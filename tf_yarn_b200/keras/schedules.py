"""Keras learning-rate schedules (``keras.optimizers.schedules``).

A schedule maps ``step`` -- Keras's ``optimizer.iterations``, the number of batches already trained (the number of
updates already applied unless the optimizer sets ``gradient_accumulation_steps``) -- to the learning rate of an
update made at that step.  The formulas are tf.keras 2.13+ / Keras 3's:

* ``ExponentialDecay``: ``initial_learning_rate * decay_rate ** p`` with ``p = step / decay_steps``
  (``floor``-ed when ``staircase``).
* ``PiecewiseConstantDecay``: ``values[i]`` where ``i`` is the number of boundaries ``b`` with ``step > b``
  (so ``values[0]`` up to and including ``boundaries[0]``); at most 16 boundaries.
* ``PolynomialDecay``: ``(initial_learning_rate - end_learning_rate) * (1 - t / d) ** power + end_learning_rate``
  with ``t = min(step, decay_steps)`` and ``d = decay_steps``; with ``cycle``, ``t = step`` and
  ``d = decay_steps * max(1, ceil(step / decay_steps))``.
* ``InverseTimeDecay``: ``initial_learning_rate / (1 + decay_rate * p)`` with ``p = step / decay_steps``
  (``floor``-ed when ``staircase``).
* ``CosineDecay``: without warm-up (``warmup_target is None``),
  ``initial_learning_rate * ((1 - alpha) * 0.5 * (1 + cos(pi * t / decay_steps)) + alpha)`` with
  ``t = min(step, decay_steps)``.  With warm-up, ``t = min(step, decay_steps + warmup_steps)``; while
  ``t < warmup_steps`` the rate is ``initial_learning_rate + (warmup_target - initial_learning_rate) * t /
  warmup_steps``, afterwards the decay above from ``warmup_target`` at ``t - warmup_steps``.
* ``CosineDecayRestarts``: period ``i`` lasts ``first_decay_steps * t_mul ** i`` steps; with ``f`` the fraction of
  its period that ``step`` has completed, ``initial_learning_rate * ((1 - alpha) * 0.5 * m_mul ** i *
  (1 + cos(pi * f)) + alpha)``.  ``t_mul`` must be at least 1.

Every schedule is evaluated in float64 and rounded to float32 once, as the fused optimizer step does on the GPU
(``ops/csrc/tfy_lr_schedule.cuh``): there the thread that advances the device step counter writes the rate of the
next update, so a captured CUDA graph follows the schedule with no host copy and no extra launch.
"""
from __future__ import annotations

import math
from typing import Any, Dict, Sequence

import numpy as np

MAX_BOUNDARIES = 16

# TfyLrKind (ops/csrc/tfy_lr_schedule.cuh)
_EXPONENTIAL, _PIECEWISE, _POLYNOMIAL, _INVERSE_TIME, _COSINE, _COSINE_RESTARTS = 1, 2, 3, 4, 5, 6


def _f32(x: float) -> float:
    return float(np.float32(x))


def _positive(name: str, v) -> float:
    v = float(v)
    if not v > 0 or not math.isfinite(v):
        raise ValueError(f"`{name}` must be a finite number > 0, got {v}")
    return v


def _finite(name: str, v) -> float:
    v = float(v)
    if not math.isfinite(v):
        raise ValueError(f"`{name}` must be a finite number, got {v}")
    return v


class LearningRateSchedule:
    """Base class: ``__call__(step)`` returns the learning rate of the update after ``step`` updates."""

    def __call__(self, step) -> float:
        raise NotImplementedError

    def get_config(self) -> Dict[str, Any]:
        raise NotImplementedError

    @classmethod
    def from_config(cls, config: Dict[str, Any]) -> "LearningRateSchedule":
        return cls(**config)

    def _device_fields(self) -> Dict[str, Any]:
        """The fields of the device struct TfyLrSchedule (``ops.native.LrSchedule``) that describe this schedule."""
        raise NotImplementedError(f"{type(self).__name__} has no device form: the fused optimizer step evaluates "
                                  "only the schedules of keras.optimizers.schedules")

    def __eq__(self, other) -> bool:
        return type(self) is type(other) and self.get_config() == other.get_config()

    def __repr__(self) -> str:
        args = ", ".join(f"{k}={v!r}" for k, v in self.get_config().items())
        return f"{type(self).__name__}({args})"


class ExponentialDecay(LearningRateSchedule):
    def __init__(self, initial_learning_rate, decay_steps, decay_rate, staircase=False, name=None):
        self.initial_learning_rate = _finite("initial_learning_rate", initial_learning_rate)
        self.decay_steps = _positive("decay_steps", decay_steps)
        self.decay_rate = _positive("decay_rate", decay_rate)
        self.staircase, self.name = bool(staircase), name

    def __call__(self, step) -> float:
        p = float(step) / self.decay_steps
        if self.staircase:
            p = math.floor(p)
        return _f32(self.initial_learning_rate * self.decay_rate ** p)

    def get_config(self):
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "decay_rate": self.decay_rate, "staircase": self.staircase, "name": self.name}

    def _device_fields(self):
        return {"kind": _EXPONENTIAL, "flags": int(self.staircase), "initial_lr": self.initial_learning_rate,
                "decay_steps": self.decay_steps, "decay_rate": self.decay_rate}


class PiecewiseConstantDecay(LearningRateSchedule):
    def __init__(self, boundaries: Sequence[float], values: Sequence[float], name=None):
        boundaries, values = list(boundaries), list(values)
        if len(boundaries) > MAX_BOUNDARIES:
            raise ValueError(f"`boundaries` holds at most {MAX_BOUNDARIES} entries, got {len(boundaries)}")
        if len(values) != len(boundaries) + 1:
            raise ValueError(f"`values` must have one more entry than `boundaries`: got {len(values)} values for "
                             f"{len(boundaries)} boundaries")
        self.boundaries = [_finite("boundaries", b) for b in boundaries]
        if any(a >= b for a, b in zip(self.boundaries, self.boundaries[1:])):
            raise ValueError(f"`boundaries` must be strictly increasing, got {self.boundaries}")
        self.values = [_f32(_finite("values", v)) for v in values]
        self.name = name

    def __call__(self, step) -> float:
        s = float(step)
        return self.values[sum(1 for b in self.boundaries if s > b)]

    def get_config(self):
        return {"boundaries": list(self.boundaries), "values": list(self.values), "name": self.name}

    def _device_fields(self):
        return {"kind": _PIECEWISE, "n_boundaries": len(self.boundaries), "initial_lr": self.values[0],
                "boundaries": self.boundaries, "values": self.values}


class PolynomialDecay(LearningRateSchedule):
    def __init__(self, initial_learning_rate, decay_steps, end_learning_rate=0.0001, power=1.0, cycle=False,
                 name=None):
        self.initial_learning_rate = _finite("initial_learning_rate", initial_learning_rate)
        self.decay_steps = _positive("decay_steps", decay_steps)
        self.end_learning_rate = _finite("end_learning_rate", end_learning_rate)
        self.power = _positive("power", power)
        self.cycle, self.name = bool(cycle), name

    def __call__(self, step) -> float:
        t, d = float(step), self.decay_steps
        if self.cycle:
            if t > 0:
                d *= math.ceil(t / self.decay_steps)
        else:
            t = min(t, self.decay_steps)
        lr = (self.initial_learning_rate - self.end_learning_rate) * (1.0 - t / d) ** self.power
        return _f32(lr + self.end_learning_rate)

    def get_config(self):
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "end_learning_rate": self.end_learning_rate, "power": self.power, "cycle": self.cycle,
                "name": self.name}

    def _device_fields(self):
        return {"kind": _POLYNOMIAL, "flags": int(self.cycle), "initial_lr": self.initial_learning_rate,
                "decay_steps": self.decay_steps, "end_lr": self.end_learning_rate, "power": self.power}


class InverseTimeDecay(LearningRateSchedule):
    def __init__(self, initial_learning_rate, decay_steps, decay_rate, staircase=False, name=None):
        self.initial_learning_rate = _finite("initial_learning_rate", initial_learning_rate)
        self.decay_steps = _positive("decay_steps", decay_steps)
        self.decay_rate = _finite("decay_rate", decay_rate)
        if self.decay_rate < 0:
            raise ValueError(f"`decay_rate` must be >= 0, got {self.decay_rate}")
        self.staircase, self.name = bool(staircase), name

    def __call__(self, step) -> float:
        p = float(step) / self.decay_steps
        if self.staircase:
            p = math.floor(p)
        return _f32(self.initial_learning_rate / (1.0 + self.decay_rate * p))

    def get_config(self):
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "decay_rate": self.decay_rate, "staircase": self.staircase, "name": self.name}

    def _device_fields(self):
        return {"kind": _INVERSE_TIME, "flags": int(self.staircase), "initial_lr": self.initial_learning_rate,
                "decay_steps": self.decay_steps, "decay_rate": self.decay_rate}


def _cosine(t: float, decay_steps: float, alpha: float, from_lr: float) -> float:
    decayed = 0.5 * (1.0 + math.cos(math.pi * (t / decay_steps)))
    return from_lr * ((1.0 - alpha) * decayed + alpha)


class CosineDecay(LearningRateSchedule):
    def __init__(self, initial_learning_rate, decay_steps, alpha=0.0, name=None, warmup_target=None,
                 warmup_steps=0):
        self.initial_learning_rate = _finite("initial_learning_rate", initial_learning_rate)
        self.decay_steps = _positive("decay_steps", decay_steps)
        self.alpha = _finite("alpha", alpha)
        self.warmup_target = None if warmup_target is None else _finite("warmup_target", warmup_target)
        self.warmup_steps = _finite("warmup_steps", warmup_steps)
        if self.warmup_steps < 0:
            raise ValueError(f"`warmup_steps` must be >= 0, got {self.warmup_steps}")
        self.name = name

    def __call__(self, step) -> float:
        s = float(step)
        if self.warmup_target is None:
            return _f32(_cosine(min(s, self.decay_steps), self.decay_steps, self.alpha, self.initial_learning_rate))
        t = min(s, self.decay_steps + self.warmup_steps)
        if t < self.warmup_steps:
            lr = (self.warmup_target - self.initial_learning_rate) * (t / self.warmup_steps) + \
                self.initial_learning_rate
        else:
            lr = _cosine(t - self.warmup_steps, self.decay_steps, self.alpha, self.warmup_target)
        return _f32(lr)

    def get_config(self):
        return {"initial_learning_rate": self.initial_learning_rate, "decay_steps": self.decay_steps,
                "alpha": self.alpha, "name": self.name, "warmup_target": self.warmup_target,
                "warmup_steps": self.warmup_steps}

    def _device_fields(self):
        warm = self.warmup_target is not None
        return {"kind": _COSINE, "flags": 2 if warm else 0, "initial_lr": self.initial_learning_rate,
                "decay_steps": self.decay_steps, "alpha": self.alpha,
                "warmup_target": self.warmup_target if warm else 0.0, "warmup_steps": self.warmup_steps}


class CosineDecayRestarts(LearningRateSchedule):
    def __init__(self, initial_learning_rate, first_decay_steps, t_mul=2.0, m_mul=1.0, alpha=0.0, name=None):
        self.initial_learning_rate = _finite("initial_learning_rate", initial_learning_rate)
        self.first_decay_steps = _positive("first_decay_steps", first_decay_steps)
        self.t_mul = _finite("t_mul", t_mul)
        if self.t_mul < 1.0:
            raise ValueError(f"`t_mul` must be >= 1 (restart periods that shrink end after a finite number of "
                             f"steps), got {self.t_mul}")
        self.m_mul = _finite("m_mul", m_mul)
        if self.m_mul < 0:
            raise ValueError(f"`m_mul` must be >= 0, got {self.m_mul}")
        self.alpha = _finite("alpha", alpha)
        self.name = name

    def __call__(self, step) -> float:
        # the same period search as the device (tfy_lr_schedule.cuh): a logarithm estimates the period, the
        # start of the period is then checked on both sides
        frac, t = float(step) / self.first_decay_steps, self.t_mul
        if t == 1.0:
            i = math.floor(frac)
            frac -= i
        else:
            i = float(math.floor(math.log1p(frac * (t - 1.0)) / math.log(t)))
            start = (t ** i - 1.0) / (t - 1.0)
            while i > 0.0 and frac < start:
                i -= 1.0
                start = (t ** i - 1.0) / (t - 1.0)
            while frac >= start + t ** i:
                start += t ** i
                i += 1.0
            frac = (frac - start) / t ** i
        decayed = 0.5 * self.m_mul ** i * (1.0 + math.cos(math.pi * frac))
        return _f32(self.initial_learning_rate * ((1.0 - self.alpha) * decayed + self.alpha))

    def get_config(self):
        return {"initial_learning_rate": self.initial_learning_rate, "first_decay_steps": self.first_decay_steps,
                "t_mul": self.t_mul, "m_mul": self.m_mul, "alpha": self.alpha, "name": self.name}

    def _device_fields(self):
        return {"kind": _COSINE_RESTARTS, "initial_lr": self.initial_learning_rate,
                "decay_steps": self.first_decay_steps, "t_mul": self.t_mul, "m_mul": self.m_mul, "alpha": self.alpha}


_BY_NAME = {c.__name__: c for c in (ExponentialDecay, PiecewiseConstantDecay, PolynomialDecay, InverseTimeDecay,
                                    CosineDecay, CosineDecayRestarts)}


def serialize(schedule: LearningRateSchedule) -> Dict[str, Any]:
    return {"class_name": type(schedule).__name__, "config": schedule.get_config()}


def deserialize(config: Dict[str, Any], custom_objects: Dict[str, type] = None) -> LearningRateSchedule:
    known = dict(_BY_NAME, **(custom_objects or {}))
    name = config.get("class_name")
    if name not in known:
        raise ValueError(f"unknown learning-rate schedule {name!r}")
    return known[name].from_config(dict(config.get("config", {})))


def is_schedule(x) -> bool:
    return isinstance(x, LearningRateSchedule)
