"""Keras-style optimizer descriptors.

A descriptor only carries hyper-parameters.  On H100 the train engine maps it to
the fused K4 kernel (``OptimizerSpec``); on CPU it is instantiated as the
equivalent ``torch.optim`` optimizer (same update formulas: tests/test_native_device_code.py checks the kernel's
update against them on the CPU, tests/fused_step_reference.py states them in float64, and
tests/test_gpu_fused_step.py holds the kernel to that reference on the GPU).
"""
from __future__ import annotations

import numbers
from typing import Iterable, Optional

import torch

from tf_yarn_b200.keras import schedules
from tf_yarn_b200.parallel.optspec import OptimizerSpec


class Optimizer:
    """``learning_rate`` is a float or a :class:`~tf_yarn_b200.keras.schedules.LearningRateSchedule`.  A schedule is
    evaluated at ``optimizer.iterations`` -- the batches already trained -- before every update: on the GPU by the
    fused step itself, which writes the next step's rate where it advances its device step counter; on the CPU by
    the engine.  As in Keras 3, the learning rate of a schedule-driven optimizer cannot be set.

    ``gradient_accumulation_steps`` (Keras 3) is ``None`` (off) or an integer ``N >= 2``.  ``iterations`` then still
    counts batches, and for batch ``s = 0, 1, ...`` with gradient ``g_s`` (the batch mean, sample and class weights
    included):

    * ``acc += g_s``, summed in fp32 in batch order;
    * if ``(s + 1) % N == 0``, the update applies ``g = acc * fl32(1/N)`` (averaged over the ranks when
      distributed) with the learning rate ``schedule(s)`` and Adam's bias correction at ``t = s + 1``, then
      ``acc = 0``;
    * the weights do not change on the other batches.  A sum not yet applied stays pending across epochs and the
      end of ``fit``, and a checkpoint carries it.
    """
    kind = "sgd"

    def __init__(self, learning_rate, gradient_accumulation_steps=None, **extra):
        self._learning_rate = learning_rate if schedules.is_schedule(learning_rate) else float(learning_rate)
        self.gradient_accumulation_steps = _check_accumulation_steps(gradient_accumulation_steps)
        self.distributed = False        # set by hvd.DistributedOptimizer
        self.extra = extra

    @property
    def learning_rate(self):
        """The float learning rate, or the schedule."""
        return self._learning_rate

    @learning_rate.setter
    def learning_rate(self, v) -> None:
        if self.schedule is not None:
            raise TypeError(f"{type(self).__name__} was created with a LearningRateSchedule as its learning_rate "
                            "argument, hence its learning rate is not settable")
        self._learning_rate = v if schedules.is_schedule(v) else float(v)

    # lr alias used by Keras 2 code
    @property
    def lr(self):
        return self.learning_rate

    @lr.setter
    def lr(self, v) -> None:
        self.learning_rate = v

    @property
    def schedule(self) -> Optional[schedules.LearningRateSchedule]:
        return self._learning_rate if schedules.is_schedule(self._learning_rate) else None

    def current_learning_rate(self, step: int = 0) -> float:
        """The learning rate of the update after ``step`` updates."""
        return float(self.schedule(step)) if self.schedule is not None else self._learning_rate

    @property
    def _lr0(self) -> float:
        """The float learning rate of the ``torch.optim`` rendition (the schedule's first; engines advance it)."""
        return self.current_learning_rate(0)

    def to_spec(self) -> OptimizerSpec:
        raise NotImplementedError

    def to_torch(self, params: Iterable[torch.nn.Parameter]) -> torch.optim.Optimizer:
        raise NotImplementedError

    def get_config(self):
        lr = schedules.serialize(self.schedule) if self.schedule is not None else self._learning_rate
        cfg = {"class_name": type(self).__name__, "learning_rate": lr, **self.extra}
        if self.gradient_accumulation_steps is not None:
            cfg["gradient_accumulation_steps"] = self.gradient_accumulation_steps
        return cfg


def _check_accumulation_steps(n):
    """``None`` or an integer ``>= 2`` (bools, floats and smaller values are refused, as by Keras 3)."""
    if n is None:
        return None
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < 2:
        raise ValueError(f"gradient_accumulation_steps must be None or an integer >= 2, got {n!r}")
    return int(n)


class SGD(Optimizer):
    def __init__(self, learning_rate: float = 0.01, momentum: float = 0.0, nesterov: bool = False,
                 weight_decay: float = 0.0, lr: float = None, gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, momentum=momentum,
                         nesterov=nesterov,
                         weight_decay=weight_decay)
        self.momentum, self.nesterov, self.weight_decay = momentum, nesterov, weight_decay

    def to_spec(self):
        return OptimizerSpec.sgd(self.learning_rate, self.momentum, 0.0, self.nesterov, self.weight_decay)

    def to_torch(self, params):
        return torch.optim.SGD(params, lr=self._lr0, momentum=self.momentum, nesterov=self.nesterov,
                               weight_decay=self.weight_decay)


class Adadelta(Optimizer):
    def __init__(self, learning_rate: float = 0.001, rho: float = 0.95, epsilon: float = 1e-7,
                 weight_decay: float = 0.0, lr: float = None, gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, rho=rho, epsilon=epsilon,
                         weight_decay=weight_decay)
        self.rho, self.epsilon, self.weight_decay = rho, epsilon, weight_decay

    def to_spec(self):
        return OptimizerSpec.adadelta(self.learning_rate, self.rho, self.epsilon, self.weight_decay)

    def to_torch(self, params):
        return torch.optim.Adadelta(params, lr=self._lr0, rho=self.rho, eps=self.epsilon,
                                    weight_decay=self.weight_decay)


class Adam(Optimizer):
    def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999,
                 epsilon: float = 1e-7, weight_decay: float = 0.0, decoupled_weight_decay: bool = False,
                 lr: float = None, gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, beta_1=beta_1,
                         beta_2=beta_2, epsilon=epsilon,
                         weight_decay=weight_decay, decoupled_weight_decay=decoupled_weight_decay)
        self.beta_1, self.beta_2, self.epsilon = beta_1, beta_2, epsilon
        self.weight_decay, self.decoupled = weight_decay, decoupled_weight_decay

    def to_spec(self):
        return OptimizerSpec.adam(self.learning_rate, self.beta_1, self.beta_2, self.epsilon, self.weight_decay,
                                  self.decoupled)

    def to_torch(self, params):
        cls = torch.optim.AdamW if self.decoupled else torch.optim.Adam
        return cls(params, lr=self._lr0, betas=(self.beta_1, self.beta_2), eps=self.epsilon,
                   weight_decay=self.weight_decay)


class AdamW(Adam):
    def __init__(self, learning_rate: float = 0.001, weight_decay: float = 0.004, **kw):
        kw.pop("decoupled_weight_decay", None)       # in get_config() of an AdamW: always True
        super().__init__(learning_rate, weight_decay=weight_decay, decoupled_weight_decay=True, **kw)


class Adagrad(Optimizer):
    def __init__(self, learning_rate: float = 0.001, initial_accumulator_value: float = 0.1,
                 epsilon: float = 1e-7, weight_decay: float = 0.0, lr: float = None,
                 gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps,
                         initial_accumulator_value=initial_accumulator_value, epsilon=epsilon,
                         weight_decay=weight_decay)
        self.initial_accumulator_value, self.epsilon, self.weight_decay = \
            initial_accumulator_value, epsilon, weight_decay

    def to_spec(self):
        return OptimizerSpec.adagrad(self.learning_rate, self.epsilon, self.weight_decay,
                                     self.initial_accumulator_value)

    def to_torch(self, params):
        return torch.optim.Adagrad(params, lr=self._lr0, eps=self.epsilon,
                                   weight_decay=self.weight_decay,
                                   initial_accumulator_value=self.initial_accumulator_value)


class Ftrl(Optimizer):
    """FTRL-proximal (``tf.keras.optimizers.Ftrl`` / ``tf.train.FtrlOptimizer``), TF's default optimizer of linear
    models and the canonical choice for the wide tower of wide-and-deep (learning_rate_power fixed at -0.5)."""
    kind = "ftrl"

    def __init__(self, learning_rate: float = 0.001, learning_rate_power: float = -0.5,
                 initial_accumulator_value: float = 0.1, l1_regularization_strength: float = 0.0,
                 l2_regularization_strength: float = 0.0, beta: float = 0.0, lr: float = None,
                 gradient_accumulation_steps: int = None):
        if learning_rate_power != -0.5:
            raise ValueError("Ftrl: only learning_rate_power=-0.5 is implemented")
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps,
                         learning_rate_power=learning_rate_power,
                         initial_accumulator_value=initial_accumulator_value,
                         l1_regularization_strength=l1_regularization_strength,
                         l2_regularization_strength=l2_regularization_strength, beta=beta)
        self.initial_accumulator_value = initial_accumulator_value
        self.l1, self.l2, self.beta = l1_regularization_strength, l2_regularization_strength, beta

    def to_spec(self):
        return OptimizerSpec.ftrl(self.learning_rate, self.l1, self.l2, self.beta, self.initial_accumulator_value)

    def to_torch(self, params):
        return TorchFtrl(params, lr=self._lr0, l1=self.l1, l2=self.l2, beta=self.beta,
                         initial_accumulator_value=self.initial_accumulator_value)


class TorchFtrl(torch.optim.Optimizer):
    """torch.optim rendition of FTRL-proximal (same formulas as the fused / parameter-server kernels)."""

    def __init__(self, params, lr=1e-3, l1=0.0, l2=0.0, beta=0.0, initial_accumulator_value=0.1):
        super().__init__(params, dict(lr=lr, l1=l1, l2=l2, beta=beta, init=initial_accumulator_value))

    @torch.no_grad()
    def step(self, closure=None):
        for grp in self.param_groups:
            lr, l1, l2, beta = grp["lr"], grp["l1"], grp["l2"], grp["beta"]
            for p in grp["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["n"] = torch.full_like(p, grp["init"])
                    st["z"] = torch.zeros_like(p)
                g, n, z = p.grad, st["n"], st["z"]
                n_new = n + g * g
                z.add_(g - (n_new.sqrt() - n.sqrt()) / lr * p)
                n.copy_(n_new)
                w = -(z - torch.sign(z) * l1) / ((beta + n_new.sqrt()) / lr + 2 * l2)
                p.copy_(torch.where(z.abs() <= l1, torch.zeros_like(w), w))


class RMSprop(Optimizer):
    """RMSprop as ``tf.keras.optimizers.RMSprop`` (Keras 2.11+ and Keras 3) defines it, per element::

        v  = rho * v + (1 - rho) * g^2
        mg = rho * mg + (1 - rho) * g               (centered only)
        inc = lr * g / sqrt(v [- mg^2] + epsilon)
        m  = momentum * m + inc;  p -= m            (momentum > 0; otherwise p -= inc)

    Unlike ``torch.optim.RMSprop``, epsilon sits inside the square root and the learning rate inside the momentum
    buffer, so a learning-rate change only scales later increments.  ``weight_decay`` is coupled, as for SGD,
    Adadelta and Adagrad here: ``g += weight_decay * p`` before the update."""
    kind = "rmsprop"

    def __init__(self, learning_rate: float = 0.001, rho: float = 0.9, momentum: float = 0.0, epsilon: float = 1e-7,
                 centered: bool = False, weight_decay: float = 0.0, lr: float = None,
                 gradient_accumulation_steps: int = None):
        if momentum < 0:
            raise ValueError(f"RMSprop momentum must be >= 0, got {momentum}")
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, rho=rho,
                         momentum=momentum, epsilon=epsilon,
                         centered=centered, weight_decay=weight_decay)
        self.rho, self.momentum, self.epsilon = rho, momentum, epsilon
        self.centered, self.weight_decay = bool(centered), weight_decay

    def to_spec(self):
        return OptimizerSpec.rmsprop(self.learning_rate, self.rho, self.momentum, self.epsilon, self.centered,
                                     self.weight_decay)

    def to_torch(self, params):
        return TorchRMSprop(params, lr=self._lr0, rho=self.rho, momentum=self.momentum, eps=self.epsilon,
                            centered=self.centered, weight_decay=self.weight_decay)


class TorchRMSprop(torch.optim.Optimizer):
    """torch.optim rendition of the Keras RMSprop (same formulas as the fused kernel; see :class:`RMSprop`)."""

    def __init__(self, params, lr=1e-3, rho=0.9, momentum=0.0, eps=1e-7, centered=False, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, rho=rho, momentum=momentum, eps=eps, centered=centered,
                                      weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        for grp in self.param_groups:
            lr, rho, mom, eps, wd = grp["lr"], grp["rho"], grp["momentum"], grp["eps"], grp["weight_decay"]
            for p in grp["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["v"] = torch.zeros_like(p)
                    if mom > 0:
                        st["m"] = torch.zeros_like(p)
                    if grp["centered"]:
                        st["mg"] = torch.zeros_like(p)
                g = p.grad + wd * p if wd else p.grad
                v = st["v"]
                v.mul_(rho).addcmul_(g, g, value=1 - rho)
                denom = v
                if grp["centered"]:
                    mg = st["mg"]
                    mg.mul_(rho).add_(g, alpha=1 - rho)
                    denom = v - mg * mg
                inc = lr * g * (denom + eps).rsqrt()
                if mom > 0:
                    m = st["m"]
                    m.mul_(mom).add_(inc)
                    p.sub_(m)
                else:
                    p.sub_(inc)


class Adamax(Optimizer):
    """Adamax as ``tf.keras.optimizers.Adamax`` defines it, per element, at update ``t = iterations + 1``::

        m = beta_1 * m + (1 - beta_1) * g
        u = max(beta_2 * u, |g|)
        p -= lr / (1 - beta_1^t) * m / (u + epsilon)

    ``torch.optim.Adamax`` puts epsilon inside the max (``max(beta_2 u, |g| + epsilon)``), so the torch rendition is
    :class:`TorchAdamax`.  ``weight_decay`` is coupled: ``g += weight_decay * p`` before the update."""
    kind = "adamax"

    def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999,
                 epsilon: float = 1e-7, weight_decay: float = 0.0, lr: float = None,
                 gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, beta_1=beta_1,
                         beta_2=beta_2, epsilon=epsilon, weight_decay=weight_decay)
        self.beta_1, self.beta_2, self.epsilon, self.weight_decay = beta_1, beta_2, epsilon, weight_decay

    def to_spec(self):
        return OptimizerSpec.adamax(self.learning_rate, self.beta_1, self.beta_2, self.epsilon, self.weight_decay)

    def to_torch(self, params):
        return TorchAdamax(params, lr=self._lr0, betas=(self.beta_1, self.beta_2), eps=self.epsilon,
                           weight_decay=self.weight_decay)


class TorchAdamax(torch.optim.Optimizer):
    """torch.optim rendition of the Keras Adamax (epsilon outside the max; see :class:`Adamax`).  Its state has the
    names of ``torch.optim.Adamax``'s: ``step``, ``exp_avg`` (m) and ``exp_inf`` (u)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-7, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        for grp in self.param_groups:
            lr, (b1, b2), eps, wd = grp["lr"], grp["betas"], grp["eps"], grp["weight_decay"]
            for p in grp["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_inf"] = torch.zeros_like(p)
                st["step"] += 1
                t = float(st["step"])
                g = p.grad + wd * p if wd else p.grad
                m, u = st["exp_avg"], st["exp_inf"]
                m.mul_(b1).add_(g, alpha=1 - b1)
                torch.maximum(u * b2, g.abs(), out=u)
                p.addcdiv_(m, u + eps, value=-lr / (1 - b1 ** t))


class Nadam(Optimizer):
    """Nadam as ``torch.optim.NAdam`` with ``momentum_decay=0.004`` (tf.keras 2's ``schedule_decay``) defines it, per
    element, at update ``t = iterations + 1``::

        mu_t = beta_1 * (1 - 0.5 * 0.96^(0.004 t));  mu_product_t = mu_product_{t-1} * mu_t
        m = beta_1 * m + (1 - beta_1) * g
        v = beta_2 * v + (1 - beta_2) * g^2
        d = sqrt(v / (1 - beta_2^t)) + epsilon
        p -= lr (1 - mu_t) / (1 - mu_product_t) * g / d + lr mu_{t+1} / (1 - mu_product_t mu_{t+1}) * m / d

    ``mu_product`` depends on the history of the step counter, so the fused step keeps it in float64 on the device and
    checkpoints carry it.  ``weight_decay`` is coupled: ``g += weight_decay * p`` before the update."""
    kind = "nadam"

    def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999,
                 epsilon: float = 1e-7, weight_decay: float = 0.0, lr: float = None,
                 gradient_accumulation_steps: int = None):
        super().__init__(lr if lr is not None else learning_rate, gradient_accumulation_steps, beta_1=beta_1,
                         beta_2=beta_2, epsilon=epsilon, weight_decay=weight_decay)
        self.beta_1, self.beta_2, self.epsilon, self.weight_decay = beta_1, beta_2, epsilon, weight_decay

    def to_spec(self):
        return OptimizerSpec.nadam(self.learning_rate, self.beta_1, self.beta_2, self.epsilon, self.weight_decay)

    def to_torch(self, params):
        return torch.optim.NAdam(params, lr=self._lr0, betas=(self.beta_1, self.beta_2), eps=self.epsilon,
                                 weight_decay=self.weight_decay, momentum_decay=0.004)


_BY_NAME = {"sgd": SGD, "adadelta": Adadelta, "adam": Adam, "adamw": AdamW, "adagrad": Adagrad, "ftrl": Ftrl,
            "rmsprop": RMSprop, "adamax": Adamax, "nadam": Nadam}


def get(identifier) -> Optimizer:
    """Resolve a string / descriptor / distributed wrapper into a descriptor."""
    if isinstance(identifier, Optimizer):
        return identifier
    if isinstance(identifier, str):
        if identifier.lower() not in _BY_NAME:
            raise ValueError(f"unknown optimizer {identifier!r}")
        return _BY_NAME[identifier.lower()]()
    inner = getattr(identifier, "_tfy_inner_optimizer", None)
    if inner is not None:
        opt = get(inner)
        opt.distributed = True
        return opt
    raise TypeError(f"cannot interpret optimizer {identifier!r}")


def from_config(cfg) -> Optimizer:
    cfg = dict(cfg)
    cls = _BY_NAME[cfg.pop("class_name").lower()]
    if isinstance(cfg.get("learning_rate"), dict):
        cfg["learning_rate"] = schedules.deserialize(cfg["learning_rate"])
    return cls(**cfg)
