"""Float64 reference of one fused optimizer step (ops/csrc/tfy_fused_step.cuh), written from the torch.optim
definitions of each optimizer and from Keras' RMSprop.  Plain NumPy: nothing here imports tf_yarn_b200.

Every step function takes ``(p, g, s1, s2, s3, h, step)`` and returns the new ``(p, s1, s2, s3)``:

* ``p``, ``s1``, ``s2``, ``s3``: the fp32 master weights and the optimizer states, as float64 arrays.  A state the
  optimizer does not use is passed through unchanged.
* ``g``: the gradient as the kernel reads it, i.e. summed over the ranks.  The step uses ``g * grad_scale / world``.
* ``h``: a :class:`Hyper`, whose fields are the float32 values the device holds, widened to float64.  So the reference
  measures the arithmetic and not the rounding of, say, ``0.999`` to float32.
* ``step``: the number of completed steps; this call performs step ``step + 1``.

What the generic fields of ``TfyOptHyper`` and the three state buffers mean for each optimizer (``flags`` is bit 0):

==========  ==============  ==========  =====  ==================  ==========  =============  ==========
optimizer   p1              p2          eps    flags               s1          s2             s3
==========  ==============  ==========  =====  ==================  ==========  =============  ==========
sgd         momentum        dampening   -      nesterov            momentum    -              -
adadelta    rho             -           eps    -                   E[g^2]      E[dx^2]        -
adam        beta1           beta2       eps    decoupled (AdamW)   m           v              -
adagrad     -               -           eps    -                   sum g^2     -              -
ftrl        l1              l2          beta   -                   n           z              -
rmsprop     rho             momentum    eps    centered            E[g^2]      momentum buf   mean g
==========  ==============  ==========  =====  ==================  ==========  =============  ==========

``weight_decay`` is coupled (``g += wd * p``) for every optimizer except AdamW.  Adagrad's initial accumulator value
and FTRL's initial ``n`` are the initial contents of ``s1``; the kernel never reads them from the hyper-parameters.
"""
from __future__ import annotations

from dataclasses import dataclass, fields

import numpy as np

FIELDS = {
    "sgd": ("momentum", "dampening", None, "nesterov"),
    "adadelta": ("rho", None, "eps", None),
    "adam": ("beta1", "beta2", "eps", "decoupled weight decay"),
    "adagrad": (None, None, "eps", None),
    "ftrl": ("l1", "l2", "beta", None),
    "rmsprop": ("rho", "momentum", "eps", "centered"),
}
STATES = {
    "sgd": ("momentum buffer", None, None),
    "adadelta": ("E[g^2]", "E[dx^2]", None),
    "adam": ("m", "v", None),
    "adagrad": ("sum of g^2", None, None),
    "ftrl": ("n", "z", None),
    "rmsprop": ("E[g^2]", "momentum buffer", "mean gradient"),
}


def f32(x) -> float:
    """``x`` as the device holds it: rounded to float32, widened back to float64."""
    return float(np.float32(x))


@dataclass
class Hyper:
    lr: float
    p1: float = 0.0
    p2: float = 0.0
    eps: float = 0.0
    wd: float = 0.0
    grad_scale: float = 1.0
    flags: int = 0
    world: int = 1

    def __post_init__(self):
        for f in fields(self):
            if f.name not in ("flags", "world"):
                setattr(self, f.name, f32(getattr(self, f.name)))


def grad(g, h: Hyper):
    return np.asarray(g, np.float64) * h.grad_scale / h.world


def sgd(p, g, s1, s2, s3, h: Hyper, step: int):
    g = grad(g, h) + h.wd * p
    if h.p1 != 0.0:
        s1 = g.copy() if step == 0 else h.p1 * s1 + (1.0 - h.p2) * g
        g = g + h.p1 * s1 if h.flags & 1 else s1
    return p - h.lr * g, s1, s2, s3


def adadelta(p, g, s1, s2, s3, h: Hyper, step: int):
    g = grad(g, h) + h.wd * p
    s1 = h.p1 * s1 + (1.0 - h.p1) * g * g
    delta = np.sqrt(s2 + h.eps) / np.sqrt(s1 + h.eps) * g
    s2 = h.p1 * s2 + (1.0 - h.p1) * delta * delta
    return p - h.lr * delta, s1, s2, s3


def adam(p, g, s1, s2, s3, h: Hyper, step: int):
    t = step + 1
    g = grad(g, h)
    if h.flags & 1:
        p = p * (1.0 - h.lr * h.wd)
    else:
        g = g + h.wd * p
    s1 = h.p1 * s1 + (1.0 - h.p1) * g
    s2 = h.p2 * s2 + (1.0 - h.p2) * g * g
    denom = np.sqrt(s2) / np.sqrt(1.0 - h.p2 ** t) + h.eps
    return p - h.lr / (1.0 - h.p1 ** t) * s1 / denom, s1, s2, s3


def adagrad(p, g, s1, s2, s3, h: Hyper, step: int):
    g = grad(g, h) + h.wd * p
    s1 = s1 + g * g
    return p - h.lr * g / (np.sqrt(s1) + h.eps), s1, s2, s3


def ftrl_linear(p, g, s1, s2, h: Hyper):
    """FTRL-proximal with learning_rate_power -0.5: the new ``n``, the new ``z`` and the unclamped weight
    ``-(z - sign(z) l1) / ((beta + sqrt(n)) / lr + 2 l2)``."""
    g = grad(g, h) + h.wd * p
    n = s1 + g * g
    z = s2 + g - (np.sqrt(n) - np.sqrt(s1)) / h.lr * p
    w = -(z - np.sign(z) * h.p1) / ((h.eps + np.sqrt(n)) / h.lr + 2.0 * h.p2)
    return n, z, w


def ftrl(p, g, s1, s2, s3, h: Hyper, step: int):
    n, z, w = ftrl_linear(p, g, s1, s2, h)
    return np.where(np.abs(z) <= h.p1, 0.0, w), n, z, s3


def rmsprop(p, g, s1, s2, s3, h: Hyper, step: int):
    g = grad(g, h) + h.wd * p
    s1 = h.p1 * s1 + (1.0 - h.p1) * g * g
    denom = s1
    if h.flags & 1:
        s3 = h.p1 * s3 + (1.0 - h.p1) * g
        denom = s1 - s3 * s3
    inc = h.lr * g / np.sqrt(denom + h.eps)
    if h.p2 > 0.0:
        s2 = h.p2 * s2 + inc
        return p - s2, s1, s2, s3
    return p - inc, s1, s2, s3


# The variants the tests run: name -> (kind, Hyper fields, initial s1).  Each switches on a different branch of the
# kernel's update; the hyper-parameters are the torch / Keras defaults where those exist.
VARIANTS = {
    "sgd": ("sgd", dict(lr=0.05), 0.0),
    "sgd_momentum_dampening": ("sgd", dict(lr=0.05, p1=0.9, p2=0.3), 0.0),
    "sgd_nesterov_wd": ("sgd", dict(lr=0.05, p1=0.9, wd=0.01, flags=1), 0.0),
    "adadelta": ("adadelta", dict(lr=1.0, p1=0.95, eps=1e-7), 0.0),
    "adam": ("adam", dict(lr=1e-3, p1=0.9, p2=0.999, eps=1e-8), 0.0),
    "adam_l2": ("adam", dict(lr=1e-3, p1=0.9, p2=0.999, eps=1e-8, wd=0.01), 0.0),
    "adamw": ("adam", dict(lr=1e-3, p1=0.9, p2=0.999, eps=1e-8, wd=0.01, flags=1), 0.0),
    "adagrad": ("adagrad", dict(lr=0.05, eps=1e-10), 0.1),
    "ftrl": ("ftrl", dict(lr=0.1, p1=0.05, p2=0.001, eps=0.1), 0.1),
    "rmsprop": ("rmsprop", dict(lr=1e-3, p1=0.9, eps=1e-7, wd=0.01), 0.0),
    "rmsprop_momentum": ("rmsprop", dict(lr=1e-3, p1=0.9, p2=0.9, eps=1e-7, wd=0.01), 0.0),
    "rmsprop_centered": ("rmsprop", dict(lr=1e-3, p1=0.9, eps=1e-7, wd=0.01, flags=1), 0.0),
    "rmsprop_momentum_centered": ("rmsprop", dict(lr=1e-3, p1=0.9, p2=0.9, eps=1e-7, wd=0.01, flags=1), 0.0),
}


def n_states(kind: str, h: Hyper) -> int:
    """How many of s1 / s2 / s3 the kernel reads and writes."""
    if kind == "rmsprop":
        return 1 + (h.p2 > 0) + (h.flags & 1)
    return 2 if kind in ("adadelta", "adam", "ftrl") else 1


STEP = {"sgd": sgd, "adadelta": adadelta, "adam": adam, "adagrad": adagrad, "ftrl": ftrl, "rmsprop": rmsprop}


def step(kind: str, p, g, s1, s2, s3, h: Hyper, n: int):
    """One update of optimizer ``kind`` (``"adamw"`` is ``"adam"`` with flags bit 0)."""
    return STEP["adam" if kind == "adamw" else kind](p, g, s1, s2, s3, h, n)
