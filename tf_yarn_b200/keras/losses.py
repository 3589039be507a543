"""Loss functions (mean over the batch), computed in fp32.

Every built-in loss also has a per-sample form (``per_sample``): one value per sample, shape ``[B]``, the mean over
the non-batch dimensions.  Keras ``sample_weight`` / ``class_weight`` training reduces it as ``sum(w * l) / B``.

The categorical and binary cross-entropies take Keras' ``label_smoothing`` ``ls`` in [0, 1]: the targets become
``y (1 - ls) + ls / C`` (C classes) and ``y (1 - ls) + ls / 2`` respectively.  With ``ls = 0`` the targets are used
as they are."""
from __future__ import annotations

from typing import Callable, Union

import torch
import torch.nn.functional as F


def sparse_categorical_crossentropy(y_true, y_pred, from_logits: bool = False):
    y_pred = y_pred.float()
    y_true = y_true.long().reshape(-1)
    y_pred = y_pred.reshape(-1, y_pred.shape[-1])
    if from_logits:
        return F.cross_entropy(y_pred, y_true)
    return F.nll_loss(torch.log(y_pred.clamp_min(1e-7)), y_true)


def _smoothing(label_smoothing) -> float:
    ls = float(label_smoothing)
    if not 0.0 <= ls <= 1.0:
        raise ValueError(f"label_smoothing must be in [0, 1], got {label_smoothing!r}")
    return ls


def _categorical_targets(y_true, y_pred, label_smoothing):
    y = y_true.float()
    ls = _smoothing(label_smoothing)
    return y * (1.0 - ls) + ls / y_pred.shape[-1] if ls else y


def _binary_targets(y_true, label_smoothing):
    y = y_true.float().reshape(-1)
    ls = _smoothing(label_smoothing)
    return y * (1.0 - ls) + 0.5 * ls if ls else y


def categorical_crossentropy(y_true, y_pred, from_logits: bool = False, label_smoothing: float = 0.0):
    y_pred = y_pred.float()
    y_true = _categorical_targets(y_true, y_pred, label_smoothing)
    logp = F.log_softmax(y_pred, dim=-1) if from_logits else torch.log(y_pred.clamp_min(1e-7))
    return -(y_true * logp).sum(dim=-1).mean()


def binary_crossentropy(y_true, y_pred, from_logits: bool = False, label_smoothing: float = 0.0):
    y_pred = y_pred.float().reshape(-1)
    y_true = _binary_targets(y_true, label_smoothing)
    if from_logits:
        return F.binary_cross_entropy_with_logits(y_pred, y_true)
    return F.binary_cross_entropy(y_pred.clamp(1e-7, 1 - 1e-7), y_true)


def mean_squared_error(y_true, y_pred):
    return F.mse_loss(y_pred.float(), y_true.float().reshape(y_pred.shape))


def mean_absolute_error(y_true, y_pred):
    return F.l1_loss(y_pred.float(), y_true.float().reshape(y_pred.shape))


def _per_row(t: torch.Tensor, batch: int) -> torch.Tensor:
    return t.reshape(batch, -1).mean(dim=1)


def sparse_categorical_crossentropy_per_sample(y_true, y_pred, from_logits: bool = False):
    batch = y_pred.shape[0]
    y_pred = y_pred.float()
    y_true = y_true.long().reshape(-1)
    y_pred = y_pred.reshape(-1, y_pred.shape[-1])
    if from_logits:
        return _per_row(F.cross_entropy(y_pred, y_true, reduction="none"), batch)
    return _per_row(F.nll_loss(torch.log(y_pred.clamp_min(1e-7)), y_true, reduction="none"), batch)


def categorical_crossentropy_per_sample(y_true, y_pred, from_logits: bool = False, label_smoothing: float = 0.0):
    y_pred = y_pred.float()
    y_true = _categorical_targets(y_true, y_pred, label_smoothing)
    logp = F.log_softmax(y_pred, dim=-1) if from_logits else torch.log(y_pred.clamp_min(1e-7))
    return _per_row(-(y_true * logp).sum(dim=-1), y_pred.shape[0])


def binary_crossentropy_per_sample(y_true, y_pred, from_logits: bool = False, label_smoothing: float = 0.0):
    batch = y_pred.shape[0]
    y_pred = y_pred.float().reshape(-1)
    y_true = _binary_targets(y_true, label_smoothing)
    if from_logits:
        return _per_row(F.binary_cross_entropy_with_logits(y_pred, y_true, reduction="none"), batch)
    return _per_row(F.binary_cross_entropy(y_pred.clamp(1e-7, 1 - 1e-7), y_true, reduction="none"), batch)


def mean_squared_error_per_sample(y_true, y_pred):
    y_pred = y_pred.float()
    return _per_row((y_pred - y_true.float().reshape(y_pred.shape)) ** 2, y_pred.shape[0])


def mean_absolute_error_per_sample(y_true, y_pred):
    y_pred = y_pred.float()
    return _per_row((y_pred - y_true.float().reshape(y_pred.shape)).abs(), y_pred.shape[0])


class SparseCategoricalCrossentropy:
    def __init__(self, from_logits: bool = False):
        self.from_logits = from_logits
        self.__name__ = "sparse_categorical_crossentropy"

    def __call__(self, y_true, y_pred):
        return sparse_categorical_crossentropy(y_true, y_pred, self.from_logits)


class CategoricalCrossentropy:
    """Keras ``CategoricalCrossentropy``: one-hot or soft targets ``[B, C]``, classes on the last axis only."""

    def __init__(self, from_logits: bool = False, label_smoothing: float = 0.0, axis: int = -1):
        if axis != -1:
            raise ValueError(f"CategoricalCrossentropy supports axis=-1 only, got axis={axis!r}")
        self.from_logits = from_logits
        self.label_smoothing = _smoothing(label_smoothing)
        self.__name__ = "categorical_crossentropy"

    def __call__(self, y_true, y_pred):
        return categorical_crossentropy(y_true, y_pred, self.from_logits, self.label_smoothing)


class BinaryCrossentropy:
    def __init__(self, from_logits: bool = False, label_smoothing: float = 0.0):
        self.from_logits = from_logits
        self.label_smoothing = _smoothing(label_smoothing)
        self.__name__ = "binary_crossentropy"

    def __call__(self, y_true, y_pred):
        return binary_crossentropy(y_true, y_pred, self.from_logits, self.label_smoothing)


_BY_NAME = {
    "sparse_categorical_crossentropy": sparse_categorical_crossentropy,
    "categorical_crossentropy": categorical_crossentropy,
    "binary_crossentropy": binary_crossentropy,
    "mse": mean_squared_error, "mean_squared_error": mean_squared_error,
    "mae": mean_absolute_error, "mean_absolute_error": mean_absolute_error,
}


_PER_SAMPLE = {
    sparse_categorical_crossentropy: sparse_categorical_crossentropy_per_sample,
    categorical_crossentropy: categorical_crossentropy_per_sample,
    binary_crossentropy: binary_crossentropy_per_sample,
    mean_squared_error: mean_squared_error_per_sample,
    mean_absolute_error: mean_absolute_error_per_sample,
}


def per_sample(identifier: Union[str, Callable]) -> Callable:
    """Per-sample form ``(y_true, y_pred) -> [B]`` of a loss.  A custom callable is used as it is and must itself
    return one loss per sample: a scalar raises ``ValueError`` (it cannot be weighted)."""
    fn = get(identifier)
    if isinstance(fn, (SparseCategoricalCrossentropy, CategoricalCrossentropy, BinaryCrossentropy)):
        base, from_logits = _PER_SAMPLE[_BY_NAME[fn.__name__]], fn.from_logits
        if isinstance(fn, SparseCategoricalCrossentropy):
            return lambda y_true, y_pred: base(y_true, y_pred, from_logits)
        ls = fn.label_smoothing
        return lambda y_true, y_pred: base(y_true, y_pred, from_logits, ls)
    for builtin, form in _PER_SAMPLE.items():
        if fn is builtin:
            return form

    def custom(y_true, y_pred):
        out = fn(y_true, y_pred)
        if not torch.is_tensor(out) or out.dim() == 0:
            raise ValueError(f"loss {name_of(identifier)!r} returns a scalar: with sample_weight or class_weight a "
                             "custom loss must return one loss per sample (shape [batch])")
        return out.float().reshape(out.shape[0], -1).mean(dim=1)
    return custom


def get(identifier: Union[str, Callable]) -> Callable:
    if callable(identifier):
        return identifier
    if identifier not in _BY_NAME:
        raise ValueError(f"unknown loss {identifier!r}")
    return _BY_NAME[identifier]


def name_of(identifier) -> str:
    return identifier if isinstance(identifier, str) else getattr(identifier, "__name__", "loss")


def serialize(identifier):
    """JSON-able description of a loss (None when it is an arbitrary callable)."""
    if identifier is None:
        return None
    if isinstance(identifier, str):
        return {"name": identifier}
    if isinstance(identifier, (SparseCategoricalCrossentropy, CategoricalCrossentropy, BinaryCrossentropy)):
        cfg = {"name": identifier.__name__, "from_logits": identifier.from_logits}
        if getattr(identifier, "label_smoothing", 0.0):      # (absent at 0: configs written without it stay as they are)
            cfg["label_smoothing"] = identifier.label_smoothing
        return cfg
    return None


def deserialize(cfg):
    if not cfg:
        return None
    if "from_logits" in cfg:
        cls = {"sparse_categorical_crossentropy": SparseCategoricalCrossentropy,
               "categorical_crossentropy": CategoricalCrossentropy,
               "binary_crossentropy": BinaryCrossentropy}[cfg["name"]]
        if "label_smoothing" in cfg:
            return cls(from_logits=cfg["from_logits"], label_smoothing=cfg["label_smoothing"])
        return cls(from_logits=cfg["from_logits"])
    return cfg["name"]
