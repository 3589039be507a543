"""Loss functions (mean over the batch), computed in fp32.

Every built-in loss also has a per-sample form (``per_sample``): one value per sample, shape ``[B]``, the mean over
the non-batch dimensions.  Keras ``sample_weight`` / ``class_weight`` training reduces it as ``sum(w * l) / B``."""
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


def categorical_crossentropy(y_true, y_pred, from_logits: bool = False):
    y_pred = y_pred.float()
    logp = F.log_softmax(y_pred, dim=-1) if from_logits else torch.log(y_pred.clamp_min(1e-7))
    return -(y_true.float() * logp).sum(dim=-1).mean()


def binary_crossentropy(y_true, y_pred, from_logits: bool = False):
    y_pred = y_pred.float().reshape(-1)
    y_true = y_true.float().reshape(-1)
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


def categorical_crossentropy_per_sample(y_true, y_pred, from_logits: bool = False):
    y_pred = y_pred.float()
    logp = F.log_softmax(y_pred, dim=-1) if from_logits else torch.log(y_pred.clamp_min(1e-7))
    return _per_row(-(y_true.float() * logp).sum(dim=-1), y_pred.shape[0])


def binary_crossentropy_per_sample(y_true, y_pred, from_logits: bool = False):
    batch = y_pred.shape[0]
    y_pred = y_pred.float().reshape(-1)
    y_true = y_true.float().reshape(-1)
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
    def __init__(self, from_logits: bool = False):
        self.from_logits = from_logits
        self.__name__ = "categorical_crossentropy"

    def __call__(self, y_true, y_pred):
        return categorical_crossentropy(y_true, y_pred, self.from_logits)


class BinaryCrossentropy:
    def __init__(self, from_logits: bool = False):
        self.from_logits = from_logits
        self.__name__ = "binary_crossentropy"

    def __call__(self, y_true, y_pred):
        return binary_crossentropy(y_true, y_pred, self.from_logits)


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
        return lambda y_true, y_pred: base(y_true, y_pred, from_logits)
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
        return {"name": identifier.__name__, "from_logits": identifier.from_logits}
    return None


def deserialize(cfg):
    if not cfg:
        return None
    if "from_logits" in cfg:
        cls = {"sparse_categorical_crossentropy": SparseCategoricalCrossentropy,
               "categorical_crossentropy": CategoricalCrossentropy,
               "binary_crossentropy": BinaryCrossentropy}[cfg["name"]]
        return cls(from_logits=cfg["from_logits"])
    return cfg["name"]
