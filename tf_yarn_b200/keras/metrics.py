"""Streaming metrics: ``update(y_true, y_pred, sample_weight=None) -> (numerator, denominator)``.

The numerator is a device tensor; the denominator (an element count) is a Python float so that
no host->device copy happens inside a CUDA-graph capture.  With ``sample_weight`` (Keras
``weighted_metrics``) the pair is ``(sum w*m, sum w)``, both device tensors, where ``m`` is the
metric of one sample (the mean over its non-batch elements)."""
from __future__ import annotations

from typing import Callable, Tuple, Union

import torch


def _weighted(m: torch.Tensor, sample_weight) -> Tuple[torch.Tensor, torch.Tensor]:
    w = sample_weight.reshape(-1).float()
    m = m.float().reshape(w.shape[0], -1).mean(dim=1)
    return (m * w).sum(), w.sum()


def sparse_categorical_accuracy(y_true, y_pred, sample_weight=None) -> Tuple[torch.Tensor, torch.Tensor]:
    pred = y_pred.reshape(-1, y_pred.shape[-1]).argmax(dim=-1)
    y_true = y_true.long().reshape(-1)
    if sample_weight is not None:
        return _weighted(pred == y_true, sample_weight)
    return (pred == y_true).sum().float(), float(y_true.numel())


def categorical_accuracy(y_true, y_pred, sample_weight=None):
    return sparse_categorical_accuracy(y_true.argmax(dim=-1), y_pred, sample_weight)


def binary_accuracy(y_true, y_pred, sample_weight=None):
    pred = (y_pred.float().reshape(-1) > 0.5)
    y_true = y_true.reshape(-1) > 0.5
    if sample_weight is not None:
        return _weighted(pred == y_true, sample_weight)
    return (pred == y_true).sum().float(), float(y_true.numel())


def mean_absolute_error(y_true, y_pred, sample_weight=None):
    d = (y_pred.float() - y_true.float().reshape(y_pred.shape)).abs()
    if sample_weight is not None:
        return _weighted(d, sample_weight)
    return d.sum(), float(d.numel())


def resolve(identifier: Union[str, Callable], loss_name: str, output_dim: int) -> Tuple[str, Callable]:
    """Keras resolves the string 'accuracy' from the loss / output shape."""
    if callable(identifier):
        return getattr(identifier, "__name__", "metric"), identifier
    if identifier in ("accuracy", "acc"):
        if loss_name == "sparse_categorical_crossentropy":
            return "accuracy", sparse_categorical_accuracy
        if loss_name == "categorical_crossentropy":
            return "accuracy", categorical_accuracy
        if loss_name == "binary_crossentropy" or output_dim == 1:
            return "accuracy", binary_accuracy
        return "accuracy", sparse_categorical_accuracy
    table = {"sparse_categorical_accuracy": sparse_categorical_accuracy,
             "categorical_accuracy": categorical_accuracy, "binary_accuracy": binary_accuracy,
             "mae": mean_absolute_error, "mean_absolute_error": mean_absolute_error}
    if identifier not in table:
        raise ValueError(f"unknown metric {identifier!r}")
    return identifier, table[identifier]
