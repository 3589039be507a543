"""Streaming metrics: ``update(y_true, y_pred, sample_weight=None) -> (numerator, denominator)``.

The numerator is a device tensor; the denominator (an element count) is a Python float so that
no host->device copy happens inside a CUDA-graph capture.  With ``sample_weight`` (Keras
``weighted_metrics``) the pair is ``(sum w*m, sum w)``, both device tensors, where ``m`` is the
metric of one sample (the mean over its non-batch elements).

``AUC``, ``Precision`` and ``Recall`` do not decompose that way: they are stateful :class:`Metric` objects that
accumulate a thresholded confusion histogram across batches (:mod:`tf_yarn_b200.ops.confusion`)."""
from __future__ import annotations

import logging
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from tf_yarn_b200.ops import confusion

logger = logging.getLogger(__name__)


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


class Metric:
    """A stateful streaming metric, as ``tf.keras.metrics.Metric``: ``update_state`` per batch, ``result`` at the end.

    The state lives on the device of the first update and is updated without a host sync, so the update can run
    inside a captured train step; ``result`` reads it back once."""

    def __init__(self, name: Optional[str] = None, dtype=None):
        self.name = name

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        raise NotImplementedError

    def result(self):
        raise NotImplementedError

    def reset_state(self) -> None:
        raise NotImplementedError

    def state_tensors(self) -> List[torch.Tensor]:
        """The device tensors holding the state (snapshot / restore around a train engine's warm-up steps)."""
        return []

    def get_config(self) -> Dict[str, Any]:
        return {"name": self.name}

    @classmethod
    def from_config(cls, config: Dict[str, Any]) -> "Metric":
        return cls(**config)

    def fresh(self) -> "Metric":
        """A new metric of the same configuration with its own, empty state."""
        return type(self).from_config(self.get_config())


_UNSUPPORTED = ("multi_label", "num_labels", "label_weights", "top_k", "class_id")


def _reject_unsupported(kwargs: Dict[str, Any]) -> None:
    for key in _UNSUPPORTED:
        if key in kwargs and kwargs[key] not in (None, False):
            raise ValueError(f"{key}={kwargs[key]!r} is not supported")
    unknown = sorted(set(kwargs) - set(_UNSUPPORTED) - {"dtype"})
    if unknown:
        raise TypeError(f"unexpected arguments {unknown}")


class _ConfusionMetric(Metric):
    """A metric computed from the thresholded confusion histogram of :mod:`tf_yarn_b200.ops.confusion`."""

    def __init__(self, num_thresholds: int, thresholds: Optional[Sequence[float]], from_logits: bool, name: str):
        super().__init__(name)
        if thresholds is not None:
            for t in thresholds:
                if not t == t:
                    raise ValueError("thresholds must not be NaN")
        self._state = confusion.ConfusionState(num_thresholds, thresholds, from_logits)

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        with torch.no_grad():
            self._state.update(y_true, y_pred, sample_weight)

    def reset_state(self) -> None:
        self._state.reset()

    def state_tensors(self) -> List[torch.Tensor]:
        return self._state.state_tensors()

    def _confusion(self):
        return confusion.confusion(self._state.histogram(), self._state.T)


class AUC(_ConfusionMetric):
    """Area under the ROC or precision-recall curve, as ``tf.keras.metrics.AUC`` (single label).

    ``thresholds`` (values in [0, 1]) replace the ``num_thresholds`` evenly spaced ones; ``-1e-7`` and ``1+1e-7`` are
    added at the ends, as Keras does, and the list is sorted."""

    def __init__(self, num_thresholds: int = 200, curve: str = "ROC", summation_method: str = "interpolation",
                 name: Optional[str] = None, dtype=None, thresholds: Optional[Sequence[float]] = None,
                 multi_label: bool = False, num_labels=None, label_weights=None, from_logits: bool = False, **kwargs):
        _reject_unsupported(dict(kwargs, multi_label=multi_label, num_labels=num_labels, label_weights=label_weights))
        curve = str(curve).upper()
        if curve not in ("ROC", "PR"):
            raise ValueError(f"curve must be 'ROC' or 'PR', got {curve!r}")
        summation_method = str(summation_method).lower()
        if summation_method not in ("interpolation", "minoring", "majoring"):
            raise ValueError(f"summation_method must be 'interpolation', 'minoring' or 'majoring', "
                             f"got {summation_method!r}")
        self.curve, self.summation_method = curve, summation_method
        self._user_thresholds = None if thresholds is None else [float(t) for t in thresholds]
        self._user_num_thresholds = int(num_thresholds)
        if thresholds is not None:
            full = [-confusion.EPSILON] + sorted(self._user_thresholds) + [1.0 + confusion.EPSILON]
            super().__init__(len(full), full, from_logits, name or "auc")
        else:
            if num_thresholds <= 1:
                raise ValueError("num_thresholds must be > 1")
            super().__init__(int(num_thresholds), None, from_logits, name or "auc")

    def result(self) -> float:
        tp, fp, fn, tn = self._confusion()
        return confusion.auc(tp, fp, fn, tn, self.curve, self.summation_method)

    def get_config(self) -> Dict[str, Any]:
        return {"num_thresholds": self._user_num_thresholds, "curve": self.curve,
                "summation_method": self.summation_method, "name": self.name, "thresholds": self._user_thresholds,
                "from_logits": self._state.from_logits}


class _PrecisionRecall(_ConfusionMetric):
    def __init__(self, thresholds, name: str, top_k=None, class_id=None, from_logits: bool = False, **kwargs):
        _reject_unsupported(dict(kwargs, top_k=top_k, class_id=class_id))
        self._scalar = thresholds is None or np.ndim(thresholds) == 0          # numbers, NumPy scalars, 0-d arrays
        vals = [0.5] if thresholds is None else ([float(thresholds)] if self._scalar else
                                                 [float(t) for t in thresholds])
        if not vals:
            raise ValueError("thresholds must not be empty")
        self._user_thresholds = None if thresholds is None else (vals[0] if self._scalar else vals)
        # one value per threshold in the order given: position of each in the sorted list the histogram uses
        self._order = np.argsort(np.asarray(vals, dtype=np.float32), kind="stable")
        self._rank = np.empty_like(self._order)
        self._rank[self._order] = np.arange(len(vals))
        super().__init__(max(len(vals), 2), vals if len(vals) >= 2 else vals * 2, from_logits, name)

    def _value(self, tp, fp, fn):
        raise NotImplementedError

    def result(self):
        tp, fp, fn, _ = self._confusion()
        v = self._value(tp, fp, fn)[self._rank]
        return float(v[0]) if self._scalar else [float(x) for x in v]

    def get_config(self) -> Dict[str, Any]:
        cfg = {"thresholds": self._user_thresholds, "name": self.name}
        if self._state.from_logits:
            cfg["from_logits"] = True
        return cfg


class Precision(_PrecisionRecall):
    """``tp / (tp + fp)`` at ``thresholds`` (default 0.5; a list gives one value per threshold), as Keras.
    ``from_logits=True`` (not in Keras) applies the sigmoid first, for heads that output logits."""

    def __init__(self, thresholds=None, top_k=None, class_id=None, name: Optional[str] = None, dtype=None,
                 from_logits: bool = False, **kwargs):
        super().__init__(thresholds, name or "precision", top_k=top_k, class_id=class_id, from_logits=from_logits,
                         **kwargs)

    def _value(self, tp, fp, fn):
        return confusion._div(tp, tp + fp)


class Recall(_PrecisionRecall):
    """``tp / (tp + fn)`` at ``thresholds`` (default 0.5; a list gives one value per threshold), as Keras."""

    def __init__(self, thresholds=None, top_k=None, class_id=None, name: Optional[str] = None, dtype=None,
                 from_logits: bool = False, **kwargs):
        super().__init__(thresholds, name or "recall", top_k=top_k, class_id=class_id, from_logits=from_logits,
                         **kwargs)

    def _value(self, tp, fp, fn):
        return confusion._div(tp, tp + fn)


METRIC_CLASSES = {"AUC": AUC, "Precision": Precision, "Recall": Recall}


def serialize(identifier) -> Any:
    """A metric spec as ``Model.save`` stores it: strings as they are, the built-in metric classes (``AUC``,
    ``Precision``, ``Recall``) by class name and config, anything else as None (not saved: ``load_model`` could not
    rebuild it)."""
    if isinstance(identifier, str):
        return identifier
    if isinstance(identifier, Metric) and METRIC_CLASSES.get(type(identifier).__name__) is type(identifier):
        return {"class_name": type(identifier).__name__, "config": identifier.get_config()}
    return None


def deserialize(spec) -> Any:
    """Inverse of :func:`serialize`; a class this version does not know is skipped (None) with a warning."""
    if isinstance(spec, dict) and "class_name" in spec:
        cls = METRIC_CLASSES.get(spec["class_name"])
        if cls is None:
            logger.warning("saved metric %r is not a known metric class: left out", spec["class_name"])
            return None
        return cls.from_config(spec["config"])
    return spec


def resolve(identifier: Union[str, Callable], loss_name: str, output_dim: int) -> Tuple[str, Callable]:
    """Keras resolves the string 'accuracy' from the loss / output shape.  A ``Metric`` object or class name
    (``"AUC"``, ``"Precision"``, ``"Recall"``) resolves to a NEW metric with its own state."""
    if isinstance(identifier, Metric):
        m = identifier.fresh()
        return m.name, m
    if isinstance(identifier, str) and identifier in METRIC_CLASSES:
        m = METRIC_CLASSES[identifier]()
        return m.name, m
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
