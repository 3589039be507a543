"""Estimator heads (``tf.estimator.BinaryClassHead``, ``MultiClassHead``, ``RegressionHead``, ``MultiLabelHead``,
``PoissonRegressionHead``, ``LogisticRegressionHead``): the loss, eval metrics and predictions a canned estimator puts
on top of its logits.

A head is passed to ``LinearEstimator``, ``DNNEstimator`` or ``DNNLinearCombinedEstimator``; the classifiers and
regressors build the equivalent head from ``n_classes`` / ``label_dimension``.  Each head gives:

* ``logits_dimension``, the number of logits per example;
* ``canned_head()``, a fresh :class:`~tf_yarn_b200.ops.head.CannedHead` (the loss; on a CUDA device one launch of the
  ``tfy_canned_head`` kernel).  A model_fn keeps the one it made for its lifetime: a CUDA graph captured with it keeps
  using its device buffers;
* ``metrics()``, fresh device-side ``Metric`` objects keyed by TF's eval-metric names (no host read per batch);
* ``predictions(logits)``, the dict ``predict()`` yields;
* ``weights``, ``features -> [B]`` weights of ``weight_column``, or ``None``.

The loss is TF2's ``SUM_OVER_BATCH_SIZE`` (the only ``loss_reduction`` accepted) and its contract is in
:mod:`tf_yarn_b200.ops.head`.  ``label_vocabulary``, ``loss_fn``, ``inverse_link_fn`` and ``name`` are not supported:
any value but ``None`` raises ``ValueError``.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, Optional, Sequence

import torch
import torch.nn.functional as F

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.keras import metrics as kmetrics
from tf_yarn_b200.ops import head as canned_head

SUM_OVER_BATCH_SIZE = "sum_over_batch_size"      # tf.keras.losses.Reduction.SUM_OVER_BATCH_SIZE, TF2's default


def _weights_fn(weight_column) -> Optional[Callable]:
    """``features -> [B] float32`` weights of ``weight_column`` (a feature key or a ``NumericColumn``), or ``None``.

    Weights are used as given (no sign check), as TF does."""
    if weight_column is None:
        return None
    key = weight_column.key if isinstance(weight_column, fc.NumericColumn) else weight_column
    if not isinstance(key, str):
        raise TypeError(f"weight_column must be a feature key or a numeric_column, got {weight_column!r}")

    def weights(features):
        if key not in features:
            raise KeyError(f"weight_column {key!r} is not among the features {sorted(features)}")
        w = features[key]
        w = w if torch.is_tensor(w) else torch.as_tensor(w)
        if not (w.dim() == 1 or (w.dim() == 2 and w.shape[1] == 1)):
            raise ValueError(f"weight_column {key!r} must have shape [B] or [B, 1], got {list(w.shape)}")
        return w.reshape(-1).float()
    return weights


class _BatchRatio(kmetrics.Metric):
    """``sum of the per-batch numerators / sum of the per-batch denominators``, 0 when the denominators sum to 0.

    ``fn(labels, logits, weights) -> (numerator, denominator)`` gives one batch's fp32 sums (``weights`` is ``None``
    without a weight column).  They are added as fp64 on the device, in batch order, with no host read per batch."""

    def __init__(self, name: str, fn: Callable):
        super().__init__(name)
        self._fn = fn
        self._sum: Optional[torch.Tensor] = None         # float64 [2]: numerator, denominator

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        num, den = self._fn(y_true, y_pred, sample_weight)
        if self._sum is None:
            self._sum = torch.zeros(2, dtype=torch.float64, device=y_pred.device)
        self._sum[0] += num
        self._sum[1] += den

    def result(self) -> float:
        if self._sum is None:
            return 0.0
        s, n = self._sum.tolist()
        return s / n if n != 0 else 0.0

    def reset_state(self) -> None:
        if self._sum is not None:
            self._sum.zero_()

    def fresh(self) -> "_BatchRatio":
        return _BatchRatio(self.name, self._fn)


class _AccuracyBaseline(kmetrics.Metric):
    """``max(m, 1 - m)`` for the (weighted) label mean ``m``: the accuracy of always predicting the majority class."""

    def __init__(self, name: str = "accuracy_baseline"):
        super().__init__(name)
        self._sum: Optional[torch.Tensor] = None         # float64 [2]: sum of the (weighted) labels, of the weights

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        y = y_true.detach().reshape(-1).double()
        if self._sum is None:
            self._sum = torch.zeros(2, dtype=torch.float64, device=y.device)
        if sample_weight is None:
            self._sum[0] += y.sum()
            self._sum[1] += y.numel()
        else:
            w = sample_weight.detach().reshape(-1).double()
            self._sum[0] += (y * w).sum()
            self._sum[1] += w.sum()

    def result(self) -> float:
        if self._sum is None:
            return 0.0
        s, n = self._sum.tolist()
        m = s / n if n else 0.0
        return max(m, 1.0 - m)

    def reset_state(self) -> None:
        if self._sum is not None:
            self._sum.zero_()


class _Column(kmetrics.Metric):
    """``inner`` on column ``k`` of ``[B, C]`` labels and logits (one class of a multi-label head)."""

    def __init__(self, inner: kmetrics.Metric, k: int):
        super().__init__(inner.name)
        self._inner, self._k = inner, k

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        C = y_pred.shape[-1]
        self._inner.update_state(y_true.reshape(-1, C)[:, self._k], y_pred.reshape(-1, C)[:, self._k], sample_weight)

    def result(self):
        return self._inner.result()

    def reset_state(self) -> None:
        self._inner.reset_state()


def _classification_head(n_classes: int) -> canned_head.CannedHead:
    if n_classes == 2:
        return canned_head.CannedHead(canned_head.BINARY, 1)
    return canned_head.CannedHead(canned_head.MULTI_CLASS, n_classes)


def _mean_of(values: Callable) -> Callable:
    """``(labels, logits, w) -> (sum_i w_i sum_j v_ij, sum_i w_i C)`` for ``values(labels, logits) -> [B, C]``: the
    weighted mean over every element (unweighted, the plain mean)."""
    def fn(labels, logits, w):
        v = values(labels, logits)
        if w is None:
            return v.sum(), float(v.numel())
        return (v.sum(dim=1) * w).sum(), v.shape[1] * w.sum()
    return fn


def _threshold_metrics(thresholds: Sequence[float]) -> Dict[str, Any]:
    """TF's ``accuracy/``, ``precision/`` and ``recall/positive_threshold_%g`` of a sigmoid head, over every
    (example, logit) pair."""
    ops: Dict[str, Any] = {}
    for t in thresholds:
        def hit(labels, logits, t=t):
            z = logits.float().reshape(logits.shape[0], -1)
            return ((torch.sigmoid(z) > t).float() == labels.float().reshape(z.shape)).float()
        ops[f"accuracy/positive_threshold_{t:g}"] = _BatchRatio(f"accuracy/positive_threshold_{t:g}", _mean_of(hit))
        ops[f"precision/positive_threshold_{t:g}"] = kmetrics.Precision(
            thresholds=t, from_logits=True, name=f"precision/positive_threshold_{t:g}")
        ops[f"recall/positive_threshold_{t:g}"] = kmetrics.Recall(
            thresholds=t, from_logits=True, name=f"recall/positive_threshold_{t:g}")
    return ops


def _classification_metrics(n_classes: int) -> Dict[str, Any]:
    head = canned_head.BINARY if n_classes == 2 else canned_head.MULTI_CLASS

    def class_ids(labels):
        # a label outside [0, n_classes) is reported by the head (CannedHead.check); clamping keeps the metrics from
        # indexing with it, and changes nothing for valid labels
        y = labels.long().reshape(-1)
        return y if n_classes == 2 else y.clamp(0, n_classes - 1)

    def accuracy(labels, logits, w):
        if n_classes == 2:
            pred = (logits.reshape(-1) > 0).long()
        else:
            pred = logits.argmax(dim=-1)
        labels = labels.long().reshape(-1)
        if w is None:
            return (pred == labels).sum().float(), float(labels.numel())
        return (w * (pred == labels).float()).sum(), w.sum()

    def average_loss(labels, logits, w):
        if w is None:
            n = labels.reshape(-1).shape[0]
            return canned_head.torch_head(head, logits, class_ids(labels), None) * n, float(n)
        return (canned_head.torch_row_losses(head, logits, class_ids(labels)) * w).sum(), w.sum()
    ops: Dict[str, Any] = {"accuracy": _BatchRatio("accuracy", accuracy),
                           "average_loss": _BatchRatio("average_loss", average_loss)}
    if n_classes == 2:
        # the rest of TF's binary head: tensorflow_estimator head/binary_class_head.py
        def label_mean(labels, logits, w):
            y = labels.float().reshape(-1)
            return (y.sum(), float(y.numel())) if w is None else ((y * w).sum(), w.sum())

        def prediction_mean(labels, logits, w):
            p = torch.sigmoid(logits.float().reshape(-1))
            return (p.sum(), float(p.numel())) if w is None else ((p * w).sum(), w.sum())

        ops.update({"auc": kmetrics.AUC(from_logits=True, name="auc"),
                    "auc_precision_recall": kmetrics.AUC(curve="PR", from_logits=True, name="auc_precision_recall"),
                    "precision": kmetrics.Precision(from_logits=True), "recall": kmetrics.Recall(from_logits=True),
                    "label/mean": _BatchRatio("label/mean", label_mean),
                    "prediction/mean": _BatchRatio("prediction/mean", prediction_mean),
                    "accuracy_baseline": _AccuracyBaseline()})
    return ops


def _regression_metrics(label_dimension: int, head: int = canned_head.REGRESSION,
                        inverse_link: Optional[Callable] = None) -> Dict[str, Any]:
    """TF's regression head (tensorflow_estimator head/regression_head.py): each weighted and averaged over all d
    outputs, ``sum_i w_i sum_j v_ij / (d sum_i w_i)``.  ``average_loss`` is the head's element loss (squared error,
    Poisson or logistic) and ``prediction/mean`` is over ``inverse_link(logits)`` when a link is given."""
    def ratio(values):
        return _mean_of(lambda labels, logits: values(labels.float().reshape(logits.shape), logits.float()))
    if head == canned_head.REGRESSION:
        loss = ratio(lambda y, z: (z - y) ** 2)
    else:
        loss = _mean_of(lambda labels, logits: canned_head.torch_element_losses(head, logits, labels))
    link = inverse_link or (lambda z: z)
    return {"average_loss": _BatchRatio("average_loss", loss),
            "label/mean": _BatchRatio("label/mean", ratio(lambda y, z: y)),
            "prediction/mean": _BatchRatio("prediction/mean", ratio(lambda y, z: link(z)))}


def _multi_label_metrics(n_classes: int, thresholds: Sequence[float], classes: Sequence[int]) -> Dict[str, Any]:
    """TF's multi-label head (tensorflow_estimator head/multi_label_head.py): ``average_loss``
    ``sum_i w_i (sum_j l_ij / C) / sum_i w_i``, AUCs over every (example, class) pair with the example's weight, the
    threshold metrics over pairs, and per listed class its probability mean and AUCs."""
    C = n_classes

    def losses(labels, logits):
        return canned_head.torch_element_losses(canned_head.MULTI_LABEL, logits, labels)
    ops: Dict[str, Any] = {
        "average_loss": _BatchRatio("average_loss", _mean_of(losses)),
        "auc": kmetrics.AUC(from_logits=True, name="auc"),
        "auc_precision_recall": kmetrics.AUC(curve="PR", from_logits=True, name="auc_precision_recall")}
    ops.update(_threshold_metrics(thresholds))
    for k in classes:
        def prob(labels, logits, k=k):
            return torch.sigmoid(logits.float().reshape(-1, C)[:, k:k + 1])
        ops[f"probability_mean/class{k}"] = _BatchRatio(f"probability_mean/class{k}", _mean_of(prob))
        ops[f"auc/class{k}"] = _Column(kmetrics.AUC(from_logits=True, name=f"auc/class{k}"), k)
        ops[f"auc_precision_recall/class{k}"] = _Column(
            kmetrics.AUC(curve="PR", from_logits=True, name=f"auc_precision_recall/class{k}"), k)
    return ops


def _classification_predictions(n_classes: int) -> Callable:
    def predictions(logits):
        logits = logits.float()
        if n_classes == 2:
            p1 = torch.sigmoid(logits.reshape(-1, 1))
            probs = torch.cat([1 - p1, p1], dim=1)
            ids = (p1 > 0.5).long()
        else:
            probs = F.softmax(logits, dim=-1)
            ids = probs.argmax(dim=-1, keepdim=True)
        return {"logits": logits, "probabilities": probs, "class_ids": ids}
    return predictions


def _regression_predictions(logits):
    return {"predictions": logits.float()}


# --------------------------------------------------------------------------------------------------- argument checks
def _check_unsupported(**args) -> None:
    for name, value in args.items():
        if value is not None:
            raise ValueError(f"{name} is not supported (got {value!r}); leave it None")


def _check_reduction(loss_reduction) -> None:
    if loss_reduction != SUM_OVER_BATCH_SIZE:
        raise ValueError(f"loss_reduction must be {SUM_OVER_BATCH_SIZE!r} (SUM_OVER_BATCH_SIZE), got "
                         f"{loss_reduction!r}")


def _check_count(name: str, value, least: int) -> int:
    if isinstance(value, bool) or not isinstance(value, int) or value < least:
        raise ValueError(f"{name} must be an integer >= {least}, got {value!r}")
    return value


def _check_thresholds(thresholds) -> tuple:
    ts = tuple(float(t) for t in (thresholds or ()))
    for t in ts:
        if not 0.0 < t < 1.0:
            raise ValueError(f"thresholds must be in (0, 1), got {t!r}")
    return ts


# ------------------------------------------------------------------------------------------------------------ heads
class _Head:
    """What every head shares; a subclass sets ``_code`` (its :mod:`tf_yarn_b200.ops.head` code) and
    ``logits_dimension``."""

    _code: int
    logits_dimension: int

    def __init__(self, weight_column, loss_reduction, **unsupported):
        _check_reduction(loss_reduction)
        _check_unsupported(**unsupported)
        self.weight_column = weight_column
        self.weights = _weights_fn(weight_column)

    def canned_head(self) -> canned_head.CannedHead:
        return canned_head.CannedHead(self._code, self.logits_dimension)

    def metrics(self) -> Dict[str, Any]:
        raise NotImplementedError

    def predictions(self, logits: torch.Tensor) -> Dict[str, torch.Tensor]:
        raise NotImplementedError


class BinaryClassHead(_Head):
    """Sigmoid cross entropy on one logit; labels 0 or 1 (soft labels in [0, 1] are used as given)."""

    def __init__(self, weight_column=None, thresholds=None, label_vocabulary=None,
                 loss_reduction: str = SUM_OVER_BATCH_SIZE, loss_fn=None, name=None):
        super().__init__(weight_column, loss_reduction, label_vocabulary=label_vocabulary, loss_fn=loss_fn, name=name)
        self.thresholds = _check_thresholds(thresholds)
        self._code, self.logits_dimension = canned_head.BINARY, 1

    def metrics(self):
        ops = _classification_metrics(2)
        ops.update(_threshold_metrics(self.thresholds))
        return ops

    def predictions(self, logits):
        return _classification_predictions(2)(logits)


class MultiClassHead(_Head):
    """Softmax cross entropy over ``n_classes`` logits; labels are class ids in ``[0, n_classes)``."""

    def __init__(self, n_classes: int, weight_column=None, label_vocabulary=None,
                 loss_reduction: str = SUM_OVER_BATCH_SIZE, loss_fn=None, name=None):
        super().__init__(weight_column, loss_reduction, label_vocabulary=label_vocabulary, loss_fn=loss_fn, name=name)
        self.n_classes = _check_count("n_classes", n_classes, 3)       # two classes: BinaryClassHead, as in TF
        self._code, self.logits_dimension = canned_head.MULTI_CLASS, self.n_classes

    def metrics(self):
        return _classification_metrics(self.n_classes)

    def predictions(self, logits):
        return _classification_predictions(self.n_classes)(logits)


class RegressionHead(_Head):
    """Squared error on ``label_dimension`` outputs; ``predictions`` are the logits."""

    def __init__(self, label_dimension: int = 1, weight_column=None, loss_reduction: str = SUM_OVER_BATCH_SIZE,
                 loss_fn=None, inverse_link_fn=None, name=None):
        super().__init__(weight_column, loss_reduction, loss_fn=loss_fn, inverse_link_fn=inverse_link_fn, name=name)
        self.logits_dimension = _check_count("label_dimension", label_dimension, 1)
        self._code = canned_head.REGRESSION

    def metrics(self):
        return _regression_metrics(self.logits_dimension)

    def predictions(self, logits):
        return _regression_predictions(logits)


class MultiLabelHead(_Head):
    """Sigmoid cross entropy on each of ``n_classes`` logits: ``[B, n_classes]`` labels, each 0 or 1 (soft labels
    are used as given).  ``thresholds`` add accuracy, precision and recall at each; ``classes_for_class_based_metrics``
    (class ids) add per-class probability means and AUCs."""

    def __init__(self, n_classes: int, weight_column=None, thresholds=None, label_vocabulary=None,
                 loss_reduction: str = SUM_OVER_BATCH_SIZE, loss_fn=None, classes_for_class_based_metrics=None,
                 name=None):
        super().__init__(weight_column, loss_reduction, label_vocabulary=label_vocabulary, loss_fn=loss_fn, name=name)
        self.n_classes = _check_count("n_classes", n_classes, 2)
        self.thresholds = _check_thresholds(thresholds)
        classes = []
        for k in classes_for_class_based_metrics or ():
            if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k < self.n_classes:
                raise ValueError(f"classes_for_class_based_metrics must be class ids in [0, {self.n_classes}), "
                                 f"got {k!r}")
            classes.append(k)
        self.classes_for_class_based_metrics = tuple(classes)
        self._code, self.logits_dimension = canned_head.MULTI_LABEL, self.n_classes

    def metrics(self):
        return _multi_label_metrics(self.n_classes, self.thresholds, self.classes_for_class_based_metrics)

    def predictions(self, logits):
        logits = logits.float()
        return {"logits": logits, "probabilities": torch.sigmoid(logits)}


class PoissonRegressionHead(_Head):
    """Poisson regression on ``label_dimension`` log-rate logits: loss ``exp(z) - y z`` (plus Stirling's term for
    ``y > 1`` with ``compute_full_loss``), labels counts ``>= 0``, ``predictions = exp(logits)``."""

    def __init__(self, label_dimension: int = 1, weight_column=None, loss_reduction: str = SUM_OVER_BATCH_SIZE,
                 compute_full_loss: bool = True, name=None):
        super().__init__(weight_column, loss_reduction, name=name)
        self.logits_dimension = _check_count("label_dimension", label_dimension, 1)
        self.compute_full_loss = bool(compute_full_loss)
        self._code = canned_head.POISSON_FULL if self.compute_full_loss else canned_head.POISSON

    def metrics(self):
        return _regression_metrics(self.logits_dimension, self._code, torch.exp)

    def predictions(self, logits):
        logits = logits.float()
        return {"predictions": torch.exp(logits), "logits": logits}


class LogisticRegressionHead(_Head):
    """A rate in ``[0, 1]`` predicted as a probability: sigmoid cross entropy on one logit,
    ``predictions = sigmoid(logits)``."""

    def __init__(self, weight_column=None, loss_reduction: str = SUM_OVER_BATCH_SIZE, name=None):
        super().__init__(weight_column, loss_reduction, name=name)
        self._code, self.logits_dimension = canned_head.LOGISTIC, 1

    def metrics(self):
        return _regression_metrics(1, self._code, torch.sigmoid)

    def predictions(self, logits):
        logits = logits.float()
        return {"predictions": torch.sigmoid(logits), "logits": logits}
