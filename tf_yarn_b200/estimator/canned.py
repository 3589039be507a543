"""Canned estimators: the Linear / DNN / DNNLinearCombined classifiers and regressors, model_to_estimator.

The reference's examples use ``tf.estimator.LinearClassifier(feature_columns, model_dir,
n_classes[, optimizer][, config])`` (reference: tf_yarn/examples/linear_classifier_example.py:49-52,
collective_all_reduce_example.py:58-62, mlflow_example.py:61-67) and
``tf.keras.estimator.model_to_estimator`` (keras_example.py:64-65).  The wide-and-deep
estimator is the BASELINE config that exercises the parameter-server path.
"""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.estimator.config import RunConfig
from tf_yarn_b200.estimator.estimator import Estimator
from tf_yarn_b200.estimator.spec import EstimatorSpec
from tf_yarn_b200.keras import metrics as kmetrics
from tf_yarn_b200.keras import optimizers as kopt
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


def _classification_head(n_classes: int) -> canned_head.CannedHead:
    if n_classes == 2:
        return canned_head.CannedHead(canned_head.BINARY, 1)
    return canned_head.CannedHead(canned_head.MULTI_CLASS, n_classes)


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


def _regression_metrics(label_dimension: int) -> Dict[str, Any]:
    """TF's regression head (tensorflow_estimator head/regression_head.py): each weighted and averaged over all d
    outputs, ``sum_i w_i sum_j v_ij / (d sum_i w_i)``."""
    d = label_dimension

    def ratio(values):
        def fn(labels, logits, w):
            v = values(labels.float().reshape(logits.shape), logits.float())
            if w is None:
                return v.sum(), float(v.numel())
            return (v.sum(dim=1) * w).sum(), d * w.sum()
        return fn
    return {"average_loss": _BatchRatio("average_loss", ratio(lambda y, z: (z - y) ** 2)),
            "label/mean": _BatchRatio("label/mean", ratio(lambda y, z: y)),
            "prediction/mean": _BatchRatio("prediction/mean", ratio(lambda y, z: z))}


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


class _WideDeepNet(nn.Module):
    """logits = linear(wide columns) + dnn(dense(deep columns))."""

    def __init__(self, linear_columns, dnn_columns, hidden_units: Sequence[int], n_out: int,
                 activation=F.relu, dropout: Optional[float] = None, sparse_combiner: str = "sum"):
        super().__init__()
        self.linear = fc.LinearModel(linear_columns, n_out, sparse_combiner) if linear_columns else None
        self.dense_features = fc.DenseFeatures(dnn_columns) if dnn_columns else None
        self.activation = activation
        self.dropout = dropout
        self.hidden = nn.ModuleList()
        if self.dense_features is not None:
            width = self.dense_features.width
            for h in hidden_units:
                self.hidden.append(nn.Linear(width, h))
                width = h
            self.logits = nn.Linear(width, n_out)
        else:
            self.logits = None

    def forward(self, features):
        out = None
        if self.linear is not None:
            out = self.linear(features)
        if self.dense_features is not None:
            x = self.dense_features(features).to(self.logits.weight.dtype)
            for layer in self.hidden:
                x = self.activation(layer(x))
                if self.dropout:
                    x = F.dropout(x, self.dropout, self.training)
            d = self.logits(x)
            out = d if out is None else out + d.to(out.dtype)
        return out


def _tf_default(opt, tower: str, n_columns: int, combined: bool):
    """An optimizer NAME gets the learning rate TF's canned estimators give it (tensorflow_estimator canned/dnn.py
    ``_LEARNING_RATE = 0.05``, linear.py ``min(0.2, 1/sqrt(n_columns))``, dnn_linear_combined.py 0.001 / ``min(0.005,
    1/sqrt(n_linear_columns))``) instead of the Keras class default (0.001); optimizer objects and callables pass
    through untouched."""
    if not isinstance(opt, str):
        return opt
    name = opt.lower()
    per_columns = 1.0 / math.sqrt(max(n_columns, 1))
    if tower == "dnn" and name in ("adagrad", "rmsprop"):
        cls = kopt.Adagrad if name == "adagrad" else kopt.RMSprop
        return cls(0.001 if combined else 0.05)
    if tower == "linear" and name in ("ftrl", "rmsprop"):
        cls = kopt.Ftrl if name == "ftrl" else kopt.RMSprop
        return cls(min(0.005 if combined else 0.2, per_columns))
    return opt


def _regression_predictions(logits):
    return {"predictions": logits.float()}


def _canned_model_fn(linear_columns, dnn_columns, hidden_units, optimizer, dropout=None, linear_optimizer=None,
                     sparse_combiner="sum", n_classes=2, label_dimension=None, weight_column=None):
    """The model_fn of every canned estimator: a classifier head for ``n_classes``, or a regression head of
    ``label_dimension`` outputs when that is given."""
    if label_dimension is not None:
        head = canned_head.CannedHead(canned_head.REGRESSION, label_dimension)
        metrics, predictions = (lambda: _regression_metrics(label_dimension)), _regression_predictions
    else:
        head = _classification_head(n_classes)
        metrics, predictions = (lambda: _classification_metrics(n_classes)), _classification_predictions(n_classes)
    weights = _weights_fn(weight_column)
    n_out = head.n_out
    combined = bool(linear_columns) and bool(dnn_columns)
    if dnn_columns:
        optimizer = _tf_default(optimizer, "dnn", len(dnn_columns), combined)
        linear_optimizer = _tf_default(linear_optimizer, "linear", len(linear_columns), combined)
    else:                                   # linear-only model: `optimizer` IS the linear optimizer
        optimizer = _tf_default(optimizer, "linear", len(linear_columns), False)

    def model_fn(features, labels, mode, params=None, config=None):
        net = _WideDeepNet(linear_columns, dnn_columns, hidden_units, n_out, dropout=dropout,
                           sparse_combiner=sparse_combiner)
        # the wide tower's parameters live under "linear."; everything else belongs to the deep tower
        per_tower = {"linear.": linear_optimizer} if (linear_optimizer is not None and linear_columns) else None
        # one head per model_fn: its device buffers outlive any CUDA graph a train step captured with it
        return EstimatorSpec(mode=mode, network=net, loss=head, optimizer=optimizer, eval_metric_ops=metrics(),
                             predictions=predictions, optimizers=per_tower, weights=weights)
    return model_fn


def _check_regression_args(label_dimension, loss_reduction) -> int:
    if isinstance(label_dimension, bool) or not isinstance(label_dimension, int) or label_dimension < 1:
        raise ValueError(f"label_dimension must be an integer >= 1, got {label_dimension!r}")
    if loss_reduction != SUM_OVER_BATCH_SIZE:
        raise ValueError(f"loss_reduction must be {SUM_OVER_BATCH_SIZE!r} (SUM_OVER_BATCH_SIZE), got "
                         f"{loss_reduction!r}")
    return label_dimension


class LinearClassifier(Estimator):
    def __init__(self, feature_columns, model_dir: Optional[str] = None, n_classes: int = 2, weight_column=None,
                 optimizer: Any = "ftrl", config: Optional[RunConfig] = None, sparse_combiner: str = "sum",
                 **_ignored):
        # FTRL is TF's default for linear models (tf.estimator.LinearClassifier)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], optimizer, sparse_combiner=sparse_combiner,
                                          n_classes=n_classes, weight_column=weight_column), model_dir, config)


class DNNClassifier(Estimator):
    def __init__(self, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 n_classes: int = 2, weight_column=None, optimizer: Any = "adagrad", dropout: Optional[float] = None,
                 config: Optional[RunConfig] = None, **_ignored):
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), optimizer, dropout,
                                          n_classes=n_classes, weight_column=weight_column), model_dir, config)


class DNNLinearCombinedClassifier(Estimator):
    """Wide & deep with TF's defaults: FTRL for the linear (wide) tower, Adagrad for the DNN (deep) tower."""

    def __init__(self, model_dir: Optional[str] = None, linear_feature_columns=None, linear_optimizer: Any = "ftrl",
                 dnn_feature_columns=None, dnn_optimizer: Any = "adagrad", dnn_hidden_units: Sequence[int] = (),
                 dnn_dropout: Optional[float] = None, n_classes: int = 2, weight_column=None,
                 config: Optional[RunConfig] = None, linear_sparse_combiner: str = "sum", **_ignored):
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units), dnn_optimizer, dnn_dropout,
                                          linear_optimizer=linear_optimizer, sparse_combiner=linear_sparse_combiner,
                                          n_classes=n_classes, weight_column=weight_column),
                         model_dir, config)


class LinearRegressor(Estimator):
    """tf.estimator.LinearRegressor: squared error, ``predictions`` = the ``label_dimension`` logits."""

    def __init__(self, feature_columns, model_dir: Optional[str] = None, label_dimension: int = 1,
                 weight_column=None, optimizer: Any = "ftrl", config: Optional[RunConfig] = None,
                 sparse_combiner: str = "sum", loss_reduction: str = SUM_OVER_BATCH_SIZE):
        d = _check_regression_args(label_dimension, loss_reduction)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], optimizer, sparse_combiner=sparse_combiner,
                                          label_dimension=d, weight_column=weight_column), model_dir, config)


class DNNRegressor(Estimator):
    """tf.estimator.DNNRegressor: squared error, ``predictions`` = the ``label_dimension`` logits."""

    def __init__(self, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 label_dimension: int = 1, weight_column=None, optimizer: Any = "adagrad",
                 dropout: Optional[float] = None, config: Optional[RunConfig] = None,
                 loss_reduction: str = SUM_OVER_BATCH_SIZE):
        d = _check_regression_args(label_dimension, loss_reduction)
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), optimizer, dropout,
                                          label_dimension=d, weight_column=weight_column), model_dir, config)


class DNNLinearCombinedRegressor(Estimator):
    """Wide & deep regression with TF's defaults: FTRL for the linear (wide) tower, Adagrad for the DNN (deep)
    tower."""

    def __init__(self, model_dir: Optional[str] = None, linear_feature_columns=None, linear_optimizer: Any = "ftrl",
                 dnn_feature_columns=None, dnn_optimizer: Any = "adagrad", dnn_hidden_units: Sequence[int] = (),
                 dnn_dropout: Optional[float] = None, label_dimension: int = 1, weight_column=None,
                 config: Optional[RunConfig] = None, linear_sparse_combiner: str = "sum",
                 loss_reduction: str = SUM_OVER_BATCH_SIZE):
        d = _check_regression_args(label_dimension, loss_reduction)
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units), dnn_optimizer, dnn_dropout,
                                          linear_optimizer=linear_optimizer, sparse_combiner=linear_sparse_combiner,
                                          label_dimension=d, weight_column=weight_column),
                         model_dir, config)


def model_to_estimator(keras_model, model_dir: Optional[str] = None, config: Optional[RunConfig] = None,
                       **_ignored) -> Estimator:
    """Estimator around a compiled mini-Keras model (loss / optimizer / metrics taken from compile())."""
    from tf_yarn_b200.keras import losses as klosses
    from tf_yarn_b200.keras import metrics as kmetrics
    if keras_model.optimizer is None or keras_model.loss is None:
        raise ValueError("compile() the Keras model before converting it to an estimator")
    keras_model.build()
    loss_fn = klosses.get(keras_model.loss)
    out_dim = keras_model.layers[-1].output_shape_[-1]
    metric_fns = dict(kmetrics.resolve(m, klosses.name_of(keras_model.loss), out_dim)
                      for m in keras_model._metrics_spec)

    def pick_features(features):
        # Keras models take a single tensor; dict inputs are concatenated in key order
        if isinstance(features, dict):
            vals = [features[k].reshape(features[k].shape[0], -1).float() for k in sorted(features)]
            return vals[0] if len(vals) == 1 else torch.cat(vals, dim=1)
        return features

    class _Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.inner = keras_model.net

        def forward(self, features):
            x = pick_features(features)
            p = next(self.inner.parameters(), None)
            if p is not None and torch.is_floating_point(x):
                x = x.to(p.dtype)
            return self.inner(x)

    def model_fn(features, labels, mode, params=None, config=None):
        return EstimatorSpec(mode=mode, network=_Net(), loss=lambda y, out: loss_fn(y, out),
                             optimizer=keras_model.optimizer, eval_metric_ops=metric_fns)
    return Estimator(model_fn, model_dir, config)
