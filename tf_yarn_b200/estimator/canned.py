"""Canned estimators: LinearClassifier, DNNClassifier, DNNLinearCombinedClassifier, model_to_estimator.

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


def _classification_loss(n_classes: int) -> Callable:
    if n_classes == 2:
        def loss(labels, logits):
            return F.binary_cross_entropy_with_logits(logits.float().reshape(-1), labels.float().reshape(-1))
    else:
        def loss(labels, logits):
            return F.cross_entropy(logits.float(), labels.long().reshape(-1))
    return loss


def _classification_metrics(n_classes: int) -> Dict[str, Callable]:
    def accuracy(labels, logits):
        if n_classes == 2:
            pred = (logits.reshape(-1) > 0).long()
        else:
            pred = logits.argmax(dim=-1)
        labels = labels.long().reshape(-1)
        return (pred == labels).sum().float(), float(labels.numel())

    def average_loss(labels, logits):
        n = labels.reshape(-1).shape[0]
        return _classification_loss(n_classes)(labels, logits) * n, float(n)
    ops: Dict[str, Any] = {"accuracy": accuracy, "average_loss": average_loss}
    if n_classes == 2:
        # the rest of TF's binary head: tensorflow_estimator head/binary_class_head.py
        def label_mean(labels, logits):
            y = labels.float().reshape(-1)
            return y.sum(), float(y.numel())

        def prediction_mean(labels, logits):
            p = torch.sigmoid(logits.float().reshape(-1))
            return p.sum(), float(p.numel())

        ops.update({"auc": kmetrics.AUC(from_logits=True, name="auc"),
                    "auc_precision_recall": kmetrics.AUC(curve="PR", from_logits=True, name="auc_precision_recall"),
                    "precision": kmetrics.Precision(from_logits=True), "recall": kmetrics.Recall(from_logits=True),
                    "label/mean": label_mean, "prediction/mean": prediction_mean,
                    "accuracy_baseline": _AccuracyBaseline()})
    return ops


class _AccuracyBaseline(kmetrics.Metric):
    """``max(m, 1 - m)`` for the label mean ``m``: the accuracy of always predicting the majority class."""

    def __init__(self, name: str = "accuracy_baseline"):
        super().__init__(name)
        self._sum: Optional[torch.Tensor] = None         # float64 [2]: sum of the labels, their count

    def update_state(self, y_true, y_pred, sample_weight=None) -> None:
        y = y_true.detach().reshape(-1).double()
        if self._sum is None:
            self._sum = torch.zeros(2, dtype=torch.float64, device=y.device)
        self._sum[0] += y.sum()
        self._sum[1] += y.numel()

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


def _canned_model_fn(linear_columns, dnn_columns, hidden_units, n_classes, optimizer, dropout=None,
                     linear_optimizer=None, sparse_combiner="sum"):
    n_out = 1 if n_classes == 2 else n_classes
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
        return EstimatorSpec(mode=mode, network=net, loss=_classification_loss(n_classes), optimizer=optimizer,
                             eval_metric_ops=_classification_metrics(n_classes),
                             predictions=_classification_predictions(n_classes), optimizers=per_tower)
    return model_fn


class LinearClassifier(Estimator):
    def __init__(self, feature_columns, model_dir: Optional[str] = None, n_classes: int = 2, optimizer: Any = "ftrl",
                 config: Optional[RunConfig] = None, sparse_combiner: str = "sum", **_ignored):
        # FTRL is TF's default for linear models (tf.estimator.LinearClassifier)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], n_classes, optimizer,
                                          sparse_combiner=sparse_combiner), model_dir, config)


class DNNClassifier(Estimator):
    def __init__(self, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 n_classes: int = 2, optimizer: Any = "adagrad", dropout: Optional[float] = None,
                 config: Optional[RunConfig] = None, **_ignored):
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), n_classes, optimizer,
                                          dropout), model_dir, config)


class DNNLinearCombinedClassifier(Estimator):
    """Wide & deep with TF's defaults: FTRL for the linear (wide) tower, Adagrad for the DNN (deep) tower."""

    def __init__(self, model_dir: Optional[str] = None, linear_feature_columns=None, linear_optimizer: Any = "ftrl",
                 dnn_feature_columns=None, dnn_optimizer: Any = "adagrad", dnn_hidden_units: Sequence[int] = (),
                 dnn_dropout: Optional[float] = None, n_classes: int = 2, config: Optional[RunConfig] = None,
                 linear_sparse_combiner: str = "sum", **_ignored):
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units), n_classes, dnn_optimizer, dnn_dropout,
                                          linear_optimizer=linear_optimizer, sparse_combiner=linear_sparse_combiner),
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
