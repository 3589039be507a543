"""Canned estimators: the Linear / DNN / DNNLinearCombined classifiers, regressors and head-taking estimators,
model_to_estimator.

The reference's examples use ``tf.estimator.LinearClassifier(feature_columns, model_dir,
n_classes[, optimizer][, config])`` (reference: tf_yarn/examples/linear_classifier_example.py:49-52,
collective_all_reduce_example.py:58-62, mlflow_example.py:61-67) and
``tf.keras.estimator.model_to_estimator`` (keras_example.py:64-65).  The wide-and-deep
estimator is the BASELINE config that exercises the parameter-server path.
"""
from __future__ import annotations

import math
from typing import Any, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.estimator.config import RunConfig
from tf_yarn_b200.estimator.estimator import Estimator
from tf_yarn_b200.estimator.head import (SUM_OVER_BATCH_SIZE, BinaryClassHead, MultiClassHead,  # noqa: F401
                                         RegressionHead, _classification_head, _classification_metrics, _Head,
                                         _regression_metrics)
from tf_yarn_b200.estimator.spec import EstimatorSpec
from tf_yarn_b200.keras import optimizers as kopt


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
    by_name = {"adagrad": kopt.Adagrad, "ftrl": kopt.Ftrl, "rmsprop": kopt.RMSprop, "adamax": kopt.Adamax,
               "nadam": kopt.Nadam}
    if tower == "dnn" and name in ("adagrad", "rmsprop", "adamax", "nadam"):
        return by_name[name](0.001 if combined else 0.05)
    if tower == "linear" and name in ("ftrl", "rmsprop", "adamax", "nadam"):
        return by_name[name](min(0.005 if combined else 0.2, per_columns))
    return opt


def _canned_model_fn(linear_columns, dnn_columns, hidden_units, optimizer, head: _Head, dropout=None,
                     linear_optimizer=None, sparse_combiner="sum"):
    """The model_fn of every canned estimator: the wide and/or deep towers under ``head``."""
    if not isinstance(head, _Head):
        raise TypeError(f"head must be one of the heads of tf_yarn_b200.estimator (BinaryClassHead, ...), got "
                        f"{head!r}")
    # one CannedHead per model_fn: its device buffers outlive any CUDA graph a train step captured with it
    loss = head.canned_head()
    n_out = head.logits_dimension
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
        return EstimatorSpec(mode=mode, network=net, loss=loss, optimizer=optimizer, eval_metric_ops=head.metrics(),
                             predictions=head.predictions, optimizers=per_tower, weights=head.weights)
    return model_fn


def _classifier_head(n_classes, weight_column) -> _Head:
    if n_classes == 2:
        return BinaryClassHead(weight_column)
    return MultiClassHead(n_classes, weight_column)


def _check_estimator_args(activation_fn=F.relu, batch_norm=False, warm_start_from=None, name="activation_fn"):
    if activation_fn not in (F.relu, torch.relu, "relu"):
        raise ValueError(f"{name} must be relu (the only activation supported), got {activation_fn!r}")
    if batch_norm:
        raise ValueError("batch_norm=True is not supported")
    if warm_start_from is not None:
        raise ValueError(f"warm_start_from is not supported (got {warm_start_from!r})")


class LinearClassifier(Estimator):
    def __init__(self, feature_columns, model_dir: Optional[str] = None, n_classes: int = 2, weight_column=None,
                 optimizer: Any = "ftrl", config: Optional[RunConfig] = None, sparse_combiner: str = "sum",
                 **_ignored):
        # FTRL is TF's default for linear models (tf.estimator.LinearClassifier)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], optimizer,
                                          _classifier_head(n_classes, weight_column),
                                          sparse_combiner=sparse_combiner), model_dir, config)


class DNNClassifier(Estimator):
    def __init__(self, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 n_classes: int = 2, weight_column=None, optimizer: Any = "adagrad", dropout: Optional[float] = None,
                 config: Optional[RunConfig] = None, **_ignored):
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), optimizer,
                                          _classifier_head(n_classes, weight_column), dropout), model_dir, config)


class DNNLinearCombinedClassifier(Estimator):
    """Wide & deep with TF's defaults: FTRL for the linear (wide) tower, Adagrad for the DNN (deep) tower."""

    def __init__(self, model_dir: Optional[str] = None, linear_feature_columns=None, linear_optimizer: Any = "ftrl",
                 dnn_feature_columns=None, dnn_optimizer: Any = "adagrad", dnn_hidden_units: Sequence[int] = (),
                 dnn_dropout: Optional[float] = None, n_classes: int = 2, weight_column=None,
                 config: Optional[RunConfig] = None, linear_sparse_combiner: str = "sum", **_ignored):
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units), dnn_optimizer,
                                          _classifier_head(n_classes, weight_column), dnn_dropout,
                                          linear_optimizer=linear_optimizer, sparse_combiner=linear_sparse_combiner),
                         model_dir, config)


class LinearRegressor(Estimator):
    """tf.estimator.LinearRegressor: squared error, ``predictions`` = the ``label_dimension`` logits."""

    def __init__(self, feature_columns, model_dir: Optional[str] = None, label_dimension: int = 1,
                 weight_column=None, optimizer: Any = "ftrl", config: Optional[RunConfig] = None,
                 sparse_combiner: str = "sum", loss_reduction: str = SUM_OVER_BATCH_SIZE):
        head = RegressionHead(label_dimension, weight_column, loss_reduction)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], optimizer, head,
                                          sparse_combiner=sparse_combiner), model_dir, config)


class DNNRegressor(Estimator):
    """tf.estimator.DNNRegressor: squared error, ``predictions`` = the ``label_dimension`` logits."""

    def __init__(self, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 label_dimension: int = 1, weight_column=None, optimizer: Any = "adagrad",
                 dropout: Optional[float] = None, config: Optional[RunConfig] = None,
                 loss_reduction: str = SUM_OVER_BATCH_SIZE):
        head = RegressionHead(label_dimension, weight_column, loss_reduction)
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), optimizer, head, dropout),
                         model_dir, config)


class DNNLinearCombinedRegressor(Estimator):
    """Wide & deep regression with TF's defaults: FTRL for the linear (wide) tower, Adagrad for the DNN (deep)
    tower."""

    def __init__(self, model_dir: Optional[str] = None, linear_feature_columns=None, linear_optimizer: Any = "ftrl",
                 dnn_feature_columns=None, dnn_optimizer: Any = "adagrad", dnn_hidden_units: Sequence[int] = (),
                 dnn_dropout: Optional[float] = None, label_dimension: int = 1, weight_column=None,
                 config: Optional[RunConfig] = None, linear_sparse_combiner: str = "sum",
                 loss_reduction: str = SUM_OVER_BATCH_SIZE):
        head = RegressionHead(label_dimension, weight_column, loss_reduction)
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units), dnn_optimizer, head, dnn_dropout,
                                          linear_optimizer=linear_optimizer, sparse_combiner=linear_sparse_combiner),
                         model_dir, config)


class LinearEstimator(Estimator):
    """tf.estimator.LinearEstimator: a linear model under any head (FTRL by default, as TF)."""

    def __init__(self, head, feature_columns, model_dir: Optional[str] = None, optimizer: Any = "ftrl",
                 config: Optional[RunConfig] = None, sparse_combiner: str = "sum", warm_start_from=None):
        _check_estimator_args(warm_start_from=warm_start_from)
        fc._check_combiner(sparse_combiner)
        super().__init__(_canned_model_fn(list(feature_columns), [], [], optimizer, head,
                                          sparse_combiner=sparse_combiner), model_dir, config)


class DNNEstimator(Estimator):
    """tf.estimator.DNNEstimator: a ReLU network under any head (Adagrad by default, as TF)."""

    def __init__(self, head, hidden_units: Sequence[int], feature_columns, model_dir: Optional[str] = None,
                 optimizer: Any = "adagrad", activation_fn=F.relu, dropout: Optional[float] = None,
                 config: Optional[RunConfig] = None, warm_start_from=None, batch_norm: bool = False):
        _check_estimator_args(activation_fn, batch_norm, warm_start_from)
        super().__init__(_canned_model_fn([], list(feature_columns), list(hidden_units), optimizer, head, dropout),
                         model_dir, config)


class DNNLinearCombinedEstimator(Estimator):
    """tf.estimator.DNNLinearCombinedEstimator: wide & deep under any head, with TF's defaults: FTRL for the linear
    (wide) tower, Adagrad for the DNN (deep) tower."""

    def __init__(self, head, model_dir: Optional[str] = None, linear_feature_columns=None,
                 linear_optimizer: Any = "ftrl", dnn_feature_columns=None, dnn_optimizer: Any = "adagrad",
                 dnn_hidden_units: Sequence[int] = (), dnn_activation_fn=F.relu, dnn_dropout: Optional[float] = None,
                 config: Optional[RunConfig] = None, batch_norm: bool = False, linear_sparse_combiner: str = "sum",
                 warm_start_from=None):
        _check_estimator_args(dnn_activation_fn, batch_norm, warm_start_from, name="dnn_activation_fn")
        fc._check_combiner(linear_sparse_combiner)
        super().__init__(_canned_model_fn(list(linear_feature_columns or []), list(dnn_feature_columns or []),
                                          list(dnn_hidden_units or ()), dnn_optimizer, head, dnn_dropout,
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
