"""Estimator specs (NamedTuples with ``_replace``, as the reference's hooks injection needs:
reference tf_yarn/tensorflow/metrics.py:128-137)."""
from __future__ import annotations

from typing import Any, Callable, Dict, NamedTuple, Optional, Sequence


class ModeKeys:
    TRAIN = "train"
    EVAL = "eval"
    PREDICT = "infer"


class GraphKeys:
    GLOBAL_STEP = "global_step"


class EstimatorSpec(NamedTuple):
    """What ``model_fn(features, labels, mode[, params][, config])`` returns.

    Torch-backed, define-by-run contract (there is no graph to hand over):

    network         ``torch.nn.Module`` mapping the features batch to outputs (logits / predictions).
                    ``None`` makes a parameter-free estimator (the step only advances global_step).
    loss            callable ``(labels, outputs) -> scalar tensor`` (TRAIN / EVAL); ``(labels, outputs, weights)``
                    when ``weights`` is set.
    optimizer       mini-Keras optimizer descriptor, its name, or a zero-arg factory (TRAIN).
    optimizers      optional ``{parameter-name prefix: optimizer}``: a different optimizer per part of the
                    network (longest matching prefix wins, ``optimizer`` is the default) -- TF's wide-and-deep
                    trains the linear tower with FTRL and the deep tower with Adagrad.
    eval_metric_ops ``{name: callable(labels, outputs) -> (numerator, denominator)}`` streaming metrics, or
                    ``{name: keras.metrics.Metric}`` (``reset_state`` / ``update_state(labels, outputs)`` /
                    ``result``, as TF2 Estimators take them).
    predictions     callable ``outputs -> dict`` (PREDICT), default identity.
    weights         optional callable ``features -> [B] float tensor``: per-example weights (a canned estimator's
                    ``weight_column``).  When set, the estimator calls ``loss(labels, outputs, w)``,
                    ``update_state(labels, outputs, sample_weight=w)`` on Metric ops and ``(num, den)`` ops as
                    ``fn(labels, outputs, w)``, in training and in evaluation; when ``None`` every call is made
                    without it.
    train_op / export_outputs are accepted for signature parity and ignored.
    """
    mode: str
    network: Any = None
    loss: Optional[Callable] = None
    optimizer: Any = None
    eval_metric_ops: Optional[Dict[str, Callable]] = None
    predictions: Optional[Callable] = None
    train_op: Any = None
    export_outputs: Any = None
    optimizers: Optional[Dict[str, Any]] = None
    weights: Optional[Callable] = None


class TrainSpec(NamedTuple):
    input_fn: Callable
    max_steps: Optional[int] = None
    hooks: Sequence[Any] = ()


class EvalSpec(NamedTuple):
    input_fn: Callable
    steps: Optional[int] = 100
    name: Optional[str] = None
    hooks: Sequence[Any] = ()
    exporters: Any = None
    start_delay_secs: int = 120
    throttle_secs: int = 600
