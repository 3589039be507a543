"""Float64 NumPy reference of the Keras AUC / Precision / Recall metrics (tf.keras 2.x ``metrics_utils.
update_confusion_matrix_variables``, ``AUC.result`` and ``AUC.interpolate_pr_auc``), written from their definitions so
the metrics can be checked without TensorFlow.

* Default thresholds (``thresholds=None``, ``T = num_thresholds``): ``t_0 = -1e-7``, ``t_j = j/(T-1)``, ``t_{T-1} =
  1+1e-7``; a prediction ``p`` is in bucket ``b = max(ceil(p*(T-1)) - 1, 0)`` (float32) and positive at ``j`` iff
  ``j <= b``.
* Explicit thresholds: ``p`` is positive at ``j`` iff ``p > t_j`` (float32 compare).
* Every element adds ``y*w`` to the true-positive side and ``(1-y)*w`` to the false-positive side of each threshold it
  is positive at (``w`` its sample's weight), and to the false-negative / true-negative side of the others.
"""
from __future__ import annotations

import numpy as np

EPS = 1e-7


def sigmoid32(x):
    x = np.asarray(x, np.float32)
    return (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)


def _inputs(y_true, y_pred, sample_weight, from_logits):
    p = np.asarray(y_pred, np.float32).reshape(-1)
    if from_logits:
        p = sigmoid32(p)
    y = np.asarray(y_true).reshape(-1).astype(np.float32)
    if np.isnan(p).any() or (p < 0).any() or (p > 1).any():
        raise ValueError("predictions must be in [0, 1]")
    if np.isnan(y).any() or (y < 0).any() or (y > 1).any():
        raise ValueError("labels must be in [0, 1]")
    w = np.ones(p.size, np.float64)
    if sample_weight is not None:
        sw = np.asarray(sample_weight, np.float32).reshape(-1).astype(np.float64)
        w = np.repeat(sw, p.size // sw.size)
    return p, y.astype(np.float64), w


def edge_values(num_thresholds):
    """Every bucket edge j/(T-1) in float32 and its float32 neighbours two steps either side, plus 0, 1, -0 and
    subnormals: the predictions where a float32 bucket computation can go wrong."""
    edges = (np.arange(num_thresholds, dtype=np.float64) / (num_thresholds - 1)).astype(np.float32)
    vals = [edges]
    for direction in (np.float32(-1), np.float32(2)):
        e = edges.copy()
        for _ in range(2):
            e = np.nextafter(e, direction).astype(np.float32)
            vals.append(e)
    tiny = np.array([0.0, -0.0, 1.0, np.float32(1e-45), np.float32(1e-40), np.finfo(np.float32).tiny,
                     np.nextafter(np.float32(1), np.float32(0))], np.float32)
    p = np.concatenate(vals + [tiny]).astype(np.float32)
    return p[(p >= 0) & (p <= 1)]


def bucket_even(p, num_thresholds):
    """``max(ceil(p*(T-1)) - 1, 0)`` in float32."""
    p = np.asarray(p, np.float32)
    s = (p * np.float32(num_thresholds - 1)).astype(np.float32)
    return np.maximum(np.ceil(s).astype(np.int64) - 1, 0)


def positive_matrix(p, num_thresholds, thresholds=None):
    """``[N, T]`` bool: is prediction i positive at threshold j."""
    p = np.asarray(p, np.float32)
    j = np.arange(num_thresholds)
    if thresholds is None:
        return j[None, :] <= bucket_even(p, num_thresholds)[:, None]
    t = np.asarray(thresholds, np.float32)
    return p[:, None] > t[None, :]


def confusion(y_true, y_pred, sample_weight=None, num_thresholds=200, thresholds=None, from_logits=False):
    """``(tp, fp, fn, tn)`` float64 ``[T]`` by direct summation over the elements, thresholds in the order given."""
    p, y, w = _inputs(y_true, y_pred, sample_weight, from_logits)
    T = num_thresholds if thresholds is None else len(thresholds)
    pos = positive_matrix(p, T, thresholds)
    yp, yn = y * w, (1.0 - y) * w
    tp = (pos * yp[:, None]).sum(axis=0)
    fp = (pos * yn[:, None]).sum(axis=0)
    fn = (~pos * yp[:, None]).sum(axis=0)
    tn = (~pos * yn[:, None]).sum(axis=0)
    return tp, fp, fn, tn


def histogram(y_true, y_pred, sample_weight=None, num_thresholds=200, thresholds=None, from_logits=False):
    """The ``[2, T+1]`` histogram the kernel accumulates (``thresholds`` sorted ascending): bucket ``b`` = positive at
    ``j <= b``, bucket ``T`` = positive nowhere."""
    p, y, w = _inputs(y_true, y_pred, sample_weight, from_logits)
    T = num_thresholds if thresholds is None else len(thresholds)
    if thresholds is None:
        b = bucket_even(p, T)
    else:
        c = (p[:, None] > np.asarray(thresholds, np.float32)[None, :]).sum(axis=1)
        b = np.where(c == 0, T, c - 1)
    h = np.zeros((2, T + 1), np.float64)
    np.add.at(h[0], b, y * w)
    np.add.at(h[1], b, (1.0 - y) * w)
    return h


def _div(a, b):
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    out = np.zeros(a.shape)
    nz = b != 0
    out[nz] = a[nz] / b[nz]
    return out


def auc_from_confusion(tp, fp, fn, tn, curve="ROC", summation_method="interpolation"):
    T = len(tp)
    if curve == "PR" and summation_method == "interpolation":
        # Davis & Goadrich: precision interpolated linearly in the true positives between adjacent thresholds
        total = 0.0
        for j in range(T - 1):
            dtp = tp[j] - tp[j + 1]
            p0, p1 = tp[j] + fp[j], tp[j + 1] + fp[j + 1]
            dp = p0 - p1
            slope = dtp / max(dp, 0.0) if max(dp, 0.0) != 0 else 0.0
            intercept = tp[j + 1] - slope * p1
            ratio = (p0 / p1) if (p0 > 0 and p1 > 0) else 1.0
            den = max(tp[j + 1] + fn[j + 1], 0.0)
            num = slope * (dtp + intercept * np.log(ratio))
            total += num / den if den != 0 else 0.0
        return float(total)
    rec = _div(tp, tp + fn)
    if curve == "ROC":
        x, y = _div(fp, fp + tn), rec
    else:
        x, y = rec, _div(tp, tp + fp)
    total = 0.0
    for j in range(T - 1):
        h = {"interpolation": (y[j] + y[j + 1]) / 2, "minoring": min(y[j], y[j + 1]),
             "majoring": max(y[j], y[j + 1])}[summation_method]
        total += (x[j] - x[j + 1]) * h
    return float(total)


def auc(y_true, y_pred, sample_weight=None, num_thresholds=200, curve="ROC", summation_method="interpolation",
        thresholds=None, from_logits=False):
    if thresholds is not None:
        thresholds = [-EPS] + sorted(float(t) for t in thresholds) + [1.0 + EPS]
    c = confusion(y_true, y_pred, sample_weight, num_thresholds, thresholds, from_logits)
    return auc_from_confusion(*c, curve=curve, summation_method=summation_method)


def precision(y_true, y_pred, sample_weight=None, thresholds=(0.5,), from_logits=False):
    tp, fp, _, _ = confusion(y_true, y_pred, sample_weight, thresholds=list(thresholds), from_logits=from_logits)
    return _div(tp, tp + fp)


def recall(y_true, y_pred, sample_weight=None, thresholds=(0.5,), from_logits=False):
    tp, _, fn, _ = confusion(y_true, y_pred, sample_weight, thresholds=list(thresholds), from_logits=from_logits)
    return _div(tp, tp + fn)
