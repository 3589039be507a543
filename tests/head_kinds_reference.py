"""The multi-label, Poisson and logistic heads (tf_yarn_b200/ops/head.py codes 3-6, estimator/head.py) in NumPy float64:
loss, logit gradient, eval metrics and fp32 error bounds.

Every logit is one element: with B rows of C logits, L = sum_i w_i sum_j l_ij / (B C) and
dL/dz_ij = w_i dl_ij/dz_ij / (B C).
    multi-label (3), logistic (6)  l = max(z, 0) - z y + log1p(exp(-|z|))     dl/dz = sigmoid(z) - y
    Poisson (4)                    l = exp(z) - y z                           dl/dz = exp(z) - y
    Poisson, full loss (5)         (4) + y log y - y + log(2 pi y) / 2 if y > 1
A Poisson label < 0 or a logistic label outside [0, 1] (NaN included) is invalid: its element adds 0 to the loss and
to the gradient and still counts in B C.
"""
import numpy as np

import confusion_reference as cref

MULTI_LABEL, POISSON, POISSON_FULL, LOGISTIC = 3, 4, 5, 6
EPS32 = float(np.finfo(np.float32).eps)


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def _zy(z, y):
    z = _f64(z)
    z = z.reshape(z.shape[0], -1)
    return z, _f64(y).reshape(z.shape)


def valid(head, y):
    """Which labels the head accepts, elementwise."""
    y = _f64(y)
    with np.errstate(invalid="ignore"):
        if head == LOGISTIC:
            return (y >= 0) & (y <= 1)
        if head in (POISSON, POISSON_FULL):
            return y >= 0
    return np.ones(y.shape, dtype=bool)


def stirling(y):
    """y log y - y + log(2 pi y) / 2 where y > 1, else 0."""
    y = _f64(y)
    big = y > 1
    ys = np.where(big, y, 2.0)
    return np.where(big, ys * np.log(ys) - ys + 0.5 * np.log(2 * np.pi * ys), 0.0)


def element_losses(head, z, y):
    """l_ij, [B, C] (0 for an invalid label)."""
    z, y = _zy(z, y)
    ok = valid(head, y)
    ys = np.where(ok, y, 0.0)
    with np.errstate(over="ignore"):
        if head in (MULTI_LABEL, LOGISTIC):
            v = np.maximum(z, 0) - z * ys + np.log1p(np.exp(-np.abs(z)))
        else:
            v = np.exp(z) - ys * z
            if head == POISSON_FULL:
                v = v + stirling(ys)
    return np.where(ok, v, 0.0)


def element_grads(head, z, y):
    """dl_ij/dz_ij, [B, C] (0 for an invalid label)."""
    z, y = _zy(z, y)
    ok = valid(head, y)
    ys = np.where(ok, y, 0.0)
    with np.errstate(over="ignore"):
        g = 1.0 / (1.0 + np.exp(-z)) - ys if head in (MULTI_LABEL, LOGISTIC) else np.exp(z) - ys
    return np.where(ok, g, 0.0)


def _w(z, w):
    return np.ones(_f64(z).shape[0]) if w is None else _f64(w).reshape(-1)


def loss(head, z, y, w=None):
    v = element_losses(head, z, y)
    return float((_w(z, w) * v.sum(axis=1)).sum() / v.size)


def dlogits(head, z, y, w=None):
    g = element_grads(head, z, y)
    return _w(z, w)[:, None] * g / g.size


# ------------------------------------------------------------------------------------------------------ eval metrics
def _ratio(num, den):
    return float(num / den) if den != 0 else 0.0


def regression_metrics(head, z, y, w=None):
    """Poisson and logistic heads: average_loss, label/mean and prediction/mean (over exp / sigmoid of the logits),
    each sum_i w_i sum_j v_ij / (d sum_i w_i)."""
    z, y = _zy(z, y)
    w = _w(z, w)
    den = z.shape[1] * w.sum()
    pred = 1.0 / (1.0 + np.exp(-z)) if head == LOGISTIC else np.exp(z)
    return {"average_loss": _ratio((w * element_losses(head, z, y).sum(axis=1)).sum(), den),
            "label/mean": _ratio((w * y.sum(axis=1)).sum(), den),
            "prediction/mean": _ratio((w * pred.sum(axis=1)).sum(), den)}


def multi_label_metrics(z, y, w=None, thresholds=(), classes=()):
    """TF's multi-label eval metrics over a whole evaluation (the batches concatenated): AUCs over every (example,
    class) pair with the example's weight, threshold metrics over pairs, and per listed class."""
    z, y = _zy(z, y)
    B, C = z.shape
    w = _w(z, w)
    sw = w.sum()
    p = 1.0 / (1.0 + np.exp(-z))
    out = {"average_loss": _ratio((w * element_losses(MULTI_LABEL, z, y).sum(axis=1)).sum(), C * sw),
           "auc": cref.auc(y, z, w, from_logits=True),
           "auc_precision_recall": cref.auc(y, z, w, curve="PR", from_logits=True)}
    for t in thresholds:
        out[f"accuracy/positive_threshold_{t:g}"] = _ratio((w[:, None] * ((p > t) == y)).sum(), C * sw)
        out[f"precision/positive_threshold_{t:g}"] = float(cref.precision(y, z, w, (t,), from_logits=True)[0])
        out[f"recall/positive_threshold_{t:g}"] = float(cref.recall(y, z, w, (t,), from_logits=True)[0])
    for k in classes:
        out[f"probability_mean/class{k}"] = _ratio((w * p[:, k]).sum(), sw)
        out[f"auc/class{k}"] = cref.auc(y[:, k], z[:, k], w, from_logits=True)
        out[f"auc_precision_recall/class{k}"] = cref.auc(y[:, k], z[:, k], w, curve="PR", from_logits=True)
    return out


# ----------------------------------------------------------------------------- fp32 error bounds (derived in the tests)
def element_scale(head, z, y):
    """Per-element magnitude S_ij with |fp32 l_ij - exact| <= 8 EPS32 S_ij."""
    z, y = _zy(z, y)
    ys = np.where(valid(head, y), y, 0.0)
    if head in (MULTI_LABEL, LOGISTIC):
        return np.abs(z) * (1 + np.abs(ys)) + 1
    with np.errstate(over="ignore"):
        s = np.exp(z) + np.abs(ys * z) + 1
    if head == POISSON_FULL:
        yb = np.where(ys > 1, ys, 0.0)
        s = s + yb * np.abs(np.log(np.maximum(yb, 1.0))) + yb + np.abs(np.log(2 * np.pi * np.maximum(yb, 1.0)))
    return s


def loss_tol(head, z, y, w=None):
    z, y = _zy(z, y)
    w = np.abs(_w(z, w))
    n = z.size
    terms = (w * np.abs(element_losses(head, z, y)).sum(axis=1)).sum()
    return EPS32 * (8 * (w * element_scale(head, z, y).sum(axis=1)).sum() + (np.log2(n) + 4) * terms) / n + 1e-30


def grad_tol(head, z, y, w=None):
    z, y = _zy(z, y)
    w = np.abs(_w(z, w))[:, None]
    ys = np.abs(np.where(valid(head, y), y, 0.0))
    g = np.abs(element_grads(head, z, y))
    if head in (MULTI_LABEL, LOGISTIC):
        e = 4 * (1 + ys) + 4 * g
    else:
        with np.errstate(over="ignore"):
            e = 4 * (np.exp(z) + ys) + 4 * g
    return EPS32 * e * w / z.size + 1e-37
