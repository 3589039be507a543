"""The canned heads' contract (tf_yarn_b200/ops/head.py) in NumPy float64: loss, logit gradient and eval metrics of the
binary, multi-class and regression heads, weighted or not.

Row i has logits z_i (C values), label y_i and weight w_i (1 without a weight column); c = 1 for the classification
heads, c = d for regression.  L = sum_i w_i sum_j l_ij / (B c) and dL/dz_ij = w_i dl_ij/dz_ij / (B c).  A multi-class
label outside [0, C) contributes nothing to either (its row still counts in B).
"""
import numpy as np

BINARY, MULTI_CLASS, REGRESSION = 0, 1, 2


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def valid_rows(head, y, C):
    """Rows whose label the head accepts (every row but the multi-class ones with a label outside [0, C))."""
    y = _f64(y)
    if head != MULTI_CLASS:
        return np.ones(y.shape[0], dtype=bool)
    y = y.reshape(-1)
    return (y > -1) & (y < C)            # a float label is truncated toward zero, as torch's .long() does


def row_losses(head, z, y):
    """sum_j l_ij of every row, [B] (0 for a rejected multi-class label)."""
    z = _f64(z)
    B = z.shape[0]
    z = z.reshape(B, -1)
    if head == BINARY:
        z, t = z[:, 0], _f64(y).reshape(-1)
        return np.maximum(z, 0) - z * t + np.log1p(np.exp(-np.abs(z)))
    if head == MULTI_CLASS:
        ok = valid_rows(head, y, z.shape[1])
        cls = np.where(ok, np.trunc(_f64(y).reshape(-1)), 0).astype(np.int64)
        m = z.max(axis=1)
        lse = m + np.log(np.exp(z - m[:, None]).sum(axis=1))
        return np.where(ok, lse - z[np.arange(B), cls], 0.0)
    return ((z - _f64(y).reshape(z.shape)) ** 2).sum(axis=1)


def element_grads(head, z, y):
    """dl_ij/dz_ij, [B, C] (zero rows for a rejected multi-class label)."""
    z = _f64(z)
    B = z.shape[0]
    z = z.reshape(B, -1)
    if head == BINARY:
        return (1.0 / (1.0 + np.exp(-z[:, 0])) - _f64(y).reshape(-1))[:, None]
    if head == MULTI_CLASS:
        ok = valid_rows(head, y, z.shape[1])
        cls = np.where(ok, np.trunc(_f64(y).reshape(-1)), 0).astype(np.int64)
        e = np.exp(z - z.max(axis=1, keepdims=True))
        g = e / e.sum(axis=1, keepdims=True)
        g[np.arange(B), cls] -= 1.0
        return np.where(ok[:, None], g, 0.0)
    return 2.0 * (z - _f64(y).reshape(z.shape))


def _per_loss(head, z):
    z = _f64(z)
    return z.shape[0] if head == MULTI_CLASS else z.size          # B c


def loss(head, z, y, w=None):
    w = np.ones(_f64(z).shape[0]) if w is None else _f64(w).reshape(-1)
    return float((w * row_losses(head, z, y)).sum() / _per_loss(head, z))


def dlogits(head, z, y, w=None):
    z = _f64(z)
    w = np.ones(z.shape[0]) if w is None else _f64(w).reshape(-1)
    return w[:, None] * element_grads(head, z, y) / _per_loss(head, z)


def _ratio(num, den):
    return float(num / den) if den != 0 else 0.0


def classifier_metrics(n_classes, z, y, w=None):
    """TF's classifier eval metrics over a whole evaluation (the batches concatenated)."""
    z = _f64(z)
    B = z.shape[0]
    w = np.ones(B) if w is None else _f64(w).reshape(-1)
    y = _f64(y).reshape(-1)
    head = BINARY if n_classes == 2 else MULTI_CLASS
    pred = (z.reshape(-1) > 0).astype(np.float64) if n_classes == 2 else z.argmax(axis=1).astype(np.float64)
    sw = w.sum()
    out = {"accuracy": _ratio((w * (pred == np.trunc(y))).sum(), sw),
           "average_loss": _ratio((w * row_losses(head, z, y)).sum(), sw)}
    if n_classes == 2:
        m = _ratio((w * y).sum(), sw)
        out.update({"label/mean": m,
                    "prediction/mean": _ratio((w / (1.0 + np.exp(-z.reshape(-1)))).sum(), sw),
                    "accuracy_baseline": max(m, 1.0 - m)})
    return out


def regressor_metrics(z, y, w=None):
    """TF's regression eval metrics: each sum_i w_i sum_j v_ij / (d sum_i w_i)."""
    z = _f64(z)
    B, d = z.shape[0], z.reshape(z.shape[0], -1).shape[1]
    z = z.reshape(B, d)
    y = _f64(y).reshape(B, d)
    w = np.ones(B) if w is None else _f64(w).reshape(-1)
    den = d * w.sum()
    return {"average_loss": _ratio((w * ((z - y) ** 2).sum(axis=1)).sum(), den),
            "label/mean": _ratio((w * y.sum(axis=1)).sum(), den),
            "prediction/mean": _ratio((w * z.sum(axis=1)).sum(), den)}


# ------------------------------------------------------------------------- fp32 error bounds (derived in the GPU test)
EPS32 = float(np.finfo(np.float32).eps)


def _element_scale(head, z, y):
    """Per-row magnitude S_i with |fp32 sum_j l_ij - exact| <= 8 EPS32 S_i."""
    z = _f64(z)
    B = z.shape[0]
    z = z.reshape(B, -1)
    if head == BINARY:
        return np.abs(z[:, 0]) * (1 + np.abs(_f64(y).reshape(-1))) + 1
    if head == MULTI_CLASS:
        C = z.shape[1]
        ok = valid_rows(head, y, C)
        cls = np.where(ok, np.trunc(_f64(y).reshape(-1)), 0).astype(np.int64)
        return np.abs(z.max(axis=1)) + np.abs(z[np.arange(B), cls]) + np.log(C) + C + 1
    return ((np.abs(z) + np.abs(_f64(y).reshape(z.shape))) ** 2).sum(axis=1) + 1


def loss_tol(head, z, y, w=None):
    z = _f64(z)
    B = z.shape[0]
    w = np.abs(np.ones(B) if w is None else _f64(w).reshape(-1))
    n = _per_loss(head, z)
    terms = w * np.abs(row_losses(head, z, y))
    return EPS32 * (8 * (w * _element_scale(head, z, y)).sum() + (np.log2(n) + 4) * terms.sum()) / n + 1e-30


def grad_tol(head, z, y, w=None):
    z = _f64(z)
    B = z.shape[0]
    z2 = z.reshape(B, -1)
    w = np.abs(np.ones(B) if w is None else _f64(w).reshape(-1))[:, None]
    g = np.abs(element_grads(head, z, y))
    if head == BINARY:
        e = 4 * (1 + np.abs(_f64(y).reshape(-1, 1))) + 4 * g
    elif head == MULTI_CLASS:
        C = z2.shape[1]
        p = np.exp(z2 - z2.max(axis=1, keepdims=True))
        p /= p.sum(axis=1, keepdims=True)
        e = (C + 8) * p + 4 * g + 2
    else:
        e = 8 * (np.abs(z2) + np.abs(_f64(y).reshape(z2.shape))) + 1
    return EPS32 * e * w / _per_loss(head, z) + 1e-37
