"""Float64 reference of the binary (Keras BinaryCrossentropy) classifier-head kernels of ops/csrc/tfy_nn.cu, with a
bound on each output's error.

The kernels: ``tfy_dense_head_fused_binary`` (logits = h W2^T + b2, loss, dW2, db2, dh = (dz W2) gate scale, db1,
stats) and ``tfy_sigmoid_xent`` (logits given: loss, dlogits, dbias, stats).  For row i, output c, with logit z,
raw target y, label smoothing ls and row weight w_i:

    t = y (1 - ls) + ls / 2      l = max(z, 0) - z t + log1p(exp(-|z|))      L_i = (1/C) sum_c l_ic
    loss = sum_i w_i L_i / B      dz = w_i (sigmoid(z) - t) / (B C)
    hit = (out > 0.5) == (y > 0.5), out = sigmoid(z) (a sigmoid layer) or z (a linear layer)

Error model (the bound tier of tests/soft_xent_reference.py, EPS32 = 2^-24, U_BF16 = 2^-8).  Each fp32 operation is
exact up to a relative EPS32; a sum of n terms in any order is within (n - 1) EPS32 sum|terms| of the exact sum; the
accurate expf / log1pf are within 2 EPS32 relative; a bf16 output adds U_BF16 |value|.  First-order terms only, then
a factor 2 of headroom:

* logits: as soft_xent_reference (e_z = (K + 1) EPS32 sum_k |h w| + |b| EPS32 fused, EPS32 |z| for the fallback).
* t = fma(y, 1 - ls, ls / 2): 3 EPS32 (|y| + ls / 2).
* sigmoid(z) = 1 / (1 + e) or e / (1 + e), e = exp(-|z|): 6 EPS32 sigmoid relative, and |sigmoid'| e_z <= e_z / 4.
* l: |dl| <= e_z (|1{z>0} - t| + 1) + |z| |dt| + 8 EPS32 (|max(z, 0)| + |z t| + log1p(e)); L and the loss sum C and B
  terms in fixed-order trees no deeper than C + B + 40: (C + B + 40) EPS32 sum |w l| / (B C) more.
* dz: (|d sigmoid| + |dt| + EPS32 (sigmoid + |t|)) w / (B C) + 4 EPS32 |dz|.
* dW2, db2, dh, db1: propagated as in soft_xent_reference.
* hits: exact, except on outputs whose model output lies within its error of 0.5 ("undecided").  The GPU tests draw
  operands on a grid of multiples of 1/8 and 1/16, whose products and K-term sums fp32 holds exactly: the kernels'
  logits are then the reference's, and so are their hits, which are checked exactly.
"""
import numpy as np

EPS32 = 2.0 ** -24
U_BF16 = 2.0 ** -8
HEADROOM = 2.0


def _f64(t):
    return t.detach().double().cpu().numpy() if hasattr(t, "detach") else np.asarray(t, dtype=np.float64)


def targets_2d(y, C):
    """Targets as [B, C] float64 ([B] is taken as [B, 1] when C = 1)."""
    y = _f64(y)
    return y.reshape(-1, C)


def weights(y, sample_w, class_w):
    """Row weights w_i = sample_w[i] * class_w[class_i]: class round(y) (half to even) for C = 1, first argmax of y
    otherwise; a class outside the table of max(C, 2) entries, or a null factor, counts as 1."""
    B, C = y.shape
    w = np.ones(B)
    if class_w is not None:
        table = _f64(class_w)
        cls = np.rint(y[:, 0]).astype(np.int64) if C == 1 else np.argmax(y, axis=1)
        inside = (cls >= 0) & (cls < len(table))
        w = w * np.where(inside, table[np.clip(cls, 0, len(table) - 1)], 1.0)
    if sample_w is not None:
        w = w * _f64(sample_w)
    return w


def sigmoid_xent(z, e_z, y, ls, w, sigmoid_out):
    """Loss, dz, hits and their bounds from float64 logits ``z`` [B, C] with per-element error bounds ``e_z``."""
    B, C = z.shape
    t = y * (1.0 - ls) + ls / 2
    dt = 3 * EPS32 * (np.abs(y) + ls / 2)
    e = np.exp(-np.abs(z))
    sg = np.where(z >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
    l = np.maximum(z, 0) - z * t + np.log1p(e)
    dl = (e_z * (np.abs((z > 0) - t) + 1) + np.abs(z) * dt
          + 8 * EPS32 * (np.maximum(z, 0) + np.abs(z * t) + np.log1p(e)))
    wl = w[:, None] * l / C
    loss = float(wl.sum() / B)
    dloss = float((np.abs(w)[:, None] * dl).sum() / (B * C) + (C + B + 40) * EPS32 * np.abs(wl).sum() / B)
    scale = (w / (B * C))[:, None]
    g = (sg - t) * scale
    dg = (6 * EPS32 * sg + e_z / 4 + dt + EPS32 * (sg + np.abs(t))) * np.abs(scale) + 4 * EPS32 * np.abs(g)
    out = sg if sigmoid_out else z
    e_out = (6 * EPS32 * sg + e_z / 4) if sigmoid_out else e_z
    undecided = np.abs(out - 0.5) <= e_out
    hit = (out > 0.5) == (y > 0.5)
    return dict(loss=loss, loss_bound=HEADROOM * dloss, dl=g, dl_bound=HEADROOM * dg,
                hits=(int((hit & ~undecided).sum()), int(undecided.sum()), hit))


def _stats(out, w, C):
    hit = out["hits"][2]
    out["w"] = w
    out["w_hits"] = float((w * hit.sum(1) / C).sum())
    return out


def fused_head(h, w2, b2, y, ls, mask, scale, sample_w, class_w, sigmoid_out):
    """Reference of tfy_dense_head_fused_binary: dict of values and bounds (numpy float64)."""
    h, w2, b2 = _f64(h), _f64(w2), _f64(b2)
    B, K = h.shape
    C = w2.shape[0]
    y = targets_2d(y, C)
    z = h @ w2.T + b2
    e_z = (K + 1) * EPS32 * (np.abs(h) @ np.abs(w2).T) + EPS32 * np.abs(b2)
    w = weights(y, sample_w, class_w)
    out = sigmoid_xent(z, e_z, y, ls, w, sigmoid_out)
    dl, ddl = out["dl"], out["dl_bound"] / HEADROOM
    gate = _f64(mask) * scale if mask is not None else np.ones((B, K))      # (the scale goes with the mask)
    n_red = B + 16
    out["dw2"] = dl.T @ h
    out["dw2_bound"] = HEADROOM * (ddl.T @ np.abs(h) + n_red * EPS32 * (np.abs(dl).T @ np.abs(h))
                                   + U_BF16 * np.abs(out["dw2"]))
    out["db2"] = dl.sum(0)
    out["db2_bound"] = HEADROOM * (ddl.sum(0) + n_red * EPS32 * np.abs(dl).sum(0) + U_BF16 * np.abs(out["db2"]))
    dh32 = (dl @ w2) * gate
    e_dh32 = ((ddl @ np.abs(w2)) + 17 * EPS32 * (np.abs(dl) @ np.abs(w2))) * np.abs(gate)
    out["dh"] = dh32
    out["dh_bound"] = HEADROOM * (e_dh32 + U_BF16 * np.abs(dh32))
    out["db1"] = dh32.sum(0)
    out["db1_bound"] = HEADROOM * (e_dh32.sum(0) + n_red * EPS32 * np.abs(dh32).sum(0) + U_BF16 * np.abs(out["db1"]))
    return _stats(out, w, C)


def sigmoid_xent_fallback(logits, bias, y, ls, sample_w, class_w, sigmoid_out):
    """Reference of tfy_sigmoid_xent (bf16 logits + bias): dict of values and bounds (numpy float64)."""
    z = _f64(logits) + (_f64(bias) if bias is not None else 0.0)
    B, C = z.shape
    y = targets_2d(y, C)
    e_z = EPS32 * np.abs(z)
    w = weights(y, sample_w, class_w)
    out = sigmoid_xent(z, e_z, y, ls, w, sigmoid_out)
    dl, ddl = out["dl"], out["dl_bound"] / HEADROOM
    out["dlogits"] = dl
    out["dlogits_bound"] = HEADROOM * (ddl + U_BF16 * np.abs(dl))
    out["dbias"] = dl.sum(0)
    out["dbias_bound"] = HEADROOM * (ddl.sum(0) + (B + 32) * EPS32 * np.abs(dl).sum(0) + U_BF16 * np.abs(out["dbias"]))
    return _stats(out, w, C)
