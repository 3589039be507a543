"""Float64 reference of the dense-target (Keras CategoricalCrossentropy) classifier-head kernels of ops/csrc/tfy_nn.cu,
with a bound on each output's error.

The kernels: ``tfy_dense_head_fused_soft`` (logits = h W2^T + b2, loss, dW2, db2, dh = (dl W2) gate scale, db1, stats)
and ``tfy_softmax_xent_soft`` (logits given: loss, dlogits, dbias, stats).  For row r with targets y_r, label
smoothing ls and weight w_r:

    t_c = y_c (1 - ls) + ls / C      S = sum_c t_c      p = softmax(v)      lse = logsumexp(v)
    l_r = sum_c t_c (lse - v_c)      dl_rc = (p_c S - t_c) w_r / B      loss = sum_r w_r l_r / B

Error model (the bound tier of tests/test_gpu_dense_kernels.py, with EPS32 = 2^-24 and U_BF16 = 2^-8, extended by
the terms t, S and p S add).  Each fp32 operation is exact up to a relative EPS32; a sum of n terms in any order is
within (n - 1) EPS32 sum|terms| of the exact sum; the SFU __expf / __logf are within 2^-21 relative (__expf) and
2^-21 absolute (__logf) over the ranges here; a bf16 output adds U_BF16 |value|.  First-order terms only, then a
factor 2 of headroom:

* logits (fused head, K-term fp32 dot products of bf16 operands, plus the bias): e_v = (K + 1) EPS32 sum_k |h w| + |b|
  EPS32.  The fallback kernel reads bf16 logits and adds the bias: e_v = EPS32 |v|.
* p: exp(v_c - mx) / sum: the logit errors move every difference v_c - mx by at most 2 max e_v, the SFU adds 2^-21, the
  C-term sum and the division (C + 2) EPS32: |dp_c| <= p_c d_p with d_p = 2 max_c e_v + 2^-21 + (C + 2) EPS32.
* t = fma(y, 1 - ls, ls / C): 3 EPS32 (|y| + ls / C).  S: C-term sum: |dS| <= sum |dt| + C EPS32 sum |t|.
* p S - t (one fma, or a product and a difference): |d(pS - t)| <= |p S| d_p + p |dS| + |dt| + 2 EPS32 (|p S| + |t|);
  times w / B: 2 more EPS32.
* l_r: |dl_r| <= sum_c |t_c| (e_lse + e_v,c) + |dt_c| |lse - v_c| + 2 C EPS32 sum_c |t_c (lse - v_c)|, with e_lse =
  max e_v + 2^-21 + EPS32 |lse| + C EPS32.  loss: sum over the rows (B EPS32 sum |w l|) and w l / B.
* dW2 = sum_r dl_r h_r^T, db2 = sum_r dl_r, db1 = sum_r dh_r: (B + 16) EPS32 sum |terms| (16-row CTA sums, then the
  slabs in CTA order) plus the propagated |d dl| |h|, then the bf16 rounding.
* dh = sum_c dl_c W_ck (C terms, 16 padded with zeros) times gate and scale: (16 + 1) EPS32 sum |dl W| scale plus sum_c
  |d dl_c| |W_ck| scale, then the bf16 rounding; db1 sums the fp32 dh.
* hits: exact, except on rows whose two largest logits are closer than 2 e_v (the argmax may go either way there).
"""
import numpy as np

EPS32 = 2.0 ** -24
U_BF16 = 2.0 ** -8
SFU = 2.0 ** -21
HEADROOM = 2.0


def _f64(t):
    return t.detach().double().cpu().numpy() if hasattr(t, "detach") else np.asarray(t, dtype=np.float64)


def weights(B, C, y, sample_w, class_w):
    """Row weights w_r = sample_w[r] * class_w[argmax_c y_rc] (a null factor counts as 1)."""
    w = np.ones(B)
    if class_w is not None:
        w = w * _f64(class_w)[np.argmax(y, axis=1)]
    if sample_w is not None:
        w = w * _f64(sample_w)
    return w


def soft_xent(v, e_v, y, ls, w):
    """Loss, dl and their bounds from float64 logits ``v`` [B, C] with per-element logit error bounds ``e_v``."""
    B, C = v.shape
    t = y * (1.0 - ls) + ls / C
    dt = 3 * EPS32 * (np.abs(y) + ls / C)
    S = t.sum(1, keepdims=True)
    dS = dt.sum(1, keepdims=True) + C * EPS32 * np.abs(t).sum(1, keepdims=True)
    mx = v.max(1, keepdims=True)
    e = np.exp(v - mx)
    p = e / e.sum(1, keepdims=True)
    lse = mx + np.log(e.sum(1, keepdims=True))
    ev_max = e_v.max(1, keepdims=True)
    d_p = 2 * ev_max + SFU + (C + 2) * EPS32
    g = p * S - t
    dg = np.abs(p * S) * d_p + p * dS + dt + 2 * EPS32 * (np.abs(p * S) + np.abs(t))
    wb = (w / B)[:, None]
    dl = g * wb
    ddl = (dg + 2 * EPS32 * np.abs(g)) * np.abs(wb)
    lterm = t * (lse - v)
    l = lterm.sum(1)
    e_lse = ev_max + SFU + EPS32 * np.abs(lse) + C * EPS32
    dlr = (np.abs(t) * (e_lse + e_v) + dt * np.abs(lse - v)).sum(1) + 2 * C * EPS32 * np.abs(lterm).sum(1)
    loss = float((w * l).sum() / B)
    dloss = float((np.abs(w) * dlr).sum() / B + (B + 2) * EPS32 * np.abs(w * l).sum() / B)
    return dict(loss=loss, loss_bound=HEADROOM * dloss, dl=dl, dl_bound=HEADROOM * ddl, p=p)


def hits(v, e_v, y):
    """(hits certain, rows whose logit argmax is undecided within the logit error)."""
    order = np.sort(v, axis=1)
    gap = order[:, -1] - order[:, -2] if v.shape[1] > 1 else np.full(v.shape[0], np.inf)
    undecided = gap <= 2 * e_v.max(1)
    hit = np.argmax(v, axis=1) == np.argmax(y, axis=1)
    return int((hit & ~undecided).sum()), int(undecided.sum()), hit


def fused_head(h, w2, b2, y, ls, mask, scale, sample_w, class_w):
    """Reference of tfy_dense_head_fused_soft: dict of values and bounds (numpy float64)."""
    h, w2, b2, y = _f64(h), _f64(w2), _f64(b2), _f64(y)
    B, K = h.shape
    C = w2.shape[0]
    v = h @ w2.T + b2
    e_v = (K + 1) * EPS32 * (np.abs(h) @ np.abs(w2).T) + EPS32 * np.abs(b2)
    w = weights(B, C, y, sample_w, class_w)
    out = soft_xent(v, e_v, y, ls, w)
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
    out["hits"] = hits(v, e_v, y)
    out["w"] = w
    return out


def softmax_xent(logits, bias, y, ls, sample_w, class_w):
    """Reference of tfy_softmax_xent_soft (bf16 logits + bias): dict of values and bounds (numpy float64)."""
    v = _f64(logits) + (_f64(bias) if bias is not None else 0.0)
    y = _f64(y)
    B, C = v.shape
    e_v = EPS32 * np.abs(v)
    w = weights(B, C, y, sample_w, class_w)
    out = soft_xent(v, e_v, y, ls, w)
    dl, ddl = out["dl"], out["dl_bound"] / HEADROOM
    out["dlogits"] = dl
    out["dlogits_bound"] = HEADROOM * (ddl + U_BF16 * np.abs(dl))
    out["dbias"] = dl.sum(0)
    out["dbias_bound"] = HEADROOM * (ddl.sum(0) + (B + 32) * EPS32 * np.abs(dl).sum(0) + U_BF16 * np.abs(out["dbias"]))
    out["hits"] = hits(v, e_v, y)
    out["w"] = w
    return out
