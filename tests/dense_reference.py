"""float64 reference of the Dense-layer kernels: the wgmma GEMMs (ops/csrc/tfy_gemm.cu, tfy_gemm2.cu), the split-K slab
sum, the fused split-K epilogue, the Dense backward (tfy_dense.cu), the fused classifier head (tfy_nn.cu) and the
parameter-server gather GEMM (tfy_ps_gemm.cu).

Plain NumPy.  Inputs are taken as given (bf16 tensors already rounded), every product and sum is float64, and each
function follows the contract the kernel comments state:

* GEMM: ``C = act(A B^T + bias)``; a bf16 output is the fp32 result rounded to nearest-even.
* split-K: K tile t (64 columns) belongs to slice ``t // per`` with ``per = ceil(k_tiles / split)``; the slice count
  is ``ceil(k_tiles / per)`` after clamping split to [1, k_tiles]; slab z holds the partial product over its columns,
  and the slabs are summed in slab order, left to right, in fp32.
* fused split-K epilogue: ``y = bf16(f32(relu(sum + bias)) * f32(1 / (1 - rate)))`` where element e = row * N + col
  is kept iff ``u(seed, step, e) >= rate``; the mask byte is 1 iff the ReLU passed AND the element was kept.
* Dense backward: ``dW = dh^T x``, ``dx = dh W``.
* classifier head: logits ``v = h W2^T + b2``, ``dlogits = w_r (softmax - onehot) / B``, ``dW2 = dlogits^T h``,
  ``db2 = colsum(dlogits)``, ``dh = (dlogits W2) * (mask1 & 1) * scale1`` (no gate and no scale without a mask),
  ``db1 = colsum(dh)``, loss ``sum_r w_r l_r / B``, ``stats += [hits, B(, sum w hit, sum w)]``.  Row weight
  ``w_r = sample_w[r] * class_w[label_r]``; a null table, or a label outside [0, C), counts as 1; such a label matches
  no class, so its row has no loss, no hit and no onehot term.
* gather GEMM: ``x = concat_t(table_t[ids[t]]) ++ numeric`` (ids outside [0, V) gather a zero row), ``xbuf = bf16(x)``
  with zero pad columns up to Kp, ``y = bf16(xbuf W^T + bias)``.

The exact tier (:func:`integers`, :func:`assert_exact`): operands that are small integers make every product exact in
fp32, and as long as the sum of |terms| of every output stays below 2^22 every partial sum is an integer that fp32
holds exactly, so the fp32 accumulator equals the float64 sum whatever the order of the additions.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from nn_reference import U_BF16, softmax_xent  # noqa: F401  (re-exported for the tests)
from ps_reference import EPS32, bf16_round  # noqa: F401  (re-exported for the tests)

BK = 64                 # K columns per tile of the split-K GEMM
EXACT_LIMIT = 2 ** 22   # sum of |terms| below which fp32 holds every partial sum exactly


# ---------------------------------------------------------------------------------------------- exact tier
def integers(rng: np.random.Generator, shape, lo: int = -15, hi: int = 15) -> np.ndarray:
    """Integer-valued float64 array, uniform in [lo, hi] (every value is a bf16 number)."""
    return rng.integers(lo, hi + 1, size=shape).astype(np.float64)


def assert_exact(a: np.ndarray, b: np.ndarray, bias: Optional[np.ndarray] = None) -> np.ndarray:
    """For C = a b^T (+ bias): asserts that every output's sum of |terms| is below 2^22; returns those sums."""
    mag = np.abs(a) @ np.abs(b).T + (0.0 if bias is None else np.abs(bias))
    assert mag.max(initial=0.0) < EXACT_LIMIT, f"exact-tier operands too large: sum |terms| = {mag.max()}"
    assert np.array_equal(a, np.round(a)) and np.array_equal(b, np.round(b)), "exact-tier operands must be integers"
    return mag


# ---------------------------------------------------------------------------------------------- GEMM
def gemm(a, b, bias=None, relu: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """a [M, K], b [N, K], bias [N] or None -> (act(a b^T + bias), sum of |terms| per output)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    c = a @ b.T
    mag = np.abs(a) @ np.abs(b).T
    if bias is not None:
        c = c + np.asarray(bias, np.float64)
        mag = mag + np.abs(np.asarray(bias, np.float64))
    return (np.maximum(c, 0.0) if relu else c), mag


def slab_count(K: int, split: int) -> int:
    """The number of K-slices (workspace slabs) a requested split runs (tfy_gemm_bf16_splitk_slabs)."""
    return len(k_slices(K, split))


def k_slices(K: int, split: int) -> List[Tuple[int, int]]:
    """Column ranges [k_lo, k_hi) of the K-slices: whole 64-column tiles, ``per`` tiles each, the last clipped to K."""
    k_tiles = -(-K // BK)
    split = min(max(split, 1), k_tiles)
    if split < 1:
        return [(0, K)]
    per = -(-k_tiles // split)
    return [(z * per * BK, min((z + 1) * per * BK, K)) for z in range(-(-k_tiles // per))]


def splitk_slabs(a, b, split: int) -> np.ndarray:
    """[S, M, N]: slab z = a[:, slice z] b[:, slice z]^T."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.stack([a[:, lo:hi] @ b[:, lo:hi].T for lo, hi in k_slices(a.shape[1], split)])


def sum_slabs_f32(slabs) -> np.ndarray:
    """The split-K reduction's contract: fp32 sum of the slabs in slab order, left to right."""
    s = np.asarray(slabs, np.float32)
    acc = s[0].copy()
    for z in range(1, s.shape[0]):
        acc = acc + s[z]
    return acc


def keep_scale_f32(rate: float) -> np.float32:
    """1.f / (1.f - rate) in IEEE fp32, as the fused epilogue computes it (1 when rate == 0)."""
    if rate <= 0.0:
        return np.float32(1.0)
    return np.float32(1.0) / (np.float32(1.0) - np.float32(rate))


def fused_epilogue(acc, bias, relu: bool, rate: float, u: Optional[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
    """acc [M, N] (the exact fp32 sum of the slabs), bias [N] or None -> (bf16 y as float64, mask bytes).

    Each step is one fp32 operation: v = acc + bias, ReLU, v * keep_scale, then bf16 rounding."""
    v = np.asarray(acc, np.float32)
    if bias is not None:
        v = v + np.asarray(bias, np.float32)[None, :]
    on = v > 0 if relu else np.ones(v.shape, bool)
    if relu:
        v = np.where(on, v, np.float32(0.0))
    if rate > 0:
        keep = (u[:v.size] >= rate).reshape(v.shape)
        v = np.where(keep, v * keep_scale_f32(rate), np.float32(0.0))
        on = on & keep
    return bf16_round(v), on.astype(np.uint8)


# ---------------------------------------------------------------------------------------------- Dense backward
def dense_bwd(dh, x, w):
    """dh [B, U], x [B, I], w [U, I] -> (dW [U, I], dx [B, I], sum|terms| of dW, sum|terms| of dx)."""
    dh = np.asarray(dh, np.float64)
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    return dh.T @ x, dh @ w, np.abs(dh).T @ np.abs(x), np.abs(dh) @ np.abs(w)


# ---------------------------------------------------------------------------------------------- classifier head
def row_weights(labels, C: int, sample_w=None, class_w=None) -> np.ndarray:
    """w_r = sample_w[r] * class_w[label_r] (a null table, or a label outside [0, C), counts as 1)."""
    labels = np.asarray(labels, np.int64)
    w = np.ones(labels.shape[0]) if sample_w is None else np.asarray(sample_w, np.float64).copy()
    if class_w is not None:
        ok = (labels >= 0) & (labels < C)
        w[ok] *= np.asarray(class_w, np.float64)[labels[ok]]
    return w


def dense_head(h, w2, b2, labels, mask1=None, scale1: float = 1.0, sample_w=None, class_w=None) -> dict:
    """The fused head's outputs (float64) and the logits it takes its decisions on; see the module docstring."""
    h = np.asarray(h, np.float64)
    w2 = np.asarray(w2, np.float64)
    labels = np.asarray(labels, np.int64)
    B, C = h.shape[0], w2.shape[0]
    valid = (labels >= 0) & (labels < C)
    logits = h @ w2.T
    _, d, _, _, rows, v = softmax_xent(logits, b2, np.where(valid, labels, 0))
    d[~valid, 0] += 1.0 / B                     # a label outside [0, C) has no onehot term ...
    rows = np.where(valid, rows, 0.0)           # ... and no loss
    wr = row_weights(labels, C, sample_w, class_w)
    d = d * wr[:, None]
    hit = valid & (np.argmax(v, 1) == labels)
    gate = np.ones(h.shape) if mask1 is None else (np.asarray(mask1) & 1) * scale1
    dh = (d @ w2) * gate
    return dict(v=v, d=d, wr=wr, loss=(wr * rows).sum() / B, rows=rows, dw2=d.T @ h, db2=d.sum(0), dh=dh,
                db1=dh.sum(0), gate=gate, stats=np.array([hit.sum(), B, (wr * hit).sum(), wr.sum()], np.float64))


# ---------------------------------------------------------------------------------------------- gather GEMM
def gather_x(tables, ids, numeric, Kp: int) -> np.ndarray:
    """tables: T fp32 [V, 64]; ids [T, B] (outside [0, V): a zero row); numeric [B, n_num] -> x [B, Kp] (zero pad)."""
    ids = np.asarray(ids, np.int64)
    T, B = ids.shape
    n_num = 0 if numeric is None else numeric.shape[1]
    x = np.zeros((B, Kp))
    for t in range(T):
        V = tables[t].shape[0]
        ok = (ids[t] >= 0) & (ids[t] < V)
        x[ok, 64 * t:64 * t + 64] = np.asarray(tables[t], np.float64)[ids[t][ok]]
    if n_num:
        x[:, 64 * T:64 * T + n_num] = numeric
    return x
