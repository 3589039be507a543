"""float64 reference of the parameter-server data plane (estimator/ps.py, estimator/ps_hbm.py, ops/csrc/tfy_ps.cu).

Plain NumPy.  It states the contract the HBM kernels must meet:

* dense push: per element, coupled weight decay first (``g = g * grad_scale + wd * w``), then
    SGD      ``w -= lr g``
    Adagrad  ``acc += g^2 ; w -= lr g / (sqrt(acc) + eps)``
    Adam     ``m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; w -= lr a0 m / (sqrt(v) a1 + eps)`` with the bias-correction
             buffer ``(a0, a1) = (1/(1-b1^t), 1/sqrt(1-b2^t))`` -- torch's formula, the one K4 and the CPU plane use
    FTRL     ``n' = n + g^2 ; z += g - (sqrt(n') - sqrt(n)) / lr w ; w = |z| <= l1 ? 0 : -(z - sgn(z) l1) / ((beta +
             sqrt(n')) / lr + 2 l2)`` (lr_power -0.5), as estimator/ps.py writes it
  Hyper-parameters follow the kernels' TfyPsSeg: p1, p2, p3 = l1, l2, beta (FTRL) | beta1, beta2, - (Adam).
* sparse push: per table only the distinct in-range ids of the batch are touched; each receives the sum of its
  gradients (x 1/L for a mean bag), added in the original (b, j) order, and the optimizer runs ONCE on it.  Rows not
  in the batch keep their values and slots (lazy Adam).  Ids < 0 or >= V are skipped.
* bag / multi-bag: sum, or mean with divisor L, of the rows; skipped ids contribute nothing.
* pull / shadow: the local copy or the bf16 shadow equals the fp32 master rounded to nearest-even; the pad columns of
  a row-padded shadow stay zero.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

SGD, ADAM, ADAGRAD, FTRL = 0, 2, 3, 4          # TfyOpt codes (ops/csrc/tfy_common.cuh)
EPS32 = float(np.finfo(np.float32).eps)


def adam_scale(t: int, beta1: float, beta2: float) -> Tuple[float, float]:
    """The bias-correction buffer of step t (1-based): (1/(1-b1^t), 1/sqrt(1-b2^t))."""
    return 1.0 / (1.0 - beta1 ** t), 1.0 / np.sqrt(1.0 - beta2 ** t)


def ftrl_w(z: np.ndarray, n: np.ndarray, lr: float, l1: float, l2: float, beta: float) -> np.ndarray:
    w = -(z - np.sign(z) * l1) / ((beta + np.sqrt(n)) / lr + 2.0 * l2)
    return np.where(np.abs(z) <= l1, 0.0, w)


def apply(opt: int, w: np.ndarray, s1, s2, g: np.ndarray, hp: Dict[str, float],
          scale: Tuple[float, float] = (1.0, 1.0)) -> None:
    """One optimizer step in place on float64 arrays (g already scaled and decayed)."""
    lr, eps = hp["lr"], hp.get("eps", 0.0)
    if opt == SGD:
        w -= lr * g
    elif opt == ADAGRAD:
        s1 += g * g
        w -= lr * g / (np.sqrt(s1) + eps)
    elif opt == ADAM:
        b1, b2 = hp["p1"], hp["p2"]
        s1 *= b1
        s1 += (1.0 - b1) * g
        s2 *= b2
        s2 += (1.0 - b2) * g * g
        w -= lr * scale[0] * s1 / (np.sqrt(s2) * scale[1] + eps)
    elif opt == FTRL:
        n_new = s1 + g * g
        s2 += g - (np.sqrt(n_new) - np.sqrt(s1)) / lr * w
        s1[...] = n_new
        w[...] = ftrl_w(s2, n_new, lr, hp["p1"], hp["p2"], hp["p3"])
    else:
        raise ValueError(f"unknown optimizer {opt}")


def dense_push(opt: int, w, s1, s2, grad, hp: Dict[str, float], grad_scale: float = 1.0,
               scale: Tuple[float, float] = (1.0, 1.0)) -> None:
    """tfy_ps_push on one variable (in place, float64)."""
    g = np.asarray(grad, np.float64) * grad_scale + hp.get("wd", 0.0) * w
    apply(opt, w, s1, s2, g, hp, scale)


def sparse_push(opt: int, tables: Sequence[np.ndarray], s1s, s2s, ids: np.ndarray, dout: np.ndarray, D: int,
                hp: Dict[str, float], mean: bool = False, grad_scale: float = 1.0, col_stride: int = 0,
                scale: Tuple[float, float] = (1.0, 1.0)) -> None:
    """tfy_ps_push_rows (T = 1) / tfy_ps_multi_push_rows (L = 1) in place.

    ids: int [T, B, L]; table t's id ids[t, b, j] receives dout[b, t*col_stride : t*col_stride + D]."""
    T, B, L = ids.shape
    V = tables[0].shape[0]
    dout = np.asarray(dout, np.float64)
    for t in range(T):
        sums: Dict[int, np.ndarray] = {}
        for b in range(B):
            for j in range(L):
                i = int(ids[t, b, j])
                if i < 0 or i >= V:
                    continue
                g = dout[b, t * col_stride:t * col_stride + D]
                sums[i] = sums[i] + g if i in sums else g.copy()
        f = grad_scale / L if mean else grad_scale
        for i, g in sums.items():
            apply(opt, tables[t][i], None if s1s is None else s1s[t][i], None if s2s is None else s2s[t][i], g * f, hp,
                  scale)


def row_counts(ids: np.ndarray, V: int) -> List[np.ndarray]:
    """Occurrences of every row of every table in one push (ids [T, B, L]): the number of terms of its gradient sum."""
    return [np.bincount(x[(x >= 0) & (x < V)], minlength=V) for x in ids.reshape(ids.shape[0], -1)]


def bag(table: np.ndarray, ids: np.ndarray, mean: bool) -> np.ndarray:
    """tfy_ps_embedding_bag: ids [B, L] -> [B, D]."""
    V, D = table.shape
    B, L = ids.shape
    out = np.zeros((B, D))
    for b in range(B):
        for j in range(L):
            i = int(ids[b, j])
            if 0 <= i < V:
                out[b] += table[i]
    return out / L if mean else out


def multi_bag(tables: Sequence[np.ndarray], ids: np.ndarray) -> np.ndarray:
    """tfy_ps_multi_bag: ids [T, B] -> sum over t of table_t[ids[t, b]]."""
    return sum(bag(tables[t], ids[t][:, None], False) for t in range(len(tables)))


def bf16_round(x) -> np.ndarray:
    """fp32 -> bf16 (round to nearest, ties to even), returned as the float64 values of the bf16 numbers."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def shadow(master: np.ndarray, cols: int, ld: int) -> np.ndarray:
    """The row-padded bf16 shadow of a [rows, cols] master: [rows, ld], pad columns zero (cols == 0: flat)."""
    if not cols:
        return bf16_round(master)
    m = np.asarray(master).reshape(-1, cols)
    out = np.zeros((m.shape[0], ld))
    out[:, :cols] = bf16_round(m)
    return out
