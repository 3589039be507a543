"""float64 reference of multi-hot and weighted categorical columns (TF's embedding_column / weighted_categorical_column
combiners), for the feature columns (estimator/feature_column.py) and the HBM kernels tfy_ps_multi_bag_weighted /
tfy_ps_multi_push_rows_weighted (ops/csrc/tfy_ps.cu).  Plain NumPy.

For table t, example b and slot j: id i = ids[t, b, j], weight w = weights[t, b, j] (1 when unweighted).
* An occurrence is present iff 0 <= i < V and w != 0.  An absent one contributes nothing and touches no row.
* S = sum_present w table[i];  den = 1 (sum), sum_present w (mean), sqrt(sum_present w^2) (sqrtn);
  out = S / den, and 0 where den == 0 (TF's div_no_nan).
* Backward: a present occurrence's gradient is w f[t, b] dout[b] with f = 1/den (0 where den == 0); within one push
  every distinct (t, i) receives the sum of its occurrences' gradients and its optimizer runs once.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import ps_reference as ref

COMBINERS = ("sum", "mean", "sqrtn")


def _w(ids: np.ndarray, weights: Optional[np.ndarray]) -> np.ndarray:
    return np.ones(ids.shape) if weights is None else np.asarray(weights, np.float64)


def present(ids: np.ndarray, weights: Optional[np.ndarray], V: int) -> np.ndarray:
    return (ids >= 0) & (ids < V) & (_w(ids, weights) != 0)


def factors(ids: np.ndarray, weights: Optional[np.ndarray], V: int, combiner: str) -> np.ndarray:
    """f = 1/den per example (ids [..., B, L] -> [..., B]), 0 where den == 0."""
    w = np.where(present(ids, weights, V), _w(ids, weights), 0.0)
    if combiner == "sum":
        den = np.ones(w.shape[:-1])
    elif combiner == "mean":
        den = w.sum(-1)
    elif combiner == "sqrtn":
        den = np.sqrt((w * w).sum(-1))
    else:
        raise ValueError(combiner)
    with np.errstate(divide="ignore"):
        return np.where(den != 0, 1.0 / np.where(den != 0, den, 1.0), 0.0)


def bag(table: np.ndarray, ids: np.ndarray, weights: Optional[np.ndarray], combiner: str) -> np.ndarray:
    """One column: ids [B, L] -> [B, D], S / den (0 where den == 0)."""
    V, D = table.shape
    B, L = ids.shape
    w = _w(ids, weights)
    pres = present(ids, weights, V)
    out = np.zeros((B, D))
    for b in range(B):
        for j in range(L):
            if pres[b, j]:
                out[b] += w[b, j] * table[ids[b, j]]
    return out * factors(ids, weights, V, combiner)[:, None]


def multi_bag(tables: Sequence[np.ndarray], ids: np.ndarray, weights: Optional[np.ndarray], combiner: str,
              col_stride: int) -> np.ndarray:
    """T columns, ids [T, B, L]: concatenated at t * col_stride, or summed (col_stride 0)."""
    T, B, _ = ids.shape
    D = tables[0].shape[1]
    parts = [bag(tables[t], ids[t], None if weights is None else weights[t], combiner) for t in range(T)]
    if col_stride == 0:
        return sum(parts)
    out = np.zeros((B, (T - 1) * col_stride + D))
    for t in range(T):
        out[:, t * col_stride:t * col_stride + D] = parts[t]
    return out


def table_grad(V: int, ids: np.ndarray, weights: Optional[np.ndarray], f: np.ndarray, dout: np.ndarray) -> np.ndarray:
    """d loss / d table of one column: ids [B, L], f [B], dout [B, D] -> [V, D]."""
    g = np.zeros((V, dout.shape[1]))
    w = _w(ids, weights)
    pres = present(ids, weights, V)
    for b in range(ids.shape[0]):
        for j in range(ids.shape[1]):
            if pres[b, j]:
                g[ids[b, j]] += w[b, j] * f[b] * dout[b]
    return g


def sparse_push(opt: int, tables, s1s, s2s, ids: np.ndarray, weights: Optional[np.ndarray], f: Optional[np.ndarray],
                dout: np.ndarray, D: int, hp, grad_scale: float = 1.0, col_stride: int = 0, scale=(1.0, 1.0)) -> None:
    """tfy_ps_multi_push_rows_weighted in place: ids / weights [T, B, L], f [T, B] (None = 1)."""
    T, B, L = ids.shape
    V = tables[0].shape[0]
    dout = np.asarray(dout, np.float64)
    w = _w(ids, weights)
    pres = present(ids, weights, V)
    for t in range(T):
        sums = {}
        for b in range(B):
            c = 1.0 if f is None else float(f[t, b])
            for j in range(L):
                if not pres[t, b, j]:
                    continue
                i = int(ids[t, b, j])
                g = w[t, b, j] * c * dout[b, t * col_stride:t * col_stride + D]
                sums[i] = sums[i] + g if i in sums else g
        for i, g in sums.items():
            ref.apply(opt, tables[t][i], None if s1s is None else s1s[t][i], None if s2s is None else s2s[t][i],
                      g * grad_scale, hp, scale)


def row_counts(ids: np.ndarray, weights: Optional[np.ndarray], V: int):
    """Present occurrences of every row of every table in one push: the number of terms of its gradient sum."""
    pres = present(ids, weights, V)
    return [np.bincount(ids[t][pres[t]], minlength=V) for t in range(ids.shape[0])]
