"""float64 reference of shared embedding columns (tf.feature_column.shared_embedding_columns): the feature columns
(estimator/feature_column.py) and the HBM push tfy_ps_multi_push_rows_shared (ops/csrc/tfy_ps.cu).  Plain NumPy.

Column t of a collection looks up table table_of[t] with its own ids [B, L_t] and weights, by the combiners of
multihot_reference.  So:
* each member's values are multihot_reference.bag of the shared table with that member's ids;
* the table's gradient is the sum over its members of multihot_reference.table_grad;
* within one push every distinct (table, row) receives the sum of its occurrences' gradients over all its columns, in
  (t, b, j) order, and its optimizer runs once.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import multihot_reference as mh
import ps_reference as ref


def member_values(table: np.ndarray, ids: Sequence[np.ndarray], weights: Sequence[Optional[np.ndarray]],
                  combiner: str):
    """[B, D] of every member of a collection."""
    return [mh.bag(table, i, w, combiner) for i, w in zip(ids, weights)]


def table_grad(V: int, ids: Sequence[np.ndarray], weights: Sequence[Optional[np.ndarray]], combiner: str,
               douts: Sequence[np.ndarray]) -> np.ndarray:
    """d loss / d table: the sum over the members of their own column's gradient."""
    return sum(mh.table_grad(V, i, w, mh.factors(i, w, V, combiner), d) for i, w, d in zip(ids, weights, douts))


def sparse_push(opt: int, tables, s1s, s2s, table_of: Sequence[int], ids: np.ndarray, weights: Optional[np.ndarray],
                f: Optional[np.ndarray], dout: np.ndarray, D: int, hp, grad_scale: float = 1.0, col_stride: int = 0,
                scale=(1.0, 1.0)) -> None:
    """tfy_ps_multi_push_rows_shared in place: tables / s1s / s2s per distinct table, ids / weights [T, B, L],
    f [T, B] (None = 1)."""
    T, B, L = ids.shape
    V = tables[0].shape[0]
    dout = np.asarray(dout, np.float64)
    w = mh._w(ids, weights)
    pres = mh.present(ids, weights, V)
    sums = {}
    for t in range(T):                       # (t, b, j) order
        for b in range(B):
            c = 1.0 if f is None else float(f[t, b])
            for j in range(L):
                if pres[t, b, j]:
                    key = (table_of[t], int(ids[t, b, j]))
                    g = w[t, b, j] * c * dout[b, t * col_stride:t * col_stride + D]
                    sums[key] = sums[key] + g if key in sums else g
    for (k, i), g in sums.items():
        ref.apply(opt, tables[k][i], None if s1s is None else s1s[k][i], None if s2s is None else s2s[k][i],
                  g * grad_scale, hp, scale)


def row_counts(table_of: Sequence[int], n_tables: int, ids: np.ndarray, weights: Optional[np.ndarray], V: int):
    """Present occurrences of every row of every distinct table in one push."""
    per_col = mh.row_counts(ids, weights, V)
    out = [np.zeros(V, np.int64) for _ in range(n_tables)]
    for t, c in enumerate(per_col):
        out[table_of[t]] += c
    return out
