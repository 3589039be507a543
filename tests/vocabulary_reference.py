"""NumPy statement of the vocabulary columns (estimator/feature_column.py VocabularyColumn), with a Python dict for the
vocabulary, for the torch path and the tfy_vocab_ids kernel (ops/csrc/tfy_features.cu) to be checked against.

With n entries, entry i has id i.  A raw value v maps to:
* -1 if v < 0 (missing);
* its id if it is an entry;
* n + ((uint64) v * 2654435761 mod 2^32) % num_oov_buckets if num_oov_buckets > 0;
* default_value otherwise.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

import crossed_reference as cref


def lookup(raw, entries, num_oov_buckets: int = 0, default_value: int = -1) -> np.ndarray:
    """[B, ...] raw integers -> int64 [B, L] ids."""
    raw = np.asarray(raw, np.int64).reshape(len(raw), -1)
    table = {int(v): i for i, v in enumerate(entries)}
    n = len(table)
    assert n == len(entries), "the reference needs distinct entries"
    out = np.empty(raw.shape, np.int64)
    for idx, v in np.ndenumerate(raw):
        v = int(v)
        if v < 0:
            out[idx] = -1
        elif v in table:
            out[idx] = table[v]
        elif num_oov_buckets > 0:
            out[idx] = n + ((v * 2654435761) % 2 ** 32) % num_oov_buckets
        else:
            out[idx] = default_value
    return out


def column_lookup(col, raw) -> np.ndarray:
    return lookup(raw, [int(v) for v in col.vocabulary.keys], col.num_oov_buckets, col.default_value)


def leaf_values(key, features: Dict[str, np.ndarray]) -> np.ndarray:
    from tf_yarn_b200.estimator import feature_column as fc
    if isinstance(key, fc.VocabularyColumn):
        return column_lookup(key, features[key.key])
    return cref.leaf_values(key, features)


def column_ids(col, features: Dict[str, np.ndarray]) -> np.ndarray:
    """[B, L] ids of any categorical column, vocabulary columns (bare, weighted or as a cross's leaf) included."""
    from tf_yarn_b200.estimator import feature_column as fc
    base = col.categorical_column if isinstance(col, fc.WeightedCategoricalColumn) else col
    if isinstance(base, fc.VocabularyColumn):
        return column_lookup(base, features[base.key])
    if isinstance(col, fc.CrossedColumn):
        return cref.cross([leaf_values(k, features) for k in col.keys], col.hash_bucket_size, col.hash_key)
    return cref.column_ids(col, features)
