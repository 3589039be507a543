"""NumPy statement of the bucketized and crossed feature columns (estimator/feature_column.py BucketizedColumn /
CrossedColumn), for the torch path and the tfy_feature_ids kernel (ops/csrc/tfy_features.cu) to be checked against.

* bucketized: element j of example b -> c + j * (n + 1), c = the number of boundaries <= x compared in float32
  (np.searchsorted(side="right")), NaN -> n.
* crossed: slot s of example b is the row-major tuple of its leaf keys' values (first key slowest); present iff every
  value is >= 0; id = h % hash_bucket_size in uint64 with h = hash_key, then h = FingerprintCat64(h, v) per value.
"""
from __future__ import annotations

import itertools
from typing import Dict

import numpy as np

M = np.uint64(0xc6a4a7935bd1e995)
DEFAULT_HASH_KEY = 0xDECAFCAFFE


def shift_mix(x: np.ndarray) -> np.ndarray:
    return x ^ (x >> np.uint64(47))


def fingerprint_cat64(a, b) -> np.ndarray:
    with np.errstate(over="ignore"):
        a = np.asarray(a, np.uint64)
        b = np.asarray(b, np.uint64)
        r = a ^ M
        r = r ^ (shift_mix(b * M) * M)
        r = r * M
        r = shift_mix(r) * M
        return shift_mix(r)


def bucketize(x: np.ndarray, boundaries) -> np.ndarray:
    """[B, k] fp32 values -> [B, k] ids."""
    x = np.asarray(x, np.float32).reshape(len(x), -1)
    b = np.asarray(boundaries, np.float32)
    c = np.searchsorted(b, x, side="right")
    c = np.where(np.isnan(x), len(b), c)
    return c + np.arange(x.shape[1]) * (len(b) + 1)


def identity(raw: np.ndarray, V: int) -> np.ndarray:
    raw = np.asarray(raw, np.int64).reshape(len(raw), -1)
    return np.where(raw < 0, -1, raw % V)


def hashed(raw: np.ndarray, V: int) -> np.ndarray:
    """categorical_column_with_hash_bucket's ids: (uint64(raw) * 2654435761 mod 2^32) % V."""
    raw = np.asarray(raw, np.int64).reshape(len(raw), -1)
    with np.errstate(over="ignore"):
        h = (raw.astype(np.uint64) * np.uint64(2654435761)) & np.uint64(0xffffffff)
    return np.where(raw < 0, -1, (h % np.uint64(V)).astype(np.int64))


def cross(values, hash_bucket_size: int, hash_key: int = DEFAULT_HASH_KEY) -> np.ndarray:
    """values: the [B, L_k] int64 component values of every leaf key, in key order -> [B, prod L_k] ids."""
    B = len(values[0])
    L = int(np.prod([v.shape[1] for v in values]))
    out = np.full((B, L), -1, np.int64)
    for b in range(B):
        for s, combo in enumerate(itertools.product(*[v[b] for v in values])):
            if min(combo) < 0:
                continue
            h = np.uint64(hash_key % 2 ** 64)
            for v in combo:
                h = fingerprint_cat64(h, np.uint64(int(v)))
            out[b, s] = int(np.uint64(h) % np.uint64(hash_bucket_size))
    return out


def leaf_values(key, features: Dict[str, np.ndarray]) -> np.ndarray:
    """A cross's leaf key (a feature name, or a column of estimator.feature_column) -> [B, L_k] values."""
    from tf_yarn_b200.estimator import feature_column as fc
    if isinstance(key, str):
        return np.asarray(features[key], np.int64).reshape(len(features[key]), -1)
    if isinstance(key, fc.BucketizedColumn):
        return bucketize(features[key.source_column.key], key.boundaries)
    return identity(features[key.key], key.num_buckets)


def column_ids(col, features: Dict[str, np.ndarray]) -> np.ndarray:
    """[B, L] ids of any categorical column of estimator.feature_column."""
    from tf_yarn_b200.estimator import feature_column as fc
    if isinstance(col, fc.BucketizedColumn):
        return bucketize(features[col.source_column.key], col.boundaries)
    if isinstance(col, fc.CrossedColumn):
        return cross([leaf_values(k, features) for k in col.keys], col.hash_bucket_size, col.hash_key)
    if isinstance(col, fc.WeightedCategoricalColumn):
        col = col.categorical_column
    return (hashed if col.hashed else identity)(features[col.key], col.num_buckets)
