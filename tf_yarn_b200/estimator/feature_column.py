"""Feature columns (``tf.feature_column`` subset) for the canned estimators.

Used by the reference's examples as ``tf.feature_column.numeric_column(name)``
(reference: tf_yarn/examples/winequality.py:44-45) and by the wide-and-deep
BASELINE config (categorical + embedding columns).
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

COMBINERS = ("sum", "mean", "sqrtn")


class NumericColumn(NamedTuple):
    key: str
    shape: Tuple[int, ...] = (1,)

    @property
    def dim(self) -> int:
        n = 1
        for s in self.shape:
            n *= s
        return n


class CategoricalColumn(NamedTuple):
    key: str
    num_buckets: int
    hashed: bool = False


class WeightedCategoricalColumn(NamedTuple):
    """A categorical column whose every id carries the value found at the same position of the float feature
    ``weight_feature_key`` (``tf.feature_column.weighted_categorical_column``)."""
    categorical_column: CategoricalColumn
    weight_feature_key: str
    dtype: torch.dtype = torch.float32

    @property
    def key(self) -> str:
        return self.categorical_column.key

    @property
    def num_buckets(self) -> int:
        return self.categorical_column.num_buckets

    @property
    def hashed(self) -> bool:
        return self.categorical_column.hashed


Categorical = Union[CategoricalColumn, WeightedCategoricalColumn]


class EmbeddingColumn(NamedTuple):
    categorical_column: Categorical
    dimension: int
    combiner: str = "mean"


class IndicatorColumn(NamedTuple):
    categorical_column: Categorical


def numeric_column(key: str, shape: Sequence[int] = (1,), **_ignored) -> NumericColumn:
    return NumericColumn(key, tuple(shape))


def categorical_column_with_identity(key: str, num_buckets: int, **_ignored) -> CategoricalColumn:
    return CategoricalColumn(key, int(num_buckets), False)


def categorical_column_with_hash_bucket(key: str, hash_bucket_size: int, **_ignored) -> CategoricalColumn:
    return CategoricalColumn(key, int(hash_bucket_size), True)


def weighted_categorical_column(categorical_column: CategoricalColumn, weight_feature_key: str,
                                dtype: torch.dtype = torch.float32) -> WeightedCategoricalColumn:
    if not isinstance(categorical_column, CategoricalColumn):
        raise ValueError(f"weighted_categorical_column wraps a categorical column, got {categorical_column!r}")
    if not dtype.is_floating_point:
        raise ValueError(f"weighted_categorical_column: dtype must be a float type, got {dtype}")
    return WeightedCategoricalColumn(categorical_column, weight_feature_key, dtype)


def _check_combiner(combiner: str) -> str:
    if combiner not in COMBINERS:
        raise ValueError(f"combiner must be one of {COMBINERS}, got {combiner!r}")
    return combiner


def embedding_column(categorical_column: Categorical, dimension: int, combiner: str = "mean",
                     **_ignored) -> EmbeddingColumn:
    return EmbeddingColumn(categorical_column, int(dimension), _check_combiner(combiner))


def indicator_column(categorical_column: Categorical) -> IndicatorColumn:
    return IndicatorColumn(categorical_column)


def _categorical(c) -> Optional[Categorical]:
    """The categorical column a wide-tower column is looked up by (None for a numeric column)."""
    c = c.categorical_column if isinstance(c, (EmbeddingColumn, IndicatorColumn)) else c
    return c if isinstance(c, (CategoricalColumn, WeightedCategoricalColumn)) else None


def _ids(col: Categorical, t: torch.Tensor) -> torch.Tensor:
    """Bucket ids of a raw id tensor; a negative raw id is missing (TF pads ragged dense input with -1) and stays -1."""
    raw = t.long()
    ids = raw
    if col.hashed:
        # cheap integer hash (Knuth multiplicative), stable across processes
        ids = (ids * 2654435761) % (2 ** 32)
    return torch.where(raw < 0, -1, ids % col.num_buckets)


def _ids_and_weights(col: Categorical, features: Dict[str, torch.Tensor]):
    """[B, L] bucket ids (-1 = missing) and, for a weighted column, the [B, L] float weights (else None)."""
    t = features[col.key]
    ids = _ids(col, t).reshape(t.shape[0], -1)
    if not isinstance(col, WeightedCategoricalColumn):
        return ids, None
    return ids, _weights(col, features, ids.shape)


def _weights(col: WeightedCategoricalColumn, features: Dict[str, torch.Tensor], shape) -> torch.Tensor:
    """The [B, L] weights of a weighted column, checked against its ids' shape."""
    if col.weight_feature_key not in features:
        raise KeyError(f"weighted_categorical_column {col.key!r} needs the weight feature {col.weight_feature_key!r}, "
                       f"which the input does not have")
    w = features[col.weight_feature_key]
    w = w.reshape(w.shape[0], -1)
    if w.shape != shape:
        raise ValueError(f"weight feature {col.weight_feature_key!r} has shape {tuple(w.shape)}, "
                         f"its ids {col.key!r} {tuple(shape)}")
    return w


class CombinedBag(nn.EmbeddingBag):
    """An embedding table [V, D] combined over the L ids of every example by TF's rule: an id is present iff it is
    >= 0 and its weight is != 0; ``S = sum_present w row``, ``out = S / den`` with den = 1 (sum), sum_present w
    (mean) or sqrt(sum_present w^2) (sqrtn), and 0 where den == 0.  Same parameters as ``nn.EmbeddingBag`` (the
    parameter-server planes serve it as one); ``mode`` keeps the reduction a one-id-per-example bag would use."""

    def __init__(self, num_embeddings: int, embedding_dim: int, combiner: str):
        super().__init__(num_embeddings, embedding_dim, mode="mean" if combiner == "mean" else "sum")
        self.combiner = _check_combiner(combiner)

    def forward(self, ids: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        present = ids >= 0
        if weights is None:
            w = present.to(self.weight.dtype)
        else:
            w = torch.where(present, weights.to(self.weight.dtype), 0.0)
        s = F.embedding_bag(ids.clamp(min=0), self.weight, mode="sum", per_sample_weights=w)
        if self.combiner == "sum":
            return s
        den = w.sum(1) if self.combiner == "mean" else (w * w).sum(1).sqrt()
        nz = den != 0
        return s / torch.where(nz, den, 1.0)[:, None] * nz[:, None].to(s.dtype)


class DenseFeatures(nn.Module):
    """Concatenate numeric / indicator / embedding columns into one dense [batch, width] tensor."""

    def __init__(self, columns: Sequence[Union[NumericColumn, EmbeddingColumn, IndicatorColumn]]):
        super().__init__()
        self.columns = list(columns)
        self.embeddings = nn.ModuleDict()
        width = 0
        for c in self.columns:
            if isinstance(c, NumericColumn):
                width += c.dim
            elif isinstance(c, EmbeddingColumn):
                emb = CombinedBag(c.categorical_column.num_buckets, c.dimension, c.combiner)
                nn.init.normal_(emb.weight, std=1.0 / c.dimension ** 0.5)
                self.embeddings[c.categorical_column.key] = emb
                width += c.dimension
            elif isinstance(c, IndicatorColumn):
                width += c.categorical_column.num_buckets
            else:
                raise TypeError(f"{c!r} cannot feed a dense layer; wrap it in embedding_column/indicator_column")
        self.width = width

    def forward(self, features: Dict[str, torch.Tensor]) -> torch.Tensor:
        parts: List[torch.Tensor] = []
        ref = None
        for c in self.columns:
            if isinstance(c, NumericColumn):
                t = features[c.key]
                parts.append(t.reshape(t.shape[0], -1))
            elif isinstance(c, EmbeddingColumn):
                ids, w = _ids_and_weights(c.categorical_column, features)
                parts.append(self.embeddings[c.categorical_column.key](ids, w))
            else:
                # the count of every bucket in the example, or the sum of its weights for a weighted column
                ids, w = _ids_and_weights(c.categorical_column, features)
                present = ids >= 0
                w = present.float() if w is None else torch.where(present, w.float(), 0.0)
                parts.append(torch.zeros(ids.shape[0], c.categorical_column.num_buckets, device=ids.device)
                             .scatter_add_(1, ids.clamp(min=0), w))
        dtype = next((p.dtype for p in parts if p.is_floating_point()), torch.float32)
        return torch.cat([p.to(dtype) for p in parts], dim=1)


class LinearModel(nn.Module):
    """Wide part: a weight per numeric dimension and per categorical bucket, plus a bias.  The buckets of one
    categorical column are combined by ``sparse_combiner`` (as an embedding column's ids are), then the columns
    are summed."""

    def __init__(self, columns: Sequence[Union[NumericColumn, Categorical]], units: int,
                 sparse_combiner: str = "sum"):
        super().__init__()
        self.columns = list(columns)
        self.units = units
        self.sparse_combiner = _check_combiner(sparse_combiner)
        n_numeric = sum(c.dim for c in self.columns if isinstance(c, NumericColumn))
        self.numeric = nn.Linear(n_numeric, units, bias=False) if n_numeric else None
        if self.numeric is not None:
            nn.init.zeros_(self.numeric.weight)
        self.tables = nn.ModuleDict()
        for c in self.columns:
            c = _categorical(c)
            if c is not None:
                emb = CombinedBag(c.num_buckets, units, sparse_combiner)
                nn.init.zeros_(emb.weight)
                self.tables[c.key] = emb
        self.bias = nn.Parameter(torch.zeros(units))

    def forward(self, features: Dict[str, torch.Tensor]) -> torch.Tensor:
        out = None
        nums = [features[c.key].reshape(features[c.key].shape[0], -1).float() for c in self.columns
                if isinstance(c, NumericColumn)]
        if nums:
            x = torch.cat(nums, dim=1)
            out = self.numeric(x.to(self.numeric.weight.dtype))
        for c in self.columns:
            cc = _categorical(c)
            if cc is not None:
                y = self.tables[cc.key](*_ids_and_weights(cc, features))
                out = y if out is None else out + y
        return out + self.bias
