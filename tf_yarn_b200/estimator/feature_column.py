"""Feature columns (``tf.feature_column`` subset) for the canned estimators.

Used by the reference's examples as ``tf.feature_column.numeric_column(name)``
(reference: tf_yarn/examples/winequality.py:44-45) and by the wide-and-deep
BASELINE config (categorical + embedding columns).
"""
from __future__ import annotations

import hashlib
import re
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
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
        """Whether the ids are hashed (a vocabulary column's never are)."""
        return isinstance(self.categorical_column, CategoricalColumn) and self.categorical_column.hashed


class BucketizedColumn(NamedTuple):
    """``tf.feature_column.bucketized_column``: element j of a numeric column of shape (k,) falls in bucket c = the
    number of boundaries <= x (TF's ``Bucketize``, ``std::upper_bound``), and its id is ``c + j * (len(boundaries) +
    1)``.  So an example has k ids, all present, and ``num_buckets = k * (len(boundaries) + 1)``.  x and the boundaries
    are compared in float32 on every path; NaN goes to the last bucket, as ``upper_bound`` puts it."""
    source_column: NumericColumn
    boundaries: Tuple[float, ...]

    @property
    def key(self) -> str:
        return f"{self.source_column.key}_bucketized"

    @property
    def num_buckets(self) -> int:
        return self.source_column.dim * (len(self.boundaries) + 1)


CROSS_HASH_KEY = 0xDECAFCAFFE
MAX_CROSS_BUCKETS = 2 ** 62         # the int64 statement of the unsigned modulo (_umod) holds below it
_U64 = 2 ** 64


class CrossedColumn(NamedTuple):
    """``tf.feature_column.crossed_column``: the Cartesian product of its leaf keys' ids, hashed into
    ``hash_bucket_size`` buckets.

    A leaf key is a raw integer feature (a string: its values are used as they are), an identity categorical column
    (its bucket ids) or a bucketized column.  Example b has, for leaf key k, L_k component values, a negative one
    being missing.  The cross has ``L = prod L_k`` slots in row-major order (the first key varies slowest).  A slot
    is present iff all its components are; its id is ``h % hash_bucket_size`` in uint64 arithmetic, with
    ``h = hash_key`` and then ``h = FingerprintCat64(h, (uint64) v)`` for each component value v in key order::

        FingerprintCat64(a, b): M = 0xc6a4a7935bd1e995
            r = a ^ M;  r ^= ShiftMix(b * M) * M;  r *= M;  r = ShiftMix(r) * M;  r = ShiftMix(r)
        ShiftMix(x) = x ^ (x >> 47)                (mod 2^64, logical shift)

    An absent slot is -1.  The formula follows TF's ``SparseCrossHashed``; that the ids are TF's own has not been
    checked against TF.  A vocabulary column's OOV buckets are not TF's either (see VocabularyColumn)."""
    keys: Tuple[Union[str, CategoricalColumn, BucketizedColumn, "VocabularyColumn"], ...]   # nested crosses flattened
    hash_bucket_size: int
    hash_key: int = CROSS_HASH_KEY

    @property
    def key(self) -> str:
        return "_X_".join(sorted(k if isinstance(k, str) else k.key for k in self.keys))

    @property
    def num_buckets(self) -> int:
        return self.hash_bucket_size


MAX_VOCABULARY = 2 ** 31 - 1            # entries of one vocabulary: its ids are int32 on the device
HASH_MULT = 2654435761                  # categorical_column_with_hash_bucket's multiplicative hash


class Vocabulary:
    """The entries of a vocabulary column, in list (or file) order, as a read-only int64 array: entry i has id i.

    Immutable.  Equality and hashing go through a SHA-256 digest of the entries computed once, so a column holding a
    million entries is as cheap a dict key as any other; it pickles its entries only.  ``tables(device)`` gives the
    keys sorted ascending with the id of each, built once per device and shared by every user of the vocabulary there
    (the torch statement and the HBM plane's id kernels), so a lookup never re-sorts or re-uploads."""

    __slots__ = ("_keys", "_digest", "_sorted", "_tables")

    def __init__(self, entries):
        keys = _vocabulary_entries(entries)
        keys.setflags(write=False)
        self._keys = keys
        self._digest = hashlib.sha256(keys.tobytes()).digest()
        order = np.argsort(keys, kind="stable")
        skeys = keys[order]
        if skeys.size > 1 and bool(np.any(skeys[1:] == skeys[:-1])):
            dup = skeys[1:][skeys[1:] == skeys[:-1]][0]
            raise ValueError(f"vocabulary has duplicate entries, e.g. {int(dup)}")
        skeys.setflags(write=False)
        ids = order.astype(np.int32)
        ids.setflags(write=False)
        self._sorted = (skeys, ids)
        self._tables: Dict[torch.device, Tuple[torch.Tensor, torch.Tensor]] = {}

    @property
    def keys(self) -> np.ndarray:
        """int64 [n] entries in id order (read-only)."""
        return self._keys

    @property
    def sorted(self) -> Tuple[np.ndarray, np.ndarray]:
        """(int64 keys sorted ascending, int32 id of each), read-only host arrays."""
        return self._sorted

    def tables(self, device) -> Tuple[torch.Tensor, torch.Tensor]:
        """The sorted keys (int64) and their ids (int32) on ``device``, uploaded on first use.  Read-only: every user
        of the vocabulary on that device shares them."""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        t = self._tables.get(device)
        if t is None:
            skeys, ids = self._sorted
            t = (torch.from_numpy(skeys.copy()).to(device), torch.from_numpy(ids.copy()).to(device))
            self._tables[device] = t
        return t

    def __len__(self) -> int:
        return int(self._keys.size)

    def __eq__(self, other) -> bool:
        return isinstance(other, Vocabulary) and self._digest == other._digest

    def __hash__(self) -> int:
        return hash(self._digest)

    def __reduce__(self):
        return Vocabulary, (self._keys,)

    def __repr__(self) -> str:
        head = ", ".join(str(int(k)) for k in self._keys[:4])
        return f"Vocabulary(n={len(self)}, [{head}{', ...' if len(self) > 4 else ''}], sha256={self._digest[:6].hex()})"


def _vocabulary_entries(entries) -> np.ndarray:
    """int64 [n] array of a vocabulary's entries, each an integer in [0, 2^63); ValueError otherwise."""
    if isinstance(entries, np.ndarray):
        if entries.ndim != 1 or entries.dtype.kind not in "iu":
            raise ValueError(f"vocabulary entries must be a 1-D array of integers in [0, 2^63), got an array of "
                             f"shape {entries.shape} and dtype {entries.dtype}")
        n = entries.size
    else:
        if isinstance(entries, (str, bytes)):
            raise ValueError(f"vocabulary must be a list of integers, got {entries!r}")
        n = len(entries)
    if n == 0:
        raise ValueError("vocabulary is empty")
    if n > MAX_VOCABULARY:
        raise ValueError(f"vocabulary has {n} entries; at most 2^31 - 1 are supported")
    if isinstance(entries, np.ndarray):
        if entries.min() < 0 or (entries.dtype.kind == "u" and int(entries.max()) >= 2 ** 63):
            raise ValueError("vocabulary entries must be integers in [0, 2^63)")
        return np.array(entries, dtype=np.int64, copy=True)       # a private copy: the caller's array stays its own
    for v in entries:
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 0 <= int(v) < 2 ** 63:
            raise ValueError(f"vocabulary entries must be integers in [0, 2^63), got {v!r}; no column here takes "
                             f"string features")
    return np.array([int(v) for v in entries], dtype=np.int64)


class VocabularyColumn(NamedTuple):
    """``tf.feature_column.categorical_column_with_vocabulary_list`` / ``_file`` over integer features.

    Entry i of ``vocabulary`` (its position in the list, its line in the file) has id i; n = len(vocabulary) and
    ``num_buckets = n + num_oov_buckets``.  A raw value v maps to:

    * -1 (missing) if v < 0, the convention of every column here (TF treats only -1 as missing for integers);
    * its id if v is in the vocabulary;
    * else, with ``num_oov_buckets > 0``: ``n + ((uint64) v * 2654435761 mod 2^32) % num_oov_buckets``, the hash of
      ``categorical_column_with_hash_bucket``.  These OOV ids are not TF's, which hashes the decimal string with
      Fingerprint64;
    * else ``default_value`` (-1, the default, is absent).

    The ids are the same on every path: the torch statement (``_vocabulary_ids``, a searchsorted over the sorted keys)
    and the HBM parameter server's ``tfy_vocab_ids`` kernel, a binary search over the same keys."""
    key: str
    vocabulary: Vocabulary
    num_oov_buckets: int = 0
    default_value: int = -1

    @property
    def num_buckets(self) -> int:
        return len(self.vocabulary) + self.num_oov_buckets


Categorical = Union[CategoricalColumn, WeightedCategoricalColumn, BucketizedColumn, CrossedColumn, VocabularyColumn]
DERIVED = (BucketizedColumn, CrossedColumn)         # columns whose ids are computed from other features


class EmbeddingColumn(NamedTuple):
    categorical_column: Categorical
    dimension: int
    combiner: str = "mean"


class SharedEmbeddingColumn(NamedTuple):
    """One member of ``tf.feature_column.shared_embedding_columns``: a column whose ids look up the table named
    ``shared_name``, which every member of the collection shares.

    Each member keeps its own ids, weights and position: in ``DenseFeatures`` it adds ``dimension`` columns where it
    stands, combined by ``combiner`` over its own ids exactly as an ``embedding_column`` would be.  The table is one
    ``[num_buckets, dimension]`` parameter, ``embeddings[shared_name]``, created once per ``DenseFeatures`` and
    initialised as an ``embedding_column``'s; its gradient is the sum of the members' gradients.  Two
    ``DenseFeatures`` built on the same collection each create their own table."""
    categorical_column: Categorical
    dimension: int
    combiner: str
    shared_name: str


class IndicatorColumn(NamedTuple):
    categorical_column: Categorical


def numeric_column(key: str, shape: Sequence[int] = (1,), **_ignored) -> NumericColumn:
    return NumericColumn(key, tuple(shape))


def categorical_column_with_identity(key: str, num_buckets: int, **_ignored) -> CategoricalColumn:
    return CategoricalColumn(key, int(num_buckets), False)


def categorical_column_with_hash_bucket(key: str, hash_bucket_size: int, **_ignored) -> CategoricalColumn:
    return CategoricalColumn(key, int(hash_bucket_size), True)


_INT_DTYPES = (None, torch.int32, torch.int64, "int32", "int64")


def _integer(fn: str, name: str, v) -> int:
    """v as an int; ValueError for anything but an integer (a float is not truncated, a bool is not a count)."""
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise ValueError(f"{fn}: {name} must be an integer, got {v!r}")
    return int(v)


def _vocabulary_column(fn: str, key: str, vocabulary: Vocabulary, num_oov_buckets, default_value, dtype):
    if not any(dtype is d or (isinstance(dtype, str) and dtype == d) for d in _INT_DTYPES):
        raise ValueError(f"{fn}: dtype must be None, torch.int32/torch.int64 or 'int32'/'int64', got {dtype!r}; no "
                         f"column here takes string features")
    n, oov, dflt = len(vocabulary), _integer(fn, "num_oov_buckets", num_oov_buckets), \
        _integer(fn, "default_value", default_value)
    if not 0 <= oov <= MAX_VOCABULARY:
        raise ValueError(f"{fn}: num_oov_buckets must be in [0, 2^31), got {num_oov_buckets}")
    if oov > 0 and dflt != -1:
        raise ValueError(f"{fn}: set either num_oov_buckets ({oov}) or default_value ({dflt}), not both")
    if not -1 <= dflt < n:
        raise ValueError(f"{fn}: default_value must be -1 or an id in [0, {n}), got {default_value}")
    return VocabularyColumn(key, vocabulary, oov, dflt)


def categorical_column_with_vocabulary_list(key: str, vocabulary_list, dtype=None, default_value: int = -1,
                                            num_oov_buckets: int = 0) -> VocabularyColumn:
    """Ids of an integer feature by its position in ``vocabulary_list`` (see VocabularyColumn).  The entries must be
    distinct integers in [0, 2^63)."""
    return _vocabulary_column("categorical_column_with_vocabulary_list", key, Vocabulary(vocabulary_list),
                              num_oov_buckets, default_value, dtype)


_DECIMAL = re.compile(r"[+-]?[0-9]+")


def _read_vocabulary_file(path: str, vocabulary_size: Optional[int]) -> List[int]:
    """The entries of a vocabulary file: one base-10 integer per line, surrounding whitespace stripped, a single
    trailing newline allowed; the first ``vocabulary_size`` lines if given."""
    with open(path, "r") as fh:
        text = fh.read()
    lines = text.split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    if vocabulary_size is not None:
        vocabulary_size = _integer("categorical_column_with_vocabulary_file", "vocabulary_size", vocabulary_size)
        if not 1 <= vocabulary_size <= len(lines):
            raise ValueError(f"vocabulary file {path!r}: vocabulary_size must be in [1, {len(lines)}] (its number of "
                             f"lines), got {vocabulary_size}")
        lines = lines[:vocabulary_size]
    out = []
    for i, line in enumerate(lines):
        s = line.strip()
        if not _DECIMAL.fullmatch(s):
            raise ValueError(f"vocabulary file {path!r}, line {i + 1}: expected one base-10 integer, got {line!r}")
        out.append(int(s))
    return out


def categorical_column_with_vocabulary_file(key: str, vocabulary_file: str, vocabulary_size: Optional[int] = None,
                                            num_oov_buckets: int = 0, default_value: Optional[int] = None,
                                            dtype=None) -> VocabularyColumn:
    """Ids of an integer feature by its line in ``vocabulary_file`` (see VocabularyColumn), read once, here."""
    fn = "categorical_column_with_vocabulary_file"
    if default_value is None:
        default_value = -1
    elif _integer(fn, "num_oov_buckets", num_oov_buckets) > 0:
        raise ValueError(f"categorical_column_with_vocabulary_file: set either num_oov_buckets ({num_oov_buckets}) "
                         f"or default_value ({default_value}), not both")
    return _vocabulary_column("categorical_column_with_vocabulary_file", key,
                              Vocabulary(_read_vocabulary_file(vocabulary_file, vocabulary_size)), num_oov_buckets,
                              default_value, dtype)


def weighted_categorical_column(categorical_column: Union[CategoricalColumn, VocabularyColumn], weight_feature_key: str,
                                dtype: torch.dtype = torch.float32) -> WeightedCategoricalColumn:
    if not isinstance(categorical_column, (CategoricalColumn, VocabularyColumn)):
        raise ValueError(f"weighted_categorical_column wraps a categorical column, got {categorical_column!r}")
    if not dtype.is_floating_point:
        raise ValueError(f"weighted_categorical_column: dtype must be a float type, got {dtype}")
    return WeightedCategoricalColumn(categorical_column, weight_feature_key, dtype)


def bucketized_column(source_column: NumericColumn, boundaries: Sequence[float]) -> BucketizedColumn:
    """Buckets of a numeric column of shape (k,) split at strictly increasing ``boundaries`` (see BucketizedColumn)."""
    if not isinstance(source_column, NumericColumn) or len(source_column.shape) != 1:
        raise ValueError(f"bucketized_column needs a numeric column of a 1-D shape, got {source_column!r}")
    bounds = tuple(float(b) for b in boundaries) if isinstance(boundaries, (list, tuple)) else ()
    if not bounds or any(a >= b for a, b in zip(bounds, bounds[1:])):
        raise ValueError(f"bucketized_column: boundaries must be a non-empty, strictly increasing list, "
                         f"got {boundaries!r}")
    return BucketizedColumn(source_column, bounds)


def crossed_column(keys: Sequence, hash_bucket_size: int, hash_key: Optional[int] = None) -> CrossedColumn:
    """The hashed cross of ``keys`` (strings, identity categorical, bucketized or crossed columns; see
    CrossedColumn)."""
    leaves: List = []
    for k in keys:
        if isinstance(k, CrossedColumn):
            leaves.extend(k.keys)
        elif isinstance(k, WeightedCategoricalColumn):
            raise ValueError(f"crossed_column does not support weight_tensor, got {k!r}")
        elif isinstance(k, CategoricalColumn) and k.hashed:
            raise ValueError(f"crossed_column does not support a hashed categorical column, got {k!r}; cross its "
                             f"raw feature {k.key!r} instead")
        elif isinstance(k, (str, CategoricalColumn, BucketizedColumn, VocabularyColumn)):
            leaves.append(k)
        else:
            raise ValueError(f"crossed_column keys must be feature names, identity categorical, vocabulary, "
                             f"bucketized or crossed columns, got {k!r}")
    if len(leaves) < 2:
        raise ValueError(f"crossed_column needs at least two keys, got {keys!r}")
    if not 1 <= int(hash_bucket_size) < MAX_CROSS_BUCKETS:
        raise ValueError(f"crossed_column: hash_bucket_size must be >= 1 and < 2^62, got {hash_bucket_size}")
    return CrossedColumn(tuple(leaves), int(hash_bucket_size), CROSS_HASH_KEY if hash_key is None else int(hash_key))


def _check_combiner(combiner: str) -> str:
    if combiner not in COMBINERS:
        raise ValueError(f"combiner must be one of {COMBINERS}, got {combiner!r}")
    return combiner


def embedding_column(categorical_column: Categorical, dimension: int, combiner: str = "mean",
                     **_ignored) -> EmbeddingColumn:
    return EmbeddingColumn(categorical_column, int(dimension), _check_combiner(combiner))


def _kind(c) -> Optional[str]:
    """What a shared collection's members must agree on: the column type (a weighted column counts as its base
    column; identity and hashed columns differ), or None for a non-categorical column."""
    c = c.categorical_column if isinstance(c, WeightedCategoricalColumn) else c
    if isinstance(c, CategoricalColumn):
        return "hashed" if c.hashed else "identity"
    if isinstance(c, VocabularyColumn):
        return "vocabulary"
    return type(c).__name__ if isinstance(c, DERIVED) else None


def shared_embedding_columns(categorical_columns: Sequence[Categorical], dimension: int, combiner: str = "mean",
                             shared_embedding_collection_name: Optional[str] = None,
                             **_ignored) -> List[SharedEmbeddingColumn]:
    """``tf.feature_column.shared_embedding_columns``: one SharedEmbeddingColumn per input, in input order, all
    looking up one table.  The members must be categorical columns of one kind with one ``num_buckets`` and distinct
    keys.  The default collection name is TF's: the sorted member keys joined by "_", then "_shared_embedding"."""
    cols = list(categorical_columns)
    if not cols:
        raise ValueError("shared_embedding_columns needs at least one categorical column")
    for c in cols:
        if _kind(c) is None:
            raise ValueError(f"shared_embedding_columns: {c!r} is not a categorical column")
    if len({_kind(c) for c in cols}) > 1:
        raise ValueError(f"shared_embedding_columns: all columns must be of one kind, got "
                         f"{sorted({_kind(c) for c in cols})}")
    if len({c.num_buckets for c in cols}) > 1:
        raise ValueError(f"shared_embedding_columns: all columns must have the same num_buckets, got "
                         f"{[c.num_buckets for c in cols]}")
    keys = [c.key for c in cols]
    if len(set(keys)) < len(keys):
        raise ValueError(f"shared_embedding_columns: a column appears twice, keys {keys}")
    if int(dimension) < 1:
        raise ValueError(f"shared_embedding_columns: dimension must be >= 1, got {dimension}")
    _check_combiner(combiner)
    name = shared_embedding_collection_name or "_".join(sorted(keys)) + "_shared_embedding"
    return [SharedEmbeddingColumn(c, int(dimension), combiner, name) for c in cols]


shared_embeddings = shared_embedding_columns          # the TF2 name


def _embedding_key(c) -> str:
    """The DenseFeatures.embeddings key of an embedding or shared embedding column."""
    return c.shared_name if isinstance(c, SharedEmbeddingColumn) else c.categorical_column.key


def indicator_column(categorical_column: Categorical) -> IndicatorColumn:
    return IndicatorColumn(categorical_column)


def _categorical(c) -> Optional[Categorical]:
    """The categorical column a wide-tower column is looked up by (None for a numeric column)."""
    c = c.categorical_column if isinstance(c, (EmbeddingColumn, IndicatorColumn)) else c
    return c if isinstance(c, (CategoricalColumn, WeightedCategoricalColumn, VocabularyColumn) + DERIVED) else None


def _device_ids(c) -> bool:
    """True for a column whose ids the HBM parameter server builds on the device (ops/features.py FeatureIds):
    bucketized, crossed and vocabulary columns, the last also inside a weighted column."""
    c = c.categorical_column if isinstance(c, WeightedCategoricalColumn) else c
    return isinstance(c, DERIVED + (VocabularyColumn,))


def _vocabulary_ids(col: VocabularyColumn, t: torch.Tensor) -> torch.Tensor:
    """Ids of a vocabulary column's raw values, same shape (see VocabularyColumn): a lower-bound search over the
    vocabulary's sorted keys, cached on the values' device."""
    raw = t.long().contiguous()
    keys, ids = col.vocabulary.tables(raw.device)
    n = keys.numel()
    pos = torch.searchsorted(keys, raw).clamp_(max=n - 1)
    hit = keys[pos] == raw
    if col.num_oov_buckets > 0:
        miss = n + (raw * HASH_MULT) % (2 ** 32) % col.num_oov_buckets     # the low 32 bits of the wrapped product
    else:
        miss = torch.full_like(raw, col.default_value)
    return torch.where(raw < 0, -1, torch.where(hit, ids[pos].long(), miss))


def _ids(col: Categorical, t: torch.Tensor) -> torch.Tensor:
    """Bucket ids of a raw id tensor; a negative raw id is missing (TF pads ragged dense input with -1) and stays -1."""
    raw = t.long()
    ids = raw
    if col.hashed:
        # cheap integer hash (Knuth multiplicative), stable across processes
        ids = (ids * 2654435761) % (2 ** 32)
    return torch.where(raw < 0, -1, ids % col.num_buckets)


def _check_source_width(col: BucketizedColumn, width: int) -> None:
    """A bucketized column's feature must have the k values per example of its shape: its ids are < k * (n + 1)."""
    if width != col.source_column.dim:
        raise ValueError(f"bucketized_column {col.key!r}: feature {col.source_column.key!r} has {width} values "
                         f"per example, the column's shape {col.source_column.shape}")


def _bucketize(col: BucketizedColumn, features: Dict[str, torch.Tensor]) -> torch.Tensor:
    """[B, k] ids of a bucketized column: bucket c + j * (len(boundaries) + 1), compared in float32, NaN last."""
    x = features[col.source_column.key]
    x = x.reshape(x.shape[0], -1).float().contiguous()
    k, n = col.source_column.dim, len(col.boundaries)
    _check_source_width(col, x.shape[1])
    bounds = torch.tensor(col.boundaries, dtype=torch.float32, device=x.device)
    c = torch.searchsorted(bounds, x, right=True)
    c = torch.where(torch.isnan(x), n, c)
    return c + torch.arange(k, device=x.device) * (n + 1)


def _shift_mix(x: torch.Tensor) -> torch.Tensor:
    return x ^ ((x >> 47) & ((1 << 17) - 1))          # logical shift of the uint64 held in an int64


def _as_i64(u: int) -> int:
    """The int64 with the bits of the uint64 u mod 2^64."""
    return (u % _U64 ^ 2 ** 63) - 2 ** 63


_M = _as_i64(0xc6a4a7935bd1e995)


def _fingerprint_cat64(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """FingerprintCat64 on uint64 values held in int64 tensors (multiplication wraps mod 2^64 either way)."""
    r = a ^ _M
    r = r ^ (_shift_mix(b * _M) * _M)
    r = r * _M
    r = _shift_mix(r) * _M
    return _shift_mix(r)


def _umod(h: torch.Tensor, n: int) -> torch.Tensor:
    """(uint64) h % n for the int64 h with the same bits (n < 2^62)."""
    return torch.where(h < 0, (h % n + _U64 % n) % n, h % n)


def _leaf_values(k, features: Dict[str, torch.Tensor]) -> torch.Tensor:
    """[B, L_k] int64 component values of a cross's leaf key (negative = missing)."""
    if isinstance(k, str):
        t = features[k]
        return t.reshape(t.shape[0], -1).long()
    if isinstance(k, BucketizedColumn):
        return _bucketize(k, features)
    t = features[k.key]
    if isinstance(k, VocabularyColumn):              # a cross hashes the vocabulary ids, as TF's does
        return _vocabulary_ids(k, t).reshape(t.shape[0], -1)
    return _ids(k, t).reshape(t.shape[0], -1)


def _cross(col: CrossedColumn, features: Dict[str, torch.Tensor]) -> torch.Tensor:
    """[B, prod L_k] ids of a crossed column, -1 where a component is missing."""
    h = present = None
    for k in col.keys:
        v = _leaf_values(k, features)
        if h is None:
            h = torch.full(v.shape[:1] + (1,), _as_i64(col.hash_key), dtype=torch.int64, device=v.device)
            present = torch.ones_like(h, dtype=torch.bool)
        B = v.shape[0]
        h = _fingerprint_cat64(h[:, :, None], v[:, None, :]).reshape(B, -1)
        present = (present[:, :, None] & (v >= 0)[:, None, :]).reshape(B, -1)
    return torch.where(present, _umod(h, col.hash_bucket_size), -1)


def _width(col, features: Dict[str, torch.Tensor]) -> int:
    """L of a column's (or a cross's leaf key's) [B, L] ids, from the features' shapes alone."""
    if isinstance(col, str):
        return features[col][0].numel()
    if isinstance(col, BucketizedColumn):
        return col.source_column.dim
    if isinstance(col, CrossedColumn):
        n = 1
        for k in col.keys:
            n *= _width(k, features)
        return n
    return features[col.key][0].numel()


def _ids_and_weights(col: Categorical, features: Dict[str, torch.Tensor]):
    """[B, L] bucket ids (-1 = missing) and, for a weighted column, the [B, L] float weights (else None).  A bucketized
    or crossed column computes its ids from the features it is built on, a vocabulary column looks its values up."""
    if isinstance(col, BucketizedColumn):
        return _bucketize(col, features), None
    if isinstance(col, CrossedColumn):
        return _cross(col, features), None
    t = features[col.key]
    base = col.categorical_column if isinstance(col, WeightedCategoricalColumn) else col
    if isinstance(base, VocabularyColumn):
        ids = _vocabulary_ids(base, t).reshape(t.shape[0], -1)
    else:
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

    def __init__(self, columns: Sequence[Union[NumericColumn, EmbeddingColumn, SharedEmbeddingColumn, IndicatorColumn,
                                               BucketizedColumn]]):
        super().__init__()
        self.columns = list(columns)
        self.embeddings = nn.ModuleDict()
        # shared name -> positions of its members in self.columns
        self.shared: Dict[str, List[int]] = {}
        width = 0
        for pos, c in enumerate(self.columns):
            if isinstance(c, NumericColumn):
                width += c.dim
            elif isinstance(c, EmbeddingColumn):
                if c.categorical_column.key in self.shared:
                    raise ValueError(f"embedding column {c.categorical_column.key!r} has the name of a shared "
                                     f"embedding collection")
                emb = CombinedBag(c.categorical_column.num_buckets, c.dimension, c.combiner)
                nn.init.normal_(emb.weight, std=1.0 / c.dimension ** 0.5)
                self.embeddings[c.categorical_column.key] = emb
                width += c.dimension
            elif isinstance(c, SharedEmbeddingColumn):
                name = c.shared_name
                if name in self.shared:
                    first = self.columns[self.shared[name][0]]
                    if (first.categorical_column.num_buckets, first.dimension, first.combiner) != \
                            (c.categorical_column.num_buckets, c.dimension, c.combiner):
                        raise ValueError(f"shared embedding collection {name!r}: members disagree on num_buckets, "
                                         f"dimension or combiner: {first!r} and {c!r}")
                    self.shared[name].append(pos)
                else:
                    if name in self.embeddings:
                        raise ValueError(f"shared embedding collection {name!r} has the name of another embedding")
                    emb = CombinedBag(c.categorical_column.num_buckets, c.dimension, c.combiner)
                    nn.init.normal_(emb.weight, std=1.0 / c.dimension ** 0.5)
                    self.embeddings[name] = emb
                    self.shared[name] = [pos]
                width += c.dimension
            elif isinstance(c, IndicatorColumn):
                width += c.categorical_column.num_buckets
            elif isinstance(c, BucketizedColumn):       # TF's dense form: the one-hot of its k ids
                width += c.num_buckets
            else:
                raise TypeError(f"{c!r} cannot feed a dense layer; wrap it in embedding_column/indicator_column")
        self.width = width

    def shared_lookup(self, name: str, features: Dict[str, torch.Tensor]) -> List[torch.Tensor]:
        """The [B, dimension] values of the members of collection ``name``, in column order.  The HBM parameter server
        replaces it on the instance with one bag and one push for the whole collection."""
        emb = self.embeddings[name]
        return [emb(*_ids_and_weights(self.columns[p].categorical_column, features)) for p in self.shared[name]]

    def forward(self, features: Dict[str, torch.Tensor]) -> torch.Tensor:
        parts: List[torch.Tensor] = []
        ref = None
        shared = {}
        for name, positions in self.shared.items():
            shared.update(zip(positions, self.shared_lookup(name, features)))
        for pos, c in enumerate(self.columns):
            if isinstance(c, NumericColumn):
                t = features[c.key]
                parts.append(t.reshape(t.shape[0], -1))
            elif isinstance(c, SharedEmbeddingColumn):
                parts.append(shared[pos])
            elif isinstance(c, EmbeddingColumn):
                ids, w = _ids_and_weights(c.categorical_column, features)
                parts.append(self.embeddings[c.categorical_column.key](ids, w))
            else:
                # the count of every bucket in the example, or the sum of its weights for a weighted column
                cat = c if isinstance(c, BucketizedColumn) else c.categorical_column
                ids, w = _ids_and_weights(cat, features)
                present = ids >= 0
                w = present.float() if w is None else torch.where(present, w.float(), 0.0)
                parts.append(torch.zeros(ids.shape[0], cat.num_buckets, device=ids.device)
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
        for c in self.columns:
            if isinstance(c, SharedEmbeddingColumn):
                raise ValueError(f"a linear model does not take shared embedding columns, got {c!r}")
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
