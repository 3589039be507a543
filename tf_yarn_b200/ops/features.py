"""Host side of ``tfy_feature_ids`` and ``tfy_vocab_ids`` (ops/csrc/tfy_features.cu): the int64 [T, B, L_max] bucket
ids of a tower's categorical columns -- identity, hashed, bucketized, crossed and vocabulary, in any mix -- computed on
the device from the raw features, one launch per kFeatMaxCols columns / kFeatMaxComps components, after one vocabulary
launch per kVocabMaxSrcs vocabulary sources."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Sequence

import torch

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import native

MAX_COLS, MAX_COMPS = 32, 64                   # kFeatMaxCols / kFeatMaxComps of tfy_features.cuh
MAX_VOCAB_SRCS = 32                            # kVocabMaxSrcs
RAW, IDENTITY, HASHED, BUCKETIZED = 0, 1, 2, 3
I32, I64, F32 = 0, 1, 2


class FeatComp(ctypes.Structure):
    """Mirror of TfyFeatComp (ops/csrc/tfy_features.cuh)."""
    _fields_ = [("src", ctypes.c_uint64), ("modulus", ctypes.c_int64), ("kind", ctypes.c_int32),
                ("dtype", ctypes.c_int32), ("width", ctypes.c_int32), ("n_bounds", ctypes.c_int32),
                ("bounds_off", ctypes.c_int32), ("pad", ctypes.c_int32)]


class FeatCol(ctypes.Structure):
    """Mirror of TfyFeatCol."""
    _fields_ = [("hash_key", ctypes.c_uint64), ("V", ctypes.c_int64), ("comp0", ctypes.c_int32),
                ("n_comps", ctypes.c_int32), ("L", ctypes.c_int32), ("crossed", ctypes.c_int32)]


class FeatureParams(ctypes.Structure):
    """Mirror of TfyFeatureParams."""
    _fields_ = [("out", ctypes.c_uint64), ("bounds", ctypes.c_uint64), ("B", ctypes.c_int32), ("L_max", ctypes.c_int32),
                ("T", ctypes.c_int32), ("n_comps", ctypes.c_int32), ("cols", FeatCol * MAX_COLS),
                ("comps", FeatComp * MAX_COMPS)]


class VocabSrc(ctypes.Structure):
    """Mirror of TfyVocabSrc."""
    _fields_ = [("src", ctypes.c_uint64), ("out", ctypes.c_uint64), ("keys", ctypes.c_uint64), ("ids", ctypes.c_uint64),
                ("n", ctypes.c_int32), ("n_oov", ctypes.c_int32), ("dflt", ctypes.c_int32), ("dtype", ctypes.c_int32),
                ("width", ctypes.c_int32), ("pad", ctypes.c_int32)]


class VocabParams(ctypes.Structure):
    """Mirror of TfyVocabParams."""
    _fields_ = [("B", ctypes.c_int32), ("S", ctypes.c_int32), ("srcs", VocabSrc * MAX_VOCAB_SRCS)]


native.declare("tfy_feature_ids", [ctypes.POINTER(FeatureParams), ctypes.c_void_p])
native.declare("tfy_vocab_ids", [ctypes.POINTER(VocabParams), ctypes.c_void_p])


def _leaves(col) -> List:
    """The components of a column: itself, or a cross's leaf keys."""
    return list(col.keys) if isinstance(col, fc.CrossedColumn) else [col]


class FeatureIds:
    """The id computation of one group of columns, its descriptors fixed at construction (the source pointers and
    widths are filled per batch).  The group's boundaries live in one fp32 device tensor owned by this object.  Its
    vocabularies are each Vocabulary's own device copy (sorted int64 keys, int32 ids), which every group, column and
    the torch statement on that device share; this object holds references to them.

    A vocabulary column -- bare, weighted or a cross's leaf -- is a source of the vocabulary launches: they translate
    its raw values into an int64 buffer, which the id launches then read as an identity component of modulus
    num_buckets.  Sources are keyed by column (its feature and vocabulary), so a raw cross leaf and a vocabulary
    column over the same feature stay apart."""

    def __init__(self, cols: Sequence, device):
        self.cols = list(cols)
        bounds: List[float] = []
        self.vocab_cols: List = []   # the vocabulary sources, in order of first use
        vocab_index: Dict = {}
        self._comps = []            # per column: [(source, kind, modulus, n_bounds, bounds_off, leaf key)], the source
        for c in self.cols:         # a feature name, or the index of a vocabulary source
            comps = []
            for k in _leaves(c):
                base = k.categorical_column if isinstance(k, fc.WeightedCategoricalColumn) else k
                if isinstance(k, str):
                    comps.append((k, RAW, 0, 0, 0, k))
                elif isinstance(k, fc.BucketizedColumn):
                    comps.append((k.source_column.key, BUCKETIZED, 0, len(k.boundaries), len(bounds), k))
                    bounds.extend(k.boundaries)
                elif isinstance(base, fc.VocabularyColumn):
                    j = vocab_index.setdefault(base, len(self.vocab_cols))
                    if j == len(self.vocab_cols):
                        self.vocab_cols.append(base)
                    comps.append((j, IDENTITY, base.num_buckets, 0, 0, base))
                else:                # identity or hashed (a weighted column's ids are its categorical column's)
                    comps.append((k.key, HASHED if k.hashed else IDENTITY, k.num_buckets, 0, 0, k))
            self._comps.append(comps)
        self.bounds = torch.tensor(bounds or [0.0], dtype=torch.float32, device=device)
        self.vocab_tables: List = []     # per source: (keys, ids) on the device, kept alive here
        self.vocab_params: List[VocabParams] = []
        if self.vocab_cols:
            self._install_vocabularies(device)
        # launches: runs of columns within both caps
        self.chunks: List[List[int]] = [[]]
        n = 0
        for t, comps in enumerate(self._comps):
            if len(comps) > MAX_COMPS:
                raise ValueError(f"column {self.cols[t].key!r} crosses {len(comps)} keys; at most {MAX_COMPS} are "
                                 f"supported")
            if len(self.chunks[-1]) == MAX_COLS or n + len(comps) > MAX_COMPS:
                self.chunks.append([])
                n = 0
            self.chunks[-1].append(t)
            n += len(comps)
        self.params = [self._static_params(chunk) for chunk in self.chunks]

    def _install_vocabularies(self, device) -> None:
        """The static part of the vocabulary launches' descriptors, pointing at each vocabulary's device copy (uploaded
        here on its first use on this device)."""
        self.vocab_tables = [c.vocabulary.tables(device) for c in self.vocab_cols]
        for j0 in range(0, len(self.vocab_cols), MAX_VOCAB_SRCS):
            p = VocabParams()
            chunk = self.vocab_cols[j0:j0 + MAX_VOCAB_SRCS]
            p.S = len(chunk)
            for s, c, (keys, ids) in zip(p.srcs, chunk, self.vocab_tables[j0:j0 + MAX_VOCAB_SRCS]):
                s.keys, s.ids = keys.data_ptr(), ids.data_ptr()
                s.n, s.n_oov, s.dflt = len(c.vocabulary), c.num_oov_buckets, c.default_value
            self.vocab_params.append(p)

    @property
    def launches(self) -> int:
        return len(self.vocab_params) + len(self.chunks)

    def _static_params(self, chunk: List[int]) -> FeatureParams:
        p = FeatureParams()
        p.bounds = self.bounds.data_ptr()
        p.T = len(chunk)
        q = 0
        for i, t in enumerate(chunk):
            c = self.cols[t]
            col = p.cols[i]
            col.V, col.comp0, col.n_comps = c.num_buckets, q, len(self._comps[t])
            col.crossed = int(isinstance(c, fc.CrossedColumn))
            col.hash_key = c.hash_key % 2 ** 64 if col.crossed else 0
            for key, kind, modulus, n_bounds, off, _ in self._comps[t]:
                comp = p.comps[q]
                comp.kind, comp.modulus, comp.n_bounds, comp.bounds_off = kind, modulus, n_bounds, off
                comp.dtype = F32 if kind == BUCKETIZED else I64
                q += 1
        p.n_comps = q
        return p

    def __call__(self, features: Dict[str, torch.Tensor], lib) -> torch.Tensor:
        """int64 [T, B, L_max] ids of the batch (-1 = missing or padding), computed on the current stream."""
        out, srcs = self.prepare(features)
        stream = torch.cuda.current_stream().cuda_stream
        for p in self.vocab_params:                  # the translated vocabulary sources first
            native.check(lib.tfy_vocab_ids(ctypes.byref(p), stream), "tfy_vocab_ids")
        for p in self.params:
            native.check(lib.tfy_feature_ids(ctypes.byref(p), stream), "tfy_feature_ids")
        del srcs                                      # stream-ordered frees: the launches are enqueued
        return out

    def prepare(self, features: Dict[str, torch.Tensor]):
        """The output tensor and the sources (kept alive by the caller until the launches are enqueued), with every
        launch's parameters (self.vocab_params, then self.params) pointing at them."""
        srcs: Dict[tuple, torch.Tensor] = {}         # one flattened source per (feature or vocabulary source, bucketized)
        translated = self._prepare_vocabularies(features, srcs)
        widths = []
        for comps in self._comps:
            w = []
            for key, kind, *_, leaf in comps:
                if isinstance(key, int):            # a vocabulary source's int64 ids
                    t = translated[key]
                else:
                    t = features[key]
                    t = t.reshape(t.shape[0], -1)
                if kind == BUCKETIZED:          # k values per example, or its ids would leave [0, num_buckets)
                    fc._check_source_width(leaf, t.shape[1])
                    t = t.float()
                elif t.dtype not in (torch.int32, torch.int64):
                    t = t.long()
                srcs[(key, kind == BUCKETIZED)] = t.contiguous()
                w.append(t.shape[1])
            widths.append(w)
        B = next(iter(srcs.values())).shape[0]
        Ls = []
        for w in widths:
            n = 1
            for x in w:
                n *= x
            Ls.append(n)
        L_max = max(Ls)
        out = torch.empty((len(self.cols), B, L_max), dtype=torch.int64, device=self.bounds.device)
        t0 = 0
        for chunk, p in zip(self.chunks, self.params):
            p.out = out.data_ptr() + t0 * B * L_max * 8
            p.B, p.L_max = B, L_max
            q = 0
            for i, t in enumerate(chunk):
                p.cols[i].L = Ls[t]
                for (key, kind, *_), w in zip(self._comps[t], widths[t]):
                    src = srcs[(key, kind == BUCKETIZED)]
                    p.comps[q].src = src.data_ptr()
                    p.comps[q].width = w
                    if kind != BUCKETIZED:
                        p.comps[q].dtype = I32 if src.dtype == torch.int32 else I64
                    q += 1
            t0 += len(chunk)
        return out, srcs

    def _prepare_vocabularies(self, features: Dict[str, torch.Tensor], srcs: Dict) -> List[torch.Tensor]:
        """The [B, width] int64 ids of every vocabulary source, views of one buffer the vocabulary launches write, with
        their raw sources (kept in srcs) and output pointers filled into self.vocab_params."""
        if not self.vocab_cols:
            return []
        raws = []
        for j, c in enumerate(self.vocab_cols):
            t = features[c.key]
            t = t.reshape(t.shape[0], -1)
            if t.dtype not in (torch.int32, torch.int64):
                t = t.long()
            raws.append(t.contiguous())
            srcs[("vocab", j)] = raws[-1]
        B = raws[0].shape[0]
        buf = torch.empty(sum(B * r.shape[1] for r in raws), dtype=torch.int64, device=self.bounds.device)
        srcs[("vocab", None)] = buf
        out, off = [], 0
        for j, r in enumerate(raws):
            w = r.shape[1]
            out.append(buf[off:off + B * w].view(B, w))
            p = self.vocab_params[j // MAX_VOCAB_SRCS]
            s = p.srcs[j % MAX_VOCAB_SRCS]
            s.src, s.out, s.width = r.data_ptr(), out[-1].data_ptr(), w
            s.dtype = I32 if r.dtype == torch.int32 else I64
            p.B = B
            off += B * w
        return out
