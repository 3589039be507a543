"""Host side of ``tfy_feature_ids`` (ops/csrc/tfy_features.cu): the int64 [T, B, L_max] bucket ids of a tower's
categorical columns -- identity, hashed, bucketized and crossed, in any mix -- computed on the device from the raw
features, one launch per kFeatMaxCols columns / kFeatMaxComps components."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Sequence

import torch

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import native

MAX_COLS, MAX_COMPS = 32, 64                   # kFeatMaxCols / kFeatMaxComps of tfy_features.cuh
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


native.declare("tfy_feature_ids", [ctypes.POINTER(FeatureParams), ctypes.c_void_p])


def _leaves(col) -> List:
    """The components of a column: itself, or a cross's leaf keys."""
    return list(col.keys) if isinstance(col, fc.CrossedColumn) else [col]


class FeatureIds:
    """The id computation of one group of columns, its descriptors fixed at construction (the source pointers and
    widths are filled per batch).  The group's boundaries live in one fp32 device tensor owned by this object."""

    def __init__(self, cols: Sequence, device):
        self.cols = list(cols)
        bounds: List[float] = []
        self._comps = []            # per column: [(feature key, kind, modulus, n_bounds, bounds_off, leaf key)]
        for c in self.cols:
            comps = []
            for k in _leaves(c):
                if isinstance(k, str):
                    comps.append((k, RAW, 0, 0, 0, k))
                elif isinstance(k, fc.BucketizedColumn):
                    comps.append((k.source_column.key, BUCKETIZED, 0, len(k.boundaries), len(bounds), k))
                    bounds.extend(k.boundaries)
                else:                # identity or hashed (a weighted column's ids are its categorical column's)
                    comps.append((k.key, HASHED if k.hashed else IDENTITY, k.num_buckets, 0, 0, k))
            self._comps.append(comps)
        self.bounds = torch.tensor(bounds or [0.0], dtype=torch.float32, device=device)
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

    @property
    def launches(self) -> int:
        return len(self.chunks)

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
        for p in self.params:
            native.check(lib.tfy_feature_ids(ctypes.byref(p), stream), "tfy_feature_ids")
        del srcs                                      # stream-ordered frees: the launches are enqueued
        return out

    def prepare(self, features: Dict[str, torch.Tensor]):
        """The output tensor and the sources (kept alive by the caller until the launches are enqueued), with every
        launch's parameters (self.params) pointing at them."""
        srcs: Dict[tuple, torch.Tensor] = {}         # one flattened source per (feature, bucketized)
        widths = []
        for comps in self._comps:
            w = []
            for key, kind, *_, leaf in comps:
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
