"""H100 data plane of the asynchronous parameter server: shards in the ps ranks' HBM.

Every task of the training cluster (chief, workers AND ps) joins one symmetric arena
(:mod:`tf_yarn_b200.parallel.symm`, rendezvous through the launcher's KV store).  A ps rank's
shard is a region of ITS arena; chief/workers reach it through the peer mapping over NVLink:

* dense pull   : ``tfy_ps_pull`` -- peer fp32 master -> local replica, ONE launch for the variables that need a
  local copy (biases, small vectors); Dense weights and embedding rows are never copied;
* GEMM pull    : the weight matrix of a Dense layer stays on the ps rank: its row-padded bf16 shadow is streamed
  by TMA into the wgmma GEMM that consumes it (forward ``tfy_gemm_bf16``, backward ``tfy_dense_bwd``: dW and
  dx in one kernel against the same remote shadow);
* sparse pull  : ``tfy_ps_embedding_bag`` / ``tfy_ps_multi_bag`` (all tables of a tower in one launch); for the
  first deep layer the gather IS the A-operand producer of the GEMM (K5, ``tfy_ps_gather_gemm``);
* push         : ``tfy_ps_push`` / ``tfy_ps_push_rows`` / ``tfy_ps_multi_push_rows`` -- gradients applied to the peer
  master with vector red/atom and the variable's own optimizer fused (SGD, Adagrad, Adam, FTRL), asynchronously
  and without locks (K6); row gradients are pushed straight out of column slices of the fused layer's dx.

The ps process only owns memory and waits for the stop barrier: no server thread is on the data path.
Control state (layout, readiness, global step) stays on the KV store / a shared-memory header, as in
the CPU data plane (:mod:`tf_yarn_b200.estimator.ps`).
"""
from __future__ import annotations

import ctypes
import logging
import os
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from tf_yarn_b200 import _task_commons
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.estimator import ps as ps_cpu
from tf_yarn_b200.ops import features as feature_ids
from tf_yarn_b200.ops import native
from tf_yarn_b200.parallel.symm import _RawCudaMemory

logger = logging.getLogger(__name__)

_vp, _i, _sz, _f, _ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float, ctypes.c_longlong
native.declare("tfy_ps_pull", [_vp, _i, _sz, _i, _vp])
native.declare("tfy_ps_push", [_vp, _i, _sz, _i, _f, _vp, _vp])
native.declare("tfy_ps_refresh_shadow", [_vp, _i, _sz, _vp])
native.declare("tfy_dense_bwd", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_ps_embedding_bag", [_vp, _vp, _vp, _i, _i, _i, _i, _ll, _i, _vp])
native.declare("tfy_ps_push_rows_scratch_bytes", [_ll], _sz)
native.declare("tfy_ps_push_rows", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _i, _i, _f, _f, _f, _f, _f, _f, _vp,
                                    _i, _vp, _sz, _vp])
native.declare("tfy_ps_multi_bag", [_vp, _vp, _vp, _i, _i, _i, _i, _ll, _vp])
native.declare("tfy_ps_multi_push_rows", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _i, _f, _f, _f, _f, _f, _f, _vp, _i,
                                          _i, _vp, _sz, _vp])
native.declare("tfy_ps_gather_gemm", [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _vp])
native.declare("tfy_ps_multi_bag_weighted", [_vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _vp, _i, _i, _i, _vp, _i, _vp,
                                             _vp])
native.declare("tfy_ps_multi_push_rows_weighted", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _i, _f, _f, _f, _f, _f,
                                                   _f, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _sz, _vp])
native.declare("tfy_ps_multi_push_rows_shared", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _i, _f, _f, _f, _f, _f,
                                                 _f, _vp, _i, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _sz, _vp])

OPT_CODES = {"sgd": native.OPT_SGD, "adagrad": native.OPT_ADAGRAD, "adam": native.OPT_ADAM,
             "ftrl": native.OPT_FTRL}
COMBINER_CODES = {"sum": 0, "mean": 1, "sqrtn": 2}      # tfy_ps_multi_bag_weighted / tfy_ps_multi_push_rows_weighted
SUM, MEAN = COMBINER_CODES["sum"], COMBINER_CODES["mean"]


class PsSeg(ctypes.Structure):
    """Mirror of TfyPsSeg (ops/csrc/tfy_ps.cu): one variable of a push / pull, with ITS optimizer."""
    _fields_ = [("remote_w", ctypes.c_uint64), ("remote_s1", ctypes.c_uint64), ("remote_s2", ctypes.c_uint64),
                ("remote_shadow", ctypes.c_uint64), ("local", ctypes.c_uint64), ("n", ctypes.c_uint64),
                ("opt", ctypes.c_int32), ("lr", ctypes.c_float), ("eps", ctypes.c_float), ("wd", ctypes.c_float),
                ("p1", ctypes.c_float), ("p2", ctypes.c_float), ("p3", ctypes.c_float), ("pad", ctypes.c_int32),
                ("cols", ctypes.c_uint32), ("shadow_ld", ctypes.c_uint32)]


def push_rows_launches(per_table: int, max_members: int = 0) -> int:
    """Kernel launches of one sparse push of `per_table` ids per column: a per-table block sort (up to 2048 ids per
    table, tfy_ps.cu kPsBlockSortMax) or the key kernel and CUB's device radix sort (histogram, scan and one kernel
    per 8-bit pass, counted here as one launch), then the short-run and long-run apply kernels.  A shared push
    (tfy_ps_multi_push_rows_shared, max_members > 0 = the most columns any one table has) takes the block sort when
    max_members * per_table <= 2048, and runs one more kernel: the per-occurrence gradient offsets, which also write
    a weighted push's factors."""
    if not max_members:
        return 3 if per_table <= 2048 else 4
    return (3 if per_table * max_members <= 2048 else 4) + 1


def push_rows_scratch(lib, n: int, device) -> torch.Tensor:
    """Device scratch of a sparse push of n ids (tfy_ps_push_rows / tfy_ps_multi_push_rows fold duplicates in it).
    Allocated per push from the caching allocator, so a captured CUDA graph keeps its own."""
    nbytes = int(lib.tfy_ps_push_rows_scratch_bytes(n)) if n > 0 else 0
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return t.data_ptr() if t is not None else None


def weighted_bag(lib, tables: torch.Tensor, ids: torch.Tensor, weights: Optional[torch.Tensor], combiner: int, D: int,
                 V: int, out: torch.Tensor, out_ld: int, col_stride: int, f: torch.Tensor,
                 numeric: Optional[torch.Tensor] = None) -> None:
    """tfy_ps_multi_bag_weighted: ids int64 [T, B, L] (-1 = missing), weights fp32 [T, B, L] or None, f fp32 [T, B]
    receives 1/den for the push."""
    T, B, L = ids.shape
    n_num = numeric.shape[1] if numeric is not None else 0
    native.check(lib.tfy_ps_multi_bag_weighted(tables.data_ptr(), ids.data_ptr(), _ptr(weights), combiner, B, L, T, D,
                                               V, out.data_ptr(), int(out.dtype == torch.bfloat16), out_ld, col_stride,
                                               _ptr(numeric), n_num, f.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream), "tfy_ps_multi_bag_weighted")


def cluster_ranks(cluster) -> Dict[str, int]:
    """Global rank of every cluster task in the symmetric arena: chief, workers, then ps."""
    keys = cluster.trainers() + [f"ps:{i}" for i in range(len(cluster.spec.get("ps", [])))]
    return {k: r for r, k in enumerate(keys)}


def join_arena(cluster):
    """Create this process's Communicator over ALL cluster tasks (collective: every task calls it)."""
    from tf_yarn_b200.parallel import runtime
    ranks = cluster_ranks(cluster)
    me = f"{cluster.task_type}:{cluster.task_id}"
    os.environ["TFY_RANK"] = str(ranks[me])
    os.environ["TFY_WORLD_SIZE"] = str(len(ranks))
    ids = [int(v) for v in os.environ.get("TFY_GPU_IDS", "").split(",") if v.strip() != ""]
    dev = ids[0] if ids else ranks[me] % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    return runtime.get_communicator(device=dev), ranks


def shard_bytes(layout: ps_cpu.Layout) -> int:
    """Bytes every rank reserves in its arena (the largest shard; fp32 master+slots, then bf16 shadows)."""
    worst = 0
    for ps in range(layout.n_ps):
        elems = layout.shard_elems[ps]
        rows = sum(int(s[0]) for (_, s), o in zip(layout.variables, layout.owner) if o == ps and len(s) == 2)
        worst = max(worst, elems * 4 + elems * 2 + rows * 16 + 4096)       # fp32 area + (row-padded) bf16 shadows
    return (worst + 4095) // 4096 * 4096


class HbmConnection:
    """Chief / worker view of the HBM shards."""

    def __init__(self, layout: ps_cpu.Layout, comm, ranks: Dict[str, int], region_off: int, names: List[str],
                 header: ps_cpu.ShmShard, network: nn.Module):
        self.layout, self.names, self.header = layout, names, header
        self.lib = native.load()
        bad = sorted({k for k in layout.kinds if k not in OPT_CODES})
        if bad:
            raise ValueError(f"the HBM parameter server fuses SGD, Adagrad, Adam and FTRL; got {bad}")
        self.var_opt = [OPT_CODES[k] for k in layout.kinds]
        arena = comm.arena
        self.ps_base = [arena.peer_base[ranks[f"ps:{i}"]] + region_off for i in range(layout.n_ps)]
        dev = torch.device(f"cuda:{comm.device}")
        self.device = dev
        params = dict(network.named_parameters())
        self.params = [params[n] for n in names]
        self.sparse: Dict[int, nn.Module] = {}      # variable index -> EmbeddingBag served sparsely
        self.gemm: Dict[int, nn.Module] = {}        # variable index -> Linear whose weight stays remote
        self._classify(network)
        self.dense_idx = [i for i in range(len(names)) if i not in self.sparse]
        # Dense-layer weights served by the remote-weight GEMMs are NEVER copied to the worker: forward streams
        # the ps rank's bf16 shadow through TMA, backward (dW, dx) reads the same shadow (tfy_dense_bwd)
        self.pull_idx = [i for i in self.dense_idx if i not in self.gemm]
        self._pull_segs = self._make_segs(for_push=False, idx=self.pull_idx)
        self._push_segs = None
        self._push_ptrs = None
        self._max_n = max([self._n4(i) for i in self.dense_idx] + [4])
        # Adam bias correction {1/(1-b1^t), 1/sqrt(1-b2^t)}: device scalars the push kernels read, refreshed from the
        # global step before every push (so a captured CUDA graph sees them advance)
        self._adam = [i for i, k in enumerate(layout.kinds) if k == "adam"]
        self.adam_scale = torch.ones(2, dtype=torch.float32, device=dev)
        self._adam_host = torch.ones(2, dtype=torch.float32).pin_memory() if self._adam else None
        # NVLink traffic / kernel launches of one step, counted on the host while a step runs eagerly (the
        # captured graph replays exactly the same launches)
        self._acct = {"pull_bytes": 0, "push_bytes": 0, "launches_per_step": 0}
        self._acct_last = dict(self._acct)

    # ------------------------------------------------------------------ addressing
    def _n4(self, i: int) -> int:
        return (self.layout.numel[i] + 3) // 4 * 4

    def master_ptr(self, i: int, slot: int = 0) -> int:
        lay = self.layout
        return self.ps_base[lay.owner[i]] + 4 * (lay.offset[i] + slot * lay.padded(i))

    def shadow_ptr(self, i: int) -> int:
        """bf16 shadow of variable i: the shadows of a ps follow its fp32 area (master + slots)."""
        lay = self.layout
        ps = lay.owner[i]
        return self.ps_base[ps] + 4 * lay.shard_elems[ps] + 2 * self._shadow_off(i)

    def shadow_ld(self, i: int) -> int:
        """Row pitch (elements) of variable i's bf16 shadow: 2-D weights are stored with rows padded to a multiple
        of 8 elements so that a TMA tensor map can describe them whatever in_features is (0 = flat)."""
        shape = self.layout.variables[i][1]
        return (int(shape[1]) + 7) // 8 * 8 if len(shape) == 2 else 0

    def _shadow_elems(self, i: int) -> int:
        shape = self.layout.variables[i][1]
        ld = self.shadow_ld(i)
        return (int(shape[0]) * ld + 7) // 8 * 8 if ld else self.layout.padded(i)

    def _shadow_off(self, i: int) -> int:
        """Element offset of variable i inside its ps's bf16 shadow area (layout order)."""
        lay = self.layout
        off = 0
        for j in range(i):
            if lay.owner[j] == lay.owner[i]:
                off += self._shadow_elems(j)
        return off

    def remote_tensor(self, i: int, slot: int = 0) -> torch.Tensor:
        """Zero-copy torch view of a peer region (used for initialisation and checkpoints)."""
        n = self.layout.numel[i]
        mem = _RawCudaMemory(self.master_ptr(i, slot), n * 4, self)
        return torch.as_tensor(mem, device=self.device).view(torch.float32)

    def _classify(self, network: nn.Module) -> None:
        by_param = {id(p): i for i, p in enumerate(self.params)}
        for mod in network.modules():
            if isinstance(mod, nn.EmbeddingBag) and id(mod.weight) in by_param and mod.mode in ("sum", "mean"):
                self.sparse[by_param[id(mod.weight)]] = mod
            elif isinstance(mod, nn.Linear) and id(mod.weight) in by_param and mod.out_features >= 8 \
                    and mod.out_features % 8 == 0:
                self.gemm[by_param[id(mod.weight)]] = mod

    def _make_segs(self, for_push: bool, idx: Optional[List[int]] = None):
        idx = self.dense_idx if idx is None else idx
        segs = (PsSeg * max(1, len(idx)))()
        for k, i in enumerate(idx):
            p = self.params[i]
            h = self.layout.hypers[i]
            segs[k].remote_w = self.master_ptr(i)
            segs[k].remote_s1 = self.master_ptr(i, 1) if self.layout.var_slots[i] >= 1 else 0
            segs[k].remote_s2 = self.master_ptr(i, 2) if self.layout.var_slots[i] >= 2 else 0
            segs[k].remote_shadow = self.shadow_ptr(i) if i in self.gemm else 0
            segs[k].local = (p.grad.data_ptr() if for_push else p.data_ptr())
            segs[k].n = self.layout.numel[i]
            segs[k].opt, segs[k].lr, segs[k].eps, segs[k].p1, segs[k].p2, segs[k].p3 = self.push_hypers(i)
            segs[k].wd = float(h["wd"])
            ld = self.shadow_ld(i) if i in self.gemm else 0
            segs[k].cols = int(self.layout.variables[i][1][1]) if ld else 0
            segs[k].shadow_ld = ld
        dev_segs = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).to(self.device)
        return dev_segs

    def push_hypers(self, i: int) -> tuple:
        """(opt, lr, eps, p1, p2, p3) of variable i as every push kernel takes them.  FTRL: l1, l2, beta in p1, p2,
        p3 (OptimizerSpec.ftrl keeps beta in eps) | Adam: beta1, beta2 in p1, p2."""
        h = self.layout.hypers[i]
        p3 = float(h["eps"]) if self.layout.kinds[i] == "ftrl" else 0.0
        return self.var_opt[i], float(h["lr"]), float(h["eps"]), float(h["p1"]), float(h["p2"]), p3

    # ------------------------------------------------------------------ install the fused ops
    def install(self, network: nn.Module) -> None:
        """Route EmbeddingBag / Linear modules through the peer-memory kernels."""
        conn = self
        for idx, mod in self.sparse.items():
            mod.forward = _make_bag_forward(conn, idx, mod)
        for idx, mod in self.gemm.items():
            mod.forward = _make_linear_forward(conn, idx, mod)
        self.fused_first = _try_fuse_first_layer(conn, network)
        self.fused_wide = _try_fuse_wide_tower(conn, network)
        self.shared_collections = _serve_shared_collections(
            conn, network, k5_features=getattr(network, "dense_features", None) if self.fused_first else None)

    # ------------------------------------------------------------------ pull / push
    def pull(self, network: nn.Module) -> None:
        """Dense pull of the variables that need a local replica (biases, small vectors): ONE launch of peer
        loads.  Embedding rows and Dense weights are not pulled (gathered / streamed by their consumers)."""
        self._acct = {"pull_bytes": 0, "push_bytes": 0, "launches_per_step": 0}      # a step starts with the pull
        if not self.pull_idx:
            return
        native.check(self.lib.tfy_ps_pull(self._pull_segs.data_ptr(), len(self.pull_idx), self._max_n, 0,
                                          torch.cuda.current_stream().cuda_stream), "tfy_ps_pull")
        self.account(pull=sum(self.layout.numel[i] * 4 for i in self.pull_idx))

    def account(self, pull: int = 0, push: int = 0, launches: int = 1) -> None:
        a = self._acct
        a["pull_bytes"] += pull
        a["push_bytes"] += push
        a["launches_per_step"] += launches

    def traffic_per_step(self) -> dict:
        """Bytes read from / written to the ps ranks over NVLink and kernels launched by the last eager step."""
        return dict(self._acct_last)

    def push(self, network: nn.Module) -> None:
        if not self.dense_idx:
            return
        for i in self.dense_idx:
            p = self.params[i]
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        ptrs = tuple(self.params[i].grad.data_ptr() for i in self.dense_idx)
        if self._push_segs is None or self._push_ptrs != ptrs:     # gradients normally keep their address
            self._push_segs, self._push_ptrs = self._make_segs(for_push=True), ptrs
        segs = self._push_segs
        native.check(self.lib.tfy_ps_push(segs.data_ptr(), len(self.dense_idx), self._max_n, 0, 1.0,
                                          self.adam_scale.data_ptr(), torch.cuda.current_stream().cuda_stream),
                     "tfy_ps_push")
        # per element: gradient applied to master (+ slots read-modify-written) on the peer
        self.account(push=sum(self.layout.numel[i] * 4 * (1 + self.layout.var_slots[i]) for i in self.dense_idx))
        self._acct_last = dict(self._acct)

    def refresh_adam_scale(self) -> None:
        """Bias correction of the asynchronous Adam from the shared global step (host side, outside any graph)."""
        if not self._adam:
            return
        h = self.layout.hypers[self._adam[0]]
        t = max(self.global_step(), 0) + 1
        self._adam_host[0] = 1.0 / (1.0 - h["p1"] ** t)
        self._adam_host[1] = 1.0 / (1.0 - h["p2"] ** t) ** 0.5
        self.adam_scale.copy_(self._adam_host, non_blocking=True)

    def refresh_shadows(self) -> None:
        segs = self._make_segs(for_push=False)
        native.check(self.lib.tfy_ps_refresh_shadow(segs.data_ptr(), len(self.dense_idx), self._max_n,
                                                    torch.cuda.current_stream().cuda_stream), "tfy_ps_refresh_shadow")
        torch.cuda.current_stream().synchronize()

    # ------------------------------------------------------------------ global step / checkpoints
    def increment_global_step(self) -> int:
        return self.header.add_global_step(1)

    def global_step(self) -> int:
        return self.header.global_step()

    def state_dict_from_ps(self, network: nn.Module) -> Dict[str, torch.Tensor]:
        torch.cuda.synchronize()
        with torch.no_grad():
            for i, p in enumerate(self.params):
                p.copy_(self.remote_tensor(i).view(p.shape))
        return network.state_dict()

    def optimizer_state(self) -> Dict[str, dict]:
        """Every variable's optimizer slots, read from the ps ranks (ps.export_slots).  The bf16 shadows are derived
        from the masters and are not part of it."""
        torch.cuda.synchronize()
        return ps_cpu.export_slots(self.layout, self.remote_tensor)


def _make_bag_forward(conn: HbmConnection, idx: int, mod: nn.EmbeddingBag):
    combiner = getattr(mod, "combiner", mod.mode)
    group = _TableGroup(conn, [idx], [fc.CategoricalColumn("", mod.num_embeddings)], mod.embedding_dim,
                        combiners=[COMBINER_CODES[combiner]], one_table=True)
    anchor = torch.zeros((), device=conn.device, requires_grad=True)

    def run(ids, weights):
        ids = ids.contiguous().long()
        if ids.dim() == 1:
            ids = ids[:, None]
        if weights is None and ids.shape[1] == 1 and combiner in ("sum", "mean"):
            return _Lookup.apply(group, ids.reshape(1, -1), None, anchor)     # one id per example: the one-table kernels
        if weights is not None:
            weights = weights.contiguous().float().reshape(ids.shape[0], -1)
            if weights.shape != ids.shape:
                raise ValueError(f"weights {tuple(weights.shape)} do not match ids {tuple(ids.shape)}")
            weights = weights[None]
        return _Lookup.apply(group, ids[None], weights, anchor)     # multi-hot, weighted or sqrtn: the weighted bag

    if isinstance(mod, fc.CombinedBag):
        def forward(ids, weights=None):
            return run(ids, weights)
    else:
        def forward(ids, offsets=None, per_sample_weights=None):
            if offsets is not None:
                raise NotImplementedError("the HBM parameter server serves [B, L] id batches; offsets are not supported")
            if per_sample_weights is not None and mod.mode != "sum":
                raise ValueError("per_sample_weights needs mode='sum' (as for torch.nn.EmbeddingBag)")
            return run(ids, per_sample_weights)
    return forward


def _make_linear_forward(conn: HbmConnection, idx: int, mod: nn.Linear):
    from tf_yarn_b200.ops.gemm import gemm_bf16
    N, K = mod.out_features, mod.in_features
    Kp = conn.shadow_ld(idx)                 # row pitch of the remote bf16 shadow (K rounded up to 8; pad columns = 0)
    shadow = conn.shadow_ptr(idx)

    class _PSLinear(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, weight, bias):
            if Kp == K:
                xb = x.to(torch.bfloat16).contiguous()
            else:                            # TMA needs 16-byte row pitches: zero-pad the activations like the shadow
                xb = torch.zeros((x.shape[0], Kp), dtype=torch.bfloat16, device=x.device)
                xb[:, :K] = x
            y = gemm_bf16(xb, None, bias=bias.to(torch.bfloat16) if bias is not None else None, b_ptr=shadow,
                          b_rows=N, b_ld=Kp, impl="1cta")       # weights stream from the ps rank over NVLink
            conn.account(pull=N * Kp * 2)
            ctx.save_for_backward(xb, weight)
            ctx.has_bias = bias is not None
            return y.to(x.dtype)

        @staticmethod
        def backward(ctx, dy):
            xb, weight = ctx.saved_tensors
            B = xb.shape[0]
            dyb = dy.to(torch.bfloat16).contiguous()
            dw = torch.empty((N, Kp), dtype=torch.bfloat16, device=dy.device)
            dx = torch.empty((B, Kp), dtype=torch.bfloat16, device=dy.device) if ctx.needs_input_grad[0] else None
            # dW = dy^T x and dx = dy W in one wgmma kernel; W is the ps rank's bf16 shadow, read over NVLink
            native.check(conn.lib.tfy_dense_bwd(dyb.data_ptr(), xb.data_ptr(), shadow, dw.data_ptr(),
                                                dx.data_ptr() if dx is not None else None, B, N, Kp,
                                                torch.cuda.current_stream().cuda_stream), "tfy_dense_bwd")
            conn.account(pull=N * Kp * 2 if dx is not None else 0)
            db = dy.float().sum(0) if ctx.has_bias else None
            gx = dx[:, :K].to(dy.dtype) if dx is not None else None
            return gx, dw[:, :K].to(weight.dtype), db

    def forward(x):
        return _PSLinear.apply(x, mod.weight, mod.bias)
    return forward


def _rows(x: Optional[torch.Tensor], rows) -> Optional[torch.Tensor]:
    """x[rows] (a slice: a view; a list of rows: a contiguous copy), or None."""
    if x is None:
        return None
    return x[rows] if isinstance(rows, slice) else x[rows].contiguous()


class _TableGroup:
    """T embedding columns of one consumer, looked up by one bag and pushed by one push; the only code that launches
    a sparse bag or push.  Column t looks up the table tables_idx[t]; columns of a shared embedding collection repeat
    their table.  The consumer's output holds column t's D values at columns [t * col_stride, t * col_stride + D) of
    each row, or all columns summed into [0, D) when col_stride is 0; combiners[t] is column t's bag combiner.

    A batch comes as ids int64 [T, B] when every column has one id per example and none is weighted (the one-id
    kernels), else as ids / weights [T, B, L] (the weighted bag).  The kernel serving it:

    * one-id bag: tfy_ps_embedding_bag for a one_table group (an unfused EmbeddingBag), else tfy_ps_multi_bag;
    * weighted bag: tfy_ps_multi_bag_weighted, once per column when the columns' combiners differ;
    * push: tables of mixed optimizers one by one (below); columns sharing tables tfy_ps_multi_push_rows_shared, so
      that each distinct (table, row) is folded and applied once; a weighted bag's push
      tfy_ps_multi_push_rows_weighted; one-id batches tfy_ps_push_rows for a one_table group, else
      tfy_ps_multi_push_rows.
    """

    def __init__(self, conn: HbmConnection, tables_idx: List[int], cat_cols, D: int = 0, col_stride: int = 0,
                 combiners: Optional[List[int]] = None, one_table: bool = False):
        lay = conn.layout
        self.conn, self.idx, self.cols = conn, tables_idx, cat_cols
        self.D, self.col_stride, self.one_table = D, col_stride, one_table
        self.combiners = combiners or [SUM] * len(tables_idx)
        self.out_ld = col_stride * len(tables_idx) if col_stride else D
        first = tables_idx[0]
        self.uniform = all(lay.kinds[i] == lay.kinds[first] and lay.hypers[i] == lay.hypers[first] for i in tables_idx)
        dev = conn.device
        ns = lay.var_slots[first]

        def ptrs(idx, slot):
            return torch.tensor([conn.master_ptr(i, slot) for i in idx], dtype=torch.int64, device=dev)
        # per column: the bags and K5's gather read tables[t]
        self.tables = ptrs(tables_idx, 0)
        self.s1 = ptrs(tables_idx, 1) if ns >= 1 else None
        self.s2 = ptrs(tables_idx, 2) if ns >= 2 else None
        # per distinct table: the shared push's {w, s1, s2} arrays and table_of[t], the index of column t's table.
        # Built from the distinct tables in order of first use, the map meets the kernel's preconditions by
        # construction: every value in [0, n_tables), every table named, none by more than max_members columns.
        self.distinct = list(dict.fromkeys(tables_idx))
        if self.shared:
            table_of = [self.distinct.index(i) for i in tables_idx]
            self.table_of = torch.tensor(table_of, dtype=torch.int32, device=dev)
            self.push_tables = ptrs(self.distinct, 0)
            self.push_s1 = ptrs(self.distinct, 1) if ns >= 1 else None
            self.push_s2 = ptrs(self.distinct, 2) if ns >= 2 else None
            self.max_members = max(table_of.count(k) for k in range(len(self.distinct)))
        # a group with a bucketized, crossed or vocabulary column (also weighted or as a cross's leaf) takes every
        # column's ids from tfy_vocab_ids + tfy_feature_ids (torch on a CPU tensor), which bound each column's ids by
        # its own V: its tables may differ in V, and the bag and push kernels are given the largest
        self.derived = any(fc._device_ids(c) for c in cat_cols)
        self.feature_ids = feature_ids.FeatureIds(cat_cols, conn.device) if self.derived else None
        self.V = max(c.num_buckets for c in cat_cols) if self.derived else cat_cols[0].num_buckets
        self.same_v = not self.derived and all(c.num_buckets == self.V and c.hashed == cat_cols[0].hashed
                                               for c in cat_cols)
        self.hp = conn.push_hypers(first)
        self.slots = ns
        self.parts = None if self.uniform else self.split()

    @property
    def shared(self) -> bool:
        """True when columns share tables: the group then pushes through tfy_ps_multi_push_rows_shared."""
        return len(set(self.idx)) < len(self.idx)

    @property
    def weighted(self) -> bool:
        return any(isinstance(c, fc.WeightedCategoricalColumn) for c in self.cols)

    def one_hot(self, features) -> bool:
        """True when the batch has one id per example in every column ([B] or [B, 1]) and no column is weighted: the
        one-id kernels (K5, tfy_ps_multi_bag) serve it.  Decided from shapes, without a device synchronisation."""
        if self.derived:                # a cross has prod L_k ids per example, a bucketized column k
            return not self.weighted and all(fc._width(c, features) == 1 for c in self.cols)
        return not self.weighted and all(features[c.key].reshape(features[c.key].shape[0], -1).shape[1] == 1
                                         for c in self.cols)

    def ids_of(self, features) -> torch.Tensor:
        """int64 [T, B] bucket ids of the batch (-1 = missing): ONE hash over the stacked columns (26 separate
        3-kernel hashes were 40 % of the step's device time in the first profile)."""
        if self.derived:
            ids = self._derived_ids(features)
            return ids.reshape(ids.shape[0], -1)
        raw = torch.stack([features[c.key].reshape(-1) for c in self.cols]).long()
        return self._bucket(raw)

    def _derived_ids(self, features) -> torch.Tensor:
        """int64 [T, B, L] ids of a group with bucketized, crossed or vocabulary columns, padded with -1: one
        tfy_vocab_ids launch per kVocabMaxSrcs vocabulary sources, then one tfy_feature_ids launch per kFeatMaxCols
        columns, on CUDA tensors; the columns' torch statement on CPU tensors."""
        if self.conn.device.type == "cuda":
            self.conn.account(launches=self.feature_ids.launches)
            return self.feature_ids(features, self.conn.lib)
        ids = [fc._ids_and_weights(c, features)[0] for c in self.cols]
        L = max(i.shape[1] for i in ids)
        return torch.stack([F.pad(i, (0, L - i.shape[1]), value=-1) for i in ids]).contiguous()

    def _bucket(self, raw: torch.Tensor) -> torch.Tensor:
        """feature_column._ids of the stacked columns (the CPU plane's mapping, -1 = missing): one call when the
        columns share V and hashing, else column by column."""
        if self.same_v:
            return fc._ids(self.cols[0], raw).contiguous()
        return torch.stack([fc._ids(c, r) for c, r in zip(self.cols, raw)]).contiguous()

    def multi_of(self, features):
        """int64 [T, B, L] bucket ids (-1 = missing), every column padded on the device to the group's largest L with
        -1, and the
        fp32 [T, B, L] weights (1 for an unweighted column) or None when no column is weighted."""
        if self.derived:
            ids = self._derived_ids(features)
            shapes = [(ids.shape[1], fc._width(c, features)) for c in self.cols]
        else:
            raws = [features[c.key] for c in self.cols]
            raws = [r.reshape(r.shape[0], -1).long() for r in raws]
            L = max(r.shape[1] for r in raws)
            ids = self._bucket(torch.stack([F.pad(r, (0, L - r.shape[1]), value=-1) for r in raws]))
            shapes = [r.shape for r in raws]
        if not self.weighted:
            return ids, None
        L = ids.shape[2]
        ws = []
        for c, shape in zip(self.cols, shapes):
            if isinstance(c, fc.WeightedCategoricalColumn):
                w = fc._weights(c, features, shape).float()
            else:
                w = torch.ones(shape, dtype=torch.float32, device=ids.device)
            ws.append(F.pad(w, (0, L - w.shape[1])))
        return ids, torch.stack(ws).contiguous()

    def split(self):
        """(member columns, group) per distinct table: a mixed-optimizer group pushes table by table."""
        out = []
        for ti in self.distinct:
            members = [t for t, i in enumerate(self.idx) if i == ti]
            shared = len(members) > 1
            out.append((members, _TableGroup(self.conn, [ti] * len(members), [self.cols[t] for t in members], self.D,
                                             self.D if shared else 0, one_table=not shared)))
        return out

    def bag(self, ids: torch.Tensor, weights: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
            out_ld: Optional[int] = None, numeric: Optional[torch.Tensor] = None):
        """Look up a batch into out (fp32 [B, out_ld] allocated when None; the weighted bag writes the numeric
        columns after the embeddings).  Returns out and, for the weighted bag, f fp32 [T, B]: each row's 1/den,
        which its push takes."""
        conn, lib, D, V = self.conn, self.conn.lib, self.D, self.V
        T, B = ids.shape[:2]
        L = ids.shape[2] if ids.dim() == 3 else 1
        out_ld = self.out_ld if out_ld is None else out_ld
        if out is None:
            out = torch.empty((B, out_ld), dtype=torch.float32, device=ids.device)
        f, launches = None, 1
        if ids.dim() == 2 and self.one_table:
            native.check(lib.tfy_ps_embedding_bag(conn.master_ptr(self.idx[0]), ids.data_ptr(), out.data_ptr(), 0, B, L,
                                                  D, V, int(self.combiners[0] == MEAN),
                                                  torch.cuda.current_stream().cuda_stream), "tfy_ps_embedding_bag")
        elif ids.dim() == 2:
            native.check(lib.tfy_ps_multi_bag(self.tables.data_ptr(), ids.data_ptr(), out.data_ptr(), 0, B, T, D, V,
                                              torch.cuda.current_stream().cuda_stream), "tfy_ps_multi_bag")
        else:
            f = torch.empty((T, B), dtype=torch.float32, device=ids.device)
            if len(set(self.combiners)) == 1:
                weighted_bag(lib, self.tables, ids, weights, self.combiners[0], D, V, out, out_ld, self.col_stride, f,
                             numeric)
            else:       # the bag takes one combiner per launch: column by column, numeric after the last
                launches = T
                for t in range(T):
                    weighted_bag(lib, self.tables[t:t + 1], ids[t:t + 1], _rows(weights, slice(t, t + 1)),
                                 self.combiners[t], D, V, out[:, self.col_stride * t:], out_ld, self.col_stride,
                                 f[t:t + 1], numeric if t == T - 1 else None)
        conn.account(pull=T * B * L * D * 4, launches=launches)
        return out, f

    def push(self, ids: torch.Tensor, dout: torch.Tensor, weights: Optional[torch.Tensor] = None,
             f: Optional[torch.Tensor] = None, combiner: int = SUM, dout_ld: Optional[int] = None) -> None:
        """Apply the row gradients of a bag's batch (ids, weights and the bag's f) with each table's optimizer.  dout
        [B, *] is laid out as the bag's output, with row pitch dout_ld (None: the bag's own out_ld).  combiner goes to
        the kernels that take one; with f given it only says that f is."""
        if self.parts is not None:              # mixed optimizers: table by table, each with its member columns
            for members, sub in self.parts:
                if sub.shared:
                    cols = [dout[:, self.col_stride * t:self.col_stride * t + self.D] for t in members]
                    sub.push(_rows(ids, members), torch.cat(cols, dim=1), _rows(weights, members), _rows(f, members),
                             combiner)
                else:
                    t = slice(members[0], members[0] + 1)
                    sub.push(ids[t], dout[:, self.col_stride * members[0]:], _rows(weights, t), _rows(f, t), combiner,
                             self.out_ld if dout_ld is None else dout_ld)
            return
        conn, lib, D, V = self.conn, self.conn.lib, self.D, self.V
        T, B = ids.shape[:2]
        L = ids.shape[2] if ids.dim() == 3 else 1
        ld = self.out_ld if dout_ld is None else dout_ld
        scratch = push_rows_scratch(lib, T * B * L, dout.device)
        hyper = (*self.hp, 1.0, conn.adam_scale.data_ptr())
        tail = (scratch.data_ptr(), scratch.numel(), torch.cuda.current_stream().cuda_stream)
        args = (ids.data_ptr(), dout.data_ptr(), int(dout.dtype == torch.bfloat16), B)
        if self.shared:
            name = "tfy_ps_multi_push_rows_shared"
            rc = lib.tfy_ps_multi_push_rows_shared(
                self.push_tables.data_ptr(), _ptr(self.push_s1), _ptr(self.push_s2), *args, T, D, V, *hyper, ld,
                self.col_stride, L, _ptr(weights), _ptr(f), combiner, len(self.distinct), self.table_of.data_ptr(),
                self.max_members, *tail)
        elif f is not None:
            name = "tfy_ps_multi_push_rows_weighted"
            rc = lib.tfy_ps_multi_push_rows_weighted(self.tables.data_ptr(), _ptr(self.s1), _ptr(self.s2), *args, T, D,
                                                     V, *hyper, ld, self.col_stride, L, _ptr(weights), f.data_ptr(),
                                                     combiner, *tail)
        elif self.one_table:                    # dout_ld 0: rows of D
            name = "tfy_ps_push_rows"
            i = self.idx[0]
            slot = [conn.master_ptr(i, s) if s <= self.slots else None for s in range(3)]
            rc = lib.tfy_ps_push_rows(*slot, *args, L, D, V, int(combiner == MEAN), *hyper, dout_ld or 0, *tail)
        else:
            name = "tfy_ps_multi_push_rows"
            rc = lib.tfy_ps_multi_push_rows(self.tables.data_ptr(), _ptr(self.s1), _ptr(self.s2), *args, T, D, V,
                                            *hyper, ld, self.col_stride, *tail)
        native.check(rc, name)
        # the rows written are those of the distinct tables; the occurrences read are every column's.  A weighted
        # push runs one kernel more than an unweighted one: the per-occurrence factors w * f (the shared push's
        # offsets kernel writes them)
        launches = push_rows_launches(B * L, self.max_members if self.shared else 0)
        conn.account(push=T * B * L * D * 4 * (1 + self.slots), launches=launches + int(f is not None and not self.shared))


class _Lookup(torch.autograd.Function):
    """An embedding lookup over a table group: group.bag forward, group.push backward.  anchor is a leaf that
    requires grad, so that the backward runs although no input does."""

    @staticmethod
    def forward(ctx, group, ids, weights, anchor):
        out, ctx.f = group.bag(ids, weights)
        ctx.group, ctx.ids, ctx.weights = group, ids, weights
        return out

    @staticmethod
    def backward(ctx, dout):
        ctx.group.push(ctx.ids, dout.contiguous().float(), ctx.weights, ctx.f, ctx.group.combiners[0])
        return None, None, None, None


def _try_fuse_wide_tower(conn: HbmConnection, network: nn.Module) -> bool:
    """The wide tower (fc.LinearModel): T per-bucket weight tables [V, units] looked up once per example and summed.
    One multi-table gather kernel forward, one multi-table push (FTRL / ... fused) backward, instead of T launches
    each plus T adds."""
    if os.environ.get("TFY_PS_FUSE_WIDE", "1") == "0":
        return False
    lin = getattr(network, "linear", None)
    if not isinstance(lin, fc.LinearModel) or not lin.tables:
        return False
    by_param = {id(p): i for i, p in enumerate(conn.params)}
    cat_cols, tables_idx = [], []
    for c in lin.columns:
        cc = fc._categorical(c)
        if cc is not None:
            emb = lin.tables[cc.key]
            ti = by_param.get(id(emb.weight))
            if ti is None or ti not in conn.sparse or not isinstance(emb, fc.CombinedBag):
                return False
            cat_cols.append(cc)
            tables_idx.append(ti)
    combiner = lin.sparse_combiner
    # every table gets the same gradient (col_stride 0)
    group = _TableGroup(conn, tables_idx, cat_cols, lin.units,
                        combiners=[COMBINER_CODES[combiner]] * len(tables_idx))
    if not (group.uniform and (group.same_v or group.derived)):     # mixed V only with the id kernel's bound
        return False
    anchor = torch.zeros((), device=conn.device, requires_grad=True)
    num_cols = [c for c in lin.columns if isinstance(c, fc.NumericColumn)]

    def forward(features):
        if combiner == "sum" and group.one_hot(features):
            out = _Lookup.apply(group, group.ids_of(features), None, anchor)
        else:       # multi-hot, weighted or non-sum: every column combined by the sparse combiner, then summed
            out = _Lookup.apply(group, *group.multi_of(features), anchor)
        if lin.numeric is not None and num_cols:
            nums = [features[c.key].reshape(features[c.key].shape[0], -1).float() for c in num_cols]
            x = nums[0] if len(nums) == 1 else torch.cat(nums, dim=1)
            out = out + lin.numeric(x.to(lin.numeric.weight.dtype))
        return out + lin.bias

    lin.forward = forward
    logger.info("wide tower: %d tables served by the multi-table gather / push kernels", len(tables_idx))
    return True


def _serve_shared_collections(conn: HbmConnection, network: nn.Module, k5_features=None) -> int:
    """Shared embedding collections of a DenseFeatures that K5 does not serve: one weighted bag launch for all the
    members of a collection (T = members, the table repeated, into a [B, C*D] buffer sliced to their positions) and
    one shared push in its backward, instead of one bag and one push per member.  k5_features is the DenseFeatures
    whose forward K5 replaced (its collections are pushed by K5's backward).  Returns the collections served."""
    by_param = {id(p): i for i, p in enumerate(conn.params)}
    served = 0
    for df in network.modules():
        if not isinstance(df, fc.DenseFeatures) or not df.shared or df is k5_features:
            continue
        lookups = {}
        for name, positions in df.shared.items():
            emb = df.embeddings[name]
            ti = by_param.get(id(emb.weight))
            if ti is None or ti not in conn.sparse or not isinstance(emb, fc.CombinedBag):
                continue
            lookups[name] = _shared_lookup(conn, ti, [df.columns[p] for p in positions])
        if lookups:
            default = df.shared_lookup

            def shared_lookup(name, features, lookups=lookups, default=default):
                return lookups[name](features) if name in lookups else default(name, features)
            df.shared_lookup = shared_lookup
            served += len(lookups)
    return served


def _shared_lookup(conn: HbmConnection, ti: int, members):
    """One collection's lookup: the members' [B, D] values from one tfy_ps_multi_bag_weighted launch, and one push of
    the table for all of them."""
    C, D = len(members), members[0].dimension
    group = _TableGroup(conn, [ti] * C, [c.categorical_column for c in members], D, D,
                        combiners=[COMBINER_CODES[members[0].combiner]] * C)
    anchor = torch.zeros((), device=conn.device, requires_grad=True)

    def lookup(features):
        out = _Lookup.apply(group, *group.multi_of(features), anchor)
        return [out[:, D * k:D * k + D] for k in range(C)]
    return lookup


def _try_fuse_first_layer(conn: HbmConnection, network: nn.Module) -> bool:
    """K5: fuse the sparse pull of the embedding rows INTO the first deep GEMM (ops/csrc/tfy_ps_gemm.cu).

    Pattern (the canned wide-and-deep / DNN networks): ``network.dense_features`` concatenates embedding columns
    of dimension 64 with one id per example followed by numeric columns (<= 64 values in total), and
    ``network.hidden[0]`` is a Linear served by the remote-weight GEMM.  The gather of the rows from the ps ranks'
    HBM becomes the A-operand producer of that GEMM; the backward (dW, dx) is one wgmma kernel against the same
    remote shadow, and the row gradients are pushed straight out of its dx.  TFY_PS_FUSE_FIRST=0 disables it."""
    from tf_yarn_b200.ops.gemm import gemm_bf16
    if os.environ.get("TFY_PS_FUSE_FIRST", "1") == "0":
        return False
    df, hidden = getattr(network, "dense_features", None), getattr(network, "hidden", None)
    if not isinstance(df, fc.DenseFeatures) or not hidden or not isinstance(hidden[0], nn.Linear):
        return False
    lin = hidden[0]
    by_param = {id(p): i for i, p in enumerate(conn.params)}
    widx = by_param.get(id(lin.weight))
    if widx is None or widx not in conn.gemm or lin.bias is None:
        return False
    emb_cols, num_cols, seen_numeric = [], [], False
    for c in df.columns:
        if isinstance(c, (fc.EmbeddingColumn, fc.SharedEmbeddingColumn)) and not seen_numeric and c.dimension == 64:
            emb_cols.append(c)
        elif isinstance(c, fc.NumericColumn):
            seen_numeric = True
            num_cols.append(c)
        else:
            return False                     # embeddings must come first, all of dimension 64
    T, n_num = len(emb_cols), sum(c.dim for c in num_cols)
    if T == 0 or n_num > 64 or lin.in_features != 64 * T + n_num:
        return False
    tables_idx = []
    for c in emb_cols:
        emb = df.embeddings[fc._embedding_key(c)]
        ti = by_param.get(id(emb.weight))
        if ti is None or ti not in conn.sparse or not isinstance(emb, fc.CombinedBag):
            return False
        tables_idx.append(ti)
    V = emb_cols[0].categorical_column.num_buckets
    if any(c.categorical_column.num_buckets != V for c in emb_cols):
        return False
    dev = conn.device
    N, K, Kp = lin.out_features, lin.in_features, conn.shadow_ld(widx)
    shadow = conn.shadow_ptr(widx)
    # table t takes columns [64 t, 64 t + 64) of the activation buffer and of dx.  The bag takes one combiner per
    # launch (a group whose columns differ is gathered table by table); the push takes each column's 1/den in f, so
    # it is told "mean" whatever the mix
    group = _TableGroup(conn, tables_idx, [c.categorical_column for c in emb_cols], 64, 64,
                        combiners=[COMBINER_CODES[c.combiner] for c in emb_cols])

    class _FusedFirst(torch.autograd.Function):
        """One id per example: the gather is the A-operand producer of the GEMM (tfy_ps_gather_gemm)."""

        @staticmethod
        def forward(ctx, ids, weights, numeric, weight, bias):
            B = ids.shape[1]
            xbuf = torch.zeros((B, Kp), dtype=torch.bfloat16, device=dev)
            y = torch.empty((B, N), dtype=torch.bfloat16, device=dev)
            bb = bias.to(torch.bfloat16)
            native.check(conn.lib.tfy_ps_gather_gemm(shadow, group.tables.data_ptr(), ids.data_ptr(),
                                                     numeric.data_ptr() if numeric is not None else None,
                                                     bb.data_ptr(), xbuf.data_ptr(), y.data_ptr(), B, N, T, n_num, Kp,
                                                     V, torch.cuda.current_stream().cuda_stream), "tfy_ps_gather_gemm")
            conn.account(pull=B * T * 64 * 4 + N * Kp * 2)
            ctx.save_for_backward(xbuf, ids, weight)
            ctx.weights, ctx.f = None, None
            return y.to(weight.dtype)

        @staticmethod
        def backward(ctx, dy):
            """dW and dx in one wgmma kernel against the remote shadow, then the push of the embedding rows straight
            out of dx."""
            xbuf, ids, weight = ctx.saved_tensors
            B = xbuf.shape[0]
            dyb = dy.to(torch.bfloat16).contiguous()
            dw = torch.empty((N, Kp), dtype=torch.bfloat16, device=dev)
            dx = torch.empty((B, Kp), dtype=torch.bfloat16, device=dev)
            native.check(conn.lib.tfy_dense_bwd(dyb.data_ptr(), xbuf.data_ptr(), shadow, dw.data_ptr(), dx.data_ptr(),
                                                B, N, Kp, torch.cuda.current_stream().cuda_stream), "tfy_dense_bwd")
            conn.account(pull=N * Kp * 2)
            group.push(ids, dx, ctx.weights, ctx.f, SUM if ctx.f is None else MEAN, Kp)
            return None, None, None, dw[:, :K].to(weight.dtype), dy.float().sum(0).to(weight.dtype)

    class _BagFirst(_FusedFirst):
        """Multi-hot or weighted batches: the weighted bag writes the activation buffer K5 would (embeddings, then
        the numeric columns), then the remote-weight GEMM; the backward is K5's, with the weighted push."""

        @staticmethod
        def forward(ctx, ids, weights, numeric, weight, bias):
            xbuf = torch.zeros((ids.shape[1], Kp), dtype=torch.bfloat16, device=dev)
            _, f = group.bag(ids, weights, xbuf, Kp, numeric)
            y = gemm_bf16(xbuf, None, bias=bias.to(torch.bfloat16), b_ptr=shadow, b_rows=N, b_ld=Kp, impl="1cta")
            conn.account(pull=N * Kp * 2)
            ctx.save_for_backward(xbuf, ids, weight)
            ctx.weights, ctx.f = weights, f
            return y.to(weight.dtype)

    class _Deferred:
        """What the patched DenseFeatures returns: the raw inputs of the fused first layer (weights is None and ids
        [T, B] for K5; ids [T, B, L] for the weighted bag)."""

        def __init__(self, ids, weights, numeric, one_hot):
            self.ids, self.weights, self.numeric, self.one_hot = ids, weights, numeric, one_hot

        def to(self, *a, **k):
            return self

    def df_forward(features):
        one_hot = group.one_hot(features)
        if one_hot:
            ids, weights = group.ids_of(features), None
        else:
            ids, weights = group.multi_of(features)
        numeric = None
        if num_cols:
            parts = [features[c.key].reshape(features[c.key].shape[0], -1).float() for c in num_cols]
            numeric = (parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)).contiguous()
        return _Deferred(ids, weights, numeric, one_hot)

    def lin_forward(x):
        if isinstance(x, _Deferred):
            fn = _FusedFirst if x.one_hot else _BagFirst
            return fn.apply(x.ids, x.weights, x.numeric, lin.weight, lin.bias)
        return _make_linear_forward(conn, widx, lin)(x)

    df.forward = df_forward
    lin.forward = lin_forward
    logger.info("K5: embedding gather of %d tables fused into the first deep GEMM (%d -> %d)", T, K, N)
    return True


# ---------------------------------------------------------------------------------------------
# connection set-up (collective over the cluster)
# ---------------------------------------------------------------------------------------------
def connect_worker(network: nn.Module, opt_desc, cluster, is_chief: bool, global_step: int,
                   opt_by_name=None, ps_state: Optional[Dict[str, dict]] = None) -> HbmConnection:
    """Chief: publish the layout, initialise the shards (the optimizer slots from `ps_state`, a checkpoint's, where
    they match: ps.init_slots) and their bf16 shadows.  Worker: wait until ready.  Both then install the kernels."""
    ps_cpu.refuse_nadam(ps_cpu._named_trainables(network), opt_desc, opt_by_name)
    if any(getattr(d, "schedule", None) is not None for d in [opt_desc, *(opt_by_name or {}).values()]):
        raise ValueError("the HBM parameter server bakes the learning rate into its push kernels and does not run "
                         "a LearningRateSchedule; use the shared-memory parameter server (TFY_PS_PLANE=shm) or a "
                         "constant learning rate")
    client = _task_commons.TaskClient.from_current()
    kv = client.kv
    n_ps = len(cluster.spec["ps"])
    named = ps_cpu._named_trainables(network)
    names = [n for n, _ in named]
    if is_chief:
        layout = ps_cpu.make_layout(named, n_ps, opt_desc, opt_by_name)
        kv[ps_cpu.KV_LAYOUT] = layout.to_json().encode()
    else:
        layout = ps_cpu.Layout.from_json(kv.wait(ps_cpu.KV_LAYOUT))
    comm, ranks = join_arena(cluster)
    region_off = comm.arena.alloc(shard_bytes(layout), align=4096)
    header_path = kv.wait("ps:0/shard").decode()
    header = ps_cpu.ShmShard(header_path, 8, create=False)
    conn = HbmConnection(layout, comm, ranks, region_off, names, header, network)
    if is_chief:
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                conn.remote_tensor(i).copy_(p.detach().reshape(-1).float())
            ps_cpu.init_slots(layout, conn.remote_tensor, ps_state)
        conn.refresh_shadows()
        header.set_global_step(global_step)
        torch.cuda.synchronize()
        kv[ps_cpu.KV_READY] = b"1"
        logger.info("HBM parameter servers initialised: %d variables on %d ps (%d sparse, %d remote-GEMM)",
                    len(names), n_ps, len(conn.sparse), len(conn.gemm))
    else:
        kv.wait(ps_cpu.KV_READY)
    conn.install(network)
    return conn


def serve(cluster, poll_secs: float = 0.2) -> None:
    """``ps`` task on H100: join the arena, reserve the shard region, publish the header, idle."""
    import time
    client = _task_commons.TaskClient.from_current()
    kv = client.kv
    idx = cluster.task_id
    layout = ps_cpu.Layout.from_json(kv.wait(ps_cpu.KV_LAYOUT))
    comm, _ = join_arena(cluster)
    off = comm.arena.alloc(shard_bytes(layout), align=4096)
    region = comm.arena.tensor(off, (shard_bytes(layout),), torch.uint8)
    region.zero_()
    torch.cuda.synchronize()
    path = os.path.join(ps_cpu._shm_dir(), f"tfy_ps_{ps_cpu._job_tag()}_{idx}")
    header = ps_cpu.ShmShard(path, 8, create=True)
    kv[f"ps:{idx}/shard"] = path.encode()
    logger.info("ps %d: %d bytes of HBM shard at arena offset %d", idx, shard_bytes(layout), off)
    import atexit
    atexit.register(header.unlink)
    while True:
        time.sleep(poll_secs)
