"""Data-parallel wrapper driven by the hand-written NVLS / P2P all-reduce kernels.

Drop-in for ``torch.nn.parallel.DistributedDataParallel`` as the reference's
PyTorch worker uses it (reference: tf_yarn/pytorch/tasks/worker.py:105-107,
arguments tf_yarn/pytorch/experiment.py:23-27):

* parameters are bucketed in reverse registration order (first bucket 1 MiB,
  then ``bucket_cap_mb``) into flat gradient buffers that live in the
  symmetric arena; every ``p.grad`` is a view into its bucket;
* a post-accumulate-grad hook makes ONE call per parameter into the native
  reducer (``ops/csrc/tfy_reducer.cpp``): it counts ready gradients and, when a
  bucket (and all its predecessors) is complete, launches the bucket's
  all-reduce kernel (``multimem.ld_reduce`` + ``multimem.st``, averaged, in
  place) on its communication stream, overlapping the rest of backward;
* :meth:`DistributedDataParallel.fuse_optimizer` replaces the per-bucket
  all-reduce by the fused reduce-scatter -> optimizer -> all-gather kernel
  (K4), so the optimizer step overlaps backward as well;
* at the end of backward the compute stream waits for the last collective;
* parameters (and, each forward, module buffers when ``broadcast_buffers``)
  are broadcast from rank 0 with the K7 kernel.

No NCCL call is issued by this wrapper.  On a CPU-only process group (gloo,
the plumbing configuration) :func:`wrap_model` returns torch's own DDP.
"""
from __future__ import annotations

import contextlib
import ctypes
from typing import List, Optional

import torch
import torch.nn as nn

from tf_yarn_b200.ops import native
from tf_yarn_b200.parallel.comm import _DT, Communicator, _stream_ptr, hyper_block, launch_code
from tf_yarn_b200.parallel.optspec import OptimizerSpec

_vp, _i, _u64, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_size_t
native.declare("tfy_reducer_create", [_vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _i], restype=_vp)
native.declare("tfy_reducer_set_fused", [_vp, _i, _i, _u64, _vp, _vp, _vp, _sz, _i, _i, _vp])
native.declare("tfy_reducer_mark_ready", [_vp, _i, _vp])
native.declare("tfy_reducer_finalize", [_vp, _vp])
native.declare("tfy_reducer_launches", [_vp], restype=ctypes.c_long)
native.declare("tfy_reducer_destroy", [_vp], restype=None)

_FIRST_BUCKET_BYTES = 1 << 20


def _view_like(flat: torch.Tensor, off: int, p: torch.Tensor) -> torch.Tensor:
    """View of ``flat[off:off+numel]`` with the shape AND memory layout of ``p``.

    autograd's gradient layout contract wants ``grad.strides == param.strides``; a channels_last conv
    weight therefore gets a channels_last view of its slice (otherwise every accumulation re-lays the
    gradient out and warns)."""
    seg = flat[off:off + p.numel()]
    if p.dim() == 4 and not p.is_contiguous() and p.is_contiguous(memory_format=torch.channels_last):
        n, c, h, w = p.shape
        return seg.view(n, h, w, c).permute(0, 3, 1, 2)
    return seg.view_as(p)


class _Bucket:
    __slots__ = ("params", "offsets", "flat", "pending", "launched", "event", "dtype", "off", "pflat", "poff",
                 "master", "s1", "s2", "hyper", "shard_n")

    def __init__(self, dtype):
        self.params: List[nn.Parameter] = []
        self.offsets: List[int] = []
        self.flat: Optional[torch.Tensor] = None
        self.pending = 0
        self.launched = False
        self.event: Optional[torch.cuda.Event] = None
        self.dtype = dtype


class DistributedDataParallel(nn.Module):
    _is_tfy_ddp = True

    def __init__(self, module: nn.Module, comm: Communicator, broadcast_buffers: bool = True,
                 bucket_cap_mb: int = 25, find_unused_parameters: bool = False,
                 gradient_as_bucket_view: bool = False, device_ids=None):
        super().__init__()
        self.module = module
        self.comm = comm
        self.broadcast_buffers = broadcast_buffers
        self.find_unused_parameters = find_unused_parameters
        self.require_backward_grad_sync = True
        self._comm_stream = torch.cuda.Stream(device=comm.device) if comm.world > 1 else None
        self._callback_queued = False
        self._next_bucket = 0            # buckets [0, _next_bucket) have been launched in this backward
        self._buckets: List[_Bucket] = []
        self._param_bucket = {}          # id(param) -> (bucket, index in bucket); tensors compare elementwise
        self._build_buckets(int(bucket_cap_mb) << 20)
        self._sync_params_and_buffers()
        # native reducer (C++): needs the kernel library and a CUDA device; the Python bookkeeping below is the
        # fallback for host-only unit tests with a fake communicator
        self._reducer = None
        self._fused = None
        self._param_index = {}
        if getattr(comm, "lib", None) is not None and torch.cuda.is_available():
            self._create_reducer()
        for b in self._buckets:
            for p in b.params:
                p.register_post_accumulate_grad_hook(self._make_hook(p))

    # ------------------------------------------------------------------ set-up
    def _build_buckets(self, cap_bytes: int) -> None:
        params = [p for p in self.module.parameters() if p.requires_grad]
        cur: Optional[_Bucket] = None
        cur_bytes = 0
        limit = _FIRST_BUCKET_BYTES
        for p in reversed(params):
            if p.dtype not in (torch.float32, torch.bfloat16):
                raise TypeError(f"unsupported parameter dtype {p.dtype}: use float32 or bfloat16")
            nbytes = p.numel() * p.element_size()
            if cur is None or cur.dtype != p.dtype or (cur_bytes + nbytes > limit and cur.params):
                if cur is not None:
                    limit = cap_bytes
                cur = _Bucket(p.dtype)
                self._buckets.append(cur)
                cur_bytes = 0
            cur.params.append(p)
            cur.offsets.append(cur_bytes // p.element_size())
            cur_bytes += (nbytes + 15) // 16 * 16
        for b in self._buckets:
            last = b.params[-1]
            n = b.offsets[-1] + (last.numel() + 7) // 8 * 8
            n = self.comm.pad_elems(n, b.dtype)
            b.off, b.flat = self.comm.arena.empty((n,), b.dtype, align=4096)
            b.flat.zero_()
            for i, (p, o) in enumerate(zip(b.params, b.offsets)):
                p.grad = _view_like(b.flat, o, p)
                self._param_bucket[id(p)] = (b, i)
            b.pending = len(b.params)

    def _create_reducer(self) -> None:
        nb = len(self._buckets)
        offs = (ctypes.c_uint64 * nb)(*[b.off for b in self._buckets])
        ns = (ctypes.c_size_t * nb)(*[b.flat.numel() for b in self._buckets])
        dts = (ctypes.c_int * nb)(*[_DT[b.dtype] for b in self._buckets])
        nps = (ctypes.c_int * nb)(*[len(b.params) for b in self._buckets])
        flat_params, pb = [], []
        for bi, b in enumerate(self._buckets):
            for p in b.params:
                self._param_index[id(p)] = len(flat_params)
                flat_params.append(p)
                pb.append(bi)
        pbs = (ctypes.c_int * len(pb))(*pb)
        lib = self.comm.lib
        self._reducer = lib.tfy_reducer_create(self.comm.arena.ctx_ref, nb, offs, ns, dts, nps, len(pb), pbs,
                                               self.comm.pick_algo_inplace())
        if not self._reducer:
            raise RuntimeError("tfy_reducer_create failed")

    @property
    def kernel_launches(self) -> int:
        """Collective / fused-step kernels launched by the reducer so far."""
        if self._reducer:
            return int(self.comm.lib.tfy_reducer_launches(self._reducer))
        return 0

    def fuse_optimizer(self, kind: str = "sgd", **hyper):
        """Move the optimizer INTO the gradient exchange: every bucket runs the fused reduce-scatter -> update
        -> all-gather kernel (K4: ``multimem.ld_reduce`` of the owned 1/world shard, SGD-momentum / Adam / Adagrad /
        Adadelta / RMSprop / Adamax / Nadam on fp32 master + sharded state, ``multimem.st`` of the new parameters) on
        the communication stream as soon as its gradients are complete, so the whole optimizer step overlaps backward.  Parameters are
        re-pointed at flat symmetric buffers.  Returns an optimizer-shaped object (``step`` / ``zero_grad`` are
        no-ops: by the time backward returns, the update is queued behind it).  Gradient clipping between
        ``backward()`` and ``step()`` is not available in this mode.

        ``hyper`` are the keyword arguments of the matching ``OptimizerSpec`` constructor, e.g.
        ``fuse_optimizer("rmsprop", lr=1e-3, rho=0.9, momentum=0.9, eps=1e-7, centered=True)`` for the Keras
        RMSprop (epsilon inside the square root, lr inside the momentum buffer), or
        ``fuse_optimizer("adamax" | "nadam", lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)`` for the Keras Adamax and
        Nadam.  Every bucket of a Nadam step keeps its own running product of the momentum schedule."""
        if not self._reducer:
            raise RuntimeError("fuse_optimizer needs the native reducer (CUDA)")
        if self._fused is not None:
            return self._fused
        kinds = {"sgd": OptimizerSpec.sgd, "adam": OptimizerSpec.adam, "adagrad": OptimizerSpec.adagrad,
                 "adadelta": OptimizerSpec.adadelta, "rmsprop": OptimizerSpec.rmsprop,
                 "adamax": OptimizerSpec.adamax, "nadam": OptimizerSpec.nadam}
        if kind not in kinds:
            raise ValueError(f"unknown fused optimizer {kind!r}")
        spec = kinds[kind](**hyper)
        comm = self.comm
        dev = f"cuda:{comm.device}"
        world = comm.world
        for bi, b in enumerate(self._buckets):
            n = b.flat.numel()
            b.shard_n = n // world
            assert b.shard_n * world == n and b.shard_n % 8 == 0, (n, world)
            b.poff, b.pflat = comm.arena.empty((n,), b.dtype, align=4096)
            b.pflat.zero_()
            for p, o in zip(b.params, b.offsets):
                view = _view_like(b.pflat, o, p)
                view.copy_(p.data)
                p.data = view
            r = comm.rank if world > 1 else 0
            b.master = b.pflat[r * b.shard_n:(r + 1) * b.shard_n].float().clone()
            b.s1 = torch.full((b.shard_n,), spec.init_s1, dtype=torch.float32, device=dev)
            b.s2 = torch.zeros(spec.s2_numel(b.shard_n), dtype=torch.float32, device=dev)
            b.hyper = torch.frombuffer(bytearray(bytes(hyper_block(spec))), dtype=torch.uint8).to(dev)
            if spec.schedule is not None:
                native.check(comm.lib.tfy_lr_schedule_sync(b.hyper.data_ptr(), _stream_ptr()), "tfy_lr_schedule_sync")
            native.check(comm.lib.tfy_reducer_set_fused(
                self._reducer, bi, _DT[b.dtype], b.poff, b.master.data_ptr(), b.s1.data_ptr(), b.s2.data_ptr(),
                b.shard_n, launch_code(spec), comm.mode, b.hyper.data_ptr()), "tfy_reducer_set_fused")
        torch.cuda.current_stream().synchronize()
        if world > 1:
            comm.barrier()
        self._fused = _FusedOptimizer(self, spec)
        # loading a model checkpoint writes the (replicated) parameters; the fp32 master shards the fused kernel
        # updates FROM must follow, or the next step would overwrite the loaded weights with the old master
        self.module.register_load_state_dict_post_hook(lambda _module, _keys: self._resync_fused_masters())
        return self._fused

    def _resync_fused_masters(self) -> None:
        """fp32 master shard of every bucket := this rank's slice of the current parameters."""
        me = self.comm.rank if self.comm.world > 1 else 0
        with torch.no_grad():
            for b in self._buckets:
                b.master.copy_(b.pflat[me * b.shard_n:(me + 1) * b.shard_n].float())

    def _sync_params_and_buffers(self) -> None:
        if self.comm.world == 1:
            return
        tensors = [p.data for p in self.module.parameters()] + [b.data for b in self.module.buffers()]
        self.comm.broadcast(tensors, root=0)
        torch.cuda.current_stream().synchronize()

    def _grad_view(self, p: nn.Parameter) -> torch.Tensor:
        b, i = self._param_bucket[id(p)]
        o = b.offsets[i]
        return _view_like(b.flat, o, p)

    # ------------------------------------------------------------------ hooks
    def _make_hook(self, p: nn.Parameter):
        bucket, idx = self._param_bucket[id(p)]
        off = bucket.offsets[idx]
        view = _view_like(bucket.flat, off, p)
        pidx = self._param_index.get(id(p), -1)

        def hook(param: nn.Parameter) -> None:
            g = param.grad
            if g is not None and g.data_ptr() != view.data_ptr():
                # the user dropped the view (zero_grad(set_to_none=True)): fold the fresh grad back in
                view.copy_(g)
                param.grad = view
            if not self.require_backward_grad_sync:
                return
            if not self._callback_queued:
                self._callback_queued = True
                torch.autograd.Variable._execution_engine.queue_callback(self._finalize_backward)
            if self._reducer:
                rc = self.comm.lib.tfy_reducer_mark_ready(self._reducer, pidx, torch.cuda.current_stream().cuda_stream)
                if rc:
                    raise RuntimeError(f"bucket collective failed to launch: {rc}")
                return
            bucket.pending -= 1
            if bucket.pending == 0:
                self._launch_ready_prefix()

        return hook

    def _launch_ready_prefix(self) -> None:
        """Launch complete buckets STRICTLY in index order (bucket i only after 0..i-1), as torch DDP does: the
        kernels of different ranks are paired by launch order on the per-CTA flag slots, so every rank must issue
        the same sequence even if autograd completes the buckets in a different order on some rank."""
        while self._next_bucket < len(self._buckets):
            b = self._buckets[self._next_bucket]
            if b.pending != 0:
                return
            self._launch(b)
            self._next_bucket += 1

    def _launch(self, bucket: _Bucket) -> None:
        bucket.launched = True
        if self.comm.world == 1:
            return
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        self._comm_stream.wait_event(ready)
        with torch.cuda.stream(self._comm_stream):
            self.comm.all_reduce_symm(bucket.flat, average=True, algo=self.comm.pick_algo_inplace())
            bucket.event = torch.cuda.Event()
            bucket.event.record(self._comm_stream)

    def _finalize_backward(self) -> None:
        self._callback_queued = False
        if self._reducer:
            rc = self.comm.lib.tfy_reducer_finalize(self._reducer, torch.cuda.current_stream().cuda_stream)
            if rc:
                raise RuntimeError(f"bucket collective failed to launch: {rc}")
            return
        for b in self._buckets[self._next_bucket:]:
            # buckets still waiting for a predecessor, or whose parameters received no gradient this step
            # (they contribute zeros -- what find_unused_parameters=True does in torch DDP), in index order
            self._launch(b)
        self._next_bucket = 0
        cur = torch.cuda.current_stream() if self.comm.world > 1 else None
        for b in self._buckets:
            if b.event is not None:
                cur.wait_event(b.event)
                b.event = None
            b.launched = False
            b.pending = len(b.params)

    # ---------------------------------------------------------------- forward
    def forward(self, *args, **kwargs):
        if self.broadcast_buffers and self.comm.world > 1 and self.require_backward_grad_sync:
            bufs = [b.data for b in self.module.buffers() if b.is_floating_point()]
            if bufs:
                self.comm.broadcast(bufs, root=0)
        return self.module(*args, **kwargs)

    @contextlib.contextmanager
    def no_sync(self):
        """Accumulate gradients locally; the next synced backward reduces the accumulated sum."""
        old = self.require_backward_grad_sync
        self.require_backward_grad_sync = False
        try:
            yield
        finally:
            self.require_backward_grad_sync = old

    def zero_grad(self, set_to_none: bool = False) -> None:  # keep the bucket views alive
        if self._fused is not None and self.require_backward_grad_sync:
            return                      # the fused kernel clears every bucket behind itself
        for b in self._buckets:
            b.flat.zero_()
            for p, o in zip(b.params, b.offsets):
                p.grad = _view_like(b.flat, o, p)

    def __del__(self):
        try:
            if getattr(self, "_reducer", None):
                self.comm.lib.tfy_reducer_destroy(self._reducer)
                self._reducer = None
        except Exception:  # noqa: BLE001
            pass

    # state_dict()/load_state_dict() are nn.Module's: keys carry the ``module.`` prefix exactly like
    # torch.nn.parallel.DistributedDataParallel, so checkpoints are interchangeable with the reference's
    # (tf_yarn/pytorch/model_ckpt.py saves ``model.module.state_dict()`` when it sees a wrapper).


class _ScheduledParamGroup(dict):
    """``param_groups[0]`` of a fused optimizer whose rate follows a LearningRateSchedule: ``["lr"]`` reads the rate
    the fused step will use next from the device (a 4-byte read), and setting it -- e.g. by a torch LR scheduler --
    raises at once, since the fused step writes every rate itself."""

    def __init__(self, opt: "_FusedOptimizer", params):
        super().__init__(params=params)
        self._opt = opt

    def __getitem__(self, key):
        if key == "lr":
            return self._opt.current_lr()
        return super().__getitem__(key)

    def __setitem__(self, key, value):
        if key in ("lr", "initial_lr"):
            raise TypeError("the learning rate of this optimizer follows a LearningRateSchedule, which the fused "
                            "step evaluates on the device; it cannot be set")
        super().__setitem__(key, value)

    def setdefault(self, key, default=None):
        if key not in self:
            self[key] = default
        return self[key]

    def __contains__(self, key):
        return key == "lr" or super().__contains__(key)


class _FusedOptimizer:
    """Optimizer-shaped handle of :meth:`DistributedDataParallel.fuse_optimizer`."""

    def __init__(self, ddp: "DistributedDataParallel", spec: OptimizerSpec):
        self._ddp, self.spec = ddp, spec
        params = [p for b in ddp._buckets for p in b.params]
        if spec.schedule is not None:
            self.param_groups = [_ScheduledParamGroup(self, params)]
        else:
            self.param_groups = [{"lr": spec.lr, "params": params}]

    def current_lr(self) -> float:
        """The learning rate of the next step (with a schedule, the one the device holds)."""
        if self.spec.schedule is None:
            return float(self.param_groups[0]["lr"])
        return float(self._ddp._buckets[0].hyper[0:4].view(torch.float32).item())

    def step(self, closure=None):
        if self.spec.schedule is not None:          # the fused step writes every rate itself
            return None
        lr = float(self.param_groups[0]["lr"])
        if lr != self.spec.lr:                       # an LR scheduler changed it: 4-byte copies, graph/stream safe
            self.set_lr(lr)
        return None

    def zero_grad(self, set_to_none: bool = False) -> None:
        return None

    def set_lr(self, lr: float) -> None:
        if self.spec.schedule is not None:
            raise TypeError("the learning rate of this optimizer follows a LearningRateSchedule, which the fused "
                            "step evaluates on the device; it cannot be set")
        self.spec.lr = float(lr)
        t = torch.tensor([lr], dtype=torch.float32).view(torch.uint8)
        for b in self._ddp._buckets:
            b.hyper[0:4].copy_(t, non_blocking=True)

    def state_dict(self) -> dict:
        comm = self._ddp.comm
        out = {"kind": "tfy_fused_ddp", "buckets": []}
        for b in self._ddp._buckets:
            out["buckets"].append({"master": b.master.cpu(), "s1": b.s1.cpu(), "s2": b.s2.cpu(),
                                   "step": int(b.hyper[24:28].view(torch.int32).item()), "rank": comm.rank})
            if self.spec.kind == "nadam":
                out["buckets"][-1]["mu_product"] = float(b.hyper[_MU_OFF:_MU_OFF + 8].view(torch.float64).item())
        return out

    def load_state_dict(self, state: dict) -> None:
        """Restore what :meth:`state_dict` saved.  The state is SHARDED (each rank owns 1/world of the fp32 master
        weights and moments) while the reference's flow saves on rank 0 only (tf_yarn/pytorch/model_ckpt.py:55-72):
        a rank that is handed another rank's shard rebuilds its fp32 master from the parameters the model checkpoint
        has just restored and restarts its moments, instead of adopting foreign values."""
        comm = self._ddp.comm
        me = comm.rank if comm.world > 1 else 0
        foreign = False
        for b, st in zip(self._ddp._buckets, state["buckets"]):
            if int(st.get("rank", 0)) == me and st["master"].numel() == b.master.numel():
                b.master.copy_(st["master"])
                b.s1.copy_(st["s1"])
                b.s2.copy_(st["s2"])
            else:
                foreign = True
                b.master.copy_(b.pflat[me * b.shard_n:(me + 1) * b.shard_n].float())
                b.s1.fill_(self.spec.init_s1)
                b.s2.zero_()
            b.hyper[24:28].copy_(torch.tensor([st["step"]], dtype=torch.int32).view(torch.uint8))
            if self.spec.kind == "nadam":
                b.hyper[_MU_OFF:_MU_OFF + 8].copy_(
                    torch.tensor([float(st.get("mu_product", 1.0))], dtype=torch.float64).view(torch.uint8))
            if self.spec.schedule is not None:      # the rate of the restored step, written by the device function
                native.check(self._ddp.comm.lib.tfy_lr_schedule_sync(b.hyper.data_ptr(), _stream_ptr()),
                             "tfy_lr_schedule_sync")
        if foreign:
            import logging
            logging.getLogger(__name__).warning(
                "rank %d: the optimizer checkpoint holds another rank's shard; fp32 master rebuilt from the restored "
                "parameters, moments restart on this rank", me)


_MU_OFF = native.NadamHyperBlock.mu_product.offset     # Nadam's running product in a bucket's hyper block


def wrap_model(model: nn.Module, device, ddp_kwargs: Optional[dict] = None, comm: Optional[Communicator] = None):
    """Data-parallel wrapper appropriate for the process: ours on H100, torch DDP on CPU/gloo."""
    import torch.distributed as dist
    ddp_kwargs = dict(ddp_kwargs or {})
    on_gpu = isinstance(device, int) or torch.device(device).type == "cuda"
    if on_gpu:
        if comm is None:
            from tf_yarn_b200.parallel import runtime
            comm = runtime.get_communicator()
        return DistributedDataParallel(model, comm, **ddp_kwargs)
    if dist.is_initialized() and dist.get_world_size() > 1:
        from torch.nn.parallel import DistributedDataParallel as TorchDDP
        return TorchDDP(model, **ddp_kwargs)
    return model
