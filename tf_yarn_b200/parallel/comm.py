"""Collectives over the symmetric arena (hand-written sm_90a kernels, no NCCL).

``Communicator`` is the data plane behind the Horovod-like facade
(:mod:`tf_yarn_b200.hvd`), the DDP-like wrapper
(:mod:`tf_yarn_b200.parallel.ddp`) and the mini-Keras train step.  It replaces
Horovod's fusion-buffer + gloo/NCCL allreduce (reference:
tf_yarn/tensorflow/tasks/gloo_allred_task.py:54) and c10d's NCCL process group
(reference: tf_yarn/pytorch/tasks/worker.py:101).
"""
from __future__ import annotations

import ctypes
from typing import Tuple,  List, Optional, Sequence

import torch

from tf_yarn_b200.ops import native
from tf_yarn_b200.parallel.optspec import OptimizerSpec  # noqa: F401  (re-export)
from tf_yarn_b200.parallel.symm import Rendezvous, SymmArena

_DT = {torch.bfloat16: native.BF16, torch.float32: native.F32}

_vp, _i, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
native.declare("tfy_grad_accumulate", [_vp, _vp, _i, _sz, _i, _vp, _i, _i, _vp])

# below this many bytes the latency-optimal one-shot kernel wins (one barrier
# pair + every rank reads everything); above it the 2-phase kernels move 1/N of
# the data per rank.
ONESHOT_MAX_BYTES = 128 * 1024


def _stream_ptr(stream: Optional[torch.cuda.Stream] = None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return s.cuda_stream


class Communicator:
    def __init__(self, arena_bytes: int = 256 << 20, fusion_bytes: int = 64 << 20,
                 rdv: Optional[Rendezvous] = None, device: Optional[int] = None, arena=None):
        self.arena = arena if arena is not None else SymmArena(arena_bytes + fusion_bytes + (1 << 20),
                                                               device=device, rdv=rdv)
        self.lib = self.arena.lib
        self.rank, self.world = self.arena.rank, self.arena.world
        self.device = self.arena.device
        self.multicast = self.arena.multicast
        self.fusion_bytes = fusion_bytes
        self.fusion_off = self.arena.alloc(fusion_bytes, align=4096)
        self._fusion_u8 = self.arena.tensor(self.fusion_off, (fusion_bytes,), torch.uint8)
        self.launches = 0  # kernels launched by this communicator (bench.py reports it)

    # ------------------------------------------------------------------ helpers
    @property
    def mode(self) -> int:
        if self.world == 1:
            return native.MODE_LOCAL
        return native.MODE_NVLS if self.multicast else native.MODE_P2P

    def pick_algo(self, nbytes: int) -> int:
        if self.world == 1 or nbytes <= ONESHOT_MAX_BYTES:
            return native.ALGO_ONESHOT
        return native.ALGO_NVLS if self.multicast else native.ALGO_TWOSHOT

    def pick_algo_inplace(self) -> int:
        """Algorithm for in-place reduction of an arena buffer (one-shot needs a separate output)."""
        return native.ALGO_NVLS if self.multicast else native.ALGO_TWOSHOT

    def pad_elems(self, n: int, dtype: torch.dtype) -> int:
        """Round an element count up so the buffer splits into world x 16-byte packs."""
        per = (16 // torch.empty((), dtype=dtype).element_size()) * self.world
        per = max(per, 8 * self.world)
        return (n + per - 1) // per * per

    # -------------------------------------------------------------- collectives
    def barrier(self, stream=None) -> None:
        native.check(self.lib.tfy_barrier(self.arena.ctx_ref, 1, _stream_ptr(stream)), "tfy_barrier")
        self.launches += 1

    def all_reduce_symm(self, t: torch.Tensor, average: bool = False, algo: Optional[int] = None,
                        out: Optional[torch.Tensor] = None, grid: int = 0, block: int = 0, stream=None):
        """All-reduce a tensor that lives in the symmetric arena.

        Two-shot / NVLS reduce in place and return ``t``; one-shot writes into
        ``out`` (any local tensor of the same shape, required) and returns it.
        """
        dt = _DT[t.dtype]
        n = t.numel()
        off = self.arena.offset_of(t)
        nbytes = n * t.element_size()
        if algo is None:
            algo = self.pick_algo(nbytes)
        if algo != native.ALGO_ONESHOT and (nbytes // 16) % self.world:
            algo = native.ALGO_ONESHOT
        scale = 1.0 / self.world if average else 1.0
        if algo == native.ALGO_ONESHOT:
            if out is None:
                out = torch.empty_like(t)
            outp = out.data_ptr()
        else:
            outp = None
        native.check(self.lib.tfy_allreduce(self.arena.ctx_ref, dt, algo, off, n, scale, outp, grid, block,
                                            _stream_ptr(stream)), "tfy_allreduce")
        self.launches += 1
        return out if algo == native.ALGO_ONESHOT else t

    def all_reduce(self, tensors: Sequence[torch.Tensor], average: bool = True, stream=None) -> None:
        """Horovod-style fused all-reduce of arbitrary CUDA tensors, in place.

        Tensors are packed into the symmetric fusion buffer (one multi-tensor
        copy), reduced by ONE kernel, and unpacked.  Chunks larger than the
        fusion buffer are processed in several rounds.
        """
        if not tensors or self.world == 1:
            return
        by_dtype = {}
        for t in tensors:
            by_dtype.setdefault(t.dtype, []).append(t)
        for dtype, group in by_dtype.items():
            if dtype not in _DT and dtype != torch.float16:
                self._all_reduce_exact(group, average, stream)
                continue
            if dtype not in _DT:
                # fp16 goes through fp32: one rounding of the fp32 sum
                tmp = [g.float() for g in group]
                self.all_reduce(tmp, average, stream)
                for g, x in zip(group, tmp):
                    g.copy_(x)
                continue
            esz = group[0].element_size()
            cap = self.fusion_bytes // esz
            batch: List[torch.Tensor] = []
            used = 0
            for t in group:
                n = t.numel()
                if n > cap:
                    self._flush(batch, dtype, average, stream)
                    batch, used = [], 0
                    flat = t.reshape(-1) if t.is_contiguous() else None
                    src = flat if flat is not None else t.contiguous().view(-1)
                    for s in range(0, n, cap):
                        piece = src[s:s + cap]
                        self._flush([piece], dtype, average, stream)
                    if flat is None:
                        t.copy_(src.view_as(t))
                    continue
                if used + n > cap:
                    self._flush(batch, dtype, average, stream)
                    batch, used = [], 0
                batch.append(t)
                used += n
            self._flush(batch, dtype, average, stream)

    def _all_reduce_exact(self, group: Sequence[torch.Tensor], average: bool, stream) -> None:
        """float64 and integer tensors, which fp32 would round (int64 above 2^24, say): every rank's bytes are
        all-gathered and summed in rank order in the tensor's own dtype, as the CPU plane's gloo sum is.  An average
        divides by the world size (integers: truncated toward zero)."""
        div = torch.full((), self.world, dtype=group[0].dtype, device=group[0].device)
        for t in group:
            src = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
            chunk = max(1, (self.fusion_bytes // self.world) // 16 * 16 // t.element_size())
            for s in range(0, src.numel(), chunk):
                piece = src[s:s + chunk]
                parts = self.all_gather(piece, stream).view(self.world, -1)
                acc = parts[0].clone()
                for r in range(1, self.world):
                    acc += parts[r]
                if average:
                    # a device tensor divisor: a true division, not a multiplication by a rounded reciprocal
                    acc = acc / div if acc.is_floating_point() else torch.div(acc, div, rounding_mode="trunc")
                piece.copy_(acc)
            if not t.is_contiguous():
                t.copy_(src.view_as(t))

    def _flush(self, batch: List[torch.Tensor], dtype, average: bool, stream) -> None:
        if not batch:
            return
        total = sum(t.numel() for t in batch)
        padded = self.pad_elems(total, dtype)
        buf = self._fusion_u8.view(dtype)[:padded]
        views = []
        o = 0
        for t in batch:
            views.append(buf[o:o + t.numel()].view_as(t) if t.is_contiguous() else buf[o:o + t.numel()].view(t.shape))
            o += t.numel()
        if padded > total:
            buf[total:].zero_()
        torch._foreach_copy_(views, list(batch))
        if self.world > 1:
            nbytes = padded * buf.element_size()
            algo = self.pick_algo(nbytes)
            if algo == native.ALGO_ONESHOT:
                out = torch.empty_like(buf)
                self.all_reduce_symm(buf, average, algo, out=out, stream=stream)
                o = 0
                outs = []
                for t in batch:
                    outs.append(out[o:o + t.numel()].view(t.shape))
                    o += t.numel()
                torch._foreach_copy_(list(batch), outs)
                return
            self.all_reduce_symm(buf, average, algo, stream=stream)
        torch._foreach_copy_(list(batch), views)

    def broadcast_symm(self, t: torch.Tensor, root: int = 0, stream=None) -> torch.Tensor:
        off = self.arena.offset_of(t)
        nbytes = t.numel() * t.element_size()
        if nbytes % 16:
            raise ValueError("broadcast_symm needs a multiple of 16 bytes")
        if self.world > 1:
            native.check(self.lib.tfy_broadcast(self.arena.ctx_ref, off, nbytes, root, int(self.multicast), 0, 0,
                                                _stream_ptr(stream)), "tfy_broadcast")
            self.launches += 1
        return t

    def broadcast(self, tensors: Sequence[torch.Tensor], root: int = 0, stream=None) -> None:
        """Broadcast arbitrary CUDA tensors from ``root``: packed into the fusion buffer (one multi-tensor
        copy), ONE broadcast kernel per fusion-buffer fill, unpacked (tensors larger than the buffer go
        through it in pieces)."""
        if self.world == 1 or not tensors:
            return
        batch: List[torch.Tensor] = []
        used = 0

        def flush():
            nonlocal batch, used
            if not batch:
                return
            views = []
            o = 0
            for t in batch:
                nb = t.numel() * t.element_size()
                views.append(self._fusion_u8[o:o + nb].view(t.dtype).view(t.shape))
                o += (nb + 15) // 16 * 16
            if self.rank == root:
                torch._foreach_copy_(views, batch)
            self.broadcast_symm(self._fusion_u8[:o], root, stream)
            if self.rank != root:
                torch._foreach_copy_(batch, views)
            batch, used = [], 0

        for t in tensors:
            nb = t.numel() * t.element_size()
            if nb > self.fusion_bytes or not t.is_contiguous():
                flush()
                flat = t.contiguous().view(-1).view(torch.uint8)
                for s in range(0, flat.numel(), self.fusion_bytes):
                    piece = flat[s:s + self.fusion_bytes]
                    padded = (piece.numel() + 15) // 16 * 16
                    buf = self._fusion_u8[:padded]
                    if self.rank == root:
                        buf[:piece.numel()].copy_(piece)
                    self.broadcast_symm(buf, root, stream)
                    if self.rank != root:
                        piece.copy_(buf[:piece.numel()])
                if not t.is_contiguous() and self.rank != root:
                    t.copy_(flat.view(t.dtype).view(t.shape))
                continue
            padded = (nb + 15) // 16 * 16
            if used + padded > self.fusion_bytes:
                flush()
            batch.append(t)
            used += padded
        flush()

    def all_gather_symm(self, t: torch.Tensor, stream=None) -> torch.Tensor:
        """``t`` is [world * shard] in the arena; rank r's slice r is valid on entry."""
        off = self.arena.offset_of(t)
        shard_bytes = t.numel() * t.element_size() // self.world
        if self.world > 1:
            native.check(self.lib.tfy_allgather(self.arena.ctx_ref, off, shard_bytes, 0, 0, _stream_ptr(stream)),
                         "tfy_allgather")
            self.launches += 1
        return t

    def all_gather(self, shard: torch.Tensor, stream=None) -> torch.Tensor:
        """Gather equal-sized local shards; returns a new [world * n] tensor."""
        n = shard.numel()
        nbytes = n * shard.element_size()
        padded = (nbytes + 15) // 16 * 16
        if padded * self.world > self.fusion_bytes:
            raise ValueError("all_gather shard too large for the fusion buffer")
        buf = self._fusion_u8[:padded * self.world].view(self.world, padded)
        buf[self.rank, :nbytes].copy_(shard.contiguous().view(-1).view(torch.uint8))
        self.all_gather_symm(buf.view(-1), stream)
        return buf[:, :nbytes].contiguous().view(-1).view(shard.dtype).clone()

    def close(self) -> None:
        self.arena.close()


# ---------------------------------------------------------------------------
# K4: fused reduce-scatter -> optimizer -> all-gather over flat buffers
# ---------------------------------------------------------------------------
def hyper_block(spec: OptimizerSpec, step: int = 0):
    """The device hyper block of ``spec`` at ``step`` completed updates.  With a learning-rate schedule, ``hp.lr`` is
    the rate of the next update and the fused step writes each later one where it advances the step counter.  Nadam's
    block (``native.NadamHyperBlock``) adds the running product of its momentum schedule, 1 before any update: a
    block for a later step gets it from a checkpoint (``FusedShardedOptimizer.load_state``)."""
    blk = native.NadamHyperBlock(mu_product=1.0) if spec.kind == "nadam" else native.HyperBlock()
    blk.hp = native.OptHyper(spec.lr, spec.p1, spec.p2, spec.eps, spec.weight_decay, 1.0, step, spec.flags, 0, 0)
    if spec.schedule is not None:
        fields = dict(spec.schedule._device_fields())
        bounds, values = fields.pop("boundaries", ()), fields.pop("values", ())
        for k, v in fields.items():
            setattr(blk.sched, k, v)
        for i, b in enumerate(bounds):
            blk.sched.boundaries[i] = b
        for i, v in enumerate(values):
            blk.sched.values[i] = v
        blk.hp.lr = float(spec.schedule(step))
    return blk


def launch_code(spec: OptimizerSpec) -> int:
    """The ``opt`` code of a fused-step launch: the optimizer, plus ``OPT_LR_SCHEDULE`` when a schedule drives the
    learning rate (its instantiations advance the rate with the step counter; the others carry no schedule code)."""
    return spec.code | (native.OPT_LR_SCHEDULE if spec.schedule is not None else 0)


class FusedShardedOptimizer:
    """Flat parameter / gradient buffers + the fused K4 step.

    * ``params``  : replicated compute parameters, one flat symmetric buffer
      (bf16 or fp32); model parameters are views into it.
    * ``grads``   : flat symmetric gradient buffer (same layout); ``.grad`` of
      every model parameter is a view into it.
    * ``master`` / ``s1`` / ``s2`` : fp32 master weights and optimizer state of
      the 1/world shard this rank owns (ZeRO-1 layout).

    ``step()`` launches ONE kernel: in-switch reduce of the owned gradient
    shard (``multimem.ld_reduce``), bf16->fp32 cast and 1/world scaling, the
    optimizer update on the fp32 master shard, and the multicast store of the
    new parameters into every rank's replica (``multimem.st``).

    ``accumulation_steps=N`` (Keras ``gradient_accumulation_steps``) adds ``flat_acc``, an fp32 accumulator of the
    gradient buffer's layout in the symmetric arena (the same offset on every rank, where the step reads the peers'
    copies): :meth:`accumulate` adds a batch's gradients into it, and :meth:`step_accumulated` applies
    ``flat_acc * fl32(1/N)`` (``grad_scale``), averaged over the ranks, and clears it.
    """

    def __init__(self, comm: Communicator, shapes: Sequence[Sequence[int]], spec: OptimizerSpec,
                 param_dtype: torch.dtype = torch.bfloat16, grad_dtype: Optional[torch.dtype] = None,
                 zero_grads: bool = True, accumulation_steps: Optional[int] = None):
        self.comm, self.spec = comm, spec
        self.accum_steps = accumulation_steps
        self.param_dtype = param_dtype
        self.grad_dtype = grad_dtype or param_dtype
        self.zero_grads = zero_grads
        dev = f"cuda:{comm.device}"
        self.numels = []
        self.offsets = []
        o = 0
        for shp in shapes:
            n = 1
            for s in shp:
                n *= int(s)
            self.offsets.append(o)
            self.numels.append(n)
            o += (n + 7) // 8 * 8            # keep every tensor 16-byte aligned in bf16
        self.shapes = [tuple(int(s) for s in shp) for shp in shapes]
        self.n_real = o
        world = comm.world
        per = 8 * world
        self.n = (o + per - 1) // per * per
        self.shard_n = self.n // world
        arena = comm.arena
        self.param_off, self.flat_params = arena.empty((self.n,), self.param_dtype, align=4096)
        self.grad_off, self.flat_grads = arena.empty((self.n,), self.grad_dtype, align=4096)
        self.flat_params.zero_()
        self.flat_grads.zero_()
        self.master = torch.zeros(self.shard_n, dtype=torch.float32, device=dev)
        self.s1 = torch.full((self.shard_n,), spec.init_s1, dtype=torch.float32, device=dev)
        self.s2 = torch.zeros(spec.s2_numel(self.shard_n), dtype=torch.float32, device=dev)
        self._block = hyper_block(spec)
        self._code = launch_code(spec)
        self._hyper_host = self._block.hp
        self.acc_off, self.flat_acc = None, None
        if accumulation_steps is not None:
            self.acc_off, self.flat_acc = arena.empty((self.n,), torch.float32, align=4096)
            self.flat_acc.zero_()
            self._hyper_host.grad_scale = 1.0 / accumulation_steps      # rounded to fp32 by the ctypes field
        self.hyper = torch.zeros(ctypes.sizeof(self._block), dtype=torch.uint8, device=dev)
        self._push_hyper()
        self._sync_scheduled_lr()
        self.param_views = [self.flat_params[o:o + n].view(shp) for o, n, shp in
                            zip(self.offsets, self.numels, self.shapes)]
        self.grad_views = [self.flat_grads[o:o + n].view(shp) for o, n, shp in
                           zip(self.offsets, self.numels, self.shapes)]
        self.grid = 0
        self.block = 0

    # -- hyper-parameters (device resident so CUDA graphs see updates) --------
    def _push_hyper(self) -> None:
        raw = bytes(self._block)
        host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
        self.hyper.copy_(host)

    def _sync_scheduled_lr(self, stream=None) -> None:
        """With a schedule: ``hp.lr = schedule(hp.step)`` written on the device by the function the fused step
        evaluates, so the rate of an installed or restored step has the bits an uninterrupted run would read."""
        if self.spec.schedule is not None:
            native.check(self.comm.lib.tfy_lr_schedule_sync(self.hyper.data_ptr(), _stream_ptr(stream)),
                         "tfy_lr_schedule_sync")

    def set_lr(self, lr: float) -> None:
        """Update lr on the device (4-byte async copy; safe between graph replays)."""
        if self.spec.schedule is not None:
            raise TypeError("the learning rate of this optimizer follows a LearningRateSchedule, which the fused "
                            "step evaluates on the device; it cannot be set")
        self._hyper_host.lr = float(lr)
        t = torch.tensor([lr], dtype=torch.float32).view(torch.uint8)
        self.hyper[0:4].copy_(t, non_blocking=True)

    def set_grad_scale(self, s: float) -> None:
        self._hyper_host.grad_scale = float(s)
        t = torch.tensor([s], dtype=torch.float32).view(torch.uint8)
        self.hyper[20:24].copy_(t, non_blocking=True)

    @property
    def step_count(self) -> int:
        return int(self.hyper[24:28].view(torch.int32).item())

    def set_step_count(self, n: int) -> None:
        """Set the device step counter; with a schedule, also the rate of the next step (``schedule(n)``)."""
        self.hyper[24:28].copy_(torch.tensor([n], dtype=torch.int32).view(torch.uint8))
        self._sync_scheduled_lr()

    def current_lr(self) -> float:
        """The learning rate of the next step (with a schedule, the one the device holds: a 4-byte read)."""
        if self.spec.schedule is not None:
            return float(self.hyper[0:4].view(torch.float32).item())
        return float(self._hyper_host.lr)

    # -- initialisation ------------------------------------------------------
    def init_from(self, tensors: Sequence[torch.Tensor], broadcast_root: Optional[int] = 0) -> None:
        """Load initial values (fp32 source of truth), optionally broadcast rank ``root``'s."""
        full = torch.zeros(self.n, dtype=torch.float32, device=self.flat_params.device)
        for o, n, t in zip(self.offsets, self.numels, tensors):
            full[o:o + n].copy_(t.detach().reshape(-1).float())
        self.load_full_master(full, broadcast_root)

    def load_full_master(self, full: torch.Tensor, broadcast_root: Optional[int] = 0) -> None:
        comm = self.comm
        if comm.world > 1 and broadcast_root is not None:
            comm.broadcast([full], root=broadcast_root)
        r = comm.rank if comm.world > 1 else 0
        self.master.copy_(full[r * self.shard_n:(r + 1) * self.shard_n])
        self.flat_params.copy_(full.to(self.param_dtype))
        torch.cuda.current_stream().synchronize()
        if comm.world > 1:
            comm.barrier()

    # -- the hot path --------------------------------------------------------
    def step(self, stream=None, elem_range: Optional[Tuple[int, int]] = None, advance: bool = True,
             block: int = 0, shard_groups: Optional[Tuple[int, int]] = None) -> None:
        """One fused update.  ``elem_range=(e0, e1)`` restricts it to that element range of the flat buffers
        (multiples of 8): a step may be split into several launches -- e.g. the gradients that are final
        early on a side stream while backward continues -- with ``advance=True`` on the LAST one only, so
        that every launch of the step sees the same step counter.  ``shard_groups=(g0, g1)`` restricts it to
        groups of 8 elements RELATIVE TO EVERY RANK'S SHARD (the complement of :meth:`overlap_step`)."""
        c = self.comm
        if shard_groups is not None:
            if self.zero_grads:
                raise ValueError("ranged steps do not clear gradients: construct with zero_grads=False")
            g0, g1 = shard_groups
            rc = c.lib.tfy_fused_step_shard_range(
                c.arena.ctx_ref, _DT[self.grad_dtype], _DT[self.param_dtype], self._code, c.mode,
                self.grad_off, self.param_off, self.shard_n,
                self.master.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr(), self.hyper.data_ptr(),
                0, 0, int(block), int(g0), int(g1), int(advance), _stream_ptr(stream))
        elif elem_range is None and advance:
            rc = c.lib.tfy_fused_step(
                c.arena.ctx_ref, _DT[self.grad_dtype], _DT[self.param_dtype], self._code, c.mode,
                self.grad_off, self.param_off, self.shard_n,
                self.master.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr(), self.hyper.data_ptr(),
                int(self.zero_grads), self.grid, self.block, _stream_ptr(stream))
        else:
            if self.zero_grads:
                raise ValueError("ranged steps do not clear gradients: construct with zero_grads=False")
            e0, e1 = elem_range if elem_range is not None else (0, self.n)
            if e0 % 8 or e1 % 8 or not 0 <= e0 <= e1 <= self.n:
                raise ValueError(f"bad element range {elem_range} for a buffer of {self.n}")
            rc = c.lib.tfy_fused_step_range(
                c.arena.ctx_ref, _DT[self.grad_dtype], _DT[self.param_dtype], self._code, c.mode,
                self.grad_off, self.param_off, self.shard_n,
                self.master.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr(), self.hyper.data_ptr(),
                0, 0, int(block), e0, e1, int(advance), _stream_ptr(stream))
        native.check(rc, "tfy_fused_step")
        c.launches += 1

    def accumulate(self, advance: bool, stream=None) -> None:
        """``flat_acc += flat_grads`` in fp32 (one launch), clearing the gradients behind it when the optimizer was
        built with ``zero_grads``.  ``advance``: this batch is not an update, so this launch advances the step counter
        (and a scheduled learning rate) instead of the fused step."""
        if self.flat_acc is None:
            raise ValueError("accumulate() needs an optimizer constructed with accumulation_steps")
        c = self.comm
        native.check(c.lib.tfy_grad_accumulate(
            self.flat_acc.data_ptr(), self.flat_grads.data_ptr(), _DT[self.grad_dtype], self.n, int(self.zero_grads),
            self.hyper.data_ptr(), int(self.spec.schedule is not None), int(advance), _stream_ptr(stream)),
            "tfy_grad_accumulate")
        c.launches += 1

    def step_accumulated(self, stream=None) -> None:
        """The update of an accumulation: the fused step over ``flat_acc`` (fp32 gradients, scaled by ``grad_scale``
        = fl32(1/N)), which clears the accumulator behind itself and advances the step counter."""
        if self.flat_acc is None:
            raise ValueError("step_accumulated() needs an optimizer constructed with accumulation_steps")
        c = self.comm
        native.check(c.lib.tfy_fused_step(
            c.arena.ctx_ref, native.F32, _DT[self.param_dtype], self._code, c.mode, self.acc_off, self.param_off,
            self.shard_n, self.master.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr(), self.hyper.data_ptr(),
            1, self.grid, self.block, _stream_ptr(stream)), "tfy_fused_step")
        c.launches += 1

    def pending_accumulation(self) -> bool:
        """True when batches have been accumulated since the last update."""
        return self.accum_steps is not None and self.step_count % self.accum_steps != 0

    def overlap_step(self, g0: int, g1: int, n_cta: int, slot0: int = 960):
        """Descriptor of the fused step of shard-relative groups ``[g0, g1)`` for the communication CTAs of a
        persistent compute kernel (``tfy_conv3x3_c32_wgrad_unpool_ov``): they reduce-scatter, update and
        all-gather those parameters over NVLink WHILE the kernel's compute CTAs run, so that part of the
        gradient exchange costs no step time.  bf16 gradients / parameters only.  The trailing
        ``step(shard_groups=(0, g0))`` of the same training step publishes the result (its exit barrier)."""
        if self.grad_dtype != torch.bfloat16 or self.param_dtype != torch.bfloat16:
            raise ValueError("overlap_step needs bf16 gradients and parameters")
        if self.spec.kind == "rmsprop":
            raise ValueError("overlap_step does not run RMSprop: its states do not fit the descriptor; "
                             "update every group with step()")
        if self.spec.kind in ("adamax", "nadam"):
            raise ValueError(f"overlap_step does not run {self.spec.kind.capitalize()}: the communication role has no "
                             "instantiation for it; update every group with step()")
        c = self.comm
        ov = native.OverlapStep()
        ov.c = c.arena.ctx
        ov.grad_off, ov.param_off, ov.shard_n = self.grad_off, self.param_off, self.shard_n
        ov.master, ov.s1, ov.s2 = self.master.data_ptr(), self.s1.data_ptr(), self.s2.data_ptr()
        ov.hp = self.hyper.data_ptr()
        ov.g0, ov.g1 = int(g0), int(min(g1, self.shard_n // 8))
        ov.opt, ov.mode, ov.n_cta, ov.slot0 = self.spec.code, c.mode, int(n_cta), int(slot0)
        return ov

    # -- checkpoint support ----------------------------------------------------
    def _states(self):
        """(name, shard) of every fp32 array the step updates; the states after ``s1`` are consecutive
        ``shard_n``-long parts of the ``s2`` buffer."""
        out = [("master", self.master), ("s1", self.s1)]
        for i in range(1, self.spec.n_states):
            out.append((f"s{i + 1}", self.s2[(i - 1) * self.shard_n:i * self.shard_n]))
        return out

    def gather_state(self) -> dict:
        """Materialise full (unsharded) fp32 master / state tensors on every rank."""
        out = {name: self._gather_full(t) for name, t in self._states()}
        out["step"] = self.step_count
        if self.spec.kind == "nadam":
            out["mu_product"] = self.mu_product
        if self.pending_accumulation():
            # the sum of the batches since the last update; over several ranks, the sum of every rank's (a
            # collective, as the gathers above): a resume puts it on rank 0, so the next update sees the same total
            # up to the order of the fp32 sums
            acc = self.flat_acc.clone()
            if self.comm.world > 1:
                self.comm.all_reduce([acc], average=False)
            out["grad_accum"] = acc
        return out

    def _gather_full(self, shard: torch.Tensor) -> torch.Tensor:
        c = self.comm
        if c.world == 1:
            return shard.clone()
        pieces = []
        chunk = max(8, (c.fusion_bytes // (4 * c.world)) // 8 * 8)
        for s in range(0, self.shard_n, chunk):
            part = shard[s:s + chunk]
            g = c.all_gather(part).view(c.world, -1)
            pieces.append(g)
        return torch.cat(pieces, dim=1).reshape(-1)

    def load_state(self, state: dict) -> None:
        r = self.comm.rank if self.comm.world > 1 else 0
        sl = slice(r * self.shard_n, (r + 1) * self.shard_n)
        for name, t in self._states():
            if name in ("master", "s1") or name in state:
                t.copy_(state[name][sl])
        self.flat_params.copy_(state["master"].to(self.flat_params.device).to(self.param_dtype))
        if self.flat_acc is not None:
            if "grad_accum" in state and r == 0:
                self.flat_acc.copy_(state["grad_accum"])
            else:
                self.flat_acc.zero_()
        self.set_step_count(int(state.get("step", 0)))
        if self.spec.kind == "nadam":
            self._mu_product_bytes().copy_(torch.tensor([float(state.get("mu_product", 1.0))],
                                                        dtype=torch.float64).view(torch.uint8))

    def _mu_product_bytes(self) -> torch.Tensor:
        off = native.NadamHyperBlock.mu_product.offset
        return self.hyper[off:off + 8]

    @property
    def mu_product(self) -> float:
        """Nadam: the running product of the momentum schedule after the completed updates (float64, on the
        device)."""
        return float(self._mu_product_bytes().view(torch.float64).item())

    def unflatten(self, full: torch.Tensor) -> List[torch.Tensor]:
        return [full[o:o + n].view(shp) for o, n, shp in zip(self.offsets, self.numels, self.shapes)]
