"""Train-step engines behind ``Model.fit``.

``GraphTrainEngine`` (H100) — the flagship path of the Horovod-style Keras
configuration:

* parameters live in ONE flat bf16 buffer in the symmetric arena, gradients in
  another; model parameters / ``.grad`` are views into them; fp32 master
  weights and optimizer state are sharded 1/world per rank;
* one training step = forward + backward (cuDNN/cuBLAS bf16 through torch
  autograd) followed by ONE hand-written kernel that does the cross-GPU
  gradient reduction, the bf16->fp32 cast + 1/world scale, the optimizer update
  on the owned shard and the all-gather of the new bf16 parameters
  (``tfy_fused_step_kernel``: multimem.ld_reduce / multimem.st over NVSwitch);
* the whole step is captured in a CUDA graph and replayed; inputs are staged
  from pinned host memory on a copy stream one step ahead; the loss is read
  back asynchronously into a pinned ring.

``EagerTrainEngine`` (CPU plumbing configuration) — plain torch ops, gloo
all-reduce of the gradients, ``torch.optim`` with the same update formulas.

With ``gradient_accumulation_steps=N`` (Keras 3) the engines count batches, not updates: batch ``s`` adds its
gradients to an fp32 sum, and batch ``s`` with ``(s + 1) % N == 0`` applies ``sum * fl32(1/N)`` (averaged over the
ranks) with the learning rate ``schedule(s)`` and Adam's bias correction at ``t = s + 1``, then clears the sum.
"""
from __future__ import annotations

import ctypes

import logging
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from tf_yarn_b200.keras import losses as loss_mod
from tf_yarn_b200.keras import weighting
from tf_yarn_b200.keras.metrics import Metric

logger = logging.getLogger(__name__)


def _to_device_batch(t, device, non_blocking=True):
    if isinstance(t, (tuple, list)):
        return type(t)(_to_device_batch(x, device, non_blocking) for x in t)
    if isinstance(t, dict):
        return {k: _to_device_batch(v, device, non_blocking) for k, v in t.items()}
    return t.to(device, non_blocking=non_blocking)


class EagerTrainEngine:
    """Reference-semantics engine for CPU (and the fp32 numerics oracle for the graph engine)."""

    def __init__(self, net: nn.Module, loss_fn: Callable, optimizer, metric_fns: Sequence[Tuple[str, Callable]],
                 device: torch.device, distributed: bool = False,
                 weighted_metric_fns: Sequence[Tuple[str, Callable]] = ()):
        self.net, self.loss_fn, self.metric_fns = net, loss_fn, list(metric_fns)
        self.weighted_metric_fns = list(weighted_metric_fns)
        self.device = device
        self.distributed = distributed
        self.opt_desc = optimizer
        self.opt = optimizer.to_torch([p for p in net.parameters() if p.requires_grad])
        self._schedule = getattr(optimizer, "schedule", None)
        self.accum_steps = getattr(optimizer, "gradient_accumulation_steps", None)
        if self.accum_steps is not None:
            # .grad is the accumulator and lives on the module's parameters: a previous fit (whose last gradients
            # stay there) must not leak into the first update.  load_state_dict puts a saved pending sum back.
            for p in net.parameters():
                p.grad = None
        self.iterations = 0                 # batches trained (Keras optimizer.iterations): a schedule's step
        self.kernel_launches = 0
        self._cw = None                     # class-weight table [C] on the device (None: no class_weight)
        self._wacc = [[0.0, 0.0] for _ in self.weighted_metric_fns]     # epoch sums (sum w*m, sum w)

    def set_class_weight(self, table: Optional[torch.Tensor]) -> None:
        """Class-weight table of the following steps (None: off)."""
        self._cw = table.to(self.device, torch.float32).reshape(-1) if table is not None else None

    # -- distributed helpers (gloo) -------------------------------------------
    def _world(self) -> int:
        import torch.distributed as dist
        return dist.get_world_size() if (self.distributed and dist.is_initialized()) else 1

    def broadcast_variables(self, root: int = 0) -> None:
        import torch.distributed as dist
        if self._world() > 1:
            for t in list(self.net.parameters()) + list(self.net.buffers()):
                dist.broadcast(t.data, src=root)

    def train_step(self, x, y, w=None) -> Dict[str, torch.Tensor]:
        self.net.train()
        x, y = _to_device_batch(x, self.device), _to_device_batch(y, self.device)
        if self.accum_steps is None:
            self.opt.zero_grad(set_to_none=False)
        out = self.net(x)
        sw = None
        if w is None and self._cw is None:
            loss = self.loss_fn(y, out)
        else:
            sw = weighting.sample_weights(y, w.to(self.device) if w is not None else None, self._cw)
            loss = weighting.weighted_loss(loss_mod.per_sample(self.loss_fn), y, out, sw)
        loss.backward()              # with accumulation: .grad += this batch's gradients (fp32, in batch order)
        if self.accum_steps is None or (self.iterations + 1) % self.accum_steps == 0:
            self._apply_gradients()
        self.iterations += 1
        logs = {"loss": loss.detach()}
        with torch.no_grad():
            for name, fn in self.metric_fns:
                if isinstance(fn, Metric):
                    fn.update_state(y, out)
                    continue
                num, den = fn(y, out)
                logs[name] = num / den
            for acc, (_, fn) in zip(self._wacc, self.weighted_metric_fns):
                if isinstance(fn, Metric):
                    fn.update_state(y, out, sample_weight=sw)
                    continue
                num, den = fn(y, out, sample_weight=sw)
                acc[0] += float(num)
                acc[1] += float(den)
        return logs

    def _apply_gradients(self) -> None:
        """The update of batch ``self.iterations``: the gradients averaged over the ranks (and, accumulating, the sum
        of the last N batches scaled by fl32(1/N)), the learning rate at ``iterations``; then, accumulating, the sum
        is cleared."""
        import torch.distributed as dist
        world = self._world()
        if world > 1:
            grads = [p.grad for p in self.net.parameters() if p.grad is not None]
            flat = torch.cat([g.reshape(-1) for g in grads])
            dist.all_reduce(flat)
            flat /= world
            o = 0
            for g in grads:
                g.copy_(flat[o:o + g.numel()].view_as(g))
                o += g.numel()
        if self._schedule is not None:
            lr = float(self._schedule(self.iterations))
            for g in self.opt.param_groups:
                g["lr"] = lr
        if self.accum_steps is not None:
            scale = float(np.float32(1.0 / self.accum_steps))
            for p in self.net.parameters():
                if p.grad is not None:
                    p.grad.mul_(scale)
            self._align_adam_step()
        self.opt.step()
        if self.accum_steps is not None:
            self.opt.zero_grad(set_to_none=False)

    def _align_adam_step(self) -> None:
        """Keras 3 applies the update of batch ``s`` with Adam's bias correction at ``t = s + 1`` (``iterations``
        counts batches); ``torch.optim.Adam`` counts its own steps, so its counter is set to ``s`` before it adds 1.
        The same holds for Adamax's bias correction and Nadam's momentum schedule."""
        from tf_yarn_b200.keras.optimizers import TorchAdamax
        if not isinstance(self.opt, (torch.optim.Adam, torch.optim.AdamW, torch.optim.NAdam, TorchAdamax)):
            return
        from torch.optim.optimizer import _get_scalar_dtype
        for grp in self.opt.param_groups:
            for p in grp["params"]:
                st = self.opt.state[p]
                if not st:                  # the lazy initialisation of the optimizer, with the step set
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if isinstance(self.opt, TorchAdamax):
                        st["exp_inf"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    else:
                        st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if grp.get("amsgrad"):
                        st["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if isinstance(self.opt, torch.optim.NAdam):     # Nadam's product advances on updates only
                        st["mu_product"] = torch.ones((), dtype=_get_scalar_dtype())
                st["step"] = torch.tensor(float(self.iterations), dtype=_get_scalar_dtype())

    @property
    def stateful_metrics(self) -> List[Metric]:
        return [fn for _, fn in self.metric_fns + self.weighted_metric_fns if isinstance(fn, Metric)]

    def pop_metrics(self) -> Dict[str, float]:
        """The weighted metrics of the steps since the last call, ``sum(w*m) / sum(w)`` over all of them, and the
        results of the stateful metrics (AUC, ...), which are then reset."""
        out = {name: fn.result() for name, fn in self.metric_fns if isinstance(fn, Metric)}
        for (name, fn), (num, den) in zip(self.weighted_metric_fns, self._wacc):
            out[name] = fn.result() if isinstance(fn, Metric) else (num / den if den else 0.0)
        self._wacc = [[0.0, 0.0] for _ in self.weighted_metric_fns]
        for m in self.stateful_metrics:
            m.reset_state()
        return out

    def set_learning_rate(self, lr: float) -> None:
        if self._schedule is not None:
            raise TypeError("the learning rate of this optimizer follows a LearningRateSchedule; it cannot be set")
        for g in self.opt.param_groups:
            g["lr"] = lr

    def get_learning_rate(self) -> float:
        if self._schedule is not None:
            return float(self._schedule(self.iterations))
        return self.opt.param_groups[0]["lr"]

    def sync_params_to_module(self) -> None:
        pass

    def _pending_accumulation(self) -> bool:
        return self.accum_steps is not None and self.iterations % self.accum_steps != 0

    def state_dict(self) -> dict:
        """With batches accumulated since the last update, the state carries their sum (``grad_accum``).  A
        checkpoint is written by one rank alone, without a collective, so over several ranks it holds that rank's part
        of the sum only.  A resume puts it back on rank 0 and zeros on the others, so the first update after it lacks
        the other ranks' pending batches while still dividing by ``world * N`` (a warning says so at save time;
        docs/Migration.md states it).  The GPU engines gather every rank's part and have no such gap."""
        st = {"kind": "eager", "optimizer": self.opt.state_dict(), "iterations": self.iterations}
        if self._pending_accumulation():
            if self._world() > 1:
                logger.warning("checkpoint in the middle of a gradient accumulation over %d ranks: only this rank's "
                               "pending gradients are saved, so the first update after resuming from it leaves out "
                               "the other ranks' pending batches", self._world())
            st["grad_accum"] = [p.grad.detach().clone() if p.grad is not None else None
                                for p in self.net.parameters() if p.requires_grad]
        return st

    def load_state_dict(self, state: dict) -> None:
        if state.get("kind") == "eager":
            self.opt.load_state_dict(state["optimizer"])
            self.iterations = int(state.get("iterations", 0))
            if self.accum_steps is not None:
                pending = state.get("grad_accum")
                first = self._world() == 1 or _rank() == 0
                for i, p in enumerate(p for p in self.net.parameters() if p.requires_grad):
                    g = pending[i] if (pending is not None and first) else None
                    p.grad = g.to(p.device).clone() if g is not None else torch.zeros_like(p)

    # fit() drives the eager engine synchronously
    pipelined = False


class GraphTrainEngine:
    """CUDA-graph train step with the fused reduce-scatter/optimizer/all-gather kernel."""

    pipelined = True
    accum_steps: Optional[int] = None        # the optimizer's gradient_accumulation_steps

    def __init__(self, net: nn.Module, loss_fn: Callable, optimizer, metric_fns: Sequence[Tuple[str, Callable]],
                 device: torch.device, distributed: bool, example_x, example_y,
                 compute_dtype: torch.dtype = torch.bfloat16, use_graph: bool = True, comm=None,
                 weighted_metric_fns: Sequence[Tuple[str, Callable]] = ()):
        from tf_yarn_b200.parallel import runtime
        from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
        self.net, self.loss_fn, self.metric_fns = net, loss_fn, list(metric_fns)
        self.weighted_metric_fns = list(weighted_metric_fns)
        self.device = device
        self.compute_dtype = compute_dtype
        self.use_graph = use_graph
        self.opt_desc = optimizer
        torch.cuda.set_device(device)
        if comm is None:
            if distributed:
                comm = runtime.get_communicator(device=device.index)
            else:
                from tf_yarn_b200.parallel.comm import Communicator
                from tf_yarn_b200.parallel.symm import SoloRendezvous
                comm = _solo_communicator(device.index)
        self.comm = comm
        self.distributed = distributed and comm.world > 1
        self.params = [p for p in net.parameters() if p.requires_grad]
        # fp32 source of truth, in the byte order of the flat buffers: conv kernels are stored
        # (O, kh, kw, I) so that the parameter seen by cuDNN is a channels_last view of its slice
        init = [p.detach().float().permute(0, 2, 3, 1).contiguous() if p.dim() == 4 else p.detach().float()
                for p in self.params]
        # gradient_accumulation_steps: two captured graphs per input slot, an accumulation batch (forward, backward,
        # accumulate + advance the step counter) and an update batch (forward, backward, accumulate, fused step over
        # the accumulator); the host picks one from its batch counter
        self.accum_steps = getattr(optimizer, "gradient_accumulation_steps", None)
        self._batch = 0                      # batches launched (the device step counter, which counts batches)
        self.fused = FusedShardedOptimizer(comm, [tuple(t.shape) for t in init], optimizer.to_spec(),
                                           param_dtype=compute_dtype, grad_dtype=compute_dtype, zero_grads=True,
                                           accumulation_steps=self.accum_steps)
        self.fused.init_from(init, broadcast_root=None)
        net.to(compute_dtype)
        # re-point the module's parameters / grads at the flat symmetric buffers
        for p, pv, gv in zip(self.params, self.fused.param_views, self.fused.grad_views):
            if p.dim() == 4:
                pv, gv = pv.permute(0, 3, 1, 2), gv.permute(0, 3, 1, 2)
            p.data, p.grad = pv, gv
        self.stream = torch.cuda.Stream(device=device)
        self.copy_stream = torch.cuda.Stream(device=device)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self._static_x = None
        self._static_y = None
        self._staging = None            # two device-side input slots filled by the copy stream
        self._slot = 0
        self._slot_free = [None, None]  # event: the step that read staging[slot] has copied it out
        self._loss = torch.zeros((), dtype=torch.float32, device=device)
        # rows: the metrics, then the weighted metrics (sum w*m, sum w)
        self._metric_acc = torch.zeros(max(1, len(self.metric_fns) + len(self.weighted_metric_fns)), 2,
                                       dtype=torch.float32, device=device)
        self._example = (example_x, example_y)
        self.kernel_launches = 0
        self._launches_per_step = 1          # the fused K4 kernel (accumulating: + the accumulate kernel)
        self._launches_per_accum_step = 1    # accumulating: the accumulate kernel of an accumulation batch
        if self.accum_steps is not None:
            self._launches_per_step = 2
        self._captured = False
        # Keras sample weighting.  The weighting mode -- (class_weight, sample_weight) -- is part of the captured
        # graphs: a step in another mode captures them again.  The class-weight table is an engine-owned device
        # buffer read by the graphs, so a new table of the same size is copied in place without a recapture;
        # sample weights get a [B] buffer per staging slot.
        self._cw: Optional[torch.Tensor] = None
        self._cw_on = False
        self._wmode = (False, False)
        self._staging_w = [None, None]

    def set_class_weight(self, table: Optional[torch.Tensor]) -> None:
        """Class-weight table ``[C]`` of the following steps (None: off)."""
        if table is None:
            self._cw_on = False
            return
        table = table.to(torch.float32).reshape(-1)
        if self._cw is None or self._cw.numel() != table.numel():
            if self._wmode[0]:
                self._captured = False       # the graphs read the old buffer
            self._cw = torch.empty(table.numel(), dtype=torch.float32, device=self.device)
        with torch.cuda.stream(self.stream):  # ordered after the steps already queued, before the next ones
            self._cw.copy_(table)
        self.stream.synchronize()
        self._cw_on = True

    # ------------------------------------------------------------------ variables
    def broadcast_variables(self, root: int = 0) -> None:
        """Make every rank start from rank ``root``'s weights (BroadcastGlobalVariablesCallback)."""
        if not self.distributed:
            return
        full = self._full_master()
        self.fused.load_full_master(full, broadcast_root=root)

    def _full_master(self) -> torch.Tensor:
        return self.fused.gather_state()["master"] if self.comm.world > 1 else self.fused.master.clone()

    def master_tensors(self) -> List[torch.Tensor]:
        """Full-precision parameters in module layout (for checkpoints / evaluation)."""
        full = self._full_master()
        out = []
        for p, t in zip(self.params, self.fused.unflatten(full)):
            out.append(t.permute(0, 3, 1, 2) if p.dim() == 4 else t)
        return out

    def sync_params_to_module(self) -> None:
        pass  # module parameters ARE the flat buffer

    # ------------------------------------------------------------------ step body
    def _apply_gradients(self, update: bool) -> int:
        """The end of a step: the fused optimizer step, or -- accumulating -- the accumulate kernel, followed on an
        update batch by the fused step over the accumulator.  Returns the launches made."""
        if self.accum_steps is None:
            self.fused.step()
            return 1
        self.fused.accumulate(advance=not update)
        if update:
            self.fused.step_accumulated()
        return 2 if update else 1

    def _next_is_update(self) -> bool:
        return self.accum_steps is None or (self._batch + 1) % self.accum_steps == 0

    def _forward_backward(self, x, y, w=None, update: bool = True) -> None:
        xin = x
        if torch.is_tensor(xin) and torch.is_floating_point(xin):
            xin = xin.to(self.compute_dtype)
        out = self.net(xin)
        sw = None
        if self._wmode == (False, False):
            loss = self.loss_fn(y, out)
        else:
            sw = weighting.sample_weights(y, w, self._cw if self._wmode[0] else None)
            loss = weighting.weighted_loss(loss_mod.per_sample(self.loss_fn), y, out, sw)
        loss.backward()
        self._loss.copy_(loss.detach())
        if self.metric_fns:
            with torch.no_grad():
                for i, (_, fn) in enumerate(self.metric_fns):
                    if isinstance(fn, Metric):          # stateful: one histogram kernel launch, state on the device
                        fn.update_state(y, out)
                        continue
                    num, den = fn(y, out)
                    self._metric_acc[i, 0] += num
                    self._metric_acc[i, 1] += den
        if self.weighted_metric_fns:
            with torch.no_grad():
                for i, (_, fn) in enumerate(self.weighted_metric_fns, start=len(self.metric_fns)):
                    if isinstance(fn, Metric):
                        fn.update_state(y, out, sample_weight=sw)
                        continue
                    num, den = fn(y, out, sample_weight=sw)
                    self._metric_acc[i, 0] += num
                    self._metric_acc[i, 1] += den
        self._apply_gradients(update)

    def _capture(self, x, y, w=None) -> None:
        self.net.train()
        # two input slots, and one captured graph per slot reading it in place: the copy stream fills slot
        # (i+1) % 2 while graph[i % 2] runs, and no staging -> static copy sits in front of every step
        self._staging = [(_clone_struct(x), _clone_struct(y)) for _ in range(2)]
        self._static_x, self._static_y = self._staging[0]
        self._wmode = (self._cw_on, w is not None)
        self._staging_w = [w.reshape(-1).float().clone() if w is not None else None for _ in range(2)]
        if getattr(self, "_loss_host", None) is None:
            # (a recapture keeps them: the loss of the step queued before it is still to be read)
            self._loss_host = [torch.zeros((), dtype=torch.float32).pin_memory() for _ in range(2)]
        self._loss_in_host = [False, False]
        self._capture_slot = None
        self._ready_ev = [torch.cuda.Event() for _ in range(2)]
        self._done_ev = [torch.cuda.Event() for _ in range(2)]
        from tf_yarn_b200.ops import native
        native.declare("tfy_memcpy_async", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p])
        self._lib = native.load()
        self._fast_copy = hasattr(self._lib, "tfy_memcpy_async")
        fused = self.fused
        snap = (fused.master.clone(), fused.s1.clone(), fused.s2.clone(), fused.flat_params.clone(),
                fused.hyper.clone(), self._metric_acc.clone(),
                fused.flat_acc.clone() if fused.flat_acc is not None else None)
        # stateful metrics allocate their device state on their first update (a warm-up step): empty until then
        metric_snap = [[t.clone() for t in m.state_tensors()] for m in self.stateful_metrics]
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            for i in range(3):          # accumulating: an accumulation, an update and an accumulation batch
                self._forward_backward(self._static_x, self._static_y, self._staging_w[0],
                                       update=self.accum_steps is None or i == 1)
        self.stream.synchronize()
        self.graphs = [None, None]
        self._acc_graphs = [None, None]
        if self.use_graph:
            # a CUDAGraph of an older engine being garbage-collected while this stream captures would
            # invalidate the capture (cudaGraphExecDestroy is not allowed then): collect now, pause GC
            import gc
            gc.collect()
            was_enabled = gc.isenabled()
            gc.disable()
            try:
                for slot in range(2):
                    for update in ((True,) if self.accum_steps is None else (True, False)):
                        g = torch.cuda.CUDAGraph()
                        sx, sy = self._staging[slot]
                        sw = self._staging_w[slot]
                        # the graphs never run concurrently (same stream), so they share one memory pool
                        pool = self.graphs[0].pool() if self.graphs[0] is not None else None
                        self._capture_slot = slot
                        with torch.cuda.graph(g, stream=self.stream, pool=pool):
                            self._forward_backward(sx, sy, sw, update)
                            if not self._loss_in_host[slot]:      # (the fast path's head kernel writes it itself)
                                self._loss_host[slot].copy_(self._loss, non_blocking=True)  # D2H node of the graph
                        self._capture_slot = None
                        (self.graphs if update else self._acc_graphs)[slot] = g
                self.graph = self.graphs[0]
            finally:
                if was_enabled:
                    gc.enable()
        # undo the warm-up steps: training starts from the user's initial state
        with torch.cuda.stream(self.stream):
            fused.master.copy_(snap[0]); fused.s1.copy_(snap[1]); fused.s2.copy_(snap[2])
            fused.flat_params.copy_(snap[3]); fused.hyper.copy_(snap[4]); self._metric_acc.copy_(snap[5])
            if snap[6] is not None:
                fused.flat_acc.copy_(snap[6])
            fused.flat_grads.zero_()
            for m, saved in zip(self.stateful_metrics, metric_snap):
                if saved:
                    for t, v in zip(m.state_tensors(), saved):
                        t.copy_(v)
                else:
                    m.reset_state()
        self.stream.synchronize()
        if self.distributed:
            self.comm.barrier()
            torch.cuda.synchronize()
        self._captured = True

    # ------------------------------------------------------------------ public
    def ensure_captured(self, x, y, w=None) -> None:
        if self._captured and self._wmode != (self._cw_on, w is not None):
            self._captured = False          # another weighting mode: capture the step graphs again
        if not self._captured:
            self._capture(_to_device_batch(x, self.device, False), _to_device_batch(y, self.device, False),
                          w.to(self.device) if w is not None else None)

    def stage_inputs(self, x, y, w=None):
        """Asynchronous copy (H2D from pinned memory, or D2D) of the next batch -- and of its sample weights
        ``w`` [B], if any -- into a staging slot.

        Runs on the copy stream, so it overlaps the step that is currently executing.  Returns a
        ticket for :meth:`launch_step`.
        """
        self.ensure_captured(x, y, w)
        slot = self._slot
        self._slot ^= 1
        sx, sy = self._staging[slot]
        sw = self._staging_w[slot]
        cs = self.copy_stream
        free = self._slot_free[slot]
        if free is not None:
            cs.wait_event(free)
        if (self._fast_copy and torch.is_tensor(x) and torch.is_tensor(y) and x.dtype == sx.dtype
                and y.dtype == sy.dtype and x.is_contiguous() and y.is_contiguous()
                and x.numel() == sx.numel() and y.numel() == sy.numel()
                and (w is None or (w.dtype == sw.dtype and w.is_contiguous() and w.numel() == sw.numel()))):
            # hot path: two cudaMemcpyAsync calls through ctypes, no stream context manager (three with weights)
            lib, sp = self._lib, cs.cuda_stream
            lib.tfy_memcpy_async(sx.data_ptr(), x.data_ptr(), x.numel() * x.element_size(), sp)
            lib.tfy_memcpy_async(sy.data_ptr(), y.data_ptr(), y.numel() * y.element_size(), sp)
            if w is not None:
                lib.tfy_memcpy_async(sw.data_ptr(), w.data_ptr(), w.numel() * w.element_size(), sp)
        else:
            with torch.cuda.stream(cs):
                _copy_struct(sx, x)
                _copy_struct(sy, y)
                if w is not None:
                    sw.copy_(w.reshape(-1), non_blocking=True)
        ev = self._ready_ev[slot]
        ev.record(cs)
        return slot, ev

    def launch_step(self, ticket) -> torch.cuda.Event:
        """Run one captured step on the staged batch; returns the event marking its completion.

        The step's loss is copied to ``loss_host(slot)`` (pinned) by the graph itself."""
        slot, ready = ticket
        st = self.stream
        st.wait_event(ready)
        update = self._next_is_update()
        if torch.cuda.current_stream() == st:
            self._launch_on_current(slot, update)
        else:
            with torch.cuda.stream(st):
                self._launch_on_current(slot, update)
        done = self._done_ev[slot]
        done.record(st)
        self._slot_free[slot] = done          # the slot may be refilled once this step has run
        self._batch += 1
        self.kernel_launches += self._launches_per_step if update else self._launches_per_accum_step
        return done

    def _launch_on_current(self, slot: int, update: bool = True) -> None:
        if self.graph is not None:
            (self.graphs if update else self._acc_graphs)[slot].replay()
        else:
            sx, sy = self._staging[slot]
            self._forward_backward(sx, sy, self._staging_w[slot], update)
            self._loss_host[slot].copy_(self._loss, non_blocking=True)

    def loss_host(self, slot: int) -> torch.Tensor:
        """Pinned scalar that receives the loss of the steps run on ``slot`` (valid once their event fired)."""
        return self._loss_host[slot]

    def read_loss_async(self, pinned_slot: torch.Tensor) -> None:
        with torch.cuda.stream(self.stream):
            pinned_slot.copy_(self._loss, non_blocking=True)

    def train_step(self, x, y, w=None) -> Dict[str, torch.Tensor]:
        """Synchronous convenience wrapper (tests, smoke): one step, returns device scalars."""
        ticket = self.stage_inputs(x, y) if w is None else self.stage_inputs(x, y, w)
        self.launch_step(ticket)
        self.stream.synchronize()
        return {"loss": self._loss.clone()}

    @property
    def stateful_metrics(self) -> List[Metric]:
        return [fn for _, fn in self.metric_fns + self.weighted_metric_fns if isinstance(fn, Metric)]

    def pop_metrics(self) -> Dict[str, float]:
        self.stream.synchronize()
        acc = self._metric_acc.cpu()
        self._metric_acc.zero_()
        out = {}
        for i, (name, fn) in enumerate(self.metric_fns):
            out[name] = fn.result() if isinstance(fn, Metric) else float(acc[i, 0] / acc[i, 1].clamp_min(1))
        for i, (name, fn) in enumerate(self.weighted_metric_fns, start=len(self.metric_fns)):
            if isinstance(fn, Metric):
                out[name] = fn.result()
            else:
                out[name] = float(acc[i, 0] / acc[i, 1]) if float(acc[i, 1]) != 0.0 else 0.0
        with torch.cuda.stream(self.stream):            # ordered before the next epoch's steps
            for m in self.stateful_metrics:
                m.reset_state()
        return out

    def set_learning_rate(self, lr: float) -> None:
        with torch.cuda.stream(self.stream):
            self.fused.set_lr(lr)

    def get_learning_rate(self) -> float:
        return self.fused.current_lr()

    def state_dict(self) -> dict:
        st = self.fused.gather_state()
        return {"kind": "fused", **{k: (v.cpu() if torch.is_tensor(v) else v) for k, v in st.items()}}

    def load_state_dict(self, state: dict) -> None:
        if state.get("kind") == "fused":
            dev = self.fused.master.device
            self.fused.load_state({k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in state.items()
                                   if k != "kind"})
            self._batch = int(state.get("step", 0))


def _rank() -> int:
    import torch.distributed as dist
    return dist.get_rank() if dist.is_initialized() else 0


_solo = {}


def _solo_communicator(device_index: int):
    """Single-GPU communicator (world=1): the fused kernel runs in LOCAL mode, no peers."""
    from tf_yarn_b200.parallel.comm import Communicator
    from tf_yarn_b200.parallel.symm import SoloRendezvous
    if device_index not in _solo:
        _solo[device_index] = Communicator(arena_bytes=1 << 30, fusion_bytes=16 << 20, rdv=SoloRendezvous(),
                                           device=device_index)
    return _solo[device_index]


def _clone_struct(t):
    if isinstance(t, (tuple, list)):
        return type(t)(_clone_struct(x) for x in t)
    if isinstance(t, dict):
        return {k: _clone_struct(v) for k, v in t.items()}
    return t.clone()


def _copy_struct(dst, src) -> None:
    if isinstance(dst, (tuple, list)):
        for d, s in zip(dst, src):
            _copy_struct(d, s)
    elif isinstance(dst, dict):
        for k in dst:
            _copy_struct(dst[k], src[k])
    else:
        dst.copy_(src, non_blocking=True)
