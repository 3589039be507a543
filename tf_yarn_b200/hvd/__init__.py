"""Horovod-shaped facade over the H100 comm runtime.

User code written for the reference's all-reduce path keeps working::

    import tf_yarn_b200.hvd as hvd
    hvd.init()
    opt = keras.optimizers.Adadelta(1.0 * hvd.size())
    opt = hvd.DistributedOptimizer(opt)
    callbacks = [hvd.keras.callbacks.BroadcastGlobalVariablesCallback(0)]

(reference: tf_yarn/examples/native_keras_with_gloo_example.py:41,65-83,
collective_all_reduce_example.py:58-69).  Instead of Horovod's C++ core + gloo
over TCP (reference: tf_yarn/tensorflow/tasks/gloo_allred_task.py:42-54) the
data plane is :class:`tf_yarn_b200.parallel.comm.Communicator`: NVLS/P2P kernels
over symmetric HBM.  With a mini-Keras optimizer the gradient all-reduce is
fused into the optimizer kernel (K4); with a ``torch.optim`` optimizer the
wrapper all-reduces the gradients through the fusion buffer before ``step()``.

Identity (rank/size/...) comes from ``HOROVOD_*`` variables exported by the
all-reduce task, else from ``RANK``/``WORLD_SIZE`` (torchrun), else 0/1.
On a CPU-only process the collectives run on a gloo process group.
"""
from __future__ import annotations

import logging
import os
from typing import Iterable, List, Optional

import torch

logger = logging.getLogger(__name__)

_state = {"initialized": False, "rank": 0, "size": 1, "local_rank": 0, "local_size": 1, "cross_rank": 0,
          "cross_size": 1, "cpu_group": False}


def init() -> None:
    env = os.environ
    if "HOROVOD_RANK" in env:
        _state.update(rank=int(env["HOROVOD_RANK"]), size=int(env["HOROVOD_SIZE"]),
                      local_rank=int(env.get("HOROVOD_LOCAL_RANK", 0)),
                      local_size=int(env.get("HOROVOD_LOCAL_SIZE", 1)),
                      cross_rank=int(env.get("HOROVOD_CROSS_RANK", 0)),
                      cross_size=int(env.get("HOROVOD_CROSS_SIZE", 1)))
    elif "RANK" in env and "WORLD_SIZE" in env:
        _state.update(rank=int(env["RANK"]), size=int(env["WORLD_SIZE"]),
                      local_rank=int(env.get("LOCAL_RANK", env["RANK"])),
                      local_size=int(env.get("LOCAL_WORLD_SIZE", env["WORLD_SIZE"])))
    _state["initialized"] = True
    if torch.cuda.is_available():
        ids = [int(v) for v in env.get("TFY_GPU_IDS", "").split(",") if v.strip() != ""]
        dev = ids[0] if ids else _state["local_rank"] % torch.cuda.device_count()
        torch.cuda.set_device(dev)
    logger.info("hvd.init: rank %d / %d (local %d / %d)", _state["rank"], _state["size"], _state["local_rank"],
                _state["local_size"])


def _check() -> None:
    if not _state["initialized"]:
        raise ValueError("Horovod facade has not been initialized; call hvd.init() first")


def is_initialized() -> bool:
    return _state["initialized"]


def rank() -> int:
    _check()
    return _state["rank"]


def size() -> int:
    _check()
    return _state["size"]


def local_rank() -> int:
    _check()
    return _state["local_rank"]


def local_size() -> int:
    _check()
    return _state["local_size"]


def cross_rank() -> int:
    _check()
    return _state["cross_rank"]


def cross_size() -> int:
    _check()
    return _state["cross_size"]


def shutdown() -> None:
    import torch.distributed as dist
    if torch.cuda.is_available():
        from tf_yarn_b200.parallel import runtime
        runtime.shutdown()
    if _state["cpu_group"] and dist.is_initialized():
        dist.destroy_process_group()
        _state["cpu_group"] = False
    _state["initialized"] = False


# ---------------------------------------------------------------------------
# data plane selection
# ---------------------------------------------------------------------------
def ensure_cpu_group() -> None:
    """gloo group for CPU-only jobs (rendezvous address exported by the all-reduce task)."""
    import torch.distributed as dist
    _check()
    if _state["size"] == 1 or dist.is_initialized():
        return
    addr = os.environ.get("HOROVOD_GLOO_RENDEZVOUS_ADDR") or os.environ.get("MASTER_ADDR", "127.0.0.1")
    port = os.environ.get("HOROVOD_GLOO_RENDEZVOUS_PORT") or os.environ.get("MASTER_PORT", "29500")
    dist.init_process_group("gloo", init_method=f"tcp://{addr}:{port}", rank=_state["rank"],
                            world_size=_state["size"])
    _state["cpu_group"] = True


def _communicator():
    """The NVLink communicator of this rank (H100 only)."""
    from tf_yarn_b200.parallel import runtime
    from tf_yarn_b200.parallel.symm import default_rendezvous
    os.environ.setdefault("TFY_RANK", str(_state["rank"]))
    os.environ.setdefault("TFY_WORLD_SIZE", str(_state["size"]))
    return runtime.get_communicator()


def _on_gpu(t: torch.Tensor) -> bool:
    return t.is_cuda


def allreduce_(tensor: torch.Tensor, average: bool = True, name: Optional[str] = None) -> torch.Tensor:
    """In-place all-reduce (sum or average)."""
    _check()
    if _state["size"] == 1:
        return tensor
    if _on_gpu(tensor):
        _communicator().all_reduce([tensor], average=average)
    else:
        import torch.distributed as dist
        ensure_cpu_group()
        dist.all_reduce(tensor)
        if average:
            tensor /= _state["size"]
    return tensor


def allreduce(tensor: torch.Tensor, average: bool = True, name: Optional[str] = None) -> torch.Tensor:
    return allreduce_(tensor.clone(), average, name)


def grouped_allreduce_(tensors: List[torch.Tensor], average: bool = True) -> List[torch.Tensor]:
    """Fused all-reduce of many tensors: one kernel over the fusion buffer."""
    _check()
    if _state["size"] == 1 or not tensors:
        return tensors
    if _on_gpu(tensors[0]):
        _communicator().all_reduce(tensors, average=average)
    else:
        import torch.distributed as dist
        ensure_cpu_group()
        flat = torch.cat([t.reshape(-1) for t in tensors])
        dist.all_reduce(flat)
        if average:
            flat /= _state["size"]
        o = 0
        for t in tensors:
            t.copy_(flat[o:o + t.numel()].view_as(t))
            o += t.numel()
    return tensors


def broadcast_(tensor: torch.Tensor, root_rank: int = 0, name: Optional[str] = None) -> torch.Tensor:
    _check()
    if _state["size"] == 1:
        return tensor
    if _on_gpu(tensor):
        _communicator().broadcast([tensor], root=root_rank)
    else:
        import torch.distributed as dist
        ensure_cpu_group()
        dist.broadcast(tensor, src=root_rank)
    return tensor


def broadcast(tensor: torch.Tensor, root_rank: int = 0, name: Optional[str] = None) -> torch.Tensor:
    return broadcast_(tensor.clone(), root_rank, name)


def allgather(tensor: torch.Tensor, name: Optional[str] = None) -> torch.Tensor:
    """Concatenate equally shaped tensors of all ranks along dim 0."""
    _check()
    if _state["size"] == 1:
        return tensor.clone()
    if _on_gpu(tensor):
        flat = _communicator().all_gather(tensor.contiguous().view(-1))
        return flat.view(_state["size"] * tensor.shape[0], *tensor.shape[1:])
    import torch.distributed as dist
    ensure_cpu_group()
    out = [torch.empty_like(tensor) for _ in range(_state["size"])]
    dist.all_gather(out, tensor)
    return torch.cat(out, dim=0)


def broadcast_parameters(params, root_rank: int = 0) -> None:
    """Broadcast a ``state_dict`` / iterable of (name, tensor) / iterable of tensors from ``root_rank``."""
    if isinstance(params, dict):
        tensors = [t for t in params.values() if torch.is_tensor(t)]
    else:
        tensors = [(p[1] if isinstance(p, tuple) else p) for p in params]
    tensors = [t.data if isinstance(t, torch.nn.Parameter) else t for t in tensors]
    if not tensors or size() == 1:
        return
    if _on_gpu(tensors[0]):
        _communicator().broadcast(tensors, root=root_rank)
    else:
        for t in tensors:
            broadcast_(t, root_rank)


def broadcast_variables(variables, root_rank: int = 0) -> None:
    """``horovod.tensorflow.broadcast_variables``: same as :func:`broadcast_parameters` for a list of tensors /
    parameters / ``(name, tensor)`` pairs or a ``state_dict``."""
    broadcast_parameters(variables, root_rank)


def broadcast_optimizer_state(optimizer: torch.optim.Optimizer, root_rank: int = 0) -> None:
    tensors = []
    for st in optimizer.state.values():
        tensors.extend(v for v in st.values() if torch.is_tensor(v))
    broadcast_parameters(tensors, root_rank)


def barrier() -> None:
    if size() == 1:
        return
    if torch.cuda.is_available():
        _communicator().barrier()
        torch.cuda.current_stream().synchronize()
    else:
        import torch.distributed as dist
        ensure_cpu_group()
        dist.barrier()


# ---------------------------------------------------------------------------
# DistributedOptimizer
# ---------------------------------------------------------------------------
class _KerasDistributedOptimizer:
    """Marker wrapper: ``Model.compile`` unwraps it and turns on the fused distributed step."""

    def __init__(self, optimizer):
        self._tfy_inner_optimizer = optimizer

    def __getattr__(self, name):
        return getattr(self._tfy_inner_optimizer, name)


def DistributedOptimizer(optimizer, named_parameters=None, **_ignored):
    """Wrap an optimizer so that gradients are averaged over all ranks before the update.

    * mini-Keras optimizer descriptor -> marker for ``compile`` (fused K4 kernel on H100);
    * a factory (callable returning a descriptor, as Estimators take) -> wrapped factory;
    * ``torch.optim.Optimizer`` -> same object whose ``step()`` first all-reduces the gradients.
    """
    from tf_yarn_b200.keras import optimizers as kopt
    if isinstance(optimizer, kopt.Optimizer):
        return _KerasDistributedOptimizer(optimizer)
    if isinstance(optimizer, torch.optim.Optimizer):
        return _wrap_torch_optimizer(optimizer)
    if callable(optimizer):
        return lambda *a, **k: DistributedOptimizer(optimizer(*a, **k))
    raise TypeError(f"cannot distribute optimizer of type {type(optimizer)}")


def _wrap_torch_optimizer(optimizer: torch.optim.Optimizer) -> torch.optim.Optimizer:
    base_step = optimizer.step

    def step(closure=None):
        grads = [p.grad for g in optimizer.param_groups for p in g["params"] if p.grad is not None]
        grouped_allreduce_(grads, average=True)
        return base_step(closure) if closure is not None else base_step()

    optimizer.step = step  # type: ignore[method-assign]
    optimizer._tfy_distributed = True  # type: ignore[attr-defined]
    return optimizer


# ---------------------------------------------------------------------------
# callbacks / hooks namespaces:  hvd.keras.callbacks.*, hvd.callbacks.*
# ---------------------------------------------------------------------------
from tf_yarn_b200.keras.callbacks import Callback as _Callback  # noqa: E402


class BroadcastGlobalVariablesCallback(_Callback):
    """At the start of training every rank adopts rank ``root_rank``'s variables."""

    def __init__(self, root_rank: int = 0):
        super().__init__()
        self.root_rank = root_rank
        self._done = False

    def on_train_begin(self, logs=None):
        if not self._done:
            self.model.broadcast_variables(self.root_rank)
            self._done = True


class MetricAverageCallback(_Callback):
    """Average the epoch-end metrics over ranks."""

    def on_epoch_end(self, epoch, logs=None):
        if logs and size() > 1:
            keys = sorted(logs)
            t = torch.tensor([float(logs[k]) for k in keys], dtype=torch.float32)
            if torch.cuda.is_available():
                t = t.cuda()
            allreduce_(t, average=True)
            for k, v in zip(keys, t.cpu().tolist()):
                logs[k] = v


class BroadcastGlobalVariablesHook:
    """Estimator hook: broadcast the model variables from ``root_rank`` before the first step."""

    def __init__(self, root_rank: int = 0, device: str = ""):
        self.root_rank = root_rank

    def begin(self):
        pass

    def after_create_session(self, estimator=None, coord=None):
        if estimator is not None:
            estimator.broadcast_variables(self.root_rank)

    def before_run(self, run_context):
        return None

    def after_run(self, run_context, run_values):
        pass

    def end(self, session=None):
        pass


class callbacks:  # hvd.callbacks.*
    BroadcastGlobalVariablesCallback = BroadcastGlobalVariablesCallback
    MetricAverageCallback = MetricAverageCallback


class keras:  # hvd.keras.callbacks.*  /  hvd.keras.DistributedOptimizer
    callbacks = callbacks
    DistributedOptimizer = staticmethod(DistributedOptimizer)
