"""``Sequential`` / ``Model``: the Keras-shaped front end of the train engines.

Accepts the call patterns of the reference's Keras path --
``model.compile(loss=..., optimizer=hvd.DistributedOptimizer(opt), metrics=[...])``
then ``model.fit(**train_params)`` with ``x`` / ``y`` / ``steps_per_epoch`` /
``epochs`` / ``callbacks`` / ``verbose`` (reference:
tf_yarn/tensorflow/tasks/gloo_allred_task.py:76-89, README.md:104-113) and
``load_model(ckpt).evaluate(dataset)`` on the evaluator (reference:
tf_yarn/tensorflow/tasks/evaluator_task.py:54-73).
"""
from __future__ import annotations

import logging
import os
import time
from typing import Any, Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import cloudpickle
import numpy as np
import torch
import torch.nn as nn

from tf_yarn_b200.keras import callbacks as cb_mod
from tf_yarn_b200.keras import layers as L
from tf_yarn_b200.keras import losses as loss_mod
from tf_yarn_b200.keras import metrics as metric_mod
from tf_yarn_b200.keras import optimizers as opt_mod
from tf_yarn_b200.keras.engine import EagerTrainEngine, GraphTrainEngine

logger = logging.getLogger(__name__)


class _Net(nn.Module):
    """The torch module executing a list of built layers."""

    def __init__(self, layers: List[L.Layer]):
        super().__init__()
        self.klayers = layers
        self.mods = nn.ModuleList([ly.module if ly.module is not None else nn.Identity() for ly in layers])
        self.image_input = len(layers) > 0 and layers[0].input_shape_ is not None and \
            len(layers[0].input_shape_) == 3

    def forward(self, x):
        if self.image_input and torch.is_tensor(x) and x.dim() == 4:
            x = x.permute(0, 3, 1, 2)      # NHWC bytes, NCHW logical == channels_last: zero copy
        training = self.training
        for ly in self.klayers:
            x = ly.call(x, training)
        if torch.is_tensor(x) and x.dim() == 4:
            x = x.permute(0, 2, 3, 1)
        return x


def default_device() -> torch.device:
    if torch.cuda.is_available():
        ids = [int(v) for v in os.environ.get("TFY_GPU_IDS", "").split(",") if v.strip() != ""]
        if ids:
            return torch.device(f"cuda:{ids[0]}")
        return torch.device(f"cuda:{torch.cuda.current_device()}")
    return torch.device("cpu")


def _as_tensor(a) -> torch.Tensor:
    if torch.is_tensor(a):
        return a
    return torch.as_tensor(np.asarray(a))


class _NoWatchdog:
    """Stand-in used when a loop runs outside ``fit`` (no watchdog armed)."""

    @staticmethod
    def beat() -> None:
        pass


_NO_WATCHDOG = _NoWatchdog()


class _ArrayBatches:
    """Batches out of in-memory arrays; pinned host memory when feeding a GPU.  With sample weights ``w`` the
    batches are ``(x, y, w)`` triples (``w`` fp32 ``[B]``), gathered with the same permutation as x and y.  ``y_dtype``:
    the labels are cast to it once, here (the dtype the train step reads)."""

    def __init__(self, x, y, batch_size: int, shuffle: bool, pin: bool, drop_remainder: bool, w=None,
                 y_dtype: Optional[torch.dtype] = None):
        self.x, self.y = _as_tensor(x), (_as_tensor(y) if y is not None else None)
        self.w = _as_tensor(w).reshape(-1).float().contiguous() if w is not None else None
        if self.x.dtype == torch.float64:
            self.x = self.x.float()
        if self.y is not None and y_dtype is not None and self.y.dtype != y_dtype:
            self.y = self.y.to(y_dtype)
        self.n = self.x.shape[0]
        if self.w is not None and self.w.shape[0] != self.n:
            raise ValueError(f"sample_weight has {self.w.shape[0]} entries for {self.n} samples")
        self.bs = batch_size
        self.shuffle = shuffle
        self.drop = drop_remainder
        self.pin = pin and torch.cuda.is_available()
        if self.pin:
            self.x = self.x.pin_memory() if not self.x.is_pinned() else self.x
            if self.y is not None:
                self.y = self.y.pin_memory() if not self.y.is_pinned() else self.y
            if self.w is not None:
                self.w = self.w.pin_memory() if not self.w.is_pinned() else self.w
            self._stage = None
            self._slot = 0

    def __len__(self) -> int:
        return self.n // self.bs if self.drop else -(-self.n // self.bs)

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, ...]]:
        if self.w is not None:
            yield from self._iter_weighted()
            return
        if not self.shuffle:
            for i in range(len(self)):
                s = slice(i * self.bs, min(self.n, (i + 1) * self.bs))
                yield self.x[s], (self.y[s] if self.y is not None else None)
            return
        perm = torch.randperm(self.n)
        if self.pin and self._stage is None:
            # gathered batches land in a small ring of pinned staging buffers
            self._stage = [(torch.empty((self.bs,) + tuple(self.x.shape[1:]), dtype=self.x.dtype).pin_memory(),
                            torch.empty((self.bs,) + tuple(self.y.shape[1:]), dtype=self.y.dtype).pin_memory()
                            if self.y is not None else None) for _ in range(4)]
        for i in range(len(self)):
            idx = perm[i * self.bs:(i + 1) * self.bs]
            if self.pin and idx.numel() == self.bs:
                sx, sy = self._stage[self._slot]
                self._slot = (self._slot + 1) % len(self._stage)
                torch.index_select(self.x, 0, idx, out=sx)
                if self.y is not None:
                    torch.index_select(self.y, 0, idx, out=sy)
                yield sx, sy
            else:
                yield self.x[idx], (self.y[idx] if self.y is not None else None)

    def _iter_weighted(self) -> Iterator[Tuple[torch.Tensor, ...]]:
        y = self.y
        if not self.shuffle:
            for i in range(len(self)):
                s = slice(i * self.bs, min(self.n, (i + 1) * self.bs))
                yield self.x[s], (y[s] if y is not None else None), self.w[s]
            return
        perm = torch.randperm(self.n)
        if self.pin and self._stage is None:
            self._stage = [(torch.empty((self.bs,) + tuple(self.x.shape[1:]), dtype=self.x.dtype).pin_memory(),
                            torch.empty((self.bs,) + tuple(y.shape[1:]), dtype=y.dtype).pin_memory()
                            if y is not None else None,
                            torch.empty((self.bs,), dtype=torch.float32).pin_memory()) for _ in range(4)]
        for i in range(len(self)):
            idx = perm[i * self.bs:(i + 1) * self.bs]
            if self.pin and idx.numel() == self.bs:
                sx, sy, sw = self._stage[self._slot]
                self._slot = (self._slot + 1) % len(self._stage)
                torch.index_select(self.x, 0, idx, out=sx)
                if y is not None:
                    torch.index_select(y, 0, idx, out=sy)
                torch.index_select(self.w, 0, idx, out=sw)
                yield sx, sy, sw
            else:
                yield self.x[idx], (y[idx] if y is not None else None), self.w[idx]


def _split_batch(item):
    """``(x, y)`` or ``(x, y, sample_weight)`` -> ``(x, y, sample_weight or None)``."""
    if isinstance(item, (tuple, list)) and len(item) >= 2:
        return item[0], item[1], (item[2] if len(item) >= 3 else None)
    return item, None, None


def _as_weights(w) -> Optional[torch.Tensor]:
    return None if w is None else _as_tensor(w).reshape(-1).float()


def _is_array(x) -> bool:
    return hasattr(x, "shape") and not hasattr(x, "__next__")


class Model:
    """Base model: a stack of layers (``Sequential``) or a wrapped ``torch.nn.Module``."""

    def __init__(self, layers: Optional[Sequence[L.Layer]] = None, name: Optional[str] = None):
        self.name = name or type(self).__name__.lower()
        self.layers: List[L.Layer] = []
        self.net: Optional[_Net] = None
        self.built = False
        self.stop_training = False
        self.optimizer: Optional[opt_mod.Optimizer] = None
        self.loss = None
        self._loss_fn: Optional[Callable] = None
        self._metrics_spec: List[Any] = []
        self._weighted_metrics_spec: List[str] = []
        self._fit_class_weight: Optional[dict] = None
        self._class_weight_pending = False      # fit() got a new class_weight (or none) for the engine
        self._engine = None
        self._device: Optional[torch.device] = None
        self.compute_dtype = torch.bfloat16
        self.use_cuda_graph = True
        self.use_fast_path = True
        self.history = None
        self._watchdog = None             # utils.watchdog.StepWatchdog while fit() runs
        self._pending_broadcast_root: Optional[int] = None
        self._pending_engine_state: Optional[dict] = None    # optimizer state of a loaded checkpoint (load_model)
        for layer in layers or []:
            self.add(layer)

    # ------------------------------------------------------------------ building
    @classmethod
    def from_torch(cls, module: nn.Module, input_shape: Optional[Sequence[int]] = None, name=None) -> "Model":
        m = cls(name=name)
        m.add(L.TorchModule(module, input_shape=input_shape))
        return m

    def add(self, layer: L.Layer) -> None:
        if self.built:
            raise RuntimeError("cannot add layers after the model was built")
        if layer.name is None:
            base = type(layer).__name__.lower()
            n = sum(1 for ly in self.layers if type(ly) is type(layer))
            layer.name = f"{base}_{n}" if n else base
        self.layers.append(layer)

    def build(self, input_shape: Optional[Sequence[int]] = None) -> None:
        if self.built:
            return
        if not self.layers:
            raise ValueError("model has no layers")
        shape = input_shape if input_shape is not None else self.layers[0]._declared_input_shape
        if shape is None and isinstance(self.layers[0], L.TorchModule):
            shape = ()               # wrapped torch modules (possibly with dict inputs) carry their own shapes
        if shape is None:
            raise ValueError("the first layer needs input_shape=... (or call build(input_shape) / fit on data)")
        shape = tuple(shape)
        for layer in self.layers:
            shape = layer.build(shape)
        self.net = _Net(self.layers)
        self.built = True

    @property
    def output_shape(self):
        return (None,) + tuple(self.layers[-1].output_shape_) if self.built else None

    def count_params(self) -> int:
        self.build()
        return sum(p.numel() for p in self.net.parameters())

    def summary(self, print_fn: Callable[[str], None] = print) -> None:
        self.build()
        lines = [f'Model: "{self.name}"', "_" * 65, f"{'Layer (type)':<30}{'Output Shape':<22}{'Param #':>12}",
                 "=" * 65]
        for ly in self.layers:
            lines.append(f"{ly.name + ' (' + type(ly).__name__ + ')':<30}"
                         f"{str((None,) + tuple(ly.output_shape_)):<22}{ly.count_params():>12,}")
        lines += ["=" * 65, f"Total params: {self.count_params():,}", "_" * 65]
        print_fn("\n".join(lines))

    # ------------------------------------------------------------------ compile
    def compile(self, optimizer="sgd", loss=None, metrics: Optional[Sequence[Any]] = None,
                compute_dtype: Optional[torch.dtype] = None, use_cuda_graph: bool = True,
                use_fast_path: bool = True, weighted_metrics: Optional[Sequence[str]] = None, **_ignored) -> None:
        """``metrics`` are unweighted; ``weighted_metrics`` (built-in metric names) are ``sum(w*m) / sum(w)`` over the
        sample weights of ``fit`` / ``evaluate`` (``class_weight`` included).  Both accept the stateful metrics
        ``"AUC"``, ``"Precision"`` and ``"Recall"``; ``metrics`` also takes such objects (``keras.metrics.AUC(...)``),
        whose names must be unique."""
        if _ignored:
            logger.warning("Model.compile: unsupported arguments ignored: %s", sorted(_ignored))
        for m in weighted_metrics or []:
            if not isinstance(m, str):
                raise ValueError(f"weighted_metrics accepts built-in metric names only, got {m!r}")
            metric_mod.resolve(m, loss_mod.name_of(loss), 2)          # unknown names fail here
        for spec in (metrics or [], weighted_metrics or []):
            resolved = [metric_mod.resolve(m, loss_mod.name_of(loss), 2) for m in spec]
            names = [name for name, _ in resolved]
            for name, fn in resolved:
                if isinstance(fn, metric_mod.Metric) and names.count(name) > 1:
                    raise ValueError(f"metric name {name!r} is used twice: give the metrics distinct names")
        self.optimizer = opt_mod.get(optimizer)
        self.loss = loss
        self._loss_fn = loss_mod.get(loss) if loss is not None else None
        self._metrics_spec = list(metrics or [])
        self._weighted_metrics_spec = list(weighted_metrics or [])
        if compute_dtype is not None:
            self.compute_dtype = compute_dtype
        self.use_cuda_graph = use_cuda_graph
        self.use_fast_path = use_fast_path
        self._engine = None

    def _metric_fns(self) -> List[Tuple[str, Callable]]:
        out_dim = self.layers[-1].output_shape_[-1] if self.layers[-1].output_shape_ else 1
        return [metric_mod.resolve(m, loss_mod.name_of(self.loss), out_dim) for m in self._metrics_spec]

    def _weighted_metric_fns(self) -> List[Tuple[str, Callable]]:
        """Resolved ``weighted_metrics``; one that is also in ``metrics`` is logged as ``weighted_<name>``."""
        out_dim = self.layers[-1].output_shape_[-1] if self.layers[-1].output_shape_ else 1
        plain = {name for name, _ in self._metric_fns()}
        out = []
        for m in self._weighted_metrics_spec:
            name, fn = metric_mod.resolve(m, loss_mod.name_of(self.loss), out_dim)
            out.append((f"weighted_{name}" if name in plain else name, fn))
        return out

    def _class_weight_table(self, class_weight: Optional[dict]) -> Optional[torch.Tensor]:
        """``class_weight`` dict -> fp32 table ``[num_classes]``.  Keys must be class indices; classes the dict
        leaves out weigh 1.0 (with a warning)."""
        if class_weight is None:
            return None
        shape = self.layers[-1].output_shape_
        n = max(int(shape[-1]), 2) if shape else None
        for k in class_weight:
            if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 0 or (n is not None and k >= n):
                raise ValueError(f"class_weight key {k!r} is not a class index in [0, {n if n is not None else 'C'})")
        n = n if n is not None else (max(int(k) for k in class_weight) + 1 if class_weight else 1)
        table = torch.ones(n, dtype=torch.float32)
        for k, v in class_weight.items():
            table[int(k)] = float(v)
        missing = [c for c in range(n) if c not in {int(k) for k in class_weight}]
        if missing:
            logger.warning("class_weight has no entry for classes %s: they weigh 1.0", missing)
        return table
    def _ensure_engine(self, x0, y0) -> None:
        if self._engine is not None:
            return
        if self._loss_fn is None or self.optimizer is None:
            raise RuntimeError("call compile(optimizer=..., loss=...) before fit()")
        if not self.built:
            self.build(tuple(x0.shape[1:]) if torch.is_tensor(x0) else None)
        self._device = self._device or default_device()
        self.net.to(self._device)
        distributed = bool(self.optimizer.distributed)
        if self._device.type == "cuda":
            plan = None
            if self.use_fast_path and self.compute_dtype == torch.bfloat16:
                from tf_yarn_b200.keras import fastpath
                plan = fastpath.build_plan(self)
            if plan is not None:
                self._engine = fastpath.FastSequentialEngine(
                    self, plan, self.net, self._loss_fn, self.optimizer, self._metric_fns(), self._device,
                    distributed, x0, y0, self.compute_dtype, self.use_cuda_graph,
                    weighted_metric_fns=self._weighted_metric_fns())
            else:
                self._engine = GraphTrainEngine(self.net, self._loss_fn, self.optimizer, self._metric_fns(),
                                                self._device, distributed, x0, y0, self.compute_dtype,
                                                self.use_cuda_graph, weighted_metric_fns=self._weighted_metric_fns())
        else:
            if distributed:
                from tf_yarn_b200 import hvd
                hvd.ensure_cpu_group()
            self._engine = EagerTrainEngine(self.net, self._loss_fn, self.optimizer, self._metric_fns(),
                                            self._device, distributed, weighted_metric_fns=self._weighted_metric_fns())
        self._restore_engine_state()
        if self._pending_broadcast_root is not None:
            self._engine.broadcast_variables(self._pending_broadcast_root)
            self._pending_broadcast_root = None

    def _restore_engine_state(self) -> None:
        """``load_model`` keeps the saved optimizer state (moments, accumulators, step count) until the train engine
        exists; training then resumes where the checkpoint left off, as with ``tf.keras.models.load_model``.  A state
        written by a different engine / world size is skipped with a warning (the weights are already restored)."""
        state, self._pending_engine_state = self._pending_engine_state, None
        if not state:
            return
        want = "eager" if isinstance(self._engine, EagerTrainEngine) else "fused"
        if state.get("kind") != want:
            logger.warning("checkpoint optimizer state is of kind %r, the engine needs %r: optimizer starts fresh",
                           state.get("kind"), want)
            return
        try:
            if self._device.type == "cuda":
                torch.cuda.synchronize(self._device)
            self._engine.load_state_dict(state)
            if self._device.type == "cuda":
                torch.cuda.synchronize(self._device)
        except Exception as exc:  # noqa: BLE001  (shape / world-size mismatch: keep training possible)
            logger.warning("could not restore the optimizer state of the checkpoint (%s): optimizer starts fresh", exc)

    def to(self, device) -> "Model":
        self._device = torch.device(device)
        return self

    # ------------------------------------------------------------------ fit
    def fit(self, x=None, y=None, batch_size: Optional[int] = None, epochs: int = 1, verbose: int = 1,
            callbacks: Optional[List[cb_mod.Callback]] = None, validation_data=None, shuffle: bool = True,
            steps_per_epoch: Optional[int] = None, initial_epoch: int = 0, validation_steps: Optional[int] = None,
            validation_split: float = 0.0, sample_weight=None, class_weight: Optional[dict] = None, **_ignored):
        """Train.  ``x`` may be an array/tensor (with ``y`` and ``batch_size``) or an iterable of
        ``(features, labels)`` or ``(features, labels, sample_weight)`` batches such as
        :class:`tf_yarn_b200.data.Dataset`.  ``validation_split`` holds out the LAST fraction of array inputs
        (before shuffling), as Keras does.  ``sample_weight`` (one weight per sample of an array ``x``) and
        ``class_weight`` (``{class index: weight}``) weigh the loss as ``sum(w*l) / B`` and the weighted metrics."""
        if _ignored:
            logger.warning("Model.fit: unsupported arguments ignored: %s", sorted(_ignored))
        if callable(x) and not torch.is_tensor(x):
            x = x()
        if callable(y):
            y = y()
        if sample_weight is not None and not _is_array(x):
            raise ValueError("sample_weight needs array inputs x; a dataset yields (x, y, sample_weight) batches instead")
        if class_weight is not None and not isinstance(class_weight, dict):
            raise ValueError("class_weight must be a dict {class index: weight}")
        if validation_split and validation_data is None:
            if not (hasattr(x, "shape") and not hasattr(x, "__next__")) or y is None:
                raise ValueError("validation_split needs array inputs x and y")
            if not 0.0 < validation_split < 1.0:
                raise ValueError("validation_split must be in (0, 1)")
            cut = int(len(x) * (1.0 - validation_split))
            validation_data = (x[cut:], y[cut:])
            x, y = x[:cut], y[:cut]
            if sample_weight is not None:
                validation_data += (sample_weight[cut:],)
                sample_weight = sample_weight[:cut]
        self._fit_class_weight = class_weight
        self._class_weight_pending = True
        if hasattr(x, "shape") and not hasattr(x, "__next__"):
            on_gpu = (self._device or default_device()).type == "cuda"
            y_dtype = None
            if on_gpu:
                # the fused classifier head reads int64 labels or fp32 targets: narrower integer labels (uint8 from
                # the Keras MNIST loader, int32) and float64 one-hot targets are cast once, not per step
                from tf_yarn_b200.keras import fastpath
                y_dtype = fastpath.label_dtype(self.loss)
            batches = _ArrayBatches(x, y, batch_size or 32, shuffle, pin=on_gpu, drop_remainder=on_gpu,
                                    w=sample_weight, y_dtype=y_dtype)
            make_iter = lambda: iter(batches)   # noqa: E731
            if steps_per_epoch is None:
                steps_per_epoch = len(batches)
            infinite = False
        else:
            dataset = x
            make_iter = lambda: iter(dataset)   # noqa: E731
            infinite = True                     # one iterator is consumed across epochs (tf.data.repeat())
            if steps_per_epoch is None:
                steps_per_epoch = getattr(dataset, "cardinality", None)
                infinite = False
        history = cb_mod.History()
        cbs = cb_mod.CallbackList([history] + list(callbacks or []), self,
                                  {"epochs": epochs, "steps": steps_per_epoch, "verbose": verbose})
        self.history = history
        self.stop_training = False
        from tf_yarn_b200.utils import watchdog
        distributed = bool(getattr(self.optimizer, "distributed", False))
        self._watchdog = watchdog.StepWatchdog(watchdog.default_timeout(distributed), "Model.fit").start()
        try:
            return self._fit_epochs(cbs, history, make_iter, infinite, initial_epoch, epochs, steps_per_epoch,
                                    validation_data, validation_steps, batch_size, verbose)
        finally:
            self._watchdog.close()
            self._watchdog = None

    def _fit_epochs(self, cbs, history, make_iter, infinite, initial_epoch, epochs, steps_per_epoch, validation_data,
                    validation_steps, batch_size, verbose):
        cbs.call("on_train_begin", None)
        it = make_iter() if infinite else None
        for epoch in range(initial_epoch, epochs):
            if self.stop_training:
                break
            cbs.call("on_epoch_begin", epoch, None)
            t0 = time.time()
            epoch_it = it if infinite else make_iter()
            logs = self._run_epoch(epoch_it, steps_per_epoch, cbs)
            if validation_data is not None:
                pair = isinstance(validation_data, (tuple, list))
                val = self.evaluate(validation_data[0] if pair else validation_data,
                                    validation_data[1] if pair else None,
                                    batch_size=batch_size or 32, steps=validation_steps, verbose=0,
                                    return_dict=True,
                                    sample_weight=validation_data[2] if pair and len(validation_data) > 2 else None)
                logs.update({f"val_{k}": v for k, v in val.items()})
            if verbose:
                msg = " - ".join(f"{k}: {_fmt(v)}" for k, v in logs.items())
                logger.info("Epoch %d/%d - %.1fs - %s", epoch + 1, epochs, time.time() - t0, msg)
            cbs.call("on_epoch_end", epoch, logs)
        cbs.call("on_train_end", None)
        return history

    def _run_epoch(self, it, steps: Optional[int], cbs: cb_mod.CallbackList) -> Dict[str, float]:
        first = None
        if self._engine is None:
            first = next(it, None)
            if first is None:
                return {}
            x0, y0, _ = _split_batch(first)
            self._ensure_engine(_as_struct(x0), _as_struct(y0))
        eng = self._engine
        if self._class_weight_pending:
            eng.set_class_weight(self._class_weight_table(self._fit_class_weight))
            self._class_weight_pending = False
        if eng.pipelined:
            return self._run_epoch_pipelined(it, steps, cbs, first)
        loss_sum, n = 0.0, 0
        metric_sums: Dict[str, float] = {}
        step = 0
        wd = self._watchdog or _NO_WATCHDOG
        while steps is None or step < steps:
            item = first if first is not None else next(it, None)
            first = None
            if item is None:
                break
            xb, yb, wb = _split_batch(item)
            if cbs.has_batch_hooks:
                cbs.call("on_train_batch_begin", step, None)
            if wb is None:
                logs = eng.train_step(_as_struct(xb), _as_struct(yb))
            else:
                logs = eng.train_step(_as_struct(xb), _as_struct(yb), _as_weights(wb))
            wd.beat()
            loss_sum += float(logs["loss"])
            for k, v in logs.items():
                if k != "loss":
                    metric_sums[k] = metric_sums.get(k, 0.0) + float(v)
            n += 1
            if cbs.has_batch_hooks:
                cbs.call("on_train_batch_end", step, {"loss": float(logs["loss"])})
            step += 1
        out = {"loss": loss_sum / max(n, 1)}
        out.update({k: v / max(n, 1) for k, v in metric_sums.items()})
        if getattr(eng, "weighted_metric_fns", None) or getattr(eng, "stateful_metrics", None):
            out.update(eng.pop_metrics())
        return out

    def _run_epoch_pipelined(self, it, steps, cbs, first) -> Dict[str, float]:
        """GPU loop: stage batch i+1 (H2D, copy stream) while step i runs.  Every captured step copies its
        loss to a pinned scalar (a D2H node of the graph); the host reads it one step late, while the
        next step is already queued, so it never stalls the GPU."""
        eng: GraphTrainEngine = self._engine
        loss_sum, n_read = 0.0, 0
        sync_every_step = cbs.needs_batch_logs
        hooks = cbs.has_batch_hooks
        wd = self._watchdog or _NO_WATCHDOG

        def fetch():
            nonlocal first
            item = first if first is not None else next(it, None)
            first = None
            if item is None:
                return None
            xb, yb, wb = _split_batch(item)
            if wb is None:
                return _as_struct(xb), _as_struct(yb)
            return _as_struct(xb), _as_struct(yb), _as_weights(wb)

        nxt = fetch()
        if nxt is None:
            return {}
        ticket = eng.stage_inputs(*nxt)
        step = 0
        pending = None                          # (slot, event) of the step whose loss is not read yet
        with torch.cuda.stream(eng.stream):     # one context for the epoch: replays go to the engine's stream
            while True:
                if hooks:
                    cbs.call("on_train_batch_begin", step, None)
                done = eng.launch_step(ticket)
                slot = ticket[0]
                step += 1
                more = steps is None or step < steps
                nxt = fetch() if more else None
                if pending is not None:         # loss of the previous step: its graph finished long ago
                    pending[1].synchronize()
                    wd.beat()                   # a step COMPLETED on the device (not merely queued)
                    loss_sum += float(eng.loss_host(pending[0]))
                    n_read += 1
                pending = (slot, done)
                if nxt is not None:
                    ticket = eng.stage_inputs(*nxt)
                if hooks:
                    logs = None
                    if sync_every_step:
                        done.synchronize()
                        logs = {"loss": float(eng.loss_host(slot))}
                    cbs.call("on_train_batch_end", step - 1, logs)
                if nxt is None:
                    break
        if pending is not None:
            pending[1].synchronize()
            loss_sum += float(eng.loss_host(pending[0]))
            n_read += 1
        out = {"loss": loss_sum / max(n_read, 1)}
        out.update(eng.pop_metrics())
        return out

    # ------------------------------------------------------------------ inference
    def _infer_batches(self, x, y, batch_size, steps, sample_weight=None):
        if callable(x) and not torch.is_tensor(x):
            x = x()
        if (y is None and isinstance(x, (tuple, list)) and len(x) in (2, 3) and all(hasattr(t, "shape") for t in x)
                and all(len(t) == len(x[0]) for t in x)):
            # ``validation_data_fn=lambda: (x_val, y_val[, w_val])``: arrays, not batches
            x, y, sample_weight = x[0], x[1], (x[2] if len(x) == 3 else sample_weight)
        if hasattr(x, "shape") and not hasattr(x, "__next__"):
            return iter(_ArrayBatches(x, y, batch_size or 32, False, pin=False, drop_remainder=False,
                                      w=sample_weight)), steps
        if sample_weight is not None:
            raise ValueError("sample_weight needs array inputs x; a dataset yields (x, y, sample_weight) batches instead")
        return iter(x), steps

    def _prep_infer(self, xb):
        dev = self._device or default_device()
        self._device = dev
        if not self.built:
            self.build(tuple(xb.shape[1:]))
        self.net.to(dev)
        xb = _move(xb, dev)
        pdt = next(self.net.parameters()).dtype if any(True for _ in self.net.parameters()) else torch.float32
        if torch.is_tensor(xb) and torch.is_floating_point(xb):
            xb = xb.to(pdt)
        return xb

    def evaluate(self, x=None, y=None, batch_size: Optional[int] = None, steps: Optional[int] = None,
                 verbose: int = 0, return_dict: bool = False, sample_weight=None, **_ignored):
        """Mean loss and metrics over ``x``; returns ``[loss, *metrics, *weighted metrics]`` (or a dict).  With sample
        weights (``sample_weight``, or ``(x, y, w)`` batches) the loss is ``sum(w*l) / N`` over the N samples and the
        weighted metrics ``sum(w*m) / sum(w)``; ``metrics`` stay unweighted."""
        it, steps = self._infer_batches(x, y, batch_size, steps, sample_weight)
        fns = self._metric_fns() if self.built and self.loss is not None else []
        wfns = self._weighted_metric_fns() if self.built and self.loss is not None else []
        loss_sum, count = 0.0, 0
        m_num = [0.0] * len(fns)
        m_den = [0.0] * len(fns)
        w_num = [0.0] * len(wfns)
        w_den = [0.0] * len(wfns)
        self.net.eval() if self.net is not None else None
        n = 0
        wd = getattr(self, "_watchdog", None)
        with torch.no_grad():
            for item in it:
                if steps is not None and n >= steps:
                    break
                xb, yb, wb = _split_batch(item)
                xb = self._prep_infer(_as_struct(xb))
                self.net.eval()
                if not fns and not wfns and self.loss is not None:
                    fns = self._metric_fns()
                    m_num, m_den = [0.0] * len(fns), [0.0] * len(fns)
                    wfns = self._weighted_metric_fns()
                    w_num, w_den = [0.0] * len(wfns), [0.0] * len(wfns)
                yb = _move(_as_struct(yb), self._device)
                wb = _move(_as_weights(wb), self._device)
                out = self.net(xb)
                if wd is not None:
                    wd.beat()
                bs = _batch_size_of(out)
                if self._loss_fn is not None:
                    if wb is None:
                        loss_sum += float(self._loss_fn(yb, out)) * bs
                    else:
                        loss_sum += float((loss_mod.per_sample(self._loss_fn)(yb, out) * wb).sum())
                count += bs
                for i, (_, fn) in enumerate(fns):
                    if isinstance(fn, metric_mod.Metric):      # streaming state on the device, read once at the end
                        fn.update_state(yb, out)
                        continue
                    a, b = fn(yb, out)
                    m_num[i] += float(a)
                    m_den[i] += float(b)
                for i, (_, fn) in enumerate(wfns):
                    if isinstance(fn, metric_mod.Metric):
                        fn.update_state(yb, out, sample_weight=wb)
                        continue
                    a, b = fn(yb, out, sample_weight=wb)
                    w_num[i] += float(a)
                    w_den[i] += float(b)
                n += 1
        res = {"loss": loss_sum / max(count, 1)}
        for i, (name, fn) in enumerate(fns):
            res[name] = fn.result() if isinstance(fn, metric_mod.Metric) else m_num[i] / max(m_den[i], 1.0)
        for i, (name, fn) in enumerate(wfns):
            if isinstance(fn, metric_mod.Metric):
                res[name] = fn.result()
            else:
                res[name] = w_num[i] / w_den[i] if w_den[i] else 0.0
        if return_dict:
            return res
        vals = list(res.values())
        return vals if len(vals) > 1 else vals[0]

    def predict(self, x, batch_size: Optional[int] = None, steps: Optional[int] = None, **_ignored) -> np.ndarray:
        it, steps = self._infer_batches(x, None, batch_size, steps)
        outs = []
        n = 0
        with torch.no_grad():
            for item in it:
                if steps is not None and n >= steps:
                    break
                xb = _split_batch(item)[0] if isinstance(item, (tuple, list)) else item
                xb = self._prep_infer(_as_struct(xb))
                self.net.eval()
                outs.append(self.net(xb).float().cpu())
                n += 1
        return torch.cat(outs).numpy() if outs else np.zeros((0,))

    def __call__(self, x, training: bool = False):
        xb = self._prep_infer(_as_struct(x))
        self.net.train(training)
        return self.net(xb)

    # ------------------------------------------------------------------ variables
    def broadcast_variables(self, root: int = 0) -> None:
        """All ranks adopt rank ``root``'s weights (applied when the engine exists)."""
        if self._engine is not None:
            self._engine.broadcast_variables(root)
        else:
            self._pending_broadcast_root = root

    def get_learning_rate(self) -> float:
        if self._engine is not None:
            return self._engine.get_learning_rate()
        return self.optimizer.current_learning_rate()

    def set_learning_rate(self, lr: float) -> None:
        self.optimizer.learning_rate = lr
        if self._engine is not None:
            self._engine.set_learning_rate(lr)

    def _param_names(self) -> List[str]:
        return [n for n, p in self.net.named_parameters() if p.requires_grad]

    def get_weights(self) -> List[np.ndarray]:
        return [t.detach().float().cpu().numpy() for t in self._fp32_state().values()]

    def set_weights(self, weights: Sequence[np.ndarray]) -> None:
        self.build()
        if isinstance(self._engine, GraphTrainEngine):     # the fp32 master copies live in the engine's shards
            raise RuntimeError("set_weights after training started on GPU: use load_weights on a fresh model")
        state = self.net.state_dict()
        if len(weights) != len(state):
            raise ValueError(f"set_weights expects {len(state)} arrays, got {len(weights)}")
        for (k, v), w in zip(state.items(), weights):
            w = torch.as_tensor(w)
            if tuple(w.shape) != tuple(v.shape):
                raise ValueError(f"shape mismatch for {k}: {tuple(w.shape)} vs {tuple(v.shape)}")
            v.copy_(w.to(v.dtype))

    def _fp32_state(self) -> Dict[str, torch.Tensor]:
        """Full-precision state dict (fp32 master weights when training on H100 in bf16)."""
        self.build()
        state = {k: v.detach().float().cpu().clone() for k, v in self.net.state_dict().items()}
        if isinstance(self._engine, GraphTrainEngine) and not self._sharded_across_ranks():
            names = self._param_names()
            for name, t in zip(names, self._engine.master_tensors()):
                state[name] = t.detach().float().cpu().contiguous()
        return state

    # ------------------------------------------------------------------ persistence
    def get_config(self) -> Dict[str, Any]:
        return {"name": self.name,
                "layers": [{"class_name": type(ly).__name__, "config": ly.get_config()} for ly in self.layers],
                "input_shape": list(self.layers[0].input_shape_) if self.built else
                (list(self.layers[0]._declared_input_shape) if self.layers[0]._declared_input_shape else None)}

    def _sharded_across_ranks(self) -> bool:
        """True when the fp32 master weights / optimizer state are split over several GPUs.  Collecting them is a
        COLLECTIVE (every rank would have to call it), while checkpoints are written by one rank alone -- the
        all-reduce task strips ``ModelCheckpoint`` from every rank but the chief, as the reference does
        (tf_yarn/tensorflow/tasks/gloo_allred_task.py:79-84) -- so single-rank readers use the replicated compute
        parameters instead (bf16-rounded on H100) and leave the optimizer state out."""
        comm = getattr(self._engine, "comm", None)
        return comm is not None and getattr(comm, "world", 1) > 1

    def save(self, filepath: str, include_optimizer: bool = True) -> None:
        """Atomically write config + fp32 weights (+ optimizer state) to ``filepath``."""
        if self._engine is not None and self._sharded_across_ranks() and not getattr(self, "_warned_sharded", False):
            self._warned_sharded = True
            logger.info("multi-rank training: the checkpoint holds this rank's replicated parameters (compute "
                        "precision) and no optimizer state; gathering the sharded fp32 state would be a collective")
        payload = {
            "format": "tf_yarn_b200.keras/1",
            "config": self.get_config(),
            "weights": self._fp32_state(),
            "compile": {"loss": loss_mod.serialize(self.loss),
                        "optimizer": self.optimizer.get_config() if self.optimizer is not None else None,
                        "metrics": [spec for spec in map(metric_mod.serialize, self._metrics_spec)
                                    if spec is not None],
                        "weighted_metrics": list(self._weighted_metrics_spec)},
            "optimizer_state": (self._engine.state_dict() if (include_optimizer and self._engine is not None
                                                              and not self._sharded_across_ranks()) else None),
        }
        os.makedirs(os.path.dirname(os.path.abspath(filepath)), exist_ok=True)
        tmp = f"{filepath}.tmp{os.getpid()}"
        with open(tmp, "wb") as f:
            cloudpickle.dump(payload, f)
        os.replace(tmp, filepath)

    def save_weights(self, filepath: str) -> None:
        tmp = f"{filepath}.tmp{os.getpid()}"
        torch.save(self._fp32_state(), tmp)
        os.replace(tmp, filepath)

    def load_weights(self, filepath: str) -> None:
        self.build()
        if isinstance(self._engine, GraphTrainEngine):     # same reason as set_weights: the fp32 master would go stale
            raise RuntimeError("load_weights after training started on GPU: load into a fresh model (or use "
                               "keras.models.load_model) before fit()")
        state = torch.load(filepath, map_location="cpu", weights_only=False)
        if isinstance(state, dict) and "weights" in state and "config" in state:
            state = state["weights"]
        self.net.load_state_dict(state)


class Sequential(Model):
    pass


def load_model(filepath: str, compile: bool = True) -> Model:
    """Rebuild a model written by :meth:`Model.save`."""
    import pickle
    with open(filepath, "rb") as f:
        payload = pickle.load(f)
    cfg = payload["config"]
    model = Sequential(name=cfg.get("name"))
    for item in cfg["layers"]:
        cls = L.LAYER_CLASSES[item["class_name"]]
        kwargs = {k: v for k, v in item["config"].items() if v is not None or k == "activation"}
        if "input_shape" in kwargs and kwargs["input_shape"] is not None:
            kwargs["input_shape"] = tuple(kwargs["input_shape"])
        model.add(cls(**kwargs))
    model.build(tuple(cfg["input_shape"]) if cfg.get("input_shape") else None)
    model.net.load_state_dict(payload["weights"])
    comp = payload.get("compile") or {}
    if compile and comp.get("loss") and comp.get("optimizer"):
        model.compile(optimizer=opt_mod.from_config(comp["optimizer"]), loss=loss_mod.deserialize(comp["loss"]),
                      metrics=[m for m in map(metric_mod.deserialize, comp.get("metrics") or []) if m is not None],
                      weighted_metrics=comp.get("weighted_metrics") or [])
        model._pending_engine_state = payload.get("optimizer_state")
    return model


def _fmt(v) -> str:
    """A log value: a float, or the list of values of a metric with several thresholds."""
    return "[" + ", ".join(f"{x:.4f}" for x in v) + "]" if isinstance(v, (list, tuple)) else f"{v:.4f}"


def _batch_size_of(out) -> int:
    """Leading dimension of a model output (a tensor, or a dict / tuple of tensors as BERT's heads return)."""
    if isinstance(out, dict):
        out = next(iter(out.values()))
    while isinstance(out, (tuple, list)):
        out = out[0]
    return int(out.shape[0])


def _as_struct(t):
    if t is None:
        return None
    if isinstance(t, (tuple, list)):
        return type(t)(_as_struct(x) for x in t)
    if isinstance(t, dict):
        return {k: _as_struct(v) for k, v in t.items()}
    t = _as_tensor(t)
    return t.float() if t.dtype == torch.float64 else t


def _move(t, device):
    if t is None:
        return None
    if isinstance(t, (tuple, list)):
        return type(t)(_move(x, device) for x in t)
    if isinstance(t, dict):
        return {k: _move(v, device) for k, v in t.items()}
    return t.to(device, non_blocking=True)
