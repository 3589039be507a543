"""``Estimator``: train / evaluate / predict driven by a ``model_fn``, checkpoints in ``model_dir``.

Torch-backed stand-in for ``tf.estimator.Estimator`` with the attributes and
methods the reference's task programs rely on (reference:
tf_yarn/tensorflow/tasks/gloo_allred_task.py:58-75 -- ``estimator._model_dir`` /
``estimator._config`` are assigned, ``estimator.train(input_fn, hooks, max_steps)``;
tf_yarn/tensorflow/tasks/evaluator_task.py:103-121 -- ``estimator.evaluate(input_fn,
steps, hooks, name, checkpoint_path)`` returning a dict holding the global step).

Three training data planes, chosen from the process's role:

* local / single process  -- plain optimizer step;
* all-reduce (``optimizer`` wrapped by ``hvd.DistributedOptimizer``) -- gradients
  averaged across ranks by ONE all-reduce kernel over the fusion buffer (NVLS / P2P kernels of
  ``ops/csrc/tfy_comm.cu`` on H100, gloo on CPU), then the optimizer step (the fully fused
  reduce-scatter -> optimizer -> all-gather kernel serves the Keras engines and the DDP wrapper);
* parameter server (``TF_CONFIG`` lists ``ps`` tasks) -- parameters live on the ps
  ranks; workers pull before and push after every step, asynchronously
  (:mod:`tf_yarn_b200.estimator.ps`).
"""
from __future__ import annotations

import inspect
import logging
import os
import tempfile
import time
from typing import Any, Callable, Dict, Iterable, List, Optional

import torch
import torch.nn as nn

from tf_yarn_b200.estimator import checkpoint as ckpt
from tf_yarn_b200.estimator import summary as summary_lib
from tf_yarn_b200.estimator.config import RunConfig
from tf_yarn_b200.estimator.hooks import (GLOBAL_STEP, SessionRunArgs, SessionRunContext, SessionRunValues)
from tf_yarn_b200.estimator.spec import EstimatorSpec, GraphKeys, ModeKeys
from tf_yarn_b200.keras import optimizers as kopt
from tf_yarn_b200.keras.metrics import Metric

logger = logging.getLogger(__name__)


def _call_model_fn(model_fn: Callable, features, labels, mode, params, config) -> EstimatorSpec:
    sig = inspect.signature(model_fn).parameters
    kwargs = {}
    if "labels" in sig:
        kwargs["labels"] = labels
    if "mode" in sig:
        kwargs["mode"] = mode
    if "params" in sig:
        kwargs["params"] = params
    if "config" in sig:
        kwargs["config"] = config
    return model_fn(features, **kwargs)


def _to_device(t, device):
    if t is None:
        return None
    if isinstance(t, dict):
        return {k: _to_device(v, device) for k, v in t.items()}
    if isinstance(t, (tuple, list)):
        return type(t)(_to_device(v, device) for v in t)
    if not torch.is_tensor(t):
        t = torch.as_tensor(t)
    if t.dtype == torch.float64:
        t = t.float()
    return t.to(device, non_blocking=True)


def _clone_tensors(t):
    if isinstance(t, dict):
        return {k: _clone_tensors(v) for k, v in t.items()}
    if isinstance(t, (tuple, list)):
        return type(t)(_clone_tensors(v) for v in t)
    return t.clone() if torch.is_tensor(t) else t


def _copy_tensors(dst, src) -> None:
    if isinstance(dst, dict):
        for k in dst:
            _copy_tensors(dst[k], src[k])
    elif isinstance(dst, (tuple, list)):
        for d, s_ in zip(dst, src):
            _copy_tensors(d, s_)
    elif torch.is_tensor(dst):
        dst.copy_(src, non_blocking=True)


def _signature(*ts):
    out = []
    for t in ts:
        if isinstance(t, dict):
            out.append(tuple((k, _signature(t[k])) for k in sorted(t)))
        elif isinstance(t, (tuple, list)):
            out.append(tuple(_signature(v) for v in t))
        elif torch.is_tensor(t):
            out.append((tuple(t.shape), str(t.dtype)))
        else:
            out.append(None)
    return tuple(out)


def _split(item):
    if isinstance(item, (tuple, list)) and len(item) == 2:
        return item[0], item[1]
    return item, None


class Estimator:
    def __init__(self, model_fn: Callable, model_dir: Optional[str] = None, config: Optional[RunConfig] = None,
                 params: Optional[Dict[str, Any]] = None, warm_start_from: Optional[str] = None):
        self._model_fn = model_fn
        self._config = config or RunConfig()
        self._model_dir = model_dir or self._config.model_dir or tempfile.mkdtemp(prefix="tfy_estimator_")
        if self._config.model_dir is None:
            self._config = self._config.replace(model_dir=self._model_dir)
        self._params = dict(params or {})
        self._warm_start_from = warm_start_from
        self._network: Optional[nn.Module] = None
        self._spec: Optional[EstimatorSpec] = None
        self._optimizer = None
        self._opt_desc: Optional[kopt.Optimizer] = None
        self._scheduled = []
        self._opt_by_name: Dict[str, kopt.Optimizer] = {}
        self._global_step = 0
        self._device: Optional[torch.device] = None
        self._ps = None
        self._ps_graph = None
        self._ps_state: Optional[Dict[str, dict]] = None
        self._last_loss_t = None
        self._pending_broadcast: Optional[int] = None
        self.last_loss: Optional[float] = None

    # -- properties the reference's tasks read / assign ---------------------------
    @property
    def model_dir(self) -> str:
        return self._model_dir

    @property
    def config(self) -> RunConfig:
        return self._config

    @property
    def params(self) -> Dict[str, Any]:
        return self._params

    @property
    def model_fn(self) -> Callable:
        return self._model_fn

    def get_global_step(self) -> int:
        return self._global_step

    # ---------------------------------------------------------------------- build
    def _default_device(self) -> torch.device:
        if torch.cuda.is_available():
            ids = [int(v) for v in os.environ.get("TFY_GPU_IDS", "").split(",") if v.strip() != ""]
            return torch.device(f"cuda:{ids[0]}" if ids else f"cuda:{torch.cuda.current_device()}")
        return torch.device("cpu")

    def _build(self, features, labels, mode: str) -> EstimatorSpec:
        spec = _call_model_fn(self._model_fn, features, labels, mode, self._params, self._config)
        if not isinstance(spec, EstimatorSpec):
            raise TypeError("model_fn must return an EstimatorSpec")
        if self._network is None:
            self._device = self._device or self._default_device()
            self._network = spec.network.to(self._device) if spec.network is not None else None
            if self._config.tf_random_seed is not None:
                torch.manual_seed(self._config.tf_random_seed)
        self._spec = spec._replace(network=self._network)
        return self._spec

    @staticmethod
    def _resolve_opt(opt):
        if opt is None:
            opt = "sgd"
        if callable(opt) and not isinstance(opt, kopt.Optimizer) and not hasattr(opt, "_tfy_inner_optimizer"):
            opt = opt()
        return kopt.get(opt)

    def _make_optimizer(self, spec: EstimatorSpec):
        desc = self._resolve_opt(spec.optimizer)
        # per-prefix optimizers (longest prefix wins); self._opt_by_name maps every parameter to its descriptor
        groups = [(pref, self._resolve_opt(o)) for pref, o in (spec.optimizers or {}).items()]
        groups.sort(key=lambda g: -len(g[0]))
        # refused before any optimizer state is set, so every later train() call refuses it again
        if any(getattr(d, "gradient_accumulation_steps", None) is not None for d in [desc, *(g for _, g in groups)]):
            raise ValueError("Estimator does not support gradient_accumulation_steps (neither the local and "
                             "all-reduce paths nor the parameter servers accumulate gradients): use Model.fit")
        self._opt_desc = desc
        named = [(n, p) for n, p in self._network.named_parameters() if p.requires_grad] \
            if self._network is not None else []
        self._opt_by_name = {}
        buckets = {}
        for n, p in named:
            d = next((gd for pref, gd in groups if n.startswith(pref)), desc)
            self._opt_by_name[n] = d
            buckets.setdefault(id(d), (d, []))[1].append(p)
        # (torch optimizer, schedule) of every bucket whose learning rate follows a LearningRateSchedule
        self._scheduled = []
        if not named:
            self._optimizer = None
        else:
            opts = [(d, d.to_torch(ps)) for d, ps in buckets.values()]
            self._optimizer = opts[0][1] if len(opts) == 1 else _MultiOptimizer([o for _, o in opts])
            self._scheduled = [(o, d.schedule) for d, o in opts if getattr(d, "schedule", None) is not None]

    def _variables(self) -> List[torch.Tensor]:
        if self._network is None:
            return []
        return [p.data for p in self._network.parameters()] + [b.data for b in self._network.buffers()]

    def broadcast_variables(self, root: int = 0) -> None:
        if self._network is None:
            self._pending_broadcast = root
            return
        from tf_yarn_b200 import hvd
        if hvd.is_initialized() and hvd.size() > 1:
            hvd.broadcast_parameters(self._variables(), root)

    # ------------------------------------------------------------------ checkpoints
    def latest_checkpoint(self) -> Optional[str]:
        return ckpt.latest_checkpoint(self._model_dir)

    def _save(self) -> str:
        payload = {"global_step": self._global_step,
                   "network": self._network.state_dict() if self._network is not None else None,
                   "optimizer": self._optimizer.state_dict() if self._optimizer is not None else None}
        if self._ps is not None:
            # the ps holds the weights and their optimizer slots: the local torch optimizer is never stepped
            payload["network"] = self._ps.state_dict_from_ps(self._network)
            payload["ps_state"] = self._ps.optimizer_state()
        path = ckpt.save_checkpoint(self._model_dir, self._global_step, payload, self._config.keep_checkpoint_max)
        logger.info("Saved checkpoint for step %d: %s", self._global_step, path)
        return path

    def _restore(self, path: Optional[str] = None, with_optimizer: bool = True) -> bool:
        path = path or self.latest_checkpoint() or self._warm_start_from
        if not path or not os.path.exists(path):
            return False
        payload = ckpt.load_checkpoint(path, map_location=self._device or "cpu")
        if self._network is not None and payload.get("network") is not None:
            self._network.load_state_dict(payload["network"])
        if with_optimizer and self._optimizer is not None and payload.get("optimizer") is not None:
            try:
                self._optimizer.load_state_dict(payload["optimizer"])
            except (ValueError, KeyError):
                logger.warning("optimizer state in %s does not match; starting it fresh", path)
        # the parameter servers' optimizer slots, for the connect_worker call in train (None: fresh slots)
        self._ps_state = payload.get("ps_state") if with_optimizer and self._ps is None else None
        self._global_step = int(payload.get("global_step", 0))
        logger.info("Restored from %s (global step %d)", path, self._global_step)
        return True

    # ------------------------------------------------------------------------ train
    def train(self, input_fn: Callable, hooks: Optional[Iterable] = None, steps: Optional[int] = None,
              max_steps: Optional[int] = None, saving_listeners=None) -> "Estimator":
        """Run training steps until ``steps`` more were done, ``max_steps`` is reached, the input is
        exhausted or a hook requests a stop."""
        from tf_yarn_b200.estimator import ps as ps_mod
        hooks = list(hooks or [])
        cfg = self._config
        cluster = cfg.cluster
        dataset = input_fn()
        it = iter(dataset)
        first = next(it, None)
        if first is None:
            return self
        features, labels = _split(first)
        spec = self._build(features, labels, ModeKeys.TRAIN)
        if self._optimizer is None and self._opt_desc is None:
            self._make_optimizer(spec)
        distributed = bool(self._opt_desc is not None and self._opt_desc.distributed)
        if distributed:
            from tf_yarn_b200 import hvd
            if not hvd.is_initialized():
                hvd.init()
            if self._device.type != "cuda":
                hvd.ensure_cpu_group()
        is_chief = cluster.is_chief
        use_ps = cluster.has_ps and cluster.task_type in ("chief", "worker")
        self._restore()
        if use_ps and self._ps is None and self._network is not None:
            if self._device.type == "cuda" and os.environ.get("TFY_PS_PLANE", "auto") != "shm":
                from tf_yarn_b200.estimator import ps_hbm
                self._ps = ps_hbm.connect_worker(self._network, self._opt_desc, cluster, is_chief,
                                                 self._global_step, opt_by_name=self._opt_by_name,
                                                 ps_state=self._ps_state)
            else:
                self._ps = ps_mod.connect_worker(self._network, self._opt_desc, cluster, is_chief,
                                                 self._global_step, opt_by_name=self._opt_by_name,
                                                 ps_state=self._ps_state)
            self._ps_state = None
            if not is_chief:
                self._global_step = self._ps.global_step()
        if self._pending_broadcast is not None:
            root, self._pending_broadcast = self._pending_broadcast, None
            self.broadcast_variables(root)

        writes_files = is_chief and cfg.model_dir is not None
        writer = summary_lib.writer(self._model_dir) if (writes_files and cfg.save_summary_steps) else None
        for h in hooks:
            h.begin()
        for h in hooks:
            try:
                h.after_create_session(self, None)
            except TypeError:
                h.after_create_session()
        if writes_files and self._global_step == 0 and \
                (cfg.save_checkpoints_steps or cfg.save_checkpoints_secs) and self.latest_checkpoint() is None:
            self._save()

        ctx = SessionRunContext(self, self._global_step)
        start_step = self._global_step
        item = first
        if self._network is not None:
            self._network.train()
        # failure detection: a synchronous all-reduce step waits on the peer ranks inside a kernel; without a
        # heartbeat a dead peer would hang this task instead of failing it (utils/watchdog.py)
        from tf_yarn_b200.utils import watchdog
        wd = watchdog.StepWatchdog(watchdog.default_timeout(distributed), "Estimator.train").start()
        try:
            item = self._train_loop(item, it, hooks, ctx, wd, distributed, steps, max_steps, start_step, writer,
                                    writes_files, cfg)
        finally:
            wd.close()
        loss = self._last_loss_t
        self.last_loss = self._read_loss(loss) if self._global_step > start_step else self.last_loss
        if writes_files and (cfg.save_checkpoints_steps or cfg.save_checkpoints_secs) and \
                self._global_step > start_step:
            st = ckpt.get_checkpoint_state(self._model_dir)
            if st is None or ckpt.step_of(st.model_checkpoint_path) != self._global_step:
                self._save()
        for h in hooks:
            try:
                h.end(None)
            except TypeError:
                h.end()
        if writer is not None:
            writer.flush()
            writer.close()
        logger.info("Loss for final step: %s.", self.last_loss)
        return self

    def _train_loop(self, item, it, hooks, ctx, wd, distributed, steps, max_steps, start_step, writer, writes_files,
                    cfg):
        last_save_time, last_save_step = time.time(), self._global_step
        last_log_time, last_log_step = time.time(), self._global_step
        while item is not None:
            if max_steps is not None and self._global_step >= max_steps:
                break
            if steps is not None and self._global_step - start_step >= steps:
                break
            features, labels = _split(item)
            wants_step = [h for h in hooks if _wants_global_step(h.before_run(ctx))]
            prev_gs = self._global_step
            loss = self._train_step(features, labels, distributed)
            wd.beat()
            self._last_loss_t = loss          # device scalar of this step (hooks may read it: one 4-byte D2H)
            if self._ps is not None:
                self._global_step = self._ps.increment_global_step()
            else:
                self._global_step += 1
            ctx.step = self._global_step
            for h in hooks:
                h.after_run(ctx, SessionRunValues(results=self._global_step if h in wants_step else None))
            gs = self._global_step
            if writer is not None and cfg.save_summary_steps and \
                    gs // cfg.save_summary_steps > (gs - 1 if self._ps is None else prev_gs) // cfg.save_summary_steps:
                self.last_loss = self._read_loss(loss)
                writer.add_scalar("loss", self.last_loss, gs)
            if cfg.log_step_count_steps and gs - last_log_step >= cfg.log_step_count_steps:
                now = time.time()
                self.last_loss = self._read_loss(loss)
                sps = (gs - last_log_step) / max(now - last_log_time, 1e-9)
                logger.info("global_step/sec: %.4g  loss = %.6g, step = %d", sps, self.last_loss, gs)
                if writer is not None:
                    writer.add_scalar("global_step/sec", sps, gs)
                last_log_time, last_log_step = now, gs
            if writes_files:
                # with asynchronous workers the chief sees the global step advance by several units
                # per local step: trigger on crossing a multiple, not on hitting it exactly
                due = (cfg.save_checkpoints_steps and
                       gs // cfg.save_checkpoints_steps > last_save_step // cfg.save_checkpoints_steps) or \
                      (cfg.save_checkpoints_secs and time.time() - last_save_time >= cfg.save_checkpoints_secs)
                if due:
                    self._save()
                    last_save_time, last_save_step = time.time(), gs
            if ctx.stop_requested:
                break
            item = next(it, None)
        return item

    def _read_loss(self, loss) -> float:
        """The loss on the host; then the loss's own ``check()`` (a canned head raises on invalid labels it flagged
        on the device), which costs no extra wait: the device has just been synchronised by the read."""
        value = float(loss)
        check = getattr(self._spec.loss, "check", None) if self._spec is not None else None
        if check is not None:
            check()
        return value

    @staticmethod
    def _loss(spec: EstimatorSpec, features, labels, outputs) -> torch.Tensor:
        if spec.weights is None:
            return spec.loss(labels, outputs)
        return spec.loss(labels, outputs, spec.weights(features))

    def _ps_step_body(self, features, labels) -> torch.Tensor:
        """pull -> forward -> backward -> push against the parameter servers (kernels only: capturable)."""
        self._ps.pull(self._network)
        self._optimizer.zero_grad(set_to_none=False)
        outputs = self._network(features)
        loss = self._loss(self._spec, features, labels, outputs)
        loss.backward()
        self._ps.push(self._network)
        return loss.detach()

    def _ps_step_cuda(self, features, labels) -> torch.Tensor:
        """H100 parameter-server step.  After three eager steps the whole pull/forward/backward/push sequence is
        captured in a CUDA graph and replayed on static input buffers: the data plane is a handful of
        microsecond-scale peer-memory kernels, so an eager step is bound by Python / launch overhead (the
        round-1 review measured it host-bound).  TFY_PS_GRAPH=0 keeps it eager."""
        if hasattr(self._ps, "refresh_adam_scale"):
            self._ps.refresh_adam_scale()
        st = self._ps_graph
        if st is None:
            st = self._ps_graph = {"warm": 0, "off": os.environ.get("TFY_PS_GRAPH", "1") == "0"}
        if st["off"]:
            return self._ps_step_body(features, labels)
        if "graph" not in st:
            prof_path = os.environ.get("TFY_PS_PROFILE")
            if prof_path and st["warm"] == 2:
                # per-kernel device times of ONE eager step (torch profiler / CUPTI), for tuning the data plane
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    loss = self._ps_step_body(features, labels)
                    torch.cuda.synchronize()
                with open(prof_path, "w") as f:
                    f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90))
            else:
                loss = self._ps_step_body(features, labels)      # eager warm-up steps
            st["warm"] += 1
            if st["warm"] >= 3:
                try:
                    sf, sl = _clone_tensors(features), _clone_tensors(labels)
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        sloss = self._ps_step_body(sf, sl)
                    st.update(graph=g, feats=sf, labels=sl, loss=sloss, sig=_signature(features, labels))
                    logger.info("parameter-server train step captured in a CUDA graph")
                except Exception as exc:  # noqa: BLE001
                    logger.warning("CUDA-graph capture of the PS step failed (%s); staying eager", exc)
                    st["off"] = True
                    st["error"] = f"{type(exc).__name__}: {exc}"[:600]
            return loss
        if _signature(features, labels) != st["sig"]:
            return self._ps_step_body(features, labels)          # odd-shaped batch: run it eagerly
        _copy_tensors(st["feats"], features)
        _copy_tensors(st["labels"], labels)
        st["graph"].replay()
        return st["loss"]

    def _train_step(self, features, labels, distributed: bool) -> torch.Tensor:
        spec = self._spec
        if self._network is None or self._optimizer is None:
            return torch.zeros(())
        features = _to_device(features, self._device)
        labels = _to_device(labels, self._device)
        if self._ps is not None and hasattr(self._ps, "traffic_per_step"):      # the peer-HBM plane (ps_hbm)
            return self._ps_step_cuda(features, labels)
        if self._ps is not None:
            self._ps.pull(self._network)
        self._optimizer.zero_grad(set_to_none=False)
        outputs = self._network(features)
        loss = self._loss(spec, features, labels, outputs)
        loss.backward()
        if self._ps is not None:
            self._ps.push(self._network)
            return loss.detach()
        if distributed:
            from tf_yarn_b200 import hvd
            grads = [p.grad for p in self._network.parameters() if p.grad is not None]
            hvd.grouped_allreduce_(grads, average=True)
        for opt, schedule in self._scheduled:          # the rate of this update: the schedule at the global step
            lr = float(schedule(self._global_step))
            for g in opt.param_groups:
                g["lr"] = lr
        self._optimizer.step()
        return loss.detach()

    # --------------------------------------------------------------------- evaluate
    def evaluate(self, input_fn: Callable, steps: Optional[int] = None, hooks: Optional[Iterable] = None,
                 checkpoint_path: Optional[str] = None, name: Optional[str] = None) -> Dict[str, Any]:
        """Metrics over ``steps`` batches of ``input_fn()`` using ``checkpoint_path`` (default: latest).

        Returns ``{"loss": ..., <metric>: ..., "global_step": step of the checkpoint}`` and writes the
        same scalars to ``<model_dir>/eval[_<name>]`` as TensorBoard events.
        """
        hooks = list(hooks or [])
        it = iter(input_fn())
        first = next(it, None)
        if first is None:
            return {}
        features, labels = _split(first)
        spec = self._build(features, labels, ModeKeys.EVAL)
        path = checkpoint_path or self.latest_checkpoint()
        if path:
            if not self._restore(path, with_optimizer=False) and checkpoint_path:
                # an explicitly named checkpoint that vanished (the chief prunes old ones: keep_checkpoint_max) must
                # not be "evaluated" with whatever weights the network happens to hold
                raise FileNotFoundError(f"checkpoint {checkpoint_path} does not exist (pruned while waiting?)")
        elif self._ps is not None and self._network is not None:
            self._ps.pull(self._network)
        gs = self._global_step
        for h in hooks:
            h.begin()
        for h in hooks:
            try:
                h.after_create_session(self, None)
            except TypeError:
                h.after_create_session()
        ctx = SessionRunContext(self, gs)
        metric_fns = dict(spec.eval_metric_ops or {})
        # values are (numerator, denominator) callables or stateful keras.metrics.Metric objects (AUC, ...), as in TF2
        stateful = {k for k, fn in metric_fns.items() if isinstance(fn, Metric)}
        for k in stateful:
            metric_fns[k].reset_state()
        num = {k: 0.0 for k in metric_fns}
        den = {k: 0.0 for k in metric_fns}
        loss_sum, n_batches = 0.0, 0
        if self._network is not None:
            self._network.eval()
        item = first
        with torch.no_grad():
            while item is not None and (steps is None or n_batches < steps):
                features, labels = _split(item)
                wants_step = [h for h in hooks if _wants_global_step(h.before_run(ctx))]
                features = _to_device(features, self._device or torch.device("cpu"))
                labels = _to_device(labels, self._device or torch.device("cpu"))
                outputs = self._network(features) if self._network is not None else features
                w = spec.weights(features) if spec.weights is not None else None
                if spec.loss is not None:
                    loss_sum += float(spec.loss(labels, outputs) if w is None else spec.loss(labels, outputs, w))
                for k, fn in metric_fns.items():
                    if k in stateful:
                        # device-side state: no host read per batch
                        if w is None:
                            fn.update_state(labels, outputs)
                        else:
                            fn.update_state(labels, outputs, sample_weight=w)
                        continue
                    a, b = fn(labels, outputs) if w is None else fn(labels, outputs, w)
                    num[k] += float(a)
                    den[k] += float(b)
                n_batches += 1
                for h in hooks:
                    h.after_run(ctx, SessionRunValues(results=gs if h in wants_step else None))
                if ctx.stop_requested:
                    break
                item = next(it, None)
        for h in hooks:
            try:
                h.end(None)
            except TypeError:
                h.end()
        check = getattr(spec.loss, "check", None)
        if check is not None:
            check()
        results: Dict[str, Any] = {"loss": loss_sum / max(n_batches, 1)}
        for k, fn in metric_fns.items():
            results[k] = fn.result() if k in stateful else num[k] / max(den[k], 1.0)
        results[GraphKeys.GLOBAL_STEP] = gs
        eval_dir = os.path.join(self._model_dir, "eval" if not name else f"eval_{name}")
        w = summary_lib.writer(eval_dir)
        for k, v in results.items():
            if k != GraphKeys.GLOBAL_STEP:
                w.add_scalar(k, v, gs)
        w.flush()
        w.close()
        logger.info("Saving dict for global step %d: %s", gs, results)
        return results

    # ---------------------------------------------------------------------- predict
    def predict(self, input_fn: Callable, checkpoint_path: Optional[str] = None, yield_single_examples: bool = True):
        it = iter(input_fn())
        first = next(it, None)
        if first is None:
            return
        features, _ = _split(first)
        spec = self._build(features, None, ModeKeys.PREDICT)
        path = checkpoint_path or self.latest_checkpoint()
        if path:
            self._restore(path, with_optimizer=False)
        if self._network is not None:
            self._network.eval()
        item = first
        with torch.no_grad():
            while item is not None:
                features, _ = _split(item)
                features = _to_device(features, self._device or torch.device("cpu"))
                outputs = self._network(features) if self._network is not None else features
                preds = spec.predictions(outputs) if spec.predictions is not None else outputs
                if yield_single_examples:
                    if isinstance(preds, dict):
                        n = next(iter(preds.values())).shape[0]
                        for i in range(n):
                            yield {k: v[i].cpu().numpy() for k, v in preds.items()}
                    else:
                        for row in preds:
                            yield row.cpu().numpy() if torch.is_tensor(row) else row
                else:
                    yield preds
                item = next(it, None)

    # ----------------------------------------------------------------------- export
    def export_saved_model(self, export_dir_base: str, serving_input_receiver_fn=None,
                           checkpoint_path: Optional[str] = None, **_ignored) -> str:
        """Write the network (weights of ``checkpoint_path``) under ``export_dir_base/<timestamp>``."""
        path = checkpoint_path or self.latest_checkpoint()
        if self._network is None:
            raise RuntimeError("export needs a built network: call train() or evaluate() first")
        if path:
            self._restore(path, with_optimizer=False)
        stamp = int(time.time())
        while True:                     # like TF: two exports within one second get distinct, increasing directories
            out = os.path.join(export_dir_base, str(stamp))
            try:
                os.makedirs(out)
                break
            except FileExistsError:
                stamp += 1
        tmp = os.path.join(out, f"saved_model.pt.tmp{os.getpid()}")
        import cloudpickle
        with open(tmp, "wb") as f:
            cloudpickle.dump({"network": self._network.to("cpu"), "global_step": self._global_step}, f)
        os.replace(tmp, os.path.join(out, "saved_model.pt"))
        self._network.to(self._device)
        return out

    export_savedmodel = export_saved_model


class _MultiOptimizer:
    """Several torch optimizers (one per parameter group of EstimatorSpec.optimizers) behind one interface."""

    def __init__(self, opts):
        self.opts = list(opts)

    @property
    def param_groups(self):
        return [g for o in self.opts for g in o.param_groups]

    def zero_grad(self, set_to_none: bool = False):
        for o in self.opts:
            o.zero_grad(set_to_none=set_to_none)

    def step(self):
        for o in self.opts:
            o.step()

    def state_dict(self):
        return {"multi": [o.state_dict() for o in self.opts]}

    def load_state_dict(self, state):
        for o, st in zip(self.opts, state["multi"]):
            o.load_state_dict(st)


def _wants_global_step(args) -> bool:
    return isinstance(args, SessionRunArgs) and args.fetches == GLOBAL_STEP
