"""Keras-style callbacks (the subset the reference's tasks and examples touch).

``ModelCheckpoint`` identity matters: the all-reduce task strips it from
non-chief ranks with an ``isinstance`` test (reference:
tf_yarn/tensorflow/tasks/gloo_allred_task.py:77-83).
"""
from __future__ import annotations

import logging
import os
from typing import Any, Callable, Dict, List, Optional

logger = logging.getLogger(__name__)


def _auto_mode(monitor: str) -> str:
    """``mode="auto"``: larger is better for accuracies and for the AUC / precision / recall metrics."""
    if "acc" in monitor or monitor.endswith(("auc", "precision", "recall")):
        return "max"
    return "min"


class Callback:
    def __init__(self):
        self.model = None
        self.params: Dict[str, Any] = {}

    def set_model(self, model) -> None:
        self.model = model

    def set_params(self, params: Dict[str, Any]) -> None:
        self.params = params

    def on_train_begin(self, logs=None): ...
    def on_train_end(self, logs=None): ...
    def on_epoch_begin(self, epoch, logs=None): ...
    def on_epoch_end(self, epoch, logs=None): ...
    def on_train_batch_begin(self, batch, logs=None): ...
    def on_train_batch_end(self, batch, logs=None): ...

    # set to True when the callback reads `logs` in on_train_batch_end: fit() then synchronises the
    # loss read-back every step instead of lagging it behind the GPU
    needs_batch_logs = False


class History(Callback):
    def on_train_begin(self, logs=None):
        self.epoch: List[int] = []
        self.history: Dict[str, List[float]] = {}

    def on_epoch_end(self, epoch, logs=None):
        self.epoch.append(epoch)
        for k, v in (logs or {}).items():
            self.history.setdefault(k, []).append(v)


class LambdaCallback(Callback):
    def __init__(self, on_epoch_begin=None, on_epoch_end=None, on_train_begin=None, on_train_end=None,
                 on_train_batch_begin=None, on_train_batch_end=None):
        super().__init__()
        for name, fn in dict(on_epoch_begin=on_epoch_begin, on_epoch_end=on_epoch_end,
                             on_train_begin=on_train_begin, on_train_end=on_train_end,
                             on_train_batch_begin=on_train_batch_begin,
                             on_train_batch_end=on_train_batch_end).items():
            if fn is not None:
                setattr(self, name, fn)
        self.needs_batch_logs = on_train_batch_end is not None


class ModelCheckpoint(Callback):
    """Save the model at the end of every ``period`` epochs to ``filepath.format(epoch=..., **logs)``."""

    def __init__(self, filepath: str, monitor: str = "val_loss", save_best_only: bool = False,
                 save_weights_only: bool = False, mode: str = "auto", period: int = 1, verbose: int = 0):
        super().__init__()
        self.filepath, self.monitor = filepath, monitor
        self.save_best_only, self.save_weights_only = save_best_only, save_weights_only
        self.period, self.verbose = period, verbose
        self._since = 0
        if mode == "auto":
            mode = _auto_mode(monitor)
        self._better = (lambda a, b: a > b) if mode == "max" else (lambda a, b: a < b)
        self.best: Optional[float] = None

    def on_epoch_end(self, epoch, logs=None):
        logs = logs or {}
        self._since += 1
        if self._since < self.period:
            return
        self._since = 0
        if self.save_best_only:
            cur = logs.get(self.monitor)
            if cur is None or (self.best is not None and not self._better(cur, self.best)):
                return
            self.best = cur
        path = self.filepath.format(epoch=epoch + 1, **logs)
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        if self.save_weights_only:
            self.model.save_weights(path)
        else:
            self.model.save(path)
        if self.verbose:
            logger.info("Epoch %d: saved model to %s", epoch + 1, path)


class LearningRateScheduler(Callback):
    def __init__(self, schedule: Callable[..., float], verbose: int = 0):
        super().__init__()
        self.schedule, self.verbose = schedule, verbose

    def on_epoch_begin(self, epoch, logs=None):
        if getattr(getattr(self.model, "optimizer", None), "schedule", None) is not None:
            raise TypeError("LearningRateScheduler cannot drive an optimizer whose learning_rate is a "
                            "LearningRateSchedule: the schedule already sets the rate of every step")
        lr = self.model.get_learning_rate()
        try:
            new = self.schedule(epoch, lr)
        except TypeError:
            new = self.schedule(epoch)
        self.model.set_learning_rate(float(new))


class TensorBoard(Callback):
    """Write epoch-level scalars as TensorBoard event files under ``log_dir``."""

    def __init__(self, log_dir: str = "logs", update_freq: str = "epoch"):
        super().__init__()
        self.log_dir = log_dir
        self._writer = None

    def on_train_begin(self, logs=None):
        from torch.utils.tensorboard import SummaryWriter
        self._writer = SummaryWriter(self.log_dir)

    def on_epoch_end(self, epoch, logs=None):
        for k, v in (logs or {}).items():
            self._writer.add_scalar(f"epoch_{k}", v, epoch)
        self._writer.flush()

    def on_train_end(self, logs=None):
        if self._writer is not None:
            self._writer.close()


class EarlyStopping(Callback):
    def __init__(self, monitor: str = "val_loss", min_delta: float = 0.0, patience: int = 0, mode: str = "auto"):
        super().__init__()
        self.monitor, self.min_delta, self.patience = monitor, min_delta, patience
        if mode == "auto":
            mode = _auto_mode(monitor)
        self._sign = 1.0 if mode == "max" else -1.0
        self.best: Optional[float] = None
        self.wait = 0

    def on_epoch_end(self, epoch, logs=None):
        cur = (logs or {}).get(self.monitor)
        if cur is None:
            return
        if self.best is None or self._sign * (cur - self.best) > self.min_delta:
            self.best, self.wait = cur, 0
        else:
            self.wait += 1
            if self.wait >= self.patience:         # Keras: stop after `patience` epochs without improvement
                self.model.stop_training = True


class CallbackList:
    def __init__(self, callbacks: Optional[List[Callback]], model, params: Dict[str, Any]):
        self.callbacks = list(callbacks or [])
        for cb in self.callbacks:
            cb.set_model(model)
            cb.set_params(params)
        self.needs_batch_logs = any(getattr(cb, "needs_batch_logs", False) for cb in self.callbacks)
        base = Callback
        self.has_batch_hooks = any(
            type(cb).on_train_batch_end is not base.on_train_batch_end
            or type(cb).on_train_batch_begin is not base.on_train_batch_begin
            or "on_train_batch_end" in cb.__dict__ or "on_train_batch_begin" in cb.__dict__
            for cb in self.callbacks)

    def call(self, hook: str, *args) -> None:
        for cb in self.callbacks:
            getattr(cb, hook)(*args)
