"""Thresholded confusion histograms behind the Keras ``AUC`` / ``Precision`` / ``Recall`` metrics.

The state of one metric is a float64 histogram ``[2, T+1]`` -- row 0 the positive weight ``y*w``, row 1 the negative
weight ``(1-y)*w`` of the predictions in each bucket -- plus an error-flag word.  Bucket ``b`` holds the predictions
that are positive at every threshold ``j <= b``; bucket ``T`` (explicit thresholds only) those positive at none.  On a
CUDA device one update is one launch of ``tfy_confusion_update`` (``ops/csrc/tfy_confusion.cu``): deterministic, no host
sync, state in persistent device buffers, so it can run inside a captured train step.  On the CPU the same histogram
is computed with float64 torch ops.  ``curves`` turns a histogram into the tf.keras 2.x results.

Soft labels contribute ``y*w`` positive and ``(1-y)*w`` negative weight on both threshold paths (tf.keras does the same
for its default evenly spaced thresholds; for explicit thresholds it differs for labels strictly between 0 and 1).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np
import torch

from tf_yarn_b200.ops import native

_vp, _i, _i64, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
native.declare("tfy_confusion_update", [_vp, _i, _vp, _i, _vp, _i64, _i64, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp])
native.declare("tfy_confusion_scratch_bytes", [_i64, _i], restype=ctypes.c_size_t)
native.declare("tfy_confusion_max_thresholds", [])

MAX_THRESHOLDS = 1000          # tfy_confusion.cu: kMaxThresholds
EPSILON = 1e-7                 # Keras backend.epsilon(): the ends of the AUC thresholds
BAD_PREDICTION, BAD_LABEL = 1, 2


def even_thresholds(num_thresholds: int) -> np.ndarray:
    """Keras's default AUC thresholds: ``-eps, 1/(T-1), ..., (T-2)/(T-1), 1+eps``."""
    t = np.arange(num_thresholds, dtype=np.float64) / (num_thresholds - 1)
    t[0], t[-1] = -EPSILON, 1.0 + EPSILON
    return t


class ConfusionState:
    """Histogram ``[2, T+1]`` and error flags of one metric, allocated on the device of the first update.

    ``thresholds=None`` selects the evenly spaced default; otherwise a sorted float32 list of ``T`` thresholds."""

    def __init__(self, num_thresholds: int, thresholds: Optional[Sequence[float]] = None, from_logits: bool = False):
        if not 2 <= num_thresholds <= MAX_THRESHOLDS:
            raise ValueError(f"num_thresholds must be in [2, {MAX_THRESHOLDS}], got {num_thresholds}")
        self.T = int(num_thresholds)
        self.thresholds = None if thresholds is None else torch.tensor(sorted(float(t) for t in thresholds),
                                                                       dtype=torch.float32)
        if self.thresholds is not None and self.thresholds.numel() != self.T:
            raise ValueError("thresholds and num_thresholds disagree")
        self.from_logits = bool(from_logits)
        self.device: Optional[torch.device] = None
        self.acc: Optional[torch.Tensor] = None        # float64 [2, T+1]
        self.flags: Optional[torch.Tensor] = None      # int32 [1] (the kernel ORs uint32 bits into it)
        self._scratch: Optional[torch.Tensor] = None
        self._thr_dev: Optional[torch.Tensor] = None

    def _allocate(self, device: torch.device) -> None:
        self.device = device
        self.acc = torch.zeros(2, self.T + 1, dtype=torch.float64, device=device)
        self.flags = torch.zeros(1, dtype=torch.int32, device=device)
        if device.type == "cuda":
            lib = native.load()
            nbytes = int(lib.tfy_confusion_scratch_bytes(0, self.T))      # the largest grid: one buffer for every N
            self._scratch = torch.zeros(nbytes, dtype=torch.uint8, device=device)
            if self.thresholds is not None:
                self._thr_dev = self.thresholds.to(device)

    def state_tensors(self):
        """The device tensors that hold the state (for snapshot / restore around a train engine's warm-up steps)."""
        return [] if self.acc is None else [self.acc, self.flags]

    def reset(self) -> None:
        if self.acc is not None:
            self.acc.zero_()
            self.flags.zero_()

    def update(self, y_true: torch.Tensor, y_pred: torch.Tensor, sample_weight: Optional[torch.Tensor] = None) -> None:
        n = y_pred.numel()
        if y_true.numel() != n:
            raise ValueError(f"labels have {y_true.numel()} elements, predictions {n}")
        if self.acc is None or self.device != y_pred.device:
            if self.acc is not None:
                raise ValueError(f"metric state lives on {self.device}, the update is on {y_pred.device}")
            self._allocate(y_pred.device)
        per_sample = 0
        if sample_weight is not None:
            sample_weight = sample_weight.reshape(-1)
            b = sample_weight.numel()
            if b == 0 or n % b:
                raise ValueError(f"{b} sample weights for {n} prediction elements")
            per_sample = n // b
        if n == 0:
            return
        if y_pred.device.type == "cuda":
            self._update_cuda(y_true, y_pred, sample_weight, n, per_sample)
        else:
            self._update_cpu(y_true, y_pred, sample_weight, per_sample)

    def _update_cuda(self, y_true, y_pred, sample_weight, n, per_sample) -> None:
        lib = native.load()
        pred = y_pred.reshape(-1)
        if pred.dtype not in (torch.float32, torch.bfloat16):
            pred = pred.float()
        pred = pred.contiguous()
        lab = y_true.reshape(-1)
        if lab.dtype not in (torch.float32, torch.int64):
            lab = lab.float()
        lab = lab.to(pred.device).contiguous()
        w = None
        if sample_weight is not None:
            w = sample_weight.to(device=pred.device, dtype=torch.float32).contiguous()
        s = torch.cuda.current_stream(pred.device).cuda_stream
        rc = lib.tfy_confusion_update(pred.data_ptr(), int(pred.dtype == torch.bfloat16), lab.data_ptr(),
                                      int(lab.dtype == torch.int64), w.data_ptr() if w is not None else None, n,
                                      per_sample, self.T, self._thr_dev.data_ptr() if self._thr_dev is not None else None,
                                      int(self.from_logits), self.acc.data_ptr(), self.flags.data_ptr(),
                                      self._scratch.data_ptr(), self._scratch.numel(), s)
        native.check(rc, "tfy_confusion_update")

    def _update_cpu(self, y_true, y_pred, sample_weight, per_sample) -> None:
        hist, flags = histogram_cpu(y_true, y_pred, sample_weight, per_sample, self.T, self.thresholds,
                                    self.from_logits)
        self.acc += hist
        self.flags |= flags

    def histogram(self) -> torch.Tensor:
        """The accumulated histogram on the host (one device-to-host copy); raises on flagged invalid input."""
        if self.acc is None:
            return torch.zeros(2, self.T + 1, dtype=torch.float64)
        flags = int(self.flags.item())
        if flags & BAD_PREDICTION:
            raise ValueError("predictions must be in [0, 1] (got a value outside it, or NaN); pass from_logits=True "
                             "for logits")
        if flags & BAD_LABEL:
            raise ValueError("labels must be in [0, 1] (got a value outside it, or NaN)")
        return self.acc.cpu()


def histogram_cpu(y_true: torch.Tensor, y_pred: torch.Tensor, sample_weight: Optional[torch.Tensor], per_sample: int,
                  num_thresholds: int, thresholds: Optional[torch.Tensor], from_logits: bool):
    """The kernel's histogram with float64 torch ops on the CPU: ``(hist [2, T+1] float64, flags int32 [1])``."""
    p = y_pred.detach().reshape(-1).cpu().float()
    if from_logits:
        p = 1.0 / (1.0 + torch.exp(-p))
    y = y_true.detach().reshape(-1).cpu()
    y32 = y.float()
    p_ok = (p >= 0) & (p <= 1)
    y_ok = (y32 >= 0) & (y32 <= 1)
    flags = torch.tensor([(0 if bool(p_ok.all()) else BAD_PREDICTION) | (0 if bool(y_ok.all()) else BAD_LABEL)],
                         dtype=torch.int32)
    ok = p_ok & y_ok
    T = num_thresholds
    if thresholds is None:
        b = (torch.ceil(p * torch.tensor(float(T - 1), dtype=torch.float32)) - 1).clamp_min(0)
        b = torch.nan_to_num(b, nan=0.0).long()
    else:
        c = torch.searchsorted(thresholds, p, side="left")          # thresholds strictly below p
        b = torch.where(c == 0, torch.full_like(c, T), c - 1)
    w = torch.ones(p.numel(), dtype=torch.float64)
    if sample_weight is not None:
        w = sample_weight.detach().reshape(-1).cpu().double().repeat_interleave(per_sample)
    yd = y32.double()
    vp = torch.where(ok, yd * w, torch.zeros_like(w))
    vn = torch.where(ok, (1.0 - yd) * w, torch.zeros_like(w))
    b = torch.where(ok, b, torch.zeros_like(b))
    hist = torch.stack([torch.bincount(b, weights=vp, minlength=T + 1), torch.bincount(b, weights=vn, minlength=T + 1)])
    return hist.double(), flags


def _div(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Division with 0 where the denominator is 0 (tf.math.divide_no_nan)."""
    out = np.zeros(np.broadcast(a, b).shape, dtype=np.float64)
    np.divide(a, b, out=out, where=(b != 0))
    return out


def confusion(hist: torch.Tensor, num_thresholds: int):
    """``(tp, fp, fn, tn)``, each float64 ``[T]``, from a histogram ``[2, T+1]``."""
    h = hist.double().numpy()
    T = num_thresholds
    pos, neg = h[0], h[1]
    tp = np.cumsum(pos[:T][::-1])[::-1]
    fp = np.cumsum(neg[:T][::-1])[::-1]
    return tp, fp, pos.sum() - tp, neg.sum() - fp


def auc(tp, fp, fn, tn, curve: str, summation_method: str) -> float:
    """tf.keras 2.x ``AUC.result()`` (and ``interpolate_pr_auc`` for PR with interpolation), in float64."""
    T = tp.shape[0]
    if curve == "PR" and summation_method == "interpolation":
        dtp = tp[:T - 1] - tp[1:]
        p = tp + fp
        dp = p[:T - 1] - p[1:]
        slope = _div(dtp, np.maximum(dp, 0))
        intercept = tp[1:] - slope * p[1:]
        both = (p[:T - 1] > 0) & (p[1:] > 0)
        ratio = np.where(both, _div(p[:T - 1], np.maximum(p[1:], 0)), np.ones_like(p[1:]))
        inc = _div(slope * (dtp + intercept * np.log(ratio)), np.maximum(tp[1:] + fn[1:], 0))
        return float(inc.sum())
    recall = _div(tp, tp + fn)
    if curve == "ROC":
        x, y = _div(fp, fp + tn), recall
    else:
        x, y = recall, _div(tp, tp + fp)
    if summation_method == "interpolation":
        h = (y[:T - 1] + y[1:]) / 2.0
    elif summation_method == "minoring":
        h = np.minimum(y[:T - 1], y[1:])
    else:
        h = np.maximum(y[:T - 1], y[1:])
    return float(((x[:T - 1] - x[1:]) * h).sum())
