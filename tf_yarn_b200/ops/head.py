"""The canned estimators' head: loss and logit gradient of the binary, multi-class and regression heads, weighted or not.

Row ``i`` has logits ``z_i`` (``C`` values), label ``y_i`` and weight ``w_i`` (``w_i = 1`` without a weight column).
With ``c = 1`` for the classification heads and ``c = d`` for regression:

==========================  =========================================  ==========================================
head                        per-element loss ``l_ij``                  ``dl/dz_ij``
==========================  =========================================  ==========================================
binary (``C = 1``)          ``max(z,0) - z*y + log1p(exp(-|z|))``      ``sigmoid(z) - y``
multi-class (``C >= 2``)    ``logsumexp(z_i) - z_{i,y_i}`` (one/row)   ``softmax(z_i)_j - [j = y_i]``
regression (``C = d``)      ``(z_ij - y_ij)^2``                        ``2 (z_ij - y_ij)``
==========================  =========================================  ==========================================

The training loss is ``L = sum_i w_i sum_j l_ij / (B c)`` (TF2's ``SUM_OVER_BATCH_SIZE``; unweighted it is the mean of
``binary_cross_entropy_with_logits`` / ``cross_entropy`` / ``mse_loss``) and ``dL/dz_ij = w_i dl_ij/dz_ij / (B c)``.
The binary label is used as the float it is; a multi-class label outside ``[0, C)`` makes its row contribute nothing
to the loss or the gradient (the row still counts in ``B``) and sets a flag that :meth:`CannedHead.check` turns into a
``ValueError`` on the host.

On a CUDA device the loss and the gradient come from one launch of ``tfy_canned_head`` (``ops/csrc/tfy_head.cu``):
labels are read in place as int32, int64 or float32, the batch sum is deterministic, and nothing syncs with the host,
so the head runs inside the captured parameter-server step.  On the CPU the same contract is computed by
:func:`torch_head` (the torch statement); unweighted, it is exactly the torch mean the classifiers have always used.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from tf_yarn_b200.ops import native

_vp, _i, _i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
native.declare("tfy_canned_head", [_vp, _vp, _i, _vp, _i64, _i, _i, _vp, _vp, _vp, _vp, _vp])
native.declare("tfy_canned_head_scratch_bytes", [_i64, _i, _i], restype=ctypes.c_size_t)

BINARY, MULTI_CLASS, REGRESSION = 0, 1, 2          # tfy_head.cuh: TfyHead
BAD_LABEL = 1
_LABEL_CODES = {torch.float32: 0, torch.int32: 1, torch.int64: 2}


def torch_row_losses(head: int, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """``sum_j l_ij`` of every row as torch ops: ``[B]``."""
    z = logits.float()
    if head == BINARY:
        return F.binary_cross_entropy_with_logits(z.reshape(-1), labels.float().reshape(-1), reduction="none")
    if head == MULTI_CLASS:
        return F.cross_entropy(z, labels.long().reshape(-1), reduction="none")
    return ((z - labels.float().reshape(z.shape)) ** 2).sum(dim=1)


def torch_head(head: int, logits: torch.Tensor, labels: torch.Tensor, weights: Optional[torch.Tensor]) -> torch.Tensor:
    """The head's training loss as torch ops (the CPU path, and the statement the kernel is tested against).

    ``logits`` are ``[B, C]`` (``[B]`` or ``[B, 1]`` for the binary head); ``labels`` hold ``B`` values (binary,
    multi-class) or ``B*d`` (regression); ``weights`` is ``None`` or ``[B]``.  Unweighted, this is the torch mean
    (``binary_cross_entropy_with_logits`` / ``cross_entropy`` / ``mse_loss``) itself."""
    z = logits.float()
    if weights is None:
        if head == BINARY:
            return F.binary_cross_entropy_with_logits(z.reshape(-1), labels.float().reshape(-1))
        if head == MULTI_CLASS:
            return F.cross_entropy(z, labels.long().reshape(-1))
        return F.mse_loss(z, labels.float().reshape(z.shape))
    n = z.shape[0] if head == MULTI_CLASS else z.numel()          # B c
    return (torch_row_losses(head, z, labels) * weights.reshape(-1)).sum() / n


class _HeadFunction(torch.autograd.Function):
    """Forward: one kernel launch writes the loss and dL/dlogits.  Backward: the saved gradient times the incoming
    scalar."""

    @staticmethod
    def forward(ctx, logits, labels, weights, head):
        loss, grad = head._launch(logits, labels, weights, with_grad=True)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None


class _DeviceState:
    """Scratch (ticket + slabs) and flag word of one head on one device, kept for the head's lifetime: a captured
    graph that launched the kernel keeps using these addresses."""

    def __init__(self, device: torch.device):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("the canned head's device buffers must be allocated before a CUDA graph is captured; "
                               "run one eager step first")
        lib = native.load()
        nbytes = int(lib.tfy_canned_head_scratch_bytes(0, 0, 0))     # the largest grid: one buffer for every batch
        self.scratch = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self.flags = torch.zeros(1, dtype=torch.int32, device=device)


class CannedHead:
    """``loss(labels, logits[, weights])`` of one canned head, with :meth:`check` for the invalid-label flag.

    ``n_out`` is the number of logits per example: 1 for the binary head, ``n_classes`` for the multi-class head and
    ``label_dimension`` for regression."""

    def __init__(self, head: int, n_out: int):
        if head not in (BINARY, MULTI_CLASS, REGRESSION):
            raise ValueError(f"unknown head {head}")
        self.head = head
        self.n_out = int(n_out)
        self._state: Dict[torch.device, _DeviceState] = {}

    def __call__(self, labels: torch.Tensor, logits: torch.Tensor,
                 weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        B = logits.shape[0]
        if self.head == REGRESSION:
            want = [(B,), (B, 1)] if self.n_out == 1 else [(B, self.n_out)]
            if tuple(labels.shape) not in want:
                raise ValueError(f"regression labels must have shape {' or '.join(str(list(s)) for s in want)}, "
                                 f"got {list(labels.shape)}")
        if weights is not None and weights.numel() != B:
            raise ValueError(f"{weights.numel()} weights for a batch of {B} examples")
        if logits.device.type != "cuda":
            return torch_head(self.head, logits, labels, weights)
        if torch.is_grad_enabled() and logits.requires_grad:
            return _HeadFunction.apply(logits, labels, weights, self)
        return self._launch(logits, labels, weights, with_grad=False)[0]

    def _launch(self, logits, labels, weights, with_grad: bool):
        dev = logits.device
        st = self._state.get(dev)
        if st is None:
            st = self._state[dev] = _DeviceState(dev)
        B = logits.shape[0]
        C = self.n_out
        z = logits.detach().float().reshape(B, C).contiguous()
        y = labels.reshape(-1)
        if y.dtype not in _LABEL_CODES:
            y = y.long() if self.head == MULTI_CLASS else y.float()
        y = y.to(dev).contiguous()
        want = B if self.head != REGRESSION else B * C
        if y.numel() != want:
            raise ValueError(f"{y.numel()} labels for {B} examples of {C} logits")
        w = None if weights is None else weights.detach().to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        loss = torch.empty((), dtype=torch.float32, device=dev)
        grad = torch.empty_like(z) if with_grad else None
        rc = native.load().tfy_canned_head(z.data_ptr(), y.data_ptr(), _LABEL_CODES[y.dtype],
                                           w.data_ptr() if w is not None else None, B, C, self.head, loss.data_ptr(),
                                           grad.data_ptr() if grad is not None else None, st.flags.data_ptr(),
                                           st.scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        native.check(rc, "tfy_canned_head")
        if grad is not None:
            grad = grad.reshape(logits.shape).to(logits.dtype)
        return loss, grad

    def check(self) -> None:
        """Raise ``ValueError`` if a multi-class label outside ``[0, n_classes)`` reached the kernel since the last
        check (and clear the flag).  Called where the estimator already reads the loss on the host."""
        for st in self._state.values():
            if int(st.flags.item()) & BAD_LABEL:
                st.flags.zero_()
                raise ValueError(f"labels must be class ids in [0, {self.n_out}): a batch held a label outside it; "
                                 "its examples were left out of the loss and the gradient")
