"""The canned estimators' head: loss and logit gradient of the binary, multi-class, regression, multi-label, Poisson and
logistic heads, weighted or not.

Row ``i`` has logits ``z_i`` (``C`` values), label ``y_i`` and weight ``w_i`` (``w_i = 1`` without a weight column).
With ``c = 1`` for the binary and multi-class heads and ``c = C`` for every other head:

==============================  =========================================  ==========================================
head                            per-element loss ``l_ij``                  ``dl/dz_ij``
==============================  =========================================  ==========================================
binary (``C = 1``)              ``max(z,0) - z*y + log1p(exp(-|z|))``      ``sigmoid(z) - y``
multi-class (``C >= 2``)        ``logsumexp(z_i) - z_{i,y_i}`` (one/row)   ``softmax(z_i)_j - [j = y_i]``
regression (``C = d``)          ``(z_ij - y_ij)^2``                        ``2 (z_ij - y_ij)``
multi-label (``C >= 2``)        the binary element function                ``sigmoid(z) - y``
Poisson (``C = d``)             ``exp(z) - y*z``                           ``exp(z) - y``
Poisson, full loss              the same ``+ y log y - y + log(2 pi y)/2``  ``exp(z) - y``
                                when ``y > 1``
logistic (``C = 1``)            the binary element function                ``sigmoid(z) - y``
==============================  =========================================  ==========================================

The training loss is ``L = sum_i w_i sum_j l_ij / (B c)`` (TF2's ``SUM_OVER_BATCH_SIZE``; unweighted it is the mean of
``binary_cross_entropy_with_logits`` / ``cross_entropy`` / ``mse_loss`` / ``poisson_nll_loss(log_input=True)``) and
``dL/dz_ij = w_i dl_ij/dz_ij / (B c)``.  Binary and multi-label labels are used as the floats they are.  A multi-class
label outside ``[0, C)`` makes its row contribute nothing to the loss or the gradient (the row still counts in ``B``);
a Poisson label ``< 0`` or a logistic label outside ``[0, 1]`` (NaN included) does the same for its element (which
still counts in ``B c``).  Either sets a flag that :meth:`CannedHead.check` turns into a ``ValueError`` on the host;
on the CPU the call itself raises.  ``exp(z)`` is not clamped: above ``z ~ 88.7`` the Poisson loss is ``inf``, as TF's.

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
MULTI_LABEL, POISSON, POISSON_FULL, LOGISTIC = 3, 4, 5, 6
HEADS = (BINARY, MULTI_CLASS, REGRESSION, MULTI_LABEL, POISSON, POISSON_FULL, LOGISTIC)
BAD_LABEL = 1
_LABEL_CODES = {torch.float32: 0, torch.int32: 1, torch.int64: 2}
_NAMES = {BINARY: "binary", MULTI_CLASS: "multi-class", REGRESSION: "regression", MULTI_LABEL: "multi-label",
          POISSON: "Poisson", POISSON_FULL: "Poisson", LOGISTIC: "logistic"}
_LABEL_RULES = {POISSON: "labels must be counts >= 0", POISSON_FULL: "labels must be counts >= 0",
                LOGISTIC: "labels must be in [0, 1]"}


def _valid_labels(head: int, y: torch.Tensor) -> torch.Tensor:
    """Which float labels a Poisson (``y >= 0``) or logistic (``0 <= y <= 1``) head accepts; NaN never."""
    return (y >= 0) & (y <= 1) if head == LOGISTIC else y >= 0


def torch_element_losses(head: int, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """``l_ij`` of every element of an elementwise head (every head but multi-class) as torch ops: ``[B, C]``."""
    z = logits.float().reshape(logits.shape[0], -1)
    y = labels.float().reshape(z.shape)
    if head in (BINARY, MULTI_LABEL, LOGISTIC):
        return F.binary_cross_entropy_with_logits(z, y, reduction="none")
    if head in (POISSON, POISSON_FULL):
        return F.poisson_nll_loss(z, y, log_input=True, full=head == POISSON_FULL, reduction="none")
    return (z - y) ** 2


def torch_row_losses(head: int, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """``sum_j l_ij`` of every row as torch ops: ``[B]``."""
    z = logits.float()
    if head == BINARY:
        return F.binary_cross_entropy_with_logits(z.reshape(-1), labels.float().reshape(-1), reduction="none")
    if head == MULTI_CLASS:
        return F.cross_entropy(z, labels.long().reshape(-1), reduction="none")
    if head == REGRESSION:
        return ((z - labels.float().reshape(z.shape)) ** 2).sum(dim=1)
    return torch_element_losses(head, z, labels).sum(dim=1)


def torch_head(head: int, logits: torch.Tensor, labels: torch.Tensor, weights: Optional[torch.Tensor]) -> torch.Tensor:
    """The head's training loss as torch ops (the CPU path, and the statement the kernel is tested against).

    ``logits`` are ``[B, C]`` (``[B]`` or ``[B, 1]`` for the binary and logistic heads); ``labels`` hold ``B`` values
    (binary, multi-class, logistic) or ``B*C`` (regression, multi-label, Poisson); ``weights`` is ``None`` or ``[B]``.
    Unweighted, this is the torch mean (``binary_cross_entropy_with_logits`` / ``cross_entropy`` / ``mse_loss`` /
    ``poisson_nll_loss``) itself.  An invalid Poisson or logistic label raises ``ValueError``."""
    z = logits.float()
    if head in (POISSON, POISSON_FULL, LOGISTIC) and not bool(_valid_labels(head, labels.float()).all()):
        raise ValueError(f"{_LABEL_RULES[head]}: a batch held a label outside it")
    if weights is None:
        if head in (BINARY, LOGISTIC):
            return F.binary_cross_entropy_with_logits(z.reshape(-1), labels.float().reshape(-1))
        if head == MULTI_CLASS:
            return F.cross_entropy(z, labels.long().reshape(-1))
        if head == MULTI_LABEL:
            return F.binary_cross_entropy_with_logits(z, labels.float().reshape(z.shape))
        if head in (POISSON, POISSON_FULL):
            return F.poisson_nll_loss(z, labels.float().reshape(z.shape), log_input=True, full=head == POISSON_FULL)
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

    ``n_out`` is the number of logits per example: 1 for the binary and logistic heads, ``n_classes`` for the
    multi-class and multi-label heads and ``label_dimension`` for regression and Poisson."""

    def __init__(self, head: int, n_out: int):
        if head not in HEADS:
            raise ValueError(f"unknown head {head}")
        self.head = head
        self.n_out = int(n_out)
        self._state: Dict[torch.device, _DeviceState] = {}

    def __call__(self, labels: torch.Tensor, logits: torch.Tensor,
                 weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        B = logits.shape[0]
        if self.head not in (BINARY, MULTI_CLASS):
            want = [(B,), (B, 1)] if self.n_out == 1 and self.head != MULTI_LABEL else [(B, self.n_out)]
            if tuple(labels.shape) not in want:
                raise ValueError(f"{_NAMES[self.head]} labels must have shape {' or '.join(str(list(s)) for s in want)}, "
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
        want = B if self.head in (BINARY, MULTI_CLASS) else B * C
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
        """Raise ``ValueError`` if a label the head does not accept (a multi-class label outside ``[0, n_classes)``,
        a Poisson label ``< 0``, a logistic label outside ``[0, 1]``) reached the kernel since the last check (and
        clear the flag).  Called where the estimator already reads the loss on the host."""
        for st in self._state.values():
            if int(st.flags.item()) & BAD_LABEL:
                st.flags.zero_()
                rule = _LABEL_RULES.get(self.head) or f"labels must be class ids in [0, {self.n_out})"
                raise ValueError(f"{rule}: a batch held a label outside it; its examples were left out of the loss "
                                 "and the gradient")
