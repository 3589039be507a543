"""Fast path of the H100 train engine: explicit forward/backward out of fused kernels.

For ``Sequential`` models made of Conv2D(3x3, valid, stride 1) / MaxPooling2D(2x2) /
Dropout / Flatten / Dense layers with relu|linear activations and a sparse-categorical or categorical
(one-hot / soft targets, label smoothing) cross-entropy head, or a binary cross-entropy head (binary or multi-label,
label smoothing) -- the MNIST-CNN of the headline benchmark, the wine MLP -- the step does not go through autograd at
all:

* convolutions are wgmma implicit GEMMs (:mod:`ops/csrc/tfy_conv.cu`): conv2 forward with
  bias + ReLU + 2x2 max-pool + dropout in the epilogue, conv2 data / weight gradients whose dz
  operand is rebuilt in shared memory from the pooled gradient (un-pool + dropout + ReLU gate
  fused, db included), the first layer's forward and weight/bias gradient with im2col built in
  shared memory;
* the long-K Dense forward is the split-K wgmma GEMM (:mod:`ops/csrc/tfy_gemm.cu`);
* the classifier head runs forward AND backward in one kernel (:mod:`ops/csrc/tfy_nn.cu`);
* weight gradients are written straight into the flat gradient buffer consumed by the fused
  reduce-scatter / optimizer / all-gather kernel (no ``grad += g`` accumulation launches).

10 launches per MNIST-CNN step, all of them our kernels (no cuBLAS / cuDNN), against 53 for the autograd engine
(profiles/launches_*.csv).  Layers or shapes outside the kernels' envelope fall back to cuDNN / cuBLAS +
the element-wise fused kernels of ``tfy_nn.cu``; models outside the grammar use the autograd engine
(:class:`GraphTrainEngine`).
"""
from __future__ import annotations

import ctypes
import os
import types
from typing import List, Optional

import torch
import torch.nn.functional as F

from tf_yarn_b200.keras import layers as L
from tf_yarn_b200.keras.engine import GraphTrainEngine
from tf_yarn_b200.ops import gemm as _gemm  # noqa: F401  (declares tfy_gemm_bf16)
from tf_yarn_b200.ops import native

_vp, _i, _sz, _f, _u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float, ctypes.c_uint32
native.declare("tfy_conv3x3_c1_fwd", [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c1_fwd_tc", [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c1_wgrad", [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp])
native.declare("tfy_bias_act_drop_fwd", [_vp, _vp, _vp, _vp, _sz, _i, _i, _f, _u32, _vp, _vp])
native.declare("tfy_bias_act_drop_fwd_f32", [_vp, _vp, _vp, _vp, _sz, _i, _i, _f, _u32, _vp, _i, _vp])
native.declare("tfy_act_drop_bwd_bias", [_vp, _vp, _vp, _vp, _f, _sz, _i, _vp, _vp, _vp, _vp])
native.declare("tfy_bias_relu_pool_drop_fwd", [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _u32, _vp, _vp])
native.declare("tfy_pool_drop_relu_bwd", [_vp, _vp, _vp, _f, _i, _i, _i, _i, _vp, _vp, _vp, _vp])
native.declare("tfy_softmax_xent", [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp])
native.declare("tfy_softmax_xent_weighted", [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp])
native.declare("tfy_softmax_xent_soft", [_vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp])
native.declare("tfy_sigmoid_xent", [_vp, _vp, _vp, _f, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_pool_fwd", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f, _u32, _vp, _vp])
native.declare("tfy_conv3x3_c32_dgrad", [_vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_wgrad", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_wgrad_scratch_elems", [], restype=ctypes.c_size_t)
native.declare("tfy_conv3x3_c1_wgrad_tc", [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_dgrad_unpool", [_vp, _vp, _f, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_wgrad_unpool", [_vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_conv3x3_c32_wgrad_unpool_ov", [_vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp])
native.declare("tfy_conv3x3_c32_wgrad_unpool_deferred", [_vp, _vp, _vp, _f, _vp, _i, _i, _i, _vp, _vp, _vp])
native.declare("tfy_conv3x3_c32_dgrad_unpool_reduce", [_vp, _vp, _f, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp,
                                                       _vp])
native.declare("tfy_conv3x3_c32_wgrad_spare_ctas", [_i, _i, _i])
native.declare("tfy_conv3x3_c32_keep_scale", [_f, ctypes.POINTER(ctypes.c_float)])
native.declare("tfy_dense_bwd", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp])
native.declare("tfy_gemm_bf16_splitk_fused", [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _u32, _vp, _i,
                                              _vp])
native.declare("tfy_dense_head_scratch_elems", [_i, _i, _i], restype=ctypes.c_size_t)
native.declare("tfy_nn_max_partial_blocks", [], restype=ctypes.c_size_t)
native.declare("tfy_dense_head_fused", [_vp, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i,
                                        _i, _vp])
native.declare("tfy_dense_head_fused_weighted", [_vp, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                 _vp, _i, _i, _i, _vp, _vp, _vp])
native.declare("tfy_dense_head_fused_soft", [_vp, _vp, _vp, _vp, _f, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                             _i, _i, _i, _vp, _vp, _vp])
native.declare("tfy_dense_head_fused_binary", [_vp, _vp, _vp, _vp, _f, _i, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                               _vp, _vp, _i, _i, _i, _vp, _vp, _vp])

PARTIAL_BLOCKS = 592


def keep_scale(lib, rate: float) -> float:
    """Scale of the kept elements of tfy_conv3x3_c32_pool_fwd's dropout at ``rate`` (the fp32 value it applies)."""
    out = ctypes.c_float(0.0)
    rc = lib.tfy_conv3x3_c32_keep_scale(float(rate), ctypes.byref(out))
    if rc != 0:
        raise RuntimeError(f"tfy_conv3x3_c32_keep_scale failed: {rc}")
    return out.value


class _Stage:
    """One fused stage of the plan."""

    def __init__(self, kind: str, **kw):
        self.kind = kind
        self.__dict__.update(kw)


def head_loss(loss):
    """``(categorical, label_smoothing, head activation)`` of a loss the fused head computes, or None.  The head computes
    softmax + cross-entropy from logits: either the loss takes logits and the last layer is linear, or the last layer
    is a softmax and the loss takes probabilities.  Sparse losses read int64 labels [B], categorical ones fp32 targets
    [B, C]."""
    from tf_yarn_b200.keras import losses as kl
    if isinstance(loss, (kl.SparseCategoricalCrossentropy, kl.CategoricalCrossentropy)):
        categorical = isinstance(loss, kl.CategoricalCrossentropy)
        return (categorical, loss.label_smoothing if categorical else 0.0,
                "linear" if loss.from_logits else "softmax")
    if isinstance(loss, str) and loss in ("sparse_categorical_crossentropy", "categorical_crossentropy"):
        return loss == "categorical_crossentropy", 0.0, "softmax"
    return None


def binary_head_loss(loss):
    """``(label_smoothing, head activation)`` of a binary cross-entropy loss the fused head computes, or None.  The head
    computes sigmoid cross-entropy from logits: either the loss takes logits and the last layer is linear, or the last
    layer is a sigmoid and the loss takes probabilities.  It reads fp32 targets [B, C] ([B] or [B, 1] when C = 1)."""
    from tf_yarn_b200.keras import losses as kl
    if isinstance(loss, kl.BinaryCrossentropy):
        return loss.label_smoothing, "linear" if loss.from_logits else "sigmoid"
    if isinstance(loss, str) and loss == "binary_crossentropy":
        return 0.0, "sigmoid"
    return None


def label_dtype(loss) -> Optional[torch.dtype]:
    """Dtype ``fit`` casts array labels to once for a softmax head's ``loss`` (None: no cast).  Binary targets are not
    cast there: whatever their dtype, the staging copy converts them to the fp32 the binary head reads."""
    head = head_loss(loss)
    if head is None:
        return None
    return torch.float32 if head[0] else torch.int64


def build_plan(model) -> Optional[List[_Stage]]:
    """Pattern-match the layer list; None if the model is outside the fast-path grammar."""
    head, binary = head_loss(model.loss), binary_head_loss(model.loss)
    # the head kernel counts the hits of the accuracy that goes with the loss; one weighted accuracy at most
    if head is not None:
        categorical, _, want_head_activation = head
        accuracies = ("accuracy", "acc", "categorical_accuracy" if categorical else "sparse_categorical_accuracy")
    elif binary is not None:
        _, want_head_activation = binary
        accuracies = ("accuracy", "acc", "binary_accuracy")
    else:
        return None
    for m in model._metrics_spec:
        if m not in accuracies:
            return None
    weighted = getattr(model, "_weighted_metrics_spec", [])
    if len(weighted) > 1 or any(m not in accuracies for m in weighted):
        return None
    layers = [ly for ly in model.layers if not isinstance(ly, L.InputLayer)]
    plan: List[_Stage] = []
    i, n = 0, len(layers)
    seen_flatten = False
    while i < n:
        ly = layers[i]
        if isinstance(ly, L.Conv2D) and not seen_flatten:
            if ly.kernel_size != (3, 3) or ly.strides != (1, 1) or ly.padding != "valid" or not ly.use_bias \
                    or ly.activation_name not in ("relu", "linear") or ly.filters % 8:
                return None
            st = _Stage("conv", layer=ly, relu=ly.activation_name == "relu", pool=False, drop=0.0)
            j = i + 1
            if j < n and type(layers[j]) is L.MaxPooling2D:      # (AveragePooling2D SUBCLASSES it: never fuse that as max)
                mp = layers[j]
                h, w, _ = ly.output_shape_
                if mp.pool_size != (2, 2) or mp.strides != (2, 2) or mp.padding != "valid" or not st.relu \
                        or h % 2 or w % 2:
                    return None
                st.pool = True
                j += 1
            if j < n and isinstance(layers[j], L.Dropout):
                st.drop = layers[j].rate
                j += 1
            plan.append(st)
            i = j
        elif isinstance(ly, L.Flatten):
            seen_flatten = True
            plan.append(_Stage("flatten"))
            i += 1
        elif isinstance(ly, L.Dense):
            last = i + 1 >= n
            if not ly.use_bias or ly.activation_name not in (("relu", "linear") if not last
                                                             else (want_head_activation,)):
                return None
            if last:
                if ly.units > 1024:
                    return None
                plan.append(_Stage("head", layer=ly))
                i += 1
            else:
                if ly.units % 8 or ly.input_shape_[-1] % 8:
                    return None
                st = _Stage("dense", layer=ly, relu=ly.activation_name == "relu", drop=0.0)
                j = i + 1
                if j < n and isinstance(layers[j], L.Dropout):
                    st.drop = layers[j].rate
                    j += 1
                plan.append(st)
                i = j
        else:
            return None
    if not plan or plan[-1].kind != "head":
        return None
    kinds = [s.kind for s in plan]
    if "conv" in kinds and "flatten" not in kinds:
        return None
    if len(model.layers[0].input_shape_ or ()) not in (1, 3):
        return None
    return plan


class FastSequentialEngine(GraphTrainEngine):
    """GraphTrainEngine whose step body is the explicit fused-kernel plan."""

    def __init__(self, model, plan: List[_Stage], *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.plan = plan
        self.lib = native.load()
        # every gradient element is overwritten by the plan's kernels each step (no accumulation), so the
        # fused optimizer step does not have to clear the gradient buffer behind itself
        self.fused.zero_grads = False
        dev = self.device
        width = 8
        for st in plan:
            if st.kind == "conv":
                width = max(width, st.layer.filters, 9 * st.layer.filters)
            elif st.kind == "dense":
                width = max(width, st.layer.units)
        # one row of `width` floats per CTA of the bias / weight-gradient reductions (their launchers refuse a grid
        # of more than tfy_nn_max_partial_blocks() CTAs)
        if int(self.lib.tfy_nn_max_partial_blocks()) != PARTIAL_BLOCKS:
            raise RuntimeError("tfy_nn.cu and fastpath.py disagree on the number of partial rows")
        self._partial = torch.zeros(PARTIAL_BLOCKS * width, dtype=torch.float32, device=dev)
        self._counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self._stats = torch.zeros(4, dtype=torch.float32, device=dev)     # hits, rows (, sum w*hit, sum w: weighted)
        self._seed = int(torch.initial_seed() & 0x7fffffff)
        self._hp = self.fused.hyper.data_ptr()
        self._k = 0
        self._acc32 = {}
        self._resolved_b = None          # batch size the plan's kernels were chosen for (_resolve)
        self._overlap = False
        self._ov_gmid = 0                # first shard group the weight-gradient kernel updates (0: none)
        self._warned = set()
        self._conv_sync = torch.zeros(1024, dtype=torch.int32, device=dev)     # grid barrier of the wgrad kernel
        self._c1_acc = torch.zeros(160 * 320, dtype=torch.float32, device=dev)   # first-layer dW/db per-CTA partials
        self._c1_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        # what the head reads: int64 labels [B] (sparse loss), or fp32 targets [B, C] and the label smoothing
        # (categorical loss: self._ls is not None; binary cross-entropy: self._binary = (label smoothing, whether the
        # model's output is the sigmoid)).  The staging slots hold labels of this dtype, so a batch of another dtype is
        # converted by the staging copy instead of being misread.
        head, binary = head_loss(model.loss), binary_head_loss(model.loss)
        categorical, ls, _ = head if head is not None else (False, 0.0, None)
        self._ls = float(ls) if categorical else None
        self._binary = (float(binary[0]), binary[1] == "sigmoid") if binary is not None else None
        self._y_dtype = torch.float32 if (categorical or binary is not None) else torch.int64

    # ------------------------------------------------------------------ helpers
    def _s(self):
        return torch.cuda.current_stream().cuda_stream

    def _chk(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed: {rc}")
        self._k += 1

    def _wb(self, layer):
        mod = layer.module
        return mod.weight, mod.bias

    @staticmethod
    def _bf16(t: torch.Tensor) -> torch.Tensor:
        return t if (t.dtype == torch.bfloat16 and t.is_contiguous()) else t.to(torch.bfloat16).contiguous()

    @staticmethod
    def _split_k(M: int, N: int, K: int, per_cta: int = 6) -> int:
        """Split factor of the wgmma GEMM for skinny-output / long-K dense layers (1 = use cuBLAS); ``per_cta``
        k-tiles per CTA (6 == the TMA ring depth)."""
        tiles = ((M + 127) // 128) * ((N + 127) // 128)
        k_tiles = (K + 63) // 64
        if K % 8 or tiles > 8 or k_tiles < 32:
            return 1
        return max(1, min(k_tiles // per_cta, 144 // tiles))

    @staticmethod
    def _tc_conv(st, B: int) -> bool:
        """True when the stage's shape is served by the wgmma implicit-GEMM kernels of ops/csrc/tfy_conv.cu."""
        ly = st.layer
        H, W, Cin = ly.input_shape_
        return (Cin == 32 and ly.filters == 64 and st.pool and st.relu and (H - 2) % 8 == 0 and (W - 2) % 8 == 0
                and B % 2 == 0)

    def _conv_drop_scale(self, st, tc: bool) -> float:
        """Scale of the kept gradients in the backward of conv stage ``st``'s dropout: the one its forward applied.
        The wgmma forward (``tc``) quantises the rate to 1/256 and scales by 256 / (256 - thr)
        (tfy_conv3x3_c32_keep_scale); the general pool kernel scales by 1 / (1 - rate)."""
        if tc:
            return keep_scale(self.lib, st.drop)
        return 1.0 / (1.0 - st.drop) if st.drop > 0 else 1.0

    def _warn_once(self, key: str, msg: str) -> None:
        if key not in self._warned:
            self._warned.add(key)
            import logging
            logging.getLogger(__name__).warning(msg)

    def _overlap_desc(self, li: int, B: int, H: int, W: int, groups_override: Optional[str]):
        """Fused-step descriptor for the communication CTAs of conv stage ``li``'s weight-gradient kernel, or None.

        Overlapped: shard-relative groups [g_mid, S/8) of EVERY rank (balanced), where g_mid*8 is at least the
        flat offset of the first parameter of the layers after ``li`` (their gradients are final by now; rank 0's
        shard starts with the still-pending convolution parameters).  The size of the overlapped part is bounded
        by what ``n_cta`` SMs can move while the weight gradient runs (TFY_OVERLAP_GROUPS overrides)."""
        fused = self.fused
        if fused.zero_grads or fused.param_dtype != torch.bfloat16 or fused.grad_dtype != torch.bfloat16:
            return None
        if self.accum_steps is not None:             # the overlap role reads the bf16 gradients, not the accumulator
            return None
        if fused.spec.kind in ("rmsprop", "adamax", "nadam"):   # no overlap role: the trailing step updates everything
            return None
        n_cta = int(self.lib.tfy_conv3x3_c32_wgrad_spare_ctas(B, H, W))
        later = [st for st in self.plan[li + 1:] if st.kind in ("conv", "dense", "head")]
        if n_cta <= 0 or not later:
            return None
        ids = [id(p) for p in self.params]
        first_later = later[0].layer.module.weight
        if id(first_later) not in ids:
            return None
        e_split = int(fused.offsets[ids.index(id(first_later))])
        groups = fused.shard_n // 8
        g_split = (e_split + 7) // 8
        if g_split >= groups:
            return None                              # rank 0's shard is all pending parameters: nothing balanced to take
        budget = int(groups_override) if groups_override is not None else 2000 * n_cta
        g_mid = max(g_split, groups - budget)
        if groups - g_mid < 64:
            return None
        self._ov_gmid = g_mid
        return fused.overlap_step(g_mid, groups, n_cta)

    def _host_loss_ptr(self):
        """Pinned scalar of the slot being captured: the head kernel stores the loss there directly (UVA), so the
        captured step needs no D2H copy node."""
        slot = getattr(self, "_capture_slot", None)
        if slot is None or not getattr(self, "_loss_host", None):
            return None
        self._loss_in_host[slot] = True
        return self._loss_host[slot].data_ptr()

    def _scratch(self, key, numel: int, dtype=torch.float32) -> torch.Tensor:
        """Engine-owned scratch buffer ``key`` of at least ``numel`` elements, zeroed when (re)allocated."""
        if key not in self._acc32 or self._acc32[key].numel() < numel:
            self._acc32[key] = torch.zeros(numel, dtype=dtype, device=self.device)
        return self._acc32[key]

    def pop_metrics(self):
        self.stream.synchronize()
        st = self._stats.cpu()
        self._stats.zero_()
        out = {}
        if self.metric_fns:
            out[self.metric_fns[0][0]] = float(st[0] / st[1].clamp_min(1))
        if self.weighted_metric_fns:
            if self._wmode == (False, False):        # every weight is 1
                out[self.weighted_metric_fns[0][0]] = float(st[0] / st[1].clamp_min(1))
            else:
                out[self.weighted_metric_fns[0][0]] = float(st[2] / st[3]) if float(st[3]) != 0.0 else 0.0
        return out

    def _stats_ptr(self):
        return self._stats.data_ptr() if (self.metric_fns or self.weighted_metric_fns) else None

    def _weight_ptrs(self, sw):
        """(sample weights, class-weight table, stream) arguments of the weighted head kernels."""
        return (sw.data_ptr() if sw is not None else None, self._cw.data_ptr() if self._wmode[0] else None,
                self._s())

    def _head_targets(self, y: torch.Tensor) -> torch.Tensor:
        """``y`` in the dtype the head reads; a categorical target must be ``[B, C]``, a binary one ``[B, C]``, or
        ``[B]`` when C = 1."""
        C = self.plan[-1].layer.units
        if self._binary is not None:
            if not ((y.dim() == 2 and y.shape[-1] == C) or (C == 1 and y.dim() == 1)):
                want = "(batch,) or (batch, 1)" if C == 1 else f"(batch, {C})"
                raise ValueError(f"binary targets of shape {tuple(y.shape)} do not match the model's output "
                                 f"(batch, {C}): pass 0/1 or soft targets of shape {want}")
        if self._ls is not None:
            if y.dim() != 2 or y.shape[-1] != C:
                raise ValueError(f"categorical targets of shape {tuple(y.shape)} do not match the model's output "
                                 f"(batch, {C}): pass one-hot or soft targets of shape (batch, {C}), or class indices "
                                 "with SparseCategoricalCrossentropy")
        return y if y.dtype == self._y_dtype else y.to(self._y_dtype)

    def _capture(self, x, y, w=None) -> None:
        self._resolve(x.shape[0])
        super()._capture(x, self._head_targets(y), w)
        with torch.cuda.stream(self.stream):
            self._stats.zero_()          # warm-up steps must not count in the epoch metrics
        self.stream.synchronize()

    # ------------------------------------------------------------------ kernel choice
    def _resolve(self, B: int) -> None:
        """Choose every stage's kernels for batch size ``B`` and allocate their scratch buffers.  Runs at capture and
        whenever a step's batch size differs from the last one resolved; the A/B switches are read here, so a change
        to one takes effect at the next capture or batch-size change."""
        env = os.environ.get
        tc_conv = env("TFY_NO_TC_CONV") != "1"         # off: cuDNN + the general pool kernels instead
        unpool_fusion = env("TFY_NO_UNPOOL_FUSION") != "1"
        tc_dense_bwd = env("TFY_NO_TC_DENSE_BWD") != "1"
        fused_head = env("TFY_NO_FUSED_HEAD") != "1"
        splitk_fuse = env("TFY_SPLITK_FUSE") == "1"
        splitk_tiles = int(env("TFY_SPLITK_TILES", "6"))
        # Gradient-exchange overlap (opt-in, TFY_OVERLAP=1): parameters whose gradients are final before the
        # convolution weight-gradient kernel starts (every layer AFTER that convolution: for the MNIST-CNN the two
        # Dense layers, 98 % of the bytes) can be reduce-scattered / updated / all-gathered by COMMUNICATION CTAs
        # inside that kernel (ops/csrc/tfy_fused_step.cuh: tfy_overlap_role) on the 4 SMs its patch grid leaves
        # idle, the trailing fused-step launch handling the rest.  Numerically equivalent (GPU test); off by default
        # because the cost of the trailing launch is the LATENCY chain signal -> in-switch reduce -> store/ack ->
        # signal, which a smaller range does not shorten.
        self._overlap = env("TFY_OVERLAP", "0") == "1"
        overlap_groups = env("TFY_OVERLAP_GROUPS")
        lib, plan = self.lib, self.plan
        for li, st in enumerate(plan):
            prev = plan[li - 1] if li > 0 else None
            st.li, st.first = li, li == 0
            st.seed = (self._seed * 2654435761 + li * 97) & 0x7fffffff
            st.gated = False         # conv: the next stage's data gradient applies this stage's ReLU gate
            if st.kind == "conv":
                ly = st.layer
                H, W, Cin = ly.input_shape_
                O = ly.filters
                st.tc = tc_conv and self._tc_conv(st, B)
                if st.tc:
                    st.fwd = "c32_pool_tc"
                elif Cin == 1 and st.relu and not st.pool:
                    st.fwd = "c1_tc" if O == 32 and tc_conv else "c1"
                else:
                    st.fwd = "cudnn"
                    self._warn_once(f"conv_fwd:{li}", f"Conv2D layer {li} ({Cin} -> {O} channels, {H}x{W}, batch {B}) is "
                                    "outside the wgmma convolution kernels' envelope (C_in 32 / C_out 64 with ReLU + 2x2 "
                                    "pool, or C_in 1): forward and backward use cuDNN")
                st.scale = self._conv_drop_scale(st, st.tc)
                if st.tc:
                    st.bwd = "unpool" if unpool_fusion else "tc"
                elif Cin == 1:
                    if not st.first:
                        raise RuntimeError("C_in=1 convolution must be the first layer")
                    st.bwd = "c1"
                else:
                    st.bwd = "cudnn"
                # the tensor-core data gradient applies the producer's ReLU gate when its output IS our input
                st.fold = (st.tc and prev is not None and prev.kind == "conv" and prev.relu and not prev.pool
                           and prev.drop == 0)
                if st.fold:
                    prev.gated = True
                    if prev.first and prev.fwd == "c1_tc":
                        prev.bwd = "c1_tc"      # first layer: dW and db in ONE tensor-core kernel
                if st.tc:                       # per-CTA fp32 partial tiles (L2 resident)
                    self._scratch("wgrad_scratch", int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()))
                st.overlap = None
            elif st.kind == "dense":
                ly = st.layer
                K, N = ly.input_shape_[-1], ly.units
                w, _ = self._wb(ly)
                st.scale = 1.0 / (1.0 - st.drop) if st.drop > 0 else 1.0
                st.split = self._split_k(B, N, K, splitk_tiles)
                tiles = ((B + 127) // 128) * ((N + 127) // 128)
                co_resident = tiles * st.split <= torch.cuda.get_device_properties(self.device).multi_processor_count
                st.splitk_fused = st.split > 1 and co_resident and splitk_fuse
                if st.split > 1:
                    st.slabs = int(lib.tfy_gemm_bf16_splitk_slabs(K, st.split))
                    self._scratch(li, st.slabs * B * N)
                    if st.splitk_fused:
                        self._scratch(("splitk_cnt", li), 2 * tiles, torch.int32)
                else:
                    self._warn_once(f"dense_fwd:{li}", f"Dense layer {li} ({K} -> {N}, batch {B}) is outside the "
                                    "split-K wgmma GEMM's envelope (long K, at most 8 output tiles): forward uses cuBLAS")
                st.tc_bwd = N % 8 == 0 and K % 8 == 0 and w.is_contiguous() and w.grad.is_contiguous() and tc_dense_bwd
                if not st.tc_bwd:
                    self._warn_once(f"dense_bwd:{li}", f"Dense layer {li} ({K} -> {N}, batch {B}) is outside "
                                    "the wgmma dense-backward kernel's envelope: cuBLAS computes dW / dx")
                st.head_gated = False   # the fused head produces this layer's gated gradient and db
            elif st.kind == "head":
                ly = st.layer
                K, C = ly.input_shape_[-1], ly.units
                st.fused = (prev is not None and prev.kind == "dense" and K in (128, 256, 512) and C <= 16
                            and fused_head)
                if st.fused:
                    prev.head_gated = True
                    self._scratch("head_scratch", int(lib.tfy_dense_head_scratch_elems(K, C, B)))   # a slab per 16 rows
                    self._scratch("head_counter", 1, torch.int32)
                else:
                    self._warn_once(f"head:{li}", f"classifier head {li} ({K} -> {C}, batch {B}) is outside "
                                    "the fused head kernel's envelope (K in 128/256/512, at most 16 classes, Dense "
                                    "predecessor): logits and gradients use cuBLAS")
        self._ov_gmid = 0
        if self._overlap:               # the last un-pool-fused weight gradient the descriptor fits
            for st in reversed(plan):
                if st.kind == "conv" and st.bwd == "unpool":
                    H, W, _ = st.layer.input_shape_
                    st.overlap = self._overlap_desc(st.li, B, H, W, overlap_groups)
                    if st.overlap is not None:
                        break
        self._resolved_b = B

    # ------------------------------------------------------------------ the step
    @torch.no_grad()
    def _forward_backward(self, x, y, sw=None, update: bool = True) -> None:
        if x.shape[0] != self._resolved_b:
            self._resolve(x.shape[0])
        self._k = 0
        saved = []
        cur = x                    # NHWC for images, [B, F] for vectors
        for st in self.plan:
            sv = types.SimpleNamespace()
            if st.kind == "head":
                self._head_fwd(st, sv, cur, saved[-1] if saved else None, y, sw)
            else:
                cur = getattr(self, f"_{st.kind}_fwd")(st, sv, cur)
            saved.append(sv)
        grad = None
        for st, sv in zip(reversed(self.plan), reversed(saved)):
            grad = getattr(self, f"_{st.kind}_bwd")(st, sv, grad)
        if self._ov_gmid:
            # the communication CTAs of the weight-gradient kernel already handled groups [g_mid, end) of every shard
            self.fused.step(shard_groups=(0, self._ov_gmid), advance=True)
            n_step = 1
        else:
            n_step = self._apply_gradients(update)
        # our kernels launched per step (library GEMMs excluded)
        if update:
            self._launches_per_step = self._k + n_step
        else:
            self._launches_per_accum_step = self._k + n_step

    def _conv_fwd(self, st, sv, x):
        lib, s, bf16 = self.lib, self._s(), torch.bfloat16
        w, b = self._wb(st.layer)
        B = x.shape[0]
        H, W, Cin = st.layer.input_shape_
        O, OH, OW = st.layer.filters, H - 2, W - 2
        sv.x = self._bf16(x) if st.fwd == "c32_pool_tc" else x
        if st.fwd == "c32_pool_tc":
            # wgmma implicit GEMM; bias + ReLU + 2x2 max-pool + dropout in the epilogue
            p = torch.empty((B, OH // 2, OW // 2, O), dtype=bf16, device=x.device)
            sv.code = torch.empty((B, OH // 2, OW // 2, O), dtype=torch.uint8, device=x.device)
            self._chk(lib.tfy_conv3x3_c32_pool_fwd(sv.x.data_ptr(), w.data_ptr(), b.data_ptr(), p.data_ptr(),
                                                   sv.code.data_ptr(), B, H, W, float(st.drop), st.seed, self._hp, s),
                      "conv3x3_c32_pool_fwd")
            return p
        if st.fwd == "cudnn":
            z = F.conv2d(self._bf16(x).permute(0, 3, 1, 2), w).permute(0, 2, 3, 1).contiguous()   # NCHW over NHWC
        else:
            # direct kernel: conv + bias + relu in one launch
            z = torch.empty((B, OH, OW, O), dtype=bf16, device=x.device)
            if st.fwd == "c1_tc":
                self._chk(lib.tfy_conv3x3_c1_fwd_tc(x.data_ptr(), int(x.dtype == torch.float32), w.data_ptr(),
                                                    b.data_ptr(), z.data_ptr(), B, H, W, s), "conv3x3_c1_fwd_tc")
            else:
                self._chk(lib.tfy_conv3x3_c1_fwd(x.data_ptr(), int(x.dtype == torch.float32), w.data_ptr(),
                                                 b.data_ptr(), z.data_ptr(), B, H, W, O, s), "conv3x3_c1_fwd")
        if st.pool:
            p = torch.empty((B, OH // 2, OW // 2, O), dtype=bf16, device=x.device)
            sv.code = torch.empty((B, OH // 2, OW // 2, O), dtype=torch.uint8, device=x.device)
            self._chk(lib.tfy_bias_relu_pool_drop_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), sv.code.data_ptr(),
                                                      B, OH, OW, O, float(st.drop), st.seed, self._hp, s),
                      "bias_relu_pool_drop_fwd")
            return p
        sv.z = z
        sv.mask = torch.empty((B, OH, OW, O), dtype=torch.uint8, device=x.device) if st.drop > 0 else None
        if st.fwd == "cudnn" or sv.mask is not None:     # (the direct kernels applied bias + ReLU already)
            self._chk(lib.tfy_bias_act_drop_fwd(z.data_ptr(), b.data_ptr() if st.fwd == "cudnn" else None, z.data_ptr(),
                                                sv.mask.data_ptr() if sv.mask is not None else None, B * OH * OW, O,
                                                int(st.relu), float(st.drop), st.seed, self._hp, s), "bias_act_drop_fwd")
        return z

    def _conv_bwd(self, st, sv, grad):
        lib, s = self.lib, self._s()
        w, b = self._wb(st.layer)
        B = grad.shape[0]
        H, W, Cin = st.layer.input_shape_
        O, OH, OW = st.layer.filters, H - 2, W - 2
        x_f32 = int(sv.x.dtype == torch.float32)
        gate = sv.x.data_ptr() if st.fold else None      # the producer's ReLU gate, applied by the tensor-core dgrad
        if st.bwd == "c1_tc":
            self._chk(lib.tfy_conv3x3_c1_wgrad_tc(sv.x.data_ptr(), x_f32, grad.data_ptr(), self._c1_acc.data_ptr(),
                                                  self._c1_cnt.data_ptr(), w.grad.data_ptr(), b.grad.data_ptr(), B, H,
                                                  W, s), "conv3x3_c1_wgrad_tc")
            return None
        if st.bwd == "unpool":
            # pool/dropout/ReLU backward fused into the operand producers of wgrad and dgrad: the 4x larger dz tensor
            # is never written; db comes out of the wgrad kernel.  When the dgrad launch follows, the wgrad CTAs only
            # store their fp32 partials (no grid barrier) and the dgrad kernel reduces them into dW / db behind its
            # main loop: the same bits either way.
            part = self._acc32["wgrad_scratch"]
            ovp = ctypes.byref(st.overlap) if st.overlap is not None else None
            if st.first:
                self._chk(lib.tfy_conv3x3_c32_wgrad_unpool_ov(
                    sv.x.data_ptr(), grad.data_ptr(), sv.code.data_ptr(), st.scale, part.data_ptr(), w.grad.data_ptr(),
                    b.grad.data_ptr(), self._conv_sync.data_ptr(), B, H, W, ovp, s), "conv3x3_c32_wgrad_unpool")
                return None
            n_part = ctypes.c_int(0)
            dx = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=grad.device)
            self._chk(lib.tfy_conv3x3_c32_wgrad_unpool_deferred(
                sv.x.data_ptr(), grad.data_ptr(), sv.code.data_ptr(), st.scale, part.data_ptr(), B, H, W, ovp,
                ctypes.byref(n_part), s), "conv3x3_c32_wgrad_unpool_deferred")
            self._chk(lib.tfy_conv3x3_c32_dgrad_unpool_reduce(
                grad.data_ptr(), sv.code.data_ptr(), st.scale, w.data_ptr(), gate, dx.data_ptr(), B, H, W,
                part.data_ptr(), n_part.value, w.grad.data_ptr(), b.grad.data_ptr(), s),
                "conv3x3_c32_dgrad_unpool_reduce")
            return dx
        if st.pool:
            dz = torch.empty((B, OH, OW, O), dtype=torch.bfloat16, device=grad.device)
            self._chk(lib.tfy_pool_drop_relu_bwd(grad.data_ptr(), sv.code.data_ptr(), dz.data_ptr(), st.scale, B, OH,
                                                 OW, O, self._partial.data_ptr(), b.grad.data_ptr(),
                                                 self._counter.data_ptr(), s), "pool_drop_relu_bwd")
        else:
            dz = grad
            relu_gate = sv.z.data_ptr() if (st.relu and sv.mask is None and not st.gated) else None
            self._chk(lib.tfy_act_drop_bwd_bias(dz.data_ptr(), sv.mask.data_ptr() if sv.mask is not None else None,
                                                relu_gate, dz.data_ptr(), st.scale, B * OH * OW, O,
                                                self._partial.data_ptr(), b.grad.data_ptr(), self._counter.data_ptr(),
                                                s), "act_drop_bwd_bias")
        if st.bwd == "c1":
            self._chk(lib.tfy_conv3x3_c1_wgrad(sv.x.data_ptr(), x_f32, dz.data_ptr(), self._partial.data_ptr(),
                                               w.grad.data_ptr(), self._counter.data_ptr(), B, H, W, O, s),
                      "conv3x3_c1_wgrad")
            return None
        if st.bwd == "tc":
            self._chk(lib.tfy_conv3x3_c32_wgrad(sv.x.data_ptr(), dz.data_ptr(), self._acc32["wgrad_scratch"].data_ptr(),
                                                w.grad.data_ptr(), self._conv_sync.data_ptr(), B, H, W, s),
                      "conv3x3_c32_wgrad")
            if st.first:
                return None
            dx = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=grad.device)
            self._chk(lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), gate, dx.data_ptr(), B, H, W, s),
                      "conv3x3_c32_dgrad")
            return dx
        gx, dw, _ = torch.ops.aten.convolution_backward(
            dz.permute(0, 3, 1, 2), self._bf16(sv.x).permute(0, 3, 1, 2), w, None, [1, 1], [0, 0], [1, 1], False,
            [0, 0], 1, [not st.first, True, False])
        w.grad.copy_(dw)
        return None if st.first else gx.permute(0, 2, 3, 1).contiguous()

    def _flatten_fwd(self, st, sv, x):
        sv.shape = x.shape
        return x.reshape(x.shape[0], -1)

    def _flatten_bwd(self, st, sv, grad):
        return grad.reshape(sv.shape) if grad is not None else None

    def _dense_fwd(self, st, sv, x):
        lib, s, ly = self.lib, self._s(), st.layer
        w, b = self._wb(ly)
        sv.x = xin = self._bf16(x)
        (B, K), N = xin.shape, ly.units
        sv.mask = torch.empty((B, N), dtype=torch.uint8, device=x.device) if (st.drop > 0 or st.relu) else None
        mask = sv.mask.data_ptr() if sv.mask is not None else None
        if st.split == 1:
            z = torch.mm(xin, w.t())
            self._chk(lib.tfy_bias_act_drop_fwd(z.data_ptr(), b.data_ptr(), z.data_ptr(), mask, B, N, int(st.relu),
                                                float(st.drop), st.seed, self._hp, s), "bias_act_drop_fwd")
            return z
        # skinny GEMM with a long K (e.g. 128 x 128 x 9216): split K over ~48 CTAs of the wgmma kernel; each K-slice
        # stores its fp32 partial in its own slab and the epilogue sums the slabs in slice order
        acc = self._acc32[st.li]
        z = torch.empty((B, N), dtype=torch.bfloat16, device=x.device)
        if st.splitk_fused:
            # ONE launch (opt-in): the K-slice CTAs of a tile meet on a counter, then each applies bias + ReLU +
            # dropout to 1/split of the tile (summing the slabs in slice order) and writes the bf16 activations and
            # the gate mask.  (The slices spin on each other: the grid must be co-resident.)  Off by default: the
            # fence + counter + spin can cost more than the short second kernel of the same CUDA graph it removes.
            self._chk(lib.tfy_gemm_bf16_splitk_fused(
                xin.data_ptr(), w.data_ptr(), acc.data_ptr(), self._acc32[("splitk_cnt", st.li)].data_ptr(),
                b.data_ptr(), z.data_ptr(), mask, B, N, K, xin.stride(0), w.stride(0), int(st.relu), float(st.drop),
                st.seed, self._hp, st.split, s), "gemm_bf16_splitk_fused")
        else:
            self._chk(lib.tfy_gemm_bf16(xin.data_ptr(), w.data_ptr(), None, acc.data_ptr(), None, B, N, K,
                                        xin.stride(0), w.stride(0), N, 0, st.split, s), "gemm_bf16(split-K)")
            self._chk(lib.tfy_bias_act_drop_fwd_f32(acc.data_ptr(), b.data_ptr(), z.data_ptr(), mask, B, N,
                                                    int(st.relu), float(st.drop), st.seed, self._hp, st.slabs, s),
                      "bias_act_drop_fwd_f32")
        return z

    def _dense_bwd(self, st, sv, grad):
        lib, s = self.lib, self._s()
        w, b = self._wb(st.layer)
        (B, I), N = sv.x.shape, st.layer.units
        if not st.head_gated:
            self._chk(lib.tfy_act_drop_bwd_bias(grad.data_ptr(), sv.mask.data_ptr() if sv.mask is not None else None,
                                                None, grad.data_ptr(), st.scale, B, N, self._partial.data_ptr(),
                                                b.grad.data_ptr(), self._counter.data_ptr(), s), "act_drop_bwd_bias")
        if not st.tc_bwd:
            torch.mm(grad.t(), sv.x, out=w.grad)
            return None if st.first else torch.mm(grad, w)
        # dW = dh^T x (straight into the flat gradient buffer) and dx = dh W in ONE wgmma kernel
        dx = None if st.first else torch.empty((B, I), dtype=torch.bfloat16, device=grad.device)
        self._chk(lib.tfy_dense_bwd(grad.data_ptr(), sv.x.data_ptr(), w.data_ptr(), w.grad.data_ptr(),
                                    dx.data_ptr() if dx is not None else None, B, N, I, s), "dense_bwd")
        return dx

    def _head_fwd(self, st, sv, x, below, y, sw):
        lib, s = self.lib, self._s()
        w, b = self._wb(st.layer)
        xin = self._bf16(x)
        (B, K), C = xin.shape, st.layer.units
        if st.fused:
            # one launch: logits, loss, dlogits, dW2, db2 and the gradient entering the previous Dense layer (its
            # ReLU / dropout gate and bias gradient included)
            prev = self.plan[st.li - 1]
            _, pb = self._wb(prev.layer)
            sv.dh = torch.empty((B, K), dtype=torch.bfloat16, device=x.device)
            rest = (below.mask.data_ptr() if below.mask is not None else None, prev.scale, self._loss.data_ptr(),
                    self._host_loss_ptr(), self._stats_ptr(), w.grad.data_ptr(), b.grad.data_ptr(), sv.dh.data_ptr(),
                    pb.grad.data_ptr(), self._acc32["head_scratch"].data_ptr(), self._acc32["head_counter"].data_ptr(),
                    B, K, C)
            args = (xin.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr()) + rest
            if self._binary is not None:
                # binary cross-entropy: fp32 targets, the label smoothing and whether the model's output is the sigmoid
                self._chk(lib.tfy_dense_head_fused_binary(*args[:4], self._binary[0], int(self._binary[1]), *rest,
                                                          *self._weight_ptrs(sw)), "dense_head_fused_binary")
            elif self._ls is not None:
                # categorical loss: fp32 targets [B, C] and the label smoothing (null weights: unweighted kernel)
                self._chk(lib.tfy_dense_head_fused_soft(xin.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(),
                                                        self._ls, *rest, *self._weight_ptrs(sw)), "dense_head_fused_soft")
            elif self._wmode == (False, False):
                self._chk(lib.tfy_dense_head_fused(*args, s), "dense_head_fused")
            else:
                # Keras sample / class weights: each row's dlogits scaled by its weight inside the kernel
                self._chk(lib.tfy_dense_head_fused_weighted(*args, *self._weight_ptrs(sw)), "dense_head_fused_weighted")
            return
        logits = torch.mm(xin, w.t())
        sv.x, sv.dlogits = xin, torch.empty((B, C), dtype=torch.bfloat16, device=x.device)
        if self._binary is not None:
            sw_ptr, cw_ptr, _ = self._weight_ptrs(sw)
            self._chk(lib.tfy_sigmoid_xent(logits.data_ptr(), b.data_ptr(), y.data_ptr(), self._binary[0],
                                           int(self._binary[1]), sw_ptr, cw_ptr, self._loss.data_ptr(),
                                           sv.dlogits.data_ptr(), b.grad.data_ptr(), self._stats_ptr(), B, C, s),
                      "sigmoid_xent")
        elif self._ls is not None:
            sw_ptr, cw_ptr, _ = self._weight_ptrs(sw)
            self._chk(lib.tfy_softmax_xent_soft(logits.data_ptr(), b.data_ptr(), y.data_ptr(), self._ls, sw_ptr, cw_ptr,
                                                self._loss.data_ptr(), sv.dlogits.data_ptr(), b.grad.data_ptr(),
                                                self._stats_ptr(), B, C, s), "softmax_xent_soft")
        elif self._wmode == (False, False):
            self._chk(lib.tfy_softmax_xent(logits.data_ptr(), b.data_ptr(), y.data_ptr(), self._loss.data_ptr(),
                                           sv.dlogits.data_ptr(), b.grad.data_ptr(), self._stats_ptr(), B, C, s),
                      "softmax_xent")
        else:
            sw_ptr, cw_ptr, _ = self._weight_ptrs(sw)
            self._chk(lib.tfy_softmax_xent_weighted(logits.data_ptr(), b.data_ptr(), y.data_ptr(), sw_ptr, cw_ptr,
                                                    self._loss.data_ptr(), sv.dlogits.data_ptr(), b.grad.data_ptr(),
                                                    self._stats_ptr(), B, C, s), "softmax_xent_weighted")

    def _head_bwd(self, st, sv, grad):
        if st.fused:
            return sv.dh          # the fused head already produced the Dense layer's gated gradient and db
        w, _ = self._wb(st.layer)
        torch.mm(sv.dlogits.t(), sv.x, out=w.grad)
        return None if st.first else torch.mm(sv.dlogits, w)
