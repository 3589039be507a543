"""Fast path of the H100 train engine: explicit forward/backward out of fused kernels.

For ``Sequential`` models made of Conv2D(3x3, valid, stride 1) / MaxPooling2D(2x2) /
Dropout / Flatten / Dense layers with relu|linear activations and a sparse-categorical
cross-entropy (from logits) head -- the MNIST-CNN of the headline benchmark, the wine MLP --
the step does not go through autograd at all:

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


def build_plan(model) -> Optional[List[_Stage]]:
    """Pattern-match the layer list; None if the model is outside the fast-path grammar."""
    from tf_yarn_b200.keras import losses as kl
    loss = model.loss
    # the fused head computes softmax + cross-entropy from logits: either the loss takes logits and the
    # last layer is linear, or the last layer is a softmax and the loss takes probabilities
    if isinstance(loss, kl.SparseCategoricalCrossentropy):
        want_head_activation = "linear" if loss.from_logits else "softmax"
    elif loss == "sparse_categorical_crossentropy":
        want_head_activation = "softmax"
    else:
        return None
    for m in model._metrics_spec:
        if m not in ("accuracy", "acc", "sparse_categorical_accuracy"):
            return None
    # the head kernel counts the (weighted) hits: one weighted accuracy at most
    weighted = getattr(model, "_weighted_metrics_spec", [])
    if len(weighted) > 1 or any(m not in ("accuracy", "acc", "sparse_categorical_accuracy") for m in weighted):
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
        # Gradient-exchange overlap (opt-in, TFY_OVERLAP=1): parameters whose gradients are final before the
        # convolution weight-gradient kernel starts (every layer AFTER that convolution: for the MNIST-CNN the two
        # Dense layers, 98 % of the bytes) can be reduce-scattered / updated / all-gathered by COMMUNICATION CTAs
        # inside that kernel (ops/csrc/tfy_fused_step.cuh: tfy_overlap_role) on the 4 SMs its patch grid leaves
        # idle, the trailing fused-step launch handling the rest.  Numerically equivalent (GPU test); off by default
        # because the cost of the trailing launch is the LATENCY chain signal -> in-switch reduce -> store/ack ->
        # signal, which a smaller range does not shorten.
        self._overlap = os.environ.get("TFY_OVERLAP", "0") == "1"
        self._ov_used = False
        self._ov_gmid = 0
        self._warned = set()
        self._conv_sync = torch.zeros(1024, dtype=torch.int32, device=dev)     # grid barrier of the wgrad kernel
        self._c1_acc = torch.zeros(160 * 320, dtype=torch.float32, device=dev)   # first-layer dW/db per-CTA partials
        self._c1_cnt = torch.zeros(1, dtype=torch.int32, device=dev)

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
    def _split_k(M: int, N: int, K: int) -> int:
        """Split factor of the wgmma GEMM for skinny-output / long-K dense layers (1 = use cuBLAS)."""
        tiles = ((M + 127) // 128) * ((N + 127) // 128)
        k_tiles = (K + 63) // 64
        if K % 8 or tiles > 8 or k_tiles < 32:
            return 1
        per_cta = int(os.environ.get("TFY_SPLITK_TILES", "6"))   # k-tiles per CTA (6 == the TMA ring depth)
        return max(1, min(k_tiles // per_cta, 144 // tiles))

    @staticmethod
    def _tc_conv(st, B: int) -> bool:
        """True when the stage is served by the wgmma implicit-GEMM kernels of ops/csrc/tfy_conv.cu."""
        if os.environ.get("TFY_NO_TC_CONV") == "1":       # A/B switch: cuDNN + separate pool kernel instead
            return False
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

    def _overlap_desc(self, li: int, B: int, H: int, W: int):
        """Fused-step descriptor for the communication CTAs of conv stage ``li``'s weight-gradient kernel, or None.

        Overlapped: shard-relative groups [g_mid, S/8) of EVERY rank (balanced), where g_mid*8 is at least the
        flat offset of the first parameter of the layers after ``li`` (their gradients are final by now; rank 0's
        shard starts with the still-pending convolution parameters).  The size of the overlapped part is bounded
        by what ``n_cta`` SMs can move while the weight gradient runs (TFY_OVERLAP_GROUPS overrides)."""
        fused = self.fused
        if not self._overlap or self._ov_used or fused.zero_grads or fused.param_dtype != torch.bfloat16 \
                or fused.grad_dtype != torch.bfloat16:
            return None
        if fused.spec.kind == "rmsprop":             # no overlap role for RMSprop: the trailing step updates everything
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
        budget = int(os.environ.get("TFY_OVERLAP_GROUPS", str(2000 * n_cta)))
        g_mid = max(g_split, groups - budget)
        if groups - g_mid < 64:
            return None
        ov = fused.overlap_step(g_mid, groups, n_cta)
        self._ov_used, self._ov_gmid = True, g_mid
        return ov

    def _host_loss_ptr(self):
        """Pinned scalar of the slot being captured: the head kernel stores the loss there directly (UVA), so the
        captured step needs no D2H copy node."""
        slot = getattr(self, "_capture_slot", None)
        if slot is None or not getattr(self, "_loss_host", None):
            return None
        self._loss_in_host[slot] = True
        return self._loss_host[slot].data_ptr()

    def _splitk_acc(self, key, slabs: int, M: int, N: int) -> torch.Tensor:
        if key not in self._acc32 or tuple(self._acc32[key].shape) != (slabs, M, N):
            self._acc32[key] = torch.zeros((slabs, M, N), dtype=torch.float32, device=self.device)
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

    def _capture(self, x, y, w=None) -> None:
        super()._capture(x, y, w)
        with torch.cuda.stream(self.stream):
            self._stats.zero_()          # warm-up steps must not count in the epoch metrics
        self.stream.synchronize()

    # ------------------------------------------------------------------ the step
    @torch.no_grad()
    def _forward_backward(self, x, y, sw=None) -> None:
        lib, s = self.lib, self._s()
        self._k = 0
        B = x.shape[0]
        bf16 = torch.bfloat16
        saved = []
        cur = x                    # NHWC for images, [B, F] for vectors
        cur_is_f32 = cur.dtype == torch.float32
        # -------- forward
        for li, st in enumerate(self.plan):
            seed = (self._seed * 2654435761 + li * 97) & 0x7fffffff
            if st.kind == "conv":
                ly = st.layer
                w, b = self._wb(ly)
                H, W, Cin = ly.input_shape_
                O = ly.filters
                OH, OW = H - 2, W - 2
                fused_pre = False
                if self._tc_conv(st, B):
                    # wgmma implicit GEMM; bias + ReLU + 2x2 max-pool + dropout in the epilogue
                    xin = cur if (cur.dtype == bf16 and cur.is_contiguous()) else cur.to(bf16).contiguous()
                    p = torch.empty((B, OH // 2, OW // 2, O), dtype=bf16, device=cur.device)
                    code = torch.empty((B, OH // 2, OW // 2, O), dtype=torch.uint8, device=cur.device)
                    self._chk(lib.tfy_conv3x3_c32_pool_fwd(xin.data_ptr(), w.data_ptr(), b.data_ptr(), p.data_ptr(),
                                                           code.data_ptr(), B, H, W, float(st.drop), seed, self._hp,
                                                           s), "conv3x3_c32_pool_fwd")
                    saved.append((xin, False, None, code))
                    cur = p
                    cur_is_f32 = False
                    continue
                if Cin == 1:
                    # direct kernel: conv + bias + relu in one launch (relu folded only when requested)
                    a = torch.empty((B, OH, OW, O), dtype=bf16, device=cur.device)
                    if st.relu and not st.pool:
                        if O == 32 and os.environ.get("TFY_NO_TC_CONV") != "1":
                            self._chk(lib.tfy_conv3x3_c1_fwd_tc(cur.data_ptr(), int(cur_is_f32), w.data_ptr(),
                                                                b.data_ptr(), a.data_ptr(), B, H, W, s),
                                      "conv3x3_c1_fwd_tc")
                        else:
                            self._chk(lib.tfy_conv3x3_c1_fwd(cur.data_ptr(), int(cur_is_f32), w.data_ptr(),
                                                             b.data_ptr(), a.data_ptr(), B, H, W, O, s),
                                      "conv3x3_c1_fwd")
                        fused_pre = True
                        z = a
                    else:
                        z = None
                else:
                    z = None
                if z is None:
                    self._warn_once(f"conv_fwd:{li}", f"Conv2D layer {li} ({Cin} -> {O} channels, {H}x{W}, batch {B}) is "
                                    "outside the wgmma convolution kernels' envelope (C_in 32 / C_out 64 with ReLU + 2x2 "
                                    "pool, or C_in 1): forward and backward use cuDNN")
                    xin = cur.to(bf16) if cur.dtype != bf16 else cur
                    zc = F.conv2d(xin.permute(0, 3, 1, 2), w)       # NCHW logical over NHWC bytes
                    z = zc.permute(0, 2, 3, 1)
                    if not z.is_contiguous():
                        z = z.contiguous()
                if st.pool:
                    p = torch.empty((B, OH // 2, OW // 2, O), dtype=bf16, device=cur.device)
                    code = torch.empty((B, OH // 2, OW // 2, O), dtype=torch.uint8, device=cur.device)
                    self._chk(lib.tfy_bias_relu_pool_drop_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), code.data_ptr(),
                                                              B, OH, OW, O, float(st.drop), seed, self._hp, s),
                              "bias_relu_pool_drop_fwd")
                    saved.append((cur, cur_is_f32, None, code))
                    cur = p
                else:
                    mask = None
                    if not fused_pre:
                        if st.drop > 0:
                            mask = torch.empty((B, OH, OW, O), dtype=torch.uint8, device=cur.device)
                        self._chk(lib.tfy_bias_act_drop_fwd(z.data_ptr(), b.data_ptr(), z.data_ptr(),
                                                            mask.data_ptr() if mask is not None else None,
                                                            B * OH * OW, O, int(st.relu), float(st.drop), seed,
                                                            self._hp, s), "bias_act_drop_fwd")
                    elif st.drop > 0:
                        mask = torch.empty((B, OH, OW, O), dtype=torch.uint8, device=cur.device)
                        self._chk(lib.tfy_bias_act_drop_fwd(z.data_ptr(), None, z.data_ptr(), mask.data_ptr(),
                                                            B * OH * OW, O, 1, float(st.drop), seed, self._hp, s),
                                  "bias_act_drop_fwd")
                    saved.append((cur, cur_is_f32, z, mask))
                    cur = z
                cur_is_f32 = False
            elif st.kind == "flatten":
                saved.append(cur.shape)
                cur = cur.reshape(B, -1)
            elif st.kind == "dense":
                ly = st.layer
                w, b = self._wb(ly)
                xin = cur.to(bf16) if cur.dtype != bf16 else cur
                mask = torch.empty((B, ly.units), dtype=torch.uint8, device=cur.device) \
                    if (st.drop > 0 or st.relu) else None
                K = xin.shape[1]
                split = self._split_k(B, ly.units, K)
                if split > 1:
                    # skinny GEMM with a long K (e.g. 128 x 128 x 9216): split K over ~48 CTAs of the
                    # wgmma kernel; each K-slice stores its fp32 partial in its own slab and the epilogue sums the
                    # slabs in slice order
                    acc = self._splitk_acc(li, int(lib.tfy_gemm_bf16_splitk_slabs(K, split)), B, ly.units)
                    z = torch.empty((B, ly.units), dtype=bf16, device=cur.device)
                    tiles = ((B + 127) // 128) * ((ly.units + 127) // 128)
                    co_resident = tiles * split <= torch.cuda.get_device_properties(cur.device).multi_processor_count
                    if co_resident and os.environ.get("TFY_SPLITK_FUSE") == "1":
                        # ONE launch (opt-in): the K-slice CTAs of a tile meet on a counter, then each applies bias +
                        # ReLU + dropout to 1/split of the tile (summing the slabs in slice order) and writes the bf16
                        # activations and the gate mask.  (The slices spin on each other: the grid must be co-resident.)
                        # Off by default: the fence + counter + spin can cost more than the short second kernel of
                        # the same CUDA graph it removes.
                        key = ("splitk_cnt", li)
                        if key not in self._acc32:
                            self._acc32[key] = torch.zeros(2 * tiles, dtype=torch.int32, device=cur.device)
                        self._chk(lib.tfy_gemm_bf16_splitk_fused(
                            xin.data_ptr(), w.data_ptr(), acc.data_ptr(), self._acc32[key].data_ptr(), b.data_ptr(),
                            z.data_ptr(), mask.data_ptr() if mask is not None else None, B, ly.units, K,
                            xin.stride(0), w.stride(0), int(st.relu), float(st.drop), seed, self._hp, split, s),
                            "gemm_bf16_splitk_fused")
                    else:
                        self._chk(lib.tfy_gemm_bf16(xin.data_ptr(), w.data_ptr(), None, acc.data_ptr(), None, B,
                                                    ly.units, K, xin.stride(0), w.stride(0), ly.units, 0, split, s),
                                  "gemm_bf16(split-K)")
                        self._chk(lib.tfy_bias_act_drop_fwd_f32(acc.data_ptr(), b.data_ptr(), z.data_ptr(),
                                                                mask.data_ptr() if mask is not None else None, B,
                                                                ly.units, int(st.relu), float(st.drop), seed, self._hp,
                                                                acc.shape[0], s), "bias_act_drop_fwd_f32")
                else:
                    self._warn_once(f"dense_fwd:{li}", f"Dense layer {li} ({K} -> {ly.units}, batch {B}) is outside the "
                                    "split-K wgmma GEMM's envelope (long K, at most 8 output tiles): forward uses cuBLAS")
                    z = torch.mm(xin, w.t())
                    self._chk(lib.tfy_bias_act_drop_fwd(z.data_ptr(), b.data_ptr(), z.data_ptr(),
                                                        mask.data_ptr() if mask is not None else None, B, ly.units,
                                                        int(st.relu), float(st.drop), seed, self._hp, s),
                              "bias_act_drop_fwd")
                saved.append((xin, mask))
                cur = z
                cur_is_f32 = False
            else:  # head
                ly = st.layer
                w, b = self._wb(ly)
                xin = cur.to(bf16) if cur.dtype != bf16 else cur
                prev = self.plan[li - 1] if li > 0 else None
                K, C = xin.shape[1], ly.units
                if (prev is not None and prev.kind == "dense" and K in (128, 256, 512) and C <= 16
                        and xin.is_contiguous() and os.environ.get("TFY_NO_FUSED_HEAD") != "1"):
                    # one launch: logits, loss, dlogits, dW2, db2 and the gradient entering the previous Dense
                    # layer (its ReLU / dropout gate and bias gradient included)
                    pmask = saved[li - 1][1]
                    pscale = 1.0 / (1.0 - prev.drop) if prev.drop > 0 else 1.0
                    _, pb = self._wb(prev.layer)
                    need = int(lib.tfy_dense_head_scratch_elems(K, C, B))      # one slab per 16 rows of the batch
                    if "head_scratch" not in self._acc32 or self._acc32["head_scratch"].numel() < need:
                        self._acc32["head_scratch"] = torch.zeros(need, dtype=torch.float32, device=cur.device)
                        self._acc32["head_counter"] = torch.zeros(1, dtype=torch.int32, device=cur.device)
                    dh = torch.empty((B, K), dtype=bf16, device=cur.device)
                    if self._wmode == (False, False):
                        self._chk(lib.tfy_dense_head_fused(
                            xin.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(),
                            pmask.data_ptr() if pmask is not None else None, pscale, self._loss.data_ptr(),
                                self._host_loss_ptr(), self._stats_ptr(), w.grad.data_ptr(), b.grad.data_ptr(),
                            dh.data_ptr(), pb.grad.data_ptr(), self._acc32["head_scratch"].data_ptr(),
                            self._acc32["head_counter"].data_ptr(), B, K, C, s), "dense_head_fused")
                    else:
                        # Keras sample / class weights: each row's dlogits scaled by its weight inside the kernel
                        self._chk(lib.tfy_dense_head_fused_weighted(
                            xin.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(),
                            pmask.data_ptr() if pmask is not None else None, pscale, self._loss.data_ptr(),
                            self._host_loss_ptr(), self._stats_ptr(), w.grad.data_ptr(), b.grad.data_ptr(),
                            dh.data_ptr(), pb.grad.data_ptr(), self._acc32["head_scratch"].data_ptr(),
                            self._acc32["head_counter"].data_ptr(), B, K, C, *self._weight_ptrs(sw)),
                            "dense_head_fused_weighted")
                    saved.append(("fused", dh))
                    continue
                self._warn_once(f"head:{li}", f"classifier head {li} ({xin.shape[1]} -> {ly.units}, batch {B}) is outside "
                                "the fused head kernel's envelope (K in 128/256/512, at most 16 classes, Dense "
                                "predecessor): logits and gradients use cuBLAS")
                logits = torch.mm(xin, w.t())
                C = ly.units
                dlogits = torch.empty((B, C), dtype=bf16, device=cur.device)
                if self._wmode == (False, False):
                    self._chk(lib.tfy_softmax_xent(logits.data_ptr(), b.data_ptr(), y.data_ptr(), self._loss.data_ptr(),
                                                   dlogits.data_ptr(), b.grad.data_ptr(), self._stats_ptr(), B, C, s),
                              "softmax_xent")
                else:
                    sw_ptr, cw_ptr, _ = self._weight_ptrs(sw)
                    self._chk(lib.tfy_softmax_xent_weighted(logits.data_ptr(), b.data_ptr(), y.data_ptr(), sw_ptr,
                                                            cw_ptr, self._loss.data_ptr(), dlogits.data_ptr(),
                                                            b.grad.data_ptr(), self._stats_ptr(), B, C, s),
                              "softmax_xent_weighted")
                saved.append((xin, dlogits))
        # -------- backward
        grad = None
        pre_gated = False          # the dgrad kernel of the next layer already applied this layer's ReLU gate
        dense_gated = False        # the fused head already produced the gated gradient + db of the Dense below
        for li in range(len(self.plan) - 1, -1, -1):
            st = self.plan[li]
            sv = saved[li]
            first = li == 0
            if st.kind == "head" and sv[0] == "fused":
                grad = sv[1]
                dense_gated = True          # the Dense layer below already has its gated gradient and db
            elif st.kind == "head":
                xin, dlogits = sv
                w, _ = self._wb(st.layer)
                torch.mm(dlogits.t(), xin, out=w.grad)
                grad = torch.mm(dlogits, w) if not first else None
            elif st.kind == "dense":
                xin, mask = sv
                ly = st.layer
                w, b = self._wb(ly)
                scale = 1.0 / (1.0 - st.drop) if st.drop > 0 else 1.0
                if dense_gated:
                    dense_gated = False
                else:
                    self._chk(lib.tfy_act_drop_bwd_bias(grad.data_ptr(), mask.data_ptr() if mask is not None else None,
                                                        None, grad.data_ptr(), scale, B, ly.units,
                                                        self._partial.data_ptr(), b.grad.data_ptr(),
                                                        self._counter.data_ptr(), s), "act_drop_bwd_bias")
                I = xin.shape[1]
                if (ly.units % 8 == 0 and I % 8 == 0 and grad.is_contiguous()
                        and xin.is_contiguous() and w.is_contiguous() and w.grad.is_contiguous()
                        and os.environ.get("TFY_NO_TC_DENSE_BWD") != "1"):
                    # dW = dh^T x (straight into the flat gradient buffer) and dx = dh W in ONE wgmma kernel
                    dx = torch.empty((B, I), dtype=bf16, device=grad.device) if not first else None
                    self._chk(lib.tfy_dense_bwd(grad.data_ptr(), xin.data_ptr(), w.data_ptr(), w.grad.data_ptr(),
                                                dx.data_ptr() if dx is not None else None, B, ly.units, I, s),
                              "dense_bwd")
                    grad = dx
                else:
                    self._warn_once(f"dense_bwd:{li}", f"Dense layer {li} ({I} -> {ly.units}, batch {B}) is outside "
                                    "the wgmma dense-backward kernel's envelope: cuBLAS computes dW / dx")
                    torch.mm(grad.t(), xin, out=w.grad)
                    grad = torch.mm(grad, w) if not first else None
            elif st.kind == "flatten":
                if grad is not None:
                    grad = grad.reshape(sv)
            else:  # conv
                xin, xin_f32, zout, aux = sv
                ly = st.layer
                w, b = self._wb(ly)
                H, W, Cin = ly.input_shape_
                O = ly.filters
                OH, OW = H - 2, W - 2
                scale = self._conv_drop_scale(st, st.pool and self._tc_conv(st, B))
                gated, pre_gated = pre_gated, False
                if (Cin == 1 and O == 32 and gated and not st.pool and aux is None and first
                        and os.environ.get("TFY_NO_TC_CONV") != "1"):
                    # first layer: dW and db in ONE tensor-core kernel (im2col built in shared memory)
                    dz = grad if grad.is_contiguous() else grad.contiguous()
                    self._chk(lib.tfy_conv3x3_c1_wgrad_tc(xin.data_ptr(), int(xin_f32), dz.data_ptr(),
                                                          self._c1_acc.data_ptr(), self._c1_cnt.data_ptr(),
                                                          w.grad.data_ptr(), b.grad.data_ptr(), B, H, W, s),
                              "conv3x3_c1_wgrad_tc")
                    grad = None
                    continue
                if (st.pool and self._tc_conv(st, B) and grad.is_contiguous()
                        and os.environ.get("TFY_NO_UNPOOL_FUSION") != "1"):
                    # pool/dropout/ReLU backward fused into the operand producers of wgrad and dgrad: the
                    # 4x larger dz tensor is never written; db comes out of the wgrad kernel.  When the dgrad
                    # launch follows, the wgrad CTAs only store their fp32 partials (no grid barrier) and the
                    # dgrad kernel reduces them into dW / db behind its main loop: the same bits either way.
                    if "wgrad_scratch" not in self._acc32:
                        self._acc32["wgrad_scratch"] = torch.empty(
                            int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()), dtype=torch.float32, device=grad.device)
                    part = self._acc32["wgrad_scratch"]
                    ov = self._overlap_desc(li, B, H, W)
                    ovp = ctypes.byref(ov) if ov is not None else None
                    n_part = ctypes.c_int(0)
                    if first:
                        self._chk(lib.tfy_conv3x3_c32_wgrad_unpool_ov(
                            xin.data_ptr(), grad.data_ptr(), aux.data_ptr(), scale, part.data_ptr(),
                            w.grad.data_ptr(), b.grad.data_ptr(), self._conv_sync.data_ptr(), B, H, W, ovp, s),
                            "conv3x3_c32_wgrad_unpool")
                    else:
                        self._chk(lib.tfy_conv3x3_c32_wgrad_unpool_deferred(
                            xin.data_ptr(), grad.data_ptr(), aux.data_ptr(), scale, part.data_ptr(), B, H, W, ovp,
                            ctypes.byref(n_part), s), "conv3x3_c32_wgrad_unpool_deferred")
                    dp = grad
                    grad = None
                    if not first:
                        prev = self.plan[li - 1]
                        fold = (prev.kind == "conv" and prev.relu and not prev.pool and prev.drop == 0
                                and saved[li - 1][2] is not None and saved[li - 1][2].data_ptr() == xin.data_ptr())
                        grad = torch.empty((B, H, W, Cin), dtype=bf16, device=dp.device)
                        self._chk(lib.tfy_conv3x3_c32_dgrad_unpool_reduce(
                            dp.data_ptr(), aux.data_ptr(), scale, w.data_ptr(), xin.data_ptr() if fold else None,
                            grad.data_ptr(), B, H, W, part.data_ptr(), n_part.value, w.grad.data_ptr(),
                            b.grad.data_ptr(), s), "conv3x3_c32_dgrad_unpool_reduce")
                        pre_gated = fold
                    continue
                if st.pool:
                    dz = torch.empty((B, OH, OW, O), dtype=bf16, device=grad.device)
                    self._chk(lib.tfy_pool_drop_relu_bwd(grad.data_ptr(), aux.data_ptr(), dz.data_ptr(), scale, B, OH,
                                                         OW, O, self._partial.data_ptr(), b.grad.data_ptr(),
                                                         self._counter.data_ptr(), s), "pool_drop_relu_bwd")
                else:
                    dz = grad if grad.is_contiguous() else grad.contiguous()
                    use_mask = aux is not None
                    self._chk(lib.tfy_act_drop_bwd_bias(dz.data_ptr(), aux.data_ptr() if use_mask else None,
                                                        zout.data_ptr() if (st.relu and not use_mask
                                                                            and not gated) else None,
                                                        dz.data_ptr(), scale, B * OH * OW, O,
                                                        self._partial.data_ptr(), b.grad.data_ptr(),
                                                        self._counter.data_ptr(), s), "act_drop_bwd_bias")
                if Cin == 1:
                    self._chk(lib.tfy_conv3x3_c1_wgrad(xin.data_ptr(), int(xin_f32), dz.data_ptr(),
                                                       self._partial.data_ptr(), w.grad.data_ptr(),
                                                       self._counter.data_ptr(), B, H, W, O, s), "conv3x3_c1_wgrad")
                    grad = None
                    if not first:
                        raise RuntimeError("C_in=1 convolution must be the first layer")
                elif self._tc_conv(st, B):
                    if "wgrad_scratch" not in self._acc32:       # per-CTA fp32 partial tiles (L2 resident)
                        self._acc32["wgrad_scratch"] = torch.empty(
                            int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()), dtype=torch.float32, device=dz.device)
                    acc = self._acc32["wgrad_scratch"]
                    self._chk(lib.tfy_conv3x3_c32_wgrad(xin.data_ptr(), dz.data_ptr(), acc.data_ptr(),
                                                        w.grad.data_ptr(), self._conv_sync.data_ptr(), B, H, W, s),
                              "conv3x3_c32_wgrad")
                    grad = None
                    if not first:
                        prev = self.plan[li - 1]
                        # fold the producer's ReLU gate into the dgrad epilogue when its output IS our input
                        fold = (prev.kind == "conv" and prev.relu and not prev.pool and prev.drop == 0
                                and saved[li - 1][2] is not None and saved[li - 1][2].data_ptr() == xin.data_ptr())
                        grad = torch.empty((B, H, W, Cin), dtype=bf16, device=dz.device)
                        self._chk(lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(),
                                                            xin.data_ptr() if fold else None, grad.data_ptr(), B, H,
                                                            W, s), "conv3x3_c32_dgrad")
                        pre_gated = fold
                    continue
                else:
                    xb = xin.to(bf16) if xin.dtype != bf16 else xin
                    dx, dw, _ = torch.ops.aten.convolution_backward(
                        dz.permute(0, 3, 1, 2), xb.permute(0, 3, 1, 2), w, None, [1, 1], [0, 0], [1, 1], False,
                        [0, 0], 1, [not first, True, False])
                    w.grad.copy_(dw)
                    grad = None
                    if not first:
                        g = dx.permute(0, 2, 3, 1)
                        grad = g if g.is_contiguous() else g.contiguous()
        if self._ov_used:
            # the communication CTAs of the weight-gradient kernel already handled groups [g_mid, end) of every shard
            self.fused.step(shard_groups=(0, self._ov_gmid), advance=True)
            self._ov_used = False
        else:
            self.fused.step()
        self._launches_per_step = self._k + 1     # our kernels launched per step (library GEMMs excluded)
