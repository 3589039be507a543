"""The conv2 tensor-core kernels (ops/csrc/tfy_conv.cu, C_in = 32 -> C_out = 64) against the float64 reference
(tests/conv2_reference.py), called through the ctypes declarations of keras/fastpath.py, at every shape class the fast
path sends them and at patch counts chosen from the device's SM count s.

Schedules.  The forward and both weight-gradient kernels tile the (H-2) x (W-2) output into 8 x 8 patches of an image
pair: P = (H-2)/8 * (W-2)/8 * B/2.  The data gradient tiles the H x W input: P = ceil(H/8) * ceil(W/8) * B/2.  The grid
is c_grid(P) (P CTAs up to s, else P spread evenly over the fewest waves).  The configurations below are derived from s
so that each kernel runs at 1 patch, fewer than s, exactly s and s + 1 patches (where some shape and even B give that
count) and at more than 2 * WG_RING * s patches, where the weight gradient's 5-stage ring and its mbarrier phases wrap
at least twice.

Exactness.  Dropout keep bits are pure functions of (seed, step, element): with a bias that makes every pooled value
positive the gate bits must equal the host-built hash's keep bits everywhere.  Argmax positions are exact wherever the
window's top two values are farther apart than twice their rounding bound plus the tag perturbation (the kernel
overwrites the two low mantissa bits, at most 3 ulp = 3 u |z|, of each compared value); ReLU gate bits and zeroed
outputs wherever the value they test is farther from 0 than its bound; the data gradient's gate is a bf16 input, so
dx is exactly 0 wherever gate <= 0.  Constant positive input regions give exact ties: the last window position must win
for a positive maximum, the first for a negative one.  The deferred weight-gradient reduction must give the same bits
as the in-kernel one, and the un-pool data gradient the same dx with and without the reduction.

Tolerances.  u = 2^-23 bounds one fp32 addition relative to the sum of the magnitudes it adds, whether it rounds (u / 2)
or truncates (tensor-core accumulation may); products of bf16 numbers are exact in fp32.  A sum whose terms pass through
at most d additions is within d u sum|terms|, and a bf16 output of it within U_BF16 |ref| + 2 d u sum|terms|.  d per
kernel (terms = the kernel's products, or its fp32 partials):

* forward: one wgmma chain of K = 9 taps * 32 channels = 288 products, + 3 for the tag, + 2 (bias add, keep scale);
  sum|terms| = (largest sum|a W| of the window + |bias|) * keep scale.
* data gradient (plain and un-pool): one chain of 9 taps * 64 channels = 576 products.
* weight gradient: a CTA of n = ceil(P / grid) patches takes them WG_GROUP = 4 at a time; per group and tap one chain of
  128 * min(4, n) pixel products, added into its fp32 tile (ceil(n / 4) additions).  The reduction over the grid's
  partials (c_wg_slice) adds at most ceil(grid / parts) partials per part and then the parts: at most 2 * grid.
  d = 128 * min(4, n) + ceil(n / 4) + 2 * grid.
* db: the fp32 product dp * scale (1), a producer thread's chain over its ceil(n / 2) patches, 2 shuffles, 16 warps in
  order, the reduction (2 * grid): d = 1 + ceil(n / 2) + 2 + 16 + 2 * grid.
* The un-pool operand is dp * scale rounded to bf16; the reference rounds it the same way (conv2_reference.unpool).

Hygiene.  Every output sits between guard bytes and is pre-filled with 0xA5; the reducing kernels run RUNS times on
the same inputs and must give the same bits; after each in-kernel reduction the grid barrier's generation word has
advanced by one and its arrival counters are back at zero.
"""
import ctypes
import hashlib
import json
import os
import types

import numpy as np
import pytest
import torch

import conv2_reference as ref
import nn_reference
from tf_yarn_b200.keras import fastpath

pytestmark = pytest.mark.gpu

U = 2.0 ** -23              # per-addition bound, truncation included
U_BF16 = nn_reference.U_BF16
GUARD = 64
RUNS = 3
SEED, STEP = 20261017, 5
WG_RING, WG_GROUP, WG_PART = 5, 4, 64 * 9 * 32 + 64
D_FWD, D_DGRAD = 288 + 3 + 2, 576
SHAPES = [(10, 10), (10, 34), (34, 10), (26, 26), (18, 42), (66, 66)]
GOLDEN_BWD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv2_bwd_b128_sha256.json")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def c_grid(p, s):
    if p <= s:
        return p
    waves = -(-p // s)
    return -(-p // waves)


def tiles_fwd(h, w):
    return ((h - 2) // 8) * ((w - 2) // 8)


def tiles_dgrad(h, w):
    return -(-h // 8) * -(-w // 8)


def configs(s):
    """(H, W, B) list covering, for the forward / weight-gradient schedule and for the data-gradient schedule, 1, < s, s,
    s + 1 and > 2 WG_RING s patches where a shape of the list (or, for s + 1 data-gradient patches, any H, W = 2 mod 8)
    and an even B give that count; then every shape at least once."""
    out = []

    def add(h, w, b):
        if (h, w, b) not in out:
            out.append((h, w, b))
    for tiles in (tiles_fwd, tiles_dgrad):
        targets = [1, s // 2, s, s + 1]
        for p in targets:
            for h, w in SHAPES:
                t = tiles(h, w)
                if p % t == 0 and p >= t:
                    add(h, w, 2 * (p // t))
                    break
            else:
                # any shape whose tile count divides p: ceil(H/8) = i + 1 for H = 8 i + 2 (likewise W)
                for i in range(1, 40):
                    for j in range(i, 200):
                        t = (i + 1) * (j + 1) if tiles is tiles_dgrad else i * j
                        if p % t == 0:
                            add(8 * i + 2, 8 * j + 2, 2 * (p // t))
                            break
                    else:
                        continue
                    break
        h, w = (26, 26) if tiles is tiles_fwd else (10, 10)
        add(h, w, 2 * (-(-(2 * WG_RING * s + 1) // tiles(h, w))))
    for h, w in SHAPES:
        if not any(c[:2] == (h, w) for c in out):
            add(h, w, 2 if (h, w) != (66, 66) else 42)
    return out


@pytest.fixture(scope="module")
def lib():
    # (importing fastpath declared the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    h = nn_reference.host_lib(str(tmp_path_factory.mktemp("conv2ref")))
    assert h is not None, "the host build of the dropout hash needs g++ and the CUDA headers"
    return ref.declare_host(h)


@pytest.fixture(scope="module")
def hp():
    from tf_yarn_b200.ops import native
    h = native.OptHyper(1.0, 0.0, 0.0, 0.0, 0.0, 1.0, STEP, 0, 0, 0)
    return torch.frombuffer(bytearray(bytes(h)), dtype=torch.uint8).cuda()


def _s():
    return torch.cuda.current_stream().cuda_stream


class Out:
    """Device output between guard bytes, pre-filled with 0xA5 so that a skipped element or a stray write shows."""

    def __init__(self, shape, dtype):
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        self.full = torch.full((2 * GUARD + n,), 0xA5, dtype=torch.uint8, device="cuda")
        self.t = self.full[GUARD:GUARD + n].view(dtype).view(shape)

    def ptr(self):
        return self.t.data_ptr()

    def get(self):
        torch.cuda.synchronize()
        assert bool((self.full[:GUARD] == 0xA5).all()) and bool((self.full[-GUARD:] == 0xA5).all()), "guard written"
        return self.t.clone()


def _np(t):
    return t.double().cpu().numpy()


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.uint8).cpu()


def _close(got, want, e, what):
    """bf16 output: |got - want| <= U_BF16 |want| + 2 e."""
    got = _np(got) if isinstance(got, torch.Tensor) else got
    tol = U_BF16 * np.abs(want) + 2.0 * e + 1e-30
    bad = ~(np.abs(got - want) <= tol)
    assert not bad.any(), (what, int(bad.sum()), float(np.abs(got - want)[bad].max()), float(tol[bad].min()))


def keep_scale_of(rate):
    """The forward's rule, stated independently of the code under test: thr = (uint32)(rate * 256 + 0.5) in fp32."""
    r = np.float32(rate)
    thr = int(np.floor(r * np.float32(256) + np.float32(0.5))) if r > 0 else 0
    return thr, np.float32(256) / np.float32(256 - thr)


def _inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(B, H, W, 32, generator=g).relu().to(torch.bfloat16)
    w = (torch.randn(64, 3, 3, 32, generator=g) * 0.06).to(torch.bfloat16)
    bias = (torch.randn(64, generator=g) * 0.1).to(torch.bfloat16)
    PH, PW = (H - 2) // 2, (W - 2) // 2
    dp = (torch.randn(B, PH, PW, 64, generator=g) * 0.5).to(torch.bfloat16)
    dz = (torch.randn(B, H - 2, W - 2, 64, generator=g) * 0.5).to(torch.bfloat16)
    return [t.cuda() for t in (a, w, bias, dp, dz)]


def run_fwd(lib, a, w, bias, rate, seed, hp_ptr):
    B, H, W, _ = a.shape
    shape = (B, (H - 2) // 2, (W - 2) // 2, 64)
    p, code = Out(shape, torch.bfloat16), Out(shape, torch.uint8)
    assert lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), p.ptr(), code.ptr(), B, H, W,
                                        rate, seed, hp_ptr, _s()) == 0
    return p.get(), code.get()


def check_fwd(host, a, w, bias, rate, p, code, step):
    """Forward outputs against the reference: keep bits, gate bits, argmax and pooled values (module docstring)."""
    B, H, W, _ = a.shape
    thr, ks = keep_scale_of(rate)
    n = B * ((H - 2) // 2) * ((W - 2) // 2) * 64
    keep = ref.keep_from_hash(ref.host_hash_u32(host, SEED, step, (n + 3) // 4), thr, n).reshape(p.shape) \
        if thr else None
    r = ref.fwd(_np(a), _np(w), _np(bias), keep, float(ks))
    code = code.cpu().numpy()
    on = (code >> 2) & 1
    if keep is not None:
        assert not (on.astype(bool) & ~keep).any(), "a dropped element lets the gradient through"
    e_v = D_FWD * U * r.mag                                            # bound of v = max + bias
    sure = np.abs(r.v) > e_v
    assert ((on == (r.code >> 2)) | ~sure).all(), "ReLU / keep bits"
    sep = r.gap > 2 * 288 * U * r.win_mag + 6 * U * np.abs(r.best)
    assert sep.mean() > 0.9
    assert (((code & 3) == (r.code & 3)) | ~sep).all(), "argmax positions"
    got = _np(p)
    assert (got[on == 0] == 0).all(), "zeroed outputs"
    both = (on == 1) & (r.code >> 2 == 1)
    _close(got[both], r.p[both], D_FWD * U * r.mag[both] * float(ks), "pooled")
    return r


def _wg_depth(P, s):
    grid = c_grid(P, s)
    n = -(-P // grid)
    return 128 * min(WG_GROUP, n) + -(-n // WG_GROUP) + 2 * grid, 1 + -(-n // 2) + 2 + 16 + 2 * grid, grid


@pytest.mark.parametrize("H,W,B", configs(_sms()))
def test_kernels_match_reference(lib, host, hp, H, W, B):
    s = _sms()
    a, w, bias, dp, dz = _inputs(B, H, W, seed=H * 1000 + W * 7 + B)
    P = tiles_fwd(H, W) * B // 2
    an, wn = _np(a), _np(w)
    n_scr = int(lib.tfy_conv3x3_c32_wgrad_scratch_elems())

    # ---- forward: rate 0 (no generator read) and rate 0.3 with the step from a device TfyOptHyper
    p0, code0 = run_fwd(lib, a, w, bias, 0.0, SEED, None)
    check_fwd(host, a, w, bias, 0.0, p0, code0, 0)
    p, code = run_fwd(lib, a, w, bias, 0.3, SEED, hp.data_ptr())
    check_fwd(host, a, w, bias, 0.3, p, code, STEP)

    # ---- data gradient, plain, with and without the gate (the previous layer's ReLU output: a)
    dzn = _np(dz)
    want, mag = ref.dgrad(dzn, wn)
    for gate in (None, a):
        dx = Out((B, H, W, 32), torch.bfloat16)
        assert lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), gate.data_ptr() if gate is not None else None,
                                         dx.ptr(), B, H, W, _s()) == 0
        got = _np(dx.get())
        if gate is None:
            _close(got, want, D_DGRAD * U * mag, "dgrad dx")
        else:
            open_ = an > 0
            assert (got[~open_] == 0).all(), "gated dx"
            _close(got[open_], want[open_], D_DGRAD * U * mag[open_], "dgrad dx (gated)")

    # ---- weight gradient with the in-kernel grid-barrier reduction
    d_w, d_b, grid = _wg_depth(P, s)
    dw_ref, dw_mag = ref.wgrad(an, dzn)
    sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
    first = None
    for run in range(RUNS):
        part = torch.full((n_scr,), float("nan"), device="cuda")
        dw = Out((64, 3, 3, 32), torch.bfloat16)
        assert lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dz.data_ptr(), part.data_ptr(), dw.ptr(), sync.data_ptr(), B,
                                         H, W, _s()) == 0
        got = dw.get()
        sy = sync.cpu()
        assert int(sy[0]) == run + 1 and not sy[1:].any(), "grid barrier state"
        if first is None:
            first = got
            _close(got, dw_ref, d_w * U * dw_mag, "wgrad dW")
        else:
            assert torch.equal(_bits(got), _bits(first)), f"wgrad dW differs on run {run}"

    # ---- fused un-pool backward with the forward's keep scale
    thr, ks = keep_scale_of(0.3)
    scale = ctypes.c_float(fastpath.keep_scale(lib, 0.3))
    assert np.float32(scale.value) == ks
    dzu, g = ref.unpool(_np(dp), code.cpu().numpy(), float(ks))
    dwu_ref, dwu_mag = ref.wgrad(an, dzu)
    db_ref, db_mag = ref.bias_grad(g)
    dxu_ref, dxu_mag = ref.dgrad(dzu, wn)
    results = {}
    sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
    for run in range(RUNS):
        part = torch.full((n_scr,), float("nan"), device="cuda")
        dw, db = Out((64, 3, 3, 32), torch.bfloat16), Out((64,), torch.bfloat16)
        assert lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale, part.data_ptr(),
                                                dw.ptr(), db.ptr(), sync.data_ptr(), B, H, W, _s()) == 0
        got = (dw.get(), db.get())
        sy = sync.cpu()
        assert int(sy[0]) == run + 1 and not sy[1:].any(), "grid barrier state (un-pool)"
        if run == 0:
            results["in_kernel"] = got
            _close(got[0], dwu_ref, d_w * U * dwu_mag, "wgrad_unpool dW")
            _close(got[1], db_ref, d_b * U * db_mag, "wgrad_unpool db")
        else:
            assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(got, results["in_kernel"])), run
    for gate in (None, a):
        for run in range(RUNS):
            part = torch.full((n_scr,), float("nan"), device="cuda")
            n_part = ctypes.c_int(-1)
            dw, db = Out((64, 3, 3, 32), torch.bfloat16), Out((64,), torch.bfloat16)
            dx = Out((B, H, W, 32), torch.bfloat16)
            gp = gate.data_ptr() if gate is not None else None
            assert lib.tfy_conv3x3_c32_wgrad_unpool_deferred(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                             part.data_ptr(), B, H, W, None, ctypes.byref(n_part),
                                                             _s()) == 0
            assert n_part.value == grid
            assert lib.tfy_conv3x3_c32_dgrad_unpool_reduce(dp.data_ptr(), code.data_ptr(), scale, w.data_ptr(), gp,
                                                           dx.ptr(), B, H, W, part.data_ptr(), n_part.value, dw.ptr(),
                                                           db.ptr(), _s()) == 0
            got = (dw.get(), db.get(), dx.get())
            assert torch.equal(_bits(got[0]), _bits(results["in_kernel"][0])), "deferred dW != in-kernel dW"
            assert torch.equal(_bits(got[1]), _bits(results["in_kernel"][1])), "deferred db != in-kernel db"
            key = "dx" if gate is None else "dx_gated"
            if key not in results:
                results[key] = got[2]
                gx = _np(got[2])
                if gate is None:
                    _close(gx, dxu_ref, D_DGRAD * U * dxu_mag, "dgrad_unpool_reduce dx")
                else:
                    open_ = an > 0
                    assert (gx[~open_] == 0).all()
                    _close(gx[open_], dxu_ref[open_], D_DGRAD * U * dxu_mag[open_], "dgrad_unpool_reduce dx (gated)")
            else:
                assert torch.equal(_bits(got[2]), _bits(results[key])), f"{key} differs on run {run}"
        # the un-pool data gradient without the reduction gives the same dx
        dx = Out((B, H, W, 32), torch.bfloat16)
        assert lib.tfy_conv3x3_c32_dgrad_unpool(dp.data_ptr(), code.data_ptr(), scale, w.data_ptr(),
                                                gate.data_ptr() if gate is not None else None, dx.ptr(), B, H, W,
                                                _s()) == 0
        assert torch.equal(_bits(dx.get()), _bits(results["dx" if gate is None else "dx_gated"])), "dgrad_unpool dx"


@pytest.mark.parametrize("H,W,B", [(8, 8, 2), (8, 8, None), (13, 13, 6), (27, 20, 4), (5, 7, 2), (20, 27, 34)])
def test_plain_data_gradient_at_any_image_size(lib, H, W, B):
    """tfy_conv3x3_c32_dgrad accepts any H, W >= 3: single tiles, partial last tiles in both directions, and (8, 8)
    at s and s + 1 patches."""
    s = _sms()
    batches = [B] if B is not None else [2 * s, 2 * (s + 1)]
    for B in batches:
        g = torch.Generator().manual_seed(H * 31 + W + B)
        dz = (torch.randn(B, H - 2, W - 2, 64, generator=g) * 0.5).to(torch.bfloat16).cuda()
        w = (torch.randn(64, 3, 3, 32, generator=g) * 0.06).to(torch.bfloat16).cuda()
        gate = torch.randn(B, H, W, 32, generator=g).to(torch.bfloat16).cuda()
        want, mag = ref.dgrad(_np(dz), _np(w))
        for gt in (None, gate):
            dx = Out((B, H, W, 32), torch.bfloat16)
            assert lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), gt.data_ptr() if gt is not None else None,
                                             dx.ptr(), B, H, W, _s()) == 0
            got = _np(dx.get())
            if gt is None:
                _close(got, want, D_DGRAD * U * mag, f"dgrad dx {H}x{W} B={B}")
            else:
                open_ = _np(gate) > 0
                assert (got[~open_] == 0).all()
                _close(got[open_], want[open_], D_DGRAD * U * mag[open_], f"gated dgrad dx {H}x{W} B={B}")


@pytest.mark.parametrize("rate", [0.3, 0.9])
@pytest.mark.parametrize("H,W,B", [(26, 26, 128), (10, 34, 6)])
def test_forward_keep_bits_exact_everywhere(lib, host, hp, H, W, B, rate):
    """A bias that makes every pooled value positive: the gate bit is the keep bit, which must equal the host-built
    hash's byte test for every element, and kept values carry the forward's keep scale."""
    a, w, _, _, _ = _inputs(B, H, W, seed=3)
    bias = torch.full((64,), 64.0, dtype=torch.bfloat16, device="cuda")
    p, code = run_fwd(lib, a, w, bias, rate, SEED, hp.data_ptr())
    thr, ks = keep_scale_of(rate)
    n = code.numel()
    keep = ref.keep_from_hash(ref.host_hash_u32(host, SEED, STEP, (n + 3) // 4), thr, n)
    got = code.cpu().numpy().reshape(-1)
    np.testing.assert_array_equal((got >> 2) & 1, keep.astype(np.uint8))
    assert abs(keep.mean() - (1 - thr / 256)) < 0.01
    r = check_fwd(host, a, w, bias, rate, p, code, STEP)
    assert (r.v > 0).all()


@pytest.mark.parametrize("H,W", [(26, 26), (66, 66)])
@pytest.mark.parametrize("sign", [1, -1])
def test_forward_exact_ties_follow_the_pinned_rule(lib, H, W, sign):
    """Constant input and weights: every z is 288 / 64 = 4.5 exactly (times sign), every window an exact tie.  The last
    position wins for a positive maximum, the first for a negative one."""
    B = 2
    a = torch.ones(B, H, W, 32, dtype=torch.bfloat16, device="cuda")
    w = torch.full((64, 3, 3, 32), sign / 64.0, dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    p, code = run_fwd(lib, a, w, bias, 0.0, SEED, None)
    r = ref.fwd(_np(a), _np(w), _np(bias))
    np.testing.assert_array_equal(code.cpu().numpy(), r.code)
    assert (r.code & 3 == (3 if sign > 0 else 0)).all()
    np.testing.assert_array_equal(_np(p), r.p)


# ---------------------------------------------------------------------------------------------- dropout adjoint
def _fast_path_scale(lib, rate):
    """The scale the fast path hands a tensor-core conv stage's backward."""
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    st = types.SimpleNamespace(kind="conv", pool=True, relu=True, drop=rate)
    return FastSequentialEngine._conv_drop_scale(types.SimpleNamespace(lib=lib), st, True)


@pytest.mark.parametrize("rate", [0.25, 0.3, 0.9])
def test_unpool_backward_is_the_adjoint_of_the_forward_dropout(lib, hp, rate):
    """Forward at `rate`, then the fused backward with the fast path's scale.  Nonnegative activations and pooled
    gradients make every term of dW and db nonnegative, so the fp32 partials the deferred weight gradient leaves (summed
    here in float64) are within d u of the float64 adjoint built with the forward's keep scale, d = the per-CTA depth of
    the module docstring: a 0.1 % scale error is far outside that."""
    B, H, W = 64, 26, 26
    s = _sms()
    a, w, bias, dp, _ = _inputs(B, H, W, seed=77)
    dp = dp.abs()
    _, code = run_fwd(lib, a, w, bias, rate, SEED, hp.data_ptr())
    _, ks = keep_scale_of(rate)
    scale = ctypes.c_float(_fast_path_scale(lib, rate))
    part = torch.full((int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()),), float("nan"), device="cuda")
    n_part = ctypes.c_int(0)
    assert lib.tfy_conv3x3_c32_wgrad_unpool_deferred(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                     part.data_ptr(), B, H, W, None, ctypes.byref(n_part), _s()) == 0
    torch.cuda.synchronize()
    parts = part[:n_part.value * WG_PART].view(n_part.value, WG_PART).double().cpu().numpy()
    total = parts.sum(0)
    dzu, g = ref.unpool(_np(dp), code.cpu().numpy(), float(ks))
    dw_ref, dw_mag = ref.wgrad(_np(a), dzu)
    db_ref, db_mag = ref.bias_grad(g)
    P = tiles_fwd(H, W) * B // 2
    grid = c_grid(P, s)
    n = -(-P // grid)
    d_w = 128 * min(WG_GROUP, n) + -(-n // WG_GROUP) + grid        # + grid: the float64 sum of fp32 partials
    d_b = 1 + -(-n // 2) + 2 + 16 + grid
    err_w = np.abs(total[:WG_PART - 64] - dw_ref.reshape(-1))
    err_b = np.abs(total[WG_PART - 64:] - db_ref)
    assert (err_w <= d_w * U * dw_mag.reshape(-1)).all(), (rate, float(scale.value), float(ks), float(err_w.max()))
    assert (err_b <= d_b * U * db_mag).all(), (rate, float(scale.value), float(ks), float(err_b.max()))


def _adjoint_model(rate):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="conv2_dropout_adjoint")
    m.add(layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)))
    m.add(layers.Conv2D(64, (3, 3), activation="relu"))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(rate))
    m.add(layers.Flatten())
    m.add(layers.Dense(10))
    return m


SCALE_ARG = {"tfy_conv3x3_c32_wgrad_unpool_ov": 3, "tfy_conv3x3_c32_wgrad_unpool_deferred": 3,
             "tfy_conv3x3_c32_wgrad_unpool": 3, "tfy_conv3x3_c32_dgrad_unpool_reduce": 2,
             "tfy_conv3x3_c32_dgrad_unpool": 2, "tfy_pool_drop_relu_bwd": 3}


class _ScaleRecorder:
    """Forwards every call to the kernel library and records the scale argument of the conv2 backward launches."""

    def __init__(self, lib):
        self._lib = lib
        self.scales = []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in SCALE_ARG:
            return fn

        def call(*args):
            self.scales.append((name, args[SCALE_ARG[name]]))
            return fn(*args)
        return call


@pytest.mark.parametrize("unfused", [False, True])
@pytest.mark.parametrize("rate", [0.25, 0.3, 0.9])
def test_engine_passes_the_forward_keep_scale_to_the_conv2_backward(monkeypatch, lib, rate, unfused):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    if unfused:
        monkeypatch.setenv("TFY_NO_UNPOOL_FUSION", "1")
    else:
        monkeypatch.delenv("TFY_NO_UNPOOL_FUSION", raising=False)
    torch.manual_seed(3)
    m = _adjoint_model(rate)
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=keras.optimizers.SGD(0.01),
              metrics=["accuracy"])
    g = torch.Generator().manual_seed(5)
    x = torch.rand(64, 28, 28, 1, generator=g)
    y = torch.randint(0, 10, (64,), generator=g)
    m.fit(x, y, batch_size=32, epochs=1, shuffle=False, verbose=0)
    eng = m._engine
    assert isinstance(eng, FastSequentialEngine)
    assert FastSequentialEngine._tc_conv(eng.plan[1], 32)
    sx = eng._static_x if eng._static_x is not None else x[:32].cuda()
    sy = eng._static_y if eng._static_y is not None else y[:32].cuda()
    rec = _ScaleRecorder(eng.lib)
    eng.lib = rec
    try:
        with torch.cuda.stream(eng.stream):
            eng._forward_backward(sx, sy)
        torch.cuda.synchronize()
    finally:
        eng.lib = rec._lib
    names = [n for n, _ in rec.scales]
    assert names == (["tfy_pool_drop_relu_bwd"] if unfused
                     else ["tfy_conv3x3_c32_wgrad_unpool_deferred", "tfy_conv3x3_c32_dgrad_unpool_reduce"]), names
    _, ks = keep_scale_of(rate)
    assert np.float32(fastpath.keep_scale(lib, rate)) == ks
    for name, sc in rec.scales:
        v = sc.value if isinstance(sc, ctypes.c_float) else sc
        assert np.float32(v) == ks, (name, v, float(ks))


# ---------------------------------------------------------------------------------------------- bit record
def _sha(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def bwd_digests(lib):
    """SHA-256 of the conv2 backward kernels' outputs at batch 128, 26 x 26 (the recorded fixture).  Inputs are seeded
    on the CPU as in test_gpu_conv2_pipeline._inputs, plus a materialised dz; the code bytes come from the forward at
    rate 0.25 (seed 1234, step 0) and the un-pool scale is its keep factor 4/3.  A change that deliberately alters a
    summation order re-records these and says so."""
    B, H, W = 128, 26, 26
    g = torch.Generator().manual_seed(11)
    a = torch.randn(B, H, W, 32, generator=g).relu().to(torch.bfloat16).cuda()
    w = (torch.randn(64, 3, 3, 32, generator=g) * 0.06).to(torch.bfloat16).cuda()
    bias = (torch.randn(64, generator=g) * 0.1).to(torch.bfloat16).cuda()
    dp = (torch.randn(B, 12, 12, 64, generator=g) * 0.5).to(torch.bfloat16).cuda()
    dz = (torch.randn(B, 24, 24, 64, generator=g) * 0.5).to(torch.bfloat16).cuda()
    pooled = torch.empty(B, 12, 12, 64, dtype=torch.bfloat16, device="cuda")
    code = torch.empty(B, 12, 12, 64, dtype=torch.uint8, device="cuda")
    assert lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(),
                                        code.data_ptr(), B, H, W, 0.25, 1234, None, _s()) == 0
    scale = ctypes.c_float(256.0 / 192.0)
    n_scr = int(lib.tfy_conv3x3_c32_wgrad_scratch_elems())
    part = torch.zeros(n_scr, dtype=torch.float32, device="cuda")
    sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
    out = {}

    dx = torch.empty(B, H, W, 32, dtype=torch.bfloat16, device="cuda")
    assert lib.tfy_conv3x3_c32_dgrad(dz.data_ptr(), w.data_ptr(), a.data_ptr(), dx.data_ptr(), B, H, W, _s()) == 0
    out["dgrad_gated_dx"] = _sha(dx)

    n_part = ctypes.c_int(0)
    dw = torch.empty(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
    db = torch.empty(64, dtype=torch.bfloat16, device="cuda")
    dx = torch.empty(B, H, W, 32, dtype=torch.bfloat16, device="cuda")
    assert lib.tfy_conv3x3_c32_wgrad_unpool_deferred(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                     part.data_ptr(), B, H, W, None, ctypes.byref(n_part), _s()) == 0
    assert lib.tfy_conv3x3_c32_dgrad_unpool_reduce(dp.data_ptr(), code.data_ptr(), scale, w.data_ptr(), a.data_ptr(),
                                                   dx.data_ptr(), B, H, W, part.data_ptr(), n_part.value,
                                                   dw.data_ptr(), db.data_ptr(), _s()) == 0
    out["deferred_dx"], out["deferred_dw"], out["deferred_db"] = _sha(dx), _sha(dw), _sha(db)

    dw = torch.empty(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
    db = torch.empty(64, dtype=torch.bfloat16, device="cuda")
    assert lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale, part.data_ptr(),
                                            dw.data_ptr(), db.data_ptr(), sync.data_ptr(), B, H, W, _s()) == 0
    out["wgrad_unpool_dw"], out["wgrad_unpool_db"] = _sha(dw), _sha(db)

    dw = torch.empty(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
    assert lib.tfy_conv3x3_c32_wgrad(a.data_ptr(), dz.data_ptr(), part.data_ptr(), dw.data_ptr(), sync.data_ptr(), B,
                                     H, W, _s()) == 0
    out["wgrad_dw"] = _sha(dw)
    torch.cuda.synchronize()
    return out


def test_backward_bit_identical_to_recorded_digest(lib):
    with open(GOLDEN_BWD) as f:
        want = json.load(f)
    got = bwd_digests(lib)
    assert got == {k: want[k] for k in got}


def test_configurations_cover_every_schedule_case():
    s = _sms()
    cfg = configs(s)
    for tiles in (tiles_fwd, tiles_dgrad):
        counts = {tiles(h, w) * b // 2 for h, w, b in cfg}
        assert min(counts) <= (1 if tiles is tiles_fwd else 4)
        assert any(1 < c < s for c in counts) and s in counts and max(counts) > 2 * WG_RING * s
        if tiles is tiles_fwd or any((s + 1) % ((i + 1) * (j + 1)) == 0 for i in range(1, 40) for j in range(i, 200)):
            assert s + 1 in counts
    assert {c[:2] for c in cfg} >= set(SHAPES)
