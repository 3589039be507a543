"""The Dense-layer kernels -- tfy_gemm_bf16 (bf16 output, split-K slabs, the fused split-K epilogue),
tfy_splitk_sum_f32, tfy_gemm2_bf16, tfy_dense_bwd, tfy_dense_head_fused(_weighted) and tfy_ps_gather_gemm -- against
the float64 reference (tests/dense_reference.py), called directly through their ctypes declarations, at the shapes
where their branches change.

Exact tier.  Operands are small integers (bf16 numbers), chosen so that every output's sum of |terms| stays below
2^22 (the generator asserts it).  Every product is then exact in fp32 and every partial sum an integer fp32 holds
exactly, so the accumulator is the float64 sum whatever the order of the additions: fp32 outputs (split-K slabs,
summed slabs) must equal the reference bit for bit, and bf16 outputs must equal its round-to-nearest-even rounding
bit for bit (outputs above 256 are full of ties, so this pins the rounding mode too).  This rests on one hardware
assumption, not measured here: wgmma's fp32 accumulation is exact when every value involved is an integer below 2^22.
If this tier ever fails, run the same inputs through torch.mm (cuBLAS on the same tensor cores) before blaming a
kernel.

Bound tier.  Gaussian operands at realistic scales.  EPS32 = 2^-24 and U_BF16 = 2^-8 are the fp32 and bf16 unit
roundoffs.  A sum whose terms each pass through at most d fp32 additions is within d EPS32 sum|terms| of the exact sum,
and a bf16 output of such a value v is within U_BF16 |v| + 2 d EPS32 sum|terms|.  As a MODEL of the tensor core (not a
measurement: wgmma's internal addition order is not documented), a wgmma K accumulation counts as a sequential fp32
sum of its K terms.  So d per kernel:

* tfy_gemm_bf16 / tfy_gemm2_bf16: K + 1 (the bias); a split-K slab: the columns of its slice; the slab sum: + S.
* tfy_gemm_bf16_splitk_fused: not in the bound tier (exact tier only: it is the MNIST forward).
* tfy_dense_bwd: dW sums over the batch, d = B; dx over the units, d = U.
* tfy_ps_gather_gemm: each 64-column chunk is one wgmma chain added into a shared-memory accumulator: Kp + chunks + 1.
* tfy_dense_head_fused: logits are 16-lane FMA chains of K / 16 terms, a 4-step shuffle tree and the bias: every logit
  is within e_v = (K / 16 + 5) EPS32 sum|h w| + |b|.  That moves ln p by at most 2 e_v, so p is within
  4 e_v + (Kx + C + 3) EPS32 relative, with Kx = 4 + 2.2 max|v - max| the __expf bound of test_gpu_nn_kernels.py;
  dlogits = w (p - onehot) / B add 2 EPS32 |p - onehot| / B and two roundings of the weight product.  dW2 and db2 are
  16-row FMA chains per CTA, then the CTA slabs summed in CTA order: d = 16 + G (G = ceil(B / 16) CTAs), plus the
  dlogits errors carried through |h|.  dh is a 16-class FMA chain and the gate scale: d = 17, plus the dlogits errors
  carried through |W2|.  db1 sums at most 16 rows per thread, one shared atomic and the G slabs: d = 17 + G, plus the
  dh errors.  The loss row is within (Kx + C + 8) EPS32 (1 + |max| + |ln se| + |v_label|) + 2^-21.41 (__logf's
  absolute error) + 4 e_v, and the rows are summed by a 5-step shuffle tree, 8 warps, G slabs and 1 / B: d = 15 + G.
  Hit counts are exact wherever the float64 gap between the two largest logits exceeds 4 e_v (twice the bound on their
  difference).

Every output sits between 0xA5 guard bytes and is pre-filled with them; the columns of a row pitch wider than N are
guards too.  Every kernel runs three times on the same inputs and must give the same bits; the head and the fused
split-K path are also captured in a CUDA graph and replayed.  Every documented refusal (-2, -3, -8) is checked by its
return code; none of them launches a kernel.
"""
import ctypes

import numpy as np
import pytest
import torch

import dense_reference as ref
import nn_reference

pytestmark = pytest.mark.gpu

EPS32, U_BF16 = ref.EPS32, ref.U_BF16
GUARD = 64
RUNS = 3
SEED, STEP = 20261017, 9
BF16, F32 = torch.bfloat16, torch.float32
RATIOS = {}                  # kernel -> largest |error| / bound seen in the bound tier (printed at the end)


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.keras import fastpath  # noqa: F401
    from tf_yarn_b200.ops import gemm, native  # noqa: F401
    return native.load()


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    h = nn_reference.host_lib(str(tmp_path_factory.mktemp("denseref")))
    assert h is not None, "the host build of the dropout generator needs g++ and the CUDA headers"
    return h


@pytest.fixture(scope="module")
def hp():
    from tf_yarn_b200.ops import native
    h = native.OptHyper(1.0, 0.0, 0.0, 0.0, 0.0, 1.0, STEP, 0, 0, 0)
    return torch.frombuffer(bytearray(bytes(h)), dtype=torch.uint8).cuda()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if RATIOS:
        print("\nlargest error / bound in the bound tier on " + torch.cuda.get_device_name(0) + ": " +
              ", ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def _s():
    return torch.cuda.current_stream().cuda_stream


class Out:
    """Device output between guard bytes, pre-filled with the same byte so that an element the kernel skips shows.
    ``cols``: the columns [cols, last dim) of a row pitch wider than the output are guards too."""

    def __init__(self, shape, dtype, cols=None):
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        self.full = torch.full((2 * GUARD + n,), 0xA5, dtype=torch.uint8, device="cuda")
        self.t = self.full[GUARD:GUARD + n].view(dtype).view(shape)
        self.cols = cols

    def ptr(self):
        return self.t.data_ptr()

    def get(self):
        torch.cuda.synchronize()
        assert bool((self.full[:GUARD] == 0xA5).all()) and bool((self.full[-GUARD:] == 0xA5).all()), "guard written"
        if self.cols is not None:
            assert bool((self.t[..., self.cols:].contiguous().view(torch.uint8) == 0xA5).all()), "pitch gap written"
            return self.t[..., :self.cols].clone()
        return self.t.clone()


def _dev(x, dtype=BF16, ld=None, fill=float("nan")):
    """float64 array [rows, cols] -> device tensor of row pitch ld (pad columns = fill), and the float64 values the
    device holds (after rounding to dtype)."""
    x = np.asarray(x, np.float64)
    t = torch.from_numpy(x).to(dtype)
    if ld is not None and ld != x.shape[-1]:
        full = torch.full((x.shape[0], ld), fill, dtype=dtype)
        full[:, :x.shape[1]] = t
        return full.cuda(), t.double().numpy()
    return t.cuda(), t.double().numpy()


def _np(t):
    return t.double().cpu().numpy()


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu()


def _exact(got, want, what):
    got = _np(got)
    bad = got != want
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:3].tolist(), got[bad][:3], want[bad][:3])


def _bound(got, want, e, what, bf16=True):
    """|got - want| <= U_BF16 |want| + 2 e for a bf16 output, <= e for an fp32 one (module docstring)."""
    got = _np(got)
    tol = (U_BF16 * np.abs(want) + 2.0 * e if bf16 else e) + 1e-30
    err = np.abs(got - want)
    bad = ~(err <= tol)
    assert not bad.any(), (what, int(bad.sum()), float(err[bad].max()), float(tol[bad].min()))
    kernel = what.split(" ")[0]
    RATIOS[kernel] = max(RATIOS.get(kernel, 0.0), float((err / tol).max(initial=0.0)))


def _repeat(launch, outs, what):
    """Launches twice more; every output must keep its bits."""
    first = [_bits(o.get()) for o in outs]
    for run in range(1, RUNS):
        launch()
        for o, f in zip(outs, first):
            assert torch.equal(_bits(o.get()), f), f"{what}: run {run} differs"


# ---------------------------------------------------------------------------------------------- tfy_gemm_bf16, bf16 out
GEMM_SHAPES = [(1, 8, 8), (7, 10, 56), (128, 128, 64), (129, 136, 72), (100, 72, 200), (300, 72, 264), (256, 384, 512),
               (1000, 10, 128), (128, 9216, 128), (128, 128, 9216), (512, 256, 1024), (512, 1024, 1680)]
# (bias, relu, operand pitch pad, output pitch pad): pitch pads are in elements; a pad of 3 sends the epilogue down
# its scalar path
GEMM_CONFIGS = [(False, False, 0, 0), (True, True, 8, 8), (True, False, 24, 3)]


def _operands(rng, tier, M, N, K, a_lo=-15):
    if tier == "exact":
        a, b, bias = ref.integers(rng, (M, K), a_lo), ref.integers(rng, (N, K)), ref.integers(rng, (N,))
        ref.assert_exact(a, b, bias)
        return a, b, bias
    return rng.standard_normal((M, K)) * 0.5, rng.standard_normal((N, K)) * 0.5, rng.standard_normal(N)


@pytest.mark.parametrize("tier", ["exact", "bound"])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_bf16_matches_reference(lib, M, N, K, tier):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    a, b, bias = _operands(rng, tier, M, N, K)
    for has_bias, relu, pad, cpad in GEMM_CONFIGS:
        lda, ldb, ldc = K + pad, K + 2 * pad, N + cpad
        ad, a64 = _dev(a, ld=lda)
        bd, b64 = _dev(b, ld=ldb)
        biasd, bias64 = _dev(bias[None])
        want, mag = ref.gemm(a64, b64, bias64[0] if has_bias else None, relu)
        c = Out((M, ldc), BF16, cols=N)

        def launch():
            assert lib.tfy_gemm_bf16(ad.data_ptr(), bd.data_ptr(), c.ptr(), None,
                                     biasd.data_ptr() if has_bias else None, M, N, K, lda, ldb, ldc, int(relu), 1,
                                     _s()) == 0
        launch()
        what = f"tfy_gemm_bf16 {tier} {(M, N, K)} bias={has_bias} relu={relu} ld={(lda, ldb, ldc)}"
        if tier == "exact":
            _exact(c.get(), ref.bf16_round(want), what)
        else:
            _bound(c.get(), want, (K + 1) * EPS32 * mag, what)
        _repeat(launch, [c], what)


# ---------------------------------------------------------------------------------------------- split-K slabs
@pytest.mark.parametrize("M,N,K,split", [(128, 128, 9216, 24), (128, 128, 9224, 24), (256, 512, 2000, 5),
                                         (100, 72, 4096, 7), (1, 8, 2048, 32), (64, 64, 128, 8), (128, 128, 9216, 1),
                                         (130, 136, 640, 3)])
def test_gemm_splitk_slabs_are_exact(lib, M, N, K, split):
    """C = nullptr: slab z holds the exact partial product over the columns of K-slice z; the slab sum is exact too."""
    rng = np.random.default_rng(M + N + K + split)
    a, b, _ = _operands(rng, "exact", M, N, K, a_lo=0)
    S = int(lib.tfy_gemm_bf16_splitk_slabs(K, split))
    assert S == ref.slab_count(K, split)
    ldc = N + (4 if M == 130 else 0)                  # a slab row pitch wider than N: its gap columns are guards
    ad, a64 = _dev(a, ld=K + 8)
    bd, b64 = _dev(b)
    want = ref.splitk_slabs(a64, b64, split)
    slabs = Out((S, M, ldc), F32, cols=N)

    def launch():
        assert lib.tfy_gemm_bf16(ad.data_ptr(), bd.data_ptr(), None, slabs.ptr(), None, M, N, K, K + 8, K, ldc, 0,
                                 split, _s()) == 0
    launch()
    what = f"split-K slabs {(M, N, K, split)}"
    _exact(slabs.get(), want, what)
    _repeat(launch, [slabs], what)
    if ldc == N:
        out = Out((M, N), F32)
        assert lib.tfy_splitk_sum_f32(slabs.ptr(), out.ptr(), S, M * N, M * N, _s()) == 0
        _exact(out.get(), want.sum(0), what + " summed")


@pytest.mark.parametrize("S,M,N", [(1, 7, 4), (3, 128, 128), (24, 128, 128), (7, 100, 72), (21, 129, 136)])
def test_splitk_sum_is_left_to_right_in_slab_order(lib, S, M, N):
    """tfy_splitk_sum_f32 on Gaussian slabs of very different scales: bit for bit the fp32 sum in slab order."""
    g = torch.Generator(device="cuda").manual_seed(S * 100 + M)
    scale = torch.logspace(-3, 3, S, device="cuda")[torch.randperm(S, device="cuda", generator=g)]
    slabs = torch.randn(S, M, N, device="cuda", generator=g) * scale[:, None, None]
    want = ref.sum_slabs_f32(slabs.cpu().numpy()).astype(np.float64)
    out = Out((M, N), F32)

    def launch():
        assert lib.tfy_splitk_sum_f32(slabs.data_ptr(), out.ptr(), S, M * N, M * N, _s()) == 0
    launch()
    _exact(out.get(), want, f"tfy_splitk_sum_f32 {(S, M, N)}")
    _repeat(launch, [out], "tfy_splitk_sum_f32")


@pytest.mark.parametrize("M,N,K", [(128, 128, 9216), (256, 384, 512), (512, 256, 1024), (512, 1024, 1680),
                                   (300, 72, 264)])
def test_gemm_bf16_python_split_k_and_auto(lib, M, N, K):
    """ops.gemm.gemm_bf16: split_k = 4 equals its own slabs summed left to right, and (exact tier) the product; the
    default path equals the direct kernel of its choice bit for bit."""
    from tf_yarn_b200.ops.gemm import GEMM2_MIN_DIM, gemm_bf16
    rng = np.random.default_rng(K)
    for tier in ("exact", "bound"):
        a, b, bias = _operands(rng, tier, M, N, K)
        ad, a64 = _dev(a)
        bd, b64 = _dev(b)
        biasd, bias64 = _dev(bias[None])
        got = gemm_bf16(ad, bd, split_k=4)
        S = int(lib.tfy_gemm_bf16_splitk_slabs(K, 4))
        slabs = Out((S, M, N), F32)
        assert lib.tfy_gemm_bf16(ad.data_ptr(), bd.data_ptr(), None, slabs.ptr(), None, M, N, K, K, K, N, 0, 4,
                                 _s()) == 0
        _exact(got, ref.sum_slabs_f32(slabs.get().cpu().numpy()).astype(np.float64), f"gemm_bf16 split 4 {tier}")
        want, mag = ref.gemm(a64, b64)
        if tier == "exact":
            _exact(got, want, "gemm_bf16 split 4")
        else:
            per = max(hi - lo for lo, hi in ref.k_slices(K, 4))
            _bound(got, want, (per + S) * EPS32 * mag, f"tfy_splitk_sum_f32 gemm {(M, N, K)}", bf16=False)
        out = gemm_bf16(ad, bd, bias=biasd[0], relu=True)
        direct = Out((M, N), BF16)
        fn = lib.tfy_gemm2_bf16 if (M >= GEMM2_MIN_DIM and N >= GEMM2_MIN_DIM) else None
        if fn is not None:
            assert fn(ad.data_ptr(), bd.data_ptr(), direct.ptr(), biasd.data_ptr(), M, N, K, K, K, N, 1, _s()) == 0
        else:
            assert lib.tfy_gemm_bf16(ad.data_ptr(), bd.data_ptr(), direct.ptr(), None, biasd.data_ptr(), M, N, K, K, K,
                                     N, 1, 1, _s()) == 0
        assert torch.equal(_bits(out), _bits(direct.get())), "gemm_bf16 default path"
        if tier == "exact":
            _exact(out, ref.bf16_round(ref.gemm(a64, b64, bias64[0], True)[0]), "gemm_bf16 default path")


def test_gemm_bf16_output_views(lib):
    """An output view 4 columns into a wider buffer: with a row pitch that is a multiple of 8 the 16-byte stores
    cannot take it and the launcher refuses it (-3); with an odd pitch the scalar epilogue writes it exactly."""
    from tf_yarn_b200.ops.gemm import gemm_bf16
    rng = np.random.default_rng(5)
    M, N, K = 100, 72, 200
    a, b, _ = _operands(rng, "exact", M, N, K)
    ad, a64 = _dev(a)
    bd, b64 = _dev(b)
    buf = torch.zeros(M, 136, dtype=BF16, device="cuda")
    with pytest.raises(RuntimeError, match="code -3"):
        gemm_bf16(ad, bd, out=buf[:, 4:4 + N])
    buf = torch.full((M, 139), 7.0, dtype=BF16, device="cuda")
    gemm_bf16(ad, bd, out=buf[:, 4:4 + N])
    torch.cuda.synchronize()
    _exact(buf[:, 4:4 + N], ref.bf16_round(ref.gemm(a64, b64)[0]), "gemm_bf16 into an odd-pitch view")
    assert bool((buf[:, :4] == 7).all()) and bool((buf[:, 4 + N:] == 7).all())


# ---------------------------------------------------------------------------------------------- fused split-K epilogue
@pytest.mark.parametrize("rate", [0.0, 0.25, 0.5])
@pytest.mark.parametrize("M,N,K,split", [(128, 128, 9216, 24), (200, 256, 4096, 16), (64, 136, 2048, 8)])
def test_gemm_splitk_fused_is_exact(lib, host, hp, M, N, K, split, rate):
    tiles = -(-M // 128) * -(-N // 128)
    S = int(lib.tfy_gemm_bf16_splitk_slabs(K, split))
    assert tiles * S <= torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(M + K + int(rate * 8))
    a, b, bias = _operands(rng, "exact", M, N, K, a_lo=0)
    ad, a64 = _dev(a, ld=K + 16)
    bd, b64 = _dev(b, ld=K + 8)
    biasd, bias64 = _dev(bias[None])
    exact = a64 @ b64.T
    u = nn_reference.uniform(host, SEED, STEP, M * N) if rate > 0 else None
    counters = torch.zeros(2 * tiles, dtype=torch.int32, device="cuda")
    for relu in (False, True):
        for has_mask in (False, True):
            for has_bias in (False, True):
                if has_bias != (relu or has_mask):
                    continue                         # bias with ReLU or mask, none without: 2 x 2 configurations
                want_y, want_m = ref.fused_epilogue(exact, bias64[0] if has_bias else None, relu, rate, u)
                acc = Out((S, M, N), F32)
                y = Out((M, N), BF16)
                m = Out((M, N), torch.uint8) if has_mask else None

                def launch():
                    assert lib.tfy_gemm_bf16_splitk_fused(
                        ad.data_ptr(), bd.data_ptr(), acc.ptr(), counters.data_ptr(),
                        biasd.data_ptr() if has_bias else None, y.ptr(), m.ptr() if m else None, M, N, K, K + 16,
                        K + 8, int(relu), ctypes.c_float(rate), SEED, hp.data_ptr(), split, _s()) == 0
                what = f"fused split-K {(M, N, K, split)} rate={rate} relu={relu} mask={has_mask}"
                outs = [y, acc] + ([m] if m else [])
                launch()
                _exact(y.get(), want_y, what)
                _exact(acc.get(), ref.splitk_slabs(a64, b64, split), what + " slabs")
                if m:
                    assert np.array_equal(m.get().cpu().numpy(), want_m), what + " mask"
                assert int(counters.abs().sum()) == 0, what + ": counters not re-armed"
                launch()
                assert int(counters.abs().sum()) == 0, what + ": counters not re-armed (second launch)"
                _repeat(launch, outs, what)
                eager = [_bits(o.get()) for o in outs]
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    launch()
                for o in outs:
                    o.t.fill_(0)
                for rep in range(3):
                    graph.replay()
                    for o, e in zip(outs, eager):
                        assert torch.equal(_bits(o.get()), e), f"{what}: graph replay {rep}"
                    assert int(counters.abs().sum()) == 0, f"{what}: counters after replay {rep}"


# ---------------------------------------------------------------------------------------------- tfy_gemm2_bf16
@pytest.mark.parametrize("tier", ["exact", "bound"])
@pytest.mark.parametrize("M,N,K,ldc", [(512, 512, 64, 512), (256, 256, 64, 264), (512, 768, 512, 768),
                                       (1000, 520, 264, 520), (4096, 1024, 128, 1024), (130, 304, 72, 312),
                                       (4096, 2048, 256, 2048), (600, 1001, 64, 1008), (512, 520, 8, 528)])
def test_gemm2_bf16_matches_reference(lib, M, N, K, ldc, tier):
    rng = np.random.default_rng(M + 3 * N + 7 * K)
    a, b, bias = _operands(rng, tier, M, N, K)
    for has_bias, relu, pad in [(False, False, 0), (True, True, 8)]:
        lda, ldb = K + pad, K + 3 * pad
        ad, a64 = _dev(a, ld=lda)
        bd, b64 = _dev(b, ld=ldb)
        biasd, bias64 = _dev(bias[None])
        want, mag = ref.gemm(a64, b64, bias64[0] if has_bias else None, relu)
        c = Out((M, ldc), BF16, cols=N)

        def launch():
            assert lib.tfy_gemm2_bf16(ad.data_ptr(), bd.data_ptr(), c.ptr(), biasd.data_ptr() if has_bias else None,
                                      M, N, K, lda, ldb, ldc, int(relu), _s()) == 0
        launch()
        what = f"tfy_gemm2_bf16 {tier} {(M, N, K, ldc)} bias={has_bias} relu={relu}"
        if tier == "exact":
            _exact(c.get(), ref.bf16_round(want), what)
        else:
            _bound(c.get(), want, (K + 1) * EPS32 * mag, what)
        _repeat(launch, [c], what)


# ---------------------------------------------------------------------------------------------- tfy_dense_bwd
@pytest.mark.parametrize("tier", ["exact", "bound"])
@pytest.mark.parametrize("B,U,I", [
    # single-shot kernel (B, U <= 128)
    (128, 128, 9216), (1, 8, 8), (5, 8, 64), (16, 8, 64), (127, 64, 72), (64, 128, 1000), (100, 72, 200),
    # tiled kernel
    (129, 8, 64), (128, 136, 264), (300, 136, 264), (1000, 256, 72), (512, 1024, 1680), (512, 256, 1024)])
def test_dense_bwd_matches_reference(lib, B, U, I, tier):
    rng = np.random.default_rng(B * 3 + U * 5 + I)
    if tier == "exact":
        dh, x, w = ref.integers(rng, (B, U)), ref.integers(rng, (B, I), 0), ref.integers(rng, (U, I))
        ref.assert_exact(dh.T, x.T)
        ref.assert_exact(dh, w.T)
    else:
        dh, x, w = rng.standard_normal((B, U)) * 0.5, np.maximum(rng.standard_normal((B, I)), 0), \
            rng.standard_normal((U, I)) * 0.05
    dhd, dh64 = _dev(dh)
    xd, x64 = _dev(x)
    wd, w64 = _dev(w)
    want_dw, want_dx, mag_dw, mag_dx = ref.dense_bwd(dh64, x64, w64)
    for want_dx_out in (True, False):
        dw = Out((U, I), BF16)
        dx = Out((B, I), BF16) if want_dx_out else None

        def launch():
            assert lib.tfy_dense_bwd(dhd.data_ptr(), xd.data_ptr(), wd.data_ptr(), dw.ptr(),
                                     dx.ptr() if dx else None, B, U, I, _s()) == 0
        launch()
        what = f"tfy_dense_bwd {tier} {(B, U, I)} dx={want_dx_out}"
        if tier == "exact":
            _exact(dw.get(), ref.bf16_round(want_dw), what + " dW")
            if dx:
                _exact(dx.get(), ref.bf16_round(want_dx), what + " dx")
        else:
            _bound(dw.get(), want_dw, B * EPS32 * mag_dw, what + " dW")
            if dx:
                _bound(dx.get(), want_dx, U * EPS32 * mag_dx, what + " dx")
        _repeat(launch, [dw] + ([dx] if dx else []), what)


# ---------------------------------------------------------------------------------------------- fused classifier head
def _head_inputs(rng, B, K, C):
    h = np.maximum(rng.standard_normal((B, K)), 0)
    w2 = rng.standard_normal((C, K)) * (2.0 / np.sqrt(K))
    b2 = rng.standard_normal(C) * 0.1
    labels = rng.integers(0, C, B)
    return h, w2, b2, labels


def _head_bounds(r, h, w2, b2, C, G):
    """Error bounds of every head output (module docstring) from the float64 reference r."""
    B, K = h.shape
    e_v = (K / 16 + 5) * EPS32 * (np.abs(h) @ np.abs(w2).T + np.abs(b2))
    ev = e_v.max(1)
    v = r["v"]
    mx = v.max(1, keepdims=True)
    p = np.exp(v - mx)
    se = p.sum(1, keepdims=True)
    p /= se
    Kx = 4 + 2.2 * np.abs(v - mx).max(1)
    lab = np.asarray(r["labels"])
    valid = (lab >= 0) & (lab < C)
    onehot = np.zeros_like(p)
    onehot[np.arange(B)[valid], lab[valid]] = 1.0
    wr = r["wr"][:, None]
    e_d = wr * ((4 * ev + (Kx + C + 3) * EPS32)[:, None] * p + 2 * EPS32 * np.abs(p - onehot)) / B \
        + 2 * EPS32 * np.abs(r["d"])
    ad = np.abs(r["d"])
    e_dw2 = (16 + G) * EPS32 * (ad.T @ np.abs(h)) + e_d.T @ np.abs(h)
    e_db2 = (16 + G) * EPS32 * ad.sum(0) + e_d.sum(0)
    e_dh = r["gate"] * (17 * EPS32 * (ad @ np.abs(w2)) + e_d @ np.abs(w2))
    e_db1 = (17 + G) * EPS32 * np.abs(r["dh"]).sum(0) + e_dh.sum(0)
    lab = np.clip(lab, 0, C - 1)
    e_row = (Kx + C + 8) * EPS32 * (1 + np.abs(mx[:, 0]) + np.abs(np.log(se[:, 0])) + np.abs(v[np.arange(B), lab])) \
        + 2 ** -21.41 + 4 * ev
    e_loss = ((r["wr"] * e_row).sum() + (15 + G) * EPS32 * np.abs(r["wr"] * r["rows"]).sum()) / B \
        + EPS32 * abs(r["loss"])
    top = np.sort(v, 1)
    gap = top[:, -1] - top[:, -2] if C > 1 else np.full(B, np.inf)
    return dict(dw2=e_dw2, db2=e_db2, dh=e_dh, db1=e_db1, loss=e_loss, ambiguous=gap <= 4 * ev)


HEAD_SHAPES = [(B, K, C) for K in (128, 256, 512) for C in (1, 2, 10, 16) for B in (1, 15, 16, 17, 128, 1000)] + \
    [(100, 256, 16), (37, 512, 3)]


@pytest.mark.parametrize("B,K,C", HEAD_SHAPES)
def test_dense_head_fused_matches_reference(lib, B, K, C):
    rng = np.random.default_rng(B * 31 + K + C)
    h, w2, b2, labels = _head_inputs(rng, B, K, C)
    hd, h64 = _dev(h)
    w2d, w264 = _dev(w2)
    b2d, b264 = _dev(b2[None])
    G = -(-B // 16)
    scratch = torch.zeros(int(lib.tfy_dense_head_scratch_elems(K, C, B)), device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    mask_bytes = rng.integers(0, 256, (B, K)).astype(np.uint8)          # high bits set: only bit 0 may count
    scale1 = 1.25
    sw = (rng.random(B) + 0.5).astype(np.float32).astype(np.float64)
    cw = (rng.random(C) * 1.5 + 0.5).astype(np.float32).astype(np.float64)
    bad_label = labels.copy()
    bad_label[B // 2] = C if B % 2 else -1
    # (weighted, mask, sample weights, class weights, labels)
    cases = [(False, None, None, None, labels), (False, mask_bytes, None, None, labels),
             (True, mask_bytes, sw, None, labels), (True, None, None, cw, labels), (True, mask_bytes, sw, cw, bad_label)]
    for weighted, mask, s_w, c_w, lab in cases:
        r = ref.dense_head(h64, w264, b264[0], lab, mask, scale1, s_w, c_w)
        r["labels"] = lab
        e = _head_bounds(r, h64, w264, b264[0], C, G)
        labd = torch.from_numpy(lab).cuda()
        maskd = torch.from_numpy(mask).cuda() if mask is not None else None
        swd = torch.from_numpy(s_w).float().cuda() if s_w is not None else None
        cwd = torch.from_numpy(c_w).float().cuda() if c_w is not None else None
        pre = [5.0, 7.0, 3.0, 11.0][:4 if weighted else 2]
        stats = torch.tensor(pre, device="cuda")
        loss, dw2, db2, dh, db1 = Out((1,), F32), Out((C, K), BF16), Out((C,), BF16), Out((B, K), BF16), Out((K,), BF16)
        outs = [loss, dw2, db2, dh, db1]

        def launch():
            args = [hd.data_ptr(), w2d.data_ptr(), b2d.data_ptr(), labd.data_ptr(),
                    maskd.data_ptr() if maskd is not None else None, ctypes.c_float(scale1), loss.ptr(), None,
                    stats.data_ptr(), dw2.ptr(), db2.ptr(), dh.ptr(), db1.ptr(), scratch.data_ptr(),
                    counter.data_ptr(), B, K, C]
            if weighted:
                rc = lib.tfy_dense_head_fused_weighted(*args, swd.data_ptr() if swd is not None else None,
                                                       cwd.data_ptr() if cwd is not None else None, _s())
            else:
                rc = lib.tfy_dense_head_fused(*args, _s())
            assert rc == 0
        what = f"tfy_dense_head_fused {(B, K, C)} weighted={weighted} mask={mask is not None} " \
               f"sw={s_w is not None} cw={c_w is not None}"
        launch()
        got = [o.get() for o in outs]
        assert float(abs(float(got[0]) - r["loss"])) <= e["loss"], (what, float(got[0]), r["loss"], e["loss"])
        RATIOS["tfy_dense_head_fused"] = max(RATIOS.get("tfy_dense_head_fused", 0.0),
                                             abs(float(got[0]) - r["loss"]) / e["loss"])
        for o, name in zip(got[1:], ("dw2", "db2", "dh", "db1")):
            _bound(o, r[name], e[name], f"{what} {name}")
        amb = e["ambiguous"]
        st = stats.cpu().numpy().astype(np.float64)
        assert st[1] == pre[1] + B, (what, st)
        hits_ref = r["stats"][0]
        assert abs(st[0] - pre[0] - hits_ref) <= amb.sum(), (what, st[0] - pre[0], hits_ref, int(amb.sum()))
        if weighted:
            w_amb = r["wr"][amb].sum()
            e_w = (13 + G + 2) * EPS32 * (r["wr"].sum() + pre[3])
            assert abs(st[2] - pre[2] - r["stats"][2]) <= w_amb + e_w + EPS32 * pre[2], (what, st, r["stats"])
            assert abs(st[3] - pre[3] - r["stats"][3]) <= e_w, (what, st, r["stats"])
        assert bool((scratch == 0).all()) and int(counter.item()) == 0, what + ": scratch / counter not cleared"
        _repeat(launch, outs, what)
        assert bool((scratch == 0).all()) and int(counter.item()) == 0, what + ": scratch / counter not cleared"


@pytest.mark.parametrize("B,K,C", [(128, 128, 10), (1000, 512, 16), (17, 256, 2)])
def test_dense_head_fused_graph_replay(lib, B, K, C):
    """Captured in a CUDA graph, the head (both variants) gives its eager bits on every replay and leaves its scratch
    and counter at zero."""
    rng = np.random.default_rng(B + K + C)
    h, w2, b2, labels = _head_inputs(rng, B, K, C)
    hd, _ = _dev(h)
    w2d, _ = _dev(w2)
    b2d, _ = _dev(b2[None])
    labd = torch.from_numpy(labels).cuda()
    maskd = torch.from_numpy(rng.integers(0, 256, (B, K)).astype(np.uint8)).cuda()
    swd = torch.from_numpy(rng.random(B) + 0.5).float().cuda()
    scratch = torch.zeros(int(lib.tfy_dense_head_scratch_elems(K, C, B)), device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    for weighted in (False, True):
        stats = torch.zeros(4 if weighted else 2, device="cuda")
        outs = [Out((1,), F32), Out((C, K), BF16), Out((C,), BF16), Out((B, K), BF16), Out((K,), BF16)]

        def launch():
            args = [hd.data_ptr(), w2d.data_ptr(), b2d.data_ptr(), labd.data_ptr(), maskd.data_ptr(),
                    ctypes.c_float(2.0), outs[0].ptr(), None, stats.data_ptr()] + [o.ptr() for o in outs[1:]] + \
                   [scratch.data_ptr(), counter.data_ptr(), B, K, C]
            rc = (lib.tfy_dense_head_fused_weighted(*args, swd.data_ptr(), None, _s()) if weighted else
                  lib.tfy_dense_head_fused(*args, _s()))
            assert rc == 0
        launch()
        eager = [_bits(o.get()) for o in outs]
        eager_stats = stats.clone()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launch()
        for rep in range(3):
            for o in outs:
                o.t.fill_(0)
            stats.zero_()
            graph.replay()
            for o, e in zip(outs, eager):
                assert torch.equal(_bits(o.get()), e), f"head graph replay {rep} weighted={weighted}"
            assert torch.equal(stats, eager_stats)
            assert bool((scratch == 0).all()) and int(counter.item()) == 0


# ---------------------------------------------------------------------------------------------- tfy_ps_gather_gemm
@pytest.mark.parametrize("tier", ["exact", "bound"])
@pytest.mark.parametrize("B,N,T,n_num", [(200, 264, 3, 13), (512, 1024, 26, 13), (64, 8, 1, 0), (1, 8, 0, 5),
                                         (129, 256, 2, 64), (300, 520, 4, 1)])
def test_ps_gather_gemm_matches_reference(lib, B, N, T, n_num, tier):
    V = 1000
    rng = np.random.default_rng(B + N + T + n_num)
    K = 64 * T + n_num
    Kp = -(-K // 8) * 8
    if tier == "exact":
        tables = [ref.integers(rng, (V, 64)) for _ in range(T)]
        numeric = ref.integers(rng, (B, n_num))
        w = ref.integers(rng, (N, K))
        bias = ref.integers(rng, (N,))
    else:
        tables = [rng.standard_normal((V, 64)) * 0.3 for _ in range(T)]
        numeric = rng.standard_normal((B, n_num))
        w = rng.standard_normal((N, K)) * 0.1
        bias = rng.standard_normal(N) * 0.1
    tables = [t.astype(np.float32).astype(np.float64) for t in tables]      # the values the fp32 tables hold
    numeric = numeric.astype(np.float32).astype(np.float64)
    ids = rng.integers(0, V, (T, B))
    if T:
        ids[0, 0] = -1
        ids[-1, -1] = V                                  # both gather a zero row
    tabd = [torch.from_numpy(t).float().cuda() for t in tables]
    ptrs = torch.tensor([t.data_ptr() for t in tabd], dtype=torch.int64, device="cuda")
    idsd = torch.from_numpy(ids).cuda()
    numd = torch.from_numpy(numeric).float().cuda() if n_num else None
    shadow, w64 = _dev(w, ld=Kp, fill=0.0)               # the shadow's pad columns are zero (its contract)
    biasd, bias64 = _dev(bias[None])
    x = ref.gather_x(tables, ids, numeric if n_num else None, Kp)
    xb = ref.bf16_round(x)
    if tier == "exact":
        ref.assert_exact(xb, np.pad(w64, ((0, 0), (0, Kp - K))), bias64[0])
    for has_bias in (True, False):
        want, mag = ref.gemm(xb[:, :K], w64, bias64[0] if has_bias else None)
        xbuf = Out((B, Kp), BF16)
        y = Out((B, N), BF16)

        def launch():
            assert lib.tfy_ps_gather_gemm(shadow.data_ptr(), ptrs.data_ptr(), idsd.data_ptr(),
                                          numd.data_ptr() if n_num else None, biasd.data_ptr() if has_bias else None,
                                          xbuf.ptr(), y.ptr(), B, N, T, n_num, Kp, V, _s()) == 0
        launch()
        what = f"tfy_ps_gather_gemm {tier} {(B, N, T, n_num)} bias={has_bias}"
        _exact(xbuf.get(), xb, what + " xbuf")
        if tier == "exact":
            _exact(y.get(), ref.bf16_round(want), what)
        else:
            _bound(y.get(), want, (Kp + T + 2) * EPS32 * mag, what)
        _repeat(launch, [xbuf, y], what)


# ---------------------------------------------------------------------------------------------- refusals
def test_documented_refusals(lib):
    """Every documented refusal returns its code before any launch: -2 for K % 8, ld % 8, N % 8 and shapes outside a
    kernel's envelope, -3 for a pointer the kernel's vector loads or stores cannot take, -8 for a fused split-K grid
    that does not fit the SMs."""
    buf = torch.zeros(1 << 22, dtype=BF16, device="cuda")          # 8 MB, 512-byte aligned
    p = buf.data_ptr()
    a, b, c, c32, bias, mask = p, p + (1 << 20), p + (2 << 20), p + (3 << 20), p + (4 << 20), p + (5 << 20)
    s = _s()

    # tfy_gemm_bf16(A, B, C, C32, bias, M, N, K, lda, ldb, ldc, relu, split_k)
    g = lib.tfy_gemm_bf16
    assert g(a, b, c, None, None, 64, 64, 60, 64, 64, 64, 0, 1, s) == -2
    assert g(a, b, c, None, None, 64, 64, 64, 68, 64, 64, 0, 1, s) == -2
    assert g(a, b, c, None, None, 64, 64, 64, 64, 68, 64, 0, 1, s) == -2
    assert g(a + 8, b, c, None, None, 64, 64, 64, 64, 64, 64, 0, 1, s) == -3
    assert g(a, b + 8, c, None, None, 64, 64, 64, 64, 64, 64, 0, 1, s) == -3
    assert g(a, b, c + 8, None, None, 64, 64, 64, 64, 64, 64, 0, 1, s) == -3        # bf16 out, 16-byte stores
    assert g(a, b, None, c32 + 8, None, 64, 64, 64, 64, 64, 64, 0, 1, s) == -3      # one fp32 slab
    assert g(a, b, None, c32 + 4, None, 64, 64, 256, 256, 256, 68, 0, 2, s) == -3   # split-K slabs
    # tfy_splitk_sum_f32(slabs, out, splits, slab, n)
    assert lib.tfy_splitk_sum_f32(c32, c, 2, 64, 62, s) == -2
    assert lib.tfy_splitk_sum_f32(c32, c, 2, 66, 64, s) == -2
    assert lib.tfy_splitk_sum_f32(c32 + 4, c, 2, 64, 64, s) == -2
    assert lib.tfy_splitk_sum_f32(c32, c + 8, 2, 64, 64, s) == -2
    assert lib.tfy_splitk_sum_f32(c32, c, 0, 64, 64, s) == -2

    # tfy_gemm_bf16_splitk_fused(A, B, acc32, counters, bias, y, mask, M, N, K, lda, ldb, relu, rate, seed, hp, split)
    counters = torch.zeros(64, dtype=torch.int32, device="cuda")
    cnt = counters.data_ptr()

    def fused(A=a, B=b, acc=c32, bs=bias, y=c, m=mask, M=128, N=128, K=1024, lda=1024, ldb=1024, split=8):
        return lib.tfy_gemm_bf16_splitk_fused(A, B, acc, cnt, bs, y, m, M, N, K, lda, ldb, 1, ctypes.c_float(0.5),
                                              SEED, None, split, s)
    assert fused(K=1020) == -2 and fused(lda=1028) == -2 and fused(ldb=1028) == -2 and fused(N=132) == -2
    assert fused(A=a + 8) == -3 and fused(B=b + 8) == -3 and fused(y=c + 8) == -3
    assert fused(acc=c32 + 8) == -3 and fused(bs=bias + 8) == -3 and fused(m=mask + 4) == -3
    assert fused(M=1024, N=256, K=2048, lda=2048, ldb=2048, split=32) == -8        # 16 tiles x 32 slices > 132 SMs

    # tfy_gemm2_bf16(A, B, C, bias, M, N, K, lda, ldb, ldc, relu)
    g2 = lib.tfy_gemm2_bf16
    assert g2(a, b, c, None, 512, 512, 60, 64, 64, 512, 0, s) == -2
    assert g2(a, b, c, None, 512, 512, 64, 68, 64, 512, 0, s) == -2
    assert g2(a, b, c, None, 512, 512, 64, 64, 68, 512, 0, s) == -2
    assert g2(a, b, c, None, 512, 512, 64, 64, 64, 513, 0, s) == -2
    assert g2(a + 8, b, c, None, 512, 512, 64, 64, 64, 512, 0, s) == -3
    assert g2(a, b + 8, c, None, 512, 512, 64, 64, 64, 512, 0, s) == -3
    assert g2(a, b, c + 8, None, 512, 512, 64, 64, 64, 512, 0, s) == -3

    # tfy_dense_bwd(dh, x, w, dw, dx, B, U, I): both kernels
    d = lib.tfy_dense_bwd
    for B, U, I in ((128, 128, 256), (256, 256, 256)):
        assert d(a, b, bias, c, c32, B, 12, I, s) == -2 and d(a, b, bias, c, c32, B, U, 12, s) == -2
        assert d(a, b, bias, c, c32, 0, U, I, s) == -2
        for k in range(5):
            ptrs = [a, b, bias, c, c32]
            ptrs[k] += 8
            assert d(*ptrs, B, U, I, s) == -3, (B, U, I, k)

    # tfy_dense_head_fused(_weighted)(h, w2, b2, labels, mask1, scale1, loss, loss_host, stats, dw2, db2, dh, db1,
    # scratch, counter, B, K, C)
    for weighted in (False, True):
        fn = lib.tfy_dense_head_fused_weighted if weighted else lib.tfy_dense_head_fused
        tail = (None, None, s) if weighted else (s,)

        def head(h=a, w2=b, dw2=c, scr=c32, B=128, K=128, C=10):
            return fn(h, w2, bias, mask, None, ctypes.c_float(1.0), bias + 64, None, None, dw2, bias + 128, None, None,
                      scr, cnt, B, K, C, *tail)
        assert head(K=192) == -2 and head(C=17) == -2 and head(C=0) == -2 and head(B=0) == -2
        assert head(h=a + 8) == -3 and head(w2=b + 8) == -3 and head(scr=c32 + 8) == -3 and head(dw2=c + 4) == -3

    # tfy_ps_gather_gemm(w_shadow, tables, ids, numeric, bias, xbuf, y, B, N, T, n_num, Kp, V)
    pg = lib.tfy_ps_gather_gemm
    assert pg(a, b, bias, None, None, c, c32, 64, 12, 1, 0, 64, 10, s) == -2
    assert pg(a, b, bias, None, None, c, c32, 64, 8, 1, 0, 68, 10, s) == -2
    assert pg(a, b, bias, mask, None, c, c32, 64, 8, 1, 65, 136, 10, s) == -2
    assert pg(a, b, bias, mask, None, c, c32, 64, 8, 2, 8, 128, 10, s) == -2
    assert pg(a + 8, b, bias, None, None, c, c32, 64, 8, 1, 0, 64, 10, s) == -3
    assert pg(a, b, bias, None, None, c + 8, c32, 64, 8, 1, 0, 64, 10, s) == -3
    assert pg(a, b, bias, None, None, c, c32 + 8, 64, 8, 1, 0, 64, 10, s) == -3
    torch.cuda.synchronize()
    assert not bool((buf != 0).any()) and not bool((counters != 0).any()), "a refused call wrote memory"
