"""The fused optimizer step (tfy_fused_step_kernel, ops/csrc/tfy_fused_step.cuh) against the float64 reference of
tests/fused_step_reference.py, for every optimizer variant, every (gradient, parameter) dtype pair and every way a step
can be split into launches, at a small odd layout and at the MNIST-CNN's 1,199,882 parameters.  The full size wraps
the grid-stride loop of the LOCAL launch (792 CTAs x 128 threads = 101,376 groups of 8 per pass) and of the U=2
multi-GPU launch (264 x 256 threads x 2 groups per batch).

Error model: one step at a time.  Before every step the test reads back the kernel's own master weights and states
and feeds them, with the gradient exactly as the buffer holds it, to the reference.  Each element of the kernel's
result must then lie within a bound computed for that element by a running error analysis of the kernel's own
sequence of fp32 operations (class ``B`` of tests/fused_step_bounds.py, which states the model).

The centre of the interval is the reference's value.  The kernel's per-element formulas are listed in
``_kernel_update``; ``tfy_opt_update_rt`` is what they mirror.  The largest error as a fraction of its bound is
printed per optimizer at the end of the module (``pytest -s``).
"""
import ctypes
from collections import defaultdict

import numpy as np
import pytest
import torch

import fused_step_reference as ref
from fused_step_bounds import B, _kernel_update

pytestmark = pytest.mark.gpu

MNIST_SHAPES = [(32, 3, 3, 1), (32,), (64, 3, 3, 32), (64,), (9216, 128), (128,), (128, 10), (10,)]
SMALL_SHAPES = [(33, 17), (129,), (7, 5, 3), (1,), (5,)]        # 561, 129, 105, 1, 5: every tensor padded to 8
# element cuts of the 3-piece ranged step, each inside a tensor: [0, 561) / [568, 697) and [320, 18752) / [18816, ...)
CUTS = {"small": (200, 640), "mnist": (9000, 600_000)}
SHAPES = {"small": SMALL_SHAPES, "mnist": MNIST_SHAPES}
DT = {"f32": torch.float32, "bf16": torch.bfloat16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32"), ("f32", "bf16")]
STEPS = 3                  # step 0 (SGD's first step, Adam's t = 1), a step at grad_scale 0.25, one more

_RATIO = defaultdict(float)


# ---------------------------------------------------------------------------------------------------------------
# the optimizer under test
# ---------------------------------------------------------------------------------------------------------------
_OPT = {}


def _fused(name, gdt, pdt, size):
    """One FusedShardedOptimizer per (variant, dtypes, size) for the whole module: the solo arena is a bump
    allocator, so the cases reuse the buffers instead of allocating new ones."""
    key = (name, gdt, pdt, size)
    if key not in _OPT:
        from tf_yarn_b200.keras.engine import _solo_communicator
        from tf_yarn_b200.parallel.comm import FusedShardedOptimizer, OptimizerSpec
        kind, hp, init = ref.VARIANTS[name]
        spec = OptimizerSpec(kind, hp["lr"], hp.get("p1", 0.0), hp.get("p2", 0.0), hp.get("eps", 0.0),
                             hp.get("wd", 0.0), hp.get("flags", 0), init)
        _OPT[key] = FusedShardedOptimizer(_solo_communicator(0), SHAPES[size], spec, param_dtype=DT[pdt],
                                          grad_dtype=DT[gdt])
    return _OPT[key]


def _hyper(name, grad_scale=1.0):
    kind, hp, _ = ref.VARIANTS[name]
    return kind, ref.Hyper(grad_scale=grad_scale, **hp)


def _reset(fo, name, seed):
    """Fresh master weights (FTRL: one in ten at exactly 0), initial states, step 0, grad_scale 1."""
    kind, _, init = ref.VARIANTS[name]
    rs = np.random.RandomState(seed)
    p0 = (rs.randn(fo.n) * 0.3).astype(np.float32)
    if kind == "ftrl":
        p0[rs.rand(fo.n) < 0.1] = 0.0
    fo.master.copy_(torch.from_numpy(p0))
    fo.flat_params.copy_(fo.master.to(fo.param_dtype))
    fo.flat_grads.zero_()
    fo.s1.fill_(init)
    fo.s2.zero_()
    fo.set_step_count(0)
    fo.set_grad_scale(1.0)
    torch.cuda.synchronize()
    return rs


def _fill_grads(fo, rs):
    """Gaussian gradients with exact +0 and -0, values whose square underflows in fp32 (~1e-25) and large ones (~1e3)."""
    n = fo.n
    g = (rs.randn(n) * 0.5).astype(np.float32)
    u = rs.rand(n)
    sign = np.where(rs.rand(n) < 0.5, -1.0, 1.0).astype(np.float32)
    g[u < 0.04] = 0.0
    g[(u >= 0.04) & (u < 0.08)] = -0.0
    tiny = (u >= 0.08) & (u < 0.12)
    g[tiny] = sign[tiny] * np.float32(1e-25) * (1 + rs.rand(int(tiny.sum()))).astype(np.float32)
    big = (u >= 0.12) & (u < 0.14)
    g[big] = sign[big] * np.float32(1e3) * (1 + rs.rand(int(big.sum()))).astype(np.float32)
    fo.flat_grads.copy_(torch.from_numpy(g).to(fo.grad_dtype))


def _states(fo, kind, h):
    """The kernel's master, s1, s2, s3 as float64 (zeros for a state the optimizer does not have)."""
    S = fo.shard_n
    f = [t.double().cpu().numpy() for t in (fo.master, fo.s1, fo.s2)]
    p, s1, buf = f
    s2 = s3 = np.zeros(S)
    if kind == "rmsprop":
        off = 0
        if h.p2 > 0:
            s2, off = buf[:S], S
        if h.flags & 1:
            s3 = buf[off:off + S]
    elif ref.n_states(kind, h) == 2:
        s2 = buf[:S]
    return p, s1, s2, s3


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _snapshot(fo):
    return {k: t.clone() for k, t in (("master", fo.master), ("s1", fo.s1), ("s2", fo.s2),
                                      ("params", fo.flat_params), ("grads", fo.flat_grads), ("hyper", fo.hyper))}


def _restore(fo, snap):
    for k, t in (("master", fo.master), ("s1", fo.s1), ("s2", fo.s2), ("params", fo.flat_params),
                 ("grads", fo.flat_grads), ("hyper", fo.hyper)):
        t.copy_(snap[k])
    torch.cuda.synchronize()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _range(fo, e0, e1, advance, mode=None, zero_grads=0):
    """tfy_fused_step_range directly: it takes modes and ranges FusedShardedOptimizer.step does not."""
    from tf_yarn_b200.ops import native
    from tf_yarn_b200.parallel.comm import _DT, launch_code
    c = fo.comm
    return c.lib.tfy_fused_step_range(
        c.arena.ctx_ref, _DT[fo.grad_dtype], _DT[fo.param_dtype], launch_code(fo.spec),
        native.MODE_LOCAL if mode is None else mode, fo.grad_off, fo.param_off, fo.shard_n, fo.master.data_ptr(),
        fo.s1.data_ptr(), fo.s2.data_ptr(), fo.hyper.data_ptr(), zero_grads, 0, 0, e0, e1, int(advance), _s())


def _pieces(fo, how, size):
    """The launches of one step as (e0, e1, launch): element ranges of the flat buffers."""
    n, G = fo.n, fo.shard_n // 8
    c1, c2 = CUTS[size]
    if how == "full":
        return [(0, n, lambda: fo.step())]
    if how == "elem3":
        return [(0, c1, lambda: fo.step(elem_range=(0, c1), advance=False)),
                (c1, c2, lambda: fo.step(elem_range=(c1, c2), advance=False)),
                (c2, n, lambda: fo.step(elem_range=(c2, n), advance=True))]
    if how == "groups2":
        g = G // 3
        return [(0, 8 * g, lambda: fo.step(shard_groups=(0, g), advance=False)),
                (8 * g, n, lambda: fo.step(shard_groups=(g, G), advance=True))]
    assert how == "edges"                   # an empty range, then a range whose end lies past the buffer (clamped)
    return [(c1, c1, lambda: fo.step(elem_range=(c1, c1), advance=False)),
            (0, c1, lambda: fo.step(elem_range=(0, c1), advance=False)),
            (c1, n, lambda: _check_rc(_range(fo, c1, n + 64 * 8, advance=True)))]


def _check_rc(rc):
    assert rc == 0, rc


def _run_step(fo, how, size, k):
    """One optimizer step, checking after every launch that nothing outside its range moved."""
    fo.zero_grads = how == "full"
    pieces = _pieces(fo, how, size)
    for i, (e0, e1, launch) in enumerate(pieces):
        before = _snapshot(fo) if how != "full" else None
        launch()
        torch.cuda.synchronize()
        if before is not None:
            for key, now in (("master", fo.master), ("s1", fo.s1), ("params", fo.flat_params),
                             ("grads", fo.flat_grads)):
                a, b = _bits(before[key]), _bits(now)
                assert torch.equal(a[:e0], b[:e0]) and torch.equal(a[e1:], b[e1:]), (how, i, key, "moved")
            assert torch.equal(before["grads"], fo.flat_grads), (how, i, "gradients changed")
            S = fo.shard_n
            for j in range(fo.s2.numel() // S):      # every state in the s2 buffer, shard_n long each
                a, b = before["s2"][j * S:(j + 1) * S], fo.s2[j * S:(j + 1) * S]
                assert torch.equal(_bits(a[:e0]), _bits(b[:e0])) and torch.equal(_bits(a[e1:]), _bits(b[e1:]))
        last = i == len(pieces) - 1
        assert fo.step_count == (k + 1 if last else k), (how, i, fo.step_count)
    if how == "full":
        assert not bool(fo.flat_grads.any()), "a full launch with zero_grads must clear every gradient"


def _check_against_reference(name, fo, before, g, h, k):
    kind = ref.VARIANTS[name][0]
    p0, s10, s20, s30 = before
    want = ref.step(kind, p0, g, s10, s20, s30, h, k)
    bounds, undecided = _kernel_update(kind, h, k, B(p0), B(g), B(s10), B(s20), B(s30))
    got = _states(fo, kind, h)
    used = [True, kind != "sgd" or h.p1 != 0.0, ref.n_states(kind, h) >= 2 and (kind != "rmsprop" or h.p2 > 0),
            kind == "rmsprop" and bool(h.flags & 1)]
    for what, on, x, w, b in zip(("p", "s1", "s2", "s3"), used, got, want, bounds):
        if not on:
            continue
        bound = b.e + 2.0 ** -40 * np.abs(w)
        assert np.isfinite(bound).all(), (name, what, "no finite bound")
        err = np.abs(x - w)
        if what == "p" and undecided is not None:
            # |z| within its bound of l1: the kernel may clamp or not; otherwise its zeros must be the reference's
            _, _, w_free = ref.ftrl_linear(p0, g, s10, s20, h)
            err = np.where(undecided & (x == 0.0), 0.0, np.where(undecided, np.abs(x - w_free), err))
            assert np.array_equal((x == 0.0)[~undecided], (w == 0.0)[~undecided]), (name, "FTRL zero pattern")
        bad = ~(err <= bound)
        assert not bad.any(), (name, what, k, int(bad.sum()), np.flatnonzero(bad)[:5], x[bad][:5], w[bad][:5],
                               bound[bad][:5])
        ratio = np.divide(err, bound, out=np.zeros_like(err), where=bound > 0)
        _RATIO[name] = max(_RATIO[name], float(ratio.max()))
    # the compute parameters are the fp32 master rounded to nearest even, bit for bit
    assert torch.equal(_bits(fo.flat_params), _bits(fo.master.to(fo.param_dtype))), (name, "parameter packing")


def _run_case(name, gdt, pdt, size, how, seed=0):
    fo = _fused(name, gdt, pdt, size)
    kind, _ = _hyper(name)
    rs = _reset(fo, name, seed)
    for k in range(STEPS):
        scale = 0.25 if k == 1 else 1.0
        fo.set_grad_scale(scale)
        _fill_grads(fo, rs)
        kind, h = _hyper(name, scale)
        torch.cuda.synchronize()
        before = _states(fo, kind, h)
        g = fo.flat_grads.double().cpu().numpy()
        _run_step(fo, how, size, k)
        _check_against_reference(name, fo, before, g, h, k)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _RATIO:
        print("\nlargest |kernel - reference| / bound per optimizer variant:")
        for name in sorted(_RATIO):
            print(f"  {name:28s} {_RATIO[name]:.3f}")


@pytest.mark.parametrize("how", ["full", "elem3", "groups2", "edges"])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
@pytest.mark.parametrize("name", sorted(ref.VARIANTS))
def test_small_layout_matches_reference(name, pair, how):
    _run_case(name, pair[0], pair[1], "small", how)


@pytest.mark.parametrize("how", ["full", "elem3"])
@pytest.mark.parametrize("pair", [("bf16", "bf16"), ("f32", "f32")], ids=lambda p: f"{p[0]}-{p[1]}")
@pytest.mark.parametrize("name", sorted(ref.VARIANTS))
def test_mnist_size_matches_reference(name, pair, how):
    """1,199,888 elements: the LOCAL grid-stride loop wraps, and its prefetch of the next batch's state runs."""
    _run_case(name, pair[0], pair[1], "mnist", how)


@pytest.mark.parametrize("name", ["adadelta", "adam"])
def test_thirty_steps_stay_near_the_reference(name):
    """30 bf16 steps without teacher forcing: the reference follows its own float64 trajectory from the same start.
    Each step's rounding is ~1e-6 of that step's update, and the update rules do not amplify it, so the master
    must stay within 1e-4 of the sum of the reference's update magnitudes."""
    fo = _fused(name, "bf16", "bf16", "mnist")
    kind, h = _hyper(name)
    rs = _reset(fo, name, 5)
    p, s1, s2, s3 = _states(fo, kind, h)
    moved = np.zeros_like(p)
    fo.zero_grads = True
    for k in range(30):
        _fill_grads(fo, rs)
        g = fo.flat_grads.double().cpu().numpy()
        fo.step()
        p_new, s1, s2, s3 = ref.step(kind, p, g, s1, s2, s3, h, k)
        moved += np.abs(p_new - p)
        p = p_new
    torch.cuda.synchronize()
    assert fo.step_count == 30
    got = fo.master.double().cpu().numpy()
    bound = 1e-4 * moved + 2.0 ** -18 * np.abs(p)        # + the fp32 rounding of p, 30 times
    assert (np.abs(got - p) <= bound).all(), float((np.abs(got - p) / bound).max())
    assert torch.equal(_bits(fo.flat_params), _bits(fo.master.to(fo.param_dtype)))


def test_grad_scale_scales_the_gradient_the_kernel_sees():
    """grad_scale 0.25 with gradient 4 g is the same step as grad_scale 1 with g, bit for bit (powers of two)."""
    fo = _fused("sgd_momentum_dampening", "f32", "f32", "small")
    out = []
    for scale, mult in ((1.0, 1.0), (0.25, 4.0)):
        rs = _reset(fo, "sgd_momentum_dampening", 3)
        fo.set_grad_scale(scale)
        _fill_grads(fo, rs)
        fo.flat_grads.mul_(mult)
        fo.zero_grads = True
        fo.step()
        torch.cuda.synchronize()
        out.append(fo.master.clone())
    assert torch.equal(out[0], out[1])
    rs = _reset(fo, "sgd_momentum_dampening", 3)
    fo.set_grad_scale(0.25)
    _fill_grads(fo, rs)
    fo.step()
    torch.cuda.synchronize()
    assert not torch.equal(fo.master, out[0])


# ---------------------------------------------------------------------------------------------------------------
# the U = 2 multi-GPU instantiations on one GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [("bf16", "bf16"), ("f32", "f32")], ids=lambda p: f"{p[0]}-{p[1]}")
@pytest.mark.parametrize("name", sorted(ref.VARIANTS))
def test_p2p_mode_at_world_one_matches_local(name, pair):
    """MODE_P2P on the solo communicator runs the multi-GPU kernel: 2 groups in flight per thread, the grid entry
    and exit barriers on the arena's own signal pad, system-scope stores.  Its per-element arithmetic is the LOCAL
    kernel's (0 + g == g for every non-zero g), so two steps with zero_grads give the LOCAL results exactly.  For
    RMSprop this is also the regression test of the multi-GPU grid: its kernels fit one 256-thread CTA per SM, and a
    grid of two per SM never finished, because its first CTAs waited at the exit barrier for CTAs that had no SM."""
    from tf_yarn_b200.ops import native
    fo = _fused(name, pair[0], pair[1], "mnist")
    results = []
    for mode in (native.MODE_LOCAL, native.MODE_P2P):
        rs = _reset(fo, name, 11)
        for k in range(2):
            _fill_grads(fo, rs)
            assert _range(fo, 0, 2 ** 64 - 1, advance=True, mode=mode, zero_grads=1) == 0
            torch.cuda.synchronize()
            assert fo.step_count == k + 1
            assert not bool(fo.flat_grads.any())
        results.append([t.clone() for t in (fo.master, fo.s1, fo.s2, fo.flat_params)])
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_nvls_mode_without_multicast_is_refused():
    from tf_yarn_b200.ops import native
    fo = _fused("adam", "bf16", "bf16", "small")
    assert fo.comm.arena.mc_base == 0
    assert _range(fo, 0, fo.n, advance=True, mode=native.MODE_NVLS) == -5


# ---------------------------------------------------------------------------------------------------------------
# the overlap role inside the conv2 weight-gradient kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sgd_momentum_dampening", "adadelta", "adam", "adagrad", "ftrl"])
def test_overlap_role_matches_single_launch(name):
    """The fast path's conv2 weight gradient (B = 128, 26 x 26 x 32 in, 12 x 12 x 64 pooled gradient) with the fused
    step of groups [g0, S/8) on its spare CTAs, then the trailing step of [0, g0): the same bits as one full launch,
    the same dw / db as the kernel without the role, and one step counted.  g0 = S/16 makes the role's loop wrap."""
    from test_gpu_conv2_kernels import _inputs
    from tf_yarn_b200.ops import native
    lib = native.load()
    B_, H, W = 128, 26, 26
    n_cta = int(lib.tfy_conv3x3_c32_wgrad_spare_ctas(B_, H, W))
    if n_cta == 0:
        pytest.skip("the weight-gradient grid fills every SM: no CTAs for the role")
    a, w, bias, dp, _ = _inputs(B_, H, W, 21)
    code = torch.empty(B_, 12, 12, 64, dtype=torch.uint8, device="cuda")
    pooled = torch.empty(B_, 12, 12, 64, dtype=torch.bfloat16, device="cuda")
    assert lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(),
                                        code.data_ptr(), B_, H, W, 0.25, 1234, None, _s()) == 0
    scale = ctypes.c_float(256.0 / 192.0)
    part = torch.zeros(int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()), dtype=torch.float32, device="cuda")

    def wgrad(ov):
        dw = torch.empty(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
        db = torch.empty(64, dtype=torch.bfloat16, device="cuda")
        sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
        assert lib.tfy_conv3x3_c32_wgrad_unpool_ov(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                   part.data_ptr(), dw.data_ptr(), db.data_ptr(), sync.data_ptr(),
                                                   B_, H, W, ctypes.byref(ov) if ov is not None else None, _s()) == 0
        return dw, db

    fo = _fused(name, "bf16", "bf16", "mnist")
    rs = _reset(fo, name, 4)
    fo.zero_grads = False
    G = fo.shard_n // 8
    g0 = G // 16
    for k in range(2):                          # step 0 (SGD's first step) and step 1
        _fill_grads(fo, rs)
        snap = _snapshot(fo)
        dw, db = wgrad(fo.overlap_step(g0, G, n_cta))
        fo.step(shard_groups=(0, g0), advance=True)
        torch.cuda.synchronize()
        assert fo.step_count == k + 1
        overlapped = _snapshot(fo)
        _restore(fo, snap)
        fo.step()
        dw0, db0 = wgrad(None)
        torch.cuda.synchronize()
        single = _snapshot(fo)
        for key in ("master", "s1", "s2", "params", "grads", "hyper"):
            assert torch.equal(_bits(overlapped[key]) if key != "hyper" else overlapped[key],
                               _bits(single[key]) if key != "hyper" else single[key]), (name, k, key)
        assert torch.equal(_bits(dw), _bits(dw0)) and torch.equal(_bits(db), _bits(db0))
