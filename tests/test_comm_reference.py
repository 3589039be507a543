"""The reference and case table of the multi-GPU collective test (tests/comm_reference.py), and the shared bound helpers
of the fused-step tests (tests/fused_step_bounds.py), on the CPU.  The GPU test trusts both, so they are pinned here."""
import hashlib
import itertools
import math

import numpy as np
import pytest
import torch

import comm_reference as cr
import fused_step_reference as ref
from fused_step_bounds import B, _kernel_update, grad_scale


def test_p2p_sum_matches_fsum_where_the_sum_is_exact():
    rs = np.random.default_rng(1)
    for world in cr.WORLDS:
        xs = [rs.integers(-(1 << 20), 1 << 20, 1000).astype(np.float32) for _ in range(world)]
        got = cr.p2p_sum(xs)
        want = [math.fsum(float(x[i]) for x in xs) for i in range(1000)]
        assert np.array_equal(got.astype(np.float64), np.array(want))


def test_p2p_sum_is_rank_order_from_plus_zero():
    one, eps = np.float32(1.0), np.float32(2.0 ** -24)
    # ((0 + 1) + eps) + eps rounds both halves away; (eps + eps) + 1 would not
    assert cr.p2p_sum([[one], [eps], [eps]])[0] == one
    assert cr.p2p_sum([[eps], [eps], [one]])[0] == np.float32(1.0 + 2.0 ** -23)
    z = cr.p2p_sum([[np.float32(-0.0)], [np.float32(-0.0)]])
    assert z[0] == 0 and not np.signbit(z[0]), "the kernel starts from +0.0f: -0 + -0 sums to +0"


def test_bf16_rounding_matches_torch():
    rs = np.random.default_rng(2)
    x = np.concatenate([(rs.standard_normal(20000) * np.exp2(rs.integers(-140, 127, 20000))).astype(np.float32),
                        np.array([0.0, -0.0, np.inf, -np.inf, 3.4e38, -3.4e38, 2.0 ** -149, 2.0 ** -133], np.float32),
                        # halfway cases, both parities
                        (np.arange(1, 200, dtype=np.uint32) << 15 | 0x3F800000).view(np.float32)])
    want = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(cr.bf16_bits(x), want)
    assert cr.bf16_bits(np.array([np.nan], np.float32))[0] & 0x7FFF == 0x7FFF


def test_p2p_allreduce_keeps_subnormals_and_propagates_inf_and_nan():
    sub = np.float32(2.0 ** -130)                        # a bf16 subnormal
    bits = cr.p2p_allreduce([[sub], [sub]], 1.0, "bf16")
    assert cr.bf16_to_f32(bits)[0] == np.float32(2.0 ** -129)
    big = np.float32(1.5 * 2.0 ** 127)
    assert np.isposinf(cr.float_of(cr.p2p_allreduce([[big], [big]], 0.5, "f32"), "f32")[0])
    assert np.isnan(cr.float_of(cr.p2p_allreduce([[np.inf], [-np.inf], [1.0]], 1.0, "f32"), "f32")[0])


def _orders(xs):
    """Every way the switch could add these fp32 values: every permutation, left to right and as a balanced pair
    tree."""
    for perm in itertools.permutations(xs):
        acc = np.float32(perm[0])
        for v in perm[1:]:
            acc = np.float32(acc + np.float32(v))
        yield acc
        while len(perm) > 1:
            perm = [np.float32(perm[i] + perm[i + 1]) if i + 1 < len(perm) else perm[i]
                    for i in range(0, len(perm), 2)]
        yield perm[0]


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_nvls_bound_contains_every_order(dtype):
    rs = np.random.default_rng(3)
    for world in (2, 3, 4, 5):
        for trial in range(60):
            xs = cr.as_dtype((rs.standard_normal(world) * np.exp2(rs.integers(-10, 10, world))).astype(np.float32),
                             dtype)
            if trial % 3 == 0:
                xs[0] = -xs[1] * np.float32(1.0 + 2.0 ** -8)     # cancellation
            for scale in (1.0, float(np.float32(1.0 / world))):
                s, a = cr.exact_sums([[x] for x in xs])
                centre, radius = cr.nvls_bound(s, a, world, scale, dtype)
                for r in _orders(list(xs)):
                    if dtype == "bf16":       # the switch rounds its fp32 sum to bf16 either way
                        rb = int(np.array([r], np.float32).view(np.uint32)[0])
                        bits = [rb >> 16] + [(rb >> 16) + 1] * bool(rb & 0xFFFF)   # toward and away from zero
                        outs = {float(cr.bf16_to_f32(np.array([b], np.uint16))[0]) for b in bits}
                    else:
                        outs = {float(r)}
                    for o in outs:
                        v = np.float32(o)
                        if scale != 1.0:
                            v = np.float32(v * np.float32(scale))
                            v = cr.float_of(cr.to_bits(np.array([v]), dtype), dtype)[0]
                        assert abs(float(v) - centre[0]) <= radius[0], (world, dtype, xs, scale, o, v, centre, radius)


def test_nvls_bound_is_tight_enough_to_see_a_dropped_rank():
    xs = [np.full(4, 1.0, np.float32)] * 4
    s, a = cr.exact_sums(xs)
    for dtype in ("f32", "bf16"):
        centre, radius = cr.nvls_bound(s, a, 4, 1.0, dtype)
        assert np.all(np.abs(3.0 - centre) > radius)


@pytest.mark.parametrize("world", cr.WORLDS)
def test_every_case_meets_the_kernels_preconditions(world):
    regions = cr.region_bytes(world)
    for c in cr.CASES:
        n, packs = cr.n_elems(c, world), cr.n_packs(c, world)
        assert n % cr.PACK[c.dtype] == 0 and n * cr.ESIZE[c.dtype] == packs * 16
        if c.algo != "oneshot":
            assert packs % world == 0
        s = cr.size_of(c, world)
        if s.grid:          # never a grid above the host's own choice
            assert s.grid <= cr.allreduce_default_grid(c.algo, packs, world, s.block)
        lo, total = cr.guarded(packs * 16)
        assert lo % 16 == 0 and total <= regions["ar"] and total <= regions["out"]
        assert lo + cr._up(packs * 16, 16) + cr.GUARD <= total
    assert sum(regions.values()) + 64 * 4096 < cr.ARENA_BYTES // 2
    for packs in cr.BCAST_PACKS:
        assert cr.guarded(packs * 16)[1] <= regions["bcast"]
    for packs in cr.GATHER_PACKS:
        assert cr.guarded(packs * 16 * world)[1] <= regions["gather"]


@pytest.mark.parametrize("world", cr.WORLDS)
def test_the_sizes_reach_the_loop_edges_they_name(world):
    for dtype in ("bf16", "f32"):
        by = {s.name: s for s in cr.sizes(world, dtype)}
        threads = lambda s: cr.pick_grid(s.shard, cr.DEFAULT_BLOCK, 2 * cr.NUM_SMS) * cr.DEFAULT_BLOCK  # noqa: E731
        assert by["sub_thread"].shard < threads(by["sub_thread"])
        t = threads(by["u_tail"])
        assert t < by["u_tail"].shard < cr.U * t and by["u_tail"].shard % t
        assert by["multi_pass"].shard > cr.GRID_PASS
        assert by["mnist"].shard * world * cr.PACK[dtype] >= cr.MNIST_PARAMS
        for name in ("grid1_block32", "grid3_block64"):
            s = by[name]
            per_pass = s.grid * s.block * cr.U
            assert s.shard > 2 * per_pass and (s.shard % per_pass) % (s.grid * s.block)


@pytest.mark.parametrize("world", cr.WORLDS)
def test_step_cases_split_where_they_say(world):
    S = cr.flat_size(cr.SMALL_SHAPES, world) // world
    c1, c2 = cr.elem3_cuts(S, world)
    pieces = cr.step_pieces("elem3", S, world)
    spans = [[cr.piece_span(p, S, r) for r in range(world)] for p in pieces]
    for r in range(world):          # the three ranges cover every shard exactly once
        cover = np.zeros(S, int)
        for sp in spans:
            lo, hi = sp[r]
            cover[lo:hi] += 1
        assert (cover == 1).all()
    if world > 1:
        assert spans[0][0] == (0, S) and spans[0][1][1] > 0, "the first range straddles the shard boundary"
        assert [sp[1] > sp[0] for sp in spans[1]].count(True) == 1, "the second range lies in one rank's shard"
    assert c1 % 8 == 0 and c2 % 8 == 0
    g = cr.case_grads(cr.flat_size(cr.SMALL_SHAPES, world), cr.StepCase("adam", ("f32", "f32"), "full", "p2p",
                                                                        "flat", solo_grad=True), 0, 0)
    assert not np.signbit(g[g == 0]).any()


def test_grad_scale_rounding_is_exact_at_powers_of_two_only():
    for world in (1, 2, 4, 8):
        assert grad_scale(ref.Hyper(lr=1.0, grad_scale=0.25, world=world)).e == 0.0
    for world in (3, 5):
        b = grad_scale(ref.Hyper(lr=1.0, grad_scale=1.0, world=world))
        assert 0.0 < b.e <= 2.0 ** -24 * b.v
        assert float(np.float32(1.0) / np.float32(world)) == b.v + b.e or \
            float(np.float32(1.0) / np.float32(world)) == b.v - b.e


# the bounds of the fused-step error analysis, as the single-GPU test computed them before the helpers moved
PINNED = {
    ("adadelta", 0, 1.0): "10a8ba54d193d2c6", ("adadelta", 1, 0.25): "35590302bdae0b12",
    ("adagrad", 0, 1.0): "f1ddd53f26883521", ("adagrad", 1, 0.25): "f8fc8e251cf2a0ff",
    ("adam", 0, 1.0): "1ce2b66f0aada14e", ("adam", 1, 0.25): "c19054cd5203d014",
    ("adam_l2", 0, 1.0): "9588cb54d3764ca2", ("adam_l2", 1, 0.25): "6ae4685e33c2d928",
    ("adamw", 0, 1.0): "31032802457e1502", ("adamw", 1, 0.25): "ee91c41aca817946",
    ("ftrl", 0, 1.0): "1b85dd6904d57d9a", ("ftrl", 1, 0.25): "25997869eba0f3bc",
    ("rmsprop", 0, 1.0): "663e08d9cb69851a", ("rmsprop", 1, 0.25): "e5109edaccff33dc",
    ("rmsprop_centered", 0, 1.0): "cc9b0261820e3b17", ("rmsprop_centered", 1, 0.25): "8e9e25a30bee339f",
    ("rmsprop_momentum", 0, 1.0): "876ba5245bae1ca0", ("rmsprop_momentum", 1, 0.25): "f95fb7248c84fe7d",
    ("rmsprop_momentum_centered", 0, 1.0): "50422ba7846bc283",
    ("rmsprop_momentum_centered", 1, 0.25): "fa39ab736c9fefc5",
    ("sgd", 0, 1.0): "b0381fe2c3879dbf", ("sgd", 1, 0.25): "9cadfb232602f173",
    ("sgd_momentum_dampening", 0, 1.0): "ba8b8846383d3ba6", ("sgd_momentum_dampening", 1, 0.25): "cdbcb38cc98902a1",
    ("sgd_nesterov_wd", 0, 1.0): "9c1a1d552991d34f", ("sgd_nesterov_wd", 1, 0.25): "0963e78de4adeda9",
}


def test_moved_bound_helpers_give_the_old_results():
    rs = np.random.RandomState(7)
    n = 64
    p = rs.randn(n) * 0.3
    g = rs.randn(n) * 0.5
    g[:4] = 0
    g[4:8] = 1e-25
    s1 = np.abs(rs.randn(n)) * 0.1
    s2 = np.abs(rs.randn(n)) * 0.01
    s3 = rs.randn(n) * 0.01
    for (name, step, gs), want in PINNED.items():
        kind, hp, init = ref.VARIANTS[name]
        h = ref.Hyper(grad_scale=gs, **hp)
        out, _ = _kernel_update(kind, h, step, B(p), B(g), B(s1 + init), B(s2), B(s3))
        d = hashlib.sha256(b"".join(np.ascontiguousarray(x.v).tobytes() + np.ascontiguousarray(x.e).tobytes()
                                    for x in out)).hexdigest()[:16]
        assert d == want, (name, step, gs)


def test_bound_at_three_ranks_covers_the_rounded_scale():
    """At world 3 the kernel multiplies by fl32(1/3): the bound around the exact 1/3 must contain that product."""
    kind, hp, _ = ref.VARIANTS["sgd"]
    h = ref.Hyper(grad_scale=1.0, world=3, **hp)
    g = np.array([3.0e3, -1.0, 0.5], np.float64)
    p = np.zeros(3)
    (pb, *_), _ = _kernel_update(kind, h, 0, B(p), B(g), B(p), B(p), B(p))
    dev = -np.float32(h.lr) * (np.float32(g) * (np.float32(1.0) / np.float32(3)))
    assert (np.abs(dev.astype(np.float64) - pb.v) <= pb.e).all()
