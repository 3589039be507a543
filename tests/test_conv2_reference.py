"""The float64 reference of the conv2 tensor-core kernels (tests/conv2_reference.py), pinned on any box: against torch
float64 conv2d / max_pool2d and autograd, on hand-worked tie windows, and against the host builds of the kernels' own
dropout hash and keep-scale rule.  Also: the fast path hands a tensor-core conv stage's backward that rule's scale."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv2_reference as ref
import nn_reference


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = nn_reference.host_lib(str(tmp_path_factory.mktemp("conv2ref")))
    if lib is None:
        pytest.skip("needs g++ and the CUDA headers")
    return ref.declare_host(lib)


def _nchw(x):
    return torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2)


def test_forward_matches_torch_conv_pool_relu():
    r = np.random.default_rng(1)
    B, H, W = 3, 10, 14
    a = r.standard_normal((B, H, W, 32))
    w = r.standard_normal((64, 3, 3, 32)) * 0.1
    b = r.standard_normal(64) * 0.3
    out = ref.fwd(a, w, b)
    z = F.conv2d(_nchw(a), torch.from_numpy(w).permute(0, 3, 1, 2))
    zp, zi = F.max_pool2d(z, 2, return_indices=True)
    want = F.relu(zp + torch.from_numpy(b).view(1, -1, 1, 1)).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(out.p, want, rtol=1e-12, atol=1e-12)
    zi = zi.permute(0, 2, 3, 1).numpy()
    pos = ((zi // (W - 2)) % 2) * 2 + (zi % 2)
    assert (out.code & 3 == pos).all()                # random data: no ties, every rule agrees
    assert ((out.code >> 2) == (want > 0)).all()
    assert (out.mag >= np.abs(out.v)).all() and (out.gap > 0).all()
    zr, mag = ref.conv(a, w)
    np.testing.assert_allclose(zr, z.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    assert (mag >= np.abs(zr)).all()


def test_backward_matches_autograd_with_dropout():
    """dgrad / un-pool / wgrad / db against autograd of conv -> pool -> +b -> ReLU -> dropout(keep, scale) in float64."""
    r = np.random.default_rng(2)
    B, H, W = 2, 18, 10
    a = r.standard_normal((B, H, W, 32))
    w = r.standard_normal((64, 3, 3, 32)) * 0.1
    b = r.standard_normal(64) * 0.3
    keep = r.random((B, (H - 2) // 2, (W - 2) // 2, 64)) >= 0.3
    scale = 256.0 / 179.0
    out = ref.fwd(a, w, b, keep, scale)
    at = _nchw(a).requires_grad_(True)
    wt = torch.from_numpy(w).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    p = F.relu(F.max_pool2d(F.conv2d(at, wt), 2) + bt.view(1, -1, 1, 1)) * _nchw(keep.astype(np.float64)) * scale
    np.testing.assert_allclose(p.permute(0, 2, 3, 1).detach().numpy(), out.p, rtol=1e-12, atol=1e-12)
    dp = r.standard_normal(out.p.shape)
    p.backward(_nchw(dp))
    dz = ref.unpool_exact(dp, out.code, scale)
    dx, dx_mag = ref.dgrad(dz, w)
    dw, dw_mag = ref.wgrad(a, dz)
    db, db_mag = ref.bias_grad(np.where(out.code & 4, dp * scale, 0.0))
    np.testing.assert_allclose(dx, at.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dw, wt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-10, atol=1e-12)
    assert (dx_mag >= np.abs(dx)).all() and (dw_mag >= np.abs(dw)).all() and (db_mag >= np.abs(db)).all()
    # the gate zeroes dx where the previous layer's ReLU output is <= 0
    gate = r.standard_normal(dx.shape)
    dxg, _ = ref.dgrad(dz, w, gate)
    assert (dxg[gate <= 0] == 0).all() and (dxg[gate > 0] == dx[gate > 0]).all()


def test_unpool_rounds_the_operand_like_the_kernel():
    """g = fp32(dp * scale); the dz operand is g in bf16 at the argmax; db sums the fp32 g."""
    dp = np.array([1.0, 1.0, -3.0, 0.5]).reshape(1, 1, 4, 1)
    code = np.array([4 | 0, 4 | 3, 4 | 1, 2], np.uint8).reshape(1, 1, 4, 1)
    scale = 256.0 / 179.0
    dz, g = ref.unpool(dp, code, scale)
    g32 = np.float32(scale)
    np.testing.assert_array_equal(g.ravel(), [g32, g32, np.float32(-3.0) * g32, 0.0])
    assert dz.shape == (1, 2, 8, 1)
    q = ref.bf16_round(np.float32(scale))
    assert dz[0, 0, 0, 0] == q and dz[0, 1, 3, 0] == q and dz[0, 0, 5, 0] == ref.bf16_round(np.float32(-3.0) * g32)
    assert np.count_nonzero(dz) == 3                  # the ungated element contributes nothing


@pytest.mark.parametrize("win,pos", [
    ([1.0, 3.0, 3.0, 0.0], 2),        # positive tie: the last of the maxima
    ([2.5, 2.5, 2.5, 2.5], 3),
    ([3.0, 1.0, 1.0, 3.0], 3),
    ([-1.0, -1.0, -2.0, -5.0], 0),    # negative tie: the first
    ([-4.0, -1.0, -3.0, -1.0], 1),
    ([-1.0, 2.0, 2.0, -3.0], 2),      # mixed signs, positive maximum
    ([-7.0, -2.0, -9.0, -2.0], 1),    # mixed magnitudes, negative maximum
    ([0.0, -1.0, 0.0, -2.0], 2),      # +0 maximum counts as positive
    ([-1.0, 5.0, 4.0, -3.0], 1),      # no tie
])
def test_tie_rule_on_hand_worked_windows(win, pos):
    assert int(ref.pool_argmax(np.array(win).reshape(4, 1))[0]) == pos
    # the same window through the whole forward: a 4 x 4 input whose z is the window (w picks channel 0 of tap 0)
    a = np.zeros((1, 4, 4, 32))
    a[0, 0:2, 0:2, 0] = np.array(win).reshape(2, 2)
    w = np.zeros((64, 3, 3, 32))
    w[:, 0, 0, 0] = 1.0
    out = ref.fwd(a, w, np.full(64, 10.0))
    assert (out.code[0, 0, 0] == (pos | 4)).all()


def test_raw_hash_top_bits_are_the_uniform_draws(host):
    for seed, step, idx0, n in [(0, 0, 0, 4096), (1234, 5, 77, 1000), (0x7fffffff, 3, (1 << 32) - 600, 600),
                                (20261016, 1 << 20, 123456789, 2048)]:
        h = ref.host_hash_u32(host, seed, step, n, idx0)
        u = nn_reference.uniform(host, seed, step, n, idx0)
        np.testing.assert_array_equal((h >> 8).astype(np.float64) * 2.0 ** -24, u)
    a = ref.host_hash_u32(host, 1, 0, 64)
    assert not np.array_equal(a, ref.host_hash_u32(host, 1, 1, 64)), "the step must change the draws"
    assert len(np.unique(a)) == 64


def test_keep_from_hash_reads_byte_e_mod_4_of_group_e_div_4():
    h = np.array([0x04030201, 0xFF00807F], np.uint32)
    np.testing.assert_array_equal(ref.keep_from_hash(h, 3, 8), [False, False, True, True, True, True, False, True])
    assert ref.keep_from_hash(h, 0, 8).all()


def _rates():
    k = np.arange(256, dtype=np.float32)
    edges = (k + np.float32(0.5)) / np.float32(256)      # (k + 0.5) / 256: exact in fp32, thr = k + 1
    below = np.nextafter(edges, np.float32(0))           # one fp32 step below: thr = k
    keras = np.array([0.0, 1e-4, 1 / 600, 0.001953125, 0.1, 0.25, 0.3, 0.4, 0.5, 0.9, 0.99, 0.996], np.float32)
    grid = np.linspace(0, 0.998, 4001, dtype=np.float32)
    return np.concatenate([edges[:-1], below, keras, grid])


def test_keep_scale_rule_at_many_rates_and_the_rounding_boundaries(host):
    rates = _rates()
    thr, scale = ref.host_keep_scale(host, rates)
    # thr = (uint32)(rate * 256 + 0.5) evaluated in fp32 (numpy float32 arithmetic rounds each operation like the
    # kernel; rate * 256 is exact, so a fused multiply-add gives the same)
    r32 = rates.astype(np.float32)
    want_thr = np.where(r32 > 0, np.floor(r32 * np.float32(256) + np.float32(0.5)), 0).astype(np.uint32)
    np.testing.assert_array_equal(thr, want_thr)
    np.testing.assert_array_equal(scale, np.float32(256) / (np.float32(256) - thr.astype(np.float32)))
    k = np.arange(255)
    np.testing.assert_array_equal(thr[:255], k + 1)
    np.testing.assert_array_equal(thr[256:510], np.arange(1, 255))
    # one step below 1/512, rate * 256 + 0.5 = 1 - 2^-25 is not an fp32 number and rounds up to 1
    assert thr[255] == 1
    # the forward's scale differs from 1 / (1 - rate) except where rate * 256 is an integer
    got = dict(zip([0.1, 0.25, 0.3, 0.4, 0.5, 0.9, 0.99], ref.host_keep_scale(host, [0.1, 0.25, 0.3, 0.4, 0.5, 0.9,
                                                                                        0.99])[1]))
    assert got[0.25] == np.float32(4 / 3) and got[0.5] == 2.0
    assert got[0.3] == np.float32(256 / 179) and got[0.9] == np.float32(256 / 26) and got[0.99] == np.float32(256 / 3)
    assert ref.host_keep_scale(host, [1e-4])[1][0] == 1.0       # below 1/512 nothing is dropped and nothing scaled


def test_native_entry_matches_the_host_rule(host):
    from tf_yarn_b200.keras import fastpath
    from tf_yarn_b200.ops import native
    try:
        lib = native.load()
    except Exception as exc:  # noqa: BLE001
        pytest.skip(f"native library not built: {exc}")
    rates = _rates()
    _, scale = ref.host_keep_scale(host, rates)
    got = np.array([fastpath.keep_scale(lib, float(r)) for r in rates], np.float32)
    np.testing.assert_array_equal(got, scale)
    assert lib.tfy_conv3x3_c32_keep_scale(0.5, None) != 0, "a null output pointer is rejected"


class _RecLib:
    def __init__(self):
        self.calls = []

    def tfy_conv3x3_c32_keep_scale(self, rate, out):
        self.calls.append(rate)
        out._obj.value = 1.25 + rate     # any value: the fast path must pass on exactly what the rule returns
        return 0


@pytest.mark.parametrize("rate", [0.0, 0.1, 0.3, 0.9, 0.99])
def test_fast_path_backward_scale_of_a_tensor_core_stage_is_the_kernel_rule(rate):
    from tf_yarn_b200.keras import layers as L
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    st = types.SimpleNamespace(kind="conv", layer=L.Conv2D(64, 3, activation="relu"), relu=True, pool=True, drop=rate)
    eng = types.SimpleNamespace(lib=_RecLib())
    assert FastSequentialEngine._conv_drop_scale(eng, st, True) == float(np.float32(1.25 + rate))
    assert eng.lib.calls == [rate]
    # a stage whose forward ran the general pool kernel keeps that kernel's 1 / (1 - rate)
    assert FastSequentialEngine._conv_drop_scale(eng, st, False) == (1.0 / (1.0 - rate) if rate > 0 else 1.0)
    assert eng.lib.calls == [rate]
    # and the backward asks for it with the stage's forward kind
    import inspect
    src = inspect.getsource(FastSequentialEngine._forward_backward)
    assert "scale = self._conv_drop_scale(st, st.pool and self._tc_conv(st, B))" in src
    assert src.count("1.0 / (1.0 - st.drop)") == 1           # only the Dense stage's own mask kernels
