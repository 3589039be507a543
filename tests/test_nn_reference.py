"""The float64 reference of the general-shape layer kernels (tests/nn_reference.py), pinned on any box: against torch
autograd in float64 on the CPU, on hand-worked tie and code-byte cases, and against the host build of the kernels'
dropout generator."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import nn_reference as ref


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = ref.host_lib(str(tmp_path_factory.mktemp("nnref")))
    if lib is None:
        pytest.skip("needs g++ and the CUDA headers")
    return lib


def _rng(seed=0):
    return np.random.default_rng(seed)


def test_conv_c1_matches_torch_conv2d():
    r = _rng(1)
    B, H, W, O = 3, 7, 9, 8
    x = r.standard_normal((B, H, W))
    w = r.standard_normal((O, 9))
    b = r.standard_normal(O)
    y, mag = ref.conv_c1_fwd(x, w, b)
    xt = torch.from_numpy(x)[:, None]
    wt = torch.from_numpy(w).view(O, 1, 3, 3).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    z = F.conv2d(xt, wt, bt)
    np.testing.assert_allclose(y, F.relu(z).permute(0, 2, 3, 1).detach().numpy(), rtol=1e-12, atol=1e-12)
    assert (mag >= np.abs(y)).all()
    # weight / bias gradient of the pre-activation
    dz = r.standard_normal((B, H - 2, W - 2, O))
    z.backward(torch.from_numpy(dz).permute(0, 3, 1, 2))
    dw, db, dw_mag, db_mag = ref.conv_c1_wgrad(x, dz)
    np.testing.assert_allclose(dw, wt.grad.view(O, 9).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12, atol=1e-12)
    assert (dw_mag >= np.abs(dw)).all() and (db_mag >= np.abs(db)).all()


def test_conv_c1_round_x_rounds_the_input_to_bf16():
    x = np.full((1, 3, 3), 1.0 + 2.0 ** -10)            # not a bf16 number: rounds to 1.0
    w = np.ones((8, 9))
    y, _ = ref.conv_c1_fwd(x, w, np.zeros(8), round_x=True)
    assert (y == 9.0).all()
    y, _ = ref.conv_c1_fwd(x, w, np.zeros(8))
    assert (y == 9.0 * (1.0 + 2.0 ** -10)).all()
    dw, _, _, _ = ref.conv_c1_wgrad(x, np.ones((1, 1, 1, 8)), round_x=True)
    assert (dw == 1.0).all()


def test_bias_relu_and_gated_backward_match_autograd():
    r = _rng(2)
    rows, C = 11, 24
    z = r.standard_normal((rows, C))
    b = r.standard_normal(C)
    y, mask, v = ref.bias_act_drop_fwd(z, b, True, 0.0, None)
    zt = torch.from_numpy(z).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    yt = F.relu(zt + bt)
    np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-15)
    assert (mask == (v > 0)).all()
    dy = r.standard_normal((rows, C))
    yt.backward(torch.from_numpy(dy))
    for gate in (mask.astype(bool), y > 0):
        dz, db, mag = ref.act_drop_bwd_bias(dy, gate, 1.0)
        np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-15)
        np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12)
        assert (mag >= np.abs(db)).all()
    # linear layer: no gate, the gradient passes through and dbias is its column sum
    dz, db, _ = ref.act_drop_bwd_bias(dy, None, 1.0)
    assert (dz == dy).all()
    np.testing.assert_allclose(db, dy.sum(0), rtol=1e-15)
    # the split-K slabs are summed before the bias
    slabs = r.standard_normal((3, rows, C))
    s, smag = ref.sum_slabs(slabs)
    np.testing.assert_allclose(s, slabs[0] + slabs[1] + slabs[2], rtol=1e-15)
    assert (smag >= np.abs(s)).all()


def test_max_pool_without_ties_matches_autograd():
    r = _rng(3)
    B, H, W, C = 2, 6, 10, 8
    z = r.standard_normal((B, H, W, C))                 # continuous draws: no ties
    b = r.standard_normal(C) * 0.3
    p, code, best = ref.pool_fwd(z, b, 0.0, None)
    zt = torch.from_numpy(z).permute(0, 3, 1, 2).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    pt = F.max_pool2d(F.relu(zt + bt[None, :, None, None]), 2)
    np.testing.assert_allclose(p, pt.permute(0, 2, 3, 1).detach().numpy(), rtol=1e-15)
    np.testing.assert_array_equal(best, F.max_pool2d(zt, 2).permute(0, 2, 3, 1).detach().numpy())
    dp = r.standard_normal(p.shape)
    pt.backward(torch.from_numpy(dp).permute(0, 3, 1, 2))
    dz, db, mag = ref.pool_bwd(dp, code, 1.0)
    # autograd sends the gradient of a window whose max + bias <= 0 nowhere; so does the code's flow bit
    np.testing.assert_allclose(dz, zt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-15)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12)
    assert (mag >= np.abs(db)).all()


def test_pool_tie_rule_and_code_bytes_worked_by_hand():
    # one image, one 2x2 window, 8 channels: the window values (00, 01, 10, 11) per channel
    wins = [(1, 1, 1, 1), (0, 2, 2, 1), (0, 1, 3, 3), (-1, -2, -3, -4), (5, 4, 5, 5), (-2, -1, -1, -2),
            (0, 0, 0, 7), (3, 3, 3, 3)]
    z = np.zeros((1, 2, 2, 8))
    for c, wv in enumerate(wins):
        for pos, val in enumerate(wv):
            z[0, pos >> 1, pos & 1, c] = val
    b = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, -3.0])
    p, code, best = ref.pool_fwd(z, b, 0.0, None)
    # first maximum in order 00, 01, 10, 11; flow bit 4 iff max + b > 0 (channel 7: 3 - 3 = 0 does not flow)
    assert list(best[0, 0, 0]) == [1, 2, 3, -1, 5, -1, 7, 3]
    assert list(code[0, 0, 0]) == [0 | 4, 1 | 4, 2 | 4, 0, 0 | 4, 1, 3 | 4, 0]
    assert list(p[0, 0, 0]) == [1, 2, 3, 0, 5, 0, 7, 0]
    # backward: the gradient of a flowing window lands on its argmax only; dbias sums the flowing ones
    dp = np.arange(1.0, 9.0).reshape(1, 1, 1, 8)
    dz, db, _ = ref.pool_bwd(dp, code, 2.0)
    want = np.zeros((1, 2, 2, 8))
    for c in range(8):
        if code[0, 0, 0, c] & 4:
            pos = code[0, 0, 0, c] & 3
            want[0, pos >> 1, pos & 1, c] = 2.0 * dp[0, 0, 0, c]
    assert (dz == want).all()
    assert list(db) == [2.0, 4.0, 6.0, 0.0, 10.0, 0.0, 14.0, 0.0]


def test_softmax_xent_matches_torch_cross_entropy():
    r = _rng(4)
    B, C = 37, 17
    lg = r.standard_normal((B, C)) * 3
    b = r.standard_normal(C)
    lab = r.integers(0, C, B)
    loss, d, db, hits, rows, v = ref.softmax_xent(lg, b, lab)
    lt = torch.from_numpy(lg).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    lref = F.cross_entropy(lt + bt, torch.from_numpy(lab))
    lref.backward()
    assert abs(loss - lref.item()) < 1e-12
    np.testing.assert_allclose(d, lt.grad.numpy(), rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-10, atol=1e-15)
    assert hits == int(((lt + bt).argmax(1) == torch.from_numpy(lab)).sum())
    np.testing.assert_allclose(rows.mean(), loss, rtol=1e-15)
    # no bias: the logits as given
    loss0, _, _, _, _, v0 = ref.softmax_xent(lg, None, lab)
    assert (v0 == lg).all()
    assert abs(loss0 - F.cross_entropy(torch.from_numpy(lg), torch.from_numpy(lab)).item()) < 1e-12


def test_softmax_hit_takes_the_first_maximum():
    lg = np.array([[1.0, 3.0, 3.0], [2.0, 2.0, 0.0], [0.0, 0.0, 0.0]])
    _, _, _, hits, _, _ = ref.softmax_xent(lg, None, np.array([2, 0, 0]))
    assert hits == 2          # row 0: argmax 1 != 2; row 1: argmax 0 == 0; row 2: argmax 0 == 0


def test_dropout_masks_come_from_the_host_generator(host):
    seed, step, rows, C, rate = 12345, 7, 5, 16, 0.5
    n = rows * C
    u = ref.uniform(host, seed, step, n)
    assert (u * 2 ** 24 == np.floor(u * 2 ** 24)).all() and (u >= 0).all() and (u < 1).all()
    # element e of the row-major matrix draws u(seed, step, e): an offset draw is the same sequence shifted
    np.testing.assert_array_equal(ref.uniform(host, seed, step, n - 3, idx0=3), u[3:])
    assert not np.array_equal(ref.uniform(host, seed, step + 1, n), u)
    z = np.ones((rows, C))
    y, mask, _ = ref.bias_act_drop_fwd(z, None, True, rate, u)
    assert (mask.reshape(-1) == (u >= rate)).all()
    assert (y.reshape(-1) == np.where(u >= rate, 2.0, 0.0)).all()
    # ReLU AND kept: a negative element never flows, whatever its draw
    y, mask, _ = ref.bias_act_drop_fwd(-z, None, True, rate, u)
    assert (mask == 0).all() and (y == 0).all()
    y, mask, _ = ref.bias_act_drop_fwd(-z, None, False, rate, u)
    assert (mask.reshape(-1) == (u >= rate)).all() and (y.reshape(-1) == np.where(u >= rate, -2.0, 0.0)).all()
    # rate 0 keeps everything and draws nothing
    y, mask, _ = ref.bias_act_drop_fwd(z, None, True, 0.0, None)
    assert (mask == 1).all() and (y == 1).all()
    # pool: the dropout index is the element index of the POOLED tensor
    B, H, W, Cp = 1, 4, 6, 8
    npool = B * (H // 2) * (W // 2) * Cp
    up = ref.uniform(host, seed, step, npool)
    p, code, _ = ref.pool_fwd(np.ones((B, H, W, Cp)), np.zeros(Cp), 0.25, up)
    assert ((code.reshape(-1) >> 2) == (up >= 0.25)).all()
    assert (p.reshape(-1) == np.where(up >= 0.25, 1.0 / 0.75, 0.0)).all()
