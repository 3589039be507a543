"""CPU tests of the float64 Dense-layer reference (tests/dense_reference.py): the reference itself against torch, the
exact tier's premise, bf16 rounding on hand-worked ties, and the split-K partition against the library's own rule."""
import numpy as np
import pytest
import torch

import dense_reference as ref


def test_gemm_matches_torch_float64():
    rng = np.random.default_rng(0)
    a, b, bias = rng.standard_normal((37, 72)), rng.standard_normal((20, 72)), rng.standard_normal(20)
    ta, tb, tbias = (torch.from_numpy(t) for t in (a, b, bias))
    for relu in (False, True):
        got, mag = ref.gemm(a, b, bias, relu)
        want = ta @ tb.T + tbias
        np.testing.assert_allclose(got, (want.relu() if relu else want).numpy(), rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(mag, (ta.abs() @ tb.abs().T + tbias.abs()).numpy(), rtol=1e-13)
    got, _ = ref.gemm(a, b)
    np.testing.assert_allclose(got, (ta @ tb.T).numpy(), rtol=1e-13, atol=1e-13)


def test_splitk_slabs_sum_to_the_product():
    rng = np.random.default_rng(1)
    a, b = rng.standard_normal((9, 9224)), rng.standard_normal((5, 9224))
    slabs = ref.splitk_slabs(a, b, 24)
    assert slabs.shape == (21, 9, 5)
    np.testing.assert_allclose(slabs.sum(0), a @ b.T, rtol=1e-10, atol=1e-10)
    # 145 tiles, 7 per slice: the last slice has 5 tiles, the last of them 8 wide
    assert ref.k_slices(9224, 24)[-1] == (8960, 9224)


def test_dense_backward_matches_torch_float64():
    rng = np.random.default_rng(2)
    dh, x, w = rng.standard_normal((13, 24)), rng.standard_normal((13, 40)), rng.standard_normal((24, 40))
    dw, dx, dw_mag, dx_mag = ref.dense_bwd(dh, x, w)
    tdh, tx, tw = (torch.from_numpy(t).requires_grad_(True) for t in (dh, x, w))
    # y = x W^T; with upstream gradient dh: dW = dh^T x, dx = dh W
    (tx @ tw.T).backward(tdh.detach())
    np.testing.assert_allclose(dw, tw.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx, tx.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dw_mag, np.abs(dh).T @ np.abs(x))
    np.testing.assert_allclose(dx_mag, np.abs(dh) @ np.abs(w))


@pytest.mark.parametrize("weighted", [False, True])
def test_dense_head_matches_autograd(weighted):
    rng = np.random.default_rng(3)
    B, K, C = 23, 16, 5
    h = np.maximum(rng.standard_normal((B, K)), 0)
    w2, b2 = rng.standard_normal((C, K)) * 0.3, rng.standard_normal(C) * 0.1
    labels = rng.integers(0, C, B)
    mask1 = rng.integers(0, 256, (B, K)).astype(np.uint8)
    scale1 = 1.5
    sw = rng.random(B) + 0.5 if weighted else None
    cw = rng.random(C) + 0.5 if weighted else None
    if weighted:
        labels[4] = C                                           # outside [0, C): weight 1 from the class table
    out = ref.dense_head(h, w2, b2, labels, mask1, scale1, sw, cw)

    th, tw, tb = (torch.from_numpy(t).requires_grad_(True) for t in (h, w2, b2))
    logits = th @ tw.T + tb
    ok = torch.from_numpy((labels >= 0) & (labels < C))
    lab = torch.from_numpy(np.where(labels < C, labels, 0))
    row = torch.nn.functional.cross_entropy(logits, lab, reduction="none") * ok
    wr = torch.ones(B, dtype=torch.float64)
    if weighted:
        wr = torch.from_numpy(sw) * torch.where(ok, torch.from_numpy(cw)[lab], torch.ones(B, dtype=torch.float64))
    # a row whose label matches no class adds nothing to the loss, but its dlogits row is p (no onehot term): the
    # gradient of logsumexp(v), which the objective below adds for those rows only
    lse_only = torch.logsumexp(logits, 1) * ~ok
    ((wr * (row + lse_only)).sum() / B).backward()
    np.testing.assert_allclose(out["loss"], float((wr * row).sum().detach() / B), rtol=1e-12)
    np.testing.assert_allclose(out["dw2"], tw.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(out["db2"], tb.grad.numpy(), rtol=1e-10, atol=1e-12)
    gate = (mask1 & 1) * scale1
    np.testing.assert_allclose(out["dh"], th.grad.numpy() * gate, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(out["db1"], (th.grad.numpy() * gate).sum(0), rtol=1e-10, atol=1e-12)
    hit = ok.numpy() & (logits.detach().numpy().argmax(1) == labels)
    np.testing.assert_array_equal(out["stats"], [hit.sum(), B, (wr.numpy() * hit).sum(), wr.numpy().sum()])
    # without a mask there is neither a gate nor the scale
    np.testing.assert_allclose(ref.dense_head(h, w2, b2, labels, None, scale1, sw, cw)["dh"], th.grad.numpy(),
                               rtol=1e-10, atol=1e-12)


def test_exact_tier_generator_rejects_large_sums():
    rng = np.random.default_rng(4)
    a, b = ref.integers(rng, (4, 9224)), ref.integers(rng, (3, 9224))
    mag = ref.assert_exact(a, b, ref.integers(rng, (3,)))
    assert mag.max() < 2 ** 22
    with pytest.raises(AssertionError):
        ref.assert_exact(np.full((1, 20000), 15.0), np.full((1, 20000), 15.0))
    with pytest.raises(AssertionError):
        ref.assert_exact(np.full((1, 8), 0.5), np.ones((1, 8)))


@pytest.mark.parametrize("K", [8, 264, 1680, 9224])
def test_exact_tier_sums_do_not_depend_on_order(K):
    """The premise of the exact tier: randomly ordered fp32 sums of the products equal the float64 sum."""
    rng = np.random.default_rng(K)
    a, b = ref.integers(rng, (6, K), 0, 15), ref.integers(rng, (4, K))
    ref.assert_exact(a, b)
    want = a @ b.T
    prods = (a[:, None, :] * b[None, :, :]).astype(np.float32)  # exact: |product| <= 225
    for _ in range(5):
        perm = rng.permutation(K)
        acc = np.zeros(want.shape, np.float32)
        for k in perm:
            acc = acc + prods[:, :, k]
        np.testing.assert_array_equal(acc.astype(np.float64), want)
        # a random split into slabs summed in a random order is the same number too
        cuts = np.sort(rng.choice(np.arange(1, K), size=min(7, K - 1), replace=False))
        parts = [p.sum(-1, dtype=np.float32) for p in np.split(prods[:, :, perm], cuts, axis=-1)]
        acc = np.zeros(want.shape, np.float32)
        for i in rng.permutation(len(parts)):
            acc = acc + parts[i]
        np.testing.assert_array_equal(acc.astype(np.float64), want)


def test_bf16_round_hand_worked_ties():
    # bf16 keeps 8 significant bits: between 256 and 512 the step is 2, between 512 and 1024 it is 4
    x = np.array([257, 259, 261, 263, 513, 514, 515, 518, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -257, -259, 256, 258],
                 np.float64)
    want = np.array([256, 260, 260, 264, 512, 512, 516, 520, 1.0, 1.0 + 2 ** -6, -256, -260, 256, 258], np.float64)
    np.testing.assert_array_equal(ref.bf16_round(x), want)
    # truncation would give 258 -> 258 but 259 -> 258, 263 -> 262: the ties above are what pins the rounding mode
    assert ref.bf16_round(np.array([259.0]))[0] != 258.0


def test_fused_epilogue_is_fp32_step_by_step():
    acc = np.array([[257.0, -3.0, 300.0, 7.0]])
    y, mask = ref.fused_epilogue(acc, np.array([2.0, 1.0, -1.0, 0.0]), True, 0.25, np.array([0.5, 0.9, 0.1, 0.3]))
    s = np.float32(1.0) / np.float32(0.75)
    np.testing.assert_array_equal(y[0], ref.bf16_round(np.array([np.float32(259) * s, 0, 0, np.float32(7) * s])))
    np.testing.assert_array_equal(mask[0], [1, 0, 0, 1])
    assert ref.keep_scale_f32(0.25) == np.float32(4.0 / 3.0) and ref.keep_scale_f32(0.0) == 1.0


def test_slab_sum_is_left_to_right():
    s = np.array([[1.0], [2.0 ** 24], [1.0], [-(2.0 ** 24)]], np.float32)
    # ((1 + 2^24) + 1) - 2^24 in fp32: 1 + 2^24 rounds to 2^24, + 1 again, - 2^24 = 0; any other order differs
    assert ref.sum_slabs_f32(s)[0] == 0.0
    assert ref.sum_slabs_f32(s[[1, 0, 2, 3]])[0] == 0.0 and ref.sum_slabs_f32(s[[0, 2, 1, 3]])[0] == 2.0


def test_gather_x_zero_rows_and_pad():
    tables = [np.arange(3 * 64, dtype=np.float64).reshape(3, 64)]
    x = ref.gather_x(tables, np.array([[2, -1, 3]]), np.ones((3, 2)), 72)
    np.testing.assert_array_equal(x[0, :64], tables[0][2])
    assert not x[1:, :64].any() and (x[:, 64:66] == 1).all() and not x[:, 66:].any()


def test_k_slices_match_the_library():
    """The partition the reference uses is the one tfy_gemm_bf16_splitk_slabs reports, for K <= 20000, split <= 200."""
    from tf_yarn_b200.ops import gemm, native  # noqa: F401  (declares tfy_gemm_bf16_splitk_slabs)
    try:
        lib = native.load()
    except Exception as exc:  # noqa: BLE001
        pytest.skip(f"native library not built: {exc}")
    for K in list(range(8, 1025, 8)) + list(range(1032, 20001, 248)) + [9216, 9224, 20000]:
        k_tiles = -(-K // 64)
        for split in list(range(0, 40)) + [63, 64, 100, 144, 145, 199, 200]:
            sl = ref.k_slices(K, split)
            assert len(sl) == int(lib.tfy_gemm_bf16_splitk_slabs(K, split)), (K, split)
            assert sl[0][0] == 0 and sl[-1][1] == K and all(p[1] == q[0] for p, q in zip(sl, sl[1:]))
            assert all(lo % 64 == 0 and hi > lo for lo, hi in sl)
            assert len(sl) <= max(1, min(max(split, 1), k_tiles))
