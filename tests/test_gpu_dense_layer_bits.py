"""Bit-level GPU tests of the Dense-layer kernels at the MNIST step's shapes (batch 128, 9216 -> 128).

The Dense backward (tfy_dense_bwd) is pinned by SHA-256 digests of its bf16 outputs in
tests/golden/dense_bwd_b128_sha256.json: wgmma does not accumulate as a sequential fp32 sum, so a float reference
cannot show that an epilogue or staging change left every byte where it was.  The two-launch split-K forward (the
GEMM into fp32 slabs, then tfy_bias_act_drop_fwd_f32) is compared byte for byte with the one-launch
tfy_gemm_bf16_splitk_fused, whose CTAs sum the same slabs in the same order themselves.
"""
import ctypes
import hashlib
import json
import os

import pytest
import torch

from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dense_bwd_b128_sha256.json")
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.ops import native
    return native.load()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _sha(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _bwd(lib, B, U, I, seed, want_dx):
    """tfy_dense_bwd on inputs seeded on the CPU: dh ~ N(0, 0.5), x = relu(N(0, 1)) (pooled activations), W ~ N(0, 0.02)."""
    g = torch.Generator().manual_seed(seed)
    dh = (torch.randn(B, U, generator=g) * 0.5).to(BF16).cuda()
    x = torch.randn(B, I, generator=g).relu().to(BF16).cuda()
    w = (torch.randn(U, I, generator=g) * 0.02).to(BF16).cuda()
    dw = torch.full((U, I), 7.0, dtype=BF16, device="cuda")
    dx = torch.full((B, I), 7.0, dtype=BF16, device="cuda") if want_dx else None
    assert lib.tfy_dense_bwd(dh.data_ptr(), x.data_ptr(), w.data_ptr(), dw.data_ptr(),
                             dx.data_ptr() if want_dx else None, B, U, I, _s()) == 0
    torch.cuda.synchronize()
    return dw, dx


def dense_bwd_digests(lib):
    """SHA-256 of tfy_dense_bwd's dW and dx: the single-shot kernel at the MNIST layer's 128 x 128 x 9216, with and
    without dx (the first-layer case), and the tiled kernel at batch 256, 256 units, 2048 in-features."""
    out = {}
    dw, dx = _bwd(lib, 128, 128, 9216, 23, True)
    out["b128_dw"], out["b128_dx"] = _sha(dw), _sha(dx)
    dw, _ = _bwd(lib, 128, 128, 9216, 23, False)
    out["b128_no_dx_dw"] = _sha(dw)
    dw, dx = _bwd(lib, 256, 256, 2048, 29, True)
    out["tiled_b256_dw"], out["tiled_b256_dx"] = _sha(dw), _sha(dx)
    return out


def test_dense_backward_bit_identical_to_recorded_digest(lib):
    with open(GOLDEN) as f:
        want = json.load(f)
    got = dense_bwd_digests(lib)
    assert got == {k: want[k] for k in got}


@pytest.mark.parametrize("drop,relu", [(0.5, 1), (0.0, 1), (0.25, 0)])
def test_one_launch_forward_is_byte_equal_to_two_launch_path(lib, drop, relu):
    """Activations and gate mask of the split-K GEMM with the fused bias / ReLU / dropout epilogue equal, byte for
    byte, the split-K GEMM into slabs followed by tfy_bias_act_drop_fwd_f32, at the engine's split of 24 K-slices;
    the tile counters are left at zero for the next launch."""
    from tf_yarn_b200.ops import native
    B, U, K = 128, 128, 9216
    split = fastpath.FastSequentialEngine._split_k(B, U, K)
    slabs = int(lib.tfy_gemm_bf16_splitk_slabs(K, split))
    assert slabs == 24
    g = torch.Generator().manual_seed(31)
    x = torch.randn(B, K, generator=g).relu().to(BF16).cuda()
    w = (torch.randn(U, K, generator=g) * 0.02).to(BF16).cuda()
    bias = (torch.randn(U, generator=g) * 0.1).to(BF16).cuda()
    h = native.OptHyper(1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 5, 0, 0, 0)
    hp = torch.frombuffer(bytearray(bytes(h)), dtype=torch.uint8).cuda()
    seed = 1234

    acc = torch.zeros(slabs, B, U, dtype=torch.float32, device="cuda")
    y2 = torch.full((B, U), 3.0, dtype=BF16, device="cuda")
    m2 = torch.full((B, U), 9, dtype=torch.uint8, device="cuda")
    assert lib.tfy_gemm_bf16(x.data_ptr(), w.data_ptr(), None, acc.data_ptr(), None, B, U, K, K, K, U, 0, split,
                             _s()) == 0
    assert lib.tfy_bias_act_drop_fwd_f32(acc.data_ptr(), bias.data_ptr(), y2.data_ptr(), m2.data_ptr(), B, U, relu,
                                         ctypes.c_float(drop), seed, hp.data_ptr(), slabs, _s()) == 0

    acc1 = torch.zeros(slabs, B, U, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    y1 = torch.full((B, U), 5.0, dtype=BF16, device="cuda")
    m1 = torch.full((B, U), 7, dtype=torch.uint8, device="cuda")
    for _ in range(2):           # the second launch reuses the counters the first one re-armed
        assert lib.tfy_gemm_bf16_splitk_fused(x.data_ptr(), w.data_ptr(), acc1.data_ptr(), cnt.data_ptr(),
                                              bias.data_ptr(), y1.data_ptr(), m1.data_ptr(), B, U, K, K, K, relu,
                                              ctypes.c_float(drop), seed, hp.data_ptr(), split, _s()) == 0
        torch.cuda.synchronize()
        assert torch.equal(y1.view(torch.int16), y2.view(torch.int16))
        assert torch.equal(m1, m2)
        assert int(cnt.abs().sum().item()) == 0
    if drop > 0:
        assert float((m1 == 0).float().mean()) > drop - 0.1
