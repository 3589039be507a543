"""conv2 forward and weight-gradient kernels (ops/csrc/tfy_conv.cu) at the batch sizes that exercise their
per-CTA patch schedules, against fp32 references, a recorded bit-exact fprop digest, and themselves.

On a 132-SM H100, batches 2, 32, 128, 160 and 232 give 1, 2, 5, 6 and 8 patches per CTA: the first patch, an odd
tail and a partial group of the MMA pipelines.
"""
import ctypes
import hashlib
import json
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

H = W = 26
BATCHES = [2, 32, 128, 160, 232]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv2_fprop_b128_sha256.json")


def _lib():
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, seed=0):
    """Seeded on the CPU, so the bytes do not depend on the device's random number generator."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(B, H, W, 32, generator=g).relu().to(torch.bfloat16)
    w = (torch.randn(64, 3, 3, 32, generator=g) * 0.06).to(torch.bfloat16)
    bias = (torch.randn(64, generator=g) * 0.1).to(torch.bfloat16)
    dp = (torch.randn(B, 12, 12, 64, generator=g) * 0.5).to(torch.bfloat16)
    return a.cuda(), w.cuda(), bias.cuda(), dp.cuda()


def run_fprop(lib, a, w, bias, drop, seed=1234):
    B = a.shape[0]
    pooled = torch.full((B, 12, 12, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    code = torch.full((B, 12, 12, 64), 0xff, dtype=torch.uint8, device="cuda")
    rc = lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(), pooled.data_ptr(),
                                      code.data_ptr(), B, H, W, drop, seed, None, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    return pooled, code


def run_wgrad(lib, a, dp, code, scale):
    B = a.shape[0]
    part = torch.full((int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()),), float("nan"), dtype=torch.float32,
                      device="cuda")
    sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
    dw = torch.zeros(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    rc = lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), code.data_ptr(), ctypes.c_float(scale),
                                          part.data_ptr(), dw.data_ptr(), db.data_ptr(), sync.data_ptr(), B, H, W,
                                          _stream())
    torch.cuda.synchronize()
    assert rc == 0
    return dw, db


def fprop_digest(lib):
    """SHA-256 of the pooled output and code bytes at batch 128 with dropout on (the recorded fixture)."""
    a, w, bias, _ = _inputs(128, seed=11)
    pooled, code = run_fprop(lib, a, w, bias, 0.5, seed=1234)
    return {"pooled": hashlib.sha256(pooled.view(torch.uint8).cpu().numpy().tobytes()).hexdigest(),
            "code": hashlib.sha256(code.cpu().numpy().tobytes()).hexdigest()}


def _close(got, ref, tol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs().max().item()
    assert err <= tol * (ref.abs().max().item() + 1e-6), f"max err {err} vs ref max {ref.abs().max().item()}"


@pytest.mark.parametrize("B", BATCHES)
def test_fprop_matches_fp32_reference(B):
    lib = _lib()
    a, w, bias, _ = _inputs(B)
    pooled, code = run_fprop(lib, a, w, bias, 0.0)
    z = F.conv2d(a.permute(0, 3, 1, 2).float(), w.permute(0, 3, 1, 2).float())
    zp, zi = F.max_pool2d(z, 2, return_indices=True)
    ref = (zp + bias.float().view(1, -1, 1, 1)).relu().permute(0, 2, 3, 1)
    _close(pooled, ref, 0.01)
    zi = zi.permute(0, 2, 3, 1)
    pos = ((zi // 24) % 2) * 2 + (zi % 2)
    assert ((code & 3).long() == pos).float().mean().item() > 0.995
    assert (((code >> 2) & 1).bool() == (ref > 0)).float().mean().item() > 0.995


def test_fprop_bit_identical_to_recorded_digest():
    with open(GOLDEN) as f:
        want = json.load(f)
    assert fprop_digest(_lib()) == {"pooled": want["pooled"], "code": want["code"]}


@pytest.mark.parametrize("B", BATCHES)
def test_wgrad_matches_fp32_reference(B):
    lib = _lib()
    a, w, bias, dp = _inputs(B)
    _, code = run_fprop(lib, a, w, bias, 0.25)
    scale = 1.0 / 0.75
    dw, db = run_wgrad(lib, a, dp, code, scale)
    # un-pool in fp32: dz[2py+dy, 2px+dx, o] = dp * scale where the code byte's gate is set and its argmax is there
    gated = torch.where((code & 4).bool(), (dp.float() * scale).to(torch.bfloat16).float(), 0.0)
    pos = (code & 3).long()
    dz = torch.zeros(B, 24, 24, 64, device="cuda")
    for dy in range(2):
        for dx in range(2):
            dz[:, dy::2, dx::2, :] = torch.where(pos == dy * 2 + dx, gated, 0.0)
    dw_ref = torch.nn.grad.conv2d_weight(a.permute(0, 3, 1, 2).float(), (64, 32, 3, 3), dz.permute(0, 3, 1, 2))
    _close(dw, dw_ref.permute(0, 2, 3, 1), 0.01)
    _close(db, gated.sum((0, 1, 2)), 0.01)


def test_wgrad_two_runs_bit_identical():
    lib = _lib()
    a, w, bias, dp = _inputs(128, seed=5)
    _, code = run_fprop(lib, a, w, bias, 0.5)
    dw0, db0 = run_wgrad(lib, a, dp, code, 2.0)
    dw1, db1 = run_wgrad(lib, a, dp, code, 2.0)
    assert torch.equal(dw0.view(torch.int16), dw1.view(torch.int16))
    assert torch.equal(db0.view(torch.int16), db1.view(torch.int16))
