"""Deferred conv2 weight-gradient reduction (ops/csrc/tfy_conv.cu): the weight-gradient kernel only stores its per-CTA
fp32 partials and the un-pool data-gradient kernel that follows reduces them.  dW, db and dx must be the same bits as
the weight-gradient kernel's own grid-barrier reduction followed by the plain data-gradient kernel.

On a 132-SM H100, batches 2, 32, 128, 160 and 232 give 9, 72, 116, 120 and 131 partials: serial sums and every
split of the partial list into thread groups, including the shorter last slice.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

H = W = 26
BATCHES = [2, 32, 128, 160, 232]


def _lib():
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(B, H, W, 32, generator=g).relu().to(torch.bfloat16)
    w = (torch.randn(64, 3, 3, 32, generator=g) * 0.06).to(torch.bfloat16)
    dp = (torch.randn(B, 12, 12, 64, generator=g) * 0.5).to(torch.bfloat16)
    code = torch.randint(0, 8, (B, 12, 12, 64), generator=g, dtype=torch.uint8)
    return a.cuda(), w.cuda(), dp.cuda(), code.cuda()


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("B", BATCHES)
def test_deferred_reduction_bit_identical_to_in_kernel_reduction(B):
    lib = _lib()
    a, w, dp, code = _inputs(B, seed=B)
    scale = ctypes.c_float(1.0 / 0.75)
    n = int(lib.tfy_conv3x3_c32_wgrad_scratch_elems())
    out = {}
    for mode in ("in_kernel", "deferred"):
        part = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
        dw = torch.full((64, 3, 3, 32), float("nan"), dtype=torch.bfloat16, device="cuda")
        db = torch.full((64,), float("nan"), dtype=torch.bfloat16, device="cuda")
        dx = torch.full((B, H, W, 32), float("nan"), dtype=torch.bfloat16, device="cuda")
        if mode == "in_kernel":
            sync = torch.zeros(1024, dtype=torch.int32, device="cuda")
            assert lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                    part.data_ptr(), dw.data_ptr(), db.data_ptr(), sync.data_ptr(),
                                                    B, H, W, _stream()) == 0
            assert lib.tfy_conv3x3_c32_dgrad_unpool(dp.data_ptr(), code.data_ptr(), scale, w.data_ptr(),
                                                    a.data_ptr(), dx.data_ptr(), B, H, W, _stream()) == 0
        else:
            n_part = ctypes.c_int(0)
            assert lib.tfy_conv3x3_c32_wgrad_unpool_deferred(a.data_ptr(), dp.data_ptr(), code.data_ptr(), scale,
                                                             part.data_ptr(), B, H, W, None, ctypes.byref(n_part),
                                                             _stream()) == 0
            assert 1 <= n_part.value <= 160
            assert lib.tfy_conv3x3_c32_dgrad_unpool_reduce(dp.data_ptr(), code.data_ptr(), scale, w.data_ptr(),
                                                           a.data_ptr(), dx.data_ptr(), B, H, W, part.data_ptr(),
                                                           n_part.value, dw.data_ptr(), db.data_ptr(),
                                                           _stream()) == 0
        torch.cuda.synchronize()
        out[mode] = (dw, db, dx)
    for name, ref, got in zip(("dw", "db", "dx"), out["in_kernel"], out["deferred"]):
        assert not torch.isnan(got.float()).any(), name
        assert torch.equal(_bits(ref), _bits(got)), name


def test_reduce_entry_rejects_a_partial_count_outside_the_scratch():
    lib = _lib()
    a, w, dp, code = _inputs(2, seed=0)
    part = torch.zeros(int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()), dtype=torch.float32, device="cuda")
    dw = torch.zeros(64, 3, 3, 32, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    dx = torch.zeros(2, H, W, 32, dtype=torch.bfloat16, device="cuda")
    for bad in (0, 161):
        assert lib.tfy_conv3x3_c32_dgrad_unpool_reduce(dp.data_ptr(), code.data_ptr(), ctypes.c_float(1.0),
                                                       w.data_ptr(), None, dx.data_ptr(), 2, H, W, part.data_ptr(),
                                                       bad, dw.data_ptr(), db.data_ptr(), _stream()) != 0
