"""Python entry points of the wgmma GEMMs: one tile per CTA with split-K and a remote-B operand
(``ops/csrc/tfy_gemm.cu``) and the persistent two-warpgroup kernel for large problems (``ops/csrc/tfy_gemm2.cu``)."""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from tf_yarn_b200.ops import native

_vp, _i = ctypes.c_void_p, ctypes.c_int
native.declare("tfy_gemm_bf16", [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp])
native.declare("tfy_gemm2_bf16", [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp])
native.declare("tfy_gemm_bf16_splitk_slabs", [_i, _i])
native.declare("tfy_splitk_sum_f32", [_vp, _vp, _i, ctypes.c_size_t, ctypes.c_size_t, _vp])

# from this many rows / columns on, the persistent kernel (tfy_gemm2.cu: two warpgroups, 128x256 tiles) is used
GEMM2_MIN_DIM = 512


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
              out: Optional[torch.Tensor] = None, split_k: int = 1, b_ptr: Optional[int] = None,
              b_rows: Optional[int] = None, b_ld: Optional[int] = None, impl: str = "auto") -> torch.Tensor:
    """``out[M,N] = act(a[M,K] @ b[N,K]^T + bias[N])`` on the Hopper tensor cores (bf16 in, fp32 acc).

    ``b`` is row-major [N, K] (the layout of a ``torch.nn.Linear`` weight).  ``b_ptr`` / ``b_rows`` /
    ``b_ld`` let the caller pass a raw device address instead -- e.g. a parameter-server shard mapped
    over NVLink (the K5 pull path); then ``b`` may be None.
    With ``split_k > 1`` the K-slices' fp32 partial products are summed in slice order (the same result on every
    run) and ``out`` is fp32.
    ``impl``: "auto" (persistent 128x256-tile kernel for large M and N, one-tile-per-CTA kernel otherwise), "1cta", or
    "2cta" (the persistent kernel; the name is kept for existing callers).
    """
    lib = native.load()
    assert a.dtype == torch.bfloat16 and a.dim() == 2 and a.stride(1) == 1
    M, K = a.shape
    if b is not None:
        assert b.dtype == torch.bfloat16 and b.dim() == 2 and b.stride(1) == 1 and b.shape[1] == K
        N, ldb, bp = b.shape[0], b.stride(0), b.data_ptr()
    else:
        N, ldb, bp = int(b_rows), int(b_ld or K), int(b_ptr)
    s = torch.cuda.current_stream().cuda_stream
    # the persistent kernel requires an output row pitch that is a multiple of 8 elements ("auto" falls back to the
    # one-tile-per-CTA kernel, whose epilogue handles any pitch; an explicit "2cta" fails loudly)
    ldc_ok = (out.stride(0) if out is not None else N) % 8 == 0
    if (split_k <= 1 and impl != "1cta" and (impl == "2cta" or (M >= GEMM2_MIN_DIM and N >= GEMM2_MIN_DIM and ldc_ok))
            and os.environ.get("TFY_GEMM2", "1") != "0"):
        if out is None:
            out = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
        assert out.dtype == torch.bfloat16 and out.stride(1) == 1
        rc = lib.tfy_gemm2_bf16(a.data_ptr(), bp, out.data_ptr(), bias.data_ptr() if bias is not None else None, M, N, K,
                                a.stride(0), ldb, out.stride(0), int(relu), s)
        native.check(rc, "tfy_gemm2_bf16")
        return out
    if split_k > 1:
        if out is None:
            out = torch.empty((M, N), dtype=torch.float32, device=a.device)
        assert out.dtype == torch.float32 and out.is_contiguous()
        slabs = torch.empty((int(lib.tfy_gemm_bf16_splitk_slabs(K, split_k)), M, N), dtype=torch.float32,
                            device=a.device)
        rc = lib.tfy_gemm_bf16(a.data_ptr(), bp, None, slabs.data_ptr(), None, M, N, K, a.stride(0), ldb, N, 0,
                               split_k, s)
        native.check(rc, "tfy_gemm_bf16")
        rc = lib.tfy_splitk_sum_f32(slabs.data_ptr(), out.data_ptr(), slabs.shape[0], M * N, M * N, s)
        native.check(rc, "tfy_splitk_sum_f32")
        return out
    else:
        if out is None:
            out = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
        assert out.dtype == torch.bfloat16 and out.stride(1) == 1
        rc = lib.tfy_gemm_bf16(a.data_ptr(), bp, out.data_ptr(), None, bias.data_ptr() if bias is not None else None,
                               M, N, K, a.stride(0), ldb, out.stride(0), int(relu), 1, s)
    native.check(rc, "tfy_gemm_bf16")
    return out
