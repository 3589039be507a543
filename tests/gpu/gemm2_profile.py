"""One launch each of the persistent two-warpgroup GEMM at 8192^3 and 4096^3 (bf16), for `ncu --set full -k regex:tfy_gemm2`.

    ncu --set full --clock-control none --import-source on -k regex:tfy_gemm2 -o gpurun_out/prof_gemm2 \
        python tests/gpu/gemm2_profile.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_yarn_b200.ops.gemm import gemm_bf16  # noqa: E402

for n in (8192, 4096):
    a = (torch.randn(n, n, device="cuda") * 0.1).bfloat16()
    b = (torch.randn(n, n, device="cuda") * 0.1).bfloat16()
    c = gemm_bf16(a, b, impl="2cta")
    torch.cuda.synchronize()
    print(n, float(c.float().abs().mean()))
