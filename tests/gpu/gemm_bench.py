"""wgmma GEMM of this repo vs cuBLAS (torch.matmul) at large shapes, bf16, on one H100.

    python tests/gpu/gemm_bench.py [--out gpurun_out/gemm_bench.json]

TFLOP/s = 2 M N K / CUDA-event time (median of 5 regions of `iters` launches, L2 flushed by rotating through
operand copies larger than the 50 MB L2); fractions are of MEASURED_PEAKS.json (bf16_tflops burst / sustained).
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tf_yarn_b200.ops.gemm import gemm_bf16  # noqa: E402


def bench(fn, n_sets, iters=10, regions=5):
    for i in range(3):
        fn(i % n_sets)
    torch.cuda.synchronize()
    ts = []
    for r in range(regions):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(iters):
            fn((r * iters + i) % n_sets)
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e) / iters)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/gemm_bench.json")
    a = ap.parse_args()
    peaks = {}
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peaks = json.load(open(p))
    burst, sust = peaks.get("bf16_tflops", 1590.0), peaks.get("bf16_tflops_sustained", 1400.0)
    rows = []
    for (M, N, K) in [(4096, 4096, 4096), (8192, 8192, 8192), (4096, 3072, 768), (4096, 768, 3072), (128, 128, 9216)]:
        per_set = (M * K + N * K) * 2
        n_sets = max(2, min(8, (160 << 20) // per_set + 1))
        A = [(torch.randn(M, K, device="cuda") * 0.1).bfloat16() for _ in range(n_sets)]
        Bm = [(torch.randn(N, K, device="cuda") * 0.1).bfloat16() for _ in range(n_sets)]
        ref = A[0].float() @ Bm[0].float().t()
        out = gemm_bf16(A[0], Bm[0], impl="1cta")
        torch.cuda.synchronize()
        err = (out.float() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        row = {"M": M, "N": N, "K": K, "rel_err": err}
        out2 = gemm_bf16(A[0], Bm[0], impl="2cta")
        torch.cuda.synchronize()
        row["rel_err_2cta"] = (out2.float() - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        for name, fn in (("ours", lambda i: gemm_bf16(A[i], Bm[i], impl="1cta")),
                         ("ours2", lambda i: gemm_bf16(A[i], Bm[i], impl="2cta")),
                         ("cublas", lambda i: torch.matmul(A[i], Bm[i].t()))):
            ms = bench(fn, n_sets)
            tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
            row[name + "_ms"] = ms
            row[name + "_tflops"] = tf
            row[name + "_of_burst_peak"] = tf / burst
            row[name + "_of_sustained_peak"] = tf / sust
        row["ours_vs_cublas"] = row["ours_tflops"] / row["cublas_tflops"]
        row["ours2_vs_cublas"] = row["ours2_tflops"] / row["cublas_tflops"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del A, Bm
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump({"peaks": {"burst": burst, "sustained": sust}, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
