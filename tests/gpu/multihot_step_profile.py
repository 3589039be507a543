"""Time the multi-hot embedding path of one wide-and-deep step per kernel (CUDA events; torch.profiler, CUDA activity).

    python tests/gpu/multihot_step_profile.py [out_dir]

Shapes of bench/wide_deep.py: 26 hashed columns of 100k buckets, batch 512, deep embeddings of 64, 13 numeric
features, first hidden layer 1024 wide.  For L ids per example (L = 1, 4, 16; weighted and unweighted, sqrtn deep and
mean wide) it times:
  deep forward : tfy_ps_multi_bag_weighted into the bf16 activation buffer, then tfy_gemm_bf16 against the shadow
                 (and, for L = 1, K5 = tfy_ps_gather_gemm, which fuses the two)
  deep backward: tfy_dense_bwd, then tfy_ps_multi_push_rows_weighted out of the dx column slices (Adagrad)
  wide         : tfy_ps_multi_bag_weighted with col_stride 0 and its push ([V, 1] FTRL tables)
Buffers are local: the peer latency of a multi-GPU job is not in these numbers.  Gathered bytes are the fp32 rows the
bag reads (present or not: every slot's id is read, a row only when present; the count is of the rows).  The card's
name and power limit are read in the same run.
"""
import collections
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

from tf_yarn_b200.estimator import ps_hbm  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402
from tf_yarn_b200.ops.gemm import gemm_bf16  # noqa: E402

T, V, B, D, N_NUM, N = 26, 100_000, 512, 64, 13, 1024
KP = (T * D + N_NUM + 7) // 8 * 8
REPS = 200


def _time(fn, reps=REPS):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def _kernels(fn, reps=20):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    kern = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = ev.name[:80]
            kern[k][0] += 1
            kern[k][1] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return {k: {"per_call": c / reps, "mean_us": round(t / c, 2)} for k, (c, t) in kern.items()}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def main(out_dir):
    lib = native.load()
    dev = torch.device("cuda")
    s = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(0)
    deep = [torch.randn(V * D, device=dev, generator=g) * 0.05 for _ in range(T)]
    deep_acc = [torch.full((V * D,), 0.1, device=dev) for _ in range(T)]
    wide = [torch.zeros(V, device=dev) for _ in range(3 * T)]           # w, n, z of FTRL
    ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=dev)   # noqa: E731
    deep_p, deep_s1 = ptr(deep), ptr(deep_acc)
    wide_p, wide_s1, wide_s2 = ptr(wide[:T]), ptr(wide[T:2 * T]), ptr(wide[2 * T:])
    shadow = (torch.randn(N, KP, device=dev, generator=g) * 0.02).to(torch.bfloat16)
    bias = torch.zeros(N, dtype=torch.bfloat16, device=dev)
    numeric = torch.randn(B, N_NUM, device=dev, generator=g)
    dy = (torch.randn(B, N, device=dev, generator=g) * 0.01).to(torch.bfloat16)
    adam = torch.ones(2, device=dev)
    results = {}
    for L in (1, 4, 16):
        ids = torch.randint(0, V, (T, B, L), device=dev, generator=g)
        if L > 1:                                                       # ragged lists padded with -1
            ids[torch.rand(T, B, L, device=dev, generator=g) < 0.25] = -1
        for weighted in (False, True):
            w = torch.rand(T, B, L, device=dev, generator=g) if weighted else None
            xbuf = torch.zeros(B, KP, dtype=torch.bfloat16, device=dev)
            f = torch.empty(T, B, device=dev)
            fw = torch.empty(T, B, device=dev)
            wide_out = torch.empty(B, 1, device=dev)
            dx = (torch.randn(B, KP, device=dev, generator=g) * 0.01).to(torch.bfloat16)   # until deep_bwd writes it
            dw = torch.empty(N, KP, dtype=torch.bfloat16, device=dev)
            dwide = torch.randn(B, 1, device=dev, generator=g) * 0.1

            def deep_bag():
                ps_hbm.weighted_bag(lib, deep_p, ids, w, 2, D, V, xbuf, KP, D, f, numeric)

            def deep_fwd():
                deep_bag()
                gemm_bf16(xbuf, None, bias=bias, b_ptr=shadow.data_ptr(), b_rows=N, b_ld=KP, impl="1cta")

            sc = ps_hbm.push_rows_scratch(lib, T * B * L, dev)    # one scratch, outside the timed calls

            def deep_push():
                native.check(lib.tfy_ps_multi_push_rows_weighted(
                    deep_p.data_ptr(), deep_s1.data_ptr(), None, ids.data_ptr(), dx.data_ptr(), 1, B, T, D, V,
                    native.OPT_ADAGRAD, 0.05, 1e-7, 0.0, 0.0, 0.0, 1.0, adam.data_ptr(), KP, D, L,
                    w.data_ptr() if w is not None else None, f.data_ptr(), 2, sc.data_ptr(), sc.numel(), s()),
                    "tfy_ps_multi_push_rows_weighted")

            def deep_bwd():
                native.check(lib.tfy_dense_bwd(dy.data_ptr(), xbuf.data_ptr(), shadow.data_ptr(), dw.data_ptr(),
                                               dx.data_ptr(), B, N, KP, s()), "tfy_dense_bwd")
                deep_push()

            def wide_bag():
                ps_hbm.weighted_bag(lib, wide_p, ids, w, 1, 1, V, wide_out, 1, 0, fw)

            def wide_push():
                native.check(lib.tfy_ps_multi_push_rows_weighted(
                    wide_p.data_ptr(), wide_s1.data_ptr(), wide_s2.data_ptr(), ids.data_ptr(), dwide.data_ptr(), 0, B,
                    T, 1, V, native.OPT_FTRL, 0.05, 0.0, 0.001, 0.01, 0.5, 1.0, adam.data_ptr(), 1, 0, L,
                    w.data_ptr() if w is not None else None, fw.data_ptr(), 1, sc.data_ptr(), sc.numel(), s()),
                    "tfy_ps_multi_push_rows_weighted")

            deep_fwd()
            wide_bag()
            torch.cuda.synchronize()
            present = int(((ids >= 0) & ((w != 0) if w is not None else True)).sum())
            r = {"present_ids": present, "gathered_bytes_deep": present * D * 4, "gathered_bytes_wide": present * 4,
                 "deep_bag_us": _time(deep_bag), "deep_fwd_us": _time(deep_fwd), "deep_push_us": _time(deep_push),
                 "deep_bwd_us": _time(deep_bwd), "wide_bag_us": _time(wide_bag), "wide_push_us": _time(wide_push)}
            if L == 1 and not weighted:
                ids2 = ids[:, :, 0].contiguous()
                y = torch.empty(B, N, dtype=torch.bfloat16, device=dev)

                def k5():
                    native.check(lib.tfy_ps_gather_gemm(shadow.data_ptr(), deep_p.data_ptr(), ids2.data_ptr(),
                                                        numeric.data_ptr(), bias.data_ptr(), xbuf.data_ptr(),
                                                        y.data_ptr(), B, N, T, N_NUM, KP, V, s()),
                                 "tfy_ps_gather_gemm")
                r["k5_fwd_us"] = _time(k5)
            r["kernels"] = _kernels(lambda: (deep_fwd(), deep_bwd(), wide_bag(), wide_push()))
            results[f"L{L}_{'weighted' if weighted else 'unweighted'}"] = r
    out = {"card": _card(), "shapes": {"T": T, "V": V, "B": B, "D": D, "Kp": KP, "N": N}, "cases": results}
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "multihot_step_profile.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
