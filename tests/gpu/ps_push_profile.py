"""Time the sparse pushes of one wide-and-deep step and split them per kernel (torch.profiler, CUDA activity).

    python tests/gpu/ps_push_profile.py [out_dir]

Shapes of bench/wide_deep.py: 26 hashed columns of 100k buckets, batch 512.  The wide tower pushes [V, 1] FTRL tables
with one fp32 gradient column (col_stride 0); the fused first deep layer pushes [V, 64] Adagrad tables out of column
slices of its bf16 dx (pitch Kp = 26*64 + 13 rounded up to 8).  Buffers are local: the peer latency of a multi-GPU
job is not in these numbers.  Prints the device time of one push (CUDA events over 500 pushes) and, per kernel, the
mean time and the number of launches per push.
"""
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

from tf_yarn_b200.estimator import ps_hbm  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

T, V, B, D = 26, 100_000, 512, 64
KP = (T * D + 13 + 7) // 8 * 8
REPS = 500


def main(out_dir):
    lib = native.load()
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    cases = {}
    for name, (d, opt, slots, gdtype, ld, cs) in {"wide_ftrl": (1, native.OPT_FTRL, 2, torch.float32, 1, 0),
                                                  "deep_adagrad": (D, native.OPT_ADAGRAD, 1, torch.bfloat16, KP, D)}.items():
        tabs = [torch.zeros(V * d, device=dev) for _ in range(T * (1 + slots))]
        ptr = [torch.tensor([t.data_ptr() for t in tabs[k * T:(k + 1) * T]], dtype=torch.int64, device=dev)
               for k in range(1 + slots)]
        ids = torch.randint(0, V, (T, B), device=dev, generator=g)
        dout = (torch.randn(B, ld, device=dev, generator=g) * 0.1).to(gdtype)
        adam = torch.ones(2, device=dev)

        def push(ptr=ptr, ids=ids, dout=dout, d=d, opt=opt, ld=ld, cs=cs, adam=adam):
            sc = ps_hbm.push_rows_scratch(lib, T * B, dev)
            native.check(lib.tfy_ps_multi_push_rows(
                ptr[0].data_ptr(), ptr[1].data_ptr(), ptr[2].data_ptr() if len(ptr) > 2 else None, ids.data_ptr(),
                dout.data_ptr(), int(dout.dtype == torch.bfloat16), B, T, d, V, opt, 0.05, 1e-7, 0.001, 0.01, 0.5,
                1.0, adam.data_ptr(), ld, cs, sc.data_ptr(), sc.numel(), torch.cuda.current_stream().cuda_stream),
                "tfy_ps_multi_push_rows")
        for _ in range(20):
            push()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(REPS):
            push()
        e1.record()
        e1.synchronize()
        per_push_us = e0.elapsed_time(e1) * 1e3 / REPS
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                push()
            torch.cuda.synchronize()
        kern = collections.defaultdict(lambda: [0, 0.0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = ev.name[:90]
                kern[k][0] += 1
                kern[k][1] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        cases[name] = {"push_us": per_push_us,
                       "kernels": {k: {"per_push": c / 50, "mean_us": t / c} for k, (c, t) in kern.items()}}
    card = torch.cuda.get_device_name()
    out = {"device": card, "cases": cases}
    print(json.dumps(out, indent=1))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "ps_push_profile.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
