"""Per-kernel breakdown of the headline MNIST-CNN training step (batch 128, Adadelta, one GPU, CUDA graph).

    python tests/gpu/step_breakdown.py OUT_DIR [--steps 300] [--regions 5]

The engine is built as ``bench/mnist.py::run_ours`` builds it; inputs rotate through a pool resident in HBM.
Reported, in ``OUT_DIR/step_breakdown.json`` and on stdout:

* the graph's step time (CUDA events around ``--steps`` replays, ``--regions`` regions, profiler off);
* for each of the step's launches, from ``torch.profiler`` (CUDA activities, a separate run): the kernel's span
  (start to end, median and spread over the steps) and its critical-path time, end minus the later of its own
  start and the previous kernel's end.  Kernels are launched with programmatic dependent launch, so a span
  includes the time a kernel waits for its predecessor; the critical-path times add up to the step;
* the MACs and the minimum HBM bytes of each kernel, computed from the shapes below, and the share of the
  applicable H100 SXM data-sheet bound (989 TFLOP/s dense bf16 or 3.35 TB/s) that the critical-path time reaches;
* the per-CTA event timeline (``tfy_conv_set_timeline``) of the conv2 forward and weight-gradient kernels,
  launched on their own at the step's shapes, split into prologue / main loop / epilogue (/ grid barrier);
* the card name, power limit and SM clock, read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

B = 128
PEAK_FLOPS = 989e12          # H100 SXM, dense bf16, data sheet
PEAK_BYTES = 3.35e12         # H100 SXM HBM3, data sheet
N_PARAMS = 1_199_882

# (substring of the kernel name, label, MACs, minimum HBM bytes) at batch B; conv1 26x26x32, conv2 24x24x64,
# pool 12x12x64, Dense 9216 -> 128 -> 10.  Bytes count each tensor the kernel must read or write once.
_A1 = B * 26 * 26 * 32 * 2                   # conv1 output = conv2 input, bf16
_P2 = B * 12 * 12 * 64                       # pooled elements
_X3 = B * 9216 * 2                           # flattened pooled activations, bf16
_W3 = 128 * 9216 * 2                         # Dense1 weight, bf16
KERNELS = [
    ("tfy_conv3x3_c1_fwd_tc_kernel", "conv1 fwd", B * 26 * 26 * 32 * 9, B * 28 * 28 * 4 + _A1),
    ("tfy_conv3x3_fprop_pool_kernel", "conv2 fprop+pool", B * 24 * 24 * 64 * 32 * 9, _A1 + _P2 * 3),
    ("tfy_gemm_bf16_kernel", "Dense1 fwd (split-K)", B * 128 * 9216, _X3 + _W3 + B * 128 * 4),
    ("tfy_bias_act_drop_fwd_kernel", "Dense1 bias/ReLU/dropout", 0, B * 128 * (4 + 2 + 1)),
    ("tfy_dense_head_fused_kernel", "Dense2 head fwd+bwd", 3 * B * 128 * 10, B * 128 * 3 + 128 * 10 * 4),
    ("tfy_dense_bwd", "Dense1 bwd (dW + dx)", 2 * B * 128 * 9216, B * 128 * 2 + _X3 + 2 * _W3 + _X3),
    ("tfy_conv3x3_wgrad_kernel", "conv2 wgrad (+unpool, db)", B * 24 * 24 * 64 * 32 * 9, _A1 + _P2 * 3),
    ("tfy_conv3x3_dgrad_kernel", "conv2 dgrad (+unpool, gate)", B * 26 * 26 * 32 * 64 * 9, _P2 * 3 + 2 * _A1),
    ("tfy_conv3x3_c1_wgrad_tc_kernel", "conv1 wgrad + db", B * 26 * 26 * 32 * 9, B * 28 * 28 * 4 + _A1),
    # Adadelta: bf16 grad + param read, param written; fp32 master + two accumulators read and written
    ("tfy_fused_step_kernel", "optimizer step", 0, N_PARAMS * (2 + 2 + 2 + 3 * 4 * 2)),
]


def classify(name: str):
    for key, label, macs, nbytes in KERNELS:
        if key in name:
            return key, label, macs, nbytes
    return name, name, 0, 0


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        fields = [f.strip() for f in out[0].split(",")]
        return dict(zip(q.split(","), fields))
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def spread(v):
    s = sorted(v)
    return {"median": statistics.median(s), "p10": s[len(s) // 10], "p90": s[(len(s) * 9) // 10],
            "min": s[0], "max": s[-1], "n": len(s)}


def build_engine():
    import torch
    from bench import mnist
    from tf_yarn_b200 import hvd
    torch.cuda.set_device(0)
    hvd.init()
    model = mnist._build_model(True, 1)
    x_host, y_host = mnist.make_pool(seed=100)
    model.fit(x_host[:3 * B], y_host[:3 * B], batch_size=B, epochs=1, shuffle=False, verbose=0)
    eng = model._engine
    assert eng.graph is not None, "the step was not captured in a CUDA graph"
    x_dev, y_dev = x_host.cuda(), y_host.cuda()
    pool = [(x_dev[b * B:(b + 1) * B], y_dev[b * B:(b + 1) * B]) for b in range(mnist.POOL_BATCHES)]
    state = {"b": 0}

    def run(n):
        for _ in range(n):
            b = state["b"]
            eng.launch_step(eng.stage_inputs(*pool[b]))
            state["b"] = (b + 1) % len(pool)
    return eng, run


def step_time(eng, run, steps, regions):
    import torch
    out = []
    with torch.cuda.stream(eng.stream):
        run(steps)
        for _ in range(regions):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(eng.stream)
            run(steps)
            e1.record(eng.stream)
            e1.synchronize()
            out.append(e0.elapsed_time(e1) * 1e3 / steps)
    return out


def profile_kernels(eng, run, steps, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with torch.cuda.stream(eng.stream):
        run(10)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            run(steps)
            torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, "step_breakdown.pt.trace.json"))
    kern = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.name.startswith(("void tfy_", "tfy_")):
            kern.append((e.time_range.start, e.time_range.end, e.name))
    kern.sort()
    return kern


def summarise(kern, steps):
    """Split the sorted kernel list into steps (each starts with conv1's forward) and attribute times."""
    first = KERNELS[0][0]
    per_step, cur = [], None
    for k in kern:
        if first in k[2]:
            cur = []
            per_step.append(cur)
        if cur is not None:
            cur.append(k)
    full = [s for s in per_step if len(s) == len(per_step[0])]
    rows = {}
    gaps, sums, walls = [], [], []
    for s in full:
        prev_end = None
        tot = 0.0
        for (t0, t1, name) in s:
            key, label, macs, nbytes = classify(name)
            r = rows.setdefault(key, {"label": label, "kernel": name.split("(")[0], "macs": macs,
                                      "min_hbm_bytes": nbytes, "span": [], "critical": []})
            r["span"].append(t1 - t0)
            crit = t1 - max(t0, prev_end) if prev_end is not None else t1 - t0
            r["critical"].append(max(crit, 0.0))
            tot += t1 - t0
            prev_end = t1 if prev_end is None else max(prev_end, t1)
        sums.append(tot)
        walls.append(s[-1][1] - s[0][0])
    for i in range(1, len(full)):
        gaps.append(full[i][0][0] - full[i - 1][-1][1])
    table = []
    for key, r in rows.items():
        crit = statistics.median(r["critical"])
        t_flop = 2.0 * r["macs"] / PEAK_FLOPS * 1e6
        t_byte = r["min_hbm_bytes"] / PEAK_BYTES * 1e6
        bound = "compute" if t_flop >= t_byte else "hbm"
        t_min = max(t_flop, t_byte)
        table.append({"label": r["label"], "kernel": r["kernel"], "macs": r["macs"],
                      "min_hbm_bytes": r["min_hbm_bytes"], "span_us": spread(r["span"]),
                      "critical_us": spread(r["critical"]), "floor_us": t_min, "bound": bound,
                      "share_of_bound": (t_min / crit) if crit > 0 else None})
    return {"steps_profiled": len(full), "launches_per_step": len(full[0]) if full else 0, "kernels": table,
            "sum_of_spans_us": spread(sums), "first_start_to_last_end_us": spread(walls),
            "gap_between_steps_us": spread(gaps) if gaps else None}


def conv_timelines(sm_mhz):
    """Per-CTA marks (SM cycles from the CTA's start) of the two conv2 kernels at the step's shapes."""
    import torch
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    lib = native.load()
    native.declare("tfy_conv_set_timeline", [ctypes.c_void_p])
    dev, bf16 = torch.device("cuda:0"), torch.bfloat16
    s = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=dev).manual_seed(7)
    a = torch.randn(B, 26, 26, 32, device=dev, generator=g).relu().to(bf16)
    w = (torch.randn(64, 3, 3, 32, device=dev, generator=g) * 0.06).to(bf16)
    bias = (torch.randn(64, device=dev, generator=g) * 0.1).to(bf16)
    pooled = torch.zeros(B, 12, 12, 64, dtype=bf16, device=dev)
    code = torch.zeros(B, 12, 12, 64, dtype=torch.uint8, device=dev)
    dp = (torch.randn(B, 12, 12, 64, device=dev, generator=g) * 0.5).to(bf16)
    part = torch.zeros(int(lib.tfy_conv3x3_c32_wgrad_scratch_elems()), dtype=torch.float32, device=dev)
    sync = torch.zeros(1024, dtype=torch.int32, device=dev)
    dw = torch.zeros(64, 3, 3, 32, dtype=bf16, device=dev)
    db = torch.zeros(64, dtype=bf16, device=dev)
    hp = torch.zeros(16, dtype=torch.float32, device=dev)
    launches = {
        "fprop": (lambda: lib.tfy_conv3x3_c32_pool_fwd(a.data_ptr(), w.data_ptr(), bias.data_ptr(),
                                                       pooled.data_ptr(), code.data_ptr(), B, 26, 26, 0.5, 1234,
                                                       hp.data_ptr(), s),
                  # (name, from slot, to slot); slot 0 is the CTA start
                  [("prologue", 0, 4), ("main_loop", 4, 11), ("epilogue_tail", 11, 9), ("exit", 9, 10)]),
        "wgrad": (lambda: lib.tfy_conv3x3_c32_wgrad_unpool(a.data_ptr(), dp.data_ptr(), code.data_ptr(),
                                                           ctypes.c_float(2.0), part.data_ptr(), dw.data_ptr(),
                                                           db.data_ptr(), sync.data_ptr(), B, 26, 26, s),
                  # slots 4 and 5 come from the MMA warpgroup's clock, 7, 8 and 10 from thread 0's: only
                  # differences within one thread are phases (all_roles_done is measured from the CTA start)
                  [("prologue", 0, 4), ("main_loop", 4, 5), ("all_roles_done", 0, 7), ("grid_barrier", 7, 8),
                   ("reduction", 8, 10)]),
    }
    tl = torch.zeros(160 * 16, dtype=torch.int64, device=dev)
    out = {}
    for name, (fn, phases) in launches.items():
        for _ in range(5):
            assert fn() == 0
        torch.cuda.synchronize()
        tl.zero_()
        lib.tfy_conv_set_timeline(tl.data_ptr())
        fn()
        torch.cuda.synchronize()
        lib.tfy_conv_set_timeline(None)
        v = tl.view(160, 16).cpu()
        v = v[v[:, 0] != 0]
        res = {"ctas": int(v.shape[0])}
        for ph, lo, hi in phases:
            d = (v[:, hi] - (v[:, lo] if lo else 0)).double()
            res[ph + "_cycles"] = {"median": float(d.median()), "max": float(d.max())}
            if sm_mhz:
                res[ph + "_us_median"] = float(d.median()) / sm_mhz
        res["end_cycles_max"] = float(v[:, 10].double().max())
        out[name] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "step_breakdown.py needs a GPU"
    os.makedirs(args.out_dir, exist_ok=True)
    eng, run = build_engine()
    regions = step_time(eng, run, args.steps, args.regions)
    card = card_info()
    kern = profile_kernels(eng, run, args.steps, args.out_dir)
    rep = summarise(kern, args.steps)
    try:
        sm_mhz = float(card.get("clocks.sm", "").split()[0])
    except (ValueError, IndexError):
        sm_mhz = None
    rep["conv2_timeline"] = conv_timelines(sm_mhz)
    rep["card"] = card
    rep["card_after"] = card_info()
    rep["label"] = args.label
    rep["step_us"] = spread(regions)
    rep["gpu"] = torch.cuda.get_device_name(0)
    path = os.path.join(args.out_dir, f"step_breakdown{('_' + args.label) if args.label else ''}.json")
    with open(path, "w") as f:
        json.dump(rep, f, indent=1)
    print(f"{rep['gpu']}  power limit {card.get('power.limit')}  SM clock {card.get('clocks.sm')} "
          f"(max {card.get('clocks.max.sm')})")
    print(f"step (graph, profiler off): {rep['step_us']['median']:.1f} us "
          f"[{rep['step_us']['min']:.1f} .. {rep['step_us']['max']:.1f}] over {args.regions} regions")
    print(f"{'kernel':34s} {'span med':>9s} {'crit med':>9s} {'p10':>7s} {'p90':>7s} {'floor':>7s} bound share")
    for r in rep["kernels"]:
        c = r["critical_us"]
        share = f"{100 * r['share_of_bound']:.1f}%" if r["share_of_bound"] else "-"
        print(f"{r['label']:34s} {r['span_us']['median']:9.2f} {c['median']:9.2f} {c['p10']:7.2f} {c['p90']:7.2f} "
              f"{r['floor_us']:7.2f} {r['bound']:7s} {share}")
    print(f"sum of spans {rep['sum_of_spans_us']['median']:.1f} us, first start to last end "
          f"{rep['first_start_to_last_end_us']['median']:.1f} us, gap between steps "
          f"{rep['gap_between_steps_us']['median'] if rep['gap_between_steps_us'] else float('nan'):.1f} us")
    print("conv2 timeline:", json.dumps(rep["conv2_timeline"]))
    print("wrote", path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
