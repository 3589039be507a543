"""Per-CTA event timeline (``tfy_gemm_set_timeline``) of the split-K Dense GEMM at the MNIST step's shape.

    python tests/gpu/gemm_timeline.py OUT_DIR [--label L]

tfy_gemm_bf16 runs on its own at M = N = 128, K = 9216 into fp32 slabs, at the engine's split (24 K-slices of 6
k-tiles) and at TFY_SPLITK_TILES=4's (36 K-slices of 4).  Reported, in ``OUT_DIR/gemm_timeline[_L].json`` and on
stdout, for each split:

* the grid (CTAs) the launch ran;
* the kernel time, CUDA events around 2000 back-to-back launches (profiler off);
* per CTA, in SM cycles from the CTA's start (median and max over CTAs; microseconds at the SM clock read in the same
  run): ``pdl_wait`` until griddepcontrol.wait returned, ``first_stage`` until the first full TMA stage landed,
  ``main_loop`` from there to the last wgmma retired, ``store`` from there to the partial tile stored;
* the spread of the CTAs' start times (global timer) and the latest CTA end, from the first CTA's start;
* the card name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from step_breakdown import card_info  # noqa: E402

M, N, K = 128, 128, 9216
PHASES = [("pdl_wait", 0, 1), ("first_stage", 1, 2), ("main_loop", 2, 3), ("store", 3, 4)]


def timeline(lib, split, sm_mhz):
    import torch
    from tf_yarn_b200.ops import native
    native.declare("tfy_gemm_set_timeline", [ctypes.c_void_p])
    g = torch.Generator().manual_seed(11)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
    w = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16).cuda()
    slabs = int(lib.tfy_gemm_bf16_splitk_slabs(K, split))
    acc = torch.empty(slabs, M, N, dtype=torch.float32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def launch():
        return lib.tfy_gemm_bf16(x.data_ptr(), w.data_ptr(), None, acc.data_ptr(), None, M, N, K, K, K, N, 0, split, s)

    for _ in range(50):
        assert launch() == 0
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 2000
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    e1.synchronize()
    kernel_us = e0.elapsed_time(e1) * 1e3 / iters

    cap = 1024
    tl = torch.zeros(cap * 16, dtype=torch.int64, device="cuda")
    lib.tfy_gemm_set_timeline(tl.data_ptr())
    assert launch() == 0
    torch.cuda.synchronize()
    lib.tfy_gemm_set_timeline(None)
    v = tl.view(cap, 16).cpu()
    v = v[v[:, 0] != 0]
    res = {"split": slabs, "ctas": int(v.shape[0]), "kernel_us": kernel_us}
    for ph, lo, hi in PHASES:
        d = (v[:, hi] - (v[:, lo] if lo else 0)).double()
        res[ph + "_cycles"] = {"median": float(d.median()), "max": float(d.max())}
        if sm_mhz:
            res[ph + "_us_median"] = float(d.median()) / sm_mhz
    start_ns = v[:, 0].double()
    res["start_spread_ns"] = float(start_ns.max() - start_ns.min())
    res["end_cycles_max"] = float(v[:, 4].double().max())
    if sm_mhz:
        res["end_us_max"] = res["end_cycles_max"] / sm_mhz
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "gemm_timeline.py needs a GPU"
    from tf_yarn_b200.ops import gemm  # noqa: F401  (declares the GEMM entry points)
    from tf_yarn_b200.ops import native
    lib = native.load()
    os.makedirs(args.out_dir, exist_ok=True)
    card = card_info()
    try:
        sm_mhz = float(card.get("clocks.sm", "").split()[0])
    except (ValueError, IndexError):
        sm_mhz = None
    rep = {"gpu": torch.cuda.get_device_name(0), "card": card, "label": args.label,
           "splits": [timeline(lib, split, sm_mhz) for split in (24, 36)], "card_after": card_info()}
    path = os.path.join(args.out_dir, f"gemm_timeline{('_' + args.label) if args.label else ''}.json")
    with open(path, "w") as f:
        json.dump(rep, f, indent=1)
    print(f"{rep['gpu']}  power limit {card.get('power.limit')}  SM clock {card.get('clocks.sm')}")
    for r in rep["splits"]:
        print(json.dumps(r))
    print("wrote", path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
