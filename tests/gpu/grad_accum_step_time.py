"""Time per batch of the MNIST-CNN fast path without and with gradient accumulation (N = 4), and the accumulate
kernel against its HBM floor.

    python tests/gpu/grad_accum_step_time.py [--regions 5] [--steps 300] [--out DIR]

Batch time: 5 alternating regions of 300 batches per configuration (batch 128, Adam), CUDA events around each
region after a warm-up.  Kernel time: CUDA events around 200 launches of tfy_grad_accumulate (bf16 source) with and
without clearing the source, on the MNIST flat gradient buffer (1.2 M elements: its 7 MB stay in L2 between
launches) and on a 64 M-element buffer (384 MB, streamed from HBM); the HBM floor is n * (2 + 4 + 4) bytes per
launch (read the gradient, read and write the accumulator), plus 2 bytes per element when it clears the source, at
the H100 SXM data-sheet bandwidth of 3.35 TB/s.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return "unknown"


def engine(n_steps):
    import numpy as np
    from tf_yarn_b200 import keras
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
    torch.manual_seed(0)
    m = keras_mnist_cnn()
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True),
              optimizer=keras.optimizers.Adam(1e-3, gradient_accumulation_steps=n_steps))
    m.build((28, 28, 1))
    rs = np.random.RandomState(0)
    x = torch.from_numpy(rs.rand(128, 28, 28, 1).astype("float32")).cuda()
    y = torch.from_numpy(rs.randint(0, 10, 128).astype("int64")).cuda()
    m._ensure_engine(x, y)
    eng = m._engine
    eng.ensure_captured(x, y)
    return eng, eng.stage_inputs(x, y)


def region(eng, ticket, steps):
    st = eng.stream
    with torch.cuda.stream(st):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        k0 = eng.kernel_launches
        a.record(st)
        for _ in range(steps):
            eng.launch_step(ticket)
        b.record(st)
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / steps, (eng.kernel_launches - k0) / steps


def kernel_time(n, clear, reps=200):
    """Time per launch of tfy_grad_accumulate on an n-element bf16 buffer.  At the MNIST size (1.2 M elements, a 7 MB
    working set) the buffers stay in the 50 MB L2 across launches, so the HBM floor only bounds it loosely; at 64 M
    elements (384 MB) every launch streams from HBM."""
    from tf_yarn_b200.ops import native
    from tf_yarn_b200.parallel import comm  # noqa: F401  (declares tfy_grad_accumulate's argument types)
    lib = native.load()
    acc = torch.zeros(n, device="cuda")
    src = torch.randn(n, device="cuda").to(torch.bfloat16)
    s = torch.cuda.current_stream().cuda_stream

    def launch():
        native.check(lib.tfy_grad_accumulate(acc.data_ptr(), src.data_ptr(), native.BF16, n, int(clear), None, 0, 0,
                                             s), "tfy_grad_accumulate")
    for _ in range(20):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    b.synchronize()
    us = a.elapsed_time(b) * 1e3 / reps
    floor_bytes = n * (2 + 4 + 4 + (2 if clear else 0))
    floor_us = floor_bytes / 3.35e12 * 1e6
    return {"n": n, "working_set_MB": round(n * (2 + 4) / 1e6, 1), "clear": clear, "us": round(us, 2),
            "hbm_floor_us": round(floor_us, 2), "floor_over_time": round(floor_us / us, 3),
            "GB_per_s": round(floor_bytes / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    engines = {"N=None": engine(None), "N=4": engine(4)}
    for eng, ticket in engines.values():
        region(eng, ticket, 40)                  # warm-up
    times = {k: [] for k in engines}
    launches = {}
    for _ in range(args.regions):
        for k, (eng, ticket) in engines.items():
            us, per = region(eng, ticket, args.steps)
            times[k].append(round(us, 2))
            launches[k] = per
    out = {"card": card(), "batch": 128, "optimizer": "adam", "regions_us_per_batch": times,
           "median_us_per_batch": {k: statistics.median(v) for k, v in times.items()},
           "launches_per_batch": launches,
           "accumulate_kernel": [kernel_time(n, clear) for n in (1199888, 64 << 20) for clear in (False, True)]}
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "grad_accum_step_time.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
