"""Time the confusion-histogram update kernel (ops/csrc/tfy_confusion.cu) and the cost of AUC in a Keras fit step.

    python tests/gpu/confusion_metric_time.py OUT_DIR

* the update at N in {128, 4096, 65536, 2^20, 2^24} elements, fp32 / bf16 predictions, with and without per-sample
  weights (fp32 labels, T = 200), timed with CUDA events over many launches after warm-up; the bytes it must move, the
  share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) that is, and a stock-torch ``bucketize`` + ``bincount``
  histogram (nondeterministic: float atomics) for comparison;
* the time per step of a Keras binary MLP ``fit`` on the CUDA-graph engine with and without ``metrics=["AUC"]``.

The card's name, power limit and SM clock are read in the same run.  Writes ``confusion_metric_time.json`` and
``confusion_metric_time.md`` under OUT_DIR.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.ops import confusion  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
T = 200


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def time_fn(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters          # microseconds


def kernel_rows():
    rows = []
    edges = torch.linspace(0, 1, T, device="cuda")
    for n in (128, 4096, 65536, 1 << 20, 1 << 24):
        for pdt in (torch.float32, torch.bfloat16):
            for weighted in (False, True):
                g = torch.Generator(device="cuda").manual_seed(n)
                p = torch.rand(n, device="cuda", generator=g).to(pdt)
                y = (torch.rand(n, device="cuda", generator=g) < 0.3).float()
                w = torch.rand(n, device="cuda", generator=g) if weighted else None
                st = confusion.ConfusionState(T)
                iters = max(20, min(2000, (1 << 26) // max(n, 1)))
                t_us = time_fn(lambda: st.update(y, p, w), iters)
                nbytes = n * (p.element_size() + 4 + (4 if weighted else 0))

                def torch_hist():
                    b = torch.bucketize(p.float(), edges)
                    ww = w if w is not None else torch.ones_like(y)
                    torch.bincount(b, weights=y * ww, minlength=T + 1)
                    torch.bincount(b, weights=(1 - y) * ww, minlength=T + 1)
                t_torch = time_fn(torch_hist, iters)
                floor_us = nbytes / HBM_BYTES_PER_S * 1e6
                rows.append({"n": n, "pred": str(pdt).replace("torch.", ""), "weighted": weighted,
                             "update_us": round(t_us, 2), "bytes": nbytes, "hbm_floor_us": round(floor_us, 2),
                             "share_of_hbm_floor": round(floor_us / t_us, 3), "torch_bucketize_bincount_us":
                             round(t_torch, 2)})
                print(rows[-1], flush=True)
    return rows


def fit_rows():
    rows = []
    n, bs, steps = 4096 * 64, 4096, 64
    g = np.random.default_rng(0)
    x = g.standard_normal((n, 64)).astype(np.float32)
    y = (x[:, 0] > 0).astype(np.float32)
    for metrics in ([], ["AUC"]):
        torch.manual_seed(0)
        m = keras.Sequential([keras.layers.Dense(256, activation="relu", input_shape=(64,)),
                              keras.layers.Dense(256, activation="relu"), keras.layers.Dense(1, activation="sigmoid")])
        m.compile(keras.optimizers.SGD(0.01), "binary_crossentropy", metrics=metrics)
        m.fit(x, y, batch_size=bs, epochs=1, shuffle=False, verbose=0)          # capture + warm-up
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.fit(x, y, batch_size=bs, epochs=1, shuffle=False, verbose=0)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) / steps * 1e6)
        rows.append({"metrics": metrics, "engine": type(m._engine).__name__, "step_us_median": round(
            float(np.median(times)), 1), "step_us_all": [round(t, 1) for t in times]})
        print(rows[-1], flush=True)
    return rows


def main(out_dir):
    assert torch.cuda.is_available(), "needs a GPU"
    os.makedirs(out_dir, exist_ok=True)
    info = card()
    res = {"card": info, "kernel": kernel_rows(), "fit": fit_rows(), "card_after": card()}
    with open(os.path.join(out_dir, "confusion_metric_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    lines = [f"Card: {info}", "", "| N | pred | weighted | update us | bytes | HBM floor us | share of floor | torch "
             "bucketize+bincount us |", "|---|---|---|---|---|---|---|---|"]
    for r in res["kernel"]:
        lines.append(f"| {r['n']} | {r['pred']} | {r['weighted']} | {r['update_us']} | {r['bytes']} | "
                     f"{r['hbm_floor_us']} | {r['share_of_hbm_floor']} | {r['torch_bucketize_bincount_us']} |")
    lines += ["", "| fit metrics | engine | us per step (median of 3 epochs) |", "|---|---|---|"]
    for r in res["fit"]:
        lines.append(f"| {r['metrics']} | {r['engine']} | {r['step_us_median']} |")
    with open(os.path.join(out_dir, "confusion_metric_time.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: confusion_metric_time.py OUT_DIR")
    main(sys.argv[1])
