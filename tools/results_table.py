#!/usr/bin/env python
"""Collect bench JSON lines (one file per run, as printed by bench.py) into markdown tables (README "Results").

    python tools/results_table.py DIR        # prints the tables of DIR/bench_*.json
Files are named bench_<config>_<impl>_N<n>_<tag>.json (one JSON object each, as printed by bench.py).
"""
import glob
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(results_dir):
    rows = {}
    for f in sorted(glob.glob(os.path.join(results_dir, "bench_*.json"))):
        m = re.match(r"bench_(.+?)_N(\d+)_(\w+)\.json", os.path.basename(f))
        if not m:
            continue
        try:
            d = json.load(open(f))
        except Exception:  # noqa: BLE001
            continue
        if "value" not in d:
            continue
        rows[(m.group(1), int(m.group(2)))] = (d, os.path.basename(f))
    return rows


def fmt(v, nd=0):
    return f"{v:,.{nd}f}" if v is not None else "–"


def table(rows, config, arms, unit):
    ns = sorted({n for (k, n) in rows if k.startswith(config + "_") or k == config})
    out = [f"| GPUs | " + " | ".join(f"{a} {unit} (device) | {a} µs/step | {a} e2e {unit}" for a in arms) + " | ours / "
           + arms[-1] + " (device, e2e) |", "|---:|" + "---:|" * (3 * len(arms) + 1)]
    for n in ns:
        cells, vals = [], {}
        for a in arms:
            d = rows.get((f"{config}_{a}", n))
            if d:
                d = d[0]
                vals[a] = (d["value"], d.get("e2e", {}).get("value"))
                cells += [fmt(d["value"]), fmt(d["ms_per_step"] * 1e3, 1), fmt(d.get("e2e", {}).get("value"))]
            else:
                cells += ["–", "–", "–"]
        ratio = "–"
        if arms[0] in vals and arms[-1] in vals and vals[arms[-1]][0]:
            r1 = vals[arms[0]][0] / vals[arms[-1]][0]
            r2 = (vals[arms[0]][1] / vals[arms[-1]][1]) if vals[arms[-1]][1] else None
            ratio = f"{r1:.1f}x, {r2:.1f}x" if r2 else f"{r1:.1f}x"
        out.append(f"| {n} | " + " | ".join(cells) + f" | {ratio} |")
    return "\n".join(out)


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: results_table.py DIR")
    rows = load(sys.argv[1])
    print("### Headline: Keras MNIST-CNN, Horovod path (samples/s)\n")
    print(table(rows, "mnist", ["ours", "standin_graph", "reference"], "samples/s"))
    base = rows.get(("mnist_ours", 1))
    if base:
        print("\nScaling efficiency (value(N) / (N * value(1))), exposed communication and parameter agreement:\n")
        print("| GPUs | efficiency (device) | efficiency (e2e) | exposed comm µs/step | params_in_sync | loss fell |")
        print("|---:|---:|---:|---:|---|---|")
        for (k, n), (d, _) in sorted(rows.items(), key=lambda kv: kv[0][1]):
            if k != "mnist_ours":
                continue
            e = d.get("e2e", {})
            print(f"| {n} | {d['value'] / (n * base[0]['value']):.3f} | "
                  f"{e.get('value', 0) / (n * base[0]['e2e']['value']):.3f} | {d.get('exposed_comm_ms', 0) * 1e3:.1f} | "
                  f"{d.get('params_in_sync')} | {e.get('loss_fell')} |")
    for cfg, arms, unit in (("resnet50", ["ours", "reference"], "img/s"), ("bert", ["ours", "standin"], "seq/s"),
                            ("wide_deep", ["ours", "standin"], "samples/s")):
        if any(k.startswith(cfg + "_") for (k, _) in rows):
            print(f"\n### {cfg}\n")
            print(table(rows, cfg, arms, unit))


if __name__ == "__main__":
    sys.exit(main())
