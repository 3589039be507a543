"""Step time of the MNIST-CNN fast path without weights, with ``class_weight`` and with ``sample_weight``.

One process, one model: after a warm-up, the three modes are timed with CUDA events in alternating regions (a change
of mode recaptures the step graphs, outside the timed window).  Prints the card name and power limit beside the
numbers, and one JSON line.

    python tests/gpu/weighted_step_time.py [--regions 5] [--steps 300]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn, synthetic_mnist  # noqa: E402


def _card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("weighted_step_time.py needs a GPU")
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    model = keras_mnist_cnn()
    model.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True),
                  optimizer=keras.optimizers.Adadelta(1.0), metrics=["accuracy"])
    B, nb = 128, 8
    x, y = synthetic_mnist(B * nb)
    x, y = torch.as_tensor(x).float(), torch.as_tensor(y).long()
    model.fit(x[:B], y[:B], batch_size=B, epochs=1, shuffle=False, verbose=0)     # builds and captures the engine
    eng = model._engine
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    assert isinstance(eng, FastSequentialEngine), type(eng).__name__
    xs = [x[i * B:(i + 1) * B].contiguous().pin_memory() for i in range(nb)]
    ys = [y[i * B:(i + 1) * B].contiguous().pin_memory() for i in range(nb)]
    ws = [torch.rand(B).pin_memory() for _ in range(nb)]
    table = torch.linspace(0.5, 2.0, 10)
    modes = {"none": (None, False), "class_weight": (table, False), "sample_weight": (None, True)}
    times = {k: [] for k in modes}
    launches = {}

    def run(n, use_w):
        ticket = eng.stage_inputs(xs[0], ys[0], ws[0] if use_w else None)
        with torch.cuda.stream(eng.stream):
            for i in range(n):
                eng.launch_step(ticket)
                b = (i + 1) % nb
                ticket = eng.stage_inputs(xs[b], ys[b], ws[b] if use_w else None)
            eng.launch_step(ticket)

    for r in range(args.regions):
        for name, (tab, use_w) in modes.items():
            eng.set_class_weight(tab)
            run(args.warmup, use_w)                 # recapture (mode change) + warm-up
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(eng.stream)
            run(args.steps - 1, use_w)
            t1.record(eng.stream)
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) / args.steps)
            launches[name] = eng._launches_per_step
        eng.pop_metrics()
    card = _card()
    print(f"card: {card}")
    for name, ts in times.items():
        ts = sorted(ts)
        print(f"{name:>14}: median {ts[len(ts) // 2] * 1e3:.1f} us/step  (min {ts[0] * 1e3:.1f}, max {ts[-1] * 1e3:.1f}; "
              f"{launches[name]} launches per step)")
    print(json.dumps({"card": card, "ms_per_step": times, "launches_per_step": launches}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
