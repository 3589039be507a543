"""Step time of the MNIST CNN with a binary head (Dense(1, sigmoid), BinaryCrossentropy(label_smoothing=0.05)) on the
fast path and on the autograd engine (use_fast_path=False), and of the headline sparse-categorical step.

One process, one model per variant (each with its own captured step graphs): after a warm-up, the three are timed with
CUDA events in alternating regions (default 5 regions of 300 steps each); the median per-step device time is
reported.  Prints the card name and power limit beside the numbers, and one JSON line.

    python tests/gpu/binary_head_step_time.py [--regions 5] [--steps 300]
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
        raise SystemExit("binary_head_step_time.py needs a GPU")
    torch.cuda.set_device(0)
    from tf_yarn_b200.keras import layers
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    B, nb = 128, 8
    x, y = synthetic_mnist(B * nb)
    x, y = torch.as_tensor(x).float(), torch.as_tensor(y).long()
    binary = (y >= 5).float().reshape(-1, 1)
    xs = [x[i * B:(i + 1) * B].contiguous().pin_memory() for i in range(nb)]
    sparse_labels = [y[i * B:(i + 1) * B].contiguous().pin_memory() for i in range(nb)]
    binary_labels = [binary[i * B:(i + 1) * B].contiguous().pin_memory() for i in range(nb)]

    def binary_cnn():
        return keras.Sequential(keras_mnist_cnn().layers[:-1] + [layers.Dense(1, activation="sigmoid")])
    bce = keras.losses.BinaryCrossentropy(label_smoothing=0.05)
    # name: (model, loss, labels, fast path)
    variants = {"binary_fast": (binary_cnn, bce, binary_labels, True),
                "binary_autograd": (binary_cnn, bce, binary_labels, False),
                "sparse_fast": (keras_mnist_cnn, keras.losses.SparseCategoricalCrossentropy(from_logits=True),
                                sparse_labels, True)}
    labels = {name: v[2] for name, v in variants.items()}
    engines = {}
    for name, (build, loss, ys, fast) in variants.items():
        torch.manual_seed(0)
        model = build()
        model.compile(loss=loss, optimizer=keras.optimizers.Adadelta(1.0), metrics=["accuracy"], use_fast_path=fast)
        model.fit(x[:B], ys[0], batch_size=B, epochs=1, shuffle=False, verbose=0)   # builds and captures
        assert isinstance(model._engine, FastSequentialEngine) == fast, type(model._engine).__name__
        engines[name] = (model, model._engine)
    times = {k: [] for k in variants}
    launches = {}

    def run(eng, ys, n):
        ticket = eng.stage_inputs(xs[0], ys[0])
        with torch.cuda.stream(eng.stream):
            for i in range(n):
                eng.launch_step(ticket)
                b = (i + 1) % nb
                ticket = eng.stage_inputs(xs[b], ys[b])
            eng.launch_step(ticket)

    for _ in range(args.regions):
        for name, (_, eng) in engines.items():
            run(eng, labels[name], args.warmup)
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(eng.stream)
            run(eng, labels[name], args.steps - 1)
            t1.record(eng.stream)
            t1.synchronize()
            times[name].append(t0.elapsed_time(t1) / args.steps)
            launches[name] = eng._launches_per_step
            eng.pop_metrics()
    card = _card()
    print(f"card: {card}")
    for name, ts in times.items():
        ts = sorted(ts)
        print(f"{name:>18}: median {ts[len(ts) // 2] * 1e3:.1f} us/step  (min {ts[0] * 1e3:.1f}, "
              f"max {ts[-1] * 1e3:.1f}; {launches[name]} launches per step)")
    print(json.dumps({"card": card, "ms_per_step": times, "launches_per_step": launches}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
