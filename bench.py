#!/usr/bin/env python
"""Benchmarks of tf_yarn_b200 against BASELINE.json's metric and configs.

Default (`--config mnist`) is the headline: samples/sec for the whole box (device-timed with CUDA events,
max over ranks) of the Keras MNIST-CNN Horovod-path config, bf16 compute, synthetic data of the MNIST
shape, random-init weights; weak scaling (128 samples per GPU per step, the Horovod keras_mnist batch).

    python bench.py --gpus 1 --steps 200 --warmup 20
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29500 bench.py --gpus 8 --steps 200 --warmup 20

Arms (`--impl`):
  ours       (default) mini-Keras + hvd facade; every step = forward/backward out of our wgmma kernels + the
             fused reduce-scatter -> Adadelta -> all-gather exchange, replayed from a CUDA graph.
  reference  the UNMODIFIED reference installed in oracle/_ref: its PyTorch worker
             (tf_yarn.pytorch.tasks.worker._train -> NCCL DistributedDataParallel) on the same model/config,
             see bench/ref_arm.py and bench/shims/README.md.
  standin    what the reference's Horovod path does on an NCCL build, written with stock PyTorch (eager, or
             CUDA-graph captured with --graph).  Not the reference itself: a second yardstick.

Other configs (`--config wide_deep | resnet50 | bert`, BASELINE.json configs 3-5) live in bench/*.py and print
the same JSON schema.

`value` is timed on the device with the input pool (269.7 MB, larger than the 50 MB L2, rotated so no batch
is re-read from L2) resident in HBM, over one region of exactly `--steps` steps (`--repeats N` times N regions
and reports the median region).  `e2e` runs the same number of steps through the public API (`model.fit`) with
per-step H2D copies from pinned host memory and a per-step D2H read of the loss.

`--dump-outputs DIR` (mnist, ours) writes what the last timed step computed -- its loss and the updated flat
parameter vector -- as DIR/loss.npy and DIR/params.npy (float32).  Inputs and initial weights are seeded, so two
builds run with the same arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "standin"])
    ap.add_argument("--config", default="mnist", choices=["mnist", "wide_deep", "resnet50", "bert"])
    ap.add_argument("--repeats", type=int, default=0, help="timed regions of --steps steps each (0 = one)")
    ap.add_argument("--graph", action="store_true", help="standin: capture the step (NCCL included) in a CUDA graph")
    ap.add_argument("--no-exposed", action="store_true", help="ours: skip the LOCAL-mode run behind exposed_comm_ms")
    ap.add_argument("--batch", type=int, default=0, help="per-GPU batch of the secondary configs (0 = default)")
    ap.add_argument("--side-tasks", action="store_true", help="bert: keep the TensorBoard side task alive during the run")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="mnist/ours: write the last timed step's loss and parameters as DIR/*.npy (float32)")
    args = ap.parse_args()
    if args.dump_outputs and (args.config != "mnist" or args.impl != "ours"):
        ap.error("--dump-outputs is implemented for --config mnist --impl ours")
    if args.config == "mnist":
        if args.impl == "reference":
            from bench import ref_arm
            return ref_arm.run_reference(args)
        from bench import mnist
        return mnist.run_standin(args) if args.impl == "standin" else mnist.run_ours(args)
    if args.config == "wide_deep":
        from bench import wide_deep
        return wide_deep.run(args)
    from bench import models
    return models.run(args)


if __name__ == "__main__":
    sys.exit(main())
