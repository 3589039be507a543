"""Size sweep of the all-reduce kernels (K1/K2/K3) and the fused step (K4, Adam) against NCCL on N H100s.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29521 tests/gpu/comm_sweep.py [--max-mb 512] [--out gpurun_out/comm_sweep_N<N>.json]

For every size: CUDA-event time of back-to-back launches after warm-up, MAX over ranks; bus bandwidth
2(N-1)/N * S / t and the fraction of the NVLS floor t_floor = S (1 + 1/N) / 770 GB/s (the measured
per-direction NVLink peer bandwidth).  Also the cost of the bare
cross-GPU barrier kernel for several grid sizes (the latency floor of every kernel here).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from tf_yarn_b200.ops import native  # noqa: E402
from tf_yarn_b200.parallel import comm as commod  # noqa: E402
from tf_yarn_b200.parallel.symm import StoreRendezvous, SymmArena  # noqa: E402

LINK_GBS = 770.0


def ev_time(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item()) * 1e3        # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-mb", type=int, default=512)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    store = dist.distributed_c10d._get_default_store()
    arena = SymmArena((args.max_mb << 20) + (700 << 20), device=local, rdv=StoreRendezvous(store, rank, world, "sweep"))
    comm = commod.Communicator(fusion_bytes=16 << 20, arena=arena)
    res = {"world": world, "multicast": bool(comm.multicast), "link_GBs": LINK_GBS, "barrier_us": {},
           "allreduce": [], "fused_adam": []}

    for grid in (1, 16, 64, 148, 296):
        us = ev_time(lambda: native.check(comm.lib.tfy_barrier(arena.ctx_ref, grid, torch.cuda.current_stream().cuda_stream),
                                          "barrier"), 200)
        res["barrier_us"][str(grid)] = us
    if rank == 0:
        print("[barrier]", json.dumps(res["barrier_us"]), flush=True)

    # launch-overhead-free numbers: 20 launches captured in a CUDA graph (what a captured train step sees)
    def graph_time(fn, reps=20):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                fn()
        return ev_time(g.replay, 10, warmup=2) / reps

    res["graph_us"] = {}
    for grid in (1, 16, 148):
        res["graph_us"][f"barrier_grid{grid}"] = graph_time(
            lambda: native.check(comm.lib.tfy_barrier(arena.ctx_ref, grid, torch.cuda.current_stream().cuda_stream), "b"))
    mark0 = arena._bump
    for label, n_params in (("fused_adadelta_320", 320), ("fused_adadelta_19k", 19_392), ("fused_adadelta_160k", 160_000),
                            ("fused_adadelta_1.2M", 1_199_882)):
        arena._bump = mark0
        fo = commod.FusedShardedOptimizer(comm, [(n_params,)], commod.OptimizerSpec.adadelta(1.0), torch.bfloat16,
                                          zero_grads=False)
        fo.init_from([torch.full((n_params,), 0.1, device="cuda")])
        fo.flat_grads.normal_()
        res["graph_us"][label] = graph_time(fo.step)
        _, buf = arena.empty((comm.pad_elems(n_params, torch.bfloat16),), torch.bfloat16)
        buf.normal_()
        if comm.multicast:
            res["graph_us"][label.replace("fused_adadelta", "nvls_allreduce")] = graph_time(
                lambda: comm.all_reduce_symm(buf, False, native.ALGO_NVLS))
        res["graph_us"][label.replace("fused_adadelta", "twoshot_allreduce")] = graph_time(
            lambda: comm.all_reduce_symm(buf, False, native.ALGO_TWOSHOT))
        del fo
    arena._bump = mark0
    if rank == 0:
        print("[graph]", json.dumps(res["graph_us"]), flush=True)

    algos = [("oneshot", native.ALGO_ONESHOT), ("twoshot", native.ALGO_TWOSHOT)]
    if comm.multicast:
        algos.append(("nvls", native.ALGO_NVLS))
    sizes = []
    b = 64 << 10
    while b <= (args.max_mb << 20):
        sizes.append(b)
        b *= 4
    if sizes[-1] != (args.max_mb << 20):
        sizes.append(args.max_mb << 20)
    mark = arena._bump
    for dtype in (torch.bfloat16, torch.float32):
        for nbytes in sizes:
            arena._bump = mark                      # reuse the same arena region for every size
            esz = 2 if dtype == torch.bfloat16 else 4
            n = comm.pad_elems(nbytes // esz, dtype)
            _, buf = arena.empty((n,), dtype)
            buf.normal_()
            out = torch.empty_like(buf) if nbytes <= (4 << 20) else None
            real = n * esz
            iters = 100 if real <= (4 << 20) else (20 if real <= (64 << 20) else 6)
            floor_us = real * (1 + 1 / world) / (LINK_GBS * 1e3)
            row = {"dtype": str(dtype)[6:], "bytes": real, "nvls_floor_us": floor_us}
            for name, algo in algos:
                if name == "oneshot" and out is None:
                    continue
                us = ev_time(lambda: comm.all_reduce_symm(buf, False, algo, out=out), iters)
                row[name + "_us"] = us
                row[name + "_busbw_GBs"] = 2 * (world - 1) / world * real / us / 1e3
            nb = buf.clone()
            us = ev_time(lambda: dist.all_reduce(nb), iters)
            row["nccl_us"] = us
            row["nccl_busbw_GBs"] = 2 * (world - 1) / world * real / us / 1e3
            best = min(v for k, v in row.items() if k.endswith("_us") and not k.startswith(("nccl", "nvls_floor")))
            row["best_over_floor"] = floor_us / best
            row["best_vs_nccl"] = row["nccl_us"] / best
            res["allreduce"].append(row)
            del nb, out
            if rank == 0:
                print("[allreduce]", json.dumps(row), flush=True)
    arena._bump = mark

    # K4 (Adam, bf16 grads/params) at model sizes: MNIST-CNN, ResNet-50, BERT-base
    for label, n_params in (("mnist_1.2M", 1_199_882), ("resnet50_25.6M", 25_557_032), ("bert_base_110M", 110_106_428)):
        if n_params * 4 > (args.max_mb << 20) + (400 << 20):
            continue
        arena._bump = mark
        fo = commod.FusedShardedOptimizer(comm, [(n_params,)], commod.OptimizerSpec.adam(1e-3), torch.bfloat16,
                                          zero_grads=False)
        fo.init_from([torch.full((n_params,), 0.1, device="cuda")])
        fo.flat_grads.normal_()
        iters = 50 if n_params < 10_000_000 else 10
        us = ev_time(fo.step, iters)
        gb = fo.flat_grads.clone()
        pref = torch.full((fo.n,), 0.1, device="cuda")
        pref.grad = torch.zeros_like(pref)
        opt = torch.optim.Adam([pref], lr=1e-3, fused=True)
        pb16 = pref.to(torch.bfloat16)

        def standin():
            dist.all_reduce(gb)
            pref.grad.copy_(gb)
            pref.grad.mul_(1.0 / world)
            opt.step()
            pb16.copy_(pref)
        us_ref = ev_time(standin, iters)
        gbytes = fo.n * 2
        row = {"model": label, "n": fo.n, "fused_us": us, "nccl_fusedadam_standin_us": us_ref,
               "nvls_floor_us": gbytes * (1 + 1 / world) / (LINK_GBS * 1e3), "speedup": us_ref / us}
        res["fused_adam"].append(row)
        if rank == 0:
            print("[fused_adam]", json.dumps(row), flush=True)
        del fo, gb, pref, opt, pb16
        torch.cuda.empty_cache()

    if rank == 0:
        out = args.out or f"gpurun_out/comm_sweep_N{world}.json"
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)
        print("SWEEP DONE", out, flush=True)
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
