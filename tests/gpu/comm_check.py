"""Multi-GPU numerics + timing check of the comm kernels (run under torchrun on H100).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29511 tests/gpu/comm_check.py [--quick]

Every kernel is compared against a plain PyTorch fp32 reference of the same op
(the expected sum is computed locally from the deterministic per-rank inputs,
and cross-checked against NCCL).  Timings use CUDA events after warm-up and are
reduced with max over ranks.  Results: gpurun_out/comm_check_N<world>.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from tf_yarn_b200.ops import native  # noqa: E402
from tf_yarn_b200.parallel import comm as commod  # noqa: E402
from tf_yarn_b200.parallel.symm import StoreRendezvous, SymmArena  # noqa: E402


class TorchSymmArena:
    """Test-only arena backed by torch.distributed._symmetric_memory (cross-check of our VMM path)."""

    def __init__(self, size_bytes, device, rank, world):
        import ctypes
        import torch.distributed._symmetric_memory as symm_mem
        self.lib = native.load()
        self.rank, self.world, self.device = rank, world, device
        total = native.FLAGS_BYTES + size_bytes
        self._t = symm_mem.empty(total, dtype=torch.uint8, device=f"cuda:{device}")
        self._t.zero_()
        self._hdl = symm_mem.rendezvous(self._t, dist.group.WORLD.group_name)
        self.size = total
        self.peer_base = [int(p) for p in self._hdl.buffer_ptrs]
        self.mc_base = int(self._hdl.multicast_ptr or 0)
        self.multicast = self.mc_base != 0
        self.base = self.peer_base[rank]
        self._bump = native.FLAGS_BYTES
        self._mem = self._t
        self.epoch = torch.zeros(native.MAX_BLOCKS * native.MAX_RANKS, dtype=torch.int32, device=f"cuda:{device}")
        self.ctx = native.CommCtx()
        for r in range(world):
            self.ctx.peer_base[r] = self.peer_base[r]
        self.ctx.mc_base = self.mc_base
        self.ctx.epoch = self.epoch.data_ptr()
        self.ctx.rank, self.ctx.world = rank, world
        self.ctx_ref = ctypes.byref(self.ctx)
        dist.barrier()

    alloc = SymmArena.alloc
    tensor = SymmArena.tensor
    empty = SymmArena.empty
    offset_of = SymmArena.offset_of

    def close(self):
        pass


def ev_time(fn, iters, warmup=5):
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
    ms = s.elapsed_time(e) / iters
    t = torch.tensor([ms], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gen(rank, n, dtype, seed=0):
    g = torch.Generator(device="cuda")
    g.manual_seed(1234 + 17 * rank + seed)
    return (torch.randn(n, generator=g, device="cuda", dtype=torch.float32) * 0.5).to(dtype)


def ref_optimizer(kind, p, g, s1, s2, hp, step):
    """fp32 reference of the fused update (same math as tfy_opt_update)."""
    lr, p1, p2, eps, wd = hp["lr"], hp["p1"], hp["p2"], hp["eps"], hp["wd"]
    if kind == "sgd":
        g = g + wd * p
        if p1 != 0:
            s1 = g.clone() if step == 0 else p1 * s1 + (1 - p2) * g
            g = g + p1 * s1 if hp.get("nesterov") else s1
        p = p - lr * g
    elif kind == "adadelta":
        g = g + wd * p
        s1 = p1 * s1 + (1 - p1) * g * g
        upd = g * torch.sqrt(s2 + eps) / torch.sqrt(s1 + eps)
        s2 = p1 * s2 + (1 - p1) * upd * upd
        p = p - lr * upd
    elif kind == "adam":
        g = g + wd * p
        s1 = p1 * s1 + (1 - p1) * g
        s2 = p2 * s2 + (1 - p2) * g * g
        t = step + 1
        bc1 = 1 - p1 ** t
        bc2 = 1 - p2 ** t
        p = p - (lr / bc1) * (s1 / (torch.sqrt(s2) / (bc2 ** 0.5) + eps))
    elif kind == "adagrad":
        g = g + wd * p
        s1 = s1 + g * g
        p = p - lr * g / (torch.sqrt(s1) + eps)
    return p, s1, s2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--backend", default="vmm", choices=["vmm", "torch", "both"])
    args = ap.parse_args()

    import faulthandler
    faulthandler.dump_traceback_later(int(os.environ.get("TFY_CHECK_DUMP_AFTER", "100")), exit=True)
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    results = {"world": world, "tests": {}, "timing": {}, "errors": []}

    def record(name, ok, detail=None):
        flag = torch.tensor([1 if ok else 0], device="cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        results["tests"][name] = {"ok": bool(flag.item()), "detail": detail}
        if rank == 0:
            print(f"[{'PASS' if flag.item() else 'FAIL'}] {name} {detail if detail is not None else ''}", flush=True)

    backends = ["vmm", "torch"] if args.backend == "both" else [args.backend]
    for backend in backends:
        tag = backend
        try:
            arena_bytes = ((1 << 30) if args.quick else (4 << 30)) + (64 << 20)
            print(f"[rank {rank}] setting up {backend} arena", flush=True)
            if backend == "vmm":
                store = dist.distributed_c10d._get_default_store()
                rdv = StoreRendezvous(store, rank, world, prefix=f"chk_{backend}")
                t0 = time.time()
                arena = SymmArena(arena_bytes, device=local, rdv=rdv)
                results[f"{tag}_setup_s"] = time.time() - t0
            else:
                arena = TorchSymmArena(arena_bytes, local, rank, world)
            comm = commod.Communicator(fusion_bytes=64 << 20, arena=arena)
        except Exception as exc:  # noqa: BLE001
            results["errors"].append(f"{backend} arena: {exc!r}\n{traceback.format_exc()}")
            if rank == 0:
                print(f"[FAIL] {backend} arena setup: {exc!r}", flush=True)
            continue
        results[f"{tag}_multicast"] = bool(comm.multicast)
        if rank == 0:
            print(f"== backend {backend}: world={world} multicast={comm.multicast} "
                  f"arena={arena.size >> 20} MiB", flush=True)

        # ---------------------------------------------------------- barrier
        for _ in range(10):
            comm.barrier()
        torch.cuda.synchronize()
        record(f"{tag}/barrier", True)

        # ---------------------------------------------------------- all-reduce numerics
        algos = [("oneshot", native.ALGO_ONESHOT), ("twoshot", native.ALGO_TWOSHOT)]
        if comm.multicast:
            algos.append(("nvls", native.ALGO_NVLS))
        for dtype in (torch.bfloat16, torch.float32):
            n = comm.pad_elems(1_199_882, dtype)
            off, buf = arena.empty((n,), dtype)
            expect = sum(gen(r, n, dtype).float() for r in range(world))
            for name, algo in algos:
                buf.copy_(gen(rank, n, dtype))
                torch.cuda.synchronize()
                dist.barrier()
                out = comm.all_reduce_symm(buf, average=False, algo=algo)
                torch.cuda.synchronize()
                err = (out.float() - expect).abs().max().item()
                tol = 1e-5 * world if dtype == torch.float32 else 0.05 * world ** 0.5
                # all ranks must hold bit-identical results
                chk = out.float().sum().double()
                lo, hi = chk.clone(), chk.clone()
                dist.all_reduce(lo, op=dist.ReduceOp.MIN)
                dist.all_reduce(hi, op=dist.ReduceOp.MAX)
                same = bool((lo == hi).item())
                record(f"{tag}/allreduce/{name}/{str(dtype)[6:]}", err <= tol and same,
                       {"max_err": err, "identical": same})
                dist.barrier()

        # fused all_reduce of a tensor list (Horovod-style API) vs NCCL
        tensors = [gen(rank, s, torch.float32, seed=i) for i, s in enumerate([10, 1280, 9216 * 128, 64, 18432, 32, 288, 32])]
        ref = [t.clone() for t in tensors]
        for t in ref:
            dist.all_reduce(t)
            t /= world
        comm.all_reduce(tensors, average=True)
        torch.cuda.synchronize()
        err = max((a - b).abs().max().item() for a, b in zip(tensors, ref))
        record(f"{tag}/allreduce/fused_list_vs_nccl", err < 1e-5, {"max_err": err})

        # ---------------------------------------------------------- broadcast / all-gather
        x = gen(rank, 4096 * 33, torch.float32)
        comm.broadcast([x], root=0)
        torch.cuda.synchronize()
        record(f"{tag}/broadcast", torch.equal(x, gen(0, 4096 * 33, torch.float32)))
        if world > 1:
            x = gen(rank, 4096 * 33, torch.float32)
            comm.broadcast([x], root=world - 1)
            torch.cuda.synchronize()
            record(f"{tag}/broadcast_root_last", torch.equal(x, gen(world - 1, 4096 * 33, torch.float32)))
        g = comm.all_gather(gen(rank, 1000, torch.float32))
        torch.cuda.synchronize()
        exp = torch.cat([gen(r, 1000, torch.float32) for r in range(world)])
        record(f"{tag}/allgather", torch.equal(g, exp))

        # ---------------------------------------------------------- fused step numerics
        shapes = [(32, 1, 3, 3), (32,), (64, 32, 3, 3), (64,), (128, 9216), (128,), (10, 128), (10,)]
        specs = {
            "adadelta": (commod.OptimizerSpec.adadelta(lr=1.0 * world, rho=0.95, eps=1e-7),
                         dict(lr=1.0 * world, p1=0.95, p2=0.0, eps=1e-7, wd=0.0)),
            "adam": (commod.OptimizerSpec.adam(lr=1e-3, weight_decay=0.01),
                     dict(lr=1e-3, p1=0.9, p2=0.999, eps=1e-8, wd=0.01)),
            "sgd": (commod.OptimizerSpec.sgd(lr=0.05, momentum=0.9, nesterov=True),
                    dict(lr=0.05, p1=0.9, p2=0.0, eps=0.0, wd=0.0, nesterov=True)),
            "adagrad": (commod.OptimizerSpec.adagrad(lr=0.05, eps=1e-10, initial_accumulator_value=0.1),
                        dict(lr=0.05, p1=0.0, p2=0.0, eps=1e-10, wd=0.0)),
        }
        for pdt, gdt in ((torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32)):
            for kind, (spec, hp) in specs.items():
                fo = commod.FusedShardedOptimizer(comm, shapes, spec, param_dtype=pdt, grad_dtype=gdt)
                init = [gen(0, int(torch.tensor(s).prod()), torch.float32, seed=100 + i).view(s) * 0.2
                        for i, s in enumerate(shapes)]
                fo.init_from(init, broadcast_root=0)
                # reference state (full, fp32)
                P = torch.zeros(fo.n, device="cuda")
                for o, nn, t in zip(fo.offsets, fo.numels, init):
                    P[o:o + nn] = t.reshape(-1)
                S1 = torch.full_like(P, spec.init_s1)
                S2 = torch.zeros_like(P)
                _, scratch_g = arena.empty((fo.n,), gdt)
                ok = True
                worst = 0.0
                for step in range(4):
                    grads_all = [gen(r, fo.n, gdt, seed=1000 + step) for r in range(world)]
                    fo.flat_grads.copy_(grads_all[rank])
                    torch.cuda.synchronize()
                    dist.barrier()
                    fo.step()
                    torch.cuda.synchronize()
                    G = sum(x.float() for x in grads_all)
                    if gdt == torch.bfloat16 and comm.mode == native.MODE_NVLS:
                        # the NVSwitch returns the bf16 sum with its own rounding (not round-to-nearest):
                        # take the reference gradient from the plain NVLS all-reduce kernel (validated
                        # above against the exact sum) so the optimizer math is compared bit-for-bit
                        scratch_g.copy_(grads_all[rank])
                        torch.cuda.synchronize()
                        dist.barrier()
                        G = comm.all_reduce_symm(scratch_g, average=False, algo=native.ALGO_NVLS).float().clone()
                        torch.cuda.synchronize()
                        dist.barrier()
                    G = G / world
                    P, S1, S2 = ref_optimizer(kind, P, G, S1, S2, hp, step)
                    got = fo.flat_params.float()
                    expect = P.to(pdt).float()
                    denom = expect.abs().clamp_min(1e-3)
                    rel = ((got - expect).abs() / denom).max().item()
                    worst = max(worst, rel)
                    # fp32: the in-switch summation order of `world` addends is not the reference's; Adadelta's
                    # rsqrt amplifies the last-bit differences
                    tol = 2e-2 if pdt == torch.bfloat16 else 2e-4 * max(1, world // 2)
                    if gdt == torch.bfloat16 and comm.mode != native.MODE_NVLS:
                        tol = max(tol, 2e-2)
                    # the replicated compute params must be exactly the (gathered) fp32 master cast down
                    if rel >= tol and rank == 0:
                        relv = (got - expect).abs() / denom
                        worst_idx = torch.topk(relv, 8).indices
                        print(f"[diag] {kind}/{pdt} step {step}: worst idx {worst_idx.tolist()} "
                              f"got {got[worst_idx].tolist()} expect {expect[worst_idx].tolist()} "
                              f"G {G[worst_idx].tolist()} n={fo.n} shard={fo.shard_n} "
                              f"n_bad={(relv >= tol).sum().item()}", flush=True)
                    ok = ok and rel < tol and bool((fo.flat_grads == 0).all().item())
                stp = fo.step_count
                ok = ok and stp == 4
                record(f"{tag}/fused/{kind}/{str(pdt)[6:]}", ok, {"max_rel_err": worst, "step": stp})
                # sharded state gather must reproduce the reference master
                st = fo.gather_state()
                merr = (st["master"] - P).abs().max().item()
                record(f"{tag}/fused/{kind}/{str(pdt)[6:]}/gather_state", merr < 1e-3, {"max_err": merr})
                dist.barrier()

        # ---------------------------------------------------------- CUDA graph replay of the fused step
        fo = commod.FusedShardedOptimizer(comm, shapes, commod.OptimizerSpec.adadelta(1.0), torch.bfloat16)
        fo.init_from([torch.ones(s, device="cuda") for s in shapes])
        gsrc = gen(rank, fo.n, torch.bfloat16, seed=7)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                fo.flat_grads.copy_(gsrc)
                fo.step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        dist.barrier()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fo.flat_grads.copy_(gsrc)
            fo.step()
        for _ in range(5):
            graph.replay()
        torch.cuda.synchronize()
        record(f"{tag}/fused/cuda_graph_replay", fo.step_count == 7, {"step": fo.step_count})

        # ---------------------------------------------------------- timings
        if backend == backends[0] or args.backend == "both":
            sizes = [("mnist_2.4MB_bf16", 1_199_882, torch.bfloat16), ("mnist_4.8MB_f32", 1_199_882, torch.float32)]
            if not args.quick:
                sizes += [("resnet50_51MB_bf16", 25_557_032, torch.bfloat16),
                          ("bert_220MB_bf16", 110_106_428, torch.bfloat16),
                          ("256MB_f32", 64 << 20, torch.float32)]
            for label, nel, dtype in sizes:
                n = comm.pad_elems(nel, dtype)
                off, buf = arena.empty((n,), dtype)
                buf.copy_(gen(rank, n, dtype))
                outb = torch.empty_like(buf)
                nbytes = n * buf.element_size()
                iters = 50 if nbytes < (32 << 20) else 10
                row = {"bytes": nbytes}
                for name, algo in algos:
                    if name == "oneshot" and nbytes > (16 << 20):
                        continue
                    ms = ev_time(lambda: comm.all_reduce_symm(buf, False, algo, out=outb), iters)
                    row[name + "_us"] = ms * 1e3
                    row[name + "_busbw_GBs"] = 2 * (world - 1) / world * nbytes / (ms * 1e-3) / 1e9 if world > 1 else None
                nb = buf.clone()
                ms = ev_time(lambda: dist.all_reduce(nb), iters)
                row["nccl_us"] = ms * 1e3
                row["nccl_busbw_GBs"] = 2 * (world - 1) / world * nbytes / (ms * 1e-3) / 1e9 if world > 1 else None
                results["timing"][f"{tag}/allreduce/{label}"] = row
                if rank == 0:
                    print(f"[time] {tag} allreduce {label}: {json.dumps(row)}", flush=True)

            # fused step vs (NCCL allreduce + cast + torch.optim) stand-in
            fsizes = [("mnist", [(32, 1, 3, 3), (32,), (64, 32, 3, 3), (64,), (128, 9216), (128,), (10, 128), (10,)])]
            if not args.quick:
                fsizes.append(("bert_base_110M", [(110_106_428,)]))
            for label, shp in fsizes:
                for kind, spec in (("adadelta", commod.OptimizerSpec.adadelta(1.0)),
                                   ("adam", commod.OptimizerSpec.adam(1e-3))):
                    fo = commod.FusedShardedOptimizer(comm, shp, spec, torch.bfloat16, zero_grads=False)
                    fo.init_from([torch.ones(s, device="cuda") * 0.1 for s in shp])
                    fo.flat_grads.copy_(gen(rank, fo.n, torch.bfloat16))
                    iters = 50 if fo.n < 10_000_000 else 10
                    ms = ev_time(fo.step, iters)
                    # graph-replayed (launch-latency free) number
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        for _ in range(10):
                            fo.step()
                    ms_g = ev_time(graph.replay, max(2, iters // 10), warmup=2) / 10
                    # stand-in: NCCL allreduce of bf16 grads -> fp32 cast/scale -> torch.optim
                    pref = torch.ones(fo.n, device="cuda") * 0.1
                    pref.grad = torch.zeros_like(pref)
                    opt = (torch.optim.Adadelta([pref], lr=1.0, rho=0.95, eps=1e-7) if kind == "adadelta"
                           else torch.optim.Adam([pref], lr=1e-3))
                    gb = gen(rank, fo.n, torch.bfloat16)
                    pb16 = pref.to(torch.bfloat16)

                    def standin():
                        dist.all_reduce(gb)
                        pref.grad.copy_(gb)
                        pref.grad.mul_(1.0 / world)
                        opt.step()
                        pb16.copy_(pref)
                    ms_ref = ev_time(standin, iters)
                    row = {"n": fo.n, "fused_us": ms * 1e3, "fused_graph_us": ms_g * 1e3,
                           "nccl_standin_us": ms_ref * 1e3}
                    results["timing"][f"{tag}/fused_step/{label}/{kind}"] = row
                    if rank == 0:
                        print(f"[time] {tag} fused_step {label} {kind}: {json.dumps(row)}", flush=True)
        dist.barrier()
        comm.close()

    if rank == 0:
        os.makedirs("gpurun_out", exist_ok=True)
        with open(f"gpurun_out/comm_check_N{world}_{args.backend}.json", "w") as f:
            json.dump(results, f, indent=1)
        n_fail = sum(1 for t in results["tests"].values() if not t["ok"]) + len(results["errors"])
        print(f"SUMMARY world={world} tests={len(results['tests'])} failed={n_fail}", flush=True)
        for e in results["errors"]:
            print(e)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
