"""Multi-GPU check of Keras learning-rate schedules in the fused K4 step.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29631 \
        tests/gpu/lr_schedule_check.py

(a) FusedShardedOptimizer in P2P and (when the GPUs support multicast) NVLS mode, Adam and RMSprop with a cosine
warm-up and a piecewise schedule, fp32 gradients / parameters: after 10 steps every rank's device learning rate is the
schedule at step 10, bit for bit on every rank, and the parameters match torch.optim on the rank-averaged gradient
driven by the schedule's rate step by step.
(b) DistributedDataParallel.fuse_optimizer("adam", lr=<schedule>) against torch DDP + Adam driven by the same rates;
a restored optimizer state writes the rate of the restored step.
"""
import copy
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

SHAPES = [(33, 17), (129,), (64, 32, 3, 3)]


def schedules():
    from tf_yarn_b200.keras import schedules as S
    return {"cosine_warmup": S.CosineDecay(0.0, 8, alpha=0.1, warmup_target=2e-3, warmup_steps=3),
            "piecewise": S.PiecewiseConstantDecay([2, 6], [2e-3, 1e-3, 2e-4])}


def gen(rank, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + rank)
    return torch.randn(n, device="cuda", generator=g)


def identical_on_all_ranks(t):
    chk = t.double().sum().reshape(1)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return bool((lo == hi).item())


def check_k4(comm, rank, world, mode_name, opt_name, sched_name):
    from tf_yarn_b200.keras import optimizers as O
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    sch = schedules()[sched_name]
    desc = O.Adam(sch) if opt_name == "adam" else O.RMSprop(sch, momentum=0.9, centered=True)
    fo = FusedShardedOptimizer(comm, SHAPES, desc.to_spec(), param_dtype=torch.float32, grad_dtype=torch.float32)
    init = [gen(0, int(torch.tensor(s).prod()), 100 + i).view(s) * 0.3 for i, s in enumerate(SHAPES)]
    fo.init_from(init, broadcast_root=0)
    ref = torch.zeros(fo.n, device="cuda", requires_grad=True)
    with torch.no_grad():
        for o, n, t in zip(fo.offsets, fo.numels, init):
            ref[o:o + n] = t.reshape(-1)
    opt = desc.to_torch([ref])
    for step in range(10):
        grads = [gen(r, fo.n, step) * 0.5 for r in range(world)]
        fo.flat_grads.copy_(grads[rank])
        torch.cuda.synchronize()
        dist.barrier()
        fo.step()
        ref.grad = sum(grads) / world
        for g in opt.param_groups:
            g["lr"] = sch(step)
        opt.step()
    torch.cuda.synchronize()
    lr = fo.hyper[0:4].view(torch.float32).clone()
    lr_ok = float(lr.item()) == sch(10) and identical_on_all_ranks(lr)
    st = fo.gather_state()
    err = ((st["master"] - ref.detach()).abs() / ref.detach().abs().clamp_min(1e-2)).max().item()
    same = identical_on_all_ranks(fo.flat_params)
    good = err < 1e-3 and same and lr_ok and fo.step_count == 10
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] k4/{mode_name}/{opt_name}/{sched_name}: max rel err {err:.2e}, "
              f"device lr {lr.item():.9g} (schedule {sch(10):.9g}), ranks identical {same}", flush=True)
    return good


def make_model():
    torch.manual_seed(11)
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(4), nn.Flatten(),
                         nn.Linear(256, 300), nn.ReLU(), nn.Linear(300, 10))


def check_ddp(comm, rank, local):
    from tf_yarn_b200.parallel.ddp import DistributedDataParallel
    sch = schedules()["cosine_warmup"]
    base = make_model().cuda()
    ref = torch.nn.parallel.DistributedDataParallel(copy.deepcopy(base), device_ids=[local])
    ref_opt = torch.optim.Adam(ref.parameters(), lr=sch(0), eps=1e-7)
    fused = DistributedDataParallel(copy.deepcopy(base), comm, bucket_cap_mb=1)
    fused_opt = fused.fuse_optimizer("adam", lr=sch, eps=1e-7)
    g = torch.Generator(device="cuda").manual_seed(100 + rank)
    for step in range(6):
        x = torch.randn(16, 3, 8, 8, device="cuda", generator=g)
        y = torch.randint(0, 10, (16,), device="cuda", generator=g)
        for grp in ref_opt.param_groups:
            grp["lr"] = sch(step)
        for m, o in ((ref, ref_opt), (fused, fused_opt)):
            o.zero_grad()
            if m is not ref:
                m.zero_grad()
            nn.functional.cross_entropy(m(x), y).backward()
            o.step()
        torch.cuda.synchronize()
    worst = 0.0
    for p, q in zip(fused.module.parameters(), ref.module.parameters()):
        worst = max(worst, (p.detach() - q.detach()).abs().max().item() / (q.detach().abs().max().item() + 1e-6))
    same = identical_on_all_ranks(torch.cat([p.detach().reshape(-1) for p in fused.module.parameters()]))
    lrs = [float(b.hyper[0:4].view(torch.float32).item()) for b in fused._buckets]
    lr_ok = all(v == sch(6) for v in lrs)
    # a restored state (step 2) writes the rate of step 2 into every bucket
    st = fused_opt.state_dict()
    for b in st["buckets"]:
        b["step"] = 2
    fused_opt.load_state_dict(st)
    torch.cuda.synchronize()
    lr_ok = lr_ok and all(float(b.hyper[0:4].view(torch.float32).item()) == sch(2) for b in fused._buckets)
    good = worst < 2e-3 and same and lr_ok
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] ddp/fused_adam_cosine_warmup: max rel diff vs torch DDP {worst:.2e}, "
              f"ranks identical {same}, device lr {lrs} (schedule {sch(6):.9g})", flush=True)
    return good


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from tf_yarn_b200.parallel import runtime
    comm = runtime.get_communicator(device=local)
    ok = True
    from tf_yarn_b200.ops import native
    multicast = comm.multicast
    for use_multicast in ([True] if multicast else []) + [False]:
        comm.multicast = use_multicast
        mode_name = {native.MODE_LOCAL: "local", native.MODE_P2P: "p2p", native.MODE_NVLS: "nvls"}[comm.mode]
        for opt_name in ("adam", "rmsprop"):
            for sched_name in schedules():
                ok = check_k4(comm, rank, world, mode_name, opt_name, sched_name) and ok
                dist.barrier()
    comm.multicast = multicast
    ok = check_ddp(comm, rank, local) and ok
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("LR SCHEDULE CHECK", "OK" if flag.item() else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if flag.item() else 1


if __name__ == "__main__":
    sys.exit(main())
