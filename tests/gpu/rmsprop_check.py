"""Multi-GPU check of the Keras RMSprop in the fused K4 step.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29627 \
        tests/gpu/rmsprop_check.py

(a) FusedShardedOptimizer in P2P and (when the GPUs support multicast) NVLS mode, every RMSprop variant, fp32
gradients / parameters, against TorchRMSprop on the full fp32 tensors with the rank-averaged gradient; the
parameters must be bit-identical on every rank, and the gathered states must match the reference's.
(b) DistributedDataParallel.fuse_optimizer("rmsprop") against torch DDP + TorchRMSprop.
"""
import copy
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

VARIANTS = {
    "plain": dict(momentum=0.0, centered=False),
    "momentum": dict(momentum=0.9, centered=False),
    "centered": dict(momentum=0.0, centered=True),
    "momentum_centered": dict(momentum=0.9, centered=True),
}
SHAPES = [(33, 17), (129,), (64, 32, 3, 3)]


def gen(rank, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + rank)
    return torch.randn(n, device="cuda", generator=g)


def identical_on_all_ranks(t):
    chk = t.double().sum().reshape(1)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return bool((lo == hi).item())


def check_k4(comm, rank, world, mode_name, variant):
    from tf_yarn_b200.keras.optimizers import RMSprop
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    desc = RMSprop(1e-3, rho=0.9, epsilon=1e-7, weight_decay=0.01, **VARIANTS[variant])
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
        opt.step()
    torch.cuda.synchronize()
    st = fo.gather_state()
    err = ((st["master"] - ref.detach()).abs() / ref.detach().abs().clamp_min(1e-2)).max().item()
    names = ["v"] + [k for k in ("m", "mg") if k in opt.state[ref]]
    serr = max(((st[f"s{i}"] - opt.state[ref][k]).abs().max() / opt.state[ref][k].abs().max().clamp_min(1e-6)).item()
               for i, k in enumerate(names, start=1))
    same = identical_on_all_ranks(fo.flat_params)
    # fp32: the reduction order of the `world` addends (in-switch for NVLS) is not the reference's
    good = err < 1e-3 and serr < 1e-3 and same and fo.step_count == 10
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] k4/{mode_name}/{variant}: max rel err {err:.2e}, state err {serr:.2e}, "
              f"ranks identical {same}", flush=True)
    return good


def make_model():
    torch.manual_seed(11)
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(4), nn.Flatten(),
                         nn.Linear(256, 300), nn.ReLU(), nn.Linear(300, 10))


def check_ddp(comm, rank, local):
    from tf_yarn_b200.keras.optimizers import TorchRMSprop
    from tf_yarn_b200.parallel.ddp import DistributedDataParallel
    hyper = dict(lr=1e-3, rho=0.9, momentum=0.9, eps=1e-7, centered=True)
    base = make_model().cuda()
    ref = torch.nn.parallel.DistributedDataParallel(copy.deepcopy(base), device_ids=[local])
    ref_opt = TorchRMSprop(ref.parameters(), **hyper)
    fused = DistributedDataParallel(copy.deepcopy(base), comm, bucket_cap_mb=1)
    fused_opt = fused.fuse_optimizer("rmsprop", **hyper)
    g = torch.Generator(device="cuda").manual_seed(100 + rank)
    for _ in range(6):
        x = torch.randn(16, 3, 8, 8, device="cuda", generator=g)
        y = torch.randint(0, 10, (16,), device="cuda", generator=g)
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
    good = worst < 2e-3 and same
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] ddp/fused_rmsprop: max rel diff vs torch DDP {worst:.2e}, "
              f"ranks identical {same}", flush=True)
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
        comm.multicast = use_multicast                # Communicator.mode follows it: P2P loads / stores otherwise
        mode_name = {native.MODE_LOCAL: "local", native.MODE_P2P: "p2p", native.MODE_NVLS: "nvls"}[comm.mode]
        for variant in VARIANTS:
            ok = check_k4(comm, rank, world, mode_name, variant) and ok
            dist.barrier()
    comm.multicast = multicast
    ok = check_ddp(comm, rank, local) and ok
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("RMSPROP CHECK", "OK" if flag.item() else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if flag.item() else 1


if __name__ == "__main__":
    sys.exit(main())
