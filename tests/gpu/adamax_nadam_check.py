"""Multi-GPU check of the Keras Adamax and Nadam in the fused K4 step.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29637 \
        tests/gpu/adamax_nadam_check.py

(a) FusedShardedOptimizer in P2P and (when the GPUs support multicast) NVLS mode, both optimizers, fp32 gradients /
parameters, against the float64 reference (tests/test_keras_adamax_nadam.py) of the rank-averaged gradient; the
parameters must be identical on every rank (params_in_sync), and so must Nadam's running product.
(b) DistributedDataParallel.fuse_optimizer("adamax" | "nadam") against torch DDP + TorchAdamax / torch.optim.NAdam.
"""
import copy
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from test_keras_adamax_nadam import CLASSES, NUMPY, nadam_mu  # noqa: E402

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


def params_in_sync(t):
    """Every rank holds rank 0's parameters bit for bit (the bench's params_in_sync)."""
    ref = t.clone()
    dist.broadcast(ref, 0)
    flag = torch.tensor([1 if torch.equal(ref, t) else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


def check_k4(comm, rank, world, mode_name, kind):
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    wd, steps = 0.01, 12
    desc = CLASSES[kind](1e-2, weight_decay=wd)
    fo = FusedShardedOptimizer(comm, SHAPES, desc.to_spec(), param_dtype=torch.float32, grad_dtype=torch.float32)
    init = [gen(0, int(torch.tensor(s).prod()), 100 + i).view(s) * 0.3 for i, s in enumerate(SHAPES)]
    fo.init_from(init, broadcast_root=0)
    p0 = torch.zeros(fo.n, device="cuda")
    for o, n, t in zip(fo.offsets, fo.numels, init):
        p0[o:o + n] = t.reshape(-1)
    grads = []
    for step in range(steps):
        per_rank = [gen(r, fo.n, step) * 0.5 for r in range(world)]
        fo.flat_grads.copy_(per_rank[rank])
        torch.cuda.synchronize()
        dist.barrier()
        fo.step()
        grads.append((sum(g.double() for g in per_rank) / world).cpu().numpy())
    torch.cuda.synchronize()
    want = NUMPY[kind](p0.double().cpu().numpy(), grads, [1e-2] * steps, range(1, steps + 1), 0.9, 0.999, 1e-7, wd)
    st = fo.gather_state()
    master = st["master"].double().cpu().numpy()
    real = np.concatenate([np.arange(o, o + n) for o, n in zip(fo.offsets, fo.numels)])
    err = float(np.abs(master[real] - want[0][real]).max()) / max(1.0, float(np.abs(want[0]).max()))
    same = identical_on_all_ranks(fo.flat_params)
    in_sync = params_in_sync(fo.flat_params)
    mu_ok = True
    if kind == "nadam":
        mu = torch.tensor([fo.mu_product], dtype=torch.float64, device="cuda")
        # the device holds beta_1 in fp32: its product follows the float64 formula of that value
        want_mu = float(np.prod([nadam_mu(float(np.float32(0.9)), t) for t in range(1, steps + 1)]))
        mu_ok = identical_on_all_ranks(mu) and abs(fo.mu_product - want_mu) < 1e-12 * want_mu
    # fp32: the reduction order of the `world` addends (in-switch for NVLS) is not the reference's
    good = err < 1e-4 and same and in_sync and mu_ok and fo.step_count == steps
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] k4/{mode_name}/{kind} world {world}: max rel err {err:.2e}, "
              f"ranks identical {same}, params_in_sync {in_sync}, mu_product ok {mu_ok}", flush=True)
    return good


def make_model():
    torch.manual_seed(11)
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(4), nn.Flatten(),
                         nn.Linear(256, 300), nn.ReLU(), nn.Linear(300, 10))


def check_ddp(comm, rank, local, kind):
    from tf_yarn_b200.parallel.ddp import DistributedDataParallel
    base = make_model().cuda()
    ref = torch.nn.parallel.DistributedDataParallel(copy.deepcopy(base), device_ids=[local])
    ref_opt = CLASSES[kind](1e-3, epsilon=1e-7).to_torch(ref.parameters())
    fused = DistributedDataParallel(copy.deepcopy(base), comm, bucket_cap_mb=1)
    fused_opt = fused.fuse_optimizer(kind, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
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
    if kind == "nadam":
        mus = [b["mu_product"] for b in fused_opt.state_dict()["buckets"]]
        good = good and all(v == mus[0] != 1.0 for v in mus)
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] ddp/fused_{kind}: max rel diff vs torch DDP {worst:.2e}, "
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
        for kind in CLASSES:
            ok = check_k4(comm, rank, world, mode_name, kind) and ok
            dist.barrier()
    comm.multicast = multicast
    for kind in CLASSES:
        ok = check_ddp(comm, rank, local, kind) and ok
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("ADAMAX NADAM CHECK", "OK" if flag.item() else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if flag.item() else 1


if __name__ == "__main__":
    sys.exit(main())
