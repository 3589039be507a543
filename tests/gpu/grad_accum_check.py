"""Multi-GPU check of Keras gradient accumulation in the fused step.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29631 \
        tests/gpu/grad_accum_check.py

FusedShardedOptimizer with bf16 gradients / parameters and ``accumulation_steps=4``, in P2P and (when the GPUs
support multicast) NVLS mode: the fused step reads the fp32 accumulator, so these runs launch its instantiations with
fp32 gradients and bf16 parameters.  Over 10 batches of per-rank gradients: the parameters move on batches 3 and 7
only, are bit-identical on every rank, and match torch Adam on the mean over ranks and batches (fp32 master); a
checkpoint taken after 6 batches (2 pending) and restored onto rank 0 continues to the same result up to the order
of the fp32 sums.
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

SHAPES = [(33, 17), (129,), (64, 32, 3, 3)]
N, BATCHES = 4, 10


def gen(rank, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed * 1000 + rank)
    return torch.randn(n, device="cuda", generator=g)


def identical_on_all_ranks(t):
    chk = t.double().sum().reshape(1)
    lo, hi = chk.clone(), chk.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return bool((lo == hi).item())


def make(comm):
    from tf_yarn_b200.keras.optimizers import Adam
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    desc = Adam(1e-2, gradient_accumulation_steps=N)
    fo = FusedShardedOptimizer(comm, SHAPES, desc.to_spec(), param_dtype=torch.bfloat16, grad_dtype=torch.bfloat16,
                               accumulation_steps=N)
    init = [gen(0, int(torch.tensor(s).prod()), 100 + i).view(s) * 0.3 for i, s in enumerate(SHAPES)]
    fo.init_from(init, broadcast_root=0)
    return desc, fo, init


def batch(fo, rank, s):
    fo.flat_grads.copy_((gen(rank, fo.n, s) * 0.5).to(torch.bfloat16))
    torch.cuda.synchronize()
    dist.barrier()
    update = (fo.step_count + 1) % N == 0
    fo.accumulate(advance=not update)
    if update:
        fo.step_accumulated()
    torch.cuda.synchronize()
    return update


def check(comm, rank, world, mode_name):
    desc, fo, init = make(comm)
    ref = torch.zeros(fo.n, device="cuda", requires_grad=True)
    with torch.no_grad():
        for o, n, t in zip(fo.offsets, fo.numels, init):
            ref[o:o + n] = t.reshape(-1)
    opt = torch.optim.Adam([ref], lr=1e-2, eps=1e-7)
    acc = torch.zeros(fo.n, device="cuda")
    moved_ok = True
    for s in range(BATCHES):
        before = fo.master.clone()
        update = batch(fo, rank, s)
        moved_ok &= (not torch.equal(before, fo.master)) == update
        acc += sum((gen(r, fo.n, s) * 0.5).to(torch.bfloat16).float() for r in range(world))
        if update:
            st = opt.state[ref]                 # Adam's bias correction at t = s + 1 (the batch count)
            if not st:
                st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(ref), torch.zeros_like(ref)
            st["step"] = torch.tensor(float(s))
            ref.grad = acc * float(torch.tensor(1.0 / N, dtype=torch.float32)) / world
            opt.step()
            acc.zero_()
    st = fo.gather_state()
    err = ((st["master"] - ref.detach()).abs() / ref.detach().abs().clamp_min(1e-2)).max().item()
    same = identical_on_all_ranks(fo.flat_params) and identical_on_all_ranks(st["master"])
    # resume: 6 batches, checkpoint (2 pending, their sum over ranks), restore, 4 more
    _, first, _ = make(comm)
    for s in range(6):
        batch(first, rank, s)
    ck = first.gather_state()
    _, resumed, _ = make(comm)
    resumed.load_state(ck)
    pending_ok = "grad_accum" in ck and (rank == 0 or float(resumed.flat_acc.abs().max()) == 0.0)
    for s in range(6, BATCHES):
        batch(resumed, rank, s)
    rs = resumed.gather_state()
    rerr = ((rs["master"] - st["master"]).abs() / st["master"].abs().clamp_min(1e-2)).max().item()
    good = err < 1e-3 and same and moved_ok and pending_ok and rerr < 1e-5 and fo.step_count == BATCHES
    if rank == 0:
        print(f"[{'PASS' if good else 'FAIL'}] {mode_name}: max rel err vs torch Adam {err:.2e}, ranks identical "
              f"{same}, moved on update batches only {moved_ok}, resume rel diff {rerr:.2e}", flush=True)
    return good


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from tf_yarn_b200.ops import native
    from tf_yarn_b200.parallel import runtime
    comm = runtime.get_communicator(device=local)
    ok = True
    multicast = comm.multicast
    for use_multicast in ([True] if multicast else []) + [False]:
        comm.multicast = use_multicast
        mode_name = {native.MODE_LOCAL: "local", native.MODE_P2P: "p2p", native.MODE_NVLS: "nvls"}[comm.mode]
        ok = check(comm, rank, world, mode_name) and ok
        dist.barrier()
    comm.multicast = multicast
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("GRAD ACCUM CHECK", "OK" if flag.item() else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if flag.item() else 1


if __name__ == "__main__":
    sys.exit(main())
