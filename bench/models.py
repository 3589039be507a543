"""BASELINE.json configs 4 and 5 through bench.py (same JSON schema and timing harness as the headline).

    python bench.py --config resnet50 [--impl ours|standin|reference] --gpus N      (config 4: PytorchExperiment
        ResNet-50 DistributedDataParallel, images/s, per-GPU batch 64, bf16 autocast, SGD momentum)
    python bench.py --config bert [--impl ours|standin] --gpus N                    (config 5: Keras BERT-base
        Horovod path, sequences/s at seq 128, per-GPU batch 32, Adam)

ours / resnet50   : torchvision ResNet-50 wrapped by tf_yarn_b200.parallel.ddp (bucketed NVLS all-reduce kernels
                    overlapped with backward, no NCCL); cuDNN/cuBLAS compute (the conv/GEMM kernels of this repo are
                    specialised for the headline model, see DESIGN.md).
standin / resnet50: torch DistributedDataParallel + NCCL written directly (what the reference's worker does).
reference/resnet50: the UNMODIFIED reference worker (bench/ref_arm.py) with a PytorchExperiment of the same model.
ours / bert       : mini-Keras BERT-base, hvd.DistributedOptimizer(Adam): CUDA-graph step + fused
                    reduce-scatter/Adam/all-gather kernel (K4), side tasks (TensorBoard) live with --side-tasks.
standin / bert    : eager bf16 step, NCCL all-reduce of a fused bf16 buffer, torch.optim.Adam(fused=True).
"""
from __future__ import annotations

import os

from bench import common

RESNET_BATCH, BERT_BATCH, BERT_SEQ = 64, 32, 128
RESNET_POOL = 8            # 8 x 64 x 3 x 224 x 224 x 4 B = 308 MB of inputs (> 50 MB L2), rotated
BERT_POOL = 8


def _record(metric, unit, world, args, warm, repeats, ms_per_step, per_gpu_batch, impl, clocks, model, extra=None):
    cfg = {"model": model, "global_batch": world * per_gpu_batch, "per_gpu_batch": per_gpu_batch,
           "seq_len": BERT_SEQ if args.config == "bert" else None, "parallelism": f"dp{world}",
           "l2": "inputs rotate through a pool larger than the 50 MB L2" if args.config == "resnet50"
                 else "activations + 220 MB of bf16 weights per step exceed the 50 MB L2"}
    cfg.update(extra or {})
    return {"metric": metric, "value": world * per_gpu_batch / (ms_per_step * 1e-3), "unit": unit, "n_gpus": world,
            "steps": args.steps, "warmup": warm, "repeats": repeats, "ms_per_step": ms_per_step,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic, random-init weights", "impl": impl, "config": cfg, "clocks": clocks}


def resnet_pool(rank: int, pinned: bool = True):
    import torch
    g = torch.Generator().manual_seed(200 + rank)
    x = torch.randn((RESNET_POOL * RESNET_BATCH, 3, 224, 224), generator=g)
    y = torch.randint(0, 1000, (RESNET_POOL * RESNET_BATCH,), generator=g)
    if pinned:
        x, y = x.pin_memory(), y.pin_memory()
    return x, y


def run_resnet50(args):
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    import torchvision
    rank, local, world = common.dist_env()
    torch.cuda.set_device(local)
    common.quiet_nccl()
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    B = args.batch or RESNET_BATCH
    torch.manual_seed(0)
    model = torchvision.models.resnet50().cuda().to(memory_format=torch.channels_last)
    fused_opt = None
    if args.impl == "ours":
        from tf_yarn_b200.parallel import runtime
        from tf_yarn_b200.parallel.ddp import DistributedDataParallel
        comm = runtime.get_communicator(device=local)
        ddp = DistributedDataParallel(model, comm, bucket_cap_mb=25)
        if hasattr(ddp, "fuse_optimizer") and os.environ.get("TFY_DDP_FUSED", "1") == "1":
            fused_opt = ddp.fuse_optimizer("sgd", lr=0.01, momentum=0.9)
    else:
        ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], bucket_cap_mb=25) if world > 1 \
            else model
    opt = fused_opt if fused_opt is not None else torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    x_host, y_host = resnet_pool(rank)
    x_dev = x_host.cuda().contiguous(memory_format=torch.channels_last)
    y_dev = y_host.cuda()
    state = {"b": 0}
    loss_box = {}

    def step(xb, yb):
        if args.impl == "ours":
            ddp.zero_grad()
        else:
            opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(ddp(xb).float(), yb)
        loss.backward()
        opt.step()
        loss_box["loss"] = loss
        return loss

    def run(n):
        b = state["b"]
        for _ in range(n):
            step(x_dev[b * B:(b + 1) * B], y_dev[b * B:(b + 1) * B])
            b = (b + 1) % RESNET_POOL
        state["b"] = b

    steps, warm = args.steps, max(3, args.warmup)
    repeats = common.pick_repeats(steps, args.repeats or 3)
    sampler = common.ClockSampler(local)
    sampler.start()
    run(warm)
    region_ms = common.timed_regions(world, steps, repeats, run, None, None, sampler)
    clocks = sampler.stop()
    ms_per_step = common.median(region_ms) / steps

    last = {"loss": 0.0}

    def e2e_region():
        b = state["b"]
        for _ in range(steps):
            xb = x_host[b * B:(b + 1) * B].cuda(non_blocking=True).contiguous(memory_format=torch.channels_last)
            yb = y_host[b * B:(b + 1) * B].cuda(non_blocking=True)
            last["loss"] = step(xb, yb).item()
            b = (b + 1) % RESNET_POOL
        state["b"] = b

    e2e_region()
    e2e_ms = common.wall_regions(world, repeats, e2e_region)
    e2e_ms_per_step = common.median(e2e_ms) / steps
    flat = torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])
    in_sync = common.all_ranks_equal(common.tensor_checksum(flat), world)
    if rank == 0:
        desc = {"ours": "torchvision ResNet-50 (25,557,032 params) under tf_yarn_b200.parallel.ddp: bucketed NVLS "
                        "all-reduce kernels on a side stream" + (" + fused per-bucket SGD-momentum step (K4)"
                                                                 if fused_opt is not None else " + torch.optim.SGD"),
                "standin": "torchvision ResNet-50 under torch DistributedDataParallel (NCCL, 25 MB buckets) + "
                           "torch.optim.SGD"}[args.impl]
        out = _record("images/sec, PytorchExperiment ResNet-50 DistributedDataParallel (whole job)", "images/s", world,
                      args, warm, repeats, ms_per_step, B, args.impl, clocks, desc)
        out["e2e"] = {"value": world * B / (e2e_ms_per_step * 1e-3), "unit": "images/s",
                      "h2d_bytes_per_step": B * (3 * 224 * 224 * 4 + 8), "d2h_bytes_per_step": 4, "steps": steps,
                      "repeats": repeats, "ms_per_step": e2e_ms_per_step, "final_loss": last["loss"]}
        out["gpu_launches"] = (getattr(ddp, "kernel_launches", 0) if args.impl == "ours" else 0)
        out["params_in_sync"] = in_sync
        common.emit(out)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def run_bert(args):
    import torch
    import torch.distributed as dist
    from tf_yarn_b200.models.bert import BertForPreTraining, pretraining_loss, synthetic_batch
    rank, local, world = common.dist_env()
    torch.cuda.set_device(local)
    common.quiet_nccl()
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    B, S = args.batch or BERT_BATCH, BERT_SEQ
    torch.manual_seed(0)
    batches = [synthetic_batch(B, S, seed=rank * 100 + i) for i in range(BERT_POOL)]
    pinned = [({k: v.pin_memory() for k, v in x.items()}, {k: v.pin_memory() for k, v in y.items()})
              for x, y in batches]
    dev = [({k: v.cuda() for k, v in x.items()}, {k: v.cuda() for k, v in y.items()}) for x, y in batches]
    steps, warm = args.steps, max(3, args.warmup)
    repeats = common.pick_repeats(steps, args.repeats or 3)
    state = {"i": 0}
    side = _start_side_tasks(rank) if args.side_tasks else None
    h2d = sum(v.numel() * v.element_size() for d in batches[0] for v in d.values())
    launches = 0
    if args.impl == "ours":
        from tf_yarn_b200 import hvd, keras
        hvd.init()
        model = keras.Model.from_torch(BertForPreTraining(), name="bert_base")
        model.compile(loss=pretraining_loss, optimizer=hvd.DistributedOptimizer(keras.optimizers.Adam(1e-4)))
        model.fit(x=iter(pinned), steps_per_epoch=4, epochs=1, verbose=0)      # builds + captures
        eng = model._engine

        def run(n):
            for _ in range(n):
                xb, yb = dev[state["i"] % BERT_POOL]
                state["i"] += 1
                eng.launch_step(eng.stage_inputs(xb, yb))

        sampler = common.ClockSampler(local)
        sampler.start()
        with torch.cuda.stream(eng.stream):
            run(warm)
            l0 = eng.kernel_launches
            dev_barrier = (lambda: eng.comm.barrier(stream=eng.stream)) if world > 1 else None
            region_ms = common.timed_regions(world, steps, repeats, run, dev_barrier, eng.stream, sampler)
            launches = (eng.kernel_launches - l0) // (repeats * (steps + 1)) * steps
        clocks = sampler.stop()

        class _Pool:
            cardinality = None

            def __iter__(self):
                while True:
                    yield pinned[state["i"] % BERT_POOL]
                    state["i"] += 1

        losses = []

        def e2e_region():
            h = model.fit(_Pool(), steps_per_epoch=steps, epochs=1, verbose=0)
            losses.append(h.history["loss"][-1])
        e2e_region()
        e2e_ms = common.wall_regions(world, repeats, e2e_region)
        final_loss = losses[-1]
        eng.stream.synchronize()
        in_sync = common.all_ranks_equal(common.tensor_checksum(eng.fused.flat_params), world)
        desc = ("mini-Keras BERT-base + pre-training heads (110,106,428 params), hvd.DistributedOptimizer(Adam): "
                "CUDA-graph step (cuDNN/cuBLAS/SDPA compute) + fused reduce-scatter/Adam/all-gather kernel")
    else:
        import torch.nn.functional as F  # noqa: F401
        net = BertForPreTraining().cuda()
        params = list(net.parameters())
        opt = torch.optim.Adam(params, lr=1e-4, fused=True)
        n_total = sum(p.numel() for p in params)
        fusion = torch.zeros(n_total, dtype=torch.bfloat16, device="cuda")
        for p in params:
            p.grad = torch.zeros_like(p)
        views, o = [], 0
        for p in params:
            views.append(fusion[o:o + p.numel()].view_as(p))
            o += p.numel()
        grads = [p.grad for p in params]

        def step(xb, yb):
            opt.zero_grad(set_to_none=False)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = net(xb)
            loss = pretraining_loss(yb, out)
            loss.backward()
            if world > 1:
                torch._foreach_copy_(views, grads)
                dist.all_reduce(fusion)
                torch._foreach_copy_(grads, views)
                torch._foreach_mul_(grads, 1.0 / world)
            opt.step()
            return loss

        def run(n):
            for _ in range(n):
                xb, yb = dev[state["i"] % BERT_POOL]
                state["i"] += 1
                step(xb, yb)

        sampler = common.ClockSampler(local)
        sampler.start()
        run(warm)
        region_ms = common.timed_regions(world, steps, repeats, run, None, None, sampler)
        clocks = sampler.stop()
        last = {"loss": 0.0}

        def e2e_region():
            for _ in range(steps):
                xh, yh = pinned[state["i"] % BERT_POOL]
                state["i"] += 1
                xb = {k: v.cuda(non_blocking=True) for k, v in xh.items()}
                yb = {k: v.cuda(non_blocking=True) for k, v in yh.items()}
                last["loss"] = step(xb, yb).item()
        e2e_region()
        e2e_ms = common.wall_regions(world, repeats, e2e_region)
        final_loss = last["loss"]
        flat = torch.cat([p.detach().reshape(-1) for p in params])
        in_sync = common.all_ranks_equal(common.tensor_checksum(flat), world)
        desc = ("torch BERT-base + pre-training heads, autocast bf16, NCCL all-reduce of a fused bf16 buffer + "
                "torch.optim.Adam(fused=True), eager")
    ms_per_step = common.median(region_ms) / steps
    e2e_ms_per_step = common.median(e2e_ms) / steps
    side_info = _stop_side_tasks(side) if side is not None else None
    if rank == 0:
        out = _record("sequences/sec, Keras BERT-base Horovod path, seq 128 (whole job)", "sequences/s", world, args,
                      warm, repeats, ms_per_step, B, args.impl, clocks, desc, {"side_tasks": side_info})
        out["e2e"] = {"value": world * B / (e2e_ms_per_step * 1e-3), "unit": "sequences/s", "h2d_bytes_per_step": h2d,
                      "d2h_bytes_per_step": 4, "steps": steps, "repeats": repeats, "ms_per_step": e2e_ms_per_step,
                      "final_loss": final_loss}
        out["gpu_launches"] = launches
        out["params_in_sync"] = in_sync
        common.emit(out)
    if world > 1:
        if args.impl == "ours":
            from tf_yarn_b200 import hvd
            hvd.shutdown()
        dist.barrier()
        dist.destroy_process_group()
    return 0


def _start_side_tasks(rank: int):
    """BASELINE config 5 runs with the TensorBoard side task alive on the box: rank 0 starts the
    repo's TensorBoard task program on a scratch log directory (CPU only) for the duration of the run."""
    if rank != 0:
        return None
    import subprocess
    import sys
    import tempfile
    logdir = tempfile.mkdtemp(prefix="tfy_bench_tb_")
    from tf_yarn_b200.estimator import summary as summary_lib
    w = summary_lib.writer(logdir)
    w.add_scalar("bench/alive", 1.0, 0)
    w.flush()
    proc = subprocess.Popen([sys.executable, "-m", "tensorboard.main", "--logdir", logdir, "--port", "0",
                             "--host", "127.0.0.1"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return {"proc": proc, "logdir": logdir}


def _stop_side_tasks(side):
    if side is None:
        return None
    alive = side["proc"].poll() is None
    side["proc"].terminate()
    try:
        side["proc"].wait(10)
    except Exception:  # noqa: BLE001
        side["proc"].kill()
    return {"tensorboard_alive_at_end": alive}


def run(args):
    if args.config == "resnet50":
        if args.impl == "reference":
            from bench import ref_arm
            return ref_arm.run_reference(args)
        return run_resnet50(args)
    if args.impl == "reference":
        import json
        if common.dist_env()[0] == 0:
            print(json.dumps({"impl": "reference", "unavailable": "the reference's Keras/Horovod path needs TensorFlow "
                              "and Horovod, which are not installable offline; see --impl standin"}))
        return 0
    return run_bert(args)
