"""Headline config: Keras MNIST-CNN, Horovod path (BASELINE.json config 2), arms `ours` and `standin`."""
from __future__ import annotations

import os
import sys

from bench import common

PER_GPU_BATCH = 128
POOL_BATCHES = 672          # 672 * 128 * 784 * 4 B = 269.7 MB  > 50 MB L2
METRIC = "samples/sec, Keras MNIST-CNN Horovod path (whole job)"
DATA = ("synthetic (MNIST-shaped, class-conditional so the loss can fall: x = 0.5*template[y] + 0.5*U(0,1)), "
        "random-init weights")
MODEL = "Keras MNIST-CNN (1,199,882 params), Adadelta(1.0*size), Horovod path"
L2_NOTE = "inputs rotate through a 269.7 MB pool (> 50 MB L2); no flush"


def make_pool(seed: int, nhwc: bool = True):
    """Learnable synthetic MNIST: ten fixed random templates (same on every rank) + per-sample noise."""
    import torch
    gt = torch.Generator().manual_seed(4242)
    templates = torch.rand((10, 28, 28), generator=gt)
    g = torch.Generator().manual_seed(seed)
    n = POOL_BATCHES * PER_GPU_BATCH
    y = torch.randint(0, 10, (n,), generator=g)
    x = torch.rand((n, 28, 28), generator=g).mul_(0.5).add_(templates[y] * 0.5)
    x = x.unsqueeze(-1) if nhwc else x.unsqueeze(1)
    return x.contiguous(), y


def base_record(world, steps, warm, repeats, ms_per_step, impl, clocks, extra_config=None):
    value = world * PER_GPU_BATCH / (ms_per_step * 1e-3)
    cfg = {"model": MODEL, "global_batch": world * PER_GPU_BATCH, "per_gpu_batch": PER_GPU_BATCH,
           "seq_len": None, "parallelism": f"dp{world}", "l2": L2_NOTE}
    cfg.update(extra_config or {})
    return {"metric": METRIC, "value": value, "unit": "samples/s", "n_gpus": world, "steps": steps,
            "warmup": warm, "repeats": repeats, "ms_per_step": ms_per_step, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": DATA, "impl": impl,
            "config": cfg, "clocks": clocks}


# ------------------------------------------------------------------------------------------------------
# ours
# ------------------------------------------------------------------------------------------------------
def _build_model(distributed: bool, world: int):
    from tf_yarn_b200 import hvd, keras
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
    import torch
    torch.manual_seed(1234)      # identical init on every rank (BroadcastGlobalVariables also runs)
    model = keras_mnist_cnn(logits=True)
    opt = keras.optimizers.Adadelta(1.0 * world)
    if distributed:
        opt = hvd.DistributedOptimizer(opt)
    model.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=opt)
    return model


def run_ours(args):
    import torch
    import torch.distributed as dist
    rank, local, world = common.dist_env()
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run")
    torch.cuda.set_device(local)
    common.quiet_nccl()
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from tf_yarn_b200 import hvd

    hvd.init()
    model = _build_model(True, world)
    callbacks = [hvd.callbacks.BroadcastGlobalVariablesCallback(0)]

    x_host, y_host = make_pool(seed=100 + rank)
    x_host, y_host = x_host.pin_memory(), y_host.pin_memory()
    h2d_bytes = PER_GPU_BATCH * (28 * 28 * 4 + 8)
    B = PER_GPU_BATCH
    steps = args.steps
    repeats = common.pick_repeats(steps, args.repeats)

    # ---- warm-up through the public API (builds the engine, captures the graph) ----------------
    warm = max(3, args.warmup)
    hist0 = model.fit(x_host[:warm * B], y_host[:warm * B], batch_size=B, epochs=1, shuffle=False, verbose=0,
                      callbacks=callbacks)
    initial_loss = hist0.history["loss"][0]
    eng = model._engine
    torch.cuda.synchronize()

    # ---- device-timed regions: inputs resident in HBM, pool larger than L2 ----------------------
    x_dev, y_dev = x_host.cuda(non_blocking=True), y_host.cuda(non_blocking=True)
    torch.cuda.synchronize()
    pool = [(x_dev[b * B:(b + 1) * B], y_dev[b * B:(b + 1) * B]) for b in range(POOL_BATCHES)]

    def make_runner(engine):
        state = {"b": 0}

        def run(n):
            b = state["b"]
            ticket = engine.stage_inputs(*pool[b])
            for i in range(n):
                engine.launch_step(ticket)
                b = (b + 1) % POOL_BATCHES
                if i + 1 < n:
                    ticket = engine.stage_inputs(*pool[b])
            state["b"] = b
        return run

    sampler = common.ClockSampler(local)
    sampler.start()                      # before any barrier, on every rank
    run = make_runner(eng)
    dev_barrier = (lambda: eng.comm.barrier(stream=eng.stream)) if world > 1 else None
    with torch.cuda.stream(eng.stream):  # replays are issued from the engine's stream (as fit() does)
        run(warm)
        launches0 = eng.kernel_launches
        run(steps)
        launches = eng.kernel_launches - launches0
        eng.stream.synchronize()
        region_ms = common.timed_regions(world, steps, repeats, run, dev_barrier, eng.stream, sampler)
    clocks = sampler.stop()
    if args.dump_outputs and rank == 0:
        eng.stream.synchronize()
        common.dump_outputs(args.dump_outputs, {"loss": eng._loss, "params": eng.fused.flat_params})
    ms_per_step = common.median(region_ms) / steps

    # ---- exposed communication: the same step with the exchange in LOCAL mode (world-1 arena) ----
    exposed_ms = 0.0
    local_ms_per_step = ms_per_step
    if world > 1 and not args.no_exposed:
        model_l = _build_model(False, world)
        model_l.fit(x_host[:warm * B], y_host[:warm * B], batch_size=B, epochs=1, shuffle=False, verbose=0)
        eng_l = model_l._engine
        run_l = make_runner(eng_l)
        with torch.cuda.stream(eng_l.stream):
            run_l(warm)
            eng_l.stream.synchronize()
            # same harness (cross-GPU barrier + untimed step before each region) so only the exchange differs
            local_regions = common.timed_regions(world, steps, repeats, run_l, None, eng_l.stream, None)
        local_ms_per_step = common.median(local_regions) / steps
        exposed_ms = max(0.0, ms_per_step - local_ms_per_step)
        del model_l, eng_l

    # ---- end-to-end regions: model.fit with per-step H2D (pinned) + per-step loss D2H ------------
    class _HostPool:
        cardinality = None

        def __init__(self, first_batch):
            self.b = first_batch

        def __iter__(self):
            while True:
                b = self.b
                self.b = (b + 1) % POOL_BATCHES
                yield (x_host[b * B:(b + 1) * B], y_host[b * B:(b + 1) * B])

    host_pool = _HostPool(warm % POOL_BATCHES)
    losses = []

    def e2e_region():
        h = model.fit(host_pool, steps_per_epoch=steps, epochs=1, verbose=0)
        losses.append(h.history["loss"][-1])

    e2e_region()                                  # untimed: first fit() after the device loop
    e2e_ms = common.wall_regions(world, repeats, e2e_region)
    e2e_ms_per_step = common.median(e2e_ms) / steps
    final_loss = losses[-1]

    # ---- the ranks must hold bit-identical parameters after all those steps ----------------------
    eng.stream.synchronize()
    in_sync = common.all_ranks_equal(common.tensor_checksum(eng.fused.flat_params), world)

    if rank == 0:
        out = base_record(world, steps, warm, repeats, ms_per_step, "ours", clocks, {
            "comm": ("NVLS multimem" if eng.comm.multicast else ("P2P" if world > 1 else "local")),
            "cuda_graph": eng.graph is not None})
        out["e2e"] = {"value": world * B / (e2e_ms_per_step * 1e-3), "unit": "samples/s",
                      "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4, "steps": steps, "repeats": repeats,
                      "ms_per_step": e2e_ms_per_step, "initial_loss": initial_loss, "final_loss": final_loss,
                      "loss_fell": bool(final_loss < 0.5 * initial_loss)}
        out["gpu_launches"] = launches
        out["exposed_comm_ms"] = exposed_ms
        out["local_mode_ms_per_step"] = local_ms_per_step
        out["params_in_sync"] = in_sync
        out["region_ms"] = {"min": min(region_ms), "median": common.median(region_ms), "max": max(region_ms)}
        common.emit(out)
    if world > 1:
        hvd.shutdown()
        dist.destroy_process_group()
    return 0 if in_sync else 3


# ------------------------------------------------------------------------------------------------------
# stand-in: stock PyTorch rendition of the reference's Horovod path on an NCCL build
# ------------------------------------------------------------------------------------------------------
def run_standin(args):
    """NCCL all-reduce of a fused bf16 gradient buffer + cast/scale + torch.optim.Adadelta.  With --graph the
    whole step (NCCL included) is captured in a CUDA graph -- the strongest thing a competent user of the
    reference's stack could do; without it the step is eager, which is what the reference does."""
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    rank, local, world = common.dist_env()
    torch.cuda.set_device(local)
    common.quiet_nccl()
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from tf_yarn_b200.models.mnist_cnn import TorchMnistCnn
    torch.manual_seed(1234)
    net = TorchMnistCnn().cuda().to(memory_format=torch.channels_last)
    params = [p for p in net.parameters()]
    opt = torch.optim.Adadelta(params, lr=1.0 * world, rho=0.95, eps=1e-7, capturable=args.graph)
    n_total = sum(p.numel() for p in params)
    fusion = torch.zeros(n_total, dtype=torch.bfloat16, device="cuda")   # Horovod fusion buffer
    x_host, y_host = make_pool(seed=100 + rank, nhwc=False)
    x_host, y_host = x_host.pin_memory(), y_host.pin_memory()
    B = PER_GPU_BATCH
    steps = args.steps
    repeats = common.pick_repeats(steps, args.repeats)
    for p in params:
        p.grad = torch.zeros_like(p)
    views, o = [], 0
    for p in params:
        views.append(fusion[o:o + p.numel()].view_as(p))
        o += p.numel()
    grads = [p.grad for p in params]
    loss_buf = torch.zeros((), device="cuda")

    def step(xb, yb):
        opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(xb)
        loss = F.nll_loss(out.float(), yb)
        loss.backward()
        if world > 1:
            torch._foreach_copy_(views, grads)     # pack (Horovod tensor fusion), bf16 on the wire
            dist.all_reduce(fusion)
            torch._foreach_copy_(grads, views)     # unpack + cast
            torch._foreach_mul_(grads, 1.0 / world)
        opt.step()
        loss_buf.copy_(loss.detach())
        return loss

    warm = max(3, args.warmup)
    x_dev, y_dev = x_host.cuda(), y_host.cuda()
    sx, sy = x_dev[:B].clone(), y_dev[:B].clone()
    state = {"b": 0}
    graph = None
    if args.graph:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                step(sx, sy)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step(sx, sy)

    def run(n):
        b = state["b"]
        for _ in range(n):
            xb, yb = x_dev[b * B:(b + 1) * B], y_dev[b * B:(b + 1) * B]
            if graph is not None:
                sx.copy_(xb, non_blocking=True)
                sy.copy_(yb, non_blocking=True)
                graph.replay()
            else:
                step(xb, yb)
            b = (b + 1) % POOL_BATCHES
        state["b"] = b

    sampler = common.ClockSampler(local)
    sampler.start()
    run(warm)
    region_ms = common.timed_regions(world, steps, repeats, run, None, None, sampler)
    clocks = sampler.stop()
    ms_per_step = common.median(region_ms) / steps

    # end to end: H2D from pinned memory + loss read every step
    last = {"loss": 0.0}

    def e2e_region():
        b = state["b"]
        for _ in range(steps):
            xb = x_host[b * B:(b + 1) * B].cuda(non_blocking=True)
            yb = y_host[b * B:(b + 1) * B].cuda(non_blocking=True)
            if graph is not None:
                sx.copy_(xb, non_blocking=True)
                sy.copy_(yb, non_blocking=True)
                graph.replay()
                last["loss"] = loss_buf.item()
            else:
                last["loss"] = step(xb, yb).item()
            b = (b + 1) % POOL_BATCHES
        state["b"] = b

    e2e_region()
    e2e_ms = common.wall_regions(world, repeats, e2e_region)
    e2e_ms_per_step = common.median(e2e_ms) / steps
    flat = torch.cat([p.detach().reshape(-1) for p in params])
    in_sync = common.all_ranks_equal(common.tensor_checksum(flat), world)
    if rank == 0:
        out = base_record(world, steps, warm, repeats, ms_per_step, "standin", clocks, {
            "model": "torch MNIST-CNN, autocast bf16, NCCL all-reduce of a fused bf16 buffer + torch.optim.Adadelta "
                     "(stock-PyTorch rendition of the reference's Horovod path)" + (", CUDA-graph captured"
                                                                                     if args.graph else ", eager"),
            "cuda_graph": bool(args.graph)})
        out["e2e"] = {"value": world * B / (e2e_ms_per_step * 1e-3), "unit": "samples/s",
                      "h2d_bytes_per_step": B * (784 * 4 + 8), "d2h_bytes_per_step": 4, "steps": steps,
                      "repeats": repeats, "ms_per_step": e2e_ms_per_step, "final_loss": last["loss"]}
        out["gpu_launches"] = 0
        out["params_in_sync"] = in_sync
        common.emit(out)
    if world > 1:
        if args.graph:
            # tearing an NCCL communicator down after it was captured in a CUDA graph hangs (observed: the
            # process sits in destroy_process_group until the launcher's timeout): leave without the teardown
            dist.barrier()
            torch.cuda.synchronize()
            sys.stdout.flush()
            os._exit(0)
        dist.destroy_process_group()
    return 0
