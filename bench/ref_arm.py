"""`bench.py --impl reference`: the UNMODIFIED reference (oracle/_ref/tf_yarn) on the headline config.

What runs is the reference's own PyTorch worker, `tf_yarn.pytorch.tasks.worker._train`
(reference: tf_yarn/pytorch/tasks/worker.py:94-122): it fetches the cloudpickled experiment function from the
application KV store, elects the master through the KV store (`choose_master`), calls
`dist.init_process_group("nccl")`, wraps the model in `torch.nn.parallel.DistributedDataParallel` with the
`DistributedDataParallelArgs` defaults (25 MB buckets), builds the `DataLoader` with a `DistributedSampler` and
calls the user's `main_fn`.  This file only plays the two roles the reference expects from its surroundings:

* the cluster side: one process per GPU (torchrun), a KV store (this repo's C++ KV server hosted by rank 0, reached
  through `bench/shims/skein`) holding the experiment, SKEIN_CONTAINER_ID in the environment;
* the user side: a `PytorchExperiment` of the same MNIST-CNN (the network of the reference's own example,
  tf_yarn/examples/pytorch/pytorch_distributed_example.py:44-67), 128 samples per GPU, bf16 autocast,
  Adadelta(1.0 * world), the same synthetic pool, with the timing loops inside `main_fn`.

Nothing of tf_yarn_b200's models, kernels or engines is imported here (only the KV client, control plane).
"""
from __future__ import annotations

import datetime
import os
import socket
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
SHIMS = os.path.join(ROOT, "bench", "shims")


def _unavailable(why: str) -> int:
    import json
    if int(os.environ.get("RANK", 0)) == 0:
        print(json.dumps({"impl": "reference", "unavailable": why}), flush=True)
    return 0


def _ensure_installed() -> str:
    """oracle/_ref is built by ``python __graft_entry__.py`` (oracle/build_ref.py) when the reference sources exist."""
    if os.path.isdir(os.path.join(REF_DIR, "tf_yarn")):
        return ""
    return "oracle/_ref is not built (the original project's sources were not available to build())"


# ------------------------------------------------------------------------------------------------------
# user side: the experiment (pickled by value with cloudpickle; runs inside the reference's worker)
# ------------------------------------------------------------------------------------------------------
def make_experiment_fn(steps: int, warmup: int, repeats: int, world: int, config: str = "mnist", batch: int = 0):
    def experiment_fn():
        import argparse
        import torch
        import torch.nn as nn
        import torch.nn.functional as F
        from tf_yarn.pytorch import DataLoaderArgs, DistributedDataParallelArgs, PytorchExperiment
        from bench import common, mnist, models

        class Net(nn.Module):            # reference: tf_yarn/examples/pytorch/pytorch_distributed_example.py:44-67
            def __init__(self):
                super().__init__()
                self.conv1 = nn.Conv2d(1, 32, 3, 1)
                self.conv2 = nn.Conv2d(32, 64, 3, 1)
                self.dropout1 = nn.Dropout(0.25)
                self.dropout2 = nn.Dropout(0.5)
                self.fc1 = nn.Linear(9216, 128)
                self.fc2 = nn.Linear(128, 10)

            def forward(self, x):
                x = F.relu(self.conv1(x))
                x = F.relu(self.conv2(x))
                x = F.max_pool2d(x, 2)
                x = self.dropout1(x)
                x = torch.flatten(x, 1)
                x = F.relu(self.fc1(x))
                x = self.dropout2(x)
                return F.log_softmax(self.fc2(x), dim=1)

        rank = int(os.environ.get("RANK", 0))
        if config == "mnist":
            B, NB = mnist.PER_GPU_BATCH, mnist.POOL_BATCHES
            make_net = lambda: Net().to(memory_format=torch.channels_last)                  # noqa: E731
            make_pool = lambda: mnist.make_pool(seed=100 + rank, nhwc=False)                  # noqa: E731
            make_opt = lambda ps: torch.optim.Adadelta(ps, lr=1.0 * world, rho=0.95, eps=1e-7)  # noqa: E731
            loss_of = lambda out, yb: F.nll_loss(out.float(), yb)                             # noqa: E731
            h2d = B * (784 * 4 + 8)
        else:                                                                               # resnet50 (config 4)
            import torchvision
            B, NB = batch or models.RESNET_BATCH, models.RESNET_POOL
            make_net = lambda: torchvision.models.resnet50().to(memory_format=torch.channels_last)  # noqa: E731
            make_pool = lambda: models.resnet_pool(rank, pinned=False)                        # noqa: E731
            make_opt = lambda ps: torch.optim.SGD(ps, lr=0.01, momentum=0.9)                   # noqa: E731
            loss_of = lambda out, yb: F.cross_entropy(out.float(), yb)                        # noqa: E731
            h2d = B * (3 * 224 * 224 * 4 + 8)

        class BatchPool(torch.utils.data.Dataset):
            """Pre-batched, pre-pinned pool: item i is batch i (the friendliest input the DataLoader can get:
            no per-sample collation, `pin_memory` finds the tensors already pinned)."""

            def __init__(self):
                x, y = make_pool()
                self.x, self.y = x.pin_memory(), y.pin_memory()

            def __len__(self):
                return NB * world          # DistributedSampler hands every rank NB of them

            def __getitem__(self, i):
                b = i % NB
                return self.x[b * B:(b + 1) * B], self.y[b * B:(b + 1) * B]

        def main_fn(ddp_model, trainloader, device, rank, tb_writer=None):
            torch.cuda.set_device(device)
            dev = torch.device(device)
            params = [p for p in ddp_model.parameters()]
            opt = make_opt(params)
            ds = trainloader.dataset
            local = dev.index or 0
            sampler = common.ClockSampler(local)
            sampler.start()

            def step(xb, yb):
                opt.zero_grad(set_to_none=True)
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = ddp_model(xb)
                loss = loss_of(out, yb)
                loss.backward()            # DDP all-reduces the 25 MB buckets (NCCL) during backward
                opt.step()
                return loss

            # device-timed: the pool resident in HBM (as in the `ours` arm)
            x_dev, y_dev = ds.x.to(dev), ds.y.to(dev)
            if x_dev.dim() == 4:
                x_dev = x_dev.contiguous(memory_format=torch.channels_last)
            state = {"b": 0}

            def run(n):
                b = state["b"]
                for _ in range(n):
                    step(x_dev[b * B:(b + 1) * B], y_dev[b * B:(b + 1) * B])
                    b = (b + 1) % NB
                state["b"] = b

            warm = max(3, warmup)
            run(warm)
            region_ms = common.timed_regions(world, steps, repeats, run, None, None, sampler)
            clocks = sampler.stop()
            ms_per_step = common.median(region_ms) / steps
            del x_dev, y_dev

            # end to end: the reference's DataLoader (DistributedSampler, pinned batches) -> H2D -> step -> loss.item()
            it = {"it": iter(trainloader)}
            last = {"loss": float("nan")}

            def next_batch():
                try:
                    return next(it["it"])
                except StopIteration:
                    it["it"] = iter(trainloader)
                    return next(it["it"])

            def e2e_region():
                for _ in range(steps):
                    xb, yb = next_batch()
                    xb = xb.to(dev, non_blocking=True)
                    if xb.dim() == 4 and config != "mnist":
                        xb = xb.contiguous(memory_format=torch.channels_last)
                    yb = yb.to(dev, non_blocking=True)
                    last["loss"] = step(xb, yb).item()

            e2e_region()
            e2e_ms = common.wall_regions(world, repeats, e2e_region)
            e2e_ms_per_step = common.median(e2e_ms) / steps
            flat = torch.cat([p.detach().reshape(-1) for p in params])
            in_sync = common.all_ranks_equal(common.tensor_checksum(flat), world)
            if rank == 0:
                if config == "mnist":
                    out = mnist.base_record(world, steps, warm, repeats, ms_per_step, "reference", clocks, {
                        "model": "the reference's PyTorch worker (tf_yarn.pytorch.tasks.worker._train, unmodified): "
                                 "torch DistributedDataParallel (bucket_cap_mb=25) over NCCL, MNIST-CNN (1,199,882 "
                                 "params), autocast bf16, torch.optim.Adadelta(1.0*size), eager",
                        "same_config": True, "cuda_graph": False})
                    unit = "samples/s"
                else:
                    ns = argparse.Namespace(config="resnet50", steps=steps)
                    out = models._record(
                        "images/sec, PytorchExperiment ResNet-50 DistributedDataParallel (whole job)", "images/s", world,
                        ns, warm, repeats, ms_per_step, B, "reference", clocks,
                        "the reference's PyTorch worker (tf_yarn.pytorch.tasks.worker._train, unmodified): torchvision "
                        "ResNet-50 under torch DistributedDataParallel (bucket_cap_mb=25) over NCCL, autocast bf16, "
                        "torch.optim.SGD(momentum 0.9), eager", {"same_config": True})
                    unit = "images/s"
                out["e2e"] = {"value": world * B / (e2e_ms_per_step * 1e-3), "unit": unit,
                              "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "steps": steps,
                              "repeats": repeats, "ms_per_step": e2e_ms_per_step, "final_loss": last["loss"]}
                out["gpu_launches"] = 0
                out["params_in_sync"] = in_sync
                out["reference_path"] = "oracle/_ref/tf_yarn/pytorch/tasks/worker.py::_train"
                common.emit(out)

        return PytorchExperiment(
            model=make_net(),
            main_fn=main_fn,
            train_dataset=BatchPool(),
            # batch_size=None: the dataset yields whole batches; prefetch_factor must be None with num_workers=0
            dataloader_args=DataLoaderArgs(batch_size=None, num_workers=0, pin_memory=True, drop_last=False,
                                           prefetch_factor=None, shuffle=False),
            ddp_args=DistributedDataParallelArgs())

    return experiment_fn


# ------------------------------------------------------------------------------------------------------
# cluster side
# ------------------------------------------------------------------------------------------------------
def _publish_kv_address(rank: int, world: int):
    """Rank 0 hosts the KV store; the others learn its address through torchrun's agent store."""
    from tf_yarn_b200.kv import start_server      # control plane only
    key = "tfy_ref_kv_addr"
    if world == 1:
        srv = start_server()
        return srv, srv.address
    from torch.distributed import TCPStore
    store = TCPStore(os.environ["MASTER_ADDR"], int(os.environ["MASTER_PORT"]), world_size=None, is_master=False,
                     timeout=datetime.timedelta(seconds=300))
    if rank == 0:
        srv = start_server()
        store.set(key, srv.address)
        return srv, srv.address
    return None, store.get(key).decode()


def run_reference(args) -> int:
    rank, local, world = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("LOCAL_RANK", 0), ("WORLD_SIZE", 1)))
    why = _ensure_installed()
    if why:
        return _unavailable(why)
    sys.path[:0] = [SHIMS, REF_DIR]
    try:
        import torch
        if not torch.cuda.is_available():
            return _unavailable("no CUDA device: the reference's worker wraps the model in DistributedDataParallel "
                                "with device_ids=[gpu] and needs NCCL")
        import cloudpickle
        import tf_yarn  # noqa: F401
        from tf_yarn import constants
        from tf_yarn.pytorch.tasks import worker as ref_worker
    except Exception as exc:  # noqa: BLE001
        return _unavailable(f"cannot import the reference: {type(exc).__name__}: {exc}")

    srv, addr = _publish_kv_address(rank, world)
    os.environ["TFY_REF_KV_ADDR"] = addr
    # environment the reference's worker expects from a skein container
    os.environ["SKEIN_CONTAINER_ID"] = f"worker_{rank}"
    os.environ.pop("TORCHELASTIC_USE_AGENT_STORE", None)   # the worker elects its own master through the KV store
    os.environ.setdefault("NCCL_DEBUG_FILE", os.path.join("/tmp", "tfy_ref_nccl_%h_%p.log"))   # it sets NCCL_DEBUG=INFO
    try:
        socket.gethostbyname(socket.getfqdn())
    except OSError:
        # the container hostname does not resolve on these boxes; choose_master() publishes socket.getfqdn()
        socket.getfqdn = lambda name="": "127.0.0.1"

    import skein
    client = skein.ApplicationClient.from_current()
    if rank == 0:
        from bench.common import pick_repeats
        cfg = getattr(args, "config", "mnist")
        repeats_n = pick_repeats(args.steps, args.repeats or (3 if cfg != "mnist" else 0))
        fn = make_experiment_fn(args.steps, args.warmup, repeats_n, world, cfg, getattr(args, "batch", 0))
        client.kv[constants.KV_EXPERIMENT_FN] = cloudpickle.dumps(fn)
    torch.cuda.set_device(local)
    ref_worker._train(local, rank, world, "nccl")
    if world > 1:
        # keep the KV server up until every rank is done with it
        client.kv[f"tfy_ref_done_{rank}"] = b"1"
        if rank == 0:
            for r in range(world):
                client.kv.wait(f"tfy_ref_done_{r}")
    if srv is not None:
        srv.stop()
    return 0
