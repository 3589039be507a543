"""PyTorch worker task: data-parallel training of a ``PytorchExperiment``.

Lifecycle parity with the reference worker (reference:
tf_yarn/pytorch/tasks/worker.py:94-214): rendezvous on a master chosen through
the KV store, ``init_process_group``, wrap the model for data-parallel
training, build the rank's dataloader, call the user's ``main_fn(model,
trainloader, device, rank, tb_writer)``, collect the TensorBoard event files.

H100 specifics:

* one process per GPU; the GPU index comes from the launcher's placement
  (``TFY_GPU_IDS``), not from ``local_index % n_gpus``;
* the gradient all-reduce is NOT NCCL: the model is wrapped in
  :class:`tf_yarn_b200.parallel.ddp.DistributedDataParallel`, whose buckets are
  reduced by the NVLS / P2P kernels over the symmetric arena.  The NCCL process
  group is still created because user code may call ``torch.distributed``
  collectives (e.g. ``dist.barrier()`` in the reference's example);
* CPU-only boxes (CI, the plumbing configuration) use gloo + torch DDP instead
  of raising "Multi-CPU training is not supported yet";
* lifecycle events are published (the reference's worker posts none, leaving
  ``Metrics`` empty) and a failing child fails the task.
"""
from __future__ import annotations

import logging
import os
import sys
import tempfile
import traceback
from typing import List, Optional

import torch
import torch.distributed as dist

from tf_yarn_b200 import _task_commons, event
from tf_yarn_b200._task_commons import (TaskClient, _get_cluster_tasks, _get_experiment, choose_master,
                                        get_task_key, rank_table, setup_logging)
from tf_yarn_b200.pytorch.experiment import DataLoaderArgs, PytorchExperiment
from tf_yarn_b200.utils import fs as filesystem

_logger = logging.getLogger(__name__)

MASTER_ADDR = "MASTER_ADDR"
MASTER_PORT = "MASTER_PORT"


def _log_sys_info() -> None:
    _logger.info("Python %s", sys.version)
    _logger.info("Pytorch %s (cuda available: %s)", torch.__version__, torch.cuda.is_available())


def _is_webdataset(dataset) -> bool:
    try:
        import webdataset as wds
    except ImportError:
        return False
    return isinstance(dataset, (wds.WebDataset, wds.DataPipeline))


def _create_dataloader(dataset, dataloader_args: DataLoaderArgs):
    """The rank's dataloader: DistributedSampler for map-style datasets, none for iterable ones."""
    if _is_webdataset(dataset):
        import webdataset as wds
        return wds.WebLoader(
            dataset, batch_size=dataloader_args.batch_size, num_workers=dataloader_args.num_workers,
            pin_memory=dataloader_args.pin_memory, drop_last=dataloader_args.drop_last,
            timeout=dataloader_args.timeout, prefetch_factor=dataloader_args.prefetch_factor,
            persistent_workers=dataloader_args.persistent_workers, shuffle=dataloader_args.shuffle)
    iterable = isinstance(dataset, torch.utils.data.IterableDataset)
    sampler = None
    if not iterable and dist.is_available() and dist.is_initialized():
        sampler = torch.utils.data.distributed.DistributedSampler(dataset, shuffle=dataloader_args.shuffle)
    if not dataloader_args.drop_last:
        _logger.error(
            "/!\\ Not dropping the last batch could result in a smaller batch size which could block your "
            "distributed training when aggregating tensors with allreduce/allgather. We strongly encourage "
            "setting DataLoaderArgs.drop_last to True")
    kwargs = dict(batch_size=dataloader_args.batch_size, num_workers=dataloader_args.num_workers,
                  pin_memory=dataloader_args.pin_memory, drop_last=dataloader_args.drop_last,
                  timeout=dataloader_args.timeout, collate_fn=dataloader_args.collate_fn)
    if dataloader_args.num_workers > 0:
        kwargs["prefetch_factor"] = dataloader_args.prefetch_factor
        kwargs["persistent_workers"] = dataloader_args.persistent_workers
    # torch forbids sampler + shuffle=True: the sampler already shuffles (the reference passes both)
    kwargs["shuffle"] = dataloader_args.shuffle if (sampler is None and not iterable) else False
    return torch.utils.data.DataLoader(dataset, sampler=sampler, **kwargs)


def _setup_master(client, rank: int) -> None:
    addr, port = choose_master(client, rank)
    os.environ[MASTER_ADDR] = addr
    os.environ[MASTER_PORT] = str(port)
    _logger.info("master: %s:%s", addr, port)


def _assigned_gpus() -> List[int]:
    return [int(x) for x in os.environ.get("TFY_GPU_IDS", "").split(",") if x.strip() != ""]


def _get_device(worker_id: int) -> Optional[int]:
    """H100 index for local process ``worker_id``; None means CPU."""
    if not torch.cuda.is_available():
        return None
    ids = _assigned_gpus()
    if ids:
        return ids[worker_id % len(ids)]
    return worker_id % torch.cuda.device_count()


def _get_collective_ops_backend(n_workers_per_executor: int) -> str:
    """nccl when every local process owns a GPU, gloo when GPUs are oversubscribed or absent."""
    if not torch.cuda.is_available():
        return "gloo"
    n_gpus = len(_assigned_gpus()) or torch.cuda.device_count()
    return "nccl" if n_workers_per_executor <= n_gpus else "gloo"


def _upload_tensorboard(local_dir: str, dest_dir: str) -> None:
    resolved_fs, _ = filesystem.resolve_filesystem_and_path(dest_dir)
    if not resolved_fs.exists(dest_dir):
        resolved_fs.mkdir(dest_dir)
    for name in os.listdir(local_dir):
        resolved_fs.put(os.path.join(local_dir, name), os.path.join(dest_dir, name))


_upload_tensorboard_on_hdfs = _upload_tensorboard


def _train(device: Optional[int], rank: int, world_size: int, collective_ops_backend: str,
           err_path: Optional[str] = None) -> None:
    try:
        _train_impl(device, rank, world_size, collective_ops_backend)
    except BaseException:
        if err_path:
            with open(err_path, "w") as f:
                f.write(traceback.format_exc())
        raise


def _train_impl(device: Optional[int], rank: int, world_size: int, collective_ops_backend: str) -> None:
    from torch.utils.tensorboard import SummaryWriter
    _logger.info("[%d] device: %s; rank: %d/%d; backend: %s", os.getpid(), device, rank, world_size,
                 collective_ops_backend)
    client = TaskClient.from_current()
    _setup_master(client, rank)
    os.environ["TFY_RANK"], os.environ["TFY_WORLD_SIZE"] = str(rank), str(world_size)
    on_gpu = device is not None and collective_ops_backend == "nccl"
    if device is not None:
        torch.cuda.set_device(device)
    dist.init_process_group(collective_ops_backend, rank=rank, world_size=world_size,
                            **({"device_id": torch.device(f"cuda:{device}")} if on_gpu else {}))
    try:
        experiment = _get_experiment(client)
        assert isinstance(experiment, PytorchExperiment)
        device_str = f"cuda:{device}" if device is not None else "cpu"
        model = experiment.model.to(device_str)
        ddp_kwargs = experiment.ddp_args._asdict() if experiment.ddp_args else {}
        if on_gpu:
            from tf_yarn_b200.parallel import ddp as tfy_ddp
            ddp_model = tfy_ddp.wrap_model(model, device_str, ddp_kwargs)
        elif world_size > 1:
            from torch.nn.parallel import DistributedDataParallel as TorchDDP
            ddp_model = TorchDDP(model, device_ids=[device] if device is not None else None, **ddp_kwargs)
        else:
            ddp_model = model
        trainloader = _create_dataloader(experiment.train_dataset, experiment.dataloader_args)
        with tempfile.TemporaryDirectory() as tmp:
            tb_writer = SummaryWriter(tmp)
            experiment.main_fn(ddp_model, trainloader, device_str, rank, tb_writer)
            tb_writer.flush()
            tb_writer.close()
            if experiment.tensorboard_hdfs_dir:
                _upload_tensorboard(tmp, os.path.join(experiment.tensorboard_hdfs_dir, f"worker{rank}"))
    finally:
        if on_gpu:
            from tf_yarn_b200.parallel import runtime
            torch.cuda.synchronize()
            runtime.shutdown()
        dist.destroy_process_group()
    _logger.info("Done training")


def main() -> None:
    setup_logging()
    _log_sys_info()
    task_key = get_task_key()
    task = task_key.to_kv_str()
    client = TaskClient.from_current()
    event.init_event(client, task, "127.0.0.1:0")
    _task_commons._setup_container_logs(client)
    error: Optional[BaseException] = None
    try:
        experiment = _get_experiment(client)   # fail fast (and publish start/stop) before spawning
        assert isinstance(experiment, PytorchExperiment), "experiment_fn must return a PytorchExperiment"
        del experiment
        cluster_tasks = _get_cluster_tasks(client)
        trainers = tuple(t for t in ("chief", "worker") if any(c.type == t for c in cluster_tasks))
        table = rank_table(cluster_tasks, roles=trainers)
        world_size = len(table)
        n_local = [t.nb_proc for t in cluster_tasks if (t.type, t.id) == (task_key.type, task_key.id)][0]
        _logger.info("Task %s; world_size: %d; cluster tasks: %s", task, world_size, cluster_tasks)
        event.start_event(client, task)
        event.broadcast_train_eval_start_timer(client, task)
        backend = _get_collective_ops_backend(n_local)
        if n_local > 1:
            import torch.multiprocessing as mp
            ctx = mp.get_context("spawn")
            tmp = tempfile.mkdtemp(prefix="tfy_worker_")
            procs = []
            for n in range(n_local):
                rank = table[(task_key.type, task_key.id, n)]
                err = os.path.join(tmp, f"err_{n}")
                p = ctx.Process(target=_train, args=(_get_device(n), rank, world_size, backend, err))
                _logger.info("starting process %d (rank %d) of task %s", n, rank, task)
                p.start()
                procs.append((p, err))
            failures = []
            for n, (p, err) in enumerate(procs):
                p.join()
                if p.exitcode != 0:
                    failures.append(f"local process {n}: " + (open(err).read() if os.path.exists(err)
                                                              else f"exit code {p.exitcode}"))
            if failures:
                raise RuntimeError("worker process(es) failed:\n" + "\n".join(failures))
        else:
            _train(_get_device(0), table[(task_key.type, task_key.id, 0)], world_size, backend)
        event.broadcast_train_eval_stop_timer(client, task)
    except BaseException as exc:  # noqa: BLE001
        error = exc
    if "stop" not in "".join(k for k in client.kv.keys(f"{task}/") if k.endswith("/stop")):
        event.stop_event(client, task, error)
    event.broadcast_container_stop_time(client, task)
    if error is not None:
        raise error


if __name__ == "__main__":
    main()
