"""Task program of ``tf_yarn_b200.distributed``: run the user's ``fn(local_rank)``.

Parity with the reference task (reference: tf_yarn/distributed/task.py:28-94)
plus what it lacks: lifecycle events (init/start/stop + timers, so ``Metrics``
is populated), collision-free global ranks for mixed roles, a GPU index per
local process and failure propagation from child processes.
"""
from __future__ import annotations

import logging
import os
import sys
import traceback
from typing import List, NamedTuple, Optional

import cloudpickle

from tf_yarn_b200 import _task_commons, event
from tf_yarn_b200._task_commons import (TaskClient, _get_cluster_tasks, catchtime, choose_master,
                                        get_pickled_experiment, get_task_key, rank_table, setup_logging)

_logger = logging.getLogger(__name__)


class TaskParameters(NamedTuple):
    task_type: str
    task_id: int            # global rank (name kept from the reference)
    world_size: int
    master_address: str
    master_port: int
    n_workers_per_executor: int = 1
    local_rank: int = 0
    device: Optional[int] = None   # H100 index assigned by the launcher (None on CPU)


def _gpu_for(local_rank: int) -> Optional[int]:
    ids = [int(x) for x in os.environ.get("TFY_GPU_IDS", "").split(",") if x.strip() != ""]
    if not ids:
        return None
    return ids[local_rank % len(ids)]


def get_task(local_rank: int = 0) -> TaskParameters:
    """Who am I: global rank, world size, master address (rendezvous through the KV store)."""
    task_key = get_task_key()
    client = TaskClient.from_current()
    cluster_tasks = _get_cluster_tasks(client)
    trainers = tuple(t for t in ("chief", "worker") if any(c.type == t for c in cluster_tasks))
    table = rank_table(cluster_tasks, roles=trainers)
    rank = table[(task_key.type, task_key.id, local_rank)]
    n_local = [t.nb_proc for t in cluster_tasks if (t.type, t.id) == (task_key.type, task_key.id)][0]
    addr, port = choose_master(client, rank)
    params = TaskParameters(task_key.type, rank, len(table), addr, port, n_local, local_rank, _gpu_for(local_rank))
    _logger.info("task %s local_rank=%d -> %s", task_key.to_kv_str(), local_rank, params)
    return params


def _child_main(pickled_fn: bytes, local_rank: int, err_path: str) -> None:
    try:
        cloudpickle.loads(pickled_fn)(local_rank)
    except BaseException:
        with open(err_path, "w") as f:
            f.write(traceback.format_exc())
        raise


def parallel_run(n_workers: int, pickled_fn: bytes) -> None:
    """One spawned process per local rank; raises if any of them fails."""
    import tempfile

    from torch import multiprocessing as mp
    ctx = mp.get_context("spawn")
    tmp = tempfile.mkdtemp(prefix="tfy_dist_")
    procs = []
    for local_rank in range(n_workers):
        err = os.path.join(tmp, f"err_{local_rank}")
        p = ctx.Process(target=_child_main, args=(pickled_fn, local_rank, err))
        p.start()
        procs.append((p, err))
    failures: List[str] = []
    for local_rank, (p, err) in enumerate(procs):
        p.join()
        if p.exitcode != 0:
            tb = open(err).read() if os.path.exists(err) else f"exit code {p.exitcode}"
            failures.append(f"local rank {local_rank}:\n{tb}")
    if failures:
        raise RuntimeError("distributed task process(es) failed:\n" + "\n".join(failures))


def main() -> None:
    setup_logging()
    _logger.info("Python %s", sys.version)
    client = TaskClient.from_current()
    task_key = get_task_key()
    task = task_key.to_kv_str()
    event.init_event(client, task, "127.0.0.1:0")
    _task_commons._setup_container_logs(client)
    error: Optional[BaseException] = None
    try:
        with catchtime("fetching experiment function"):
            pickled = get_pickled_experiment(client)
        cluster_tasks = _get_cluster_tasks(client)
        n_local = [t.nb_proc for t in cluster_tasks if (t.type, t.id) == (task_key.type, task_key.id)]
        n_local = n_local[0] if n_local else 1
        event.start_event(client, task)
        event.broadcast_train_eval_start_timer(client, task)
        if n_local > 1:
            parallel_run(n_local, pickled)
        else:
            cloudpickle.loads(pickled)(0)
        event.broadcast_train_eval_stop_timer(client, task)
    except BaseException as exc:  # noqa: BLE001
        error = exc
    event.stop_event(client, task, error)
    event.broadcast_container_stop_time(client, task)
    if error is not None:
        raise error


if __name__ == "__main__":
    main()
