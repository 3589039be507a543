"""Cluster bootstrap of the parameter-server task (reference: tf_yarn/tensorflow/cluster.py:14-71).

Every cluster task publishes ``<task>/init = "host:port"`` and waits for all the others
(the INIT barrier); the aggregated addresses become ``TF_CONFIG``, from which the Estimator
facade derives its role.  There is no gRPC server to start: the ps data plane is direct
memory access (shared memory on CPU, peer HBM over NVLink on H100), so ``start_tf_server``
only records the role.
"""
from __future__ import annotations

import json
import logging
from typing import Dict, List, Optional, Tuple

from tf_yarn_b200 import _internal, event
from tf_yarn_b200._task_commons import get_task_key
from tf_yarn_b200.topologies import ContainerTask

logger = logging.getLogger(__name__)


def aggregate_spec(client, all_tasks: List[ContainerTask]) -> Dict[str, List[str]]:
    """Wait for ``<type>:<id>/init`` of every cluster task -> ``{"worker": [addr, ...], "ps": [...]}``."""
    spec: Dict[str, List[str]] = {}
    for task in sorted(all_tasks, key=lambda t: (t.type, t.id)):
        addr = event.wait(client, f"{task.to_container_key().to_kv_str()}/init")
        spec.setdefault(task.type, []).append(addr)
    return spec


def start_cluster(host_port: Tuple[str, int], client, all_tasks: List[ContainerTask]) -> Dict[str, List[str]]:
    """Publish this task's address, then aggregate everybody's (the init barrier)."""
    host, port = host_port
    event.init_event(client, get_task_key().to_kv_str(), f"{host}:{port}")
    return aggregate_spec(client, all_tasks)


def setup_tf_config(cluster_spec: Dict[str, List[str]]) -> None:
    """Exclusively set ``TF_CONFIG`` for this task."""
    task_type, task_id = get_task_key()
    cfg = {"cluster": cluster_spec,
           "environment": "google" if _is_fake_google_env(task_type) else "",
           "task": {"type": task_type, "index": task_id}}
    _internal.xset_environ(TF_CONFIG=json.dumps(cfg))


def start_tf_server(cluster_spec: Dict[str, List[str]], session_config=None) -> Optional[dict]:
    """chief / worker: returns a descriptor of the (virtual) server; ps / evaluator: None."""
    task_type, task_id = get_task_key()
    if not _is_fake_google_env(task_type):
        return None
    server = {"job_name": task_type, "task_index": task_id, "cluster": cluster_spec, "config": session_config}
    logger.info("role %s:%d joined cluster %s", task_type, task_id, {k: len(v) for k, v in cluster_spec.items()})
    return server


def _is_fake_google_env(task_type: str) -> bool:
    return task_type not in ("evaluator", "ps")
