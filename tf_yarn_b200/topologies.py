"""Task topologies: which roles a job has and what each instance gets.

API parity with the reference (reference: tf_yarn/topologies.py:7-160) --
``TaskSpec``, ``NodeLabel``, ``ContainerKey``, ``ContainerTask``,
``single_server_topology``, ``ps_strategy_topology`` -- re-targeted at ONE
8xH100 NVSwitch box: a ``NodeLabel.GPU`` task instance is pinned to
``nb_proc_per_worker`` H100s by the local launcher instead of being a YARN
container on a ``gpu``-labelled node.
"""
from __future__ import annotations

import logging
import re
from enum import Enum
from typing import Dict, NamedTuple, Optional, Union

logger = logging.getLogger(__name__)

# container caps of the reference (MiB / cores); kept so existing configs validate identically
MAX_MEMORY_CONTAINER = 48 * 2 ** 10
MAX_VCORES_CONTAINER = 48
ALL_TASK_TYPES = {"chief", "worker", "ps", "evaluator", "tensorboard"}
# roles that are side processes, never part of the training cluster (barriers, world size)
SIDE_TASK_TYPES = ("evaluator", "tensorboard")

_MEM_UNITS = {
    "": 1, "b": 1,
    "k": 10 ** 3, "kb": 10 ** 3, "m": 10 ** 6, "mb": 10 ** 6, "g": 10 ** 9, "gb": 10 ** 9, "t": 10 ** 12,
    "tb": 10 ** 12,
    "kib": 2 ** 10, "mib": 2 ** 20, "gib": 2 ** 30, "tib": 2 ** 40,
}


def parse_memory(value: Union[int, str]) -> int:
    """Memory in MiB from an int (MiB) or a string such as ``"2 GiB"`` / ``"512 MiB"``.

    Strings are rounded up to the next MiB, like skein's ``Resources``.
    """
    if isinstance(value, bool):
        raise TypeError("memory must be an int (MiB) or a string like '2 GiB'")
    if isinstance(value, int):
        if value < 0:
            raise ValueError("memory must be >= 0")
        return value
    if isinstance(value, float):
        return int(-(-value // 1))
    m = re.fullmatch(r"\s*([0-9]*\.?[0-9]+)\s*([a-zA-Z]*)\s*", str(value))
    if not m or m.group(2).lower() not in _MEM_UNITS:
        raise ValueError(f"cannot parse memory specification {value!r}")
    nbytes = float(m.group(1)) * _MEM_UNITS[m.group(2).lower()]
    if m.group(2) == "":
        return int(float(m.group(1)))
    return int(-(-nbytes // 2 ** 20))


class NodeLabel(Enum):
    """Where a task instance runs: host CPU only, or pinned to H100 GPU(s)."""
    CPU = ""
    GPU = "gpu"


class ContainerKey(NamedTuple):
    type: str
    id: int

    def to_kv_str(self) -> str:
        return f"{self.type}:{self.id}"

    @staticmethod
    def from_kv_str(kv_str: str) -> Optional["ContainerKey"]:
        try:
            task_type, task_id = kv_str.rsplit(":", 1)
            return ContainerKey(task_type, int(task_id))
        except ValueError:
            logger.warning("%r is not a task key (expected '<type>:<id>')", kv_str)
            return None


class ContainerTask(NamedTuple):
    type: str
    id: int
    nb_proc: int

    def to_container_key(self) -> ContainerKey:
        return ContainerKey(self.type, self.id)

    def to_kv_str(self) -> str:
        return f"{self.type}:{self.id}:{self.nb_proc}"


class TaskSpec:
    """Resources of one role.

    memory : MiB as int, or a string like ``"2 GiB"``; vcores : host cores;
    instances : number of task instances of this role; nb_proc_per_worker :
    processes (== GPUs for ``NodeLabel.GPU``) per instance.
    """
    __slots__ = ("_memory", "_vcores", "instances", "label", "nb_proc_per_worker",
                 "tb_termination_timeout_seconds", "tb_model_dir", "tb_extra_args")

    def __init__(self, memory: Union[int, str], vcores: int, instances: int = 1, nb_proc_per_worker: int = 1,
                 label: NodeLabel = NodeLabel.CPU, tb_termination_timeout_seconds: int = -1,
                 tb_model_dir: Optional[str] = None, tb_extra_args: Optional[str] = None):
        self._memory = parse_memory(memory)
        self._vcores = int(vcores)
        self.instances = instances
        self.nb_proc_per_worker = nb_proc_per_worker
        self.label = label
        self.tb_termination_timeout_seconds = tb_termination_timeout_seconds
        self.tb_model_dir = tb_model_dir
        self.tb_extra_args = tb_extra_args

    @property
    def memory(self) -> int:
        return self._memory

    @memory.setter
    def memory(self, value: Union[int, str]) -> None:
        self._memory = parse_memory(value)

    @property
    def vcores(self) -> int:
        return self._vcores

    @vcores.setter
    def vcores(self, value: int) -> None:
        self._vcores = int(value)

    def __repr__(self) -> str:
        return (f"TaskSpec(memory={self.memory}, vcores={self.vcores}, instances={self.instances}, "
                f"nb_proc_per_worker={self.nb_proc_per_worker}, label={self.label})")


def _check_general_topology(task_specs: Dict[str, TaskSpec]) -> None:
    unknown = set(task_specs) - ALL_TASK_TYPES
    if unknown:
        raise ValueError(f"task_specs.keys() must be a subset of: {ALL_TASK_TYPES} (got {sorted(unknown)})")
    if "chief" not in task_specs or task_specs["chief"].instances != 1:
        raise ValueError("exactly one 'chief' task is required")
    for task_type, spec in task_specs.items():
        if spec.memory > MAX_MEMORY_CONTAINER:
            raise ValueError(f"{task_type}: Can not demand more memory than {MAX_MEMORY_CONTAINER} MiB per task")
        if spec.vcores > MAX_VCORES_CONTAINER:
            raise ValueError(f"{task_type}: Can not demand more vcores than {MAX_VCORES_CONTAINER} per task")
        if spec.nb_proc_per_worker > spec.vcores:
            raise ValueError(f"{task_type}: Can not run more processes per instance than vcores ({spec.vcores})")


def _check_ps_topology(task_specs: Dict[str, TaskSpec]) -> None:
    _check_general_topology(task_specs)
    for side in SIDE_TASK_TYPES:
        if side in task_specs and (task_specs[side].instances > 1 or task_specs[side].nb_proc_per_worker > 1):
            raise ValueError(f"no more than one '{side}' task is allowed")
    if "ps" not in task_specs or not task_specs["ps"].instances:
        raise ValueError("task_specs must contain at least a single 'ps' task for multi-worker training")


def single_server_topology(memory: Union[int, str] = MAX_MEMORY_CONTAINER,
                           vcores: int = MAX_VCORES_CONTAINER) -> Dict[str, TaskSpec]:
    topology = {
        "chief": TaskSpec(memory=memory, vcores=vcores),
        "evaluator": TaskSpec(memory=memory, vcores=vcores),
        "tensorboard": TaskSpec(memory=memory, vcores=vcores),
    }
    _check_general_topology(topology)
    return topology


def ps_strategy_topology(nb_workers: int = 2, nb_ps: int = 1, memory: Union[int, str] = MAX_MEMORY_CONTAINER,
                         vcores: int = MAX_VCORES_CONTAINER) -> Dict[str, TaskSpec]:
    """chief + workers + ps (+ evaluator + tensorboard): the asynchronous parameter-server layout."""
    topology = {
        "chief": TaskSpec(memory=memory, vcores=vcores),
        "evaluator": TaskSpec(memory=memory, vcores=vcores),
        "worker": TaskSpec(memory=memory, vcores=vcores, instances=nb_workers),
        "ps": TaskSpec(memory=memory, vcores=vcores, instances=nb_ps),
        "tensorboard": TaskSpec(memory=memory, vcores=vcores, instances=1),
    }
    _check_ps_topology(topology)
    return topology


def allreduce_topology(nb_workers: int = 8, memory: Union[int, str] = MAX_MEMORY_CONTAINER,
                       vcores: int = MAX_VCORES_CONTAINER, label: NodeLabel = NodeLabel.GPU,
                       with_evaluator: bool = True, with_tensorboard: bool = False) -> Dict[str, TaskSpec]:
    """chief + (nb_workers - 1) workers, one H100 each: the synchronous all-reduce layout
    (the reference builds this by hand in native_keras_with_gloo_example.py:98-104)."""
    if nb_workers < 1:
        raise ValueError("nb_workers must be >= 1")
    topology = {"chief": TaskSpec(memory=memory, vcores=vcores, label=label)}
    if nb_workers > 1:
        topology["worker"] = TaskSpec(memory=memory, vcores=vcores, instances=nb_workers - 1, label=label)
    if with_evaluator:
        topology["evaluator"] = TaskSpec(memory=memory, vcores=vcores)
    if with_tensorboard:
        topology["tensorboard"] = TaskSpec(memory=memory, vcores=vcores)
    _check_general_topology(topology)
    return topology
