"""Local application launcher: the single-box stand-in for skein + YARN.

The reference submits a ``skein.ApplicationSpec`` (one ``Service`` per task
type) to a Java ApplicationMaster that starts one YARN container per task
instance and hosts the KV store (reference: tf_yarn/client.py:179-269).  On one
8xH100 box the same contract is met by:

* one OS process (own session / process group) per task instance, started with
  the task's command line, environment and a private working directory;
* GPU placement: every ``NodeLabel.GPU`` instance is pinned to
  ``nb_proc_per_worker`` H100s, handed out round-robin (``TFY_GPU_IDS``);
* the KV rendezvous server hosted in the launcher process (``tf_yarn_b200.kv``);
* per-task log files (the "container logs");
* an application report with YARN-like ``state`` / ``final_status`` derived from
  the exit codes: any task exiting non-zero fails the application and the rest
  of the tasks are killed (``max_restarts=0`` semantics, client.py:233).
"""
from __future__ import annotations

import getpass
import logging
import os
import shutil
import signal
import subprocess
import tempfile
import time
import uuid
from typing import Dict, List, NamedTuple, Optional

from tf_yarn_b200 import kv as kvmod
from tf_yarn_b200.topologies import ContainerKey, NodeLabel

logger = logging.getLogger(__name__)

REPO_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class ServiceSpec(NamedTuple):
    """One role of the application (skein ``Service`` stand-in)."""
    script: str                     # bash script run for every instance
    instances: int
    nb_proc: int
    label: NodeLabel
    memory: int                     # MiB (accounting + exported as TFY_MEMORY_MB; no rlimit: CUDA reserves huge VA)
    vcores: int                     # CPU cores the instance is pinned to (sched affinity), see _cpu_plan
    env: Dict[str, str]
    files: Dict[str, str]           # target (relative to task workdir) -> source path


class ApplicationSpec(NamedTuple):
    services: Dict[str, ServiceSpec]
    name: str = "RunOnB200"
    queue: str = "default"
    user: str = ""


class ApplicationReport(NamedTuple):
    id: str
    name: str
    state: str                      # accepted | running | finished | failed | killed
    final_status: str               # undefined | succeeded | failed | killed
    start_time: float
    finish_time: Optional[float]
    tracking_url: str
    user: str
    queue: str


class FinalStatus:
    SUCCEEDED = "succeeded"
    FAILED = "failed"
    KILLED = "killed"
    UNDEFINED = "undefined"


class TaskProcess:
    def __init__(self, key: ContainerKey, popen: subprocess.Popen, log_path: str, gpus: List[int], workdir: str):
        self.key, self.popen, self.log_path, self.gpus, self.workdir = key, popen, log_path, gpus, workdir

    @property
    def container_id(self) -> str:
        return f"container_{self.key.type}_{self.key.id}"

    @property
    def returncode(self) -> Optional[int]:
        return self.popen.poll()


def visible_gpus() -> List[int]:
    """GPU indices the launcher may hand out."""
    env = os.environ.get("TFY_VISIBLE_GPUS")
    if env is not None:
        return [int(x) for x in env.split(",") if x.strip() != ""]
    try:
        import torch
        return list(range(torch.cuda.device_count()))
    except Exception:  # noqa: BLE001
        return []


class LocalApplication:
    """A running application: task processes + KV store (skein ``ApplicationClient`` stand-in)."""

    def __init__(self, spec: ApplicationSpec, workdir: Optional[str] = None, kill_grace_secs: float = 5.0):
        self.id = f"application_{int(time.time())}_{uuid.uuid4().hex[:6]}"
        self.spec = spec
        self.name = spec.name
        self.start_time = time.time()
        self.finish_time: Optional[float] = None
        self._final_status = FinalStatus.UNDEFINED
        self._own_workdir = workdir is None
        self.workdir = workdir or tempfile.mkdtemp(prefix=f"tfy_{self.id}_")
        self.log_dir = os.path.join(self.workdir, "logs")
        os.makedirs(self.log_dir, exist_ok=True)
        self.kill_grace_secs = kill_grace_secs
        self.server = kvmod.start_server()
        self.kv = kvmod.KVClient(self.server.address)
        self.processes: List[TaskProcess] = []
        self.placement: Dict[str, List[int]] = {}
        try:
            self._start_all()
        except BaseException:
            self.shutdown(FinalStatus.FAILED)
            raise

    # ------------------------------------------------------------------ start
    def _cpu_plan(self) -> Dict[str, List[int]]:
        """Disjoint CPU sets, ``vcores`` per task instance -- what YARN's vcore accounting (cgroups) gives the
        reference's containers (reference: tf_yarn/client.py:232, skein.model.Resources(memory, vcores)).  With
        eight trainers, an evaluator and TensorBoard on one host the 100-microsecond host loops of the trainers
        must not share cores with the side tasks.  GPU tasks are served first; when the box has fewer cores than
        the topology asks for, the remaining tasks share the cores left (at least one) instead of failing.
        TFY_PIN_CPUS=0 disables pinning."""
        if os.environ.get("TFY_PIN_CPUS", "1") == "0" or not hasattr(os, "sched_getaffinity"):
            return {}
        avail = sorted(os.sched_getaffinity(0))
        order = sorted(self.spec.services.items(), key=lambda kv: 0 if kv[1].label == NodeLabel.GPU else 1)
        want = sum(max(1, svc.vcores) * svc.instances for _, svc in order)
        if want > len(avail):
            logger.warning("topology asks for %d vcores, the box has %d: CPU pinning is partial", want, len(avail))
        plan: Dict[str, List[int]] = {}
        cursor = 0
        for task_type, svc in order:
            for task_id in range(svc.instances):
                n = max(1, svc.vcores)
                if cursor + n <= len(avail):
                    cpus = avail[cursor:cursor + n]
                    cursor += n
                else:
                    cpus = avail[cursor:] or avail[-max(1, min(n, len(avail))):]
                plan[ContainerKey(task_type, task_id).to_kv_str()] = cpus
        return plan

    def _start_all(self) -> None:
        gpus = visible_gpus()
        cursor = 0
        self.cpu_plan = self._cpu_plan()
        for task_type, svc in self.spec.services.items():
            for task_id in range(svc.instances):
                key = ContainerKey(task_type, task_id)
                assigned: List[int] = []
                if svc.label == NodeLabel.GPU and gpus:
                    for _ in range(max(1, svc.nb_proc)):
                        assigned.append(gpus[cursor % len(gpus)])
                        cursor += 1
                    if cursor > len(gpus):
                        logger.warning("more GPU task processes than GPUs (%d): %s shares GPUs %s",
                                       len(gpus), key.to_kv_str(), assigned)
                self.placement[key.to_kv_str()] = assigned
                self.processes.append(self._start_task(key, svc, assigned))

    def _start_task(self, key: ContainerKey, svc: ServiceSpec, gpus: List[int]) -> TaskProcess:
        task_dir = os.path.join(self.workdir, f"{key.type}_{key.id}")
        os.makedirs(task_dir, exist_ok=True)
        for target, source in (svc.files or {}).items():
            dst = os.path.join(task_dir, target)
            os.makedirs(os.path.dirname(dst) or task_dir, exist_ok=True)
            if os.path.lexists(dst):
                continue
            try:
                os.symlink(os.path.abspath(source), dst)
            except OSError:
                if os.path.isdir(source):
                    shutil.copytree(source, dst)
                else:
                    shutil.copy(source, dst)
        # <log_dir>/<container id>/task.log: the container id is the 2nd-to-last URL component,
        # which is what ContainerLogStatus.by_container_id parses (as with YARN log URLs)
        os.makedirs(os.path.join(self.log_dir, f"container_{key.type}_{key.id}"), exist_ok=True)
        log_path = os.path.join(self.log_dir, f"container_{key.type}_{key.id}", "task.log")
        env = dict(os.environ)
        env.update(svc.env or {})
        pythonpath = [task_dir, REPO_ROOT] + [p for p in (svc.env or {}).get("PYTHONPATH", "").split(":")
                                              if p and p != "."]
        pythonpath += [p for p in os.environ.get("PYTHONPATH", "").split(":") if p]
        env.update({
            "PYTHONPATH": ":".join(dict.fromkeys(pythonpath)),
            kvmod.KV_ADDR_ENV: self.server.address,
            "TFY_TASK_KEY": key.to_kv_str(),
            "SKEIN_CONTAINER_ID": f"{key.type}_{key.id}",
            "CONTAINER_ID": f"container_{key.type}_{key.id}",
            "TFY_APP_ID": self.id,
            "TFY_LOG_FILE": log_path,
            "TFY_GPU_IDS": ",".join(str(g) for g in gpus),
            "TFY_HOST": "127.0.0.1",
            "PYTHONUNBUFFERED": "1",
            "TFY_MEMORY_MB": str(svc.memory),
            "TFY_VCORES": str(svc.vcores),
        })
        if svc.label != NodeLabel.GPU and os.environ.get("TFY_CPU_TASKS_SEE_GPUS", "0") != "1":
            # a task without the GPU label runs on the host CPUs, as on a YARN node without GPUs: it must neither
            # compute on GPU 0 next to the trainer that owns it nor pick a GPU-only data plane its peers do not use
            env["CUDA_VISIBLE_DEVICES"] = ""
        cpus = getattr(self, "cpu_plan", {}).get(key.to_kv_str())
        argv = ["bash", "-c", svc.script]
        if cpus and shutil.which("taskset"):
            argv = ["taskset", "-c", ",".join(str(c) for c in cpus)] + argv
            env["TFY_CPUS"] = ",".join(str(c) for c in cpus)
            env.setdefault("OMP_NUM_THREADS", str(len(cpus)))
        logf = open(log_path, "ab", buffering=0)
        popen = subprocess.Popen(argv, cwd=task_dir, env=env, stdout=logf,
                                 stderr=subprocess.STDOUT, stdin=subprocess.DEVNULL, start_new_session=True)
        logf.close()
        logger.info("started %s pid=%d gpus=%s cpus=%s log=%s", key.to_kv_str(), popen.pid, gpus, cpus, log_path)
        return TaskProcess(key, popen, log_path, gpus, task_dir)

    # ----------------------------------------------------------------- status
    def report(self) -> ApplicationReport:
        if self._final_status == FinalStatus.UNDEFINED:
            codes = [p.returncode for p in self.processes]
            failed = [p for p, c in zip(self.processes, codes) if c not in (None, 0)]
            if failed:
                for p in failed:
                    why = " [step watchdog: no training progress, a peer rank is probably gone]" \
                        if p.returncode == 75 else ""           # utils/watchdog.py EXIT_CODE
                    logger.error("task %s exited with code %s%s (log: %s)", p.key.to_kv_str(), p.returncode, why,
                                 p.log_path)
                self._finish(FinalStatus.FAILED)
            elif all(c == 0 for c in codes):
                self._finish(FinalStatus.SUCCEEDED)
        if self._final_status == FinalStatus.UNDEFINED:
            state = "running"
        else:
            state = {"succeeded": "finished", "failed": "failed", "killed": "killed"}[self._final_status]
        return ApplicationReport(self.id, self.name, state, self._final_status, self.start_time,
                                 self.finish_time, f"file://{self.log_dir}", self.spec.user or _whoami(),
                                 self.spec.queue)

    def _finish(self, status: str) -> None:
        if self._final_status != FinalStatus.UNDEFINED:
            return
        self._final_status = status
        self.finish_time = time.time()
        self._kill_all()

    def _kill_all(self) -> None:
        alive = [p for p in self.processes if p.returncode is None]
        for p in alive:
            _signal_group(p.popen, signal.SIGTERM)
        deadline = time.time() + self.kill_grace_secs
        for p in alive:
            try:
                p.popen.wait(max(0.0, deadline - time.time()))
            except subprocess.TimeoutExpired:
                _signal_group(p.popen, signal.SIGKILL)
                try:
                    p.popen.wait(5)
                except subprocess.TimeoutExpired:
                    logger.error("task %s (pid %d) did not die", p.key.to_kv_str(), p.popen.pid)

    def shutdown(self, status: str = FinalStatus.SUCCEEDED) -> None:
        """Stop every task and the KV store (``app.shutdown`` of skein)."""
        self._finish(status)
        self._kill_all()
        self.close()

    def close(self) -> None:
        """Release the KV server; log files stay on disk."""
        try:
            self.kv.close()
        except Exception:  # noqa: BLE001
            pass
        if self.server is not None:
            self.server.stop()
            self.server = None

    # ------------------------------------------------------------------- logs
    def logs(self) -> Dict[str, str]:
        out = {}
        for p in self.processes:
            try:
                with open(p.log_path, errors="replace") as f:
                    out[p.container_id] = f.read()
            except OSError:
                out[p.container_id] = ""
        return out

    def cleanup(self) -> None:
        if self._own_workdir:
            shutil.rmtree(self.workdir, ignore_errors=True)


def _signal_group(popen: subprocess.Popen, sig: int) -> None:
    """Signal exactly the process group this launcher created for the task."""
    try:
        os.killpg(popen.pid, sig)       # start_new_session => pgid == pid
    except (ProcessLookupError, PermissionError):
        pass


def _whoami() -> str:
    try:
        return getpass.getuser()
    except Exception:  # noqa: BLE001
        return "unknown"


class LocalClient:
    """Submits applications on this box (skein ``Client`` stand-in)."""

    def __init__(self, workdir: Optional[str] = None):
        self.workdir = workdir
        self._apps: Dict[str, LocalApplication] = {}

    def submit_and_connect(self, spec: ApplicationSpec) -> LocalApplication:
        wd = None
        if self.workdir:
            wd = os.path.join(self.workdir, f"app_{len(self._apps)}_{uuid.uuid4().hex[:6]}")
            os.makedirs(wd, exist_ok=True)
        app = LocalApplication(spec, workdir=wd)
        self._apps[app.id] = app
        return app

    def application_report(self, app_id: str) -> ApplicationReport:
        return self._apps[app_id].report()

    def application_logs(self, app_id: str) -> Dict[str, str]:
        return self._apps[app_id].logs()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False
