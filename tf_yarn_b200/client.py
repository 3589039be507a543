"""Client-side driver: submit an experiment to the box, watch it, report on it.

``run_on_yarn`` keeps the reference's name and signature (reference:
tf_yarn/client.py:299-469) so user scripts switch over by changing an import;
``run_on_b200`` is an alias.  What changes is the substrate: instead of a
skein/YARN application, :mod:`tf_yarn_b200.launcher.local` starts one process per
task instance on this 8xH100 box, pins GPU-labelled instances to H100s and
hosts the KV rendezvous store.  YARN-only arguments (``queue``, ``acls``,
``file_systems``, ``pyenv_zip_path``, ``cuda_runtime_hdfs_path``) are accepted
and ignored with a debug log.

Lifecycle (same as the reference): publish ``cluster_instances`` and the
cloudpickled ``experiment_fn`` to the KV store, poll the application report,
aggregate the tasks' lifecycle events into a text report + :class:`Metrics`,
forward evaluator statistics / TensorBoard URL / task logs to the experiment
tracker, raise :class:`RunFailed` on failure and retry the WHOLE application up
to ``nb_retries`` more times.
"""
from __future__ import annotations

import importlib
import json
import logging
import os
import signal
import sys
import threading
import time
from contextlib import contextmanager, suppress
from datetime import timedelta
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Tuple, Union

import cloudpickle

from tf_yarn_b200 import (_env, _internal, constants, evaluator_metrics, metrics, mlflow, tensorboard, topologies)
from tf_yarn_b200._task_commons import catchtime, is_chief, is_evaluator, is_worker
from tf_yarn_b200.launcher.local import (ApplicationReport, ApplicationSpec, FinalStatus, LocalApplication,
                                         LocalClient, ServiceSpec)
from tf_yarn_b200.topologies import ContainerKey

logger = logging.getLogger(__name__)

ExperimentFn = Union[Callable[[], Any], Callable[[int], Any]]

DEFAULT_POLL_EVERY_SECS = float(os.environ.get("TFY_POLL_EVERY_SECS", "0.5"))


class LocalCluster(NamedTuple):
    """Everything the client holds about one submitted application (``SkeinCluster`` stand-in)."""
    client: LocalClient
    app: LocalApplication
    tasks: List[Tuple[str, int, int]]
    event_listener: threading.Thread
    events: Dict[ContainerKey, Dict[str, str]]


SkeinCluster = LocalCluster  # name used by code written against the reference


class ContainerLogStatus(NamedTuple):
    log_urls: Dict[ContainerKey, str] = dict()
    container_status: Dict[ContainerKey, str] = dict()

    def by_container_id(self) -> Dict[str, Tuple[ContainerKey, str]]:
        """``{container_id: (task key, status)}``; the id is the second-to-last component of the log URL."""
        containers: Dict[str, Tuple[ContainerKey, str]] = {}
        if len(self.log_urls) != len(self.container_status):
            logger.warning("logs_urls and container_status dicts have not the same length")
            return containers
        for (task_key, url), status in zip(self.log_urls.items(), self.container_status.values()):
            containers[self._get_container_id(url)] = (task_key, status)
        return containers

    @staticmethod
    def _get_container_id(url: str) -> str:
        if not url:
            return ""
        parts = url.split("/")
        return parts[-2] if len(parts) > 1 else ""


class RunFailed(Exception):
    """``run_on_yarn`` failed."""


# ---------------------------------------------------------------------------
# application set-up
# ---------------------------------------------------------------------------
def _setup_task_env(files: Optional[Dict[str, str]] = None, env: Optional[Dict[str, str]] = None,
                    n_try: int = 0) -> Tuple[Dict[str, str], Dict[str, str]]:
    """Files and environment common to every task of one attempt."""
    task_files = dict(files or {})
    task_env = dict(env or {})
    task_env["TF_YARN_N_TRY"] = str(n_try)
    task_env["TFY_N_TRY"] = str(n_try)
    # modules/packages passed via ``files`` are importable: the task workdir leads PYTHONPATH
    task_env["PYTHONPATH"] = ".:" + task_env.get("PYTHONPATH", "")
    task_env.update(mlflow.task_env())
    return task_files, task_env


def _setup_to_use_cuda_archive(env: Dict[str, str], pre_script_hook: str, cuda_runtime_hdfs_path: str) -> str:
    """The reference ships a CUDA runtime tarball from HDFS (client.py:154-167); the box already has
    CUDA 12.9, so this only validates the arguments the same way and leaves the hook untouched."""
    if "LD_LIBRARY_PATH" not in env:
        logger.warning("No LD_LIBRARY_PATH found in env. The cuda archive option is ignored on a H100 box.")
        return pre_script_hook
    logger.info("cuda_runtime_hdfs_path=%s ignored: the box's CUDA toolkit is used", cuda_runtime_hdfs_path)
    return pre_script_hook


def _setup_cluster_spec(task_instances: List[Tuple[str, int, int]], app) -> None:
    """Publish ``cluster_instances`` = training-cluster roles (side tasks excluded)."""
    cluster_instances = [t for t in task_instances if t[0] not in topologies.SIDE_TASK_TYPES]
    app.kv[constants.KV_CLUSTER_INSTANCES] = json.dumps(cluster_instances).encode()


def _setup_local_cluster(
        task_specs: Dict[str, topologies.TaskSpec], *, custom_task_module: Optional[str] = None,
        local_client: Optional[LocalClient] = None, files: Optional[Dict[str, str]] = None,
        env: Optional[Dict[str, str]] = None, queue: str = "default", name: str = "RunOnB200", n_try: int = 0,
        pre_script_hook: Optional[str] = None, cuda_runtime_hdfs_path: Optional[str] = None,
        interpreter: Optional[str] = None) -> LocalCluster:
    env = dict(env or {})
    pre_script_hook = pre_script_hook or ""
    if cuda_runtime_hdfs_path:
        pre_script_hook = _setup_to_use_cuda_archive(env, pre_script_hook, cuda_runtime_hdfs_path)
    task_files, task_env = _setup_task_env(files, env, n_try)
    trainer_labels = {task_specs[t].label for t in ("chief", "worker") if t in task_specs}
    if len(trainer_labels) > 1 and "ps" not in task_specs:
        logger.warning("chief and worker tasks carry different node labels: synchronous all-reduce training needs every "
                       "trainer on a GPU (NVLink kernels) or every trainer on the CPU (gloo), not a mix")
    if "ps" in task_specs and any(task_specs[t].label != topologies.NodeLabel.GPU
                                  for t in ("chief", "worker", "ps") if t in task_specs):
        # the peer-HBM parameter-server plane needs EVERY trainer and ps on a GPU; any CPU-labelled one (the
        # reference's default ps_strategy_topology()) puts the whole application on the shared-memory plane
        task_env.setdefault("TFY_PS_PLANE", "shm")

    services: Dict[str, ServiceSpec] = {}
    for task_type, spec in task_specs.items():
        service_env = dict(task_env)
        if spec.tb_termination_timeout_seconds >= 0:
            service_env["TB_TERMINATION_TIMEOUT_SECONDS"] = str(spec.tb_termination_timeout_seconds)
        if spec.tb_model_dir:
            service_env["TB_MODEL_DIR"] = str(spec.tb_model_dir)
        if spec.tb_extra_args:
            service_env["TB_EXTRA_ARGS"] = str(spec.tb_extra_args)
        cmd = _env.gen_task_cmd(interpreter, task_type, custom_task_module)
        script = "set -e\n" + (pre_script_hook + "\n" if pre_script_hook else "") + "exec " + cmd
        services[task_type] = ServiceSpec(script=script, instances=spec.instances, nb_proc=spec.nb_proc_per_worker,
                                          label=spec.label, memory=spec.memory, vcores=spec.vcores,
                                          env=service_env, files=task_files)

    container_info = [(t, s.instances, s.nb_proc_per_worker) for t, s in task_specs.items()]
    events: Dict[ContainerKey, Dict[str, str]] = {
        task.to_container_key(): {} for task in _internal.iter_tasks(container_info)}
    if local_client is None:
        local_client = LocalClient()
    with catchtime("submitting application"):
        app = local_client.submit_and_connect(ApplicationSpec(services, name=name, queue=queue))
    stop_listening = threading.Event()
    listener = threading.Thread(target=_aggregate_events, args=(app.kv, events, stop_listening), daemon=True)
    listener.stop_event = stop_listening  # type: ignore[attr-defined]
    listener.start()
    return LocalCluster(local_client, app, container_info, listener, events)


_setup_skein_cluster = _setup_local_cluster


def _run_on_cluster(experiment_fn: ExperimentFn, cluster: LocalCluster,
                    eval_monitor_log_thresholds: Optional[Dict[str, Tuple[float, float]]] = None, n_try: int = 0,
                    poll_every_secs: float = DEFAULT_POLL_EVERY_SECS) -> Optional[metrics.Metrics]:
    # serialize early: a non-picklable experiment must fail before tasks wait on it
    with catchtime("serializing experiment function"):
        serialized_fn = cloudpickle.dumps(experiment_fn)
    return _execute_and_await_termination(cluster, serialized_fn, eval_monitor_log_thresholds, n_try=n_try,
                                          poll_every_secs=poll_every_secs)


def _default_acls_all_access() -> Dict[str, Any]:
    return {"enable": True, "ui_users": ["*"], "view_users": ["*"]}


# ---------------------------------------------------------------------------
# public entry point
# ---------------------------------------------------------------------------
def run_on_yarn(
        experiment_fn: ExperimentFn,
        task_specs: Dict[str, topologies.TaskSpec],
        *,
        pyenv_zip_path: Union[str, Dict[topologies.NodeLabel, str], None] = None,
        skein_client: Optional[LocalClient] = None,
        files: Optional[Dict[str, str]] = None,
        env: Dict[str, str] = {},
        queue: str = "default",
        acls: Any = None,
        file_systems: Optional[List[str]] = None,
        eval_monitor_log_thresholds: Optional[Dict[str, Tuple[float, float]]] = None,
        nb_retries: int = 0,
        custom_task_module: Optional[str] = None,
        name: str = "RunOnB200",
        pre_script_hook: Optional[str] = None,
        cuda_runtime_hdfs_path: Optional[str] = None,
        poll_every_secs: float = DEFAULT_POLL_EVERY_SECS,
) -> Optional[metrics.Metrics]:
    """Run an experiment on the local 8xH100 box.

    Parameters keep the reference's meaning (reference: tf_yarn/client.py:317-417):

    experiment_fn
        Zero-argument function building the experiment (``Experiment`` /
        ``KerasExperiment`` / ``PytorchExperiment``); evaluated inside every
        task.  For ``tf_yarn_b200.distributed`` it is ``fn(local_rank)`` itself.
    task_specs
        ``{role: TaskSpec}`` with roles from chief / worker / ps / evaluator /
        tensorboard.
    files
        ``{target: source}`` made available in every task's working directory,
        which is on ``PYTHONPATH``.
    env
        Extra environment variables for every task.
    eval_monitor_log_thresholds
        ``{metric: (low, high)}`` for the evaluator statistics the client logs.
    nb_retries
        How many more times the WHOLE application is re-run after a failure.
    custom_task_module
        Module run as ``python -m <module>`` in chief/worker/ps/evaluator tasks
        instead of the default parameter-server task.
    pre_script_hook
        bash executed in every task before the task program.
    pyenv_zip_path
        A python interpreter path (str) or ``{NodeLabel: interpreter}``; archives
        are not needed on a single box, ``None`` uses the current interpreter.
    skein_client
        A :class:`tf_yarn_b200.launcher.local.LocalClient` to reuse.

    Raises
    ------
    RunFailed
        If the final status of the application is ``"failed"``.
    """
    if nb_retries < 0:
        raise ValueError(f"nb_retries must be greater or equal to 0. Got {nb_retries}")
    for ignored, value in (("queue", queue if queue != "default" else None), ("acls", acls),
                           ("file_systems", file_systems)):
        if value:
            logger.debug("run_on_yarn(%s=...) has no meaning on a single box; ignored", ignored)
    interpreter = _setup_pyenvs(pyenv_zip_path)
    files = _add_editable_requirements(files)

    n_try = 0
    while True:
        logger.info("Try: %d", n_try + 1)
        try:
            with catchtime("setting up the local cluster"):
                cluster = _setup_skein_cluster(
                    task_specs=task_specs, local_client=skein_client, files=files, env=env, queue=queue, name=name,
                    n_try=n_try, custom_task_module=custom_task_module, pre_script_hook=pre_script_hook,
                    cuda_runtime_hdfs_path=cuda_runtime_hdfs_path, interpreter=interpreter)
            with _shutdown_on_exception(cluster.app):
                _setup_cluster_spec(cluster.tasks, cluster.app)
                return _run_on_cluster(experiment_fn, cluster, eval_monitor_log_thresholds, n_try,
                                       poll_every_secs=poll_every_secs)
        except Exception:
            n_try += 1
            if n_try == nb_retries + 1:
                raise
            logger.exception("Retrying user application ... %d remaining attempts", nb_retries + 1 - n_try)
    return None  # unreachable; keeps type checkers happy


run_on_b200 = run_on_yarn


def _add_editable_requirements(files: Optional[Dict[str, str]]) -> Dict[str, str]:
    """The reference ships editable (``pip -e``) installs to the containers (client.py:498-505); on one
    box they are importable already, so this only normalises ``files``."""
    from tf_yarn_b200 import packaging
    files = dict(files or {})
    for dirname, path in packaging.get_editable_requirements().items():
        files.setdefault(dirname, path)
    return files


def _setup_pyenvs(pyenv_zip_path: Union[str, Dict[topologies.NodeLabel, str], None]) -> Optional[str]:
    """Interpreter used for the tasks.  A dict per NodeLabel is collapsed (one box => one env)."""
    if pyenv_zip_path is None:
        return None
    if isinstance(pyenv_zip_path, dict):
        pyenv_zip_path = pyenv_zip_path.get(topologies.NodeLabel.GPU) or next(iter(pyenv_zip_path.values()))
    if os.path.isfile(pyenv_zip_path) and os.access(pyenv_zip_path, os.X_OK):
        return pyenv_zip_path
    logger.debug("pyenv_zip_path=%s is not an interpreter; tasks use %s", pyenv_zip_path, sys.executable)
    return None


def get_safe_experiment_fn(full_fn_name: str, *args) -> Callable[[], Any]:
    """Experiment function that is imported BY NAME inside the task instead of being pickled.

    ``full_fn_name`` is ``"package.module.function"``; ``args`` are passed to it.
    (reference: tf_yarn/client.py:472-495)
    """
    module_name, fn_name = full_fn_name.rsplit(".", 1)

    def _safe_exp_fn():
        module = importlib.import_module(module_name)
        return getattr(module, fn_name)(*args)

    return _safe_exp_fn


@contextmanager
def _shutdown_on_exception(app):
    """Ctrl-C kills the application (KILLED); any other exception fails it (FAILED) and propagates."""
    if threading.current_thread() is threading.main_thread():
        with suppress(ValueError):
            signal.signal(signal.SIGINT, signal.default_int_handler)
    try:
        yield
    except (KeyboardInterrupt, SystemExit):
        with suppress(Exception):
            app.shutdown(FinalStatus.KILLED)
        logger.error("Application killed on user request")
    except Exception:
        with suppress(Exception):
            app.shutdown(FinalStatus.FAILED)
        logger.exception("Application shutdown due to an exception")
        raise


# ---------------------------------------------------------------------------
# watch loop
# ---------------------------------------------------------------------------
def _execute_and_await_termination(
        cluster: LocalCluster, serialized_fn: bytes,
        eval_monitor_log_thresholds: Optional[Dict[str, Tuple[float, float]]] = None, n_try: int = 0,
        poll_every_secs: float = DEFAULT_POLL_EVERY_SECS) -> Optional[metrics.Metrics]:
    app = cluster.app
    app.kv[constants.KV_EXPERIMENT_FN] = serialized_fn
    all_tasks = list(_internal.iter_tasks(cluster.tasks))
    eval_metrics_logger = evaluator_metrics.EvaluatorMetricsLogger(
        [t for t in all_tasks if t.type == "evaluator"], app, eval_monitor_log_thresholds, n_try=n_try)
    tb_url_event = tensorboard.url_event_name(all_tasks)
    tensorboard_url_logger = metrics.OneShotMetricsLogger(
        app, [(tb_url_event, tensorboard.URL_EVENT_LABEL)] if tb_url_event else [], n_try)

    state = None
    container_log_urls: Dict[str, str] = {}
    while True:
        report = cluster.client.application_report(app.id)
        if state != report.state:
            logger.info("Application report for %s (state: %s)%s", app.id, report.state, _format_app_report(report))
        if report.state == "running":
            with suppress(Exception):
                for key in app.kv.keys():
                    if "/logs" in key and key not in container_log_urls:
                        container_log_urls[key] = app.kv.wait(key).decode()
        if report.final_status != FinalStatus.UNDEFINED:
            # last look at the side channels (a short job may end within one poll period)
            with suppress(Exception):
                eval_metrics_logger.log()
                tensorboard_url_logger.log()
            # drain: give the aggregator a moment to receive the last PUTs, then stop it
            _join_listener(cluster.event_listener)
            log_events, result_metrics, container_status = _handle_events(cluster.events, n_try)
            logger.info(log_events)
            logger.info("container logs: %s", ", ".join(v for v in container_log_urls.values() if v))
            logs = _get_app_logs(cluster.client, app)
            _save_logs_to_mlflow(logs, container_status.by_container_id(), n_try)
            app.close()
            if report.final_status == FinalStatus.FAILED:
                failed = [f"{k.to_kv_str()}: {s}" for k, s in container_status.container_status.items()
                          if s in ("FAILED", "KILLED")]
                tails = _failed_log_tails(logs, container_status)
                raise RunFailed(f"application {app.id} failed ({'; '.join(failed)}); logs in {app.log_dir}\n"
                                + log_events + tails)
            break
        eval_metrics_logger.log()
        tensorboard_url_logger.log()
        time.sleep(poll_every_secs)
        state = report.state
    result_metrics.log_mlflow(n_try)
    return result_metrics


def _failed_log_tails(logs: Optional[Dict[str, str]], status: "ContainerLogStatus", n_lines: int = 15) -> str:
    """Last lines of the log of every task that died without publishing a ``stop`` event."""
    if not logs:
        return ""
    out = []
    for container_id, (task, st) in status.by_container_id().items():
        if st == "KILLED" and logs.get(container_id):
            tail = "\n".join(logs[container_id].rstrip().splitlines()[-n_lines:])
            out.append(f"\n--- last lines of {task.to_kv_str()} ({container_id}):\n{tail}")
    return "".join(out)


def _join_listener(listener: threading.Thread, settle_secs: float = 0.3) -> None:
    time.sleep(settle_secs)
    stop = getattr(listener, "stop_event", None)
    if stop is not None:
        stop.set()
    listener.join(timeout=5)


def _save_logs_to_mlflow(logs: Optional[Dict[str, str]], containers: Dict[str, Tuple[ContainerKey, str]],
                         n_try: int) -> None:
    if not logs:
        return
    for key, text in logs.items():
        if key in containers:
            task, status = containers[key]
            filename = mlflow.format_key(f"{task.to_kv_str()}_{status}_{n_try}")
        else:
            filename = mlflow.format_key(f"{key}_{n_try}")
        mlflow.save_text_to_mlflow(text, filename)


def _format_app_report(report: ApplicationReport) -> str:
    attrs = ["queue", "start_time", "finish_time", "final_status", "tracking_url", "user"]
    return os.linesep + os.linesep.join(f"{attr:>16}: {getattr(report, attr) or ''}" for attr in attrs)


def _aggregate_events(kv, events: Dict[ContainerKey, Dict[str, str]],
                      stop: Optional[threading.Event] = None) -> None:
    """Collect every ``"<type>:<id>/<stage>"`` PUT into ``events[task][stage]``.

    Runs on a daemon thread for the life of the application; ends when the KV
    server goes away or ``stop`` is set.
    """
    with suppress(ConnectionError, OSError):
        for key, value in kv.events(event_type="PUT", stop=stop):
            if "/" not in key:
                continue
            task_key_str, stage = key.rsplit("/", 1)
            if ":" not in task_key_str:
                continue
            task = ContainerKey.from_kv_str(task_key_str)
            if task is None:
                continue
            if task not in events:
                logger.debug("event for a task that is not part of the application: %s", key)
                continue
            events[task][stage] = value.decode() if isinstance(value, (bytes, bytearray)) else value


def _handle_events(events: Dict[ContainerKey, Dict[str, str]],
                   n_try: int) -> Tuple[str, metrics.Metrics, ContainerLogStatus]:
    """Turn the aggregated lifecycle events into a text report, Metrics and per-task statuses.

    Status: FAILED if ``stop`` carries a traceback, SUCCEEDED if ``stop`` is empty,
    KILLED if some events but no ``stop``, REQUESTED if the task never reported.
    Global training time = max(stop) - min(start) over chief+workers, only when
    every one of them reported both timers without an exception; same for evaluators.
    """
    header: List[str] = []
    details: List[str] = []
    train_start: List[float] = []
    train_stop: List[float] = []
    eval_start: List[float] = []
    eval_stop: List[float] = []
    valid_training_time = valid_eval_time = True
    container_duration: Dict[ContainerKey, Optional[timedelta]] = {}
    train_eval_time_per_node: Dict[ContainerKey, Optional[timedelta]] = {}
    log_urls: Dict[ContainerKey, str] = {}
    statuses: Dict[ContainerKey, str] = {}

    for task_key, stages in sorted(events.items()):
        if "stop" in stages:
            status = "FAILED" if stages["stop"] else "SUCCEEDED"
        elif stages:
            status = "KILLED"
        else:
            status = "REQUESTED"
        exception = stages.get("stop", "")
        log_urls[task_key] = stages.get("logs", "")
        statuses[task_key] = status

        container_duration[task_key] = None
        if "container_start_time" in stages and "container_stop_time" in stages:
            container_duration[task_key] = timedelta(
                seconds=float(stages["container_stop_time"]) - float(stages["container_start_time"]))

        train_eval_time_per_node[task_key] = None
        trains = is_worker(task_key.type) or is_chief(task_key.type)
        if "train_eval_start_time" in stages and "train_eval_stop_time" in stages and not exception:
            t0, t1 = float(stages["train_eval_start_time"]), float(stages["train_eval_stop_time"])
            train_eval_time_per_node[task_key] = timedelta(seconds=t1 - t0)
            if trains:
                train_start.append(t0)
                train_stop.append(t1)
            elif is_evaluator(task_key.type):
                eval_start.append(t0)
                eval_stop.append(t1)
        elif trains:
            valid_training_time = False
        elif is_evaluator(task_key.type):
            valid_eval_time = False

        header.append(f"{task_key.to_kv_str():>16}  {stages.get('init', '')}  {status}  {log_urls[task_key]}"
                      f"  Container duration: {container_duration[task_key]}"
                      f"  Training/evaluation duration : {train_eval_time_per_node[task_key]}")
        if exception:
            details.append(f"Exception in task {task_key.to_kv_str()}:")
            details.append(exception)

    training_time = (timedelta(seconds=max(train_stop) - min(train_start))
                     if valid_training_time and train_start else None)
    eval_time = timedelta(seconds=max(eval_stop) - min(eval_start)) if valid_eval_time and eval_start else None
    header.append(f"Training time = {training_time}")
    header.append(f"Evaluation time = {eval_time}")
    result = metrics.Metrics(training_time, eval_time, container_duration, train_eval_time_per_node)
    text = (os.linesep + os.linesep.join(header) + os.linesep * (1 + bool(details)) + os.linesep.join(details))
    return text, result, ContainerLogStatus(log_urls, statuses)


def _get_app_logs(client: LocalClient, app) -> Optional[Dict[str, str]]:
    """Task logs by container id (the YARN log-aggregation fetch of client.py:748-765 is a file read here)."""
    try:
        return client.application_logs(app.id)
    except Exception:  # noqa: BLE001
        logger.warning("Cannot collect logs", exc_info=True)
        return None
