"""``python -m tf_yarn_b200.bin.check_hadoop_env`` -- same entry point name as the reference's environment check.

The reference (tf_yarn/bin/check_hadoop_env.py:26-172) verifies the Hadoop variables, does a round trip
of a small file through HDFS with TensorFlow's filesystem layer, launches a one-container application that
re-reads the file and posts ``result`` to the KV store, and writes everything to ``check_hadoop_env.log``
in the working directory.  There is neither Hadoop nor YARN on a H100 box: this module keeps the command,
the hidden ``--file`` container mode, the ``result`` key and the log file, and runs the single-box
equivalents (toolchain, native kernels, GPUs + peer access, KV store, file round trip through
:mod:`tf_yarn_b200.utils.fs`, one-task application through the local launcher) implemented in
:mod:`tf_yarn_b200.bin.check_env`.
"""
from __future__ import annotations

import argparse
import logging
import os
import sys
import tempfile
import uuid

from tf_yarn_b200.bin import check_env as _impl

logger = logging.getLogger(__name__)

EXPECTED_CONTENT = "Hello tf-yarn!"
RESULT_CHECK_FILE = "check_hadoop_env.log"


def write_dummy_file(directory: str) -> str:
    """Write the probe file through the framework's filesystem layer and return its path."""
    from tf_yarn_b200.utils import fs
    path = os.path.join(directory, f"hello_tf_yarn_{uuid.uuid4().hex}.txt")
    filesystem, resolved = fs.resolve_filesystem_and_path(path)
    with filesystem.open(resolved, "wb") as fd:
        fd.write(EXPECTED_CONTENT.encode())
    return path


def read_file(path: str) -> str:
    from tf_yarn_b200.utils import fs
    filesystem, resolved = fs.resolve_filesystem_and_path(path)
    with filesystem.open(resolved, "rb") as fd:
        return fd.read().decode()


def check_env() -> bool:
    """Environment variables the launcher and the kernels rely on (the reference checks JAVA_HOME & co.)."""
    ok = True
    cuda_home = os.environ.get("CUDA_HOME") or ("/usr/local/cuda" if os.path.isdir("/usr/local/cuda") else None)
    logger.info("CUDA_HOME: %s", cuda_home or "MISSING")
    ok = ok and cuda_home is not None
    for var in ("TFY_KV_ADDR", "TFY_TASK_KEY"):
        if var in os.environ:
            logger.info("%s=%s (set: running inside a task container)", var, os.environ[var])
    return ok and _impl.check_toolchain()


def add_file_handler() -> None:
    fh = logging.FileHandler(RESULT_CHECK_FILE)
    fh.setLevel(logging.INFO)
    fh.setFormatter(logging.Formatter("%(asctime)s - %(name)s - %(levelname)s - %(message)s"))
    logging.getLogger().addHandler(fh)
    logger.info("results will be written in %s/%s", os.getcwd(), RESULT_CHECK_FILE)


def _container_fn(path: str):
    def fn(local_rank: int):
        main(["--file", path])
    return fn


def launch_remote_check(path: str) -> bool:
    """One-task application that re-reads the probe file and posts ``result`` (reference: :70-105)."""
    from tf_yarn_b200 import TaskSpec
    from tf_yarn_b200.distributed import run_on_yarn
    try:
        run_on_yarn(_container_fn(path), {"worker": TaskSpec(memory="1 GiB", vcores=1)}, name="check_hadoop_env")
        return True
    except Exception as exc:  # noqa: BLE001
        logger.error("remote check failed: %s", exc)
        return False


def main(argv=None) -> int:
    parser = argparse.ArgumentParser(prog="check_hadoop_env")
    parser.add_argument("--file", help=argparse.SUPPRESS)
    args = parser.parse_args(argv)
    if args.file:
        # executed inside a task container
        from tf_yarn_b200._task_commons import TaskClient
        result = False
        try:
            result = read_file(args.file) == EXPECTED_CONTENT
            logger.info("check file round trip %s", result)
        finally:
            TaskClient.from_current().kv["result"] = str(result).encode()
        if not result:
            raise RuntimeError("probe file content mismatch")
        return 0
    logging.basicConfig(level=logging.INFO)
    logging.getLogger().setLevel(logging.INFO)      # (basicConfig is a no-op when handlers already exist)
    add_file_handler()
    check_ok = check_env()
    logger.info("check environment variables: %s", check_ok)
    if check_ok:
        check_ok = _impl.check_native() and _impl.check_gpus() and _impl.check_kv()
        logger.info("check local kernels / GPUs / KV store: %s", check_ok)
    if check_ok:
        with tempfile.TemporaryDirectory() as tmp:
            path = write_dummy_file(tmp)
            check_ok = read_file(path) == EXPECTED_CONTENT
            logger.info("check local file round trip: %s", check_ok)
            if check_ok:
                check_ok = launch_remote_check(path)
                logger.info("remote_check: %s", check_ok)
    logger.info("H100 box setup: %s", "OK" if check_ok else "KO")
    return 0 if check_ok else 1


if __name__ == "__main__":
    sys.exit(main())
