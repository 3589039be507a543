"""``check_b200_env``: is this box ready to run tf_yarn_b200 jobs?

The reference ships ``check_hadoop_env`` (reference: tf_yarn/bin/check_hadoop_env.py:26-172): it checks
environment variables, writes/reads a file on HDFS and launches a one-container application that
re-reads the file and posts a ``result`` key.  The single-box equivalent checks the toolchain, the
native libraries, the GPUs and their peer access, the KV store, and launches a one-task application
that reads a file written by the client and reports back through the KV store.
"""
from __future__ import annotations

import argparse
import logging
import os
import shutil
import sys
import tempfile

logger = logging.getLogger("check_b200_env")


def check_toolchain() -> bool:
    ok = True
    for tool in ("nvcc", "g++"):
        path = shutil.which(tool) or (os.path.exists(f"/usr/local/cuda/bin/{tool}") and f"/usr/local/cuda/bin/{tool}")
        logger.info("%-6s %s", tool, path or "MISSING")
        ok = ok and bool(path)
    return ok


def check_native() -> bool:
    try:
        from tf_yarn_b200.ops import build
        build.build_all(verbose=False)
        from tf_yarn_b200.ops import native
        native.load()
        logger.info("native libraries built and loadable")
        return True
    except Exception as exc:  # noqa: BLE001
        logger.error("native libraries: %s", exc)
        return False


def check_gpus() -> bool:
    import torch
    if not torch.cuda.is_available():
        logger.warning("no CUDA device visible: only the CPU (gloo / shared-memory) data planes will work")
        return True
    n = torch.cuda.device_count()
    ok = True
    for i in range(n):
        prop = torch.cuda.get_device_properties(i)
        logger.info("GPU %d: %s sm_%d%d %.0f GB %d SMs", i, prop.name, prop.major, prop.minor,
                    prop.total_memory / 2 ** 30, prop.multi_processor_count)
        if (prop.major, prop.minor) != (9, 0):
            logger.warning("GPU %d is not sm_90 (H100): the kernels are compiled for sm_90a only", i)
            ok = False
    for i in range(n):
        for j in range(n):
            if i != j and not torch.cuda.can_device_access_peer(i, j):
                logger.error("no peer access %d -> %d (NVLink/NVSwitch required)", i, j)
                ok = False
    return ok


def check_kv() -> bool:
    from tf_yarn_b200 import kv
    srv = kv.start_server()
    try:
        c = kv.KVClient(srv.address)
        c["probe"] = b"ok"
        good = c.wait("probe", timeout=5) == b"ok"
        logger.info("KV store (%s) round trip: %s", "native" if srv.native else "python", good)
        return good
    finally:
        srv.stop()


def _probe_task_fn(path: str):
    def fn(local_rank: int):
        from tf_yarn_b200._task_commons import TaskClient
        with open(path) as f:
            ok = f.read() == "tf_yarn_b200"
        TaskClient.from_current().kv["result"] = str(ok).encode()
    return fn


def check_launch() -> bool:
    from tf_yarn_b200 import TaskSpec
    from tf_yarn_b200.distributed import run_on_yarn
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "probe.txt")
        with open(path, "w") as f:
            f.write("tf_yarn_b200")
        try:
            run_on_yarn(_probe_task_fn(path), {"worker": TaskSpec(memory="1 GiB", vcores=1)}, name="check_env")
            logger.info("one-task application: SUCCEEDED")
            return True
        except Exception as exc:  # noqa: BLE001
            logger.error("one-task application failed: %s", exc)
            return False


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--skip-launch", action="store_true", help="do not start the one-task application")
    args = ap.parse_args(argv)
    logging.basicConfig(level="INFO", format="%(message)s")
    results = {"toolchain": check_toolchain(), "native": check_native(), "gpus": check_gpus(), "kv": check_kv()}
    if not args.skip_launch:
        results["launch"] = check_launch()
    for k, v in results.items():
        logger.info("%-10s %s", k, "OK" if v else "FAILED")
    return 0 if all(results.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
