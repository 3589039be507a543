"""Recipe for ``oracle/_ref/``: the original tf-yarn package, installed unmodified, that the benchmark's reference
arm (``bench.py --impl reference``) and the control-plane shim test run against.

The original project is pure Python, so its build is a ``pip install --target`` of its source checkout: offline,
without dependencies (the shims under ``bench/shims`` stand in for skein / cluster-pack / webdataset).  The source
checkout is ``$TFY_REFERENCE_SRC`` (default ``/root/reference``); without it nothing is installed and the arm and
the test report the reference as unavailable.  ``oracle/_ref/`` is git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")


def reference_src() -> str:
    return os.environ.get("TFY_REFERENCE_SRC", "/root/reference")


def installed() -> bool:
    return os.path.isdir(os.path.join(REF_DIR, "tf_yarn"))


def build(verbose: bool = True) -> bool:
    """Install the original package into oracle/_ref/ unless it is there already; False when there is no source."""
    if installed():
        return True
    src = reference_src()
    if not os.path.isfile(os.path.join(src, "setup.py")):
        if verbose:
            sys.stderr.write(f"[oracle] no reference sources at {src}: oracle/_ref not built\n")
        return False
    with tempfile.TemporaryDirectory(prefix="tfy_ref", dir=HERE) as tmp:
        cmd = [sys.executable, "-m", "pip", "install", "--quiet", "--no-index", "--no-deps", "--no-build-isolation",
               "--no-cache-dir", "--target", os.path.join(tmp, "_ref"), src]
        res = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, PIP_NO_INPUT="1"))
        if res.returncode != 0:
            raise RuntimeError(f"pip install of the reference failed:\n{res.stdout}\n{res.stderr}")
        os.replace(os.path.join(tmp, "_ref"), REF_DIR)      # complete install or none
    if verbose:
        sys.stderr.write(f"[oracle] installed the reference into {REF_DIR}\n")
    return True


if __name__ == "__main__":
    build()
