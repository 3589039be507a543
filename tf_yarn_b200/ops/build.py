"""In-tree native build for tf_yarn_b200 (sm_90a only: NVIDIA H100).

Two shared objects are produced next to the sources (they are git-ignored and
rebuilt by ``build_all`` whenever a source or a flag changes):

* ``tf_yarn_b200/ops/lib/libtfy_b200.so`` -- every CUDA kernel + the VMM /
  multicast symmetric-memory runtime (nvcc, ``-gencode
  arch=compute_90a,code=sm_90a -lineinfo``).
* ``tf_yarn_b200/kv/libtfy_kv.so`` -- the C++ key-value rendezvous server
  (g++, no CUDA), the stand-in for the skein ApplicationMaster KV store.

The libraries expose a plain C ABI and are loaded with ``ctypes``; there is no
JIT cache outside the repo and no dependence on the torch C++ ABI.
"""
from __future__ import annotations

import concurrent.futures
import contextlib
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "lib", "obj")
CUDA_LIB = os.path.join(LIBDIR, "libtfy_b200.so")
KV_DIR = os.path.join(os.path.dirname(HERE), "kv")
KV_LIB = os.path.join(KV_DIR, "libtfy_kv.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


@contextlib.contextmanager
def _build_lock(path: str):
    """Exclusive inter-process lock: the N rank processes a launcher starts in a fresh checkout must not compile
    and link the same paths concurrently (one builds, the others wait and then find everything up to date)."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as fh:
        fcntl.flock(fh, fcntl.LOCK_EX)
        try:
            yield
        finally:
            fcntl.flock(fh, fcntl.LOCK_UN)


def have_nvcc() -> bool:
    try:
        _nvcc()
        return True
    except RuntimeError:
        return False


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; tf_yarn_b200 kernels need the CUDA 12.9 toolkit")


def _digest(path: str, extra: str = "") -> str:
    h = hashlib.sha1()
    h.update(extra.encode())
    with open(path, "rb") as f:
        h.update(f.read())
    # headers are few: hash them all into every object's key
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cuh", ".h")):
            with open(os.path.join(CSRC, name), "rb") as f:
                h.update(f.read())
    return h.hexdigest()


def cuda_sources() -> List[str]:
    return sorted(
        os.path.join(CSRC, n) for n in os.listdir(CSRC) if n.endswith((".cu", ".cpp"))
    )


def _compile_one(src: str, verbose: bool) -> str:
    os.makedirs(OBJDIR, exist_ok=True)
    base = os.path.basename(src)
    obj = os.path.join(OBJDIR, base + ".o")
    stamp = obj + ".sha1"
    key = _digest(src, " ".join(NVCC_FLAGS))
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == key:
        return obj
    tmp_obj = obj + f".tmp{os.getpid()}"
    cmd = [_nvcc()] + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", tmp_obj]
    if src.endswith(".cpp"):
        cmd = [_nvcc(), "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-x", "cu",
               "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
               "-I", CSRC, "-c", src, "-o", tmp_obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = os.path.join(OBJDIR, base + ".log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if res.returncode != 0:
        with contextlib.suppress(OSError):
            os.remove(tmp_obj)
        raise RuntimeError(f"nvcc failed for {base}:\n{res.stdout}\n{res.stderr}")
    os.replace(tmp_obj, obj)
    if verbose:
        sys.stderr.write(f"[tf_yarn_b200.build] compiled {base}\n")
    with open(stamp + ".tmp", "w") as f:
        f.write(key)
    os.replace(stamp + ".tmp", stamp)
    return obj


def build_cuda(verbose: bool = False) -> str:
    """Compile every ``.cu``/``.cpp`` under ``ops/csrc`` for sm_90a and link them."""
    srcs = cuda_sources()
    with _build_lock(os.path.join(LIBDIR, ".build.lock")):
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
            objs = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
        newest = max(os.path.getmtime(o) for o in objs)
        if os.path.exists(CUDA_LIB) and os.path.getmtime(CUDA_LIB) >= newest:
            return CUDA_LIB
        tmp = CUDA_LIB + f".tmp{os.getpid()}"
        cmd = [_nvcc(), "-shared", "-o", tmp] + objs + ["-cudart", "static", "-lpthread", "-ldl", "-lrt"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
        os.replace(tmp, CUDA_LIB)       # a process that dlopen()s concurrently sees the old or the new file, never half
        if verbose:
            sys.stderr.write(f"[tf_yarn_b200.build] linked {CUDA_LIB}\n")
        return CUDA_LIB


def build_kv(verbose: bool = False) -> str:
    """Compile the C++ KV rendezvous server (host only)."""
    src = os.path.join(KV_DIR, "kv_server.cpp")
    if os.path.exists(KV_LIB) and os.path.getmtime(KV_LIB) >= os.path.getmtime(src):
        return KV_LIB
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        raise RuntimeError("g++ not found")
    tmp = KV_LIB + f".tmp{os.getpid()}"
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", src, "-o", tmp]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"g++ failed for kv_server.cpp:\n{res.stdout}\n{res.stderr}")
    os.replace(tmp, KV_LIB)
    if verbose:
        sys.stderr.write(f"[tf_yarn_b200.build] built {KV_LIB}\n")
    return KV_LIB


def build_all(verbose: bool = True, require_cuda: bool = True) -> None:
    """Build everything.  ``require_cuda=False`` (CPU CI): without nvcc only the host-side KV server is built."""
    build_kv(verbose)
    if not require_cuda and not have_nvcc():
        if verbose:
            sys.stderr.write("[tf_yarn_b200.build] nvcc not found: CUDA libraries skipped\n")
        return
    build_cuda(verbose)


def sass_dump(out_dir: str) -> None:
    """Write cuobjdump -sass of the CUDA library (evidence for profiles/)."""
    os.makedirs(out_dir, exist_ok=True)
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump")
    res = subprocess.run([cuobjdump, "-sass", CUDA_LIB], capture_output=True, text=True)
    with open(os.path.join(out_dir, "libtfy_b200.sass"), "w") as f:
        f.write(res.stdout)


if __name__ == "__main__":
    build_all(verbose=True)
