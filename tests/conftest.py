import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("TFY_POLL_EVERY_SECS", "0.2")
# The CPU tests work on tiny tensors: one intra-op thread is faster than eight and, above all, immune to the
# OpenMP spin-barrier collapse on a contended / oversubscribed box (a 64-element embedding_bag took 27 ms with 8
# threads under load).  Child processes (launcher tasks, torchrun) inherit the setting.
if not os.path.exists("/dev/nvidia0"):          # (GPU boxes keep their threads for the fp32 reference computations)
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    os.environ.setdefault("MKL_NUM_THREADS", "1")


def pytest_configure(config):
    try:
        import torch
        if not torch.cuda.is_available():
            torch.set_num_threads(1)
    except Exception:  # noqa: BLE001
        pass
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `pytest -m gpu`)")
    config.addinivalue_line("markers", "slow: multi-process integration test")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no GPU in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _native_libraries_built():
    """Build the in-tree native libraries ONCE, before any test spawns worker processes: in a fresh checkout
    every child would otherwise start its own nvcc build (and multi-process tests would time out)."""
    from tf_yarn_b200.ops import build
    try:
        # without nvcc (CPU-only CI runners) only the KV server is built; gpu-marked tests are skipped anyway
        build.build_all(verbose=False, require_cuda=False)
    except RuntimeError as exc:
        import warnings
        warnings.warn(f"native build incomplete: {exc}")
    yield
