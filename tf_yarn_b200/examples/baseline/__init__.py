"""The BASELINE.json configurations as runnable examples (not in the reference tree: they exercise its three
training paths -- Horovod all-reduce, parameter server, torch DDP -- at realistic sizes).

Every example runs at full size on a H100 box and at toy size on a CPU-only box (``EXAMPLE_SMALL=1`` forces the toy
size); all data is synthetic (no network).
"""
import os

import torch


def small() -> bool:
    return os.environ.get("EXAMPLE_SMALL", "0" if torch.cuda.is_available() else "1") == "1"


def n_trainers(default: int = 8) -> int:
    """One trainer per GPU (at most ``default``); two processes on a CPU-only box."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return max(1, min(default, n)) if n else 2
