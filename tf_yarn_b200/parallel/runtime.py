"""Process-wide communication runtime (one Communicator per process == per GPU)."""
from __future__ import annotations

import os
import threading
from typing import Optional

_lock = threading.Lock()
_comm = None


def get_communicator(rdv=None, device: Optional[int] = None):
    """The process's :class:`Communicator`, created on first use.

    Sizes: ``TFY_ARENA_MB`` (default 2048) of symmetric HBM for flat parameter /
    gradient buffers, ``TFY_FUSION_MB`` (default 64) for the Horovod-style fusion
    buffer.  H100 has 80 GB of HBM3; the defaults fit BERT-base fp32 grads
    (440 MB) with room to spare.
    """
    global _comm
    with _lock:
        if _comm is None:
            from tf_yarn_b200.parallel.comm import Communicator
            arena_mb = int(os.environ.get("TFY_ARENA_MB", "2048"))
            fusion_mb = int(os.environ.get("TFY_FUSION_MB", "64"))
            _comm = Communicator(arena_bytes=arena_mb << 20, fusion_bytes=fusion_mb << 20, rdv=rdv, device=device)
        return _comm


def set_communicator(comm) -> None:
    global _comm
    with _lock:
        _comm = comm


def shutdown() -> None:
    global _comm
    with _lock:
        if _comm is not None:
            _comm.close()
            _comm = None
