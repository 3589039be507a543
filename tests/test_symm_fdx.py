"""Host-side test of the POSIX-fd exchange used to share VMM allocations between ranks.

Runs the real C++ code path (connect / SCM_RIGHTS / accept ordering) with several
processes and no GPU: every rank sends to all peers BEFORE accepting, which must not
deadlock (a first version waited for an ack and hung on the H100 box).
"""
import multiprocessing as mp
import os
import tempfile
import uuid

import pytest


def _worker(rank, world, prefix, q):
    from tf_yarn_b200.ops import native
    lib = native.load()
    import ctypes
    lib.tfy_fdx_selftest.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    rc = lib.tfy_fdx_selftest(rank, world, prefix.encode(), 20000)
    q.put((rank, rc, lib.tfy_symm_last_error().decode()))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_fd_exchange_all_to_all(world):
    from tf_yarn_b200.ops import native
    native.load()            # build once here: in a fresh checkout the children would all compile (and time out)
    ctx = mp.get_context("spawn")
    prefix = os.path.join(tempfile.gettempdir(), f"tfy_fdx_{uuid.uuid4().hex[:8]}")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, prefix, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=60) for _ in range(world)]
    for p in procs:
        p.join(30)
    assert sorted(r for r, _, _ in results) == list(range(world))
    assert all(rc == 0 for _, rc, _ in results), results
