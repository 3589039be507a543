"""Symmetric HBM arena: one VMM allocation per rank, mapped on every rank.

``SymmArena`` drives the four-step handshake implemented in
``ops/csrc/tfy_symm.cpp`` (allocate+listen, swap fds, create multicast, bind)
with barriers through a :class:`Rendezvous` -- the launcher's KV store when a
job runs under ``run_on_yarn``, or a ``torch.distributed`` store when the ranks
were started by ``torchrun``.

Allocation inside the arena is a deterministic bump allocator: every rank
performs the same sequence of ``alloc`` calls (SPMD), hence every buffer has
the same offset on every rank and a peer address is ``peer_base[r] + offset``.
The first ``FLAGS_BYTES`` of the arena are the signal pad of the device-side
barrier.
"""
from __future__ import annotations

import ctypes
import os
import tempfile
import uuid
from typing import Optional, Sequence

import torch

from tf_yarn_b200.ops import native


# ---------------------------------------------------------------------------
# rendezvous
# ---------------------------------------------------------------------------
class Rendezvous:
    """Minimal host-side rendezvous: blocking get, set, barrier."""

    rank: int
    world: int

    def set(self, key: str, value: bytes) -> None:
        raise NotImplementedError

    def get(self, key: str) -> bytes:
        raise NotImplementedError

    def barrier(self, name: str) -> None:
        self.set(f"{name}/{self.rank}", b"1")
        for r in range(self.world):
            self.get(f"{name}/{r}")


class KVRendezvous(Rendezvous):
    """Rendezvous over the launcher's KV store (no torch.distributed involved)."""

    def __init__(self, kv, rank: int, world: int, prefix: str = "symm"):
        self.kv, self.rank, self.world, self.prefix = kv, rank, world, prefix

    def set(self, key: str, value: bytes) -> None:
        self.kv.put(f"{self.prefix}/{key}", value)

    def get(self, key: str) -> bytes:
        return self.kv.wait(f"{self.prefix}/{key}")


class StoreRendezvous(Rendezvous):
    """Rendezvous over a c10d Store (torchrun-started jobs, e.g. bench.py)."""

    def __init__(self, store, rank: int, world: int, prefix: str = "tfy_symm"):
        self.store, self.rank, self.world, self.prefix = store, rank, world, prefix

    def set(self, key: str, value: bytes) -> None:
        self.store.set(f"{self.prefix}/{key}", value)

    def get(self, key: str) -> bytes:
        return self.store.get(f"{self.prefix}/{key}")


class SoloRendezvous(Rendezvous):
    def __init__(self):
        self.rank, self.world, self._d = 0, 1, {}

    def set(self, key, value):
        self._d[key] = value

    def get(self, key):
        return self._d[key]


def default_rendezvous(prefix: str = "tfy_symm") -> Rendezvous:
    """Pick the rendezvous of the current process: launcher KV, else torch.distributed, else solo."""
    import torch.distributed as dist
    from tf_yarn_b200 import kv as kvmod
    if os.environ.get(kvmod.KV_ADDR_ENV) and os.environ.get("TFY_RANK") is not None:
        client = kvmod.KVClient()
        return KVRendezvous(client, int(os.environ["TFY_RANK"]), int(os.environ["TFY_WORLD_SIZE"]),
                            prefix=f"{prefix}/{os.environ.get('TFY_N_TRY', '0')}")
    if dist.is_available() and dist.is_initialized():
        store = dist.distributed_c10d._get_default_store()
        return StoreRendezvous(store, dist.get_rank(), dist.get_world_size(), prefix)
    return SoloRendezvous()


# ---------------------------------------------------------------------------
# arena
# ---------------------------------------------------------------------------
class _RawCudaMemory:
    """Expose a raw device range through __cuda_array_interface__ (zero copy)."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self._owner = owner
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None,
        }


class SymmArena:
    _seq = 0

    def __init__(self, size_bytes: int, device: Optional[int] = None, rdv: Optional[Rendezvous] = None,
                 timeout_s: float = 120.0):
        if not torch.cuda.is_available():
            raise RuntimeError("SymmArena needs a CUDA device (H100)")
        self.lib = native.load()
        self.rdv = rdv if rdv is not None else default_rendezvous()
        self.rank, self.world = self.rdv.rank, self.rdv.world
        self.device = torch.cuda.current_device() if device is None else device
        torch.cuda.set_device(self.device)
        torch.cuda.init()
        seq = SymmArena._seq
        SymmArena._seq += 1
        self._tag = f"arena{seq}"
        # socket prefix agreed through rank 0
        if self.rank == 0:
            prefix = os.path.join(tempfile.gettempdir(), f"tfy_symm_{uuid.uuid4().hex[:12]}")
            self.rdv.set(f"{self._tag}/sock", prefix.encode())
        prefix = self.rdv.get(f"{self._tag}/sock").decode() if self.world > 1 else "/tmp/tfy_symm_solo"
        total = native.FLAGS_BYTES + int(size_bytes)
        self._h = self.lib.tfy_symm_open(self.device, self.rank, self.world, total, prefix.encode())
        if not self._h:
            raise RuntimeError("tfy_symm_open: " + self.lib.tfy_symm_last_error().decode())
        tmo = int(timeout_s * 1000)
        self.multicast = False
        dbg = os.environ.get("TFY_SYMM_DEBUG") == "1"

        def trace(msg):
            if dbg:
                print(f"[symm rank {self.rank}] {msg}", flush=True)
        trace("arena allocated, listening")
        if self.world > 1:
            self.rdv.barrier(f"{self._tag}/listening")
            trace("exchanging memory handles")
            native.check(self.lib.tfy_symm_exchange(self._h, tmo), "tfy_symm_exchange")
            self.rdv.barrier(f"{self._tag}/exchanged")
            trace("peers mapped; multicast setup")
            # two ranks on ONE physical GPU (a ps sharing the chief's device on a small box) cannot both join a
            # multicast object: fall back to plain peer mappings, which work within a device as well
            try:
                me = str(torch.cuda.get_device_properties(self.device).uuid)
            except Exception:  # noqa: BLE001
                me = f"dev{self.device}"
            self.rdv.set(f"{self._tag}/dev/{self.rank}", me.encode())
            devs = [self.rdv.get(f"{self._tag}/dev/{r}") for r in range(self.world)]
            shared_device = len(set(devs)) < self.world
            if os.environ.get("TFY_DISABLE_NVLS") == "1" or shared_device:
                rc = 1
            else:
                rc = self.lib.tfy_symm_mc_create(self._h, tmo)
                if rc < 0:
                    native.check(rc, "tfy_symm_mc_create")
            # all ranks must agree (rank 0 failing implies everyone got rc=1)
            self.rdv.set(f"{self._tag}/mc/{self.rank}", str(rc).encode())
            ok = all(self.rdv.get(f"{self._tag}/mc/{r}") == b"0" for r in range(self.world))
            if ok:
                rc = self.lib.tfy_symm_mc_bind(self._h)
                self.rdv.set(f"{self._tag}/mcb/{self.rank}", str(rc).encode())
                ok = all(self.rdv.get(f"{self._tag}/mcb/{r}") == b"0" for r in range(self.world))
                self.multicast = bool(ok)
            self.rdv.barrier(f"{self._tag}/ready")
            trace(f"ready, multicast={self.multicast}")
        self.size = int(self.lib.tfy_symm_size(self._h))
        self.peer_base = [int(self.lib.tfy_symm_peer_ptr(self._h, r)) for r in range(self.world)]
        self.mc_base = int(self.lib.tfy_symm_mc_ptr(self._h)) if self.multicast else 0
        self.base = self.peer_base[self.rank]
        self._bump = native.FLAGS_BYTES
        self._mem = torch.as_tensor(_RawCudaMemory(self.base, self.size, self), device=f"cuda:{self.device}")
        self.epoch = torch.zeros(native.MAX_BLOCKS * native.MAX_RANKS, dtype=torch.int32,
                                 device=f"cuda:{self.device}")
        self.ctx = native.CommCtx()
        for r in range(self.world):
            self.ctx.peer_base[r] = self.peer_base[r]
        self.ctx.mc_base = self.mc_base
        self.ctx.epoch = self.epoch.data_ptr()
        self.ctx.rank = self.rank
        self.ctx.world = self.world
        self.ctx_ref = ctypes.byref(self.ctx)

    # -- symmetric allocation ------------------------------------------------
    def alloc(self, nbytes: int, align: int = 256) -> int:
        off = (self._bump + align - 1) // align * align
        if off + nbytes > self.size:
            raise MemoryError(f"symmetric arena exhausted: need {nbytes} at {off}, size {self.size}")
        self._bump = off + nbytes
        return off

    def tensor(self, offset: int, shape: Sequence[int], dtype: torch.dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        return self._mem[offset:offset + nbytes].view(dtype).view(*shape)

    def empty(self, shape: Sequence[int], dtype: torch.dtype, align: int = 256):
        n = 1
        for s in shape:
            n *= int(s)
        off = self.alloc(n * torch.empty((), dtype=dtype).element_size(), align)
        return off, self.tensor(off, shape, dtype)

    def offset_of(self, t: torch.Tensor) -> int:
        off = t.data_ptr() - self.base
        if off < 0 or off >= self.size:
            raise ValueError("tensor does not live in this symmetric arena")
        return off

    def close(self) -> None:
        if getattr(self, "_h", None):
            torch.cuda.synchronize(self.device)
            self.lib.tfy_symm_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
