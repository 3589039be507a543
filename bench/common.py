"""Shared measurement harness of bench.py (all arms, all configs).

Timing rules implemented here:

* the clock sampler (NVML, 2 ms period) is started on EVERY rank BEFORE the barrier that precedes the
  timed region, so no rank enters the region late because of NVML initialisation;
* a timed region is exactly ``steps`` steps between two CUDA events on the launching stream; it is
  preceded by a host barrier + ``cuda.synchronize()``, a device-side cross-GPU barrier and ONE untimed step
  (so the skew of leaving the host barrier is absorbed outside the region), and followed by a synchronize;
* a short region (the driver's ``--steps 20`` is ~2 ms) is repeated ``repeats`` times and the MEDIAN region
  is reported; each region is first reduced with MAX over ranks.  ``steps`` in the JSON stays the number of
  steps of ONE region, ``repeats`` is printed next to it.
"""
from __future__ import annotations

import json
import os
import threading
import time
from typing import Callable, List, Optional


class ClockSampler:
    """Samples SM clock + throttle reasons through NVML on a thread while the timed regions run."""

    REASONS = {
        "hw_slowdown": 0x0000000000000008, "sw_power_cap": 0x0000000000000004,
        "hw_thermal_slowdown": 0x0000000000000040, "sw_thermal_slowdown": 0x0000000000000020,
        "hw_power_brake_slowdown": 0x0000000000000080,
    }

    def __init__(self, gpu_index: int, period_s: float = 0.002):
        self.gpu, self.period = gpu_index, period_s
        self.samples: List[float] = []
        self.reasons = set()
        self.max_mhz = None
        self._stop = threading.Event()
        self._armed = threading.Event()
        self._t = None
        self._h = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self._nv = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(self._physical_index(gpu_index))
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM))
        except Exception:  # noqa: BLE001
            self._h = None

    @staticmethod
    def _physical_index(logical: int) -> int:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        ids = [v for v in vis.split(",") if v.strip() != ""]
        if ids and logical < len(ids) and ids[logical].strip().isdigit():
            return int(ids[logical])
        return logical

    def start(self):
        """Start the sampling thread (NVML is already initialised by the constructor)."""
        if self._h is None:
            return
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def arm(self, on: bool = True):
        """Only samples taken while armed (= inside a timed region) are kept."""
        (self._armed.set if on else self._armed.clear)()

    def _run(self):
        nv = self._nv
        while not self._stop.is_set():
            if self._armed.is_set():
                try:
                    mhz = float(nv.nvmlDeviceGetClockInfo(self._h, nv.NVML_CLOCK_SM))
                    mask = nv.nvmlDeviceGetCurrentClocksEventReasons(self._h)
                    if self._armed.is_set():
                        self.samples.append(mhz)
                        for name, bit in self.REASONS.items():
                            if mask & bit:
                                self.reasons.add(name)
                except Exception:  # noqa: BLE001
                    pass
            self._stop.wait(self.period)

    def stop(self):
        if self._h is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvml unavailable"], "samples": 0}
        self._stop.set()
        if self._t is not None:
            self._t.join(2)
        sm = sorted(self.samples)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": self.max_mhz,
                "reasons": sorted(self.reasons), "samples": len(sm)}


def dist_env():
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)),
            int(os.environ.get("WORLD_SIZE", 1)))


def quiet_nccl():
    """NCCL_DEBUG=VERSION/INFO makes NCCL print on stdout, in front of the JSON line."""
    if os.environ.get("NCCL_DEBUG", "").upper() in ("VERSION", "INFO"):
        os.environ["NCCL_DEBUG"] = "WARN"


def host_barrier(world: int):
    import torch
    import torch.distributed as dist
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def max_over_ranks(values: List[float], world: int) -> List[float]:
    import torch
    import torch.distributed as dist
    if world == 1:
        return list(values)
    t = torch.tensor(values, device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(v) for v in t.tolist()]


def pick_repeats(steps: int, requested: int = 0) -> int:
    """Number of timed regions of ``steps`` steps: one unless more are requested (the median is reported)."""
    return requested if requested > 0 else 1


def dump_outputs(out_dir: str, arrays) -> None:
    """Write each tensor of ``arrays`` (name -> tensor) as ``out_dir/<name>.npy`` in float32."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"),
                t.detach().float().reshape(-1).cpu().numpy().astype(np.float32))


def median(vals: List[float]) -> float:
    s = sorted(vals)
    n = len(s)
    return s[n // 2] if n % 2 else 0.5 * (s[n // 2 - 1] + s[n // 2])


def timed_regions(world: int, steps: int, repeats: int, run_steps: Callable[[int], None],
                  device_barrier: Optional[Callable[[], None]] = None, stream=None,
                  sampler: Optional[ClockSampler] = None) -> List[float]:
    """Device-timed regions of exactly ``steps`` steps; returns the per-region ms, MAX over ranks.

    ``run_steps(n)`` enqueues n steps on ``stream`` (the current stream when None);
    ``device_barrier()`` enqueues a cross-GPU barrier kernel on the same stream (None for arms whose step
    already contains a blocking collective: one untimed step then plays that role).
    """
    import torch
    ms = []
    for _ in range(repeats):
        host_barrier(world)
        st = stream if stream is not None else torch.cuda.current_stream()
        if device_barrier is not None:
            device_barrier()
        run_steps(1)                       # untimed: absorbs the skew of leaving the host barrier
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if sampler is not None:
            sampler.arm(True)
        start.record(st)
        run_steps(steps)
        end.record(st)
        end.synchronize()
        if sampler is not None:
            sampler.arm(False)
        torch.cuda.synchronize()
        ms.append(start.elapsed_time(end))
    return max_over_ranks(ms, world)


def wall_regions(world: int, repeats: int, run_region: Callable[[], None]) -> List[float]:
    """End-to-end (wall clock) regions: barrier + synchronize on both sides, MAX over ranks."""
    import torch
    ms = []
    for _ in range(repeats):
        host_barrier(world)
        t0 = time.perf_counter()
        run_region()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    host_barrier(world)
    return max_over_ranks(ms, world)


def tensor_checksum(t) -> List[int]:
    """Exact integer checksums of a tensor's bytes (two moments, so permutations are caught as well)."""
    import torch
    v = t.detach().contiguous().view(torch.uint8).to(torch.int64)
    idx = torch.arange(v.numel(), device=v.device, dtype=torch.int64) % 8191 + 1
    return [int(v.sum().item()), int((v * idx).sum().item())]


def all_ranks_equal(vals: List[int], world: int) -> bool:
    import torch
    import torch.distributed as dist
    if world == 1:
        return True
    mine = torch.tensor(vals, device="cuda", dtype=torch.int64)
    got = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(got, mine)
    return all(bool((g == got[0]).all().item()) for g in got)


def emit(obj: dict):
    print(json.dumps(obj), flush=True)
