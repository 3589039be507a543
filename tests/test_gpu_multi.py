"""Multi-GPU tests (run with `pytest -m gpu` on a box with >= 2 H100s; skipped otherwise).

The stand-alone checks under tests/gpu/ are launched with torch.distributed.run, one process per GPU:
every collective / fused-step kernel against an fp32 PyTorch reference and against NCCL, the parameter-server
data plane end to end, and the headline bench's own cross-rank assertions (`params_in_sync`).
"""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(n, script_args, port, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", str(port)] + script_args
    return subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_comm_kernels_multi_gpu(tmp_path):
    n = min(_ngpu(), 8)
    res = _torchrun(n, ["tests/gpu/comm_check.py", "--quick"], 29611)
    assert res.returncode == 0, res.stdout[-4000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("SUMMARY")][-1]
    assert "failed=0" in line, res.stdout[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_headline_bench_ranks_stay_in_sync():
    n = min(_ngpu(), 8)
    res = _torchrun(n, ["bench.py", "--gpus", str(n), "--steps", "20", "--warmup", "3", "--repeats", "3"], 29612)
    assert res.returncode == 0, res.stdout[-4000:]
    rec = json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("{")][-1])
    assert rec["params_in_sync"] is True
    assert rec["e2e"]["loss_fell"] is True
    assert rec["gpu_launches"] > 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_ddp_wrapper_matches_torch_ddp():
    n = min(_ngpu(), 8)
    res = _torchrun(n, ["tests/gpu/ddp_check.py"], 29613)
    assert res.returncode == 0 and "DDP CHECK OK" in res.stdout, res.stdout[-4000:]
