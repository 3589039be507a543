"""The summation order of the conv2 weight gradient's per-CTA partials (ops/csrc/tfy_conv_index.cuh: c_wg_slice),
built for the host and checked against a re-enactment of the rule the weight-gradient kernel's own reduction has
always followed.  The deferred reduction in the data-gradient kernel calls the same function, so its dW / db are
the same bits as the in-kernel reduction's only if this rule is kept exactly."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"

WG_THREADS = 672                   # threads of the weight-gradient CTA
TOTAL4 = (64 * 9 * 32 + 64) // 4   # float4 outputs: the dW tile, then db


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("wgorder") / "libwgorder.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "conv_order_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_wg_slice.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p]
    lib.tfy_host_wg_slice.restype = None
    return lib


def c_grid(n_patches, sms=132):
    """Compute CTAs of the persistent conv2 kernels (tfy_conv.cu: c_grid)."""
    if n_patches <= sms:
        return n_patches
    waves = -(-n_patches // sms)
    return -(-n_patches // waves)


def reference_rule(n_cmp, owner):
    per = -(-TOTAL4 // n_cmp)
    lo = owner * per
    hi = min(lo + per, TOTAL4)
    length = max(hi - lo, 0)
    parts = WG_THREADS // length if length > 0 and 2 * length <= WG_THREADS else 1
    return lo, length, parts, per


# n_cmp of batches 2, 32, 128, 160 and 232 on 132 SMs (9 * B / 2 patches of 8 x 8 pixel pairs), plus the extremes
N_CMP = sorted({c_grid(9 * b // 2) for b in (2, 32, 128, 160, 232)} | {1, 13, 14, 132, 160})


def test_batches_give_the_expected_partial_counts():
    assert [c_grid(9 * b // 2) for b in (2, 32, 128, 160, 232)] == [9, 72, 116, 120, 131]


@pytest.mark.parametrize("n_cmp", N_CMP)
def test_slice_and_parts_follow_the_reference_rule(lib, n_cmp):
    out = (ctypes.c_int * 4)()
    covered = np.zeros(TOTAL4, dtype=np.int32)
    for owner in range(n_cmp):
        lib.tfy_host_wg_slice(TOTAL4, n_cmp, owner, WG_THREADS, out)
        assert tuple(out) == reference_rule(n_cmp, owner), (n_cmp, owner)
        covered[out[0]:out[0] + out[1]] += 1
    assert (covered == 1).all()          # every output has exactly one owner, so exactly one order
