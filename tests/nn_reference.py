"""float64 reference of the fast path's general-shape layer kernels (ops/csrc/tfy_nn.cu, the C_in = 1 kernels of
ops/csrc/tfy_conv.cu).

Plain NumPy.  Inputs are taken as given (bf16 tensors already rounded), every op is computed in float64, and each
function follows the contract the kernel comments state:

* C_in = 1 conv forward: ``y = relu(sum_t x[.., tap t] w[o, t] + b[o])``; the tensor-core kernel rounds x to bf16 first
  (``round_x``).
* C_in = 1 conv weight gradient: ``dW[o, t] = sum over pixels of x[pixel + tap t] dz[pixel, o]`` and (tensor-core
  kernel) ``db = colsum(dz)``.
* bias + activation + dropout over a row-major [rows, C] matrix: element e is kept iff ``u(seed, step, e) >= rate``,
  kept values are scaled by 1/(1-rate), and the mask byte is 1 iff the ReLU passed AND the element was kept.  The
  _f32 variant sums its split-K slabs in slab order before the bias.
* gated backward: ``dz = dy * gate * scale``, the gate from the mask bytes or from ``y > 0`` (or none), and
  ``dbias = colsum(dz)``.
* 2x2 max-pool forward: ``p = dropout(relu(max over the window of z + b))``; the argmax is the FIRST maximum in the
  (dy, dx) order 00, 01, 10, 11; the dropout index is the element index of the POOLED tensor; the code byte is
  ``argmax | 4 * flows``.  Backward: the inverse scatter, and ``dbias = colsum`` of the pooled gradient.
* softmax cross-entropy: mean loss, ``dlogits = (softmax - onehot) / B``, ``dbias`` = column sums of dlogits,
  ``stats += [hits, B]`` with the argmax the first maximum.

The dropout draws come from the kernels' own generator (tfy_uniform, ops/csrc/tfy_common.cuh) built for the host from
tests/native/device_code_host.cpp (:func:`host_lib`), not from a re-implementation of the hash.
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
from typing import Optional, Tuple

import numpy as np

from ps_reference import EPS32, bf16_round  # noqa: F401  (re-exported for the tests)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"
U_BF16 = 2.0 ** -8          # unit roundoff of bf16 (8 significant bits, round to nearest)


def host_lib(out_dir: str) -> Optional[ctypes.CDLL]:
    """Host build of tests/native/device_code_host.cpp (tfy_host_uniform & co.) in out_dir; None without g++ or the
    CUDA headers."""
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        return None
    out = os.path.join(out_dir, "libnnref_host.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "device_code_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(res.stderr[-3000:])
    lib = ctypes.CDLL(out)
    lib.tfy_host_uniform.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_uniform.restype = None
    return lib


def uniform(lib, seed: int, step: int, n: int, idx0: int = 0) -> np.ndarray:
    """u(seed, step, idx0 + i) for i < n, as the kernels draw it (float32 multiples of 2^-24, returned as float64)."""
    out = np.empty(n, np.float32)
    lib.tfy_host_uniform(seed, step, idx0, out.ctypes.data, n)
    return out.astype(np.float64)


def keep(u: Optional[np.ndarray], rate: float, n: int) -> np.ndarray:
    """Keep decisions of n elements: u >= rate (all kept when rate == 0)."""
    if rate <= 0.0 or u is None:
        return np.ones(n, bool)
    return u[:n] >= rate


# ---------------------------------------------------------------------------------------------- C_in = 1 convolution
def taps(x: np.ndarray) -> np.ndarray:
    """x [B, H, W] -> the 3x3 windows [B, H-2, W-2, 9] (tap t = 3 kh + kw)."""
    B, H, W = x.shape
    return np.stack([x[:, kh:kh + H - 2, kw:kw + W - 2] for kh in range(3) for kw in range(3)], axis=-1)


def conv_c1_fwd(x, w, b, round_x: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """x [B, H, W], w [O, 9], b [O] -> (y = relu(conv + b) [B, H-2, W-2, O], sum of |terms| per output)."""
    x = bf16_round(x) if round_x else np.asarray(x, np.float64)
    t = taps(x)
    w = np.asarray(w, np.float64)
    b = np.asarray(b, np.float64)
    z = t @ w.T + b
    mag = np.abs(t) @ np.abs(w).T + np.abs(b)
    return np.maximum(z, 0.0), mag


def conv_c1_wgrad(x, dz, round_x: bool = False):
    """x [B, H, W], dz [B, H-2, W-2, O] -> (dW [O, 9], db [O], sum|x dz| [O, 9], sum|dz| [O])."""
    x = bf16_round(x) if round_x else np.asarray(x, np.float64)
    t = taps(x).reshape(-1, 9)
    d = np.asarray(dz, np.float64).reshape(t.shape[0], -1)
    return d.T @ t, d.sum(0), np.abs(d).T @ np.abs(t), np.abs(d).sum(0)


# ---------------------------------------------------------------------------------------------- bias / act / dropout
def bias_act_drop_fwd(z, bias, relu: bool, rate: float, u: Optional[np.ndarray]):
    """z [rows, C] (or the sum of the split-K slabs), bias [C] or None -> (y, mask bytes, pre-activation v)."""
    v = np.asarray(z, np.float64) + (0.0 if bias is None else np.asarray(bias, np.float64))
    on = v > 0.0 if relu else np.ones(v.shape, bool)
    a = np.where(on, v, 0.0) if relu else v
    k = keep(u, rate, v.size).reshape(v.shape)
    scale = 1.0 / (1.0 - rate) if rate > 0 else 1.0
    y = np.where(k, a * scale, 0.0)
    return y, (on & k).astype(np.uint8), v


def sum_slabs(slabs) -> Tuple[np.ndarray, np.ndarray]:
    """The _f32 variant's input: (sum over slabs in slab order, sum of |slab values|)."""
    s = np.asarray(slabs, np.float64)
    return s.sum(0), np.abs(s).sum(0)


def act_drop_bwd_bias(dy, gate: Optional[np.ndarray], scale: float):
    """dy [rows, C]; gate [rows, C] bool (mask bit, or y > 0) or None -> (dz, dbias, sum|dz| per column)."""
    dy = np.asarray(dy, np.float64)
    dz = dy if gate is None else np.where(gate, dy * scale, 0.0)
    return dz, dz.sum(0), np.abs(dz).sum(0)


# ---------------------------------------------------------------------------------------------- 2x2 max-pool
def pool_fwd(z, bias, rate: float, u: Optional[np.ndarray]):
    """z [B, H, W, C], bias [C] -> (p [B, H/2, W/2, C], code bytes, pooled maxima of z)."""
    z = np.asarray(z, np.float64)
    B, H, W, C = z.shape
    win = np.stack([z[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)], axis=0)      # [4, B, PH, PW, C]
    arg = np.argmax(win, axis=0)                                                       # first maximum
    best = np.take_along_axis(win, arg[None], 0)[0]
    v = best + np.asarray(bias, np.float64)
    on = v > 0.0
    k = keep(u, rate, v.size).reshape(v.shape)
    scale = 1.0 / (1.0 - rate) if rate > 0 else 1.0
    p = np.where(on & k, v * scale, 0.0)
    return p, (arg | (4 * (on & k))).astype(np.uint8), best


def pool_bwd(dp, code, scale: float):
    """dp, code [B, PH, PW, C] -> (dz [B, 2 PH, 2 PW, C], dbias [C], sum|dz| per column)."""
    dp = np.asarray(dp, np.float64)
    code = np.asarray(code)
    d = np.where(code & 4, dp * scale, 0.0)
    arg = code & 3
    B, PH, PW, C = dp.shape
    dz = np.zeros((B, 2 * PH, 2 * PW, C))
    for pos in range(4):
        dz[:, pos >> 1::2, pos & 1::2] = np.where(arg == pos, d, 0.0)
    return dz, d.reshape(-1, C).sum(0), np.abs(d).reshape(-1, C).sum(0)


# ---------------------------------------------------------------------------------------------- softmax head
def softmax_xent(logits, bias, labels):
    """logits [B, C], bias [C] or None, labels [B] -> (mean loss, dlogits, dbias, hits, per-row losses, logits+b)."""
    v = np.asarray(logits, np.float64) + (0.0 if bias is None else np.asarray(bias, np.float64))
    B, C = v.shape
    labels = np.asarray(labels, np.int64)
    mx = v.max(1, keepdims=True)
    e = np.exp(v - mx)
    se = e.sum(1, keepdims=True)
    p = e / se
    rows = np.arange(B)
    l = (mx[:, 0] + np.log(se[:, 0])) - v[rows, labels]
    onehot = np.zeros_like(v)
    onehot[rows, labels] = 1.0
    d = (p - onehot) / B
    hits = int((np.argmax(v, 1) == labels).sum())
    return l.mean(), d, d.sum(0), hits, l, v
