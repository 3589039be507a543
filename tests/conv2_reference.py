"""float64 reference of the conv2 tensor-core kernels (ops/csrc/tfy_conv.cu: C_in = 32 -> C_out = 64, 3x3, VALID).

Plain NumPy, batch by batch in chunks so that B in the hundreds fits in memory.  Inputs are taken as given (bf16
tensors already rounded); every op is computed in float64 and follows the contract the kernel comments state:

* Forward (tfy_conv3x3_fprop_pool_kernel): ``z = conv3x3(a, W)``, a 2x2 max-pool, ``+ bias``, ReLU and dropout.
  - Tie rule: the kernel replaces the two low mantissa bits of each fp32 value of the window by its position
    dy * 2 + dx and takes fmaxf.  Among EQUAL maxima the last position therefore wins when the maximum is positive
    (or +0) and the first when it is negative.  This is not the first-maximum rule of the general pool kernel
    (nn_reference.pool_fwd).
  - Dropout: pooled element e (flat NHWC index) is kept iff byte e & 3 of the raw hash of group e >> 2 is >= thr
    (:func:`keep_from_hash`, hashes from the host build of the kernel's own hash), and kept values are scaled by
    256 / (256 - thr) (the host build of c_keep_scale).
  - Code byte: ``argmax | 4 * (v > 0 and kept)`` with ``v`` = pooled max + bias.
* Data gradient: ``dx[b, y, x, c] = sum_{kh, kw, o} dz[b, y - kh, x - kw, o] W[o, kh, kw, c]``, zeroed where a gate is
  given and ``gate <= 0``.
* Un-pool (the operand producers of the fused backward kernels): ``g = dp * scale`` in fp32 where the code byte's
  gate bit is set, else 0; the dz operand is ``g`` rounded to bf16 at the argmax position of the window; db sums the
  fp32 ``g`` themselves.
* Weight gradient: ``dW[o, kh, kw, c] = sum_{b, y, x} dz[b, y, x, o] a[b, y + kh, x + kw, c]`` and ``db = sum g``.

Every function also returns ``sum |terms|`` per output, the scale of its fp32 rounding error.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Optional

import numpy as np

from ps_reference import bf16_round

CHUNK = 32                  # images per float64 block


def host_hash_u32(lib, seed: int, step: int, n: int, idx0: int = 0) -> np.ndarray:
    """Raw 32-bit dropout hashes of element groups idx0 .. idx0 + n - 1 (host build of the forward's own hash)."""
    out = np.empty(n, np.uint32)
    lib.tfy_host_hash_u32(seed, step, idx0, out.ctypes.data, n)
    return out


def host_keep_scale(lib, rates) -> tuple:
    """(thr, keep scale) of each rate from the host build of c_drop_thr / c_keep_scale (fp32 rates)."""
    r = np.ascontiguousarray(rates, np.float32)
    thr = np.empty(r.size, np.uint32)
    scale = np.empty(r.size, np.float32)
    lib.tfy_host_keep_scale(r.ctypes.data, thr.ctypes.data, scale.ctypes.data, r.size)
    return thr, scale


def declare_host(lib: ctypes.CDLL) -> ctypes.CDLL:
    lib.tfy_host_hash_u32.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_hash_u32.restype = None
    lib.tfy_host_keep_scale.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_keep_scale.restype = None
    return lib


def keep_from_hash(hashes: np.ndarray, thr: int, n: int) -> np.ndarray:
    """Keep decision of pooled elements 0 .. n - 1: byte e & 3 of hashes[e >> 2] >= thr."""
    e = np.arange(n, dtype=np.int64)
    byte = (hashes[e >> 2].astype(np.uint64) >> (8 * (e & 3)).astype(np.uint64)) & 0xFF
    return byte >= thr


# ---------------------------------------------------------------------------------------------- convolution
def conv(a, w):
    """a [B, H, W, 32], w [64, 3, 3, 32] -> (z [B, H-2, W-2, 64], sum|a w| per output)."""
    a = np.asarray(a, np.float64)
    w = np.asarray(w, np.float64)
    B, H, W, _ = a.shape
    O = w.shape[0]
    z = np.zeros((B, H - 2, W - 2, O))
    mag = np.zeros_like(z)
    for b0 in range(0, B, CHUNK):
        ac = a[b0:b0 + CHUNK]
        for kh in range(3):
            for kw in range(3):
                x = ac[:, kh:kh + H - 2, kw:kw + W - 2]
                z[b0:b0 + CHUNK] += x @ w[:, kh, kw, :].T
                mag[b0:b0 + CHUNK] += np.abs(x) @ np.abs(w[:, kh, kw, :]).T
    return z, mag


def pool_argmax(win: np.ndarray) -> np.ndarray:
    """win [4, ...] (window positions dy * 2 + dx) -> argmax position with the forward kernel's tie rule: among equal
    maxima the last position for a maximum >= 0, the first for a negative one."""
    mx = win.max(0)
    is_max = win == mx[None]
    first = np.argmax(is_max, 0)
    last = 3 - np.argmax(is_max[::-1], 0)
    return np.where(mx >= 0, last, first)


class Fwd(NamedTuple):
    p: np.ndarray           # pooled output [B, PH, PW, 64]
    code: np.ndarray        # code bytes (uint8)
    mag: np.ndarray         # sum|terms| of the pooled value (the largest of the window's), + |bias|
    v: np.ndarray           # pooled maximum + bias (what ReLU tests)
    best: np.ndarray        # pooled maximum of z
    gap: np.ndarray         # top value minus the runner-up of the window (0 for a tie)
    win_mag: np.ndarray     # largest sum|terms| in the window


def fwd(a, w, bias, keep: Optional[np.ndarray] = None, keep_scale: float = 1.0) -> Fwd:
    """Forward of tfy_conv3x3_c32_pool_fwd; keep: [B, PH, PW, 64] bool (None: nothing dropped)."""
    z, mag = conv(a, w)
    win = np.stack([z[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)], 0)
    wmag = np.stack([mag[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)], 0).max(0)
    arg = pool_argmax(win)
    best = np.take_along_axis(win, arg[None], 0)[0]
    srt = np.sort(win, 0)
    gap = srt[3] - srt[2]
    b = np.asarray(bias, np.float64)
    v = best + b
    on = v > 0.0
    if keep is not None:
        on = on & keep.reshape(v.shape)
    p = np.where(on, v * keep_scale, 0.0)
    code = (arg | (4 * on)).astype(np.uint8)
    return Fwd(p, code, wmag + np.abs(b), v, best, gap, wmag)


# ---------------------------------------------------------------------------------------------- backward
def unpool(dp, code, scale: float):
    """dp, code [B, PH, PW, 64] -> (dz operand [B, 2 PH, 2 PW, 64], g [B, PH, PW, 64]).  g = fp32(dp * scale) where the
    gate bit is set (as float64); the operand holds g rounded to bf16 at the window's argmax position."""
    dp32 = np.asarray(dp, np.float32)
    code = np.asarray(code)
    g = np.where(code & 4, dp32 * np.float32(scale), np.float32(0.0)).astype(np.float64)
    gq = bf16_round(g)
    B, PH, PW, C = g.shape
    dz = np.zeros((B, 2 * PH, 2 * PW, C))
    arg = code & 3
    for pos in range(4):
        dz[:, pos >> 1::2, pos & 1::2] = np.where(arg == pos, gq, 0.0)
    return dz, g


def unpool_exact(dp, code, scale: float) -> np.ndarray:
    """The exact adjoint of the forward's pool + dropout: dz [B, 2 PH, 2 PW, 64] = dp * scale at the gated argmax."""
    d = np.where(np.asarray(code) & 4, np.asarray(dp, np.float64) * scale, 0.0)
    B, PH, PW, C = d.shape
    dz = np.zeros((B, 2 * PH, 2 * PW, C))
    arg = np.asarray(code) & 3
    for pos in range(4):
        dz[:, pos >> 1::2, pos & 1::2] = np.where(arg == pos, d, 0.0)
    return dz


def dgrad(dz, w, gate=None):
    """dz [B, H-2, W-2, 64], w [64, 3, 3, 32], gate [B, H, W, 32] or None -> (dx [B, H, W, 32], sum|dz w|)."""
    dz = np.asarray(dz, np.float64)
    w = np.asarray(w, np.float64)
    B, OH, OW, O = dz.shape
    H, W = OH + 2, OW + 2
    C = w.shape[3]
    dx = np.zeros((B, H, W, C))
    mag = np.zeros_like(dx)
    for b0 in range(0, B, CHUNK):
        dzp = np.zeros((min(CHUNK, B - b0), H + 2, W + 2, O))
        dzp[:, 2:2 + OH, 2:2 + OW] = dz[b0:b0 + CHUNK]
        for kh in range(3):
            for kw in range(3):
                x = dzp[:, 2 - kh:2 - kh + H, 2 - kw:2 - kw + W]
                dx[b0:b0 + CHUNK] += x @ w[:, kh, kw, :]
                mag[b0:b0 + CHUNK] += np.abs(x) @ np.abs(w[:, kh, kw, :])
    if gate is not None:
        dx = np.where(np.asarray(gate) > 0, dx, 0.0)
    return dx, mag


def wgrad(a, dz):
    """a [B, H, W, 32], dz [B, H-2, W-2, 64] -> (dW [64, 3, 3, 32], sum|dz a|)."""
    a = np.asarray(a, np.float64)
    dz = np.asarray(dz, np.float64)
    B, OH, OW, O = dz.shape
    C = a.shape[3]
    dw = np.zeros((O, 3, 3, C))
    mag = np.zeros_like(dw)
    for b0 in range(0, B, CHUNK):
        d = dz[b0:b0 + CHUNK].reshape(-1, O)
        for kh in range(3):
            for kw in range(3):
                x = a[b0:b0 + CHUNK, kh:kh + OH, kw:kw + OW].reshape(-1, C)
                dw[:, kh, kw] += d.T @ x
                mag[:, kh, kw] += np.abs(d).T @ np.abs(x)
    return dw, mag


def bias_grad(g):
    """g [B, PH, PW, 64] (the gated, scaled pooled gradient) -> (db [64], sum|g|)."""
    g = np.asarray(g, np.float64).reshape(-1, np.shape(g)[-1])
    return g.sum(0), np.abs(g).sum(0)
