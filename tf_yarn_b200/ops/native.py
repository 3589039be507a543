"""ctypes bindings of ``libtfy_b200.so`` (the sm_90a kernel library).

The library is built in-tree by :mod:`tf_yarn_b200.ops.build`.  On a machine
with a GPU a missing/unloadable library is a hard error: the kernels ARE the
product, there is no silent eager fallback.
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional

from tf_yarn_b200.ops import build

MAX_RANKS = 16
MAX_BLOCKS = 1024
FLAGS_BYTES = MAX_BLOCKS * MAX_RANKS * 4

BF16, F32 = 0, 1
ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS = 0, 1, 2
OPT_SGD, OPT_ADADELTA, OPT_ADAM, OPT_ADAGRAD, OPT_FTRL, OPT_RMSPROP, OPT_ADAMAX, OPT_NADAM = range(8)
MODE_LOCAL, MODE_P2P, MODE_NVLS = 0, 1, 2


class CommCtx(ctypes.Structure):
    _fields_ = [
        ("peer_base", ctypes.c_uint64 * MAX_RANKS),
        ("mc_base", ctypes.c_uint64),
        ("epoch", ctypes.c_void_p),
        ("rank", ctypes.c_int32),
        ("world", ctypes.c_int32),
    ]


class OptHyper(ctypes.Structure):
    _fields_ = [
        ("lr", ctypes.c_float),
        ("p1", ctypes.c_float),
        ("p2", ctypes.c_float),
        ("eps", ctypes.c_float),
        ("weight_decay", ctypes.c_float),
        ("grad_scale", ctypes.c_float),
        ("step", ctypes.c_int32),
        ("flags", ctypes.c_int32),
        ("done", ctypes.c_uint32),
        ("pad", ctypes.c_uint32),
    ]


LR_MAX_BOUNDARIES = 16
OPT_LR_SCHEDULE = 0x100          # or-ed into a fused step's opt code: hp heads a HyperBlock whose schedule it evaluates
LR_CONSTANT, LR_EXPONENTIAL, LR_PIECEWISE, LR_POLYNOMIAL, LR_INVERSE_TIME, LR_COSINE, LR_COSINE_RESTARTS = range(7)


class LrSchedule(ctypes.Structure):
    """Mirror of TfyLrSchedule (ops/csrc/tfy_lr_schedule.cuh)."""
    _fields_ = [
        ("kind", ctypes.c_int32),
        ("flags", ctypes.c_int32),
        ("n_boundaries", ctypes.c_int32),
        ("pad", ctypes.c_int32),
        ("initial_lr", ctypes.c_double),
        ("decay_steps", ctypes.c_double),
        ("decay_rate", ctypes.c_double),
        ("end_lr", ctypes.c_double),
        ("power", ctypes.c_double),
        ("alpha", ctypes.c_double),
        ("warmup_target", ctypes.c_double),
        ("warmup_steps", ctypes.c_double),
        ("t_mul", ctypes.c_double),
        ("m_mul", ctypes.c_double),
        ("boundaries", ctypes.c_double * LR_MAX_BOUNDARIES),
        ("values", ctypes.c_float * (LR_MAX_BOUNDARIES + 1)),
        ("pad2", ctypes.c_int32),
    ]


class HyperBlock(ctypes.Structure):
    """Mirror of TfyHyperBlock (ops/csrc/tfy_common.cuh): the device-resident hyper-parameters of a fused optimizer,
    followed by its learning-rate schedule (read only by a step launched with ``OPT_LR_SCHEDULE``)."""
    _fields_ = [
        ("hp", OptHyper),
        ("sched", LrSchedule),
    ]


class NadamHyperBlock(ctypes.Structure):
    """Mirror of TfyNadamHyperBlock (ops/csrc/tfy_common.cuh): a HyperBlock followed by Nadam's running product
    ``mu_product`` of its momentum schedule (float64, 1 before the first update), which the fused step advances."""
    _fields_ = [
        ("hp", OptHyper),
        ("sched", LrSchedule),
        ("mu_product", ctypes.c_double),
    ]


class OverlapStep(ctypes.Structure):
    """Mirror of TfyOverlapStep (ops/csrc/tfy_fused_step.cuh): a fused gradient-exchange / optimizer step that the
    communication CTAs of a persistent compute kernel run next to the compute."""
    _fields_ = [
        ("c", CommCtx),
        ("grad_off", ctypes.c_uint64),
        ("param_off", ctypes.c_uint64),
        ("shard_n", ctypes.c_size_t),
        ("master", ctypes.c_void_p),
        ("s1", ctypes.c_void_p),
        ("s2", ctypes.c_void_p),
        ("hp", ctypes.c_void_p),
        ("g0", ctypes.c_size_t),
        ("g1", ctypes.c_size_t),
        ("opt", ctypes.c_int32),
        ("mode", ctypes.c_int32),
        ("n_cta", ctypes.c_int32),
        ("slot0", ctypes.c_int32),
    ]


_lib: Optional[ctypes.CDLL] = None
_lock = threading.Lock()


def _declare(lib: ctypes.CDLL) -> None:
    vp, i, u64, sz, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_size_t, ctypes.c_float
    ctxp = ctypes.POINTER(CommCtx)
    lib.tfy_symm_last_error.restype = ctypes.c_char_p
    lib.tfy_symm_open.restype = vp
    lib.tfy_symm_open.argtypes = [i, i, i, sz, ctypes.c_char_p]
    lib.tfy_symm_exchange.argtypes = [vp, i]
    lib.tfy_symm_mc_supported.argtypes = [vp]
    lib.tfy_symm_mc_create.argtypes = [vp, i]
    lib.tfy_symm_mc_bind.argtypes = [vp]
    lib.tfy_symm_peer_ptr.restype = u64
    lib.tfy_symm_peer_ptr.argtypes = [vp, i]
    lib.tfy_symm_mc_ptr.restype = u64
    lib.tfy_symm_mc_ptr.argtypes = [vp]
    lib.tfy_symm_size.restype = u64
    lib.tfy_symm_size.argtypes = [vp]
    lib.tfy_symm_close.argtypes = [vp]
    lib.tfy_symm_close.restype = None

    lib.tfy_barrier.argtypes = [ctxp, i, vp]
    if hasattr(lib, "tfy_lr_schedule_sync"):
        lib.tfy_lr_schedule_sync.argtypes = [vp, vp]
    lib.tfy_allreduce.argtypes = [ctxp, i, i, u64, sz, f, vp, i, i, vp]
    lib.tfy_broadcast.argtypes = [ctxp, u64, sz, i, i, i, i, vp]
    lib.tfy_allgather.argtypes = [ctxp, u64, sz, i, i, vp]
    lib.tfy_fused_step.argtypes = [ctxp, i, i, i, i, u64, u64, sz, vp, vp, vp, vp, i, i, i, vp]
    if hasattr(lib, "tfy_fused_step_range"):
        lib.tfy_fused_step_range.argtypes = [ctxp, i, i, i, i, u64, u64, sz, vp, vp, vp, vp, i, i, i, sz, sz, i, vp]
    if hasattr(lib, "tfy_fused_step_shard_range"):
        lib.tfy_fused_step_shard_range.argtypes = [ctxp, i, i, i, i, u64, u64, sz, vp, vp, vp, vp, i, i, i, sz, sz, i,
                                                   vp]
    for name, (args, restype) in _EXTRA_DECLS.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.argtypes = args
            fn.restype = restype


# filled by other op modules (loss kernels, GEMM, PS) before the first load()
_EXTRA_DECLS = {}


def declare(name: str, argtypes, restype=ctypes.c_int) -> None:
    _EXTRA_DECLS[name] = (argtypes, restype)
    if _lib is not None and hasattr(_lib, name):
        getattr(_lib, name).argtypes = argtypes
        getattr(_lib, name).restype = restype


def load() -> ctypes.CDLL:
    """Load (building if necessary) the kernel library."""
    global _lib
    with _lock:
        if _lib is None:
            path = build.CUDA_LIB
            if not os.path.exists(path) or os.environ.get("TFY_REBUILD") == "1":
                path = build.build_cuda(verbose=False)
            lib = ctypes.CDLL(path)
            _declare(lib)
            _lib = lib
        return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        detail = ""
        if _lib is not None:
            detail = _lib.tfy_symm_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed with code {rc} {detail}")
