"""The update formulas of the fused K4 kernel (ops/csrc/tfy_fused_step.cuh: tfy_step_consts + tfy_opt_update_rt), built
for the host and checked against torch.optim on the CPU -- through the framework's own chain: mini-Keras optimizer
-> OptimizerSpec (hyper-parameter packing) -> TfyOptHyper (device struct) -> per-element update, with exact
sqrt / rsqrt / division in place of the SFU approximations.  It covers every optimizer, AdamW, Nesterov momentum,
weight decay and the 1/world gradient scaling, on every box.  On an H100, test_gpu_fused_step.py runs the kernel itself
for all six optimizers, every (gradient, parameter) dtype pair, ranged and split launches, the MNIST-CNN's size, the
U=2 multi-GPU instantiations at world 1 and the overlap role, against the float64 reference of
fused_step_reference.py."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.ops import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("optmath") / "liboptmath.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "device_code_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_opt_step.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
    lib.tfy_host_opt_step.restype = None
    return lib


CASES = {
    "sgd": keras.optimizers.SGD(0.1),
    "sgd_momentum": keras.optimizers.SGD(0.05, momentum=0.9),
    "sgd_nesterov_wd": keras.optimizers.SGD(0.05, momentum=0.9, nesterov=True, weight_decay=0.01),
    "adadelta": keras.optimizers.Adadelta(1.0),
    "adam": keras.optimizers.Adam(0.01),
    "adam_l2": keras.optimizers.Adam(0.01, weight_decay=0.1),
    "adamw": keras.optimizers.AdamW(0.01, weight_decay=0.1),
    "adagrad": keras.optimizers.Adagrad(0.1),
    "ftrl": keras.optimizers.Ftrl(0.1, l1_regularization_strength=0.002, l2_regularization_strength=0.001, beta=0.1),
}


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("world", [1, 4])
def test_kernel_update_matches_torch_optim(lib, name, world):
    desc = CASES[name]
    spec = desc.to_spec()
    n = 257
    g = torch.Generator().manual_seed(11)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = desc.to_torch([ref])
    # the device-side state, initialised the way FusedShardedOptimizer does
    p = p0.clone().contiguous()
    s1 = torch.full((n,), spec.init_s1)
    s2 = torch.zeros(n)
    hyper = native.OptHyper(spec.lr, spec.p1, spec.p2, spec.eps, spec.weight_decay, 1.0, 0, spec.flags, 0, 0)
    for step in range(7):
        grad = torch.randn(n, generator=g) * (0.5 + 0.2 * step)
        # the kernel receives the SUM over ranks and scales by 1/world: feed it world x the averaged gradient
        summed = (grad * world).contiguous()
        lib.tfy_host_opt_step(spec.code, ctypes.byref(hyper), world, p.data_ptr(), summed.data_ptr(), s1.data_ptr(),
                              s2.data_ptr(), n)
        ref.grad = grad.clone()
        opt.step()
    assert hyper.step == 7                                   # the device step counter drives Adam's bias correction
    err = (p - ref.detach()).abs().max().item()
    assert err < 5e-6 * max(1.0, ref.detach().abs().max().item()), (name, err)
    if name == "ftrl":
        assert int((p == 0).sum()) == int((ref.detach() == 0).sum())      # L1 zeroes exactly the same coordinates


def test_dropout_generator_is_uniform_stateless_and_step_dependent(lib):
    """tfy_uniform(seed, step, index) (ops/csrc/tfy_common.cuh): the forward draws a mask, the backward kernels re-derive
    it from the same (seed, step, index) -- so it must be a pure function -- and a replayed CUDA graph must draw a new
    mask every step because the step is read from device memory."""
    lib.tfy_host_uniform.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_uniform.restype = None

    def draw(seed, step, idx0, n=200_000):
        out = torch.empty(n)
        lib.tfy_host_uniform(seed, step, idx0, out.data_ptr(), n)
        return out
    u = draw(1234, 0, 0)
    assert 0.0 <= float(u.min()) and float(u.max()) < 1.0
    assert abs(float(u.mean()) - 0.5) < 0.005 and abs(float(u.var()) - 1 / 12) < 0.002
    hist = torch.histc(u, bins=20, min=0, max=1) / u.numel()
    assert float((hist - 0.05).abs().max()) < 0.003                                   # flat
    for rate in (0.25, 0.5):
        assert abs(float((u >= rate).float().mean()) - (1 - rate)) < 0.005           # keep probability of the kernels
    assert torch.equal(u, draw(1234, 0, 0))                                           # pure function of its arguments
    assert torch.equal(u[1000:2000], draw(1234, 0, 1000, 1000))                       # indexable anywhere (tiles, re-draws)
    for other in (draw(1234, 1, 0), draw(1235, 0, 0)):                                # new step / new seed: new mask
        assert abs(float(((u >= 0.5) == (other >= 0.5)).float().mean()) - 0.5) < 0.01
        assert abs(float(torch.corrcoef(torch.stack([u, other]))[0, 1])) < 0.01
    lag = torch.corrcoef(torch.stack([u[:-1], u[1:]]))[0, 1]                          # neighbours are uncorrelated
    assert abs(float(lag)) < 0.01
    big = draw(7, 3, (1 << 32) - 500, 1000)                                           # 64-bit indices do not wrap into repeats
    assert not torch.equal(big[:500], big[500:])


def test_bf16_pack_rounds_to_nearest_even_like_torch(lib):
    """TfyPack<bf16>::pack / unpack: the fp32 master -> bf16 parameter store of the fused step (and every bf16 epilogue)."""
    lib.tfy_host_bf16_roundtrip.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_bf16_roundtrip.restype = None
    g = torch.Generator().manual_seed(5)
    x = torch.cat([torch.randn(4096, generator=g) * 10 ** torch.randint(-6, 6, (4096,), generator=g).float(),
                   torch.tensor([0.0, -0.0, 1.0, 1.00390625, 1.01171875, 3.3895314e38, 1e-40, -1e-40])])   # ties, huge, denormal
    x = x[: x.numel() // 8 * 8].contiguous()
    out = torch.empty_like(x)
    lib.tfy_host_bf16_roundtrip(x.data_ptr(), out.data_ptr(), x.numel() // 8)
    ref = x.bfloat16().float()
    same = (out == ref) | (out.isnan() & ref.isnan())
    assert bool(same.all()), (x[~same][:5], out[~same][:5], ref[~same][:5])


@pytest.mark.parametrize("tiles_x,tiles_y,pairs,n_cta", [(3, 3, 64, 144), (3, 3, 64, 148), (1, 1, 5, 3), (4, 2, 7, 5),
                                                          (3, 3, 1, 148), (2, 5, 33, 37), (3, 3, 8, 8)])
def test_persistent_conv_ctas_cover_every_patch_exactly_once(lib, tiles_x, tiles_y, pairs, n_cta):
    """CPatchIter (ops/csrc/tfy_conv_index.cuh): CTA b of n_cta walks patches b, b + n_cta, b + 2 n_cta, ... decomposed
    into (image pair, tile row, tile column) INCREMENTALLY (no division in the hot loop).  Over all CTAs every patch
    of the batch must come up exactly once, in the order the division-based decomposition gives."""
    lib.tfy_host_patch_walk.argtypes = [ctypes.c_int] * 7 + [ctypes.c_void_p]
    lib.tfy_host_patch_walk.restype = None
    tiles = tiles_x * tiles_y
    n_patches = tiles * pairs
    seen = {}
    for explicit in (0, 1):                       # default n_cta = gridDim.x, or a grid with extra (communication) CTAs
        seen.clear()
        for b in range(min(n_cta, n_patches)):
            count = (n_patches - b + n_cta - 1) // n_cta
            out = (ctypes.c_int * (3 * count))()
            grid = n_cta if not explicit else n_cta + 4
            lib.tfy_host_patch_walk(tiles_x, tiles_y, n_cta, b, grid, explicit, count, out)
            for i in range(count):
                p = b + i * n_cta
                want = (p // tiles, (p % tiles) // tiles_x, p % tiles_x)
                got = (out[3 * i], out[3 * i + 1], out[3 * i + 2])
                assert got == want, (b, i, got, want)
                assert got not in seen
                seen[got] = b
        assert len(seen) == n_patches


def test_ctypes_mirrors_match_the_c_structs(lib):
    """tf_yarn_b200/ops/native.py mirrors the structs the kernels take by value / read from device memory; a drifted
    field would silently corrupt peer addresses or hyper-parameters.  Sizes, offsets and enum values come from the real
    headers (sizeof / offsetof in a host build)."""
    import re
    from tf_yarn_b200.ops import native
    from tf_yarn_b200.parallel import optspec
    lib.tfy_host_struct_layout.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    lib.tfy_host_struct_layout.restype = ctypes.c_int

    def c_layout(which):
        buf = (ctypes.c_int * 32)()
        n = lib.tfy_host_struct_layout(which, buf, 32)
        return list(buf[:n])

    def mirror(cls):
        return [ctypes.sizeof(cls)] + [getattr(cls, name).offset for name, _ in cls._fields_]

    ctx = c_layout(0)
    assert ctx[:6] == mirror(native.CommCtx)
    assert ctx[6:] == [native.MAX_RANKS, native.MAX_BLOCKS, native.FLAGS_BYTES]
    assert c_layout(1) == mirror(native.OptHyper)
    assert c_layout(2) == mirror(native.OverlapStep)
    assert c_layout(3) == [native.BF16, native.F32, native.ALGO_ONESHOT, native.ALGO_TWOSHOT, native.ALGO_NVLS,
                           native.OPT_SGD, native.OPT_ADADELTA, native.OPT_ADAM, native.OPT_ADAGRAD, native.OPT_FTRL,
                           native.MODE_LOCAL, native.MODE_P2P, native.MODE_NVLS]
    assert (optspec.OPT_SGD, optspec.OPT_ADADELTA, optspec.OPT_ADAM, optspec.OPT_ADAGRAD, optspec.OPT_FTRL) == \
        (native.OPT_SGD, native.OPT_ADADELTA, native.OPT_ADAM, native.OPT_ADAGRAD, native.OPT_FTRL)

    # TfyPsSeg lives in a .cu file: compare field ORDER and types textually with the ctypes mirror
    from tf_yarn_b200.estimator.ps_hbm import PsSeg
    src = open(os.path.join(CSRC, "tfy_ps.cu")).read()
    body = src[src.index("struct TfyPsSeg {"):]
    body = body[: body.index("};")]
    fields = []
    for line in body.splitlines()[1:]:
        line = line.split("//")[0].strip()
        m = re.match(r"(uint64_t|int32_t|uint32_t|float)\s+([^;]+);", line)
        if m:
            fields += [(name.strip(), m.group(1)) for name in m.group(2).split(",")]
    ctype_of = {"uint64_t": ctypes.c_uint64, "int32_t": ctypes.c_int32, "uint32_t": ctypes.c_uint32, "float": ctypes.c_float}
    assert [(n, ctype_of[t]) for n, t in fields] == list(PsSeg._fields_)
