"""Keras gradient accumulation (``gradient_accumulation_steps``) on CPU: argument validation and configs; the CPU
engine against a float64 NumPy transcription of the contract (tests/fused_step_reference.py for the updates) for
every optimizer, with and without a schedule, at N = 2, 3 and 4; save -> load_model -> resume in the middle of an
accumulation; the device header built for the host (tests/native/grad_accum_host.cpp); the fast-path planner's
overlap fallback; and the Estimator's refusal."""
import ctypes
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fused_step_reference as ref  # noqa: E402

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.keras import optimizers as kopt  # noqa: E402
from tf_yarn_b200.keras import schedules  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"

ALL = (kopt.SGD, kopt.Adadelta, kopt.Adam, kopt.AdamW, kopt.Adagrad, kopt.Ftrl, kopt.RMSprop)


# ---------------------------------------------------------------------------------------------- the argument
@pytest.mark.parametrize("cls", ALL, ids=lambda c: c.__name__)
def test_every_optimizer_accepts_and_round_trips_the_argument(cls):
    opt = cls(gradient_accumulation_steps=4)
    assert opt.gradient_accumulation_steps == 4
    cfg = opt.get_config()
    assert cfg["gradient_accumulation_steps"] == 4
    again = kopt.from_config(cfg)
    assert type(again) is cls and again.get_config() == cfg
    # off: the config of every existing optimizer is what it was
    plain = cls().get_config()
    assert "gradient_accumulation_steps" not in plain and cls().gradient_accumulation_steps is None
    assert list(cls(gradient_accumulation_steps=2).get_config())[:-1] == list(plain)


@pytest.mark.parametrize("bad", [0, 1, -2, 2.0, 3.5, True, False, "4"])
@pytest.mark.parametrize("cls", ALL, ids=lambda c: c.__name__)
def test_invalid_values_raise_value_error_naming_the_argument(cls, bad):
    with pytest.raises(ValueError, match="gradient_accumulation_steps"):
        cls(gradient_accumulation_steps=bad)


def test_get_compile_and_distributed_wrapper_keep_the_argument():
    assert kopt.get("adam").gradient_accumulation_steps is None
    from tf_yarn_b200 import hvd
    inner = kopt.RMSprop(gradient_accumulation_steps=3)
    assert kopt.get(hvd.DistributedOptimizer(inner)).gradient_accumulation_steps == 3
    m = _model(kopt.Adam(1e-3, gradient_accumulation_steps=2))
    m2 = _model(kopt.from_config(m.optimizer.get_config()))
    assert m2.optimizer.gradient_accumulation_steps == 2


# ---------------------------------------------------------------------------------------------- the CPU engine
def _model(opt, seed=0):
    torch.manual_seed(seed)
    m = keras.Sequential([keras.layers.Dense(3, input_shape=(8,))])
    m.compile(optimizer=opt, loss="mse")
    return m


def _data(n=96):
    rs = np.random.RandomState(1)
    x = rs.randn(n, 8).astype("float32")
    y = rs.randn(n, 3).astype("float32")
    return torch.from_numpy(x), torch.from_numpy(y)


class _Record(keras.callbacks.Callback):
    def __init__(self):
        super().__init__()
        self.after = []

    def on_train_batch_end(self, batch, logs=None):
        self.after.append([p.detach().clone() for p in self.model.net.parameters()])


# name -> (descriptor factory, reference kind, Hyper fields, initial s1)
CASES = {
    "sgd": (lambda **k: kopt.SGD(0.05, **k), "sgd", dict(lr=0.05), 0.0),
    "sgd_momentum": (lambda **k: kopt.SGD(0.05, momentum=0.9, **k), "sgd", dict(lr=0.05, p1=0.9), 0.0),
    "sgd_nesterov": (lambda **k: kopt.SGD(0.05, momentum=0.9, nesterov=True, **k), "sgd",
                     dict(lr=0.05, p1=0.9, flags=1), 0.0),
    "adadelta": (lambda **k: kopt.Adadelta(1.0, **k), "adadelta", dict(lr=1.0, p1=0.95, eps=1e-7), 0.0),
    "adam": (lambda **k: kopt.Adam(0.01, **k), "adam", dict(lr=0.01, p1=0.9, p2=0.999, eps=1e-7), 0.0),
    "adamw": (lambda **k: kopt.AdamW(0.01, weight_decay=0.05, **k), "adam",
              dict(lr=0.01, p1=0.9, p2=0.999, eps=1e-7, wd=0.05, flags=1), 0.0),
    "adagrad": (lambda **k: kopt.Adagrad(0.05, **k), "adagrad", dict(lr=0.05, eps=1e-7), 0.1),
    "ftrl": (lambda **k: kopt.Ftrl(0.1, l1_regularization_strength=0.01, l2_regularization_strength=0.001, beta=0.1,
                                   **k), "ftrl", dict(lr=0.1, p1=0.01, p2=0.001, eps=0.1), 0.1),
    "rmsprop": (lambda **k: kopt.RMSprop(0.01, **k), "rmsprop", dict(lr=0.01, p1=0.9, eps=1e-7), 0.0),
    "rmsprop_centered_momentum": (lambda **k: kopt.RMSprop(0.01, momentum=0.5, centered=True, **k), "rmsprop",
                                  dict(lr=0.01, p1=0.9, p2=0.5, eps=1e-7, flags=1), 0.0),
}
SCHEDULE = schedules.PiecewiseConstantDecay([2, 5, 8], [1.0, 0.5, 0.25, 0.125])     # a factor on the base rate


def _mse_grads(params, x, y):
    """float64 gradients of Keras' mean squared error of a Dense layer: mean over the batch and the outputs."""
    w, b = params
    d = 2.0 * (x @ w.T + b - y) / y.size
    return [d.T @ x, d.sum(0)]


def transcription(case, n_steps, x, y, p0, batch, schedule=None, lr_at=None, adam_t=None):
    """The contract, batch by batch, in float64: the weights after every batch, and the update batches.
    ``lr_at`` / ``adam_t`` replace the batch index at which the schedule / Adam's bias correction are read."""
    _, kind, fields, init = CASES[case]
    params = [np.asarray(p, np.float64) for p in p0]
    s1 = [np.full_like(p, init) for p in params]
    s2 = [np.zeros_like(p) for p in params]
    s3 = [np.zeros_like(p) for p in params]
    acc = [np.zeros_like(p) for p in params]
    after, updates = [], []
    for s in range(len(x) // batch):
        xb, yb = np.asarray(x[s * batch:(s + 1) * batch], np.float64), np.asarray(y[s * batch:(s + 1) * batch],
                                                                                 np.float64)
        acc = [a + g for a, g in zip(acc, _mse_grads(params, xb, yb))]
        if (s + 1) % n_steps == 0:
            k = len(updates)
            at = lr_at(s, k) if lr_at else s
            lr = fields["lr"] * float(schedule(at)) if schedule is not None else fields["lr"]
            h = ref.Hyper(**{**fields, "lr": lr, "grad_scale": 1.0 / n_steps})
            t = adam_t(s, k) if adam_t else s
            out = [ref.step(kind, p, a, a1, a2, a3, h, t) for p, a, a1, a2, a3 in zip(params, acc, s1, s2, s3)]
            params, s1, s2, s3 = [list(z) for z in zip(*out)]
            acc = [np.zeros_like(p) for p in params]
            updates.append(s)
        after.append([p.copy() for p in params])
    return after, updates


def _run(case, n_steps, schedule=None, epochs=1):
    make = CASES[case][0]
    base = CASES[case][2]["lr"]
    lr = schedules.PiecewiseConstantDecay(schedule.boundaries, [base * v for v in schedule.values]) \
        if schedule is not None else base
    opt = make(gradient_accumulation_steps=n_steps)
    if schedule is not None:
        opt._learning_rate = lr
    m = _model(opt)
    m.build((8,))
    p0 = [p.detach().clone() for p in m.net.parameters()]
    rec = _Record()
    x, y = _data()
    m.fit(x, y, batch_size=8, epochs=epochs, shuffle=False, verbose=0, callbacks=[rec])
    return m, p0, rec.after, x, y


@pytest.mark.parametrize("n_steps", [2, 3, 4])
@pytest.mark.parametrize("case", sorted(CASES))
def test_cpu_engine_follows_the_contract(case, n_steps):
    m, p0, after, x, y = _run(case, n_steps)
    want, updates = transcription(case, n_steps, x.numpy(), y.numpy(), [p.numpy() for p in p0], 8)
    assert updates == [s for s in range(12) if s % n_steps == n_steps - 1]
    assert m._engine.iterations == 12
    prev = p0
    for s, (got, exp) in enumerate(zip(after, want)):
        changed = any(not torch.equal(a, b) for a, b in zip(got, prev))
        assert changed == (s in updates), s                       # the weights move on batches kN - 1 only
        for a, b in zip(got, exp):
            np.testing.assert_allclose(a.numpy(), b, rtol=2e-5, atol=2e-6, err_msg=f"batch {s}")
        prev = got


@pytest.mark.parametrize("n_steps", [2, 3, 4])
@pytest.mark.parametrize("case", ["sgd_momentum", "adam", "rmsprop_centered_momentum"])
def test_cpu_engine_reads_the_schedule_and_adams_step_at_the_batch_index(case, n_steps):
    m, p0, after, x, y = _run(case, n_steps, SCHEDULE)
    args = (case, n_steps, x.numpy(), y.numpy(), [p.numpy() for p in p0], 8, SCHEDULE)
    want, _ = transcription(*args)
    for a, b in zip(after[-1], want[-1]):
        np.testing.assert_allclose(a.numpy(), b, rtol=2e-5, atol=2e-6)
    assert m.get_learning_rate() == pytest.approx(CASES[case][2]["lr"] * float(SCHEDULE(12)))
    # the transcription tells the alternatives apart: a schedule read at the update count ...
    by_update, _ = transcription(*args, lr_at=lambda s, k: k)
    assert not np.allclose(by_update[-1][0], want[-1][0], rtol=1e-4, atol=0)
    if CASES[case][1] == "adam":            # ... and Adam's bias correction at the update count
        by_update, _ = transcription(*args, adam_t=lambda s, k: k)
        assert not np.allclose(by_update[-1][0], want[-1][0], rtol=1e-4, atol=0)


@pytest.mark.parametrize("case", ["sgd_momentum", "sgd_nesterov"])
def test_sgd_momentums_first_step_branch_gives_the_same_update(case):
    """The fused step treats a step counter of 0 as SGD's first step (the buffer starts as the gradient).  Counting
    batches, the first update of an accumulation sees N - 1 instead: with Keras' zero dampening and a zero initial
    buffer, both branches give the same values."""
    _, kind, fields, _ = CASES[case]
    rs = np.random.RandomState(3)
    p, g = rs.randn(64), rs.randn(64)
    h = ref.Hyper(**{**fields, "grad_scale": 0.25})
    z = np.zeros(64)
    first = ref.step(kind, p, g, z, z, z, h, 0)
    later = ref.step(kind, p, g, z, z, z, h, 3)
    for a, b in zip(first, later):
        np.testing.assert_array_equal(a, b)


def test_save_load_model_resume_in_the_middle_of_an_accumulation_is_bit_identical(tmp_path):
    x, y = _data()
    make = lambda: kopt.Adam(schedules.ExponentialDecay(0.01, 4, 0.8), gradient_accumulation_steps=5)  # noqa: E731
    straight = _model(make())
    straight.fit(x, y, batch_size=8, epochs=2, shuffle=False, verbose=0)         # 24 batches, 4 updates
    first = _model(make())
    first.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0)            # 12 batches: 2 pending
    assert first._engine.iterations == 12
    path = str(tmp_path / "m.tfy")
    first.save(path)
    loaded = keras.models.load_model(path)
    assert loaded.optimizer.gradient_accumulation_steps == 5
    loaded.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0)
    assert loaded._engine.iterations == 24
    for a, b in zip(loaded.net.parameters(), straight.net.parameters()):
        assert torch.equal(a.detach(), b.detach())
    # the pending sum is part of the state only while an accumulation is open
    assert "grad_accum" in first._engine.state_dict()
    first.fit(x[:24], y[:24], batch_size=8, epochs=1, shuffle=False, verbose=0)   # batches 12..14: update at 14
    assert "grad_accum" not in first._engine.state_dict()


@pytest.mark.parametrize("before", ["plain", "accumulating"])
def test_a_recompiled_accumulating_fit_starts_from_a_zero_sum(before):
    """.grad holds the last batch's gradients after a plain fit, and the pending sum after an accumulating one; a new
    accumulating optimizer must not fold either into its first update."""
    x, y = _data()
    m = _model(kopt.SGD(0.1, gradient_accumulation_steps=3 if before == "accumulating" else None))
    m.fit(x[:32], y[:32], batch_size=8, epochs=1, shuffle=False, verbose=0)          # 4 batches (1 pending at N=3)
    assert any(p.grad is not None and float(p.grad.abs().max()) > 0 for p in m.net.parameters())
    fresh = _model(kopt.SGD(0.1, gradient_accumulation_steps=2))
    fresh.build((8,))
    fresh.net.load_state_dict(m.net.state_dict())
    m.compile(optimizer=kopt.SGD(0.1, gradient_accumulation_steps=2), loss="mse")
    for mm in (m, fresh):
        mm.fit(x[32:48], y[32:48], batch_size=8, epochs=1, shuffle=False, verbose=0)  # 2 batches: one update
    for a, b in zip(m.net.parameters(), fresh.net.parameters()):
        assert torch.equal(a.detach(), b.detach())


# ---------------------------------------------------------------------------------------------- the device header
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("gradaccum") / "libgradaccum.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "grad_accum_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_grad_accumulate.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t]
    lib.tfy_host_grad_accumulate.restype = None
    lib.tfy_host_batch_advance.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    lib.tfy_host_batch_advance.restype = None
    return lib


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_host_build_sums_in_fp32_in_batch_order(lib, dtype):
    g = torch.Generator().manual_seed(5)
    n = 4096 + 8
    acc = torch.zeros(n, dtype=torch.float32)
    want = torch.zeros(n, dtype=torch.float32)
    for _ in range(4):
        src = (torch.randn(n, generator=g) * 10.0 ** torch.randint(-3, 3, (n,), generator=g)).to(dtype)
        lib.tfy_host_grad_accumulate(acc.data_ptr(), src.data_ptr(), int(dtype == torch.bfloat16), n)
        want = want + src.float()
    assert torch.equal(acc, want)


@pytest.mark.parametrize("n_steps", [2, 3, 4])
def test_host_build_advances_the_counter_and_the_scheduled_rate_once_per_batch(lib, n_steps):
    from tf_yarn_b200.parallel.comm import hyper_block
    sch = schedules.ExponentialDecay(0.1, 3, 0.5)
    spec = kopt.SGD(sch).to_spec()
    blk = hyper_block(spec)
    from tf_yarn_b200.ops import native
    assert ctypes.sizeof(blk) == ctypes.sizeof(native.HyperBlock)
    read = []
    for s in range(4 * n_steps):
        assert blk.hp.step == s
        update = (s + 1) % n_steps == 0
        if update:
            read.append((s, blk.hp.lr))         # the rate the fused step of batch s reads
        lib.tfy_host_batch_advance(ctypes.byref(blk), 1, int(update))
    assert blk.hp.step == 4 * n_steps
    for s, lr in read:
        assert lr == pytest.approx(float(sch(s)), rel=3e-7)
    assert [s for s, _ in read] == [k * n_steps - 1 for k in range(1, 5)]
    const = hyper_block(kopt.SGD(0.1).to_spec())
    for s in range(2 * n_steps):
        lib.tfy_host_batch_advance(ctypes.byref(const), 0, int((s + 1) % n_steps == 0))
    assert const.hp.step == 2 * n_steps and const.hp.lr == pytest.approx(0.1)


# ---------------------------------------------------------------------------------------------- fast-path planner
def test_fast_path_planner_falls_back_from_overlap_when_accumulating():
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"the planner consulted {name} for an accumulating optimizer")

    eng = FastSequentialEngine.__new__(FastSequentialEngine)
    eng.fused = types.SimpleNamespace(zero_grads=False, param_dtype=torch.bfloat16, grad_dtype=torch.bfloat16,
                                      spec=types.SimpleNamespace(kind="adam"))
    eng.lib, eng.plan, eng.accum_steps = NoLib(), [], 4
    assert eng._overlap_desc(0, 128, 26, 26, None) is None
    # off: the planner goes on to ask the kernel library for its spare CTAs, as before
    eng.accum_steps = None
    eng.lib = types.SimpleNamespace(tfy_conv3x3_c32_wgrad_spare_ctas=lambda *a: 0)
    assert eng._overlap_desc(0, 128, 26, 26, None) is None


# ---------------------------------------------------------------------------------------------- Estimator
@pytest.mark.parametrize("where", ["optimizer", "optimizers", "distributed"])
def test_estimator_refuses_gradient_accumulation(tmp_path, where):
    from tf_yarn_b200 import hvd
    from tf_yarn_b200.estimator.estimator import Estimator
    from tf_yarn_b200.estimator.spec import EstimatorSpec

    def model_fn(features, labels, mode, params):
        acc = kopt.SGD(0.1, gradient_accumulation_steps=2)
        kw = {"optimizer": acc} if where == "optimizer" else \
            {"optimizer": "sgd", "optimizers": {"0.": acc}} if where == "optimizers" else \
            {"optimizer": hvd.DistributedOptimizer(acc)}
        return EstimatorSpec(mode=mode, network=torch.nn.Sequential(torch.nn.Linear(1, 1)),
                             loss=lambda l, o: ((o - l) ** 2).mean(), **kw)

    est = Estimator(model_fn, model_dir=str(tmp_path))
    x = torch.ones(4, 1)
    for _ in range(2):           # a second train() on the same Estimator refuses it too
        with pytest.raises(ValueError, match="gradient_accumulation_steps"):
            est.train(lambda: iter([(x, x)] * 2), steps=2)
