"""Keras learning-rate schedules on CPU: every schedule, and the device function built for the host
(tests/native/lr_schedule_host.cpp), against an independent float64 NumPy reference (tests/lr_schedule_reference.py);
argument validation; configs; optimizers driven by a schedule (config round trips, save -> load_model -> resume,
the TypeError of LearningRateScheduler / set_learning_rate); the CPU engine against torch.optim driven step by step by
the reference rate; the fused-step hyper block; an estimator with a schedule on the shared-memory parameter server;
and the HBM parameter server's refusal."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import lr_schedule_reference as ref  # noqa: E402

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.keras import schedules  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"
# float32 rounding of a float64 value, plus the last bits of transcendental functions: 2 ulp of float32 relative,
# and an absolute floor of 1e-7 of the initial rate for rates that decay to zero
RTOL, ATOL_REL = 2.5e-7, 1e-7

BIG = 10 ** 7


def _cases():
    """(name, schedule, reference function, steps to check)."""
    S = schedules
    out = []

    def add(name, sch, fn, extra):
        steps = sorted({0, 1, 2, BIG - 1, BIG, *[s for s in extra if s >= 0]})
        out.append((name, sch, fn, steps))

    for stair in (False, True):
        add(f"exponential_stair{int(stair)}", S.ExponentialDecay(0.1, 100, 0.96, staircase=stair),
            lambda s, st=stair: ref.exponential(s, 0.1, 100, 0.96, st), [99, 100, 101, 199, 200, 201, 12345])
        add(f"inverse_time_stair{int(stair)}", S.InverseTimeDecay(0.5, 30, 0.7, staircase=stair),
            lambda s, st=stair: ref.inverse_time(s, 0.5, 30, 0.7, st), [29, 30, 31, 59, 60, 61, 999])
    bounds, vals = [10, 50, 100, 1000], [1.0, 0.5, 0.1, 0.05, 0.001]
    add("piecewise", S.PiecewiseConstantDecay(bounds, vals), lambda s: ref.piecewise(s, bounds, vals),
        [b + d for b in bounds for d in (-1, 0, 1)])
    b16 = [10 * (i + 1) for i in range(16)]
    v16 = [1.0 / (i + 1) for i in range(17)]
    add("piecewise16", S.PiecewiseConstantDecay(b16, v16), lambda s: ref.piecewise(s, b16, v16),
        [b + d for b in b16 for d in (-1, 0, 1)])
    for cycle in (False, True):
        for power in (1.0, 0.5, 2.0):
            add(f"polynomial_p{power}_cycle{int(cycle)}",
                S.PolynomialDecay(0.1, 200, end_learning_rate=0.001, power=power, cycle=cycle),
                lambda s, c=cycle, p=power: ref.polynomial(s, 0.1, 200, 0.001, p, c),
                [199, 200, 201, 399, 400, 401, 555])
    add("cosine", S.CosineDecay(0.1, 1000, alpha=0.05), lambda s: ref.cosine(s, 0.1, 1000, 0.05),
        [499, 500, 501, 999, 1000, 1001])
    add("cosine_warmup", S.CosineDecay(0.0, 1000, alpha=0.0, warmup_target=0.2, warmup_steps=100),
        lambda s: ref.cosine(s, 0.0, 1000, 0.0, 0.2, 100), [99, 100, 101, 1099, 1100, 1101, 600])
    add("cosine_warmup_from_nonzero", S.CosineDecay(0.01, 500, alpha=0.1, warmup_target=0.1, warmup_steps=37),
        lambda s: ref.cosine(s, 0.01, 500, 0.1, 0.1, 37), [36, 37, 38, 536, 537, 538])
    restarts = [9, 10, 11, 29, 30, 31, 69, 70, 71, 149, 150, 151, 12345]
    add("restarts_t2", S.CosineDecayRestarts(0.1, 10, t_mul=2.0, m_mul=0.9, alpha=0.01),
        lambda s: ref.cosine_restarts(s, 0.1, 10, 2.0, 0.9, 0.01), restarts)
    add("restarts_t1", S.CosineDecayRestarts(0.1, 10, t_mul=1.0, m_mul=0.5),
        lambda s: ref.cosine_restarts(s, 0.1, 10, 1.0, 0.5), restarts)
    add("restarts_t1.5", S.CosineDecayRestarts(0.05, 8, t_mul=1.5, m_mul=1.0, alpha=0.0),
        lambda s: ref.cosine_restarts(s, 0.05, 8, 1.5, 1.0, 0.0), [7, 8, 9, 19, 20, 21, 37, 38, 39, 64, 65, 66])
    return out


CASES = _cases()


def _close(got, want, initial):
    got, want = float(got), float(np.float32(want))
    return abs(got - want) <= RTOL * abs(want) + ATOL_REL * abs(initial)


def _initial(sch):
    cfg = sch.get_config()
    return max(abs(cfg.get("initial_learning_rate", 0.0)), abs(cfg.get("warmup_target") or 0.0),
               max(cfg.get("values", [0.0])))


@pytest.mark.parametrize("name,sch,fn,steps", CASES, ids=[c[0] for c in CASES])
def test_host_schedule_matches_the_float64_reference(name, sch, fn, steps):
    for s in steps:
        got, want = sch(s), fn(s)
        if name.startswith("piecewise"):
            assert got == float(want), (s, got, want)                    # piecewise: exact
        else:
            assert _close(got, want, _initial(sch)), (s, got, float(want))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("lrsched") / "liblrsched.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "lr_schedule_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_lr_schedule.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    lib.tfy_host_lr_schedule.restype = ctypes.c_float
    lib.tfy_host_lr_schedule_layout.argtypes = [ctypes.c_void_p, ctypes.c_int]
    return lib


def _device_struct(sch):
    from tf_yarn_b200.parallel.comm import hyper_block
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    return hyper_block(OptimizerSpec.sgd(sch)).sched


@pytest.mark.parametrize("name,sch,fn,steps", CASES, ids=[c[0] for c in CASES])
def test_host_build_of_the_device_function_matches_the_reference_and_the_python_schedule(lib, name, sch, fn, steps):
    st = _device_struct(sch)
    for s in steps:
        got = lib.tfy_host_lr_schedule(ctypes.byref(st), s)
        want = fn(s)
        if name.startswith("piecewise"):
            assert got == float(want), (s, got, want)
        else:
            assert _close(got, want, _initial(sch)), (s, got, float(want))
        # the host writes the first rate and the rate of a restored step with the Python schedule: the same float
        assert got == sch(s), (s, got, sch(s))


def test_ctypes_mirrors_match_the_schedule_structs(lib):
    buf = (ctypes.c_int * 40)()
    n = lib.tfy_host_lr_schedule_layout(buf, 40)
    got = list(buf[:n])
    cls = native.LrSchedule
    want = [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    want += [native.LR_MAX_BOUNDARIES, native.LR_EXPONENTIAL, native.LR_PIECEWISE, native.LR_POLYNOMIAL,
             native.LR_INVERSE_TIME, native.LR_COSINE, native.LR_COSINE_RESTARTS]
    want += [ctypes.sizeof(native.HyperBlock), native.HyperBlock.hp.offset, native.HyperBlock.sched.offset,
             native.OPT_LR_SCHEDULE]
    assert got == want
    assert schedules.MAX_BOUNDARIES == native.LR_MAX_BOUNDARIES
    kinds = {type(c[1]).__name__: c[1]._device_fields()["kind"] for c in CASES}
    assert kinds == {"ExponentialDecay": native.LR_EXPONENTIAL, "InverseTimeDecay": native.LR_INVERSE_TIME,
                     "PiecewiseConstantDecay": native.LR_PIECEWISE, "PolynomialDecay": native.LR_POLYNOMIAL,
                     "CosineDecay": native.LR_COSINE, "CosineDecayRestarts": native.LR_COSINE_RESTARTS}


@pytest.mark.parametrize("make,arg", [
    (lambda: schedules.ExponentialDecay(0.1, 0, 0.9), "decay_steps"),
    (lambda: schedules.ExponentialDecay(0.1, -5, 0.9), "decay_steps"),
    (lambda: schedules.InverseTimeDecay(0.1, 0, 0.5), "decay_steps"),
    (lambda: schedules.InverseTimeDecay(0.1, 10, -0.5), "decay_rate"),
    (lambda: schedules.PolynomialDecay(0.1, 0), "decay_steps"),
    (lambda: schedules.PolynomialDecay(0.1, 10, power=0), "power"),
    (lambda: schedules.CosineDecay(0.1, 0), "decay_steps"),
    (lambda: schedules.CosineDecay(0.1, 10, warmup_target=0.2, warmup_steps=-1), "warmup_steps"),
    (lambda: schedules.CosineDecayRestarts(0.1, 0), "first_decay_steps"),
    (lambda: schedules.CosineDecayRestarts(0.1, 10, t_mul=0.5), "t_mul"),
    (lambda: schedules.CosineDecayRestarts(0.1, 10, m_mul=-1.0), "m_mul"),
    (lambda: schedules.PiecewiseConstantDecay([10, 5], [1.0, 0.5, 0.1]), "boundaries"),
    (lambda: schedules.PiecewiseConstantDecay([10, 10], [1.0, 0.5, 0.1]), "boundaries"),
    (lambda: schedules.PiecewiseConstantDecay([10, 20], [1.0, 0.5]), "values"),
    (lambda: schedules.PiecewiseConstantDecay(list(range(1, 18)), [0.1] * 18), "boundaries"),
    (lambda: schedules.ExponentialDecay(float("nan"), 10, 0.9), "initial_learning_rate"),
])
def test_invalid_arguments_raise_value_error_naming_the_argument(make, arg):
    with pytest.raises(ValueError, match=f"`{arg}`"):
        make()


def test_sixteen_boundaries_are_accepted():
    s = schedules.PiecewiseConstantDecay(list(range(1, 17)), [float(i) for i in range(17)])
    assert [s(i) for i in (0, 1, 2, 16, 17)] == [0.0, 0.0, 1.0, 15.0, 16.0]


@pytest.mark.parametrize("name,sch,fn,steps", CASES[:1] + CASES[4:5] + CASES[-6:], ids=lambda x: x if isinstance(
    x, str) else "")
def test_config_round_trip(name, sch, fn, steps):
    d = schedules.serialize(sch)
    back = schedules.deserialize(d)
    assert type(back) is type(sch) and back == sch and back.get_config() == sch.get_config()
    assert type(sch).from_config(sch.get_config()) == sch
    assert [back(s) for s in steps] == [sch(s) for s in steps]
    with pytest.raises(ValueError, match="unknown learning-rate schedule"):
        schedules.deserialize({"class_name": "Nope", "config": {}})


def test_keras_optimizers_namespace_exposes_the_schedules():
    assert keras.optimizers.schedules is schedules
    for n in ("LearningRateSchedule", "ExponentialDecay", "PiecewiseConstantDecay", "PolynomialDecay",
              "InverseTimeDecay", "CosineDecay", "CosineDecayRestarts", "serialize", "deserialize"):
        assert hasattr(keras.optimizers.schedules, n)


OPTIMIZERS = ["SGD", "Adadelta", "Adam", "AdamW", "Adagrad", "Ftrl", "RMSprop"]


@pytest.mark.parametrize("cls", OPTIMIZERS)
def test_every_optimizer_accepts_a_schedule(cls):
    sch = schedules.CosineDecay(0.01, 100, warmup_target=0.05, warmup_steps=10)
    opt = getattr(keras.optimizers, cls)(learning_rate=sch)
    assert opt.learning_rate is sch and opt.lr is sch and opt.schedule is sch
    assert opt.current_learning_rate(0) == sch(0) and opt.current_learning_rate(50) == sch(50)
    spec = opt.to_spec()
    assert spec.schedule is sch and spec.lr == sch(0)
    back = keras.optimizers.from_config(opt.get_config())
    assert type(back) is type(opt) and back.learning_rate == sch and back.get_config() == opt.get_config()
    with pytest.raises(TypeError, match="not settable"):
        opt.learning_rate = 0.1
    with pytest.raises(TypeError, match="not settable"):
        opt.lr = 0.1
    if cls not in ("AdamW",):
        via_lr = getattr(keras.optimizers, cls)(lr=sch)
        assert via_lr.learning_rate is sch
    # the torch.optim rendition starts at the schedule's first rate
    p = torch.nn.Parameter(torch.zeros(3))
    assert opt.to_torch([p]).param_groups[0]["lr"] == sch(0)


@pytest.mark.parametrize("cls", OPTIMIZERS)
def test_a_float_learning_rate_behaves_as_before(cls):
    opt = getattr(keras.optimizers, cls)(learning_rate=0.02)
    assert opt.learning_rate == 0.02 and opt.schedule is None and opt.to_spec().schedule is None
    assert opt.get_config()["learning_rate"] == 0.02
    opt.learning_rate = 0.03
    assert opt.lr == 0.03 and opt.to_spec().lr == 0.03
    from tf_yarn_b200.parallel.comm import hyper_block, launch_code
    blk = hyper_block(opt.to_spec())
    assert launch_code(opt.to_spec()) == opt.to_spec().code and blk.sched.kind == 0
    assert bytes(blk.hp) == bytes(native.OptHyper(*[getattr(blk.hp, f) for f, _ in native.OptHyper._fields_]))


def test_hyper_block_of_a_schedule():
    from tf_yarn_b200.parallel.comm import hyper_block, launch_code
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    sch = schedules.PiecewiseConstantDecay([5, 9], [0.3, 0.2, 0.1])
    spec = OptimizerSpec.adam(sch, 0.9, 0.999, 1e-7)
    assert launch_code(spec) == native.OPT_ADAM | native.OPT_LR_SCHEDULE
    blk = hyper_block(spec, step=7)
    assert blk.hp.step == 7 and blk.hp.lr == np.float32(0.2) and blk.hp.p1 == np.float32(0.9)
    assert blk.sched.kind == native.LR_PIECEWISE and blk.sched.n_boundaries == 2
    assert list(blk.sched.boundaries[:2]) == [5.0, 9.0] and list(blk.sched.values[:3]) == [
        float(np.float32(v)) for v in (0.3, 0.2, 0.1)]


class _Custom(schedules.LearningRateSchedule):
    def __call__(self, step):
        return 0.1

    def get_config(self):
        return {}


def test_a_schedule_without_device_form_is_refused_by_the_fused_step():
    from tf_yarn_b200.parallel.comm import hyper_block
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    with pytest.raises(NotImplementedError, match="no device form"):
        hyper_block(OptimizerSpec.sgd(_Custom()))


def _model(opt, seed=0):
    torch.manual_seed(seed)
    m = keras.Sequential([keras.layers.Dense(16, activation="relu", input_shape=(8,)), keras.layers.Dense(3)])
    m.compile(optimizer=opt, loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True))
    return m


def _data(n=96):
    rs = np.random.RandomState(1)
    x = rs.randn(n, 8).astype("float32")
    y = (x[:, 0] > 0).astype("int64") + (x[:, 1] > 0.5).astype("int64")
    return torch.from_numpy(x), torch.from_numpy(y)


SCHEDULE_OPTS = {
    "sgd_exponential": lambda: keras.optimizers.SGD(schedules.ExponentialDecay(0.2, 3, 0.7), momentum=0.9),
    "adam_cosine_warmup": lambda: keras.optimizers.Adam(
        schedules.CosineDecay(0.0, 10, warmup_target=0.01, warmup_steps=4)),
    "rmsprop_piecewise": lambda: keras.optimizers.RMSprop(schedules.PiecewiseConstantDecay([3, 7], [0.01, 5e-3, 1e-3]),
                                                         momentum=0.5, centered=True),
    "adadelta_polynomial": lambda: keras.optimizers.Adadelta(schedules.PolynomialDecay(1.0, 8, 0.1, power=2.0)),
}


REFERENCE_RATES = {
    "sgd_exponential": lambda s: ref.exponential(s, 0.2, 3, 0.7),
    "adam_cosine_warmup": lambda s: ref.cosine(s, 0.0, 10, 0.0, 0.01, 4),
    "rmsprop_piecewise": lambda s: ref.piecewise(s, [3, 7], [0.01, 5e-3, 1e-3]),
    "adadelta_polynomial": lambda s: ref.polynomial(s, 1.0, 8, 0.1, 2.0),
}


@pytest.mark.parametrize("name", sorted(SCHEDULE_OPTS))
def test_cpu_engine_matches_torch_optim_driven_by_the_reference_rate(name):
    x, y = _data()
    m = _model(SCHEDULE_OPTS[name]())
    # the reference: the same network and torch.optim, the rate set by hand from the schedule before every update
    ref_net = _model(SCHEDULE_OPTS[name]())
    for mm in (m, ref_net):
        if not mm.built:
            mm.build((8,))
    net = ref_net.net
    net.load_state_dict(m.net.state_dict())
    sch = SCHEDULE_OPTS[name]().schedule
    opt = SCHEDULE_OPTS[name]().to_torch([p for p in net.parameters() if p.requires_grad])
    loss_fn = torch.nn.CrossEntropyLoss()
    for i in range(12):
        for g in opt.param_groups:
            g["lr"] = float(np.float32(REFERENCE_RATES[name](i)))
        opt.zero_grad()
        loss_fn(net(x[i * 8:(i + 1) * 8]), y[i * 8:(i + 1) * 8]).backward()
        opt.step()
    m.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0)
    assert m._engine.iterations == 12
    assert m.get_learning_rate() == sch(12)
    for a, b in zip(m.net.parameters(), net.parameters()):
        torch.testing.assert_close(a.detach(), b.detach(), rtol=1e-6, atol=1e-7)


def test_save_load_model_resume_continues_the_schedule(tmp_path):
    x, y = _data()
    make = SCHEDULE_OPTS["adam_cosine_warmup"]
    straight = _model(make())
    straight.fit(x, y, batch_size=8, epochs=2, shuffle=False, verbose=0)     # 24 updates
    first = _model(make())
    first.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0)        # 12 updates
    path = str(tmp_path / "m.tfy")
    first.save(path)
    loaded = keras.models.load_model(path)
    assert isinstance(loaded.optimizer.learning_rate, schedules.CosineDecay)
    assert loaded.optimizer.learning_rate == make().learning_rate
    loaded.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0)
    assert loaded._engine.iterations == 24
    for a, b in zip(loaded.get_weights(), straight.get_weights()):
        np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=1e-5, atol=1e-6)


def test_compile_round_trips_the_schedule_through_the_optimizer_config():
    sch = schedules.InverseTimeDecay(0.1, 5, 0.5, staircase=True)
    m = _model(keras.optimizers.SGD(sch))
    cfg = m.optimizer.get_config()
    m2 = _model(keras.optimizers.from_config(cfg))
    assert m2.optimizer.learning_rate == sch and m2.get_learning_rate() == sch(0)


def test_learning_rate_scheduler_and_set_learning_rate_raise_type_error_on_a_schedule():
    x, y = _data(16)
    m = _model(keras.optimizers.Adam(schedules.ExponentialDecay(1e-3, 10, 0.9)))
    with pytest.raises(TypeError, match="LearningRateSchedule"):
        m.fit(x, y, batch_size=8, epochs=1, verbose=0,
              callbacks=[keras.callbacks.LearningRateScheduler(lambda epoch, lr: lr * 0.5)])
    with pytest.raises(TypeError):
        m.set_learning_rate(0.5)
    # a float learning rate: the callback works as before
    m = _model(keras.optimizers.Adam(1e-3))
    m.fit(x, y, batch_size=8, epochs=2, verbose=0,
          callbacks=[keras.callbacks.LearningRateScheduler(lambda epoch, lr: 1e-3 * 0.5 ** epoch)])
    assert m.get_learning_rate() == pytest.approx(5e-4)


def test_estimator_local_applies_the_schedule_at_the_global_step(tmp_path):
    from tf_yarn_b200.estimator.estimator import Estimator
    from tf_yarn_b200.estimator.spec import EstimatorSpec
    sch = schedules.ExponentialDecay(0.3, 2, 0.5, staircase=True)
    seen = []

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(1))

        def forward(self, x):
            return self.w * x

    def model_fn(features, labels, mode, params):
        def loss(labels_, out):
            return ((out - labels_) ** 2).mean()
        return EstimatorSpec(mode=mode, network=Net(), loss=loss, optimizer=lambda: keras.optimizers.SGD(sch))

    est = Estimator(model_fn, model_dir=str(tmp_path))
    orig = torch.optim.SGD.step

    def spy(self, closure=None):
        seen.append(self.param_groups[0]["lr"])
        return orig(self, closure)
    x = torch.ones(4, 1)
    torch.optim.SGD.step = spy
    try:
        est.train(lambda: iter([(x, x * 2.0)] * 6), steps=6)
    finally:
        torch.optim.SGD.step = orig
    assert seen == [sch(i) for i in range(6)]


def test_hbm_parameter_server_refuses_a_schedule():
    from tf_yarn_b200.estimator import ps_hbm
    net = torch.nn.Linear(2, 1)
    with pytest.raises(ValueError, match="HBM parameter server"):
        ps_hbm.connect_worker(net, keras.optimizers.Adam(schedules.ExponentialDecay(1e-3, 10, 0.9)), None, True, 0)
    with pytest.raises(ValueError, match="HBM parameter server"):
        ps_hbm.connect_worker(net, keras.optimizers.Adam(1e-3), None, True, 0,
                              opt_by_name={"weight": keras.optimizers.SGD(schedules.CosineDecay(0.1, 10))})


def test_shared_memory_parameter_server_push_follows_the_schedule(tmp_path):
    from tf_yarn_b200.estimator import ps
    sch = schedules.PiecewiseConstantDecay([1, 3], [0.5, 0.25, 0.125])
    net = torch.nn.Linear(3, 1, bias=False)
    named = ps._named_trainables(net)
    layout = ps.make_layout(named, 1, keras.optimizers.SGD(sch))
    shard = ps.ShmShard(str(tmp_path / "shard"), layout.shard_elems[0], create=True)
    try:
        conn = ps.WorkerConnection(layout, [shard], [n for n, _ in named], [sch])
        conn._region(0).zero_()
        shard.set_global_step(0)
        want = np.zeros(3)
        for step in range(5):
            net.weight.grad = torch.ones(1, 3)
            conn.push(net)
            conn.increment_global_step()
            want -= sch(step)
        np.testing.assert_allclose(conn._region(0).numpy(), want, rtol=1e-6)
    finally:
        shard.unlink()


def test_a_push_uses_one_global_step_for_all_its_variables(tmp_path):
    from tf_yarn_b200.estimator import ps
    sch = schedules.PiecewiseConstantDecay([0, 1, 2], [0.5, 0.25, 0.125, 0.0625])
    net = torch.nn.Linear(3, 1)
    named = ps._named_trainables(net)
    layout = ps.make_layout(named, 1, keras.optimizers.SGD(sch))
    shard = ps.ShmShard(str(tmp_path / "shard"), layout.shard_elems[0], create=True)
    try:
        conn = ps.WorkerConnection(layout, [shard], [n for n, _ in named], [sch, sch])
        for i in range(2):
            conn._region(i).zero_()
        shard.set_global_step(0)
        real = conn.global_step

        def racing():                       # another worker advances the step between two reads
            v = real()
            shard.add_global_step(1)
            return v
        conn.global_step = racing
        net.weight.grad, net.bias.grad = torch.ones(1, 3), torch.ones(1)
        conn.push(net)
        np.testing.assert_allclose(conn._region(0).numpy(), [-0.5] * 3)
        np.testing.assert_allclose(conn._region(1).numpy(), [-0.5])
    finally:
        shard.unlink()


def test_fused_ddp_param_group_reads_the_device_rate_and_refuses_to_be_set():
    from types import SimpleNamespace
    from tf_yarn_b200.parallel.comm import hyper_block
    from tf_yarn_b200.parallel.ddp import _FusedOptimizer
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    sch = schedules.ExponentialDecay(0.1, 2, 0.5)
    spec = OptimizerSpec.adam(sch)
    blk = hyper_block(spec, step=3)
    p = torch.nn.Parameter(torch.zeros(4))
    bucket = SimpleNamespace(params=[p], hyper=torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8))
    opt = _FusedOptimizer(SimpleNamespace(_buckets=[bucket]), spec)
    assert opt.param_groups[0]["lr"] == sch(3) and "lr" in opt.param_groups[0]
    assert opt.param_groups[0]["params"] == [p]
    bucket.hyper[0:4].copy_(torch.tensor([sch(5)], dtype=torch.float32).view(torch.uint8))
    assert opt.param_groups[0]["lr"] == sch(5)           # follows what the fused step wrote
    with pytest.raises(TypeError, match="LearningRateSchedule"):
        opt.param_groups[0]["lr"] = 0.5
    with pytest.raises(TypeError, match="LearningRateSchedule"):
        opt.param_groups[0].setdefault("initial_lr", opt.param_groups[0]["lr"])   # what a torch LR scheduler does
    assert opt.step() is None
    const = _FusedOptimizer(SimpleNamespace(_buckets=[bucket]), OptimizerSpec.adam(1e-3))
    assert type(const.param_groups[0]) is dict and const.param_groups[0]["lr"] == 1e-3
