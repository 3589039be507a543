"""Keras Adamax and Nadam on CPU: the fused K4 update built for the host (tests/native/adamax_nadam_host.cpp) against
TorchAdamax / torch.optim.NAdam and against an independent float64 NumPy transcription of the update rules, over many
steps, at world 1 and 4, with and without weight decay, across a learning-rate change and under a schedule; the
descriptors, their specs and serialisation; save -> load_model -> resume, with and without gradient accumulation;
the canned estimators' names; the shared-memory parameter server's lazy Adamax push; and both parameter-server
planes refusing Nadam."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import ps
from tf_yarn_b200.keras import schedules
from tf_yarn_b200.ops import native
from tf_yarn_b200.parallel.comm import hyper_block
from tf_yarn_b200.parallel.optspec import OPT_ADAMAX, OPT_NADAM, OptimizerSpec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"
CLASSES = {"adamax": keras.optimizers.Adamax, "nadam": keras.optimizers.Nadam}


def nadam_mu(b1, t):
    return b1 * (1.0 - 0.5 * 0.96 ** (0.004 * t))


def numpy_adamax(p, grads, lrs, ts, b1, b2, eps, wd):
    """The tf.keras Adamax update in float64, written from its definition (one lr and one t per update)."""
    p = np.asarray(p, np.float64).copy()
    m, u = np.zeros_like(p), np.zeros_like(p)
    for g, lr, t in zip(grads, lrs, ts):
        g = np.asarray(g, np.float64) + wd * p
        m = b1 * m + (1 - b1) * g
        u = np.maximum(b2 * u, np.abs(g))
        p = p - lr / (1 - b1 ** t) * m / (u + eps)
    return p, m, u


def numpy_nadam(p, grads, lrs, ts, b1, b2, eps, wd):
    """Nadam (torch.optim.NAdam, momentum_decay = 0.004) in float64; returns p, m, v and the running product."""
    p = np.asarray(p, np.float64).copy()
    m, v, prod = np.zeros_like(p), np.zeros_like(p), 1.0
    for g, lr, t in zip(grads, lrs, ts):
        g = np.asarray(g, np.float64) + wd * p
        mu, mu_next = nadam_mu(b1, t), nadam_mu(b1, t + 1)
        prod *= mu
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        d = np.sqrt(v / (1 - b2 ** t)) + eps
        p = p - lr * (1 - mu) / (1 - prod) * g / d - lr * mu_next / (1 - prod * mu_next) * m / d
    return p, m, v, prod


NUMPY = {"adamax": numpy_adamax, "nadam": numpy_nadam}


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("adamax_nadam") / "libadamax_nadam.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "adamax_nadam_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_adamax_nadam_step.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 4 + \
        [ctypes.c_int]
    lib.tfy_host_adamax_nadam_step.restype = None
    return lib


class HostK4:
    """The device-side state of one shard and its hyper block, as FusedShardedOptimizer allocates them."""

    def __init__(self, lib, spec, p0):
        self.lib, self.spec = lib, spec
        n = p0.numel()
        self.p = p0.clone().contiguous()
        self.s1 = torch.full((n,), spec.init_s1)
        self.s2 = torch.zeros(spec.s2_numel(n))
        self.blk = hyper_block(spec)
        self.hyper = self.blk.hp

    def step(self, summed_grad, world):
        self.lib.tfy_host_adamax_nadam_step(ctypes.byref(self.blk), self.spec.code, int(self.spec.schedule is not None),
                                            world, self.p.data_ptr(), summed_grad.data_ptr(), self.s1.data_ptr(),
                                            self.s2.data_ptr(), self.p.numel())


def test_layout_of_the_nadam_hyper_block(lib):
    out = (ctypes.c_int * 16)()
    n = lib.tfy_host_nadam_layout(out, 16)
    got = list(out[:n])
    assert got == [ctypes.sizeof(native.NadamHyperBlock), native.NadamHyperBlock.hp.offset,
                   native.NadamHyperBlock.sched.offset, native.NadamHyperBlock.mu_product.offset,
                   native.OPT_ADAMAX, native.OPT_NADAM]
    assert native.NadamHyperBlock.mu_product.offset == ctypes.sizeof(native.HyperBlock)
    assert (OPT_ADAMAX, OPT_NADAM) == (6, 7)


def _close(a, want, tol=2e-5):
    scale = max(1.0, float(np.abs(want).max()))
    return float(np.abs(np.asarray(a, np.float64) - want).max()) < tol * scale


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("world", [1, 4])
@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_kernel_update_matches_torch_and_the_formulas(lib, kind, world, wd):
    desc = CLASSES[kind](0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-7, weight_decay=wd)
    spec = desc.to_spec()
    assert spec.n_states == 2
    n, steps = 257, 60
    g = torch.Generator().manual_seed(11)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = desc.to_torch([ref])
    k4 = HostK4(lib, spec, p0)
    grads = []
    for step in range(steps):
        grad = torch.randn(n, generator=g) * (0.5 + 0.02 * step)
        grads.append(grad.numpy().copy())
        # the kernel receives the SUM over ranks and scales by 1/world: feed it world x the averaged gradient
        k4.step((grad * world).contiguous(), world)
        ref.grad = grad.clone()
        opt.step()
    assert k4.hyper.step == steps
    want = NUMPY[kind](p0.numpy(), grads, [0.01] * steps, range(1, steps + 1), 0.9, 0.999, 1e-7, wd)
    assert _close(ref.detach().numpy(), want[0]), kind
    assert _close(k4.p.numpy(), want[0]), kind
    # the states the kernel keeps: s1 = m, s2 = u (Adamax) or v (Nadam)
    assert _close(k4.s1.numpy(), want[1]) and _close(k4.s2.numpy(), want[2])
    st = opt.state[ref]
    assert torch.allclose(k4.s1, st["exp_avg"], rtol=1e-4, atol=1e-7)
    assert torch.allclose(k4.s2, st["exp_inf" if kind == "adamax" else "exp_avg_sq"], rtol=1e-4, atol=1e-9)
    if kind == "nadam":
        # the device holds beta_1 in fp32: its product follows the float64 formula of that value
        b1 = float(np.float32(0.9))
        assert k4.blk.mu_product == pytest.approx(np.prod([nadam_mu(b1, t) for t in range(1, steps + 1)]), rel=1e-12,
                                                  abs=0)
        assert float(st["mu_product"]) == pytest.approx(want[3], rel=1e-5, abs=0)


def test_torch_adamax_differs_from_the_keras_rule():
    """torch.optim.Adamax puts epsilon inside the max (u = max(beta_2 u, |g| + eps), p -= ... m / u): after one
    gradient of epsilon's order and then zeros, its norm decays onto epsilon while the Keras rule's is u + eps."""
    p0 = torch.linspace(-1, 1, 32)
    grads = [torch.full((32,), 1e-3)] + [torch.zeros(32)] * 9
    ours, theirs = torch.nn.Parameter(p0.clone()), torch.nn.Parameter(p0.clone())
    a = keras.optimizers.Adamax(0.1, beta_2=0.5, epsilon=1e-3).to_torch([ours])
    b = torch.optim.Adamax([theirs], lr=0.1, betas=(0.9, 0.5), eps=1e-3)
    assert isinstance(a, keras.optimizers.TorchAdamax)
    for grad in grads:
        ours.grad, theirs.grad = grad.clone(), grad.clone()
        a.step()
        b.step()
    want = numpy_adamax(p0.numpy(), [x.numpy() for x in grads], [0.1] * 10, range(1, 11), 0.9, 0.5, 1e-3, 0.0)[0]
    assert _close(ours.detach().numpy(), want, 1e-6)
    assert float(np.abs(theirs.detach().numpy() - want).max()) > 1e-3


@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_learning_rate_change_mid_run(lib, kind):
    desc = CLASSES[kind](0.02, weight_decay=0.001)
    spec = desc.to_spec()
    n = 64
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = desc.to_torch([ref])
    k4 = HostK4(lib, spec, p0)
    lrs, grads = [0.02] * 10 + [0.002] * 10, []
    for lr in lrs:
        grad = torch.randn(n, generator=g)
        grads.append(grad.numpy().copy())
        k4.hyper.lr = lr                       # what FusedShardedOptimizer.set_lr writes
        for grp in opt.param_groups:
            grp["lr"] = lr
        k4.step(grad.contiguous(), 1)
        ref.grad = grad.clone()
        opt.step()
    want = NUMPY[kind](p0.numpy(), grads, lrs, range(1, 21), 0.9, 0.999, 1e-7, 0.001)[0]
    assert _close(k4.p.numpy(), want) and _close(ref.detach().numpy(), want)


@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_scheduled_rate_is_advanced_with_the_step(lib, kind):
    sched = schedules.ExponentialDecay(0.01, decay_steps=4, decay_rate=0.7)
    spec = CLASSES[kind](sched).to_spec()
    assert spec.schedule is sched
    n, steps = 96, 25
    g = torch.Generator().manual_seed(8)
    p0 = torch.randn(n, generator=g)
    k4 = HostK4(lib, spec, p0)
    grads = []
    for _ in range(steps):
        grad = torch.randn(n, generator=g)
        grads.append(grad.numpy().copy())
        k4.step(grad.contiguous(), 1)
    assert k4.hyper.step == steps and k4.hyper.lr == pytest.approx(float(sched(steps)), rel=1e-6)
    lrs = [float(sched(s)) for s in range(steps)]
    want = NUMPY[kind](p0.numpy(), grads, lrs, range(1, steps + 1), 0.9, 0.999, 1e-7, 0.0)
    assert _close(k4.p.numpy(), want[0])
    if kind == "nadam":
        assert k4.blk.mu_product == pytest.approx(want[3], rel=1e-6, abs=0)


def test_name_resolution_spec_packing_and_config_round_trip():
    for name, cls in (("adamax", keras.optimizers.Adamax), ("Adamax", keras.optimizers.Adamax),
                      ("nadam", keras.optimizers.Nadam), ("Nadam", keras.optimizers.Nadam)):
        opt = keras.optimizers.get(name)
        assert type(opt) is cls and opt.learning_rate == 0.001
        assert (opt.beta_1, opt.beta_2, opt.epsilon) == (0.9, 0.999, 1e-7)
    for kind, code in (("adamax", 6), ("nadam", 7)):
        d = CLASSES[kind](0.005, beta_1=0.8, beta_2=0.99, epsilon=1e-6, weight_decay=0.01,
                          gradient_accumulation_steps=3)
        spec = d.to_spec()
        assert (spec.kind, spec.code, OptimizerSpec.KINDS[kind]) == (kind, code, code)
        assert (spec.lr, spec.p1, spec.p2, spec.eps, spec.weight_decay, spec.flags) == \
            pytest.approx((0.005, 0.8, 0.99, 1e-6, 0.01, 0))
        assert spec.n_states == 2 and spec.s2_numel(64) == 64
        cfg = d.get_config()
        assert cfg["class_name"] == CLASSES[kind].__name__ and cfg["gradient_accumulation_steps"] == 3
        again = keras.optimizers.from_config(cfg)
        assert type(again) is CLASSES[kind] and again.get_config() == cfg
        assert CLASSES[kind](lr=0.3).learning_rate == 0.3
        sched = CLASSES[kind](schedules.ExponentialDecay(0.01, 4, 0.5))
        back = keras.optimizers.from_config(sched.get_config())
        assert isinstance(back.learning_rate, schedules.ExponentialDecay) and back.get_config() == sched.get_config()
    assert type(hyper_block(OptimizerSpec.nadam())) is native.NadamHyperBlock
    assert hyper_block(OptimizerSpec.nadam()).mu_product == 1.0
    assert type(hyper_block(OptimizerSpec.adamax())) is native.HyperBlock
    nad = keras.optimizers.Nadam(0.01).to_torch([torch.nn.Parameter(torch.zeros(2))])
    assert isinstance(nad, torch.optim.NAdam) and nad.defaults["momentum_decay"] == 0.004
    assert not nad.defaults["decoupled_weight_decay"]


def _xy(n=96, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 4, generator=g)
    return x, (x[:, 0] + x[:, 1] > 0).long()


def _fresh(optimizer):
    torch.manual_seed(5)
    m = keras.Sequential([keras.layers.Dense(6, activation="tanh", input_shape=(4,)), keras.layers.Dense(2)])
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=optimizer)
    m._device = torch.device("cpu")
    return m


@pytest.mark.parametrize("accum", [None, 3])
@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_cpu_fit_save_load_resume_equals_an_uninterrupted_run(tmp_path, kind, accum):
    x, y = _xy(64)

    def opt():
        return CLASSES[kind](0.01, weight_decay=0.001, gradient_accumulation_steps=accum)
    straight = _fresh(opt())
    h = straight.fit(x, y, batch_size=16, epochs=3, shuffle=False, verbose=0)
    assert h.history["loss"][-1] < h.history["loss"][0]
    first = _fresh(opt())
    first.fit(x, y, batch_size=16, epochs=2, shuffle=False, verbose=0)
    path = str(tmp_path / "ckpt-2")
    first.save(path)
    resumed = keras.models.load_model(path)
    resumed._device = torch.device("cpu")
    assert type(resumed.optimizer) is CLASSES[kind]
    assert resumed.optimizer.get_config() == opt().get_config()
    resumed.fit(x, y, batch_size=16, epochs=1, shuffle=False, verbose=0)
    for a, b in zip(resumed.get_weights(), straight.get_weights()):
        assert np.array_equal(a, b)
    eng = straight._engine
    assert isinstance(eng.opt, keras.optimizers.TorchAdamax if kind == "adamax" else torch.optim.NAdam)
    # 12 batches: t = s + 1 of every update batch s (all of them, or every third one when accumulating)
    ts = [s + 1 for s in range(12) if accum is None or (s + 1) % accum == 0]
    for p, q in zip(eng.net.parameters(), resumed._engine.net.parameters()):
        st = eng.opt.state[p]
        assert float(st["step"]) == float(resumed._engine.opt.state[q]["step"]) == ts[-1]
        if kind == "nadam":
            want = float(np.prod([nadam_mu(0.9, t) for t in ts]))
            assert float(st["mu_product"]) == pytest.approx(want, rel=1e-5, abs=0)
            assert float(resumed._engine.opt.state[q]["mu_product"]) == float(st["mu_product"])


def test_canned_estimators_accept_the_names():
    from tf_yarn_b200.estimator import canned
    from tf_yarn_b200.estimator import feature_column as fc
    num = fc.numeric_column("x", shape=(4,))

    def resolved(est, tower_optimizers=False):
        spec = est._model_fn({"x": torch.zeros(2, 4)}, None, "train")
        return spec.optimizers if tower_optimizers else spec.optimizer

    for name, cls in (("Adamax", keras.optimizers.Adamax), ("nadam", keras.optimizers.Nadam)):
        dnn = resolved(canned.DNNClassifier([8], [num], optimizer=name))
        assert type(dnn) is cls and dnn.learning_rate == 0.05
        lin = resolved(canned.LinearRegressor([num] * 100, optimizer=name))          # min(0.2, 1/sqrt(100))
        assert type(lin) is cls and lin.learning_rate == pytest.approx(0.1)
        wd = canned.DNNLinearCombinedClassifier(linear_feature_columns=[num], dnn_feature_columns=[num],
                                                dnn_hidden_units=[8], linear_optimizer=name, dnn_optimizer=name)
        assert type(resolved(wd)) is cls and resolved(wd).learning_rate == pytest.approx(0.001)
        assert resolved(wd, True)["linear."].learning_rate == pytest.approx(0.005)


class _BagNet(torch.nn.Module):
    def __init__(self, V=12, D=8):
        super().__init__()
        self.emb = torch.nn.EmbeddingBag(V, D, mode="sum")
        self.out = torch.nn.Linear(D, 3)

    def forward(self, ids):
        return self.out(self.emb(ids))


def _connection(tmp_path, net, desc):
    named = ps._named_trainables(net)
    layout = ps.make_layout(named, 2, desc)
    shards = [ps.ShmShard(str(tmp_path / f"shard{i}"), layout.shard_elems[i], create=True) for i in range(2)]
    for s in shards:
        s.data.zero_()
    conn = ps.WorkerConnection(layout, shards, [n for n, _ in named])
    with torch.no_grad():
        for i, (_, p) in enumerate(named):
            conn._region(i).copy_(p.detach().reshape(-1))
    shards[0].set_global_step(0)
    return conn, shards


def test_ps_adamax_push_is_lazy_and_matches_a_float64_reference(tmp_path):
    lr, b1, b2, eps, wd = 0.01, 0.9, 0.999, 1e-7, 0.001
    desc = keras.optimizers.Adamax(lr, weight_decay=wd)
    torch.manual_seed(0)
    V = 12
    net = _BagNet(V)
    conn, shards = _connection(tmp_path, net, desc)
    lay = conn.layout
    assert lay.kinds == ["adamax"] * 3 and lay.var_slots == [2, 2, 2]
    assert ps.slot_names("adamax", lay.hypers[0]) == ("m", "u")
    # reference: float64 value, m, u per variable, updated row by row on the rows the batch touched
    ref = {n: [p.detach().double().clone(), torch.zeros_like(p, dtype=torch.float64),
               torch.zeros_like(p, dtype=torch.float64)] for n, p in net.named_parameters()}
    untouched = [V - 1, V - 2, 0]
    g = torch.Generator().manual_seed(1)
    for step in range(8):
        ids = torch.randint(1, V - 2, (6, 4), generator=g)
        ids[:, 0] = ids[0, 0]                                  # one row repeated in every example
        y = torch.randint(0, 3, (6,), generator=g)
        conn.pull(net)
        net.zero_grad()
        torch.nn.functional.cross_entropy(net(ids), y).backward()
        t = step + 1
        for name, p in net.named_parameters():
            w, m, u = ref[name]
            gr = p.grad.double()
            rows = p.shape[0]
            hit = (gr.reshape(rows, -1) != 0).any(dim=1)
            gg = gr + wd * w
            m2, u2, w2 = m.reshape(rows, -1), u.reshape(rows, -1), w.reshape(rows, -1)
            gh = gg.reshape(rows, -1)[hit]
            m2[hit] = b1 * m2[hit] + (1 - b1) * gh
            u2[hit] = torch.maximum(b2 * u2[hit], gh.abs())
            w2[hit] = w2[hit] - lr / (1 - b1 ** t) * m2[hit] / (u2[hit] + eps)
        emb_before = conn._region(0).clone().view(V, -1)
        conn.push(net)
        assert torch.equal(conn._region(0).view(V, -1)[untouched], emb_before[untouched])
        conn.increment_global_step()
    for i, (name, p) in enumerate(net.named_parameters()):
        w, m, u = ref[name]
        for s, want in enumerate((w, m, u)):
            got = conn._region(i, s).double().view(p.shape)
            assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (name, s, (got - want).abs().max().item())
    # rows no batch touched keep their initial value and zero slots; the exported slots carry the names
    emb = conn._region(0).view(V, -1)
    assert torch.equal(emb[untouched], ref["emb.weight"][0][untouched].float())
    assert float(conn._region(0, 1).view(V, -1)[untouched].abs().max()) == 0.0
    slots = conn.optimizer_state()
    assert slots["emb.weight"]["slot_names"] == ["m", "u"] and slots["emb.weight"]["kind"] == "adamax"
    for s in shards:
        s.unlink()


@pytest.mark.parametrize("plane", ["shm", "hbm"])
def test_both_parameter_server_planes_refuse_nadam(plane):
    from tf_yarn_b200.estimator import ps_hbm
    connect = ps.connect_worker if plane == "shm" else ps_hbm.connect_worker
    net = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    with pytest.raises(ValueError, match=r"Nadam \(variable '0.weight'\).*use Adam"):
        connect(net, keras.optimizers.Nadam(), cluster=None, is_chief=True, global_step=0)
    by_name = {"1.bias": keras.optimizers.Nadam()}
    with pytest.raises(ValueError, match=r"'1.bias'.*use Adam"):
        connect(net, keras.optimizers.Adam(), cluster=None, is_chief=True, global_step=0, opt_by_name=by_name)
    # the HBM plane fuses neither optimizer (its layout check refuses Adamax too)
    assert "adamax" not in ps_hbm.OPT_CODES and "nadam" not in ps_hbm.OPT_CODES
