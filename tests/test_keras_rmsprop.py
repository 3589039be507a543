"""Keras RMSprop on CPU: the fused K4 update built for the host (tests/native/rmsprop_host.cpp) against TorchRMSprop and
against an independent float64 NumPy transcription of the tf.keras formulas; the descriptor, its spec packing and
serialisation; save -> load_model -> resume; a learning-rate change mid-run; the shared-memory parameter-server push;
and the canned estimators' default learning rate."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import ps
from tf_yarn_b200.ops import native
from tf_yarn_b200.parallel.optspec import OPT_RMSPROP, OptimizerSpec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"

VARIANTS = {
    "plain": dict(momentum=0.0, centered=False),
    "momentum": dict(momentum=0.9, centered=False),
    "centered": dict(momentum=0.0, centered=True),
    "momentum_centered": dict(momentum=0.9, centered=True),
}


def numpy_rmsprop(p, grads, lrs, rho, momentum, eps, centered, wd):
    """The tf.keras RMSprop update in float64, written from its definition (one lr per step)."""
    p = np.asarray(p, np.float64).copy()
    v, m, mg = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
    for g, lr in zip(grads, lrs):
        g = np.asarray(g, np.float64) + wd * p
        v = rho * v + (1 - rho) * g * g
        if centered:
            mg = rho * mg + (1 - rho) * g
            denom = v - mg * mg + eps
        else:
            denom = v + eps
        inc = lr * g / np.sqrt(denom)
        if momentum > 0:
            m = momentum * m + inc
            p = p - m
        else:
            p = p - inc
    return p


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("rmsprop") / "librmsprop.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "rmsprop_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    lib.tfy_host_rmsprop_step.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
    lib.tfy_host_rmsprop_step.restype = None
    return lib


class HostK4:
    """The device-side state of one shard, laid out as FusedShardedOptimizer allocates it."""

    def __init__(self, lib, spec, p0):
        self.lib, self.spec = lib, spec
        n = p0.numel()
        self.p = p0.clone().contiguous()
        self.s1 = torch.full((n,), spec.init_s1)
        self.s2 = torch.zeros(spec.s2_numel(n))
        self.hyper = native.OptHyper(spec.lr, spec.p1, spec.p2, spec.eps, spec.weight_decay, 1.0, 0, spec.flags, 0, 0)

    def step(self, summed_grad, world):
        self.lib.tfy_host_rmsprop_step(ctypes.byref(self.hyper), world, self.p.data_ptr(), summed_grad.data_ptr(),
                                       self.s1.data_ptr(), self.s2.data_ptr(), self.p.numel())


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("world", [1, 4])
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_kernel_update_matches_torch_rmsprop_and_the_formulas(lib, variant, world, wd):
    desc = keras.optimizers.RMSprop(0.01, rho=0.9, epsilon=1e-7, weight_decay=wd, **VARIANTS[variant])
    spec = desc.to_spec()
    n = 257
    g = torch.Generator().manual_seed(11)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = desc.to_torch([ref])
    k4 = HostK4(lib, spec, p0)
    grads = []
    for step in range(7):
        grad = torch.randn(n, generator=g) * (0.5 + 0.2 * step)
        grads.append(grad.numpy().copy())
        # the kernel receives the SUM over ranks and scales by 1/world: feed it world x the averaged gradient
        k4.step((grad * world).contiguous(), world)
        ref.grad = grad.clone()
        opt.step()
    assert k4.hyper.step == 7
    want = numpy_rmsprop(p0.numpy(), grads, [0.01] * 7, 0.9, VARIANTS[variant]["momentum"], 1e-7,
                         VARIANTS[variant]["centered"], wd)
    scale = max(1.0, float(np.abs(want).max()))
    assert float(np.abs(ref.detach().numpy() - want).max()) < 5e-6 * scale, variant
    assert float(np.abs(k4.p.numpy() - want).max()) < 5e-6 * scale, variant
    # the states the kernel keeps are the ones the torch rendition keeps, in the documented order
    st = opt.state[ref]
    assert torch.allclose(k4.s1, st["v"], rtol=1e-5, atol=1e-7)
    extra = [st[k] for k in ("m", "mg") if k in st]
    assert k4.s2.numel() == max(8, n * len(extra))
    for i, t in enumerate(extra):
        assert torch.allclose(k4.s2[i * n:(i + 1) * n], t, rtol=1e-5, atol=1e-7)


def test_learning_rate_change_scales_later_increments_only(lib):
    """lr sits inside the momentum buffer: after a change, the increments already in the buffer keep the old lr.
    torch.optim.RMSprop applies lr outside the buffer (and epsilon outside the root), so it takes a different path."""
    desc = keras.optimizers.RMSprop(0.02, momentum=0.9, centered=True)
    spec = desc.to_spec()
    n = 64
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.clone())
    opt = desc.to_torch([ref])
    plain_torch = torch.nn.Parameter(p0.clone())
    topt = torch.optim.RMSprop([plain_torch], lr=0.02, alpha=0.9, eps=1e-7, momentum=0.9, centered=True)
    k4 = HostK4(lib, spec, p0)
    lrs, grads = [0.02] * 4 + [0.002] * 4, []
    for lr in lrs:
        grad = torch.randn(n, generator=g)
        grads.append(grad.numpy().copy())
        k4.hyper.lr = lr
        for grp in opt.param_groups + topt.param_groups:
            grp["lr"] = lr
        k4.step(grad.contiguous(), 1)
        ref.grad, plain_torch.grad = grad.clone(), grad.clone()
        opt.step()
        topt.step()
    want = numpy_rmsprop(p0.numpy(), grads, lrs, 0.9, 0.9, 1e-7, True, 0.0)
    assert float(np.abs(k4.p.numpy() - want).max()) < 5e-6
    assert float(np.abs(ref.detach().numpy() - want).max()) < 5e-6
    assert float(np.abs(plain_torch.detach().numpy() - want).max()) > 1e-3


def test_name_resolution_spec_packing_and_config_round_trip():
    for name in ("rmsprop", "RMSprop", "RMSProp"):
        assert type(keras.optimizers.get(name)) is keras.optimizers.RMSprop
    d = keras.optimizers.RMSprop(0.005, rho=0.8, momentum=0.5, epsilon=1e-6, centered=True, weight_decay=0.01)
    spec = d.to_spec()
    assert (spec.kind, spec.code, OPT_RMSPROP, native.OPT_RMSPROP) == ("rmsprop", 5, 5, 5)
    assert (spec.lr, spec.p1, spec.p2, spec.eps, spec.weight_decay, spec.flags) == \
        pytest.approx((0.005, 0.8, 0.5, 1e-6, 0.01, 1))
    assert spec.n_states == 3 and spec.s2_numel(64) == 128
    assert OptimizerSpec.rmsprop().n_states == 1 and OptimizerSpec.rmsprop().s2_numel(64) == 8
    assert OptimizerSpec.rmsprop(momentum=0.9).n_states == 2 and OptimizerSpec.rmsprop(centered=True).n_states == 2
    cfg = d.get_config()
    assert cfg["class_name"] == "RMSprop"
    again = keras.optimizers.from_config(cfg)
    assert type(again) is keras.optimizers.RMSprop and again.get_config() == cfg
    assert keras.optimizers.RMSprop(lr=0.3).learning_rate == 0.3
    with pytest.raises(ValueError, match="momentum"):
        keras.optimizers.RMSprop(momentum=-0.1)


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


def test_cpu_fit_learns_and_save_load_resume_equals_an_uninterrupted_run(tmp_path):
    x, y = _xy(64)

    def opt():
        return keras.optimizers.RMSprop(0.01, momentum=0.9, centered=True)
    straight = _fresh(opt())
    h = straight.fit(x, y, batch_size=16, epochs=3, shuffle=False, verbose=0)
    assert h.history["loss"][-1] < h.history["loss"][0]
    first = _fresh(opt())
    first.fit(x, y, batch_size=16, epochs=2, shuffle=False, verbose=0)
    path = str(tmp_path / "ckpt-2")
    first.save(path)
    resumed = keras.models.load_model(path)
    resumed._device = torch.device("cpu")
    assert type(resumed.optimizer) is keras.optimizers.RMSprop
    assert resumed.optimizer.get_config() == opt().get_config()
    resumed.fit(x, y, batch_size=16, epochs=1, shuffle=False, verbose=0)
    for a, b in zip(resumed.get_weights(), straight.get_weights()):
        assert np.allclose(a, b, atol=1e-6)
    # by name, with Keras' defaults
    named = _fresh("rmsprop")
    h = named.fit(x, y, batch_size=16, epochs=3, shuffle=False, verbose=0)
    assert type(named.optimizer) is keras.optimizers.RMSprop and named.optimizer.learning_rate == 0.001
    assert h.history["loss"][-1] < h.history["loss"][0]


def test_learning_rate_scheduler_reaches_the_cpu_engine():
    x, y = _xy(32)
    m = _fresh(keras.optimizers.RMSprop(0.01, momentum=0.9))
    sched = keras.callbacks.LearningRateScheduler(lambda epoch, lr: 0.01 if epoch == 0 else 0.001)
    m.fit(x, y, batch_size=16, epochs=2, shuffle=False, verbose=0, callbacks=[sched])
    assert m._engine.opt.param_groups[0]["lr"] == pytest.approx(0.001)
    assert isinstance(m._engine.opt, keras.optimizers.TorchRMSprop)


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


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_ps_push_applies_the_rmsprop_update(tmp_path, variant):
    desc = keras.optimizers.RMSprop(0.01, weight_decay=0.001, **VARIANTS[variant])
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Tanh(), torch.nn.Linear(7, 3))
    ref = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Tanh(), torch.nn.Linear(7, 3))
    ref.load_state_dict(net.state_dict())
    conn, shards = _connection(tmp_path, net, desc)
    slots = 1 + int(VARIANTS[variant]["momentum"] > 0) + int(VARIANTS[variant]["centered"])
    lay = conn.layout
    assert lay.var_slots == [slots] * 4 and lay.slots == slots
    # Linear(5, 7), Linear(7, 3) round-robin over 2 ps: weights on ps 0, biases on ps 1 (padded to 8)
    assert lay.shard_elems == [(40 + 24) * (1 + slots), (8 + 8) * (1 + slots)]
    again = ps.Layout.from_json(lay.to_json())          # what the workers derive from the published layout
    assert again.var_slots == lay.var_slots and again.shard_elems == lay.shard_elems
    opt = desc.to_torch(ref.parameters())
    g = torch.Generator().manual_seed(1)
    for _ in range(6):
        x, y = torch.randn(16, 5, generator=g), torch.randint(0, 3, (16,), generator=g)
        conn.pull(net)
        net.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        conn.push(net)
        conn.increment_global_step()
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(x), y).backward()
        opt.step()
    conn.pull(net)
    for (n, a), (_, b) in zip(net.named_parameters(), ref.named_parameters()):
        assert torch.allclose(a, b, atol=2e-6, rtol=1e-5), (n, (a - b).abs().max().item())
    for s in shards:
        s.unlink()


def test_mixed_layout_slot_counts_follow_each_variables_hyper_parameters():
    by_name = {"0.weight": keras.optimizers.RMSprop(momentum=0.9, centered=True),
               "0.bias": keras.optimizers.RMSprop(centered=True)}
    net = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    lay = ps.make_layout(ps._named_trainables(net), 1, keras.optimizers.RMSprop(), by_name)
    assert lay.kinds == ["rmsprop"] * 4 and lay.var_slots == [3, 2, 1, 1]
    assert lay.shard_elems == [16 * 4 + 8 * 3 + 8 * 2 + 8 * 2]


def test_canned_estimators_give_rmsprop_tfs_default_learning_rate():
    from tf_yarn_b200.estimator import canned
    from tf_yarn_b200.estimator import feature_column as fc
    num = fc.numeric_column("x", shape=(4,))

    def resolved(est, tower_optimizers=False):
        spec = est._model_fn({"x": torch.zeros(2, 4)}, None, "train")
        return spec.optimizers if tower_optimizers else spec.optimizer

    dnn = resolved(canned.DNNClassifier([8], [num], optimizer="RMSProp"))
    assert type(dnn) is keras.optimizers.RMSprop and dnn.learning_rate == 0.05
    lin = resolved(canned.LinearClassifier([num] * 100, optimizer="rmsprop"))        # min(0.2, 1/sqrt(100))
    assert type(lin) is keras.optimizers.RMSprop and lin.learning_rate == pytest.approx(0.1)
    lin = resolved(canned.LinearClassifier([num], optimizer="rmsprop"))
    assert lin.learning_rate == pytest.approx(0.2)
    wd = canned.DNNLinearCombinedClassifier(linear_feature_columns=[num], dnn_feature_columns=[num],
                                            dnn_hidden_units=[8], linear_optimizer="rmsprop", dnn_optimizer="rmsprop")
    assert resolved(wd).learning_rate == pytest.approx(0.001)
    assert resolved(wd, True)["linear."].learning_rate == pytest.approx(0.005)
    assert resolved(canned.DNNClassifier([8], [num], optimizer="sgd")) == "sgd"       # other names stay untouched
