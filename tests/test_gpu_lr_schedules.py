"""GPU tests of Keras learning-rate schedules in the fused K4 step (run with `pytest -m gpu` on an H100).

LOCAL mode on one GPU: after N steps -- eager launches and replayed CUDA graphs -- the device hp->lr equals the
schedule at step N for each of the six schedules, and the parameters match torch.optim driven by the schedule's rate
step by step; eager launches and graph replay give the same bits; resume mid-schedule continues it; a constant rate
still launches the instantiations without schedule code; the MNIST-CNN fast path with Adam, RMSprop and Adadelta
follows a schedule at 10 launches per step.  With 2+ GPUs, tests/gpu/lr_schedule_check.py covers the P2P and NVLS
transports and DDP `fuse_optimizer`.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(33, 17), (129,), (7, 5, 3)]


def _schedules():
    from tf_yarn_b200.keras import schedules as S
    return {
        "exponential": S.ExponentialDecay(0.05, 4, 0.8),
        "exponential_staircase": S.ExponentialDecay(0.05, 4, 0.8, staircase=True),
        "piecewise": S.PiecewiseConstantDecay([3, 7, 11], [0.05, 0.02, 0.01, 0.004]),
        "polynomial_cycle": S.PolynomialDecay(0.05, 6, end_learning_rate=0.001, power=2.0, cycle=True),
        "inverse_time": S.InverseTimeDecay(0.05, 5, 0.5, staircase=True),
        "cosine_warmup": S.CosineDecay(0.0, 12, alpha=0.1, warmup_target=0.05, warmup_steps=5),
        "cosine_restarts": S.CosineDecayRestarts(0.05, 3, t_mul=2.0, m_mul=0.8, alpha=0.05),
    }


def _fused(spec, dtype=torch.float32, zero_grads=True):
    from tf_yarn_b200.keras.engine import _solo_communicator
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    return FusedShardedOptimizer(_solo_communicator(0), SHAPES, spec, param_dtype=dtype, grad_dtype=dtype,
                                 zero_grads=zero_grads)


def _device_lr(fo) -> float:
    return float(fo.hyper[0:4].view(torch.float32).item())


def _grads(n, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    init = [torch.randn(s, device="cuda", generator=g) * 0.3 for s in SHAPES]
    return init, [[torch.randn(s, device="cuda", generator=g) * 0.5 for s in SHAPES] for _ in range(n)]


def _opt(name, schedule):
    from tf_yarn_b200.keras import optimizers as O
    return {"sgd_momentum": lambda: O.SGD(schedule, momentum=0.9), "adam": lambda: O.Adam(schedule),
            "rmsprop": lambda: O.RMSprop(schedule, momentum=0.5, centered=True),
            "adadelta": lambda: O.Adadelta(schedule)}[name]()


OPTS = ["adadelta", "adam", "rmsprop", "sgd_momentum"]


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("sched", sorted(_schedules()))
def test_device_rate_and_parameters_follow_the_schedule(sched, opt):
    schedule = _schedules()[sched]
    desc = _opt(opt, schedule)
    fo = _fused(desc.to_spec())
    init, grads = _grads(16)
    fo.init_from(init, broadcast_root=None)
    assert _device_lr(fo) == schedule(0)
    ref = [t.clone().requires_grad_(True) for t in init]
    topt = desc.to_torch(ref)
    for step, gs in enumerate(grads):
        for gv, gr, r in zip(fo.grad_views, gs, ref):
            gv.copy_(gr)
            r.grad = gr.clone()
        fo.step()
        for grp in topt.param_groups:
            grp["lr"] = schedule(step)
        topt.step()
        torch.cuda.synchronize()
        assert fo.step_count == step + 1
        assert _device_lr(fo) == schedule(step + 1), (step, _device_lr(fo), schedule(step + 1))
    assert fo.current_lr() == schedule(16)
    st = fo.gather_state()
    for t, r in zip(fo.unflatten(st["master"]), ref):
        torch.testing.assert_close(t, r.detach(), rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("sched", sorted(_schedules()))
def test_split_launches_advance_the_rate_once_per_step(sched):
    schedule = _schedules()[sched]
    from tf_yarn_b200.keras.optimizers import Adam
    whole = _fused(Adam(schedule).to_spec(), zero_grads=False)
    split = _fused(Adam(schedule).to_spec(), zero_grads=False)
    init, grads = _grads(9)
    whole.init_from(init, broadcast_root=None)
    split.init_from(init, broadcast_root=None)
    groups = split.shard_n // 8
    for gs in grads:
        for fo in (whole, split):
            for gv, gr in zip(fo.grad_views, gs):
                gv.copy_(gr)
        whole.step(shard_groups=(0, groups), advance=True)
        split.step(shard_groups=(0, groups // 3), advance=False)
        split.step(shard_groups=(groups // 3, groups), advance=True)
    torch.cuda.synchronize()
    assert split.step_count == 9 and _device_lr(split) == schedule(9) == _device_lr(whole)
    assert torch.equal(split.master, whole.master) and torch.equal(split.s2, whole.s2)


@pytest.mark.parametrize("sched", sorted(_schedules()))
def test_an_installed_or_restored_rate_has_the_bits_the_fused_step_writes(sched):
    """The rate written for a restored step n (set_step_count) is the one the fused step writes advancing from n - 1:
    both come from the same device function."""
    from tf_yarn_b200.keras.optimizers import SGD
    schedule = _schedules()[sched]
    restored, stepped = _fused(SGD(schedule).to_spec()), _fused(SGD(schedule).to_spec())
    steps = list(range(1, 200)) + [1001, 4097, 65537, 10 ** 7]
    got, want = [], []
    for n in steps:
        restored.set_step_count(n)
        stepped.set_step_count(n - 1)
        stepped.flat_grads.zero_()
        stepped.step()
        got.append(restored.hyper[0:4].clone())
        want.append(stepped.hyper[0:4].clone())
    torch.cuda.synchronize()
    assert torch.equal(torch.stack(got), torch.stack(want))
    host = torch.tensor([schedule(n) for n in steps], dtype=torch.float32)
    dev = torch.stack(got).view(torch.float32).reshape(-1).cpu()
    torch.testing.assert_close(dev, host, rtol=2.5e-7, atol=1e-9)


def test_graph_replay_gives_the_bits_of_eager_launches():
    from tf_yarn_b200.keras import schedules as S
    from tf_yarn_b200.keras.optimizers import Adam
    schedule = S.CosineDecay(0.0, 20, warmup_target=0.02, warmup_steps=6)
    init, grads = _grads(1)
    eager, graphed = _fused(Adam(schedule).to_spec(), torch.bfloat16), _fused(Adam(schedule).to_spec(), torch.bfloat16)
    for fo in (eager, graphed):
        fo.init_from(init, broadcast_root=None)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        snap = graphed.hyper.clone(), graphed.master.clone(), graphed.s1.clone(), graphed.s2.clone()
        with torch.cuda.graph(g, stream=s):
            for gv, gr in zip(graphed.grad_views, grads[0]):
                gv.copy_(gr.to(torch.bfloat16))
            graphed.step()
        # capture does not run the step: the state is still the initial one
        assert torch.equal(graphed.hyper, snap[0]) and torch.equal(graphed.master, snap[1])
        for _ in range(25):
            g.replay()
    for _ in range(25):
        for gv, gr in zip(eager.grad_views, grads[0]):
            gv.copy_(gr.to(torch.bfloat16))
        eager.step()
    torch.cuda.synchronize()
    assert graphed.step_count == eager.step_count == 25
    assert _device_lr(graphed) == _device_lr(eager) == schedule(25)
    assert torch.equal(graphed.master, eager.master) and torch.equal(graphed.flat_params, eager.flat_params)
    assert torch.equal(graphed.s1, eager.s1) and torch.equal(graphed.s2, eager.s2)


def test_resume_mid_schedule_continues_it():
    from tf_yarn_b200.keras import schedules as S
    from tf_yarn_b200.keras.optimizers import RMSprop
    schedule = S.PiecewiseConstantDecay([4, 8], [0.01, 0.005, 0.001])
    init, grads = _grads(12)

    def run(fo, gs):
        for g in gs:
            for gv, gr in zip(fo.grad_views, g):
                gv.copy_(gr)
            fo.step()
        torch.cuda.synchronize()

    straight = _fused(RMSprop(schedule, momentum=0.9).to_spec())
    straight.init_from(init, broadcast_root=None)
    run(straight, grads)
    first = _fused(RMSprop(schedule, momentum=0.9).to_spec())
    first.init_from(init, broadcast_root=None)
    run(first, grads[:6])
    st = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in first.gather_state().items()}
    resumed = _fused(RMSprop(schedule, momentum=0.9).to_spec())
    assert _device_lr(resumed) == schedule(0)
    resumed.load_state({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in st.items()})
    torch.cuda.synchronize()
    assert resumed.step_count == 6 and _device_lr(resumed) == schedule(6)
    run(resumed, grads[6:])
    assert _device_lr(resumed) == schedule(12) == _device_lr(straight)
    assert torch.equal(resumed.master, straight.master) and torch.equal(resumed.s2, straight.s2)


def test_a_constant_rate_is_untouched_and_set_lr_is_refused_for_a_schedule():
    from tf_yarn_b200.keras import schedules as S
    from tf_yarn_b200.keras.optimizers import Adam
    from tf_yarn_b200.ops import native
    fo = _fused(Adam(1e-3).to_spec())
    assert fo._code == native.OPT_ADAM
    init, grads = _grads(3)
    fo.init_from(init, broadcast_root=None)
    for g in grads:
        for gv, gr in zip(fo.grad_views, g):
            gv.copy_(gr)
        fo.step()
    torch.cuda.synchronize()
    assert _device_lr(fo) == float(torch.tensor(1e-3, dtype=torch.float32)) and fo.step_count == 3
    fo.set_lr(2e-3)
    torch.cuda.synchronize()
    assert _device_lr(fo) == float(torch.tensor(2e-3, dtype=torch.float32))
    sched = _fused(Adam(S.ExponentialDecay(1e-3, 10, 0.5)).to_spec())
    assert sched._code == native.OPT_ADAM | native.OPT_LR_SCHEDULE
    with pytest.raises(TypeError, match="LearningRateSchedule"):
        sched.set_lr(2e-3)


def _train(make_opt, fast=True, epochs=2):
    import numpy as np
    from tf_yarn_b200 import keras
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
    torch.manual_seed(7)
    m = keras_mnist_cnn()
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=make_opt(),
              use_fast_path=fast)
    rs = np.random.RandomState(0)
    y = rs.randint(0, 10, 512).astype("int64")
    x = (rs.rand(512, 28, 28, 1) * 0.5 + (y[:, None, None, None] / 20.0)).astype("float32")
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    m.fit(torch.from_numpy(x), torch.from_numpy(y), batch_size=128, epochs=epochs, shuffle=False, verbose=0,
          callbacks=[Rec()])
    torch.cuda.synchronize()
    return m, losses


def _fast_opt(name):
    from tf_yarn_b200.keras import optimizers as O
    from tf_yarn_b200.keras import schedules as S
    return {"adam_cosine_warmup": lambda: O.Adam(S.CosineDecay(0.0, 6, warmup_target=1e-3, warmup_steps=2)),
            "rmsprop_exponential": lambda: O.RMSprop(S.ExponentialDecay(1e-3, 2, 0.7)),
            "adadelta_piecewise": lambda: O.Adadelta(S.PiecewiseConstantDecay([3, 5], [1.0, 0.5, 0.1]))}[name]()


@pytest.mark.parametrize("name", ["adadelta_piecewise", "adam_cosine_warmup", "rmsprop_exponential"])
def test_fastpath_follows_the_schedule_at_ten_launches_per_step(name):
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m1, l1 = _train(lambda: _fast_opt(name))
    m2, l2 = _train(lambda: _fast_opt(name))
    eng = m1._engine
    sch = m1.optimizer.schedule
    assert isinstance(eng, FastSequentialEngine) and eng._launches_per_step == 10
    assert eng.fused._code & 0x100
    assert eng.fused.step_count == 8 and _device_lr(eng.fused) == sch(8) and m1.get_learning_rate() == sch(8)
    assert len(l1) == 8 and all(math.isfinite(v) for v in l1)
    assert l1 == l2 and torch.equal(eng.fused.master, m2._engine.fused.master)      # bit reproducible


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_p2p_nvls_and_ddp_fused_schedules_multi_gpu():
    n = min(_ngpu(), 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29631", "tests/gpu/lr_schedule_check.py"]
    res = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert res.returncode == 0 and "LR SCHEDULE CHECK OK" in res.stdout, res.stdout[-4000:]
