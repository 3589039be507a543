"""GPU tests of the Keras Adamax and Nadam in the fused K4 step (run with `pytest -m gpu` on an H100).

LOCAL mode on one GPU: both optimizers for every gradient / parameter dtype pair, with a constant and a scheduled
learning rate and over an fp32 gradient accumulator, against the float64 reference of tests/test_keras_adamax_nadam.py;
a checkpoint resume bit-identical to an uninterrupted run, Nadam's running product included; the MNIST-CNN fast path
against the autograd engine; and the overlap planner's fall-back to the trailing step.  With 2+ GPUs,
tests/gpu/adamax_nadam_check.py covers the P2P and NVLS transports and the DDP wrapper.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_keras_adamax_nadam import CLASSES, NUMPY, nadam_mu

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(33, 17), (129,), (7, 5, 3)]          # 561 + 129 + 105 elements: odd sizes, padded inside the flat buffer
PAIRS = {"bf16_bf16": (torch.bfloat16, torch.bfloat16), "f32_f32": (torch.float32, torch.float32),
         "bf16_f32": (torch.bfloat16, torch.float32), "f32_bf16": (torch.float32, torch.bfloat16)}


def nadam_product(ts, beta_1=0.9):
    """Nadam's running product after the updates at ``ts``, in float64 from beta_1 as the device holds it (fp32)."""
    return float(np.prod([nadam_mu(float(np.float32(beta_1)), t) for t in ts]))


def _fused(spec, param_dtype, grad_dtype, accumulation_steps=None):
    from tf_yarn_b200.keras.engine import _solo_communicator
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    return FusedShardedOptimizer(_solo_communicator(0), SHAPES, spec, param_dtype=param_dtype, grad_dtype=grad_dtype,
                                 accumulation_steps=accumulation_steps)


def _flat(ts):
    return np.concatenate([t.detach().double().cpu().numpy().reshape(-1) for t in ts])


@pytest.mark.parametrize("how", ["constant", "scheduled", "accumulated"])
@pytest.mark.parametrize("pair", sorted(PAIRS))
@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_fused_step_local_matches_the_float64_reference(kind, pair, how):
    from tf_yarn_b200.keras import schedules
    grad_dtype, param_dtype = PAIRS[pair]
    sched = schedules.ExponentialDecay(0.01, decay_steps=5, decay_rate=0.6) if how == "scheduled" else None
    wd = 0.01
    desc = CLASSES[kind](sched if sched is not None else 0.01, weight_decay=wd)
    n_acc = 3 if how == "accumulated" else None
    fo = _fused(desc.to_spec(), param_dtype, grad_dtype, n_acc)
    g = torch.Generator(device="cuda").manual_seed(3)
    init = [torch.randn(s, device="cuda", generator=g) * 0.3 for s in SHAPES]
    fo.init_from(init, broadcast_root=None)
    p0 = _flat(init)
    batches = 30
    grads, lrs, ts, acc = [], [], [], None
    for s in range(batches):
        gs = [(torch.randn(sh, device="cuda", generator=g) * 0.5).to(grad_dtype) for sh in SHAPES]
        for gv, gr in zip(fo.grad_views, gs):
            gv.copy_(gr)
        if n_acc is None:
            fo.step()
            grads.append(_flat(gs))
        else:
            update = (s + 1) % n_acc == 0
            fo.accumulate(advance=not update)
            # the kernel sums the batches in fp32 and scales by fl32(1/N)
            acc = [a + b.float() for a, b in zip(acc, gs)] if acc is not None else [b.float() for b in gs]
            if not update:
                continue
            fo.step_accumulated()
            grads.append(_flat([a * np.float32(1.0 / n_acc) for a in acc]))
            acc = None
        lrs.append(float(sched(s)) if sched is not None else 0.01)
        ts.append(s + 1)
    torch.cuda.synchronize()
    assert fo.step_count == batches
    want = NUMPY[kind](p0, grads, lrs, ts, 0.9, 0.999, 1e-7, wd)
    st = fo.gather_state()
    scale = max(1.0, float(np.abs(want[0]).max()))
    got = _flat(fo.unflatten(st["master"]))
    assert float(np.abs(got - want[0]).max()) < 1e-4 * scale, (kind, pair, how)
    for name, ref in (("s1", want[1]), ("s2", want[2])):
        err = float(np.abs(_flat(fo.unflatten(st[name])) - ref).max())
        assert err < 1e-4 * max(1e-3, float(np.abs(ref).max())), (name, err)
    for pv, t in zip(fo.param_views, fo.unflatten(st["master"])):
        assert torch.equal(pv, t.to(param_dtype))                  # compute params = fp32 master cast down
    if kind == "nadam":
        assert st["mu_product"] == pytest.approx(nadam_product(ts), rel=1e-12, abs=0)
    else:
        assert "mu_product" not in st


@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_gather_and_load_state_resume_is_bit_identical(kind):
    spec = CLASSES[kind](0.01).to_spec()
    g = torch.Generator(device="cuda").manual_seed(5)
    init = [torch.randn(s, device="cuda", generator=g) * 0.3 for s in SHAPES]
    grads = [[torch.randn(s, device="cuda", generator=g) for s in SHAPES] for _ in range(8)]

    def run(fo, steps):
        for gs in steps:
            for gv, gr in zip(fo.grad_views, gs):
                gv.copy_(gr)
            fo.step()
        torch.cuda.synchronize()

    straight = _fused(spec, torch.bfloat16, torch.bfloat16)
    straight.init_from(init, broadcast_root=None)
    run(straight, grads)
    first = _fused(spec, torch.bfloat16, torch.bfloat16)
    first.init_from(init, broadcast_root=None)
    run(first, grads[:3])
    st = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in first.gather_state().items()}
    assert st["step"] == 3 and set(st) >= {"master", "s1", "s2"}
    resumed = _fused(spec, torch.bfloat16, torch.bfloat16)
    resumed.load_state({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in st.items()})
    if kind == "nadam":
        assert resumed.mu_product == first.mu_product != 1.0
    run(resumed, grads[3:])
    assert resumed.step_count == 8
    for name in ("master", "s1", "s2", "flat_params"):
        assert torch.equal(getattr(resumed, name), getattr(straight, name)), name
    if kind == "nadam":
        assert resumed.mu_product == straight.mu_product
    with pytest.raises(ValueError, match=kind.capitalize()):
        straight.overlap_step(0, 8, 4)


def _mnist_like():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="mnist_cnn_adamax_nadam")
    m.add(layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)))
    m.add(layers.Conv2D(64, (3, 3), activation="relu"))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(0.0))
    m.add(layers.Flatten())
    m.add(layers.Dense(128, activation="relu"))
    m.add(layers.Dropout(0.0))
    m.add(layers.Dense(10))
    return m


def _train(kind, fast=True, epochs=2, lr=1e-3):
    """Learnable synthetic MNIST (the label shifts the image brightness), dropout off, fixed seeds."""
    from tf_yarn_b200 import keras
    torch.manual_seed(7)
    m = _mnist_like()
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=CLASSES[kind](lr),
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


@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_fastpath_learns_and_tracks_the_autograd_engine(kind):
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m_fast, l_fast = _train(kind)
    eng = m_fast._engine
    assert isinstance(eng, FastSequentialEngine) and eng.fused.spec.kind == kind
    assert eng._launches_per_step == 10
    assert len(l_fast) == 8 and all(math.isfinite(v) for v in l_fast)
    assert sum(l_fast[-4:]) < sum(l_fast[:4]), l_fast                 # loss falls
    if kind == "nadam":
        assert eng.fused.mu_product == pytest.approx(nadam_product(range(1, 9)), rel=1e-12, abs=0)
    # Adam-family first increments are sign-like (about lr * sign(g) whatever |g|), so bf16 noise that flips a
    # near-zero gradient moves that weight by whole increments.  With lr = 1e-4 those moves stay on the scale the
    # fast-path-vs-autograd tolerance was set for.
    m_ref, l_ref = _train(kind, fast=False, epochs=1, lr=1e-4)
    m_fast, l_fast = _train(kind, fast=True, epochs=1, lr=1e-4)
    assert not isinstance(m_ref._engine, FastSequentialEngine)
    for a, b in zip(l_fast, l_ref):
        assert abs(a - b) < 0.03 * max(1.0, abs(b)), (l_fast, l_ref)
    for a, b in zip(m_fast.get_weights(), m_ref.get_weights()):
        a, b = torch.as_tensor(a), torch.as_tensor(b)
        denom = b.abs().max().clamp_min(2e-2)
        assert ((a - b).abs().max() / denom) < 0.15, ((a - b).abs().max(), denom)


@pytest.mark.parametrize("kind", ["adamax", "nadam"])
def test_overlap_opt_in_falls_back_to_the_trailing_step(monkeypatch, kind):
    monkeypatch.setenv("TFY_OVERLAP", "0")
    m0, l0 = _train(kind)
    monkeypatch.setenv("TFY_OVERLAP", "1")
    monkeypatch.setenv("TFY_OVERLAP_GROUPS", "20000")
    m1, l1 = _train(kind)
    eng = m1._engine
    assert eng._overlap and eng._ov_gmid == 0, f"{kind} must not take the overlap role"
    assert eng.fused.step_count == 8
    assert l0 == l1 and torch.equal(m0._engine.fused.master, eng.fused.master)


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_p2p_nvls_and_ddp_fused_adamax_nadam_multi_gpu():
    counts = sorted({2, min(_ngpu(), 8)})
    for n in counts:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
               "--master-addr", "127.0.0.1", "--master-port", "29637", "tests/gpu/adamax_nadam_check.py"]
        res = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
        assert res.returncode == 0 and "ADAMAX NADAM CHECK OK" in res.stdout, res.stdout[-4000:]
