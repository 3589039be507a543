"""GPU tests of the Keras RMSprop in the fused K4 step (run with `pytest -m gpu` on an H100).

LOCAL mode on one GPU: every variant (plain, momentum, centered, both) against TorchRMSprop in fp32, through the full,
element-range and shard-group launches; the sharded-state checkpoint with its third state; the MNIST-CNN fast path
(learning, bit reproducibility, agreement with the autograd engine); and the overlap planner's fall-back to the
trailing step.  With 2+ GPUs, tests/gpu/rmsprop_check.py covers the P2P and NVLS transports and the DDP wrapper.
"""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = {
    "plain": dict(momentum=0.0, centered=False),
    "momentum": dict(momentum=0.9, centered=False),
    "centered": dict(momentum=0.0, centered=True),
    "momentum_centered": dict(momentum=0.9, centered=True),
}
SHAPES = [(33, 17), (129,), (7, 5, 3)]          # 561 + 129 + 105 elements: odd sizes, padded inside the flat buffer


def _fused(spec, dtype, zero_grads=True):
    from tf_yarn_b200.keras.engine import _solo_communicator
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    return FusedShardedOptimizer(_solo_communicator(0), SHAPES, spec, param_dtype=dtype, grad_dtype=dtype,
                                 zero_grads=zero_grads)


def _launch(fo, how):
    if how == "full":
        fo.step()
    elif how == "elem_range":
        mid = 600                                            # inside the second tensor
        fo.step(elem_range=(0, mid), advance=False)
        fo.step(elem_range=(mid, fo.n), advance=True)
    else:
        groups = fo.shard_n // 8
        fo.step(shard_groups=(0, groups // 3), advance=False)
        fo.step(shard_groups=(groups // 3, groups), advance=True)


@pytest.mark.parametrize("how", ["full", "elem_range", "shard_groups"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_fused_step_local_matches_torch_rmsprop(variant, dtype, how):
    from tf_yarn_b200.keras.optimizers import RMSprop
    desc = RMSprop(1e-3, rho=0.9, epsilon=1e-7, weight_decay=0.01, **VARIANTS[variant])
    spec = desc.to_spec()
    fo = _fused(spec, dtype, zero_grads=(how == "full"))
    assert fo.s2.numel() == max(8, fo.shard_n * (spec.n_states - 1))
    g = torch.Generator(device="cuda").manual_seed(3)
    init = [torch.randn(s, device="cuda", generator=g) * 0.3 for s in SHAPES]
    fo.init_from(init, broadcast_root=None)
    ref = [t.clone().requires_grad_(True) for t in init]
    opt = desc.to_torch(ref)
    for step in range(20):
        # the reference sees exactly the gradient the kernel reads (bf16-rounded in the bf16 case)
        grads = [(torch.randn(s, device="cuda", generator=g) * 0.5).to(dtype) for s in SHAPES]
        for gv, gr, r in zip(fo.grad_views, grads, ref):
            gv.copy_(gr)
            r.grad = gr.float()
        _launch(fo, how)
        opt.step()
    torch.cuda.synchronize()
    assert fo.step_count == 20
    st = fo.gather_state()
    assert set(st) == {"master", "step"} | {f"s{i}" for i in range(1, spec.n_states + 1)}
    for t, r in zip(fo.unflatten(st["master"]), ref):
        torch.testing.assert_close(t, r.detach(), rtol=1e-4, atol=1e-5)
    for pv, t in zip(fo.param_views, fo.unflatten(st["master"])):
        assert torch.equal(pv, t.to(dtype))                  # compute params = fp32 master cast down
    names = ["v"] + [k for k, on in (("m", VARIANTS[variant]["momentum"] > 0), ("mg", VARIANTS[variant]["centered"]))
                     if on]
    for i, name in enumerate(names, start=1):
        for t, r in zip(fo.unflatten(st[f"s{i}"]), ref):
            torch.testing.assert_close(t, opt.state[r][name], rtol=1e-4, atol=1e-6)


def test_gather_and_load_state_round_trip_keeps_the_third_state():
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    spec = OptimizerSpec.rmsprop(1e-3, 0.9, 0.9, 1e-7, centered=True)
    g = torch.Generator(device="cuda").manual_seed(5)
    init = [torch.randn(s, device="cuda", generator=g) * 0.3 for s in SHAPES]
    grads = [[torch.randn(s, device="cuda", generator=g) for s in SHAPES] for _ in range(6)]

    def run(fo, steps):
        for gs in steps:
            for gv, gr in zip(fo.grad_views, gs):
                gv.copy_(gr)
            fo.step()
        torch.cuda.synchronize()

    straight = _fused(spec, torch.float32)
    straight.init_from(init, broadcast_root=None)
    run(straight, grads)
    first = _fused(spec, torch.float32)
    first.init_from(init, broadcast_root=None)
    run(first, grads[:3])
    st = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in first.gather_state().items()}
    assert st["step"] == 3 and st["s2"].numel() == st["s3"].numel() == first.shard_n
    assert float(st["s2"].abs().max()) > 0 and float(st["s3"].abs().max()) > 0
    assert not torch.equal(st["s2"], st["s3"])
    resumed = _fused(spec, torch.float32)
    resumed.load_state({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in st.items()})
    assert torch.equal(resumed.s2.cpu(), first.s2.cpu())
    run(resumed, grads[3:])
    assert resumed.step_count == 6
    assert torch.equal(resumed.master, straight.master) and torch.equal(resumed.s2, straight.s2)


def _mnist_like():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="mnist_cnn_rmsprop")
    m.add(layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)))
    m.add(layers.Conv2D(64, (3, 3), activation="relu"))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(0.0))
    m.add(layers.Flatten())
    m.add(layers.Dense(128, activation="relu"))
    m.add(layers.Dropout(0.0))
    m.add(layers.Dense(10))
    return m


def _train(fast=True, epochs=3, lr=1e-3):
    """Learnable synthetic MNIST (the label shifts the image brightness), dropout off, fixed seeds."""
    import numpy as np
    from tf_yarn_b200 import keras
    torch.manual_seed(7)
    m = _mnist_like()
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True),
              optimizer=keras.optimizers.RMSprop(lr, momentum=0.9, centered=True), use_fast_path=fast)
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


def test_fastpath_rmsprop_learns_reproducibly_and_tracks_the_autograd_engine():
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m1, l1 = _train()
    m2, l2 = _train()
    assert isinstance(m1._engine, FastSequentialEngine) and m1._engine.fused.spec.kind == "rmsprop"
    assert m1._engine.fused.spec.n_states == 3
    assert len(l1) == 12 and all(math.isfinite(v) for v in l1)
    assert sum(l1[-4:]) < sum(l1[:4]), l1                            # loss falls
    assert l1 == l2, (l1, l2)                                        # bit-identical losses ...

    def bits(t):
        return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)
    assert torch.equal(bits(m1._engine.fused.flat_params), bits(m2._engine.fused.flat_params))
    assert torch.equal(bits(m1._engine.fused.master), bits(m2._engine.fused.master))   # ... and parameters
    assert torch.equal(bits(m1._engine.fused.s2), bits(m2._engine.fused.s2))

    # RMSprop's early increments are sign-like (the first centered one is 3.3 lr sign(g) whatever |g|) and the
    # momentum buffer carries them on, so bf16 noise that flips a near-zero gradient moves that weight by several
    # increments.  With lr = 1e-4 those moves stay on the scale the fast-path-vs-autograd tolerance was set for.
    m_ref, l_ref = _train(fast=False, epochs=1, lr=1e-4)
    m_fast, l_fast = _train(fast=True, epochs=1, lr=1e-4)
    assert not isinstance(m_ref._engine, FastSequentialEngine)
    for a, b in zip(l_fast, l_ref):
        assert math.isfinite(a) and abs(a - b) < 0.03 * max(1.0, abs(b)), (l_fast, l_ref)
    for a, b in zip(m_fast.get_weights(), m_ref.get_weights()):
        a, b = torch.as_tensor(a), torch.as_tensor(b)
        denom = b.abs().max().clamp_min(2e-2)
        assert ((a - b).abs().max() / denom) < 0.15, ((a - b).abs().max(), denom)


def test_overlap_opt_in_falls_back_to_the_trailing_step(monkeypatch):
    from tf_yarn_b200.parallel.optspec import OptimizerSpec
    with pytest.raises(ValueError, match="RMSprop"):
        _fused(OptimizerSpec.rmsprop(), torch.bfloat16, zero_grads=False).overlap_step(0, 8, 4)
    monkeypatch.setenv("TFY_OVERLAP", "0")
    m0, l0 = _train(epochs=2)
    monkeypatch.setenv("TFY_OVERLAP", "1")
    monkeypatch.setenv("TFY_OVERLAP_GROUPS", "20000")
    m1, l1 = _train(epochs=2)
    eng = m1._engine
    assert eng._overlap and eng._ov_gmid == 0, "RMSprop must not take the overlap role"
    assert eng.fused.step_count == 8
    assert sum(l1[-4:]) < sum(l1[:4]), l1
    assert l0 == l1 and torch.equal(m0._engine.fused.master, eng.fused.master)


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_p2p_nvls_and_ddp_fused_rmsprop_multi_gpu():
    n = min(_ngpu(), 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29627", "tests/gpu/rmsprop_check.py"]
    res = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert res.returncode == 0 and "RMSPROP CHECK OK" in res.stdout, res.stdout[-4000:]
