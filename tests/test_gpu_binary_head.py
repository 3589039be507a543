"""GPU tests of the binary (Keras BinaryCrossentropy) classifier head.

* tfy_dense_head_fused_binary and tfy_sigmoid_xent against the float64 reference of tests/binary_xent_reference.py:
  every output within the bound derived there, in EPS32 = 2^-24 terms -- a K-term fp32 logit carries (K + 1) EPS32
  sum|h w| (EPS32 |z| for the fallback's bf16 logits), the accurate expf / log1pf 2 EPS32 each, the loss (C + B + 40)
  EPS32 sum|w l| / B for its fixed-order sums, dz 6 EPS32 sigmoid plus the propagated logit and target errors, and
  every bf16 output 2^-8 of its value, all doubled for headroom.  Guard bytes around the outputs are intact.
* Exact checks: the operands lie on a grid of multiples of 1/8 and 1/16, which fp32 sums without rounding, so the
  kernels' logits are exact and their hit counts equal the reference's; two launches give the same bits; a CUDA-graph
  replay gives the launch's bits.  Logits out to |z| = 80 give a finite loss and no NaN.
* The fast path: the MNIST CNN with a Dense(1, sigmoid) head and an MLP with a multi-label Dense(10, sigmoid) head
  track the autograd engine (use_fast_path=False) under SGD: every step's loss within 0.05, the final weights within
  5 % in L2, the last two Dense layers' kernels within 10 % and their biases' largest difference within 15 % of their
  scale or 0.0075, the epoch accuracy within 0.02; sample / class
  weights and gradient accumulation under an ExponentialDecay rate keep the softmax head's launch counts;
  save -> load_model -> resume equals an uninterrupted run.
"""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import binary_xent_reference as ref  # noqa: E402

pytestmark = pytest.mark.gpu
GUARD = 64                 # guard elements after every output
# (targets, label smoothing, weighting, model output is the sigmoid)
CASES = [("hard", 0.0, "none", True), ("hard", 0.1, "sample", False), ("soft", 0.0, "class", True),
         ("soft", 0.1, "both", False), ("hard", 0.0, "class", False), ("soft", 0.1, "none", True)]
CASE_IDS = ["-".join(str(f) for f in c) for c in CASES]
BATCHES = (1, 15, 16, 17, 128, 4099)


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(shape, dtype):
    n = int(np.prod(shape)) if shape else 1
    full = torch.full((n + GUARD,), -7.0, dtype=dtype, device="cuda")
    return full, full[:n].view(shape)


def _guards_intact(bufs):
    for full, view in bufs:
        assert bool((full[view.numel():] == -7.0).all()), "an output was written past its end"


def _grid(shape, g, scale, lim, step):
    """Normal values rounded to multiples of ``step``, within +-lim."""
    return ((torch.randn(shape, device="cuda", generator=g) * scale / step).round().clamp(-lim / step, lim / step)
            * step)


def _targets(B, C, case, g):
    kind, ls, weighting, sig = case
    if kind == "hard":
        y = torch.randint(0, 2, (B, C), device="cuda", generator=g).float()
    else:
        y = torch.rand(B, C, device="cuda", generator=g)
    if C == 1 and B % 2:
        y = y.reshape(B)                    # [B] targets when C = 1 (odd batches)
    sw = torch.rand(B, device="cuda", generator=g) * 2 if weighting in ("sample", "both") else None
    cw = torch.rand(max(C, 2), device="cuda", generator=g) * 3 if weighting in ("class", "both") else None
    return y.contiguous(), ls, sw, cw, sig


def _check(name, got, want, bound):
    err = np.abs(got.double().cpu().numpy().reshape(np.shape(want)) - want)
    bad = err > bound
    assert not bad.any(), (name, float(err.max()), float(np.max(err / np.maximum(bound, 1e-300))))


def _check_stats(stats, want, B, C, weighted, n_runs):
    # grid operands: the kernel's fp32 logits are the reference's, so its hits are the reference's exactly (a logit
    # of 0 gives a sigmoid of exactly 0.5 in both, a logit of exactly 0.5 compares equal in both)
    assert stats[0].item() == n_runs * int(want["hits"][2].sum())
    assert stats[1].item() == n_runs * B * C
    if weighted:                             # (the kernel adds to the -7 the two sums start from)
        assert stats[2].item() + 7.0 == pytest.approx(n_runs * want["w_hits"], rel=1e-5, abs=1e-4)
        assert stats[3].item() + 7.0 == pytest.approx(n_runs * want["w"].sum(), rel=1e-5, abs=1e-4)
    else:
        assert stats[2].item() == -7.0 and stats[3].item() == -7.0, "the unweighted kernel writes 2 stats"


# ------------------------------------------------------------------------------------------------ fused head
def _head_operands(B, K, C, case, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    h = _grid((B, K), g, 1.0, 2.0, 1 / 8).relu().bfloat16()
    w2 = _grid((C, K), g, 0.2, 0.5, 1 / 16).bfloat16()
    b2 = _grid((C,), g, 0.5, 2.0, 1 / 8).bfloat16()
    mask = (torch.rand(B, K, device="cuda", generator=g) > 0.4).to(torch.uint8)
    return (h, w2, b2, mask) + _targets(B, C, case, g)


class _HeadOut:
    def __init__(self, lib, B, K, C):
        self.loss = _guarded((), torch.float32)
        self.stats = torch.tensor([0.0, 0.0, -7.0, -7.0], device="cuda")
        self.dw2 = _guarded((C, K), torch.bfloat16)
        self.db2 = _guarded((C,), torch.bfloat16)
        self.dh = _guarded((B, K), torch.bfloat16)
        self.db1 = _guarded((K,), torch.bfloat16)
        self.scratch = torch.zeros(int(lib.tfy_dense_head_scratch_elems(K, C, B)), device="cuda")
        self.counter = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.host = torch.zeros(1, dtype=torch.float32).pin_memory()

    def tail(self):
        return (self.loss[1].data_ptr(), self.host.data_ptr(), self.stats.data_ptr(), self.dw2[1].data_ptr(),
                self.db2[1].data_ptr(), self.dh[1].data_ptr(), self.db1[1].data_ptr(), self.scratch.data_ptr(),
                self.counter.data_ptr())

    def outputs(self):
        return [self.loss[1].clone(), self.dw2[1].clone(), self.db2[1].clone(), self.dh[1].clone(), self.db1[1].clone()]

    def bufs(self):
        return [self.loss, self.dw2, self.db2, self.dh, self.db1]


def _binary_head(lib, o, h, w2, b2, y, ls, sig, mask, scale, sw, cw, B, K, C):
    return lib.tfy_dense_head_fused_binary(
        h.data_ptr(), w2.data_ptr(), b2.data_ptr(), y.data_ptr(), ctypes.c_float(ls), int(sig),
        mask.data_ptr() if mask is not None else None, ctypes.c_float(scale), *o.tail(), B, K, C,
        sw.data_ptr() if sw is not None else None, cw.data_ptr() if cw is not None else None, _stream())


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("B,K,C", [(B, K, C) for B in BATCHES for K in (128, 256, 512) for C in (1, 3, 16)])
def test_fused_binary_head_matches_the_float64_reference(lib, B, K, C, case):
    h, w2, b2, mask, y, ls, sw, cw, sig = _head_operands(B, K, C, case, seed=B * 7 + K + C + CASES.index(case))
    o = _HeadOut(lib, B, K, C)
    runs = []
    for _ in range(2):
        assert _binary_head(lib, o, h, w2, b2, y, ls, sig, mask, 2.0, sw, cw, B, K, C) == 0
        torch.cuda.synchronize()
        runs.append(o.outputs())
        assert bool((o.scratch == 0).all()) and int(o.counter.item()) == 0
    for a, b in zip(*runs):                  # fixed-order sums: the same bits on every launch
        assert torch.equal(a, b)
    assert o.host.item() == o.loss[1].item()             # the pinned host copy of the loss
    _guards_intact(o.bufs())
    want = ref.fused_head(h, w2, b2, y, ls, mask, 2.0, sw, cw, sig)
    _check("loss", o.loss[1], want["loss"], want["loss_bound"])
    for name in ("dw2", "db2", "dh", "db1"):
        _check(name, getattr(o, name)[1], want[name], want[name + "_bound"])
    _check_stats(o.stats, want, B, C, sw is not None or cw is not None, n_runs=2)


def test_fused_binary_head_replays_in_a_cuda_graph(lib):
    B, K, C = 128, 128, 1
    h, w2, b2, mask, y, ls, sw, cw, sig = _head_operands(B, K, C, CASES[3], seed=5)
    o = _HeadOut(lib, B, K, C)
    assert _binary_head(lib, o, h, w2, b2, y, ls, sig, mask, 2.0, sw, cw, B, K, C) == 0
    torch.cuda.synchronize()
    direct = o.outputs()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert _binary_head(lib, o, h, w2, b2, y, ls, sig, mask, 2.0, sw, cw, B, K, C) == 0
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(direct, o.outputs()):
        assert torch.equal(a, b)
    assert bool((o.scratch == 0).all()) and int(o.counter.item()) == 0


@pytest.mark.parametrize("sig", [True, False])
def test_fused_binary_head_is_finite_at_extreme_logits(lib, sig):
    B, K, C = 64, 128, 3
    g = torch.Generator(device="cuda").manual_seed(11)
    h = torch.zeros(B, K, device="cuda").bfloat16()
    w2 = torch.zeros(C, K, device="cuda").bfloat16()
    b2 = torch.tensor([80.0, -80.0, 40.0], device="cuda").bfloat16()       # |z| up to 80
    y = torch.randint(0, 2, (B, C), device="cuda", generator=g).float()
    o = _HeadOut(lib, B, K, C)
    assert _binary_head(lib, o, h, w2, b2, y, 0.1, sig, None, 1.0, None, None, B, K, C) == 0
    torch.cuda.synchronize()
    for t in o.outputs():
        assert bool(torch.isfinite(t.float()).all())
    want = ref.fused_head(h, w2, b2, y, 0.1, None, 1.0, None, None, sig)
    _check("loss", o.loss[1], want["loss"], want["loss_bound"])
    _check("db2", o.db2[1], want["db2"], want["db2_bound"])
    assert o.stats[0].item() == want["hits"][0]


def test_binary_entry_points_refuse_bad_arguments(lib):
    B, K, C = 16, 128, 3
    h, w2, b2, mask, y, _, _, _, _ = _head_operands(B, K, C, CASES[0], seed=1)
    o = _HeadOut(lib, B, K, C)
    for ls in (-0.1, 1.5, float("nan")):
        assert _binary_head(lib, o, h, w2, b2, y, ls, True, mask, 1.0, None, None, B, K, C) == -2
    assert _binary_head(lib, o, h, w2, b2, y, 0.0, True, mask, 1.0, None, None, B, 64, C) == -2     # K
    assert _binary_head(lib, o, h, w2, b2, y, 0.0, True, mask, 1.0, None, None, B, K, 17) == -2     # C > 16
    lg = torch.zeros(B, C, dtype=torch.bfloat16, device="cuda")
    rest = (None, None, o.loss[1].data_ptr(), o.dh[1].data_ptr(), None, None)
    assert lib.tfy_sigmoid_xent(lg.data_ptr(), None, y.data_ptr(), ctypes.c_float(2.0), 1, *rest, B, C,
                                _stream()) == -2
    assert lib.tfy_sigmoid_xent(lg.data_ptr(), None, None, ctypes.c_float(0.0), 1, *rest, B, C, _stream()) == -2
    assert lib.tfy_sigmoid_xent(lg.data_ptr(), None, y.data_ptr(), ctypes.c_float(0.0), 1, *rest, 1 << 16, 1 << 16,
                                _stream()) == -2
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ fallback
def _fallback_operands(B, C, case, seed, lim=8.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lg = _grid((B, C), g, 3.0, lim, 1 / 8).bfloat16()
    bx = _grid((C,), g, 0.5, 2.0, 1 / 8).bfloat16()
    return (lg, bx) + _targets(B, C, case, g)


def _sigmoid_xent(lib, lg, bx, y, ls, sig, sw, cw, bufs, B, C):
    loss, dl, db, stats = bufs
    return lib.tfy_sigmoid_xent(lg.data_ptr(), bx.data_ptr(), y.data_ptr(), ctypes.c_float(ls), int(sig),
                                sw.data_ptr() if sw is not None else None, cw.data_ptr() if cw is not None else None,
                                loss[1].data_ptr(), dl[1].data_ptr(), db[1].data_ptr(), stats.data_ptr(), B, C,
                                _stream())


def _xent_bufs(B, C):
    return (_guarded((), torch.float32), _guarded((B, C), torch.bfloat16), _guarded((C,), torch.bfloat16),
            torch.tensor([0.0, 0.0, -7.0, -7.0], device="cuda"))


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("B,C", [(B, C) for B in BATCHES for C in (1, 40)])
def test_sigmoid_xent_fallback_matches_the_float64_reference(lib, B, C, case):
    lg, bx, y, ls, sw, cw, sig = _fallback_operands(B, C, case, seed=B * 5 + C + CASES.index(case))
    bufs = _xent_bufs(B, C)
    runs = []
    for _ in range(2):
        assert _sigmoid_xent(lib, lg, bx, y, ls, sig, sw, cw, bufs, B, C) == 0
        torch.cuda.synchronize()
        runs.append([b[1].clone() for b in bufs[:3]])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    _guards_intact(bufs[:3])
    want = ref.sigmoid_xent_fallback(lg, bx, y, ls, sw, cw, sig)
    _check("loss", bufs[0][1], want["loss"], want["loss_bound"])
    _check("dlogits", bufs[1][1], want["dlogits"], want["dlogits_bound"])
    _check("dbias", bufs[2][1], want["dbias"], want["dbias_bound"])
    _check_stats(bufs[3], want, B, C, sw is not None or cw is not None, n_runs=2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert _sigmoid_xent(lib, lg, bx, y, ls, sig, sw, cw, bufs, B, C) == 0
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(runs[0], [b[1] for b in bufs[:3]]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("sig", [True, False])
def test_sigmoid_xent_fallback_is_finite_at_extreme_logits(lib, sig):
    B, C = 257, 40
    lg, bx, y, _, _, _, _ = _fallback_operands(B, C, CASES[0], seed=3, lim=80.0)
    lg = (lg.float() * 16).clamp(-80, 80).bfloat16()                     # |z| out to 80
    bufs = _xent_bufs(B, C)
    assert _sigmoid_xent(lib, lg, bx, y, 0.1, sig, None, None, bufs, B, C) == 0
    torch.cuda.synchronize()
    for b in bufs[:3]:
        assert bool(torch.isfinite(b[1].float()).all())
    want = ref.sigmoid_xent_fallback(lg, bx, y, 0.1, None, None, sig)
    _check("loss", bufs[0][1], want["loss"], want["loss_bound"])
    _check("dlogits", bufs[1][1], want["dlogits"], want["dlogits_bound"])


# ------------------------------------------------------------------------------------------------ the fast path
def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _mnist_binary(dropout=0.0):
    """The MNIST CNN with a Dense(1, sigmoid) head (its dropout rates at 0 by default: the fast path and the autograd
    engine draw different masks)."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    return keras.Sequential([layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)),
                             layers.Conv2D(64, (3, 3), activation="relu"), layers.MaxPooling2D(pool_size=(2, 2)),
                             layers.Dropout(dropout), layers.Flatten(), layers.Dense(128, activation="relu"),
                             layers.Dropout(2 * dropout), layers.Dense(1, activation="sigmoid")])


def _mlp_multilabel():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    return keras.Sequential([layers.Dense(128, activation="relu", input_shape=(256,)),
                             layers.Dense(10, activation="sigmoid")])


def _mnist_data(steps):
    from tf_yarn_b200.models.mnist_cnn import synthetic_mnist
    x, y = synthetic_mnist(128 * steps, seed=3)
    return x, (torch.as_tensor(y) >= 5).float()


def _multilabel_data(steps):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(128 * steps, 256, generator=g)
    proj = torch.randn(256, 10, generator=g)
    return x, (x @ proj > 0).float()


def _fit(build, x, y, loss, fast=True, opt=None, seed=7, **fit_kw):
    from tf_yarn_b200 import keras
    torch.manual_seed(seed)
    m = build()
    m.compile(loss=loss, optimizer=opt or keras.optimizers.SGD(0.05), metrics=["accuracy"], use_fast_path=fast,
              weighted_metrics=["accuracy"] if fit_kw else None)
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    hist = m.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0, callbacks=[Rec()], **fit_kw)
    torch.cuda.synchronize()
    return m, losses, hist.history


def _tracks(fast, slow, loss_tol, weight_tol):
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    (mf, lf, hf), (ms, ls_, hs) = fast, slow
    assert isinstance(mf._engine, FastSequentialEngine) and not isinstance(ms._engine, FastSequentialEngine)
    assert len(lf) == len(ls_)
    diffs = [abs(a - b) for a, b in zip(lf, ls_)]
    print("max / mean loss difference", max(diffs), sum(diffs) / len(diffs))
    assert all(math.isfinite(a) for a in lf)
    assert max(diffs) < loss_tol, (max(diffs), lf[-5:], ls_[-5:])
    wf = [torch.as_tensor(a).float() for a in mf.get_weights()]
    ws = [torch.as_tensor(b).float() for b in ms.get_weights()]
    flat_f, flat_s = torch.cat([a.reshape(-1) for a in wf]), torch.cat([b.reshape(-1) for b in ws])
    rel = float((flat_f - flat_s).norm() / flat_s.norm())
    print("all weights", rel)
    assert rel < weight_tol, rel
    # each tensor of the last two Dense layers, whose gradients the head kernel computes: kernels within 10 % in L2;
    # biases, which 200 SGD steps move by a few 1e-3 only, within 15 % of their scale or 0.0075 (the per-step bf16
    # noise of their batch sums adds up to about 0.004)
    for a, b in zip(wf[-4:], ws[-4:]):
        rel = float((a - b).norm() / b.norm().clamp_min(1e-3))
        scaled = float((a - b).abs().max() / b.abs().max().clamp_min(0.05))
        print("weight difference", tuple(a.shape), rel, scaled, float(b.abs().max()))
        assert (rel < 2 * weight_tol) if a.dim() > 1 else (scaled < 0.15), (tuple(a.shape), rel, scaled)
    for k in hf:
        print("history", k, hf[k], hs[k])
        assert abs(hf[k][0] - hs[k][0]) < (0.02 if "acc" in k else loss_tol), (k, hf[k], hs[k])


@pytest.mark.parametrize("probability", [True, False], ids=["sigmoid_layer", "from_logits"])
def test_binary_mnist_fastpath_tracks_the_autograd_engine(probability):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    x, y = _mnist_data(200)
    if probability:
        build, loss = _mnist_binary, keras.losses.BinaryCrossentropy(label_smoothing=0.05)
    else:
        build = lambda: keras.Sequential(_mnist_binary().layers[:-1] + [layers.Dense(1)])  # noqa: E731
        loss = keras.losses.BinaryCrossentropy(from_logits=True)
    fast = _fit(build, x, y, loss)
    slow = _fit(build, x, y, loss, fast=False)
    assert fast[0]._engine._launches_per_step == 10
    _tracks(fast, slow, loss_tol=0.05, weight_tol=0.05)


def test_multilabel_fastpath_tracks_the_autograd_engine():
    from tf_yarn_b200 import keras
    x, y = _multilabel_data(300)
    loss = keras.losses.BinaryCrossentropy(label_smoothing=0.1)
    fast = _fit(_mlp_multilabel, x, y, loss)
    slow = _fit(_mlp_multilabel, x, y, loss, fast=False)
    _tracks(fast, slow, loss_tol=0.05, weight_tol=0.05)


@pytest.mark.parametrize("weights", ["sample", "class", "both"])
def test_weighted_binary_fastpath_keeps_ten_launches_and_tracks_the_autograd_engine(weights):
    from tf_yarn_b200 import keras
    x, y = _mnist_data(100)
    kw = {}
    if weights in ("sample", "both"):
        kw["sample_weight"] = torch.rand(len(y), generator=torch.Generator().manual_seed(4)) * 2
    if weights in ("class", "both"):
        kw["class_weight"] = {0: 0.5, 1: 2.0}
    loss = keras.losses.BinaryCrossentropy(label_smoothing=0.05)
    fast = _fit(_mnist_binary, x, y, loss, **kw)
    slow = _fit(_mnist_binary, x, y, loss, fast=False, **kw)
    assert fast[0]._engine._launches_per_step == 10 and fast[0]._engine._wmode != (False, False)
    _tracks(fast, slow, loss_tol=0.05, weight_tol=0.05)


def test_binary_fastpath_under_gradient_accumulation_and_a_schedule_keeps_its_launch_counts():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import schedules
    x, y = _mnist_data(8)
    opt = keras.optimizers.Adam(schedules.ExponentialDecay(1e-3, 2, 0.9), gradient_accumulation_steps=4)
    m, losses, _ = _fit(lambda: _mnist_binary(0.25), x, y, keras.losses.BinaryCrossentropy(label_smoothing=0.1),
                        opt=opt, sample_weight=torch.rand(len(y), generator=torch.Generator().manual_seed(2)))
    eng = m._engine
    assert eng._launches_per_step == 11 and eng._launches_per_accum_step == 10
    assert all(math.isfinite(v) for v in losses)


def test_binary_save_load_resume_equals_an_uninterrupted_run(tmp_path):
    from tf_yarn_b200 import keras
    x, y = _mnist_data(12)
    loss = keras.losses.BinaryCrossentropy(label_smoothing=0.05)
    make = lambda: keras.optimizers.Adam(1e-3)  # noqa: E731

    def model():
        torch.manual_seed(7)
        m = _mnist_binary(0.25)
        m.compile(loss=loss, optimizer=make(), metrics=["accuracy"])
        return m
    straight = model()
    straight.fit(x, y, batch_size=128, epochs=2, shuffle=False, verbose=0)
    first = model()
    first.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0)
    path = str(tmp_path / "m.tfy")
    first.save(path)
    loaded = keras.models.load_model(path)
    loaded.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0)
    torch.cuda.synchronize()
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    assert isinstance(loaded._engine, FastSequentialEngine)
    for a, b in zip(loaded.get_weights(), straight.get_weights()):
        assert torch.equal(_bits(torch.as_tensor(a)), _bits(torch.as_tensor(b)))


def test_binary_targets_of_the_wrong_shape_are_refused():
    from tf_yarn_b200 import keras
    x, _ = _mnist_data(2)
    with pytest.raises(ValueError, match=r"\(128, 3\).*\(batch, 1\)"):
        _fit(_mnist_binary, x, torch.zeros(256, 3), keras.losses.BinaryCrossentropy())
