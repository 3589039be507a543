"""GPU tests of the dense-target (Keras CategoricalCrossentropy, label_smoothing) classifier head.

* tfy_dense_head_fused_soft and tfy_softmax_xent_soft against the float64 reference of tests/soft_xent_reference.py,
  within the bound derived there: every output, guard bytes around them, three launches with the same bits and a
  CUDA-graph replay.
* One-hot targets with ls = 0 give every output of the sparse kernels bit for bit, weighted and unweighted.
* The fast path: the MNIST CNN fitted on to_categorical(y) with CategoricalCrossentropy trains to the same bits as
  with SparseCategoricalCrossentropy on y (with and without sample / class weights; on 2 GPUs through
  tests/gpu/categorical_head_check.py); label smoothing tracks the autograd engine; int32 / uint8 labels train like
  int64 ones.
"""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import soft_xent_reference as ref  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 64                 # guard elements after every output
CASES = ["plain", "mask_weights_ls_onehot", "mask_weights_ls_soft", "ls_soft_unweighted"]


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(shape, dtype):
    """Output buffer with GUARD trailing elements of a fixed pattern; returns (full buffer, view)."""
    n = int(np.prod(shape)) if shape else 1
    full = torch.full((n + GUARD,), -7.0, dtype=dtype, device="cuda")
    return full, full[:n].view(shape)


def _guards_intact(bufs):
    for full, view in bufs:
        tail = full[view.numel():]
        assert bool((tail == -7.0).all()), "an output was written past its end"


def _inputs(B, C, case, g, onehot=None):
    """Targets [B, C], ls, sample / class weights of a case."""
    labels = torch.randint(0, C, (B,), device="cuda", generator=g)
    soft = case.endswith("soft") if onehot is None else not onehot
    if soft:                                # unnormalised soft targets (rows do not sum to 1)
        y = torch.rand(B, C, device="cuda", generator=g) * 1.5
    else:
        y = torch.nn.functional.one_hot(labels, C).float()
    ls = 0.1 if "ls" in case else 0.0
    weighted = "weights" in case
    sw = torch.rand(B, device="cuda", generator=g) * 2 if weighted else None
    cw = torch.rand(C, device="cuda", generator=g) * 3 if weighted else None
    return labels, y.contiguous(), ls, sw, cw


def _check(name, got, want, bound):
    err = np.abs(got.double().cpu().numpy().reshape(np.shape(want)) - want)
    bad = err > bound
    assert not bad.any(), (name, float(err.max()), float(np.max(err / np.maximum(bound, 1e-300))))


def _check_stats(stats, out, B, weighted, n_runs=1):
    certain, undecided, hit = out["hits"]
    got = stats[0].item() / n_runs
    assert certain <= got <= certain + undecided, (got, certain, undecided)
    assert stats[1].item() == n_runs * B
    if weighted:                            # (the kernel adds to the -7 the two sums start from)
        assert stats[3].item() + 7.0 == pytest.approx(n_runs * out["w"].sum(), rel=1e-5, abs=1e-4)
        if undecided == 0:
            assert stats[2].item() + 7.0 == pytest.approx(n_runs * (out["w"] * hit).sum(), rel=1e-5, abs=1e-4)
    else:
        assert stats[2].item() == -7.0 and stats[3].item() == -7.0, "the unweighted kernel writes 2 stats"


# ------------------------------------------------------------------------------------------------ fused head
def _head_operands(B, K, C, case, seed, onehot=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    h = torch.randn(B, K, device="cuda", generator=g).relu().bfloat16()
    w2 = (torch.randn(C, K, device="cuda", generator=g) * 0.2).bfloat16()
    b2 = (torch.randn(C, device="cuda", generator=g) * 0.1).bfloat16()
    mask = (torch.rand(B, K, device="cuda", generator=g) > 0.4).to(torch.uint8) if "mask" in case else None
    labels, y, ls, sw, cw = _inputs(B, C, case, g, onehot)
    return h, w2, b2, mask, labels, y, ls, sw, cw


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

    def tail(self):
        return (self.loss[1].data_ptr(), None, self.stats.data_ptr(), self.dw2[1].data_ptr(), self.db2[1].data_ptr(),
                self.dh[1].data_ptr(), self.db1[1].data_ptr(), self.scratch.data_ptr(), self.counter.data_ptr())

    def outputs(self):
        return [self.loss[1].clone(), self.dw2[1].clone(), self.db2[1].clone(), self.dh[1].clone(), self.db1[1].clone()]

    def bufs(self):
        return [self.loss, self.dw2, self.db2, self.dh, self.db1]


def _soft_head(lib, o, h, w2, b2, y, ls, mask, scale, sw, cw, B, K, C):
    return lib.tfy_dense_head_fused_soft(
        h.data_ptr(), w2.data_ptr(), b2.data_ptr(), y.data_ptr(), ctypes.c_float(ls),
        mask.data_ptr() if mask is not None else None, ctypes.c_float(scale), *o.tail(), B, K, C,
        sw.data_ptr() if sw is not None else None, cw.data_ptr() if cw is not None else None, _stream())


HEAD_SHAPES = [(B, K, C) for B in (1, 16, 17, 128, 1000) for K in (128, 256, 512) for C in (2, 10, 16)]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("B,K,C", HEAD_SHAPES)
def test_fused_soft_head_matches_the_float64_reference(lib, B, K, C, case):
    h, w2, b2, mask, _, y, ls, sw, cw = _head_operands(B, K, C, case, seed=B * 7 + K + C + len(case))
    scale = 2.0
    o = _HeadOut(lib, B, K, C)
    runs = []
    for _ in range(3):
        assert _soft_head(lib, o, h, w2, b2, y, ls, mask, scale, sw, cw, B, K, C) == 0
        torch.cuda.synchronize()
        runs.append(o.outputs())
        assert bool((o.scratch == 0).all()) and int(o.counter.item()) == 0
    for run in runs[1:]:                    # fixed-order sums: the same bits on every launch
        for a, b in zip(runs[0], run):
            assert torch.equal(a, b)
    _guards_intact(o.bufs())
    want = ref.fused_head(h, w2, b2, y, ls, mask, scale, sw, cw)
    _check("loss", o.loss[1], want["loss"], want["loss_bound"])
    for name in ("dw2", "db2", "dh", "db1"):
        _check(name, getattr(o, name)[1], want[name], want[name + "_bound"])
    _check_stats(o.stats, want, B, sw is not None, n_runs=3)


@pytest.mark.parametrize("case", ["plain", "mask_weights_ls_soft"])
def test_fused_soft_head_replays_in_a_cuda_graph(lib, case):
    B, K, C = 128, 128, 10
    h, w2, b2, mask, _, y, ls, sw, cw = _head_operands(B, K, C, case, seed=5)
    o = _HeadOut(lib, B, K, C)
    assert _soft_head(lib, o, h, w2, b2, y, ls, mask, 2.0, sw, cw, B, K, C) == 0
    torch.cuda.synchronize()
    direct = o.outputs()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert _soft_head(lib, o, h, w2, b2, y, ls, mask, 2.0, sw, cw, B, K, C) == 0
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(direct, o.outputs()):
        assert torch.equal(a, b)
    assert bool((o.scratch == 0).all()) and int(o.counter.item()) == 0


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("B,K,C", HEAD_SHAPES)
def test_fused_soft_head_is_the_sparse_head_bit_for_bit_on_one_hot_targets(lib, B, K, C, weighted):
    case = "mask_weights" if weighted else "mask"
    h, w2, b2, mask, labels, y, _, sw, cw = _head_operands(B, K, C, case, seed=B + K * 3 + C, onehot=True)
    soft, sparse = _HeadOut(lib, B, K, C), _HeadOut(lib, B, K, C)
    assert _soft_head(lib, soft, h, w2, b2, y, 0.0, mask, 2.0, sw, cw, B, K, C) == 0
    args = (h.data_ptr(), w2.data_ptr(), b2.data_ptr(), labels.data_ptr(), mask.data_ptr(), ctypes.c_float(2.0),
            *sparse.tail(), B, K, C)
    if weighted:
        rc = lib.tfy_dense_head_fused_weighted(*args, sw.data_ptr(), cw.data_ptr(), _stream())
    else:
        rc = lib.tfy_dense_head_fused(*args, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    for a, b in zip(soft.outputs(), sparse.outputs()):
        assert torch.equal(a, b)
    assert torch.equal(soft.stats, sparse.stats)


def test_soft_entry_points_refuse_bad_arguments(lib):
    B, K, C = 16, 128, 10
    h, w2, b2, mask, _, y, _, _, _ = _head_operands(B, K, C, "mask", seed=1)
    o = _HeadOut(lib, B, K, C)
    for ls in (-0.1, 1.5, float("nan")):
        assert _soft_head(lib, o, h, w2, b2, y, ls, mask, 1.0, None, None, B, K, C) == -2
    assert _soft_head(lib, o, h, w2, b2, y, 0.0, mask, 1.0, None, None, B, 64, C) == -2       # K outside the envelope
    assert _soft_head(lib, o, h, w2, b2, y, 0.0, mask, 1.0, None, None, B, K, 17) == -2       # C > 16
    lg = torch.zeros(B, C, dtype=torch.bfloat16, device="cuda")
    args = (lg.data_ptr(), None, y.data_ptr())
    rest = (None, None, o.loss[1].data_ptr(), o.dh[1].data_ptr(), None, None)
    assert lib.tfy_softmax_xent_soft(*args, ctypes.c_float(2.0), *rest, B, C, _stream()) == -2
    assert lib.tfy_softmax_xent_soft(*args, ctypes.c_float(0.0), *rest, 1 << 16, 1 << 16, _stream()) == -2   # B*C
    assert lib.tfy_softmax_xent_soft(lg.data_ptr(), None, None, ctypes.c_float(0.0), *rest, B, C, _stream()) == -2
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ fallback
def _fallback_operands(B, C, case, seed, onehot=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lg = (torch.randn(B, C, device="cuda", generator=g) * 2).bfloat16()
    bx = (torch.randn(C, device="cuda", generator=g) * 0.1).bfloat16()
    labels, y, ls, sw, cw = _inputs(B, C, case, g, onehot)
    return lg, bx, labels, y, ls, sw, cw


def _soft_xent(lib, lg, bx, y, ls, sw, cw, bufs, B, C):
    loss, dl, db, stats = bufs
    return lib.tfy_softmax_xent_soft(lg.data_ptr(), bx.data_ptr(), y.data_ptr(), ctypes.c_float(ls),
                                     sw.data_ptr() if sw is not None else None,
                                     cw.data_ptr() if cw is not None else None, loss[1].data_ptr(), dl[1].data_ptr(),
                                     db[1].data_ptr(), stats.data_ptr(), B, C, _stream())


def _xent_bufs(B, C):
    return (_guarded((), torch.float32), _guarded((B, C), torch.bfloat16), _guarded((C,), torch.bfloat16),
            torch.tensor([0.0, 0.0, -7.0, -7.0], device="cuda"))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("B,C", [(B, C) for B in (1, 16, 17, 128, 1000) for C in (17, 100)])
def test_soft_xent_fallback_matches_the_float64_reference(lib, B, C, case):
    lg, bx, _, y, ls, sw, cw = _fallback_operands(B, C, case, seed=B * 5 + C + len(case))
    bufs = _xent_bufs(B, C)
    runs = []
    for _ in range(3):
        assert _soft_xent(lib, lg, bx, y, ls, sw, cw, bufs, B, C) == 0
        torch.cuda.synchronize()
        runs.append([b[1].clone() for b in bufs[:3]])
    for run in runs[1:]:
        for a, b in zip(runs[0], run):
            assert torch.equal(a, b)
    _guards_intact(bufs[:3])
    want = ref.softmax_xent(lg, bx, y, ls, sw, cw)
    _check("loss", bufs[0][1], want["loss"], want["loss_bound"])
    _check("dlogits", bufs[1][1], want["dlogits"], want["dlogits_bound"])
    _check("dbias", bufs[2][1], want["dbias"], want["dbias_bound"])
    _check_stats(bufs[3], want, B, sw is not None, n_runs=3)
    # a CUDA-graph replay gives the launch's bits
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert _soft_xent(lib, lg, bx, y, ls, sw, cw, bufs, B, C) == 0
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(runs[0], [b[1] for b in bufs[:3]]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("B,C", [(1, 17), (17, 100), (1000, 40), (3000, 10)])
def test_soft_xent_fallback_is_the_sparse_kernel_bit_for_bit_on_one_hot_targets(lib, B, C, weighted):
    lg, bx, labels, y, _, sw, cw = _fallback_operands(B, C, "weights" if weighted else "plain", seed=B + C,
                                                      onehot=True)
    soft, sparse = _xent_bufs(B, C), _xent_bufs(B, C)
    assert _soft_xent(lib, lg, bx, y, 0.0, sw, cw, soft, B, C) == 0
    loss, dl, db, stats = sparse
    if weighted:
        rc = lib.tfy_softmax_xent_weighted(lg.data_ptr(), bx.data_ptr(), labels.data_ptr(), sw.data_ptr(),
                                           cw.data_ptr(), loss[1].data_ptr(), dl[1].data_ptr(), db[1].data_ptr(),
                                           stats.data_ptr(), B, C, _stream())
    else:
        rc = lib.tfy_softmax_xent(lg.data_ptr(), bx.data_ptr(), labels.data_ptr(), loss[1].data_ptr(),
                                  dl[1].data_ptr(), db[1].data_ptr(), stats.data_ptr(), B, C, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    for a, b in zip(soft, sparse):
        assert torch.equal(a[1] if isinstance(a, tuple) else a, b[1] if isinstance(b, tuple) else b)


# ------------------------------------------------------------------------------------------------ the fast path
def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _no_dropout():
    """The MNIST CNN with its dropout rates at 0: the fast path and the autograd engine draw different masks."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    return keras.Sequential([layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)),
                             layers.Conv2D(64, (3, 3), activation="relu"), layers.MaxPooling2D(pool_size=(2, 2)),
                             layers.Dropout(0.0), layers.Flatten(), layers.Dense(128, activation="relu"),
                             layers.Dropout(0.0), layers.Dense(10)])


def _fit(loss, y, steps=50, fast=True, build=None, **fit_kw):
    """MNIST CNN (or ``build()``) from seed 7, ``steps`` batches of 128: (model, per-step losses, epoch logs,
    weights)."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn, synthetic_mnist
    torch.manual_seed(7)
    m = (build or keras_mnist_cnn)()
    m.compile(loss=loss, optimizer=keras.optimizers.Adadelta(1.0), metrics=["accuracy"], use_fast_path=fast,
              weighted_metrics=["accuracy"] if fit_kw else None)
    x, _ = synthetic_mnist(128 * steps, seed=3)
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    hist = m.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0, callbacks=[Rec()], **fit_kw)
    torch.cuda.synchronize()
    return m, losses, hist.history, [torch.as_tensor(w) for w in m.get_weights()]


def _one_hot(y):
    """Keras' to_categorical(y, 10)."""
    return torch.nn.functional.one_hot(y.long(), 10).float()


def _labels(steps=50):
    from tf_yarn_b200.models.mnist_cnn import synthetic_mnist
    return synthetic_mnist(128 * steps, seed=3)[1]


def _same_bits(a, b):
    assert a[1] == b[1], "per-step losses differ"
    assert a[2] == b[2], (a[2], b[2])
    assert torch.equal(_bits(a[0]._engine.fused.flat_params), _bits(b[0]._engine.fused.flat_params))
    assert torch.equal(a[0]._engine.fused.master, b[0]._engine.fused.master)
    for p, q in zip(a[3], b[3]):
        assert torch.equal(_bits(p), _bits(q))


@pytest.mark.parametrize("weights", ["none", "sample", "class", "both"])
def test_categorical_fastpath_trains_the_sparse_bits(weights):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    y = _labels()
    kw = {}
    if weights in ("sample", "both"):
        kw["sample_weight"] = torch.rand(len(y), generator=torch.Generator().manual_seed(4)) * 2
    if weights in ("class", "both"):
        kw["class_weight"] = {c: 0.25 + 0.3 * c for c in range(10)}
    sparse = _fit(keras.losses.SparseCategoricalCrossentropy(from_logits=True), y, **kw)
    onehot = _one_hot(y)
    cat = _fit(keras.losses.CategoricalCrossentropy(from_logits=True), onehot, **kw)
    for m in (sparse[0], cat[0]):
        assert isinstance(m._engine, FastSequentialEngine) and m._engine._launches_per_step == 10
    assert cat[0]._engine._staging[0][1].dtype == torch.float32
    _same_bits(sparse, cat)


def test_label_smoothing_fastpath_tracks_the_autograd_engine():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    y = _one_hot(_labels(20))
    loss = keras.losses.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1)
    m_fast, l_fast, _, _ = _fit(loss, y, steps=20, build=_no_dropout)
    m_ref, l_ref, _, _ = _fit(loss, y, steps=20, fast=False, build=_no_dropout)
    assert isinstance(m_fast._engine, FastSequentialEngine) and not isinstance(m_ref._engine, FastSequentialEngine)
    assert m_fast._engine._ls == pytest.approx(0.1) and m_fast._engine._launches_per_step == 10
    assert len(l_fast) == len(l_ref) == 20
    for a, b in zip(l_fast, l_ref):
        assert math.isfinite(a) and abs(a - b) < 0.03 * max(1.0, abs(b)), (l_fast, l_ref)


def test_categorical_fastpath_under_gradient_accumulation_keeps_its_launch_count():
    from tf_yarn_b200 import keras
    torch.manual_seed(7)
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn, synthetic_mnist
    m = keras_mnist_cnn()
    m.compile(loss=keras.losses.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1),
              optimizer=keras.optimizers.Adadelta(1.0, gradient_accumulation_steps=2), metrics=["accuracy"])
    x, y = synthetic_mnist(128 * 4, seed=3)
    m.fit(x, _one_hot(y), batch_size=128, epochs=1, shuffle=False, verbose=0)
    eng = m._engine
    assert eng._launches_per_step == 11 and eng._launches_per_accum_step == 10


@pytest.mark.parametrize("dtype", [torch.int32, torch.uint8])
def test_narrow_integer_labels_train_like_int64_labels(dtype):
    from tf_yarn_b200 import keras
    loss = keras.losses.SparseCategoricalCrossentropy(from_logits=True)
    y = _labels(10)
    wide = _fit(loss, y, steps=10)
    narrow = _fit(loss, y.to(dtype), steps=10)
    _same_bits(wide, narrow)
    # a dataset of narrow labels: the int64 staging slots convert them on the copy
    from tf_yarn_b200.models.mnist_cnn import synthetic_mnist
    x = synthetic_mnist(128 * 10, seed=3)[0]

    def batches(yy):
        return [(x[i:i + 128], yy[i:i + 128]) for i in range(0, len(yy), 128)]
    runs = []
    for yy in (y, y.to(dtype)):
        torch.manual_seed(7)
        from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
        m = keras_mnist_cnn()
        m.compile(loss=loss, optimizer=keras.optimizers.Adadelta(1.0), metrics=["accuracy"])
        h = m.fit(batches(yy), epochs=1, verbose=0, steps_per_epoch=10)
        torch.cuda.synchronize()
        runs.append((h.history, m._engine.fused.master.clone()))
    assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1])


def test_categorical_targets_of_the_wrong_width_are_refused():
    from tf_yarn_b200 import keras
    with pytest.raises(ValueError, match=r"\(128, 7\).*10"):
        _fit(keras.losses.CategoricalCrossentropy(from_logits=True), torch.zeros(128 * 2, 7), steps=2)


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_categorical_fastpath_trains_the_sparse_bits_on_two_gpus():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29641", "tests/gpu/categorical_head_check.py"]
    res = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert res.returncode == 0 and "CATEGORICAL HEAD CHECK OK" in res.stdout, res.stdout[-4000:]
