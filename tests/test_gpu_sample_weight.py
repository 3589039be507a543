"""GPU tests of Keras sample weighting: the weighted fused classifier head and softmax cross-entropy kernels against
fp32 references, and the fast-path engine under sample_weight / class_weight (exactness, reproducibility,
recapture on a change of weighting mode)."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = ["sample", "class", "both"]


def _weights(B, C, mode, g, dev="cuda"):
    sw = torch.rand(B, device=dev, generator=g) * 2 if mode in ("sample", "both") else None
    cw = torch.rand(C, device=dev, generator=g) * 3 if mode in ("class", "both") else None
    if sw is not None:
        sw[::7] = 0.0                                     # zeros included
    if cw is not None:
        cw[0] = 0.0
    return sw, cw


def _reference(logits, y, sw, cw, B, C):
    """Loss sum(w*l)/B and its gradient (softmax - onehot) * w / B; a label outside [0, C) has no one-hot entry and
    contributes no loss (as in the kernels), and weighs 1 in the class table."""
    valid = (y >= 0) & (y < C)
    yc = y.clamp(0, C - 1)
    w = torch.ones(B, device=y.device)
    if cw is not None:
        w = torch.where(valid, cw[yc], torch.ones_like(w))
    if sw is not None:
        w = sw * w
    onehot = torch.nn.functional.one_hot(yc, C).float() * valid[:, None].float()
    lse = torch.logsumexp(logits, dim=1)
    ce = lse - (onehot * logits).sum(1)
    grad_loss = (w * ce).sum() / B                         # gradient source (onehot 0 on invalid rows)
    loss = (w * ce * valid.float()).sum() / B
    hit = (logits.argmax(1) == y).float()
    return grad_loss, loss.item(), [hit.sum().item(), float(B), (hit * w).sum().item(), w.sum().item()]


def _close(a, b, tol=0.02):
    scale = b.abs().max().item() + 1e-6
    assert (a.float() - b).abs().max().item() <= tol * scale, ((a.float() - b).abs().max().item(), scale)


@pytest.mark.parametrize("mode", MODES + ["class_bad_label"])
@pytest.mark.parametrize("B,K,C", [(128, 128, 10), (100, 256, 16), (37, 512, 3)])
def test_weighted_fused_head_matches_autograd(B, K, C, mode):
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernel)
    from tf_yarn_b200.ops import native
    lib = native.load()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(B + K + C + len(mode))
    h = torch.randn(B, K, device=dev, generator=g).relu().bfloat16()
    w2 = (torch.randn(C, K, device=dev, generator=g) * 0.2).bfloat16()
    b2 = (torch.randn(C, device=dev, generator=g) * 0.1).bfloat16()
    y = torch.randint(0, C, (B,), device=dev, generator=g)
    sw, cw = _weights(B, C, "class" if mode == "class_bad_label" else mode, g)
    if mode == "class_bad_label":
        y[3], y[11] = C + 2, -1
    mask = (torch.rand(B, K, device=dev, generator=g) > 0.4).to(torch.uint8)
    scale = 2.0
    loss = torch.zeros((), device=dev)
    stats = torch.zeros(4, device=dev)
    dw2 = torch.zeros(C, K, dtype=torch.bfloat16, device=dev)
    db2 = torch.zeros(C, dtype=torch.bfloat16, device=dev)
    dh = torch.zeros(B, K, dtype=torch.bfloat16, device=dev)
    db1 = torch.zeros(K, dtype=torch.bfloat16, device=dev)
    scratch = torch.zeros(int(lib.tfy_dense_head_scratch_elems(K, C, B)), device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    hf = h.float().requires_grad_(True)
    wf = w2.float().requires_grad_(True)
    bf = b2.float().requires_grad_(True)
    logits = hf @ wf.t() + bf
    grad_loss, ref_loss, ref_stats = _reference(logits, y, sw, cw, B, C)
    grad_loss.backward()
    ref_dh = hf.grad * mask.float() * scale
    for _ in range(2):      # twice: the scratch buffer and the counter must come back clean
        rc = lib.tfy_dense_head_fused_weighted(
            h.data_ptr(), w2.data_ptr(), b2.data_ptr(), y.data_ptr(), mask.data_ptr(), ctypes.c_float(scale),
            loss.data_ptr(), None, stats.data_ptr(), dw2.data_ptr(), db2.data_ptr(), dh.data_ptr(), db1.data_ptr(),
            scratch.data_ptr(), counter.data_ptr(), B, K, C, sw.data_ptr() if sw is not None else None,
            cw.data_ptr() if cw is not None else None, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert abs(loss.item() - ref_loss) < 1e-3 * max(1.0, abs(ref_loss))
        _close(dw2, wf.grad)
        _close(db2, bf.grad)
        _close(dh, ref_dh)
        _close(db1, ref_dh.sum(0))
        assert bool((scratch == 0).all()) and int(counter.item()) == 0
    assert stats[0].item() == 2 * ref_stats[0] and stats[1].item() == 2 * B
    assert stats[2].item() == pytest.approx(2 * ref_stats[2], rel=1e-5, abs=1e-4)
    assert stats[3].item() == pytest.approx(2 * ref_stats[3], rel=1e-5, abs=1e-4)


@pytest.mark.parametrize("mode", MODES + ["class_bad_label"])
@pytest.mark.parametrize("B,C", [(128, 10), (100, 16), (37, 3), (3000, 40)])
def test_weighted_softmax_xent_matches_autograd(B, C, mode):
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernel)
    from tf_yarn_b200.ops import native
    lib = native.load()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(B * 3 + C + len(mode))
    lg = torch.randn(B, C, device=dev, generator=g).bfloat16()
    bx = (torch.randn(C, device=dev, generator=g) * 0.1).bfloat16()
    y = torch.randint(0, C, (B,), device=dev, generator=g)
    sw, cw = _weights(B, C, "class" if mode == "class_bad_label" else mode, g)
    if mode == "class_bad_label":
        y[3], y[11] = C + 2, -1
    loss = torch.zeros((), device=dev)
    dl = torch.empty(B, C, dtype=torch.bfloat16, device=dev)
    dbx = torch.empty(C, dtype=torch.bfloat16, device=dev)
    stats = torch.zeros(4, device=dev)
    lr_ = (lg.float() + bx.float()).requires_grad_(True)
    grad_loss, ref_loss, ref_stats = _reference(lr_, y, sw, cw, B, C)
    grad_loss.backward()
    results = []
    for _ in range(2):
        rc = lib.tfy_softmax_xent_weighted(lg.data_ptr(), bx.data_ptr(), y.data_ptr(),
                                           sw.data_ptr() if sw is not None else None,
                                           cw.data_ptr() if cw is not None else None, loss.data_ptr(), dl.data_ptr(),
                                           dbx.data_ptr(), stats.data_ptr(), B, C,
                                           torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert abs(loss.item() - ref_loss) < 1e-3 * max(1.0, abs(ref_loss))
        torch.testing.assert_close(dl.float(), lr_.grad, rtol=2e-2, atol=1e-4)
        _close(dbx, lr_.grad.sum(0))
        results.append((loss.clone(), dl.clone(), dbx.clone()))
    for a, b in zip(*results):               # fixed-order sums: the same bits on every launch
        assert torch.equal(a, b)
    assert stats[0].item() == 2 * ref_stats[0] and stats[1].item() == 2 * B
    assert stats[2].item() == pytest.approx(2 * ref_stats[2], rel=1e-5, abs=1e-4)
    assert stats[3].item() == pytest.approx(2 * ref_stats[3], rel=1e-5, abs=1e-4)


def _mnist_like(drop1=0.0, drop2=0.0, padding="valid"):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="mnist_cnn_weighted_test")
    m.add(layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1), padding=padding))
    m.add(layers.Conv2D(64, (3, 3), activation="relu"))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(drop1))
    m.add(layers.Flatten())
    m.add(layers.Dense(128, activation="relu"))
    m.add(layers.Dropout(drop2))
    m.add(layers.Dense(10))
    return m


def _data(n, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 28, 28, 1, generator=g), torch.randint(0, 10, (n,), generator=g)


CW = {c: 0.25 + 0.3 * c for c in range(10)}


def _train(fast=True, drop=(0.0, 0.0), fits=({},), steps=4, metrics=("accuracy",), weighted_metrics=None,
           optimizer=None, padding="valid", device=None):
    """Train from seed 7 with one ``fit`` per entry of ``fits`` (its keyword arguments); returns the model, the
    per-step losses and the full-precision weights."""
    from tf_yarn_b200 import keras
    torch.manual_seed(7)
    m = _mnist_like(*drop, padding=padding)
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True),
              optimizer=optimizer or keras.optimizers.Adadelta(1.0), metrics=list(metrics),
              weighted_metrics=weighted_metrics, use_fast_path=fast)
    if device is not None:
        m._device = torch.device(device)
    x, y = _data(128 * steps)
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    hists = []
    for kw in fits:
        kw = dict(kw)
        if "sample_weight" in kw and callable(kw["sample_weight"]):
            kw["sample_weight"] = kw["sample_weight"](y)
        hists.append(m.fit(x, y, batch_size=128, epochs=1, shuffle=False, verbose=0, callbacks=[Rec()], **kw))
    torch.cuda.synchronize()
    return m, losses, [torch.as_tensor(w) for w in m.get_weights()], hists


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _assert_bit_identical(a, b):
    m1, l1, w1, _ = a
    m2, l2, w2, _ = b
    assert l1 == l2, (l1, l2)
    assert torch.equal(_bits(m1._engine.fused.flat_params), _bits(m2._engine.fused.flat_params))
    for p, q in zip(w1, w2):
        assert torch.equal(_bits(p), _bits(q))


def test_fastpath_class_weight_matches_autograd_engine():
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m_fast, l_fast, wf, _ = _train(True, fits=({"class_weight": CW},))
    m_ref, l_ref, wr, _ = _train(False, fits=({"class_weight": CW},))
    assert isinstance(m_fast._engine, FastSequentialEngine)
    assert not isinstance(m_ref._engine, FastSequentialEngine)
    assert len(l_fast) == len(l_ref) == 4
    for a, b in zip(l_fast, l_ref):
        assert math.isfinite(a) and abs(a - b) < 0.03 * max(1.0, abs(b)), (l_fast, l_ref)
    for a, b in zip(wf, wr):
        denom = b.abs().max().clamp_min(2e-2)
        assert ((a - b).abs().max() / denom) < 0.15, ((a - b).abs().max(), denom)


def test_fastpath_weights_are_exact():
    """All-ones sample weights train bit for bit like no weights; class_weight=cw like sample_weight=cw[y]."""
    table = torch.tensor([CW[c] for c in range(10)])
    plain = _train(True, drop=(0.25, 0.5))
    ones = _train(True, drop=(0.25, 0.5), fits=({"sample_weight": lambda y: torch.ones(len(y))},))
    _assert_bit_identical(plain, ones)
    by_class = _train(True, drop=(0.25, 0.5), fits=({"class_weight": CW},))
    by_sample = _train(True, drop=(0.25, 0.5), fits=({"sample_weight": lambda y: table[y]},))
    _assert_bit_identical(by_class, by_sample)
    assert plain[0]._engine._launches_per_step == by_class[0]._engine._launches_per_step \
        == by_sample[0]._engine._launches_per_step == 10


def test_weighted_fastpath_training_is_bitwise_reproducible():
    sw = lambda y: torch.rand(len(y), generator=torch.Generator().manual_seed(3))  # noqa: E731
    kw = ({"sample_weight": sw, "class_weight": CW},)
    a = _train(True, drop=(0.25, 0.5), fits=kw, weighted_metrics=["accuracy"])
    b = _train(True, drop=(0.25, 0.5), fits=kw, weighted_metrics=["accuracy"])
    _assert_bit_identical(a, b)
    h = a[3][0].history
    assert set(h) == {"loss", "accuracy", "weighted_accuracy"} and h["accuracy"] != h["weighted_accuracy"]


def test_weighted_metrics_of_the_fast_path_match_the_autograd_engine():
    from tf_yarn_b200 import keras
    sw = lambda y: torch.rand(len(y), generator=torch.Generator().manual_seed(3))  # noqa: E731
    kw = ({"sample_weight": sw, "class_weight": CW},)
    opt = keras.optimizers.SGD(0.0)              # the parameters stay put: both engines score the same model
    fast = _train(True, fits=kw, weighted_metrics=["accuracy"], optimizer=opt)
    ref = _train(False, fits=kw, weighted_metrics=["accuracy"], optimizer=keras.optimizers.SGD(0.0))
    hf, hr = fast[3][0].history, ref[3][0].history
    assert abs(hf["weighted_accuracy"][0] - hr["weighted_accuracy"][0]) < 0.02
    assert abs(hf["accuracy"][0] - hr["accuracy"][0]) < 0.02


def test_changing_the_weighting_mode_recaptures_and_continues():
    """Unweighted, then class_weight, then sample_weight on one model: every change recaptures the step graphs, the
    fast path stays in use and training continues from the current state (all-ones weights are exact, so the run
    equals three unweighted epochs bit for bit, dropout and step counter included)."""
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    ones = {c: 1.0 for c in range(10)}
    captures = []
    orig = FastSequentialEngine._capture

    def counting(self, *a, **k):
        captures.append(1)
        return orig(self, *a, **k)
    FastSequentialEngine._capture = counting
    try:
        mixed = _train(True, drop=(0.25, 0.5),
                       fits=({}, {"class_weight": ones}, {"sample_weight": lambda y: torch.ones(len(y))}))
    finally:
        FastSequentialEngine._capture = orig
    plain = _train(True, drop=(0.25, 0.5), fits=({}, {}, {}))
    eng = mixed[0]._engine
    assert isinstance(eng, FastSequentialEngine) and len(captures) == 3
    assert eng._wmode == (False, True)
    assert eng.fused.step_count == plain[0]._engine.fused.step_count == 12
    _assert_bit_identical(mixed, plain)
    # a new table of the same size is copied in place: no recapture
    before = list(eng.graphs)
    eng.set_class_weight(torch.full((10,), 2.0))
    assert eng.graphs == before


def test_model_outside_the_fast_path_trains_weighted_like_the_eager_engine():
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.engine import EagerTrainEngine, GraphTrainEngine
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    sw = lambda y: torch.rand(len(y), generator=torch.Generator().manual_seed(3)) * 2  # noqa: E731
    kw = ({"sample_weight": sw, "class_weight": CW},)
    gpu = _train(True, fits=kw, padding="same", optimizer=keras.optimizers.SGD(0.05), weighted_metrics=["accuracy"])
    cpu = _train(True, fits=kw, padding="same", optimizer=keras.optimizers.SGD(0.05), weighted_metrics=["accuracy"],
                 device="cpu")
    assert isinstance(gpu[0]._engine, GraphTrainEngine) and not isinstance(gpu[0]._engine, FastSequentialEngine)
    assert isinstance(cpu[0]._engine, EagerTrainEngine)
    for a, b in zip(gpu[1], cpu[1]):
        assert math.isfinite(a) and abs(a - b) < 0.03 * max(1.0, abs(b)), (gpu[1], cpu[1])
    for a, b in zip(gpu[2], cpu[2]):
        assert ((a - b).abs().max() / b.abs().max().clamp_min(2e-2)) < 0.05
    ha, hb = gpu[3][0].history, cpu[3][0].history
    assert abs(ha["weighted_accuracy"][0] - hb["weighted_accuracy"][0]) < 0.05
