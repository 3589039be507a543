"""Keras label_smoothing on the categorical and binary cross-entropies, and the fast path's categorical head, on the CPU.

* Every loss form (class, functional, per-sample) with ls in {0, 0.1, 1}, from logits or probabilities, one-hot and
  soft targets, against a float64 NumPy statement of Keras' formulas; the weighted per-sample forms; the argument
  checks; serialize / deserialize and Model.save / load_model.
* The eager engine trains with it, and at ls = 0 bit for bit like the unsmoothed loss.
* fastpath.build_plan's grammar for categorical losses, the engine's label dtype and target check, fit's one-time
  label cast, and the categorical step's launches (the recorder of tests/test_fastpath_step_trace.py): the sparse
  step's, except the head launch.
"""
import json
import os
import sys
import types
from contextlib import ExitStack
from unittest import mock

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.keras import fastpath, weighting  # noqa: E402
from tf_yarn_b200.keras import layers as L  # noqa: E402
from tf_yarn_b200.keras import losses as kl  # noqa: E402
from tf_yarn_b200.keras.engine import GraphTrainEngine  # noqa: E402
from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402
import test_fastpath_step_trace as trace  # noqa: E402

EPS = 1e-7
LS = [0.0, 0.1, 1.0]


# ------------------------------------------------------------------------------------------------ NumPy statement
def _np_softmax(z):
    z = z - z.max(-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(-1, keepdims=True)


def np_categorical(y, out, from_logits, ls):
    """Keras: t = y (1 - ls) + ls / C; -sum_c t_c log p_c per sample (p clipped to [eps, 1 - eps])."""
    y = y.astype(np.float64)
    t = y * (1 - ls) + ls / y.shape[-1]
    p = _np_softmax(out) if from_logits else np.clip(out, EPS, 1 - EPS)
    return -(t * np.log(p)).sum(-1)


def np_binary(y, out, from_logits, ls):
    """Keras: t = y (1 - ls) + ls / 2; per element max(x, 0) - x t + log(1 + e^-|x|) from logits, else
    -(t log p + (1 - t) log(1 - p)) with p clipped to [eps, 1 - eps]."""
    t = y.astype(np.float64).reshape(-1) * (1 - ls) + 0.5 * ls
    x = out.astype(np.float64).reshape(-1)
    if from_logits:
        return np.maximum(x, 0) - x * t + np.log1p(np.exp(-np.abs(x)))
    p = np.clip(x, EPS, 1 - EPS)
    return -(t * np.log(p) + (1 - t) * np.log(1 - p))


def _categorical_data(soft, from_logits, B=9, C=5, seed=0):
    rng = np.random.default_rng(seed)
    y = rng.random((B, C)) * 1.5 if soft else np.eye(C)[rng.integers(0, C, B)]
    z = rng.normal(size=(B, C)) * 2
    out = z if from_logits else _np_softmax(z)
    return y.astype(np.float32), out.astype(np.float32)


def _binary_data(soft, from_logits, B=11, seed=1):
    rng = np.random.default_rng(seed)
    y = rng.random((B, 1)) if soft else rng.integers(0, 2, (B, 1)).astype(np.float64)
    z = rng.normal(size=(B, 1)) * 2
    out = z if from_logits else 1 / (1 + np.exp(-z))
    return y.astype(np.float32), out.astype(np.float32)


def _t(a):
    return torch.from_numpy(np.asarray(a))


# ------------------------------------------------------------------------------------------------ losses
@pytest.mark.parametrize("soft", [False, True])
@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("ls", LS)
def test_categorical_crossentropy_matches_keras(ls, from_logits, soft):
    y, out = _categorical_data(soft, from_logits)
    want = np_categorical(y, out, from_logits, ls)
    forms = {"class": kl.CategoricalCrossentropy(from_logits=from_logits, label_smoothing=ls)(_t(y), _t(out)),
             "functional": kl.categorical_crossentropy(_t(y), _t(out), from_logits=from_logits, label_smoothing=ls),
             "per_sample mean": kl.per_sample(kl.CategoricalCrossentropy(from_logits, ls))(_t(y), _t(out)).mean()}
    for name, got in forms.items():
        assert float(got) == pytest.approx(want.mean(), rel=2e-6, abs=2e-6), name
    per = kl.categorical_crossentropy_per_sample(_t(y), _t(out), from_logits=from_logits, label_smoothing=ls)
    np.testing.assert_allclose(per.numpy(), want, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("soft", [False, True])
@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("ls", LS)
def test_binary_crossentropy_matches_keras(ls, from_logits, soft):
    y, out = _binary_data(soft, from_logits)
    want = np_binary(y, out, from_logits, ls)
    forms = {"class": kl.BinaryCrossentropy(from_logits=from_logits, label_smoothing=ls)(_t(y), _t(out)),
             "functional": kl.binary_crossentropy(_t(y), _t(out), from_logits=from_logits, label_smoothing=ls),
             "per_sample mean": kl.per_sample(kl.BinaryCrossentropy(from_logits, ls))(_t(y), _t(out)).mean()}
    for name, got in forms.items():
        assert float(got) == pytest.approx(want.mean(), rel=2e-6, abs=2e-6), name
    per = kl.binary_crossentropy_per_sample(_t(y), _t(out), from_logits=from_logits, label_smoothing=ls)
    np.testing.assert_allclose(per.numpy(), want, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("ls", LS)
def test_weighted_per_sample_forms_compose_with_smoothing(ls):
    """sum(w * l) / B with w = sample_weight * class_weight[argmax y] (Keras' SUM_OVER_BATCH_SIZE)."""
    y, out = _categorical_data(True, True, B=8)
    sw = np.linspace(0.0, 2.0, 8).astype(np.float32)
    cw = np.array([0.5, 1.0, 2.0, 0.0, 3.0], dtype=np.float32)
    w = sw * cw[y.argmax(-1)]
    loss = kl.CategoricalCrossentropy(from_logits=True, label_smoothing=ls)
    got = weighting.weighted_loss(kl.per_sample(loss), _t(y), _t(out),
                                  weighting.sample_weights(_t(y), _t(sw), _t(cw)))
    assert float(got) == pytest.approx((w * np_categorical(y, out, True, ls)).sum() / 8, rel=2e-6)
    yb, ob = _binary_data(True, True, B=8)
    got = weighting.weighted_loss(kl.per_sample(kl.BinaryCrossentropy(True, ls)), _t(yb), _t(ob), _t(sw))
    assert float(got) == pytest.approx((sw * np_binary(yb, ob, True, ls)).sum() / 8, rel=2e-6)


@pytest.mark.parametrize("bad", [-0.1, 1.5, float("nan")])
def test_label_smoothing_outside_zero_one_is_refused(bad):
    y, out = _categorical_data(False, True)
    for make in (lambda: kl.CategoricalCrossentropy(label_smoothing=bad),
                 lambda: kl.BinaryCrossentropy(label_smoothing=bad),
                 lambda: kl.categorical_crossentropy(_t(y), _t(out), label_smoothing=bad),
                 lambda: kl.binary_crossentropy(_t(y[:, :1]), _t(out[:, :1]), label_smoothing=bad)):
        with pytest.raises(ValueError, match="label_smoothing"):
            make()


def test_axis_other_than_the_last_is_refused():
    with pytest.raises(ValueError, match="axis"):
        kl.CategoricalCrossentropy(axis=1)
    assert kl.CategoricalCrossentropy(axis=-1).label_smoothing == 0.0


def test_sparse_categorical_crossentropy_has_no_label_smoothing():
    with pytest.raises(TypeError):
        kl.SparseCategoricalCrossentropy(label_smoothing=0.1)


def test_serialize_carries_label_smoothing_only_when_nonzero():
    for cls in (kl.CategoricalCrossentropy, kl.BinaryCrossentropy):
        cfg = kl.serialize(cls(from_logits=True, label_smoothing=0.2))
        assert cfg == {"name": cls(False).__name__, "from_logits": True, "label_smoothing": 0.2}
        back = kl.deserialize(json.loads(json.dumps(cfg)))
        assert isinstance(back, cls) and back.from_logits and back.label_smoothing == 0.2
        assert kl.serialize(cls(from_logits=True)) == {"name": cls(False).__name__, "from_logits": True}
        old = kl.deserialize({"name": cls(False).__name__, "from_logits": False})       # a config written before
        assert isinstance(old, cls) and old.label_smoothing == 0.0


def _tiny(loss, metrics=("accuracy",)):
    m = keras.Sequential([L.Dense(8, activation="relu", input_shape=(6,)), L.Dense(4)])
    m.compile(loss=loss, optimizer=keras.optimizers.SGD(0.1), metrics=list(metrics))
    return m


def test_model_save_keeps_label_smoothing(tmp_path):
    m = _tiny(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.2))
    m.build()
    path = str(tmp_path / "m.tfy")
    m.save(path)
    back = keras.models.load_model(path)
    assert isinstance(back.loss, kl.CategoricalCrossentropy)
    assert back.loss.label_smoothing == 0.2 and back.loss.from_logits


def _data(n=64, C=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 6, generator=g)
    y = torch.nn.functional.one_hot(torch.randint(0, C, (n,), generator=g), C).float()
    return x, y


def _train(loss, **fit_kw):
    torch.manual_seed(3)
    m = _tiny(loss, metrics=())         # (a plain callable loss would resolve "accuracy" to the sparse one)
    m.to("cpu")
    x, y = _data()
    h = m.fit(x, y, batch_size=16, epochs=2, shuffle=False, verbose=0, **fit_kw)
    return h.history, [torch.as_tensor(w).clone() for w in m.get_weights()]


def _unsmoothed(y, out):        # the categorical cross-entropy from logits as it was before label smoothing
    return -(y.float() * torch.nn.functional.log_softmax(out.float(), dim=-1)).sum(dim=-1).mean()


def _unsmoothed_per_sample(y, out):
    return -(y.float() * torch.nn.functional.log_softmax(out.float(), dim=-1)).sum(dim=-1)


@pytest.mark.parametrize("weighted", [False, True])
def test_eager_engine_at_ls_zero_is_the_unsmoothed_loss_bit_for_bit(weighted):
    kw = {"sample_weight": np.linspace(0.5, 1.5, 64)} if weighted else {}
    h0, w0 = _train(_unsmoothed_per_sample if weighted else _unsmoothed, **kw)
    h1, w1 = _train(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.0), **kw)
    assert h0["loss"] == h1["loss"]
    for a, b in zip(w0, w1):
        assert torch.equal(a, b)


def test_eager_engine_trains_with_label_smoothing():
    def smoothed(y, out):
        t = y.float() * 0.9 + 0.1 / out.shape[-1]
        return -(t * torch.nn.functional.log_softmax(out.float(), dim=-1)).sum(dim=-1).mean()
    h0, w0 = _train(smoothed)
    h1, w1 = _train(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
    assert h1["loss"][-1] < h1["loss"][0]
    np.testing.assert_allclose(h0["loss"], h1["loss"], rtol=1e-6)
    for a, b in zip(w0, w1):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    assert _train(kl.CategoricalCrossentropy(True, 0.1))[0]["loss"] != _train(kl.CategoricalCrossentropy(True))[0]["loss"]


# ------------------------------------------------------------------------------------------------ fast-path grammar
def _plan(loss, metrics=("accuracy",), weighted=None, head="linear"):
    m = keras.Sequential([L.Dense(128, activation="relu", input_shape=(64,)), L.Dense(10, activation=head)])
    m.compile(loss=loss, optimizer="sgd", metrics=list(metrics), weighted_metrics=weighted)
    m.build()
    return fastpath.build_plan(m)


LOGITS = kl.CategoricalCrossentropy(from_logits=True)


@pytest.mark.parametrize("metric", ["accuracy", "acc", "categorical_accuracy"])
def test_build_plan_accepts_categorical_losses(metric):
    assert _plan(LOGITS, [metric]) is not None
    assert _plan(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.3), [metric]) is not None
    assert _plan("categorical_crossentropy", [metric], head="softmax") is not None
    assert _plan(kl.CategoricalCrossentropy(label_smoothing=0.1), [metric], head="softmax") is not None
    assert _plan(LOGITS, [metric], weighted=[metric]) is not None


def test_build_plan_refuses_what_the_categorical_head_does_not_compute():
    assert _plan(LOGITS, ["sparse_categorical_accuracy"]) is None
    assert _plan(LOGITS, ["accuracy"], weighted=["sparse_categorical_accuracy"]) is None
    assert _plan(LOGITS, ["mae"]) is None
    assert _plan(LOGITS, head="tanh") is None
    assert _plan(LOGITS, head="softmax") is None                     # logits loss after a softmax layer
    assert _plan("categorical_crossentropy") is None                 # probability loss after a linear layer
    assert _plan(kl.categorical_crossentropy, head="softmax") is None   # a plain callable: outside the grammar
    assert _plan(kl.SparseCategoricalCrossentropy(True), ["categorical_accuracy"]) is None


def test_label_dtype_is_what_the_head_reads():
    assert fastpath.label_dtype(LOGITS) == torch.float32
    assert fastpath.label_dtype("categorical_crossentropy") == torch.float32
    assert fastpath.label_dtype(kl.SparseCategoricalCrossentropy()) == torch.int64
    assert fastpath.label_dtype("sparse_categorical_crossentropy") == torch.int64
    assert fastpath.label_dtype("mse") is None and fastpath.label_dtype(kl.BinaryCrossentropy()) is None


def test_fit_casts_the_labels_once():
    from tf_yarn_b200.keras.models import _ArrayBatches
    y = np.arange(10, dtype=np.uint8) % 3
    b = _ArrayBatches(np.zeros((10, 4), np.float32), y, 5, False, pin=False, drop_remainder=False,
                      y_dtype=torch.int64)
    assert b.y.dtype == torch.int64 and b.y.tolist() == y.tolist()
    assert all(yb.dtype == torch.int64 for _, yb in b)
    same = _ArrayBatches(np.zeros((10, 4), np.float32), y, 5, False, pin=False, drop_remainder=False)
    assert same.y.dtype == torch.uint8


# ------------------------------------------------------------------------------------------------ the engine on the CPU
def _engine(loss, build=keras_mnist_cnn):
    stack = ExitStack()
    rec = trace._Recorder()
    stack.enter_context(mock.patch.object(native, "load", lambda: rec))
    stack.enter_context(mock.patch.object(GraphTrainEngine, "__init__", trace._stub_engine_init))
    stack.enter_context(mock.patch.object(torch.cuda, "get_device_properties",
                                          lambda dev=None: types.SimpleNamespace(multi_processor_count=132)))
    stack.enter_context(mock.patch.object(fastpath.FastSequentialEngine, "_s", lambda self: 0))
    env = {k: v for k, v in os.environ.items() if k not in trace.SWITCHES}
    stack.enter_context(mock.patch.dict(os.environ, env, clear=True))
    torch.manual_seed(0)
    m = build()
    m.compile(loss=loss, optimizer="sgd", metrics=["accuracy"])
    m._device = torch.device("cpu")
    m.build()
    plan = fastpath.build_plan(m)
    assert plan is not None
    return stack, rec, fastpath.FastSequentialEngine(m, plan, m.net, "adadelta")


def test_engine_reads_the_label_dtype_of_its_loss():
    stack, _, eng = _engine(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
    with stack:
        assert eng._ls == pytest.approx(0.1) and eng._y_dtype == torch.float32
        y = torch.eye(10, dtype=torch.float64)[:4]
        assert eng._head_targets(y).dtype == torch.float32
        with pytest.raises(ValueError, match=r"\(4, 7\).*\(batch, 10\)"):
            eng._head_targets(torch.zeros(4, 7))
        with pytest.raises(ValueError, match=r"\(4,\)"):
            eng._head_targets(torch.zeros(4, dtype=torch.int64))
    stack, _, eng = _engine(kl.SparseCategoricalCrossentropy(from_logits=True))
    with stack:
        assert eng._ls is None and eng._y_dtype == torch.int64
        y = torch.arange(4, dtype=torch.uint8)
        assert eng._head_targets(y).dtype == torch.int64 and eng._head_targets(y).tolist() == [0, 1, 2, 3]
        y64 = torch.arange(4)
        assert eng._head_targets(y64) is y64                 # int64 labels: today's path, no copy


def _step(loss, y, weights=None, env=None, build=keras_mnist_cnn):
    stack, rec, eng = _engine(loss, build)
    with stack:
        if env:
            stack.enter_context(mock.patch.dict(os.environ, env))
        C = eng.plan[-1].layer.units
        if weights == "class":
            eng._cw, eng._wmode = torch.linspace(0.5, 2.0, C), (True, False)
        elif weights == "sample":
            eng._wmode = (False, True)
        B = y.shape[0]
        g = torch.Generator().manual_seed(B)
        x = torch.rand((B,) + tuple(eng.plan[0].layer.input_shape_), generator=g)
        sw = torch.rand(B, generator=g) if weights == "sample" else None
        rec.calls, rec.roles = [], lambda ptr: trace._roles(eng, x, y, sw)(ptr)
        eng._forward_backward(x, y, sw)
        return [trace._fmt_call(c) for c in rec.calls], eng._launches_per_step


@pytest.mark.parametrize("env", [None, {"TFY_NO_FUSED_HEAD": "1"}])
@pytest.mark.parametrize("weights", [None, "sample", "class"])
def test_categorical_step_is_the_sparse_step_but_for_the_head_launch(weights, env):
    labels = torch.randint(0, 10, (128,), generator=torch.Generator().manual_seed(1))
    onehot = torch.nn.functional.one_hot(labels, 10).float()
    sparse, n_sparse = _step(trace.LOGITS, labels, weights, env)
    cat, n_cat = _step(kl.CategoricalCrossentropy(from_logits=True, label_smoothing=0.1), onehot, weights, env)
    assert n_sparse == n_cat and len(sparse) == len(cat)
    if env is None:
        assert n_cat == 10
    differ = [i for i, (a, b) in enumerate(zip(sparse, cat)) if a != b]
    assert len(differ) == 1, differ
    i = differ[0]
    fused = env is None
    want_sparse = ("tfy_dense_head_fused" if weights is None else "tfy_dense_head_fused_weighted") if fused else \
        ("tfy_softmax_xent" if weights is None else "tfy_softmax_xent_weighted")
    assert sparse[i].startswith(want_sparse + "(")
    name = "tfy_dense_head_fused_soft" if fused else "tfy_softmax_xent_soft"
    assert cat[i].startswith(name + "(")
    args = cat[i][len(name) + 1:-1].split(", ")
    s_args = sparse[i][len(want_sparse) + 1:-1].split(", ")
    ls = float(np.float32(0.1))
    if fused:
        # (h, w2, b2, y, ls, <the sparse launch's arguments after y>, sample_w, class_w, stream)
        assert args[3] == "y" and float(args[4]) == pytest.approx(ls)
        tail = s_args[4:] if weights is not None else s_args[4:-1] + ["null", "null", s_args[-1]]
        assert args[5:] == tail
    else:
        # (logits, bias, y, ls, sample_w, class_w, <the weighted launch's arguments after class_w>)
        assert args[2] == "y" and float(args[3]) == pytest.approx(ls)
        if weights is not None:
            assert args[4:] == s_args[3:]

