"""Keras sample weighting on the eager (CPU) engine: ``fit(sample_weight=, class_weight=)``, ``(x, y, w)`` batches,
``evaluate(sample_weight=)`` and ``compile(weighted_metrics=)``, against hand-written torch references of
``loss = sum(w * l) / B``."""
import logging

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tf_yarn_b200 import data, keras

N, LR = 24, 0.1


def _model(units, activation=None, loss="mse", metrics=None, weighted_metrics=None, seed=0):
    torch.manual_seed(seed)
    m = keras.Sequential()
    m.add(keras.layers.Dense(8, activation="relu", input_shape=(4,)))
    m.add(keras.layers.Dense(units, activation=activation))
    m.compile(loss=loss, optimizer=keras.optimizers.SGD(LR), metrics=metrics or [],
              weighted_metrics=weighted_metrics)
    m._device = torch.device("cpu")
    m.build()
    return m


def _x(n=N, seed=0):
    return torch.randn(n, 4, generator=torch.Generator().manual_seed(seed))


def _labels(n=N, classes=3, seed=1):
    return torch.randint(0, classes, (n,), generator=torch.Generator().manual_seed(seed))


def _weights(n=N, seed=2):
    return torch.rand(n, generator=torch.Generator().manual_seed(seed)) * 2


def _one_step(m, x, y, **kw):
    """One SGD step on the whole batch; returns (loss, weights after the step)."""
    h = m.fit(x, y, batch_size=len(x), epochs=1, shuffle=False, verbose=0, **kw)
    return h.history["loss"][0], [torch.as_tensor(w) for w in m.get_weights()]


def _reference_step(weights, x, y, w, per_sample):
    w1, b1, w2, b2 = [t.clone().double().requires_grad_(True) for t in weights]
    out = F.linear(F.relu(F.linear(x.double(), w1, b1)), w2, b2)
    y = y.double() if y.is_floating_point() else y
    loss = (per_sample(y, out) * w.double()).sum() / len(x)
    loss.backward()
    return float(loss), [(t - LR * t.grad).detach().float() for t in (w1, b1, w2, b2)]


_CASES = {
    "sparse_ce_logits": (3, None, lambda: keras.losses.SparseCategoricalCrossentropy(from_logits=True), _labels,
                         lambda y, o: F.cross_entropy(o, y, reduction="none")),
    "sparse_ce_probs": (3, "softmax", lambda: "sparse_categorical_crossentropy", _labels,
                        lambda y, o: -torch.log(o.softmax(-1).gather(1, y[:, None])[:, 0].clamp_min(1e-7))),
    "categorical_ce": (3, "softmax", lambda: "categorical_crossentropy", lambda: F.one_hot(_labels(), 3).float(),
                       lambda y, o: -(y * torch.log(o.softmax(-1).clamp_min(1e-7))).sum(-1)),
    "binary_ce": (1, "sigmoid", lambda: "binary_crossentropy", lambda: _labels(classes=2)[:, None].float(),
                  lambda y, o: F.binary_cross_entropy(o.sigmoid().clamp(1e-7, 1 - 1e-7), y, reduction="none")[:, 0]),
    "mse": (2, None, lambda: "mse", lambda: torch.randn(N, 2, generator=torch.Generator().manual_seed(3)),
            lambda y, o: ((o - y) ** 2).mean(1)),
    "mae": (2, None, lambda: "mae", lambda: torch.randn(N, 2, generator=torch.Generator().manual_seed(3)),
            lambda y, o: (o - y).abs().mean(1)),
}


@pytest.mark.parametrize("case", sorted(_CASES))
def test_weighted_sgd_step_matches_torch_reference(case):
    units, act, loss, make_y, per_sample = _CASES[case]
    m = _model(units, act, loss())
    x, y, w = _x(), make_y(), _weights()
    init = [torch.as_tensor(t) for t in m.get_weights()]
    loss_val, after = _one_step(m, x, y, sample_weight=w)
    ref_loss, ref_after = _reference_step(init, x, y, w, per_sample)
    assert loss_val == pytest.approx(ref_loss, rel=1e-5, abs=1e-6)
    for a, b in zip(after, ref_after):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["sparse", "one_hot", "binary"])
def test_class_weight_equals_the_matching_sample_weight(kind):
    units, act, loss, y = {
        "sparse": (3, None, "sparse_categorical_crossentropy", _labels()),
        "one_hot": (3, "softmax", "categorical_crossentropy", F.one_hot(_labels(), 3).float()),
        "binary": (1, "sigmoid", "binary_crossentropy", _labels(classes=2)[:, None].float()),
    }[kind]
    cw = {0: 0.5, 1: 2.0, 2: 3.0} if units == 3 else {0: 0.25, 1: 4.0}
    cls = y.argmax(-1) if kind == "one_hot" else y.reshape(-1).round().long()
    table = torch.tensor([cw[c] for c in range(len(cw))])
    l1, p1 = _one_step(_model(units, act, loss), _x(), y, class_weight=cw)
    l2, p2 = _one_step(_model(units, act, loss), _x(), y, sample_weight=table[cls])
    assert l1 == pytest.approx(l2, rel=1e-6)
    for a, b in zip(p1, p2):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)
    # both: the product
    sw = _weights()
    l3, p3 = _one_step(_model(units, act, loss), _x(), y, class_weight=cw, sample_weight=sw)
    l4, p4 = _one_step(_model(units, act, loss), _x(), y, sample_weight=sw * table[cls])
    assert l3 == pytest.approx(l4, rel=1e-6)
    for a, b in zip(p3, p4):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)


def test_missing_classes_weigh_one_with_a_warning(caplog):
    y = _labels()
    with caplog.at_level(logging.WARNING):
        l1, p1 = _one_step(_model(3, loss="sparse_categorical_crossentropy"), _x(), y, class_weight={1: 2.0})
    assert "class_weight" in caplog.text and "[0, 2]" in caplog.text
    l2, p2 = _one_step(_model(3, loss="sparse_categorical_crossentropy"), _x(), y,
                       sample_weight=torch.where(y == 1, 2.0, 1.0))
    assert l1 == pytest.approx(l2, rel=1e-6)


def test_bad_arguments_raise_value_error():
    x, y = _x(), _labels()
    for bad in ({3: 1.0}, {-1: 1.0}, {"a": 1.0}, {0.5: 1.0}):
        with pytest.raises(ValueError, match="class_weight"):
            _model(3, loss="sparse_categorical_crossentropy").fit(x, y, batch_size=8, verbose=0, class_weight=bad)

    def scalar_loss(y_true, y_pred):
        return ((y_pred - y_true) ** 2).mean()
    m = _model(1, loss=scalar_loss)
    with pytest.raises(ValueError, match="per sample"):
        m.fit(x, y[:, None].float(), batch_size=8, verbose=0, sample_weight=_weights())
    m = _model(1, loss=scalar_loss)
    m.fit(x, y[:, None].float(), batch_size=8, verbose=0)             # unweighted: a scalar loss is fine
    with pytest.raises(ValueError, match="weighted_metrics"):
        _model(3, loss="sparse_categorical_crossentropy", weighted_metrics=[lambda a, b: (a.sum(), 1.0)])
    with pytest.raises(ValueError, match="sample_weight"):
        _model(3, loss="sparse_categorical_crossentropy").fit(iter([(x, y)]), steps_per_epoch=1, verbose=0,
                                                               sample_weight=_weights())


def test_custom_per_sample_loss_with_weights():
    def per_sample_mse(y_true, y_pred):
        return ((y_pred - y_true) ** 2).mean(dim=1)
    y, w = torch.randn(N, 2), _weights()
    l1, p1 = _one_step(_model(2, loss=per_sample_mse), _x(), y, sample_weight=w)
    l2, p2 = _one_step(_model(2, loss="mse"), _x(), y, sample_weight=w)
    assert l1 == pytest.approx(l2, rel=1e-6)
    for a, b in zip(p1, p2):
        torch.testing.assert_close(a, b)


def test_zero_weights_leave_parameters_unchanged():
    m = _model(3, loss="sparse_categorical_crossentropy")
    before = [torch.as_tensor(t) for t in m.get_weights()]
    h = m.fit(_x(), _labels(), batch_size=8, epochs=2, shuffle=True, verbose=0, sample_weight=torch.zeros(N))
    assert h.history["loss"] == [0.0, 0.0]
    for a, b in zip(before, m.get_weights()):
        assert torch.equal(a, torch.as_tensor(b))


def test_zeroing_one_class_matches_training_on_the_other_class_alone():
    x, y = _x(), _labels(classes=2)
    keep = y == 1
    k = int(keep.sum())
    l1, p1 = _one_step(_model(2, loss="sparse_categorical_crossentropy"), x, y, class_weight={0: 0.0, 1: 1.0})
    # the loss divides by the whole batch B: the plain mean over the kept samples, scaled by k / B
    l2, _ = _one_step(_model(2, loss="sparse_categorical_crossentropy"), x[keep], y[keep])
    assert l1 == pytest.approx(l2 * k / N, rel=1e-5)
    l3, p3 = _one_step(_model(2, loss="sparse_categorical_crossentropy"), x[keep], y[keep],
                       sample_weight=torch.full((k,), k / N))
    assert l1 == pytest.approx(l3, rel=1e-5)
    for a, b in zip(p1, p3):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_metrics_stay_unweighted_and_weighted_metrics_get_the_prefix():
    x, y = _x(), _labels()
    w = torch.where(y == 0, 3.0, 0.5)
    m = _model(3, loss="sparse_categorical_crossentropy", metrics=["accuracy"], weighted_metrics=["accuracy"])
    m.optimizer.learning_rate = 0.0
    h = m.fit(x, y, batch_size=8, epochs=1, shuffle=False, verbose=0, sample_weight=w)
    assert set(h.history) == {"loss", "accuracy", "weighted_accuracy"}
    with torch.no_grad():
        hit = (m.net(x).argmax(-1) == y).float()
    assert h.history["accuracy"][0] == pytest.approx(float(hit.mean()), abs=1e-6)
    assert h.history["weighted_accuracy"][0] == pytest.approx(float((hit * w).sum() / w.sum()), abs=1e-6)
    res = m.evaluate(x, y, sample_weight=w, return_dict=True)
    assert res["accuracy"] == pytest.approx(float(hit.mean()), abs=1e-6)
    assert res["weighted_accuracy"] == pytest.approx(float((hit * w).sum() / w.sum()), abs=1e-6)
    only = _model(3, loss="sparse_categorical_crossentropy", weighted_metrics=["accuracy"])
    assert set(only.evaluate(x, y, return_dict=True)) == {"loss", "accuracy"}


def test_evaluate_sample_weight_validation_triples_and_datasets():
    x, y, w = _x(), _labels(), _weights()
    m = _model(3, "softmax", loss="sparse_categorical_crossentropy", weighted_metrics=["accuracy"])
    with torch.no_grad():
        per = F.nll_loss(m.net(x).clamp_min(1e-7).log(), y, reduction="none")
    res = m.evaluate(x, y, sample_weight=w, batch_size=5, return_dict=True)
    assert res["loss"] == pytest.approx(float((per * w).sum() / N), rel=1e-5)
    assert m.evaluate((x, y, w), batch_size=7, return_dict=True)["loss"] == pytest.approx(res["loss"], rel=1e-6)
    ds = data.Dataset.from_tensor_slices((x, y, w)).batch(6)
    assert m.evaluate(ds, return_dict=True)["loss"] == pytest.approx(res["loss"], rel=1e-6)
    # validation_data triple, validation_split with weights
    h = m.fit(x, y, batch_size=8, epochs=1, verbose=0, validation_data=(x, y, w))
    assert h.history["val_loss"][0] == pytest.approx(m.evaluate(x, y, sample_weight=w, return_dict=True)["loss"],
                                                     rel=1e-5)
    m2 = _model(3, loss="sparse_categorical_crossentropy")
    h2 = m2.fit(x, y, batch_size=6, epochs=1, verbose=0, sample_weight=w, validation_split=0.25, shuffle=False)
    assert h2.history["val_loss"][0] == pytest.approx(
        m2.evaluate(x[18:], y[18:], sample_weight=w[18:], return_dict=True)["loss"], rel=1e-5)


def test_dataset_triples_train_like_sample_weight():
    x, y, w = _x(), _labels(), _weights()
    m1 = _model(3, loss="sparse_categorical_crossentropy")
    h1 = m1.fit(x, y, batch_size=8, epochs=2, shuffle=False, verbose=0, sample_weight=w)
    m2 = _model(3, loss="sparse_categorical_crossentropy")
    h2 = m2.fit(data.Dataset.from_tensor_slices((x, y, w)).batch(8), epochs=2, verbose=0)
    assert h1.history["loss"] == pytest.approx(h2.history["loss"], rel=1e-6)
    for a, b in zip(m1.get_weights(), m2.get_weights()):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-7)


def test_shuffled_weights_stay_with_their_samples():
    # a weight of zero on every sample but one: whatever the order, only that sample moves the parameters
    x, y = _x(), _labels()
    w = torch.zeros(N)
    w[5] = 1.0
    m1 = _model(3, loss="sparse_categorical_crossentropy")
    m1.fit(x, y, batch_size=N, epochs=1, shuffle=True, verbose=0, sample_weight=w)
    m2 = _model(3, loss="sparse_categorical_crossentropy")
    m2.fit(x[5:6], y[5:6], batch_size=1, epochs=1, shuffle=False, verbose=0, sample_weight=torch.tensor([1.0 / N]))
    for a, b in zip(m1.get_weights(), m2.get_weights()):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-7)


def test_weighted_metrics_survive_save_and_load(tmp_path):
    m = _model(3, loss="sparse_categorical_crossentropy", metrics=["accuracy"], weighted_metrics=["accuracy"])
    m.fit(_x(), _labels(), batch_size=8, epochs=1, verbose=0)
    path = str(tmp_path / "m.ckpt")
    m.save(path)
    m2 = keras.models.load_model(path)
    assert m2._weighted_metrics_spec == ["accuracy"]
    assert set(m2.evaluate(_x(), _labels(), return_dict=True)) == {"loss", "accuracy", "weighted_accuracy"}
