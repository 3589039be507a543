"""Keras AUC / Precision / Recall on the CPU: the float64 NumPy reference against hand-worked cases and the exact
Mann-Whitney AUC; the bucket function of the kernel built for the host at every float32 neighbour of every bucket edge;
the torch CPU histogram against the reference; the compile / fit / evaluate / save / callbacks API; and the binary
canned estimators' TF eval keys."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.stats
import torch

import confusion_reference as ref
from tf_yarn_b200 import data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import confusion

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"


# ----------------------------------------------------------------------------------------------- the reference itself
def test_reference_hand_cases():
    y = np.array([0, 0, 1, 1])
    assert ref.auc(y, [0.1, 0.2, 0.8, 0.9]) == pytest.approx(1.0)
    assert ref.auc(y, [0.9, 0.8, 0.2, 0.1]) == pytest.approx(0.0)
    assert ref.auc(y, [0.5, 0.5, 0.5, 0.5]) == pytest.approx(0.5)
    # thresholds [-eps, 0.5, 1+eps]: p = [0.3, 0.7, 0.7, 0.3] against y = [0, 0, 1, 1]
    # tp = [2, 1, 0], fp = [2, 1, 0], fn = [0, 1, 2], tn = [0, 1, 2]
    tp, fp, fn, tn = ref.confusion(y, [0.3, 0.7, 0.7, 0.3], num_thresholds=3)
    assert tp.tolist() == [2, 1, 0] and fp.tolist() == [2, 1, 0] and fn.tolist() == [0, 1, 2] and tn.tolist() == [0, 1, 2]
    # ROC: points (1, 1), (0.5, 0.5), (0, 0) -> 0.5.  PR (majoring): recall 1 -> 0.5 -> 0, precision 0.5, 0.5, 0
    assert ref.auc_from_confusion(tp, fp, fn, tn) == pytest.approx(0.5)
    assert ref.auc_from_confusion(tp, fp, fn, tn, "PR", "majoring") == pytest.approx(0.5 * 0.5 + 0.5 * 0.5)
    assert ref.auc_from_confusion(tp, fp, fn, tn, "PR", "minoring") == pytest.approx(0.5 * 0.5 + 0.5 * 0.0)
    # Davis-Goadrich between (tp, p) = (2, 4) and (1, 2): slope 1/2, intercept 0 -> (1/2)*(1)/2 = 0.25; then
    # (1, 2) -> (0, 0): p_{j+1} = 0, log term 1 -> slope 1/2 * 1 / max(tp+fn, 0) = 0.5 * 1 / 2 = 0.25
    assert ref.auc_from_confusion(tp, fp, fn, tn, "PR", "interpolation") == pytest.approx(0.5)
    assert ref.precision(y, [0.3, 0.7, 0.7, 0.3]).tolist() == [0.5]
    assert ref.recall(y, [0.3, 0.7, 0.9, 0.8], thresholds=[0.75, 0.5]).tolist() == [1.0, 1.0]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_reference_roc_matches_the_exact_mann_whitney_auc(seed):
    """Predictions in the middle of buckets (ties count 1/2): the trapezoid sum is the exact AUC."""
    rng = np.random.default_rng(seed)
    T = 101
    k = rng.integers(0, T - 1, 500)
    p = ((k + 0.5) / (T - 1)).astype(np.float32)
    y = (rng.random(500) < 0.2 + 0.6 * p).astype(np.int64)
    u = scipy.stats.mannwhitneyu(p[y == 1], p[y == 0]).statistic
    exact = u / ((y == 1).sum() * (y == 0).sum())
    assert ref.auc(y, p, num_thresholds=T) == pytest.approx(exact, abs=1e-12)


# --------------------------------------------------------------------------------- the bucket function on the host
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("confusion") / "libconfusion.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "confusion_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.tfy_host_conf_bucket_even.argtypes = [vp, i, i, vp]
    lib.tfy_host_conf_bucket_even.restype = None
    lib.tfy_host_conf_bucket_sorted.argtypes = [vp, i, vp, i, vp]
    lib.tfy_host_conf_bucket_sorted.restype = None
    return lib


@pytest.mark.parametrize("T", [2, 3, 200, 1000])
def test_host_built_bucket_function_matches_the_reference_at_every_edge(host_lib, T):
    p = np.ascontiguousarray(ref.edge_values(T))
    out = np.zeros(p.size, np.int32)
    host_lib.tfy_host_conf_bucket_even(p.ctypes.data, p.size, T, out.ctypes.data)
    np.testing.assert_array_equal(out, ref.bucket_even(p, T))
    # explicit (sorted) thresholds at the same edges: positive at j iff p > t_j
    thr = np.ascontiguousarray(np.sort(np.unique((np.arange(T) / (T - 1)).astype(np.float32))))
    host_lib.tfy_host_conf_bucket_sorted(p.ctypes.data, p.size, thr.ctypes.data, thr.size, out.ctypes.data)
    c = (p[:, None] > thr[None, :]).sum(axis=1)
    np.testing.assert_array_equal(out, np.where(c == 0, thr.size, c - 1))


# ------------------------------------------------------------------------------- the torch CPU path vs the reference
def _data(n, seed, labels="int", weights=False, logits=False):
    g = np.random.default_rng(seed)
    p = g.random(n).astype(np.float32)
    if labels == "int":
        y = (g.random(n) < p).astype(np.int64)
    elif labels == "float":
        y = (g.random(n) < p).astype(np.float32)
    else:
        y = g.random(n).astype(np.float32)
    w = None
    if weights:
        w = g.random(n).astype(np.float32) * 3
        w[g.random(n) < 0.2] = 0.0
    if logits:
        p = (g.standard_normal(n) * 3).astype(np.float32)
    return y, p, w


@pytest.mark.parametrize("T", [2, 3, 200, 1000])
@pytest.mark.parametrize("labels", ["int", "float", "soft"])
@pytest.mark.parametrize("weights", [False, True])
def test_cpu_histogram_matches_the_reference(T, labels, weights):
    y, p, w = _data(3000, T, labels, weights)
    st = confusion.ConfusionState(T)
    st.update(torch.from_numpy(y), torch.from_numpy(p), None if w is None else torch.from_numpy(w))
    h = st.histogram().numpy()
    want = ref.histogram(y, p, w, T)
    np.testing.assert_allclose(h, want, rtol=1e-12, atol=1e-9)
    tp, fp, fn, tn = confusion.confusion(torch.from_numpy(h), T)
    for a, b in zip((tp, fp, fn, tn), ref.confusion(y, p, w, T)):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-9)
    if not weights:
        assert h.sum() == p.size


@pytest.mark.parametrize("curve", ["ROC", "PR"])
@pytest.mark.parametrize("method", ["interpolation", "minoring", "majoring"])
@pytest.mark.parametrize("T", [2, 3, 200, 1000])
def test_auc_matches_the_reference(curve, method, T):
    y, p, w = _data(2000, 7, "int", True)
    m = keras.metrics.AUC(num_thresholds=T, curve=curve, summation_method=method)
    for s in range(0, 2000, 500):                                  # streamed over four batches
        m.update_state(torch.from_numpy(y[s:s + 500]), torch.from_numpy(p[s:s + 500]),
                       sample_weight=torch.from_numpy(w[s:s + 500]))
    assert m.result() == pytest.approx(ref.auc(y, p, w, T, curve, method), rel=1e-10, abs=1e-12)


def test_auc_explicit_thresholds_and_from_logits():
    y, x, _ = _data(1500, 3, "float", logits=True)
    thr = [0.8, 0.1, 0.5, 0.3]
    m = keras.metrics.AUC(thresholds=thr, from_logits=True, curve="PR")
    m.update_state(torch.from_numpy(y), torch.from_numpy(x))
    assert m.result() == pytest.approx(ref.auc(y, x, thresholds=thr, from_logits=True, curve="PR"), rel=1e-10)
    m = keras.metrics.AUC(from_logits=True)
    m.update_state(torch.from_numpy(y), torch.from_numpy(x))
    assert m.result() == pytest.approx(ref.auc(y, x, from_logits=True), rel=1e-10)


@pytest.mark.parametrize("labels", ["int", "float", "soft"])
def test_precision_recall_match_the_reference_in_the_order_given(labels):
    y, p, w = _data(2500, 11, labels, True)
    thr = [0.7, 0.2, 0.5, 0.5, 0.95]
    P, R = keras.metrics.Precision(thresholds=thr), keras.metrics.Recall(thresholds=thr)
    for m in (P, R):
        m.update_state(torch.from_numpy(y), torch.from_numpy(p), torch.from_numpy(w))
    np.testing.assert_allclose(P.result(), ref.precision(y, p, w, thr), rtol=1e-12)
    np.testing.assert_allclose(R.result(), ref.recall(y, p, w, thr), rtol=1e-12)
    P1 = keras.metrics.Precision()
    P1.update_state(torch.from_numpy(y), torch.from_numpy(p))
    assert isinstance(P1.result(), float)
    assert P1.result() == pytest.approx(float(ref.precision(y, p)[0]), rel=1e-12)


@pytest.mark.parametrize("thr", [0.5, np.float32(0.5), np.float64(0.5), np.array(0.5)])
def test_scalar_thresholds_of_any_numeric_type(thr):
    y, p, _ = _data(500, 4, "int")
    m = keras.metrics.Precision(thresholds=thr)
    m.update_state(torch.from_numpy(y), torch.from_numpy(p))
    assert isinstance(m.result(), float)
    assert m.result() == pytest.approx(float(ref.precision(y, p)[0]), rel=1e-12)


def test_precision_with_no_positive_prediction_is_zero():
    m = keras.metrics.Precision(thresholds=0.9)
    m.update_state(torch.tensor([1, 0]), torch.tensor([0.1, 0.2]))
    assert m.result() == 0.0


@pytest.mark.parametrize("y,p,what", [([0, 1], [0.5, 1.5], "predictions"), ([0, 1], [0.5, float("nan")], "predictions"),
                                       ([0, 2], [0.5, 0.5], "labels"), ([0, -1], [0.5, 0.5], "labels")])
def test_invalid_inputs_raise_on_result(y, p, what):
    m = keras.metrics.AUC()
    m.update_state(torch.tensor(y), torch.tensor(p))
    with pytest.raises(ValueError, match=what):
        m.result()


# ------------------------------------------------------------------------------------------------------------ the API
def test_unsupported_arguments_name_themselves():
    for kw in (dict(multi_label=True), dict(num_labels=3), dict(label_weights=[1.0])):
        with pytest.raises(ValueError, match=next(iter(kw))):
            keras.metrics.AUC(**kw)
    for kw in (dict(top_k=2), dict(class_id=1)):
        with pytest.raises(ValueError, match=next(iter(kw))):
            keras.metrics.Precision(**kw)
        with pytest.raises(ValueError, match=next(iter(kw))):
            keras.metrics.Recall(**kw)
    with pytest.raises(ValueError, match="num_thresholds"):
        keras.metrics.AUC(num_thresholds=1001)


def test_resolve_accepts_class_names_and_objects_not_lowercase_auc():
    name, m = keras.metrics.resolve("AUC", "binary_crossentropy", 1)
    assert name == "auc" and isinstance(m, keras.metrics.AUC)
    obj = keras.metrics.AUC(name="my_auc", curve="PR")
    name, m = keras.metrics.resolve(obj, "binary_crossentropy", 1)
    assert name == "my_auc" and m is not obj and m.curve == "PR"
    assert keras.metrics.resolve("Precision", "mse", 1)[0] == "precision"
    assert keras.metrics.resolve("Recall", "mse", 1)[0] == "recall"
    with pytest.raises(ValueError, match="unknown metric"):
        keras.metrics.resolve("auc", "mse", 1)


def _binary_model(seed=0):
    torch.manual_seed(seed)
    m = keras.Sequential([keras.layers.Dense(8, activation="relu", input_shape=(4,)),
                          keras.layers.Dense(1, activation="sigmoid")])
    return m


def _binary_data(n=256, seed=0):
    g = np.random.default_rng(seed)
    x = g.standard_normal((n, 4)).astype(np.float32)
    y = (x[:, 0] + 0.5 * g.standard_normal(n) > 0).astype(np.float32)
    return x, y


def test_duplicate_metric_names_are_rejected():
    m = _binary_model()
    with pytest.raises(ValueError, match="'auc' is used twice"):
        m.compile("sgd", "binary_crossentropy", metrics=["AUC", keras.metrics.AUC()])
    m.compile("sgd", "binary_crossentropy", metrics=["AUC", keras.metrics.AUC(name="auc_pr", curve="PR")])


def test_fit_reports_streaming_auc_per_epoch_and_val_keys():
    x, y = _binary_data()
    m = _binary_model()
    m.compile(keras.optimizers.SGD(0.0), "binary_crossentropy",
              metrics=["AUC", keras.metrics.Precision(name="prec"), "Recall", "accuracy"])
    hist = m.fit(x, y, batch_size=64, epochs=2, shuffle=False, verbose=0, validation_data=(x[:128], y[:128]))
    h = hist.history
    for k in ("auc", "prec", "recall", "accuracy", "val_auc", "val_prec", "val_recall", "val_accuracy"):
        assert k in h and len(h[k]) == 2, k
    p = m.predict(x, batch_size=64).reshape(-1)
    want = ref.auc(y, p)
    # learning rate 0: both epochs see the same predictions; reset between epochs keeps them equal
    assert h["auc"][0] == pytest.approx(want, rel=1e-9) and h["auc"][1] == pytest.approx(want, rel=1e-9)
    assert h["val_auc"][0] == pytest.approx(ref.auc(y[:128], p[:128]), rel=1e-9)
    assert h["prec"][0] == pytest.approx(float(ref.precision(y, p)[0]), rel=1e-9)
    res = m.evaluate(x, y, batch_size=50, return_dict=True)
    assert res["auc"] == pytest.approx(want, rel=1e-9)


def test_weighted_metrics_auc_uses_sample_weight():
    x, y = _binary_data(200, 1)
    w = np.random.default_rng(5).random(200).astype(np.float32)
    m = _binary_model(1)
    m.compile(keras.optimizers.SGD(0.0), "binary_crossentropy", metrics=["AUC"], weighted_metrics=["AUC"])
    res = m.evaluate(x, y, batch_size=64, sample_weight=w, return_dict=True)
    p = m.predict(x, batch_size=64).reshape(-1)
    assert res["auc"] == pytest.approx(ref.auc(y, p), rel=1e-9)
    assert res["weighted_auc"] == pytest.approx(ref.auc(y, p, w), rel=1e-9)
    hist = m.fit(x, y, batch_size=50, epochs=1, shuffle=False, verbose=0, sample_weight=w)
    assert hist.history["weighted_auc"][0] == pytest.approx(ref.auc(y, p, w), rel=1e-9)


def test_save_load_model_keeps_metric_configs(tmp_path):
    x, y = _binary_data(64)
    m = _binary_model()
    m.compile("sgd", "binary_crossentropy",
              metrics=["accuracy", "AUC", keras.metrics.AUC(num_thresholds=50, curve="PR", summation_method="minoring",
                                                            name="pr"),
                       keras.metrics.Recall(thresholds=[0.3, 0.6], name="rec")])
    m.fit(x, y, batch_size=32, epochs=1, verbose=0)
    m.save(str(tmp_path / "m.ckpt"))
    m2 = keras.models.load_model(str(tmp_path / "m.ckpt"))
    specs = m2._metrics_spec
    assert specs[0] == "accuracy" and specs[1] == "AUC"
    assert isinstance(specs[2], keras.metrics.AUC) and specs[2].get_config() == m._metrics_spec[2].get_config()
    assert specs[3].get_config() == {"thresholds": [0.3, 0.6], "name": "rec"}
    res = m2.evaluate(x, y, batch_size=32, return_dict=True)
    assert isinstance(res["rec"], list) and len(res["rec"]) == 2 and "pr" in res


class _MeanPrediction(keras.metrics.Metric):
    """A user-defined stateful metric (not one load_model can rebuild)."""

    def __init__(self, name="mean_pred"):
        super().__init__(name)
        self.reset_state()

    def update_state(self, y_true, y_pred, sample_weight=None):
        self.s += float(y_pred.float().sum())
        self.n += y_pred.numel()

    def result(self):
        return self.s / max(self.n, 1)

    def reset_state(self):
        self.s, self.n = 0.0, 0


def test_user_defined_metric_is_left_out_of_the_save(tmp_path, caplog):
    x, y = _binary_data(64)
    m = _binary_model()
    m.compile("sgd", "binary_crossentropy", metrics=["AUC", _MeanPrediction()])
    res = m.evaluate(x, y, batch_size=32, return_dict=True)
    assert res["mean_pred"] == pytest.approx(float(m.predict(x, batch_size=32).mean()), rel=1e-5)
    m.save(str(tmp_path / "m.ckpt"))
    m2 = keras.models.load_model(str(tmp_path / "m.ckpt"))
    assert m2._metrics_spec == ["AUC"]
    assert keras.metrics.deserialize({"class_name": "NoSuchMetric", "config": {}}) is None
    assert "NoSuchMetric" in caplog.text


def test_weighted_metrics_alone_cover_every_evaluate_batch():
    """With weighted_metrics and no plain metrics, evaluate accumulates over all batches, not the last one."""
    x, y = _binary_data(250, 3)
    w = np.random.default_rng(6).random(250).astype(np.float32)
    m = _binary_model(3)
    m.compile(keras.optimizers.SGD(0.0), "binary_crossentropy", weighted_metrics=["accuracy"])
    res = m.evaluate(x, y, batch_size=64, sample_weight=w, return_dict=True)
    p = m.predict(x, batch_size=64).reshape(-1)
    hit = ((p > 0.5) == (y > 0.5)).astype(np.float64)
    assert res["accuracy"] == pytest.approx(float((hit * w).sum() / w.sum()), rel=1e-6)


def test_callbacks_auto_mode_maximises_auc_precision_recall(tmp_path):
    for mon in ("val_auc", "auc", "val_precision", "recall", "val_acc"):
        cb = keras.callbacks.EarlyStopping(monitor=mon)
        assert cb._sign == 1.0, mon
        ck = keras.callbacks.ModelCheckpoint(str(tmp_path / "x"), monitor=mon)
        assert ck._better(2, 1), mon
    assert keras.callbacks.EarlyStopping(monitor="val_loss")._sign == -1.0
    assert not keras.callbacks.ModelCheckpoint(str(tmp_path / "x"), monitor="val_loss")._better(2, 1)


# ---------------------------------------------------------------------------------------------- canned estimators
BINARY_KEYS = {"auc", "auc_precision_recall", "precision", "recall", "label/mean", "prediction/mean",
               "accuracy_baseline"}


def _est_data(n=240, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 5, generator=g)
    y = ((x[:, 0] - x[:, 1] + 0.7 * torch.randn(n, generator=g)) > 0).long()
    return x, y


def _check_binary_eval(e, x, y):
    evalf = lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(64)   # noqa: E731
    res = e.evaluate(evalf)
    assert BINARY_KEYS <= set(res)
    logits = np.concatenate([np.asarray(r["logits"]).reshape(-1)
                             for r in e.predict(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(64))])
    yn = y.numpy()
    assert res["auc"] == pytest.approx(ref.auc(yn, logits, from_logits=True), rel=1e-9)
    assert res["auc_precision_recall"] == pytest.approx(ref.auc(yn, logits, curve="PR", from_logits=True), rel=1e-9)
    assert res["precision"] == pytest.approx(float(ref.precision(yn, logits, from_logits=True)[0]), rel=1e-9)
    assert res["recall"] == pytest.approx(float(ref.recall(yn, logits, from_logits=True)[0]), rel=1e-9)
    assert res["label/mean"] == pytest.approx(yn.mean(), rel=1e-6)
    assert res["prediction/mean"] == pytest.approx(ref.sigmoid32(logits).astype(np.float64).mean(), rel=1e-5)
    m = yn.mean()
    assert res["accuracy_baseline"] == pytest.approx(max(m, 1 - m), rel=1e-12)
    # accuracy and average_loss keep their computation: logits > 0, mean binary cross-entropy over the batches
    assert res["accuracy"] == pytest.approx(((logits > 0).astype(np.int64) == yn).mean(), rel=1e-9)
    lg = torch.from_numpy(logits).double()
    bce = torch.nn.functional.binary_cross_entropy_with_logits(lg, y.double()).item()
    assert res["average_loss"] == pytest.approx(bce, rel=1e-4)
    return res


def test_binary_linear_classifier_reports_tf_binary_head_keys(tmp_path):
    x, y = _est_data()
    e = est.LinearClassifier([fc.numeric_column("x", shape=(5,))], model_dir=str(tmp_path), n_classes=2,
                             optimizer=lambda: keras.optimizers.Adam(0.05),
                             config=est.RunConfig(save_checkpoints_steps=20, log_step_count_steps=None))
    e.train(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(32).repeat(), max_steps=20)
    _check_binary_eval(e, x, y)


def test_binary_wide_and_deep_reports_tf_binary_head_keys(tmp_path):
    x, y = _est_data(seed=1)
    e = est.DNNLinearCombinedClassifier(model_dir=str(tmp_path), linear_feature_columns=[fc.numeric_column("x", shape=(5,))],
                                        dnn_feature_columns=[fc.numeric_column("x", shape=(5,))], dnn_hidden_units=[8],
                                        dnn_optimizer=lambda: keras.optimizers.Adam(0.01),
                                        config=est.RunConfig(save_checkpoints_steps=20, log_step_count_steps=None))
    e.train(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(32).repeat(), max_steps=20)
    _check_binary_eval(e, x, y)


def test_multiclass_head_keeps_its_key_set(tmp_path):
    x, _ = _est_data()
    y = (x[:, 0] > 0).long() + (x[:, 1] > 0.5).long()
    e = est.LinearClassifier([fc.numeric_column("x", shape=(5,))], model_dir=str(tmp_path), n_classes=3,
                             optimizer=lambda: keras.optimizers.Adam(0.05),
                             config=est.RunConfig(save_checkpoints_steps=10, log_step_count_steps=None))
    e.train(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(32).repeat(), max_steps=10)
    res = e.evaluate(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(64))
    assert set(res) == {"loss", "accuracy", "average_loss", "global_step"}


def test_metric_objects_in_eval_metric_ops_reset_between_evaluations(tmp_path):
    x, y = _est_data(seed=2)
    e = est.LinearClassifier([fc.numeric_column("x", shape=(5,))], model_dir=str(tmp_path), n_classes=2,
                             optimizer=lambda: keras.optimizers.Adam(0.05),
                             config=est.RunConfig(save_checkpoints_steps=10, log_step_count_steps=None))
    e.train(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(32).repeat(), max_steps=10)
    feed = lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(64)    # noqa: E731
    r1, r2 = e.evaluate(feed), e.evaluate(feed)
    assert r1["auc"] == r2["auc"] and r1["precision"] == r2["precision"] and 0.0 < r1["auc"] <= 1.0
