"""The estimator heads and the head-taking estimators on the CPU: the multi-label, Poisson and logistic heads' torch
statement and the host build of their kernel math (ops/csrc/tfy_head.cuh) against the float64 reference
(tests/head_kinds_reference.py); argument validation of every head and estimator; each of the six classifiers and
regressors against its ``*Estimator(head=...)`` twin, bit for bit; each new head trained, evaluated, used to predict,
exported and resumed; the multi-label metrics against the reference; and a multi-process run on the shared-memory
parameter-server plane with ``MultiLabelHead``."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import head_kinds_reference as ref
from tf_yarn_b200 import data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import head as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"
KINDS = [ref.MULTI_LABEL, ref.POISSON, ref.POISSON_FULL, ref.LOGISTIC]
KIND_IDS = ["multi_label", "poisson", "poisson_full", "logistic"]


# ------------------------------------------------------------------------------------------------- inputs
def kinds_inputs(head, B, C, seed, weighted=True, label_dtype=torch.float32, zmax=4.0, poisson_hi=20.0, bad=False):
    """Random logits (5 % at -80 and 5 % at +80, or at +poisson_hi for the Poisson heads), labels of the head (Poisson
    counts 0, 1, small, 1e4 and 1e6), and weights with zeros and negatives.  ``bad`` puts invalid labels in rows 1 and
    B - 1 (and NaN in row 2 for float labels)."""
    g = np.random.default_rng(seed)
    z = (g.standard_normal((B, C)) * zmax / 3).astype(np.float32)
    hi = poisson_hi if head in (ref.POISSON, ref.POISSON_FULL) else 80.0
    z.reshape(-1)[g.random(B * C) < 0.05] = hi
    z.reshape(-1)[g.random(B * C) < 0.05] = -80.0
    floats = label_dtype == torch.float32
    if head == ref.MULTI_LABEL:
        y = (g.random((B, C)) < 0.3).astype(np.float64)
        if floats:
            y[g.random((B, C)) < 0.2] = 0.25
    elif head == ref.LOGISTIC:
        y = g.integers(0, 2, (B, C)).astype(np.float64)
        if floats:
            r = g.random((B, C))
            y = np.where(r < 0.6, g.random((B, C)), y)
    else:
        y = g.choice([0.0, 1.0, 2.0, 3.0, 7.0, 40.0, 1e4, 1e6], (B, C), p=[.2, .2, .15, .15, .1, .1, .05, .05])
        if floats:
            y[g.random((B, C)) < 0.2] = 2.5
            y[g.random((B, C)) < 0.1] = 0.5
    if bad and B > 2:
        y[1, 0] = 2.0 if head == ref.LOGISTIC else -1.0
        y[B - 1, C - 1] = -1.0 if head == ref.LOGISTIC else -3.0
        if floats:
            y[2, 0] = np.nan
    w = g.choice([0.0, -0.5, 0.25, 1.0, 1.5, 3.0], B).astype(np.float32) if weighted else None
    yt = torch.from_numpy(y).to(label_dtype)
    if C == 1 and head != ref.MULTI_LABEL:
        yt = yt.reshape(B)
    return torch.from_numpy(z), yt, None if w is None else torch.from_numpy(w)


def _np(t):
    return None if t is None else t.double().numpy()


# ------------------------------------------------------------------------- the torch statement vs the reference
CASES = [(ref.MULTI_LABEL, C, B) for C in (2, 10, 100) for B in (1, 7, 64)] + \
    [(h, d, B) for h in (ref.POISSON, ref.POISSON_FULL) for d in (1, 3) for B in (1, 7, 300)] + \
    [(ref.LOGISTIC, 1, B) for B in (1, 7, 300)]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("head,C,B", CASES)
def test_torch_statement_matches_the_reference(head, C, B, weighted):
    z, y, w = kinds_inputs(head, B, C, seed=B * 31 + C + head, weighted=weighted, poisson_hi=80.0)
    zr = z.clone().requires_grad_(True)
    loss = H.CannedHead(head, C)(y, zr, w)
    loss.backward()
    zn, yn, wn = z.double().numpy(), y.double().numpy(), _np(w)
    assert abs(loss.item() - ref.loss(head, zn, yn, wn)) <= ref.loss_tol(head, zn, yn, wn)
    np.testing.assert_array_less(np.abs(zr.grad.double().numpy() - ref.dlogits(head, zn, yn, wn)),
                                 ref.grad_tol(head, zn, yn, wn) + 1e-45)


@pytest.mark.parametrize("head", KINDS, ids=KIND_IDS)
def test_unweighted_torch_statement_is_the_torch_mean(head):
    C = 1 if head == ref.LOGISTIC else 4
    z, y, _ = kinds_inputs(head, 33, C, seed=head, weighted=False)
    got = H.CannedHead(head, C)(y, z)
    if head in (ref.MULTI_LABEL, ref.LOGISTIC):
        want = F.binary_cross_entropy_with_logits(z.reshape(-1), y.float().reshape(-1))
    else:
        want = F.poisson_nll_loss(z, y.reshape(z.shape), log_input=True, full=head == ref.POISSON_FULL)
    assert torch.equal(got, want)


@pytest.mark.parametrize("head", [ref.POISSON, ref.POISSON_FULL, ref.LOGISTIC], ids=KIND_IDS[1:])
def test_invalid_labels_raise_on_the_cpu(head):
    z, y, w = kinds_inputs(head, 16, 1, seed=3, bad=True)
    rule = "labels must be in \\[0, 1\\]" if head == ref.LOGISTIC else "labels must be counts >= 0"
    with pytest.raises(ValueError, match=rule):
        H.CannedHead(head, 1)(y, z, w)
    with pytest.raises(ValueError, match=rule):
        H.CannedHead(head, 1)(y, z)


def test_label_shapes_are_checked():
    z = torch.zeros(8, 3)
    with pytest.raises(ValueError, match="multi-label labels must have shape \\[8, 3\\]"):
        H.CannedHead(H.MULTI_LABEL, 3)(torch.zeros(8), z)
    with pytest.raises(ValueError, match="Poisson labels must have shape \\[8, 3\\]"):
        H.CannedHead(H.POISSON, 3)(torch.zeros(8, 2), z)
    with pytest.raises(ValueError, match="logistic labels must have shape \\[8\\] or \\[8, 1\\]"):
        H.CannedHead(H.LOGISTIC, 1)(torch.zeros(8, 2), z[:, :1])
    for shape in ((8,), (8, 1)):                    # [B] and [B, 1] for one output
        H.CannedHead(H.POISSON, 1)(torch.zeros(shape), z[:, :1])
        H.CannedHead(H.LOGISTIC, 1)(torch.zeros(shape), z[:, :1])
    with pytest.raises(ValueError, match="unknown head"):
        H.CannedHead(7, 1)


# ------------------------------------------------------------------------------------ the kernel's math, host-built
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("head_kinds") / "libhead_kinds.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "head_kinds_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.tfy_host_head_kinds.argtypes = [i, vp, vp, i, vp, vp, vp]
    lib.tfy_host_head_kinds.restype = None
    return lib


@pytest.mark.parametrize("head,C,B", CASES)
def test_host_built_head_math_matches_the_reference(host_lib, head, C, B):
    z, y, _ = kinds_inputs(head, B, C, seed=B + 7 * C + head, poisson_hi=80.0, bad=True)
    zn = np.ascontiguousarray(z.numpy(), dtype=np.float32)
    yn = np.ascontiguousarray(y.numpy().astype(np.float32).reshape(-1))
    n = B * C
    loss, grad, ok = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.int32)
    host_lib.tfy_host_head_kinds(head, zn.ctypes.data, yn.ctypes.data, n, loss.ctypes.data, grad.ctypes.data,
                                 ok.ctypes.data)
    zd, yd = z.double().numpy(), y.double().numpy()
    assert (ok.reshape(B, C) == 1).tolist() == ref.valid(head, yd.reshape(B, C)).tolist()
    err = np.abs(loss.astype(np.float64).reshape(B, C) - ref.element_losses(head, zd, yd))
    np.testing.assert_array_less(err, 8 * ref.EPS32 * ref.element_scale(head, zd, yd))
    np.testing.assert_array_less(np.abs(grad.astype(np.float64).reshape(B, C) - ref.element_grads(head, zd, yd)),
                                 ref.grad_tol(head, zd, yd) * n)


@pytest.mark.parametrize("full", [False, True])
def test_host_built_poisson_at_the_stirling_edges(host_lib, full):
    """y in {0, 1, just above 1, 2, large} (Stirling's term starts at y > 1) against |z| up to 80."""
    head = ref.POISSON_FULL if full else ref.POISSON
    ys = np.array([0.0, 1.0, np.nextafter(np.float32(1), np.float32(2)), 2.0, 40.0, 1e4, 1e6, 3e7], np.float32)
    zs = np.array([-80.0, -5.0, 0.0, 1e-3, 2.0, 17.0, 80.0], np.float32)
    z, y = np.meshgrid(zs, ys)
    z, y = np.ascontiguousarray(z.reshape(-1, 1)), np.ascontiguousarray(y.reshape(-1))
    n = y.size
    loss, grad, ok = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.int32)
    host_lib.tfy_host_head_kinds(head, z.ctypes.data, y.ctypes.data, n, loss.ctypes.data, grad.ctypes.data,
                                 ok.ctypes.data)
    zd, yd = z.astype(np.float64), y.astype(np.float64).reshape(-1, 1)
    err = np.abs(loss.astype(np.float64) - ref.element_losses(head, zd, yd).reshape(-1))
    np.testing.assert_array_less(err, 8 * ref.EPS32 * ref.element_scale(head, zd, yd).reshape(-1))
    torch_loss = F.poisson_nll_loss(torch.from_numpy(z).reshape(-1), torch.from_numpy(y), log_input=True, full=full,
                                    reduction="none").double().numpy()
    np.testing.assert_array_less(np.abs(torch_loss - ref.element_losses(head, zd, yd).reshape(-1)),
                                 8 * ref.EPS32 * ref.element_scale(head, zd, yd).reshape(-1))


# --------------------------------------------------------------------------------------------- argument validation
def _cols():
    return [fc.numeric_column("x", (3,))]


def test_head_arguments_are_validated():
    for bad in (1, 0, 2.0, True, "3"):
        with pytest.raises(ValueError, match="n_classes"):
            est.MultiLabelHead(bad)
    for bad in (2, 1, True):
        with pytest.raises(ValueError, match="n_classes"):
            est.MultiClassHead(bad)
    for cls in (est.RegressionHead, est.PoissonRegressionHead):
        for bad in (0, -1, 1.5, True):
            with pytest.raises(ValueError, match="label_dimension"):
                cls(bad)
    for bad in ([0.0], [1.0], [0.5, 1.5], [-0.1]):
        with pytest.raises(ValueError, match="thresholds"):
            est.BinaryClassHead(thresholds=bad)
        with pytest.raises(ValueError, match="thresholds"):
            est.MultiLabelHead(3, thresholds=bad)
    for bad in ([3], [-1], [1.0], [True]):
        with pytest.raises(ValueError, match="classes_for_class_based_metrics"):
            est.MultiLabelHead(3, classes_for_class_based_metrics=bad)
    makers = [lambda **k: est.BinaryClassHead(**k), lambda **k: est.MultiClassHead(3, **k),
              lambda **k: est.RegressionHead(**k), lambda **k: est.MultiLabelHead(3, **k),
              lambda **k: est.PoissonRegressionHead(**k), lambda **k: est.LogisticRegressionHead(**k)]
    for make in makers:
        make(loss_reduction=est.SUM_OVER_BATCH_SIZE, name=None)
        with pytest.raises(ValueError, match="loss_reduction"):
            make(loss_reduction="sum")
        with pytest.raises(ValueError, match="name"):
            make(name="head")
        with pytest.raises(TypeError, match="weight_column"):
            make(weight_column=3)
    for make in makers[:4]:
        with pytest.raises(ValueError, match="loss_fn"):
            make(loss_fn=lambda y, z: z)
    for make in (makers[0], makers[1], makers[3]):
        with pytest.raises(ValueError, match="label_vocabulary"):
            make(label_vocabulary=["a", "b", "c"])
        make(label_vocabulary=None)
    with pytest.raises(ValueError, match="inverse_link_fn"):
        est.RegressionHead(inverse_link_fn=torch.exp)


def test_estimator_arguments_are_validated():
    head = est.MultiLabelHead(3)
    with pytest.raises(TypeError, match="head"):
        est.DNNEstimator(3, [4], _cols())
    with pytest.raises(ValueError, match="activation_fn"):
        est.DNNEstimator(head, [4], _cols(), activation_fn=torch.tanh)
    with pytest.raises(ValueError, match="batch_norm"):
        est.DNNEstimator(head, [4], _cols(), batch_norm=True)
    with pytest.raises(ValueError, match="warm_start_from"):
        est.DNNEstimator(head, [4], _cols(), warm_start_from="/tmp/ckpt")
    with pytest.raises(ValueError, match="warm_start_from"):
        est.LinearEstimator(head, _cols(), warm_start_from="/tmp/ckpt")
    with pytest.raises(ValueError, match="dnn_activation_fn"):
        est.DNNLinearCombinedEstimator(head, dnn_feature_columns=_cols(), dnn_hidden_units=[4],
                                       dnn_activation_fn=F.sigmoid)
    with pytest.raises(ValueError, match="batch_norm"):
        est.DNNLinearCombinedEstimator(head, dnn_feature_columns=_cols(), dnn_hidden_units=[4], batch_norm=True)
    with pytest.raises(ValueError, match="combiner"):
        est.LinearEstimator(head, _cols(), sparse_combiner="max")
    for act in (F.relu, torch.relu, "relu"):
        est.DNNEstimator(head, [4], _cols(), activation_fn=act)


def test_estimators_get_tf_default_learning_rates():
    head = est.PoissonRegressionHead()
    lin = est.LinearEstimator(head, _cols())
    dnn = est.DNNEstimator(head, [4], _cols())
    comb = est.DNNLinearCombinedEstimator(head, linear_feature_columns=_cols(), dnn_feature_columns=_cols(),
                                          dnn_hidden_units=[4])
    feats, y = {"x": torch.randn(4, 3)}, torch.ones(4)
    for e, want in ((lin, (keras.optimizers.Ftrl, 0.2)), (dnn, (keras.optimizers.Adagrad, 0.05))):
        spec = e._model_fn(feats, y, est.ModeKeys.TRAIN)
        assert isinstance(spec.optimizer, want[0]) and spec.optimizer.learning_rate == pytest.approx(want[1])
    spec = comb._model_fn(feats, y, est.ModeKeys.TRAIN)
    assert isinstance(spec.optimizer, keras.optimizers.Adagrad) and spec.optimizer.learning_rate == pytest.approx(1e-3)
    lin_opt = spec.optimizers["linear."]
    assert isinstance(lin_opt, keras.optimizers.Ftrl) and lin_opt.learning_rate == pytest.approx(0.005)


# ------------------------------------------------------------------------- the six estimators and their twins
def _class_batches(n, B, n_classes, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = torch.randn(B, 3, generator=g)
        cat = torch.randint(0, 7, (B,), generator=g)
        logit = x @ torch.tensor([1.0, -2.0, 0.5]) + (cat.float() - 3) * 0.3
        if n_classes is None:
            y = logit.reshape(B, 1) + 0.1 * torch.randn(B, 1, generator=g)
        elif n_classes == 2:
            y = (logit > 0).long()
        else:
            y = torch.bucketize(logit, torch.tensor([-1.0, 1.0]))
        out.append(({"x": x, "cat": cat, "w": torch.rand(B, generator=g) * 2}, y))
    return out


def _twin_pairs(model_dir):
    """(original, twin) constructors: each classifier and regressor, and the head-taking estimator with the equivalent
    head."""
    cat = fc.categorical_column_with_identity("cat", 7)
    lin_cols = [cat, fc.numeric_column("x", (3,))]
    dnn_cols = [fc.embedding_column(cat, 4), fc.numeric_column("x", (3,))]
    cfg = est.RunConfig(tf_random_seed=0, log_step_count_steps=None, save_checkpoints_steps=100)
    pairs = {}
    for kind, n_classes in (("binary", 2), ("multiclass", 3), ("regressor", None)):
        if n_classes is None:
            head = lambda: est.RegressionHead(weight_column="w")  # noqa: E731
            lin, dnn, comb = est.LinearRegressor, est.DNNRegressor, est.DNNLinearCombinedRegressor
            extra = {}
        else:
            head = (lambda: est.BinaryClassHead(weight_column="w")) if n_classes == 2 else \
                (lambda n=n_classes: est.MultiClassHead(n, weight_column="w"))
            lin, dnn, comb = est.LinearClassifier, est.DNNClassifier, est.DNNLinearCombinedClassifier
            extra = {"n_classes": n_classes}

        def d(name, kind=kind):
            return os.path.join(model_dir, kind, name)
        pairs[(kind, "linear")] = (
            lambda lin=lin, extra=extra, d=d: lin(lin_cols, model_dir=d("a"), weight_column="w", config=cfg, **extra),
            lambda head=head, d=d: est.LinearEstimator(head(), lin_cols, model_dir=d("b"), config=cfg))
        pairs[(kind, "dnn")] = (
            lambda dnn=dnn, extra=extra, d=d: dnn([8], dnn_cols, model_dir=d("c"), weight_column="w", config=cfg,
                                                  **extra),
            lambda head=head, d=d: est.DNNEstimator(head(), [8], dnn_cols, model_dir=d("d"), config=cfg))
        pairs[(kind, "combined")] = (
            lambda comb=comb, extra=extra, d=d: comb(model_dir=d("e"), linear_feature_columns=lin_cols,
                                                     dnn_feature_columns=dnn_cols, dnn_hidden_units=[8],
                                                     weight_column="w", config=cfg, **extra),
            lambda head=head, d=d: est.DNNLinearCombinedEstimator(head(), model_dir=d("f"),
                                                                  linear_feature_columns=lin_cols,
                                                                  dnn_feature_columns=dnn_cols, dnn_hidden_units=[8],
                                                                  config=cfg))
    return pairs


@pytest.mark.parametrize("tower", ["linear", "dnn", "combined"])
@pytest.mark.parametrize("kind", ["binary", "multiclass", "regressor"])
def test_each_canned_estimator_equals_its_head_twin(tmp_path, kind, tower):
    """Same seed, TF's default optimizers: bit-identical parameters after a few steps, identical evaluate() dicts
    and predictions."""
    original, twin = _twin_pairs(str(tmp_path))[(kind, tower)]
    batches = _class_batches(6, 32, {"binary": 2, "multiclass": 3, "regressor": None}[kind], seed=1)
    nets, results, preds = [], [], []
    for make in (original, twin):
        e = make()
        torch.manual_seed(0)
        e.train(lambda: iter(batches), max_steps=5)
        nets.append({n: p.detach().clone() for n, p in e._network.named_parameters()})
        results.append(e.evaluate(lambda: iter(batches)))
        preds.append(list(e.predict(lambda: iter([f for f, _ in batches[:1]]))))
    assert nets[0].keys() == nets[1].keys()
    for n in nets[0]:
        assert torch.equal(nets[0][n], nets[1][n]), n
    assert results[0] == results[1]
    assert len(preds[0]) == len(preds[1]) == 32
    for a, b in zip(preds[0], preds[1]):
        assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


# ------------------------------------------------------------------------------------ the new heads end to end
def _kind_batches(kind, n, B, seed, C=3):
    """Features x (3 numbers) and cat (7 ids); labels of the head that depend on them; weights w in [0, 2)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    proj = torch.tensor([[1.0, -1.0, 0.5], [-2.0, 0.5, 1.0], [0.5, 1.5, -1.0]])[:, :C]
    for _ in range(n):
        x = torch.randn(B, 3, generator=g)
        cat = torch.randint(0, 7, (B,), generator=g)
        s = x @ proj + (cat.float() - 3).reshape(B, 1) * 0.3
        if kind == "multi_label":
            y = (torch.rand(B, C, generator=g) < torch.sigmoid(2 * s)).long()
        elif kind == "poisson":
            y = torch.poisson(torch.exp(0.5 * s[:, 0]), generator=g)
        else:
            y = torch.sigmoid(s[:, 0])
        out.append(({"x": x, "cat": cat, "w": torch.rand(B, generator=g) * 2}, y))
    return out


def _kind_estimator(kind, model_dir, tower="combined", weight_column="w"):
    head = {"multi_label": lambda: est.MultiLabelHead(3, weight_column=weight_column, thresholds=[0.3, 0.5],
                                                      classes_for_class_based_metrics=[0, 2]),
            "poisson": lambda: est.PoissonRegressionHead(weight_column=weight_column),
            "logistic": lambda: est.LogisticRegressionHead(weight_column=weight_column)}[kind]()
    cat = fc.categorical_column_with_identity("cat", 7)
    cfg = est.RunConfig(tf_random_seed=0, log_step_count_steps=None, save_checkpoints_steps=20)
    if tower == "linear":
        return est.LinearEstimator(head, [cat, fc.numeric_column("x", (3,))], model_dir=model_dir, config=cfg,
                                   optimizer=lambda: keras.optimizers.SGD(0.1))
    if tower == "dnn":
        return est.DNNEstimator(head, [16], [fc.embedding_column(cat, 4), fc.numeric_column("x", (3,))],
                                model_dir=model_dir, config=cfg, optimizer=lambda: keras.optimizers.Adam(0.02))
    return est.DNNLinearCombinedEstimator(
        head, model_dir=model_dir, linear_feature_columns=[cat, fc.numeric_column("x", (3,))],
        dnn_feature_columns=[fc.embedding_column(cat, 4), fc.numeric_column("x", (3,))], dnn_hidden_units=[16],
        linear_optimizer=lambda: keras.optimizers.SGD(0.1), dnn_optimizer=lambda: keras.optimizers.Adam(0.02),
        config=cfg)


EXPECTED_KEYS = {
    "multi_label": {"loss", "average_loss", "auc", "auc_precision_recall", "global_step"}
    | {f"{m}/positive_threshold_{t}" for m in ("accuracy", "precision", "recall") for t in ("0.3", "0.5")}
    | {f"{m}/class{k}" for m in ("probability_mean", "auc", "auc_precision_recall") for k in (0, 2)},
    "poisson": {"loss", "average_loss", "label/mean", "prediction/mean", "global_step"},
    "logistic": {"loss", "average_loss", "label/mean", "prediction/mean", "global_step"},
}


@pytest.mark.parametrize("tower", ["linear", "dnn", "combined"])
@pytest.mark.parametrize("kind", ["multi_label", "poisson", "logistic"])
def test_new_head_trains_evaluates_predicts_exports_and_resumes(tmp_path, kind, tower):
    train = _kind_batches(kind, 40, 64, seed=1)
    evalb = _kind_batches(kind, 3, 128, seed=2)
    e = _kind_estimator(kind, str(tmp_path / "m"), tower)
    before = e.evaluate(lambda: iter(evalb))
    e.train(lambda: iter(train), max_steps=40)
    res = e.evaluate(lambda: iter(evalb))
    assert set(res) == EXPECTED_KEYS[kind] and res["global_step"] == 40
    assert res["average_loss"] < before["average_loss"], (before, res)      # it learned
    if kind == "multi_label":
        assert res["auc"] > 0.75, res
    preds = list(e.predict(lambda: iter([f for f, _ in evalb[:1]])))
    assert len(preds) == 128
    p = preds[0]
    if kind == "multi_label":
        assert set(p) == {"logits", "probabilities"} and p["probabilities"].shape == (3,)
        np.testing.assert_allclose(p["probabilities"], 1 / (1 + np.exp(-p["logits"].astype(np.float64))), rtol=1e-6)
    else:
        assert set(p) == {"logits", "predictions"} and p["predictions"].shape == (1,)
        link = np.exp if kind == "poisson" else (lambda v: 1 / (1 + np.exp(-v)))
        np.testing.assert_allclose(p["predictions"], link(p["logits"].astype(np.float64)), rtol=1e-6)
    path = e.export_saved_model(str(tmp_path / "export"))
    assert os.path.exists(os.path.join(path, "saved_model.pt"))
    again = _kind_estimator(kind, str(tmp_path / "m"), tower)
    assert again.evaluate(lambda: iter(evalb)) == res                    # restored from the checkpoint
    again.train(lambda: iter(train), max_steps=50)
    assert again.get_global_step() == 50


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", ["multi_label", "poisson", "logistic"])
def test_evaluate_matches_the_reference(tmp_path, kind, weighted):
    batches = _kind_batches(kind, 3, 50, seed=7)
    if weighted:
        batches[0][0]["w"][:5] = 0.0
    e = _kind_estimator(kind, str(tmp_path), "dnn", weight_column="w" if weighted else None)
    res = e.evaluate(lambda: iter(batches))
    with torch.no_grad():
        zs = [e._network(f).double().numpy() for f, _ in batches]
    z = np.concatenate(zs)
    y = torch.cat([yb for _, yb in batches]).double().numpy()
    w = torch.cat([f["w"] for f, _ in batches]).double().numpy() if weighted else None
    code = {"multi_label": ref.MULTI_LABEL, "poisson": ref.POISSON_FULL, "logistic": ref.LOGISTIC}[kind]
    if kind == "multi_label":
        want = ref.multi_label_metrics(z, y, w, thresholds=(0.3, 0.5), classes=(0, 2))
    else:
        want = ref.regression_metrics(code, z, y, w)
    assert set(want) | {"loss", "global_step"} == set(res)
    for k, v in want.items():
        assert res[k] == pytest.approx(v, rel=1e-5, abs=1e-6), k
    losses = [ref.loss(code, zb, yb.double().numpy(), f["w"].double().numpy() if weighted else None)
              for zb, (f, yb) in zip(zs, batches)]
    assert res["loss"] == pytest.approx(np.mean(losses), rel=1e-5, abs=1e-9)


def test_binary_head_thresholds_add_metrics(tmp_path):
    batches = _class_batches(3, 40, 2, seed=4)
    plain = est.DNNEstimator(est.BinaryClassHead(weight_column="w"), [8], _cols(), model_dir=str(tmp_path / "a"),
                             config=est.RunConfig(tf_random_seed=0))
    thr = est.DNNEstimator(est.BinaryClassHead(weight_column="w", thresholds=[0.25, 0.5]), [8], _cols(),
                           model_dir=str(tmp_path / "b"), config=est.RunConfig(tf_random_seed=0))
    a, b = plain.evaluate(lambda: iter(batches)), thr.evaluate(lambda: iter(batches))
    extra = {f"{m}/positive_threshold_{t}" for m in ("accuracy", "precision", "recall") for t in ("0.25", "0.5")}
    assert set(b) == set(a) | extra
    assert all(a[k] == b[k] for k in a)
    assert b["precision/positive_threshold_0.5"] == a["precision"] and b["recall/positive_threshold_0.5"] == a["recall"]
    with torch.no_grad():
        z = torch.cat([thr._network(f) for f, _ in batches]).double().numpy().reshape(-1)
    y = torch.cat([yb for _, yb in batches]).double().numpy()
    w = torch.cat([f["w"] for f, _ in batches]).double().numpy()
    p = 1 / (1 + np.exp(-z))
    for t in (0.25, 0.5):
        assert b[f"accuracy/positive_threshold_{t:g}"] == pytest.approx((w * ((p > t) == y)).sum() / w.sum(), rel=1e-6)


def test_invalid_labels_raise_in_train_and_evaluate_on_the_cpu(tmp_path):
    for kind, bad in (("poisson", -1.0), ("logistic", 1.5)):
        batches = _kind_batches(kind, 3, 16, seed=3)
        batches[1][1][4] = bad
        e = _kind_estimator(kind, str(tmp_path / kind), "linear")
        rule = "labels must be counts >= 0" if kind == "poisson" else "labels must be in \\[0, 1\\]"
        with pytest.raises(ValueError, match=rule):
            e.train(lambda: iter(batches), steps=3)
        with pytest.raises(ValueError, match=rule):
            e.evaluate(lambda: iter(batches))


# ------------------------------------------------------------------------- multi-process, shared-memory ps plane
def _ps_experiment(model_dir):
    def experiment_fn():
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200 import keras
        from tf_yarn_b200.estimator import feature_column as fc
        from tf_yarn_b200.tensorflow import Experiment
        g = torch.Generator().manual_seed(0)
        n = 4096
        x = torch.randn(n, 3, generator=g)
        cat = torch.randint(0, 10, (n,), generator=g)
        s = x @ torch.tensor([[1.0, -1.0, 0.5], [-2.0, 0.5, 1.0], [0.5, 1.5, -1.0]]) + \
            (cat.float() - 4.5).reshape(n, 1) * 0.5
        y = (torch.rand(n, 3, generator=g) < torch.sigmoid(3 * s)).long()
        w = torch.rand(n, generator=g) * 2
        feats = {"x": x, "cat": cat, "w": w}
        train = lambda: data.Dataset.from_tensor_slices((feats, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa
        evalf = lambda: data.Dataset.from_tensor_slices((feats, y)).batch(1024)  # noqa: E731
        cat_col = fc.categorical_column_with_identity("cat", 10)
        e = est.DNNLinearCombinedEstimator(
            est.MultiLabelHead(3, weight_column="w"), model_dir=model_dir,
            linear_feature_columns=[cat_col, fc.numeric_column("x", (3,))],
            dnn_feature_columns=[fc.embedding_column(cat_col, 4), fc.numeric_column("x", (3,))],
            dnn_hidden_units=[16], linear_optimizer=lambda: keras.optimizers.SGD(0.05),
            dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1),
            config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=600),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_trains_a_multi_label_wide_and_deep_estimator(tmp_path):
    """chief + 2 workers + 2 ps + evaluator: the weighted multi-label head learns its three labels."""
    import sys

    import cloudpickle

    from tf_yarn_b200.estimator import summary
    from tf_yarn_b200.tensorflow import TaskSpec, run_on_yarn
    cloudpickle.register_pickle_by_value(sys.modules[__name__])
    model_dir = str(tmp_path / "model")
    run_on_yarn(_ps_experiment(model_dir),
                {"chief": TaskSpec("1 GiB", 1), "worker": TaskSpec("1 GiB", 1, instances=2),
                 "ps": TaskSpec("1 GiB", 1, instances=2), "evaluator": TaskSpec("1 GiB", 1)})
    sc = summary.read_scalars(os.path.join(model_dir, "eval"))
    auc = [v for n, v in zip(sc["name"], sc["value"]) if n == "auc"]
    avg = [v for n, v in zip(sc["name"], sc["value"]) if n == "average_loss"]
    assert auc and auc[-1] > 0.85, auc
    assert avg and avg[-1] < 0.45, avg
