"""The canned regressors and weight_column on the CPU: construction errors; the head's torch statement and the host build
of its kernel math (ops/csrc/tfy_head.cuh) against the float64 reference (tests/canned_head_reference.py); unweighted
losses and metrics bit-equal to the formulas the classifiers used before weighting existed; train / evaluate /
predict / export / resume of the three regressors; weighted training and evaluation against the reference; and a
multi-process run on the shared-memory parameter-server plane."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import canned_head_reference as ref
from tf_yarn_b200 import data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.estimator import canned
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import head as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"


# ------------------------------------------------------------------------------------------------- inputs
def head_inputs(head, B, C, seed, zmax=8.0, weighted=True, label_dtype=torch.int64, bad=False):
    """Random logits (a few at +-80), labels of the head, and weights with zeros and negatives."""
    g = np.random.default_rng(seed)
    z = (g.standard_normal((B, C)) * zmax / 3).astype(np.float32)
    z.reshape(-1)[g.random(B * C) < 0.05] = 80.0
    z.reshape(-1)[g.random(B * C) < 0.05] = -80.0
    if head == ref.BINARY:
        y = (g.random(B) < 0.5).astype(np.float64)
        if label_dtype == torch.float32:
            y[g.random(B) < 0.3] = 0.25            # soft labels are used as given
    elif head == ref.MULTI_CLASS:
        y = g.integers(0, C, B).astype(np.float64)
        if bad and B > 2:
            y[1], y[B - 1] = C, -1
    else:
        y = g.standard_normal((B, C)) * 3
    w = None
    if weighted:
        w = g.choice([0.0, -0.5, 0.25, 1.0, 1.5, 3.0], B).astype(np.float32)
    zt = torch.from_numpy(z)
    yt = torch.from_numpy(y).to(label_dtype)
    if head == ref.REGRESSION and C == 1:
        yt = yt.reshape(B)
    wt = None if w is None else torch.from_numpy(w)
    return zt, yt, wt


def _np(t):
    return None if t is None else t.double().numpy()


# --------------------------------------------------------------------------------------------- construction
def _cols():
    return [fc.numeric_column("x", (3,))]


@pytest.mark.parametrize("bad", [0, -1, 1.5, True, "2"])
def test_bad_label_dimension(bad):
    for cls in (est.LinearRegressor, est.DNNRegressor):
        args = ([8],) if cls is est.DNNRegressor else ()
        with pytest.raises(ValueError, match="label_dimension"):
            cls(*args, _cols(), label_dimension=bad)
    with pytest.raises(ValueError, match="label_dimension"):
        est.DNNLinearCombinedRegressor(linear_feature_columns=_cols(), label_dimension=bad)


@pytest.mark.parametrize("reduction", ["sum", "none", "sum_by_nonzero_weights", None])
def test_only_sum_over_batch_size_is_accepted(reduction):
    assert est.SUM_OVER_BATCH_SIZE == "sum_over_batch_size"
    for make in (lambda r: est.LinearRegressor(_cols(), loss_reduction=r),
                 lambda r: est.DNNRegressor([4], _cols(), loss_reduction=r),
                 lambda r: est.DNNLinearCombinedRegressor(dnn_feature_columns=_cols(), dnn_hidden_units=[4],
                                                          loss_reduction=r)):
        make(est.SUM_OVER_BATCH_SIZE)
        with pytest.raises(ValueError, match="loss_reduction"):
            make(reduction)


def _batches(n, B, d=1, seed=0, w_shape=None, weight_key="w"):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = torch.randn(B, 3, generator=g)
        y = (x @ torch.tensor([[1.0], [-2.0], [0.5]])).repeat(1, d) + 0.1 * torch.arange(d)
        feats = {"x": x, weight_key: torch.rand(B if w_shape is None else w_shape, generator=g) * 2}
        out.append((feats, y.reshape(B) if d == 1 else y))
    return out


def _input(batches):
    return lambda: iter(batches)


def test_weight_shape_missing_key_and_label_shape_errors(tmp_path):
    e = est.LinearRegressor(_cols(), model_dir=str(tmp_path / "a"), weight_column="w")
    with pytest.raises(ValueError, match=r"\[B\] or \[B, 1\]"):
        e.train(_input(_batches(1, 8, w_shape=(8, 2))), steps=1)
    e = est.LinearRegressor(_cols(), model_dir=str(tmp_path / "b"), weight_column="weight_of_example")
    with pytest.raises(KeyError, match="weight_of_example"):
        e.train(_input(_batches(1, 8)), steps=1)
    e = est.DNNRegressor([4], _cols(), model_dir=str(tmp_path / "c"), label_dimension=3)
    bad = [(f, y[:, :2]) for f, y in _batches(1, 8, d=3)]
    with pytest.raises(ValueError, match="regression labels"):
        e.train(_input(bad), steps=1)
    e = est.DNNRegressor([4], _cols(), model_dir=str(tmp_path / "d"))
    with pytest.raises(ValueError, match="regression labels"):
        e.train(_input([(f, y.reshape(8, 1, 1)) for f, y in _batches(1, 8)]), steps=1)
    with pytest.raises(TypeError, match="weight_column"):
        est.DNNRegressor([4], _cols(), weight_column=3)
    # [B, 1] weights are accepted
    e = est.LinearRegressor(_cols(), model_dir=str(tmp_path / "e"), weight_column="w")
    e.train(_input(_batches(1, 8, w_shape=(8, 1))), steps=1)


# ------------------------------------------------------------------------- the torch statement vs the reference
CASES = [(ref.BINARY, 1, B) for B in (1, 7, 300)] + [(ref.MULTI_CLASS, C, B) for C in (2, 3, 10, 1000) for B in (1, 64)] \
    + [(ref.REGRESSION, d, B) for d in (1, 3) for B in (1, 7, 300)]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("head,C,B", CASES)
def test_torch_statement_matches_the_reference(head, C, B, weighted):
    z, y, w = head_inputs(head, B, C, seed=B * 31 + C, weighted=weighted,
                          label_dtype=torch.float32 if head != ref.MULTI_CLASS else torch.int64)
    zr = z.clone().requires_grad_(True)
    loss = H.CannedHead(head, C)(y, zr if head != ref.BINARY else zr.reshape(B, 1), w)
    loss.backward()
    assert abs(loss.item() - ref.loss(head, z, y, _np(w))) <= ref.loss_tol(head, z, y, _np(w))
    np.testing.assert_array_less(np.abs(zr.grad.double().numpy() - ref.dlogits(head, z, y, _np(w))),
                                 ref.grad_tol(head, z, y, _np(w)) + 1e-45)


def test_zero_weight_rows_change_nothing():
    for head, C in ((ref.BINARY, 1), (ref.MULTI_CLASS, 5), (ref.REGRESSION, 3)):
        z, y, w = head_inputs(head, 40, C, seed=C)
        w[:10] = 0.0
        z2 = z.clone()
        z2[:10] = torch.randn(10, C) * 50             # whatever the zero-weight rows hold
        a = z.clone().requires_grad_(True)
        b = z2.clone().requires_grad_(True)
        la, lb = H.CannedHead(head, C)(y, a, w), H.CannedHead(head, C)(y, b, w)
        la.backward()
        lb.backward()
        assert la.item() == pytest.approx(lb.item(), rel=1e-6)
        assert torch.equal(a.grad[10:], b.grad[10:]) and not b.grad[:10].any()


# ------------------------------------------------------------------------------------ the kernel's math, host-built
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    out = str(tmp_path_factory.mktemp("head") / "libhead.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-Wl,-Bsymbolic", "-include",
           os.path.join(ROOT, "tests", "native", "cuda_device_shim.h"), "-I", CUDA_INC, "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "head_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.tfy_host_head_elementwise.argtypes = [i, vp, vp, i, vp, vp]
    lib.tfy_host_head_multi.argtypes = [vp, vp, i, i, vp, vp]
    lib.tfy_host_head_class_of_f32.argtypes = [vp, i, i, vp]
    for f in (lib.tfy_host_head_elementwise, lib.tfy_host_head_multi, lib.tfy_host_head_class_of_f32):
        f.restype = None
    return lib


def _host(lib, head, z, y):
    z = np.ascontiguousarray(z.numpy(), dtype=np.float32)
    B, C = z.shape
    loss = np.zeros(B if head == ref.MULTI_CLASS else B * C, np.float32)
    grad = np.zeros(B * C, np.float32)
    if head == ref.MULTI_CLASS:
        yy = np.ascontiguousarray(y.numpy().astype(np.int64))
        lib.tfy_host_head_multi(z.ctypes.data, yy.ctypes.data, B, C, loss.ctypes.data, grad.ctypes.data)
    else:
        yy = np.ascontiguousarray(y.numpy().astype(np.float32).reshape(-1))
        lib.tfy_host_head_elementwise(head, z.ctypes.data, yy.ctypes.data, B * C, loss.ctypes.data, grad.ctypes.data)
    return loss.astype(np.float64).reshape(B, -1).sum(axis=1), grad.astype(np.float64).reshape(B, C)


@pytest.mark.parametrize("head,C,B", CASES + [(ref.MULTI_CLASS, 7, 50)])
def test_host_built_head_math_matches_the_reference(host_lib, head, C, B):
    z, y, _ = head_inputs(head, B, C, seed=B + 7 * C, label_dtype=torch.float32 if head != ref.MULTI_CLASS else
                          torch.int64, bad=True)
    rows, grad = _host(host_lib, head, z, y)
    want_rows = ref.row_losses(head, z, y)
    tol_rows = 8 * ref.EPS32 * ref._element_scale(head, z.double().numpy(), y.double().numpy())
    np.testing.assert_array_less(np.abs(rows - want_rows), tol_rows)
    per = B if head == ref.MULTI_CLASS else B * C
    np.testing.assert_array_less(np.abs(grad - ref.element_grads(head, z, y)), ref.grad_tol(head, z, y) * per)
    if head == ref.MULTI_CLASS and B > 2:
        assert rows[1] == 0 and rows[B - 1] == 0 and not grad[1].any()


def test_host_built_float_label_to_class(host_lib):
    v = np.array([0.0, 0.9, 2.0, 2.99, 3.0, -0.5, -1.0, np.nan, np.inf, -np.inf, 1e30], np.float32)
    out = np.zeros(v.size, np.int32)
    host_lib.tfy_host_head_class_of_f32(v.ctypes.data, v.size, 3, out.ctypes.data)
    assert out.tolist() == [0, 0, 2, 2, -1, 0, -1, -1, -1, -1, -1]
    ok = ref.valid_rows(ref.MULTI_CLASS, v, 3)
    assert (out >= 0).tolist() == ok.tolist()


# ------------------------------------------------------------------------- unweighted: bit-equal to the old formulas
def _old_loss(n_classes):
    if n_classes == 2:
        return lambda y, z: F.binary_cross_entropy_with_logits(z.float().reshape(-1), y.float().reshape(-1))
    return lambda y, z: F.cross_entropy(z.float(), y.long().reshape(-1))


def _old_metrics(n_classes, batches):
    """evaluate()'s (numerator, denominator) accumulation of the classifiers' metrics before this head existed."""
    num, den = {}, {}

    def add(k, a, b):
        num[k] = num.get(k, 0.0) + float(a)
        den[k] = den.get(k, 0.0) + float(b)
    ys = []
    for y, z in batches:
        pred = (z.reshape(-1) > 0).long() if n_classes == 2 else z.argmax(dim=-1)
        lab = y.long().reshape(-1)
        add("accuracy", (pred == lab).sum().float(), float(lab.numel()))
        n = y.reshape(-1).shape[0]
        add("average_loss", _old_loss(n_classes)(y, z) * n, float(n))
        if n_classes == 2:
            yf = y.float().reshape(-1)
            add("label/mean", yf.sum(), float(yf.numel()))
            p = torch.sigmoid(z.float().reshape(-1))
            add("prediction/mean", p.sum(), float(p.numel()))
            ys.append(y.detach().reshape(-1).double())
    out = {k: num[k] / max(den[k], 1.0) for k in num}
    if n_classes == 2:
        s = torch.zeros(2, dtype=torch.float64)
        for y in ys:
            s[0] += y.sum()
            s[1] += y.numel()
        m = s[0].item() / s[1].item()
        out["accuracy_baseline"] = max(m, 1 - m)
    return out


@pytest.mark.parametrize("n_classes", [2, 3, 10])
def test_unweighted_cpu_loss_and_metrics_are_bit_equal_to_the_old_formulas(n_classes):
    head = ref.BINARY if n_classes == 2 else ref.MULTI_CLASS
    C = 1 if n_classes == 2 else n_classes
    batches = []
    for s in range(5):
        z, y, _ = head_inputs(head, 33 + s, C, seed=s, weighted=False)
        batches.append((y, z))
        got = canned._classification_head(n_classes)(y, z)
        assert torch.equal(got, _old_loss(n_classes)(y, z))
    ops = canned._classification_metrics(n_classes)
    for k, m in ops.items():
        if isinstance(m, keras.metrics.Metric):
            m.reset_state()
            for y, z in batches:
                m.update_state(y, z)
    old = _old_metrics(n_classes, batches)
    for k, v in old.items():
        assert ops[k].result() == v, k                 # exactly: same statements, same fp64 order


def test_unweighted_regression_loss_is_mse_mean():
    for d in (1, 3):
        z, y, _ = head_inputs(ref.REGRESSION, 17, d, seed=d, weighted=False, label_dtype=torch.float32)
        assert torch.equal(H.CannedHead(H.REGRESSION, d)(y, z), F.mse_loss(z, y.reshape(z.shape)))


# --------------------------------------------------------------------------------- the three regressors end to end
def _regressors(model_dir, d, weight_column=None):
    cols = _cols()
    cfg = est.RunConfig(save_checkpoints_steps=20, log_step_count_steps=None, tf_random_seed=0)
    return {
        "linear": lambda: est.LinearRegressor(cols, model_dir=model_dir + "/linear", label_dimension=d,
                                              weight_column=weight_column, config=cfg,
                                              optimizer=lambda: keras.optimizers.SGD(0.05)),
        "dnn": lambda: est.DNNRegressor([16], cols, model_dir=model_dir + "/dnn", label_dimension=d,
                                        weight_column=weight_column, config=cfg,
                                        optimizer=lambda: keras.optimizers.Adam(0.02)),
        "combined": lambda: est.DNNLinearCombinedRegressor(
            model_dir=model_dir + "/combined", linear_feature_columns=cols, dnn_feature_columns=cols,
            dnn_hidden_units=[16], label_dimension=d, weight_column=weight_column, config=cfg,
            linear_optimizer=lambda: keras.optimizers.SGD(0.05), dnn_optimizer=lambda: keras.optimizers.Adam(0.02)),
    }


@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("kind", ["linear", "dnn", "combined"])
def test_regressor_trains_evaluates_predicts_exports_and_resumes(tmp_path, kind, d):
    make = _regressors(str(tmp_path), d, weight_column="w")[kind]
    train = _batches(60, 32, d=d, seed=1)
    evalb = _batches(4, 64, d=d, seed=2)
    e = make()
    e.train(_input(train), max_steps=60)
    res = e.evaluate(_input(evalb))
    assert set(res) == {"loss", "average_loss", "label/mean", "prediction/mean", "global_step"}
    assert res["global_step"] == 60
    # label variance is ~5.25: a fitted linear relation is far below it
    assert res["average_loss"] < 1.0, res
    preds = list(e.predict(lambda: iter([f for f, _ in evalb[:1]])))
    assert len(preds) == 64 and set(preds[0]) == {"predictions"} and preds[0]["predictions"].shape == (d,)
    path = e.export_saved_model(str(tmp_path / "export" / kind))
    assert os.path.exists(os.path.join(path, "saved_model.pt"))
    again = make()
    assert again.evaluate(_input(evalb)) == res            # restored from the checkpoint: the same metrics
    again.train(_input(train), max_steps=80)
    assert again.get_global_step() == 80


# ------------------------------------------------------------------------- weighted training and evaluation
@pytest.mark.parametrize("kind", ["classifier", "regressor", "multiclass"])
def test_weighted_step_gradients_match_the_reference(tmp_path, kind):
    """One SGD step with learning rate 1 on a linear model: the weight change is -X^T dL/dz, dL/dz from the
    reference."""
    B, d = 24, 3
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 4, generator=g)
    w = torch.tensor([0.0, -0.5, 0.25, 1.0, 2.0, 0.125] * 4)
    if kind == "classifier":
        y, n_out, head = (torch.rand(B, generator=g) < 0.5).long(), 1, ref.BINARY
        e = est.LinearClassifier([fc.numeric_column("x", (4,))], model_dir=str(tmp_path), weight_column="w",
                                 optimizer=lambda: keras.optimizers.SGD(1.0))
    elif kind == "multiclass":
        y, n_out, head = torch.randint(0, 5, (B,), generator=g), 5, ref.MULTI_CLASS
        e = est.LinearClassifier([fc.numeric_column("x", (4,))], model_dir=str(tmp_path), weight_column="w",
                                 n_classes=5, optimizer=lambda: keras.optimizers.SGD(1.0))
    else:
        y, n_out, head = torch.randn(B, d, generator=g), d, ref.REGRESSION
        e = est.LinearRegressor([fc.numeric_column("x", (4,))], model_dir=str(tmp_path), weight_column="w",
                                label_dimension=d, optimizer=lambda: keras.optimizers.SGD(1.0))
    feats = {"x": x, "w": w}
    spec = e._build(feats, y, est.ModeKeys.TRAIN)
    lin = e._network.linear
    params0 = {n: p.detach().clone() for n, p in e._network.named_parameters()}
    z = e._network(feats).detach()
    e.train(_input([(feats, y)]), steps=1)
    dz = ref.dlogits(head, z.numpy(), y.numpy(), w.numpy())          # [B, n_out]
    xd = x.double().numpy()
    for n, p in e._network.named_parameters():
        delta = (p.detach().double() - params0[n].double()).numpy()
        if n.endswith("bias"):
            want = -dz.sum(axis=0)
        else:
            want = -(xd.T @ dz).T.reshape(delta.shape)
        np.testing.assert_allclose(delta, want, rtol=1e-4, atol=1e-6, err_msg=n)
    assert spec.weights is not None and lin is not None and n_out == z.shape[1]


@pytest.mark.parametrize("kind", ["classifier", "regressor"])
def test_zero_weight_examples_change_nothing_in_training(tmp_path, kind):
    """Examples of weight 0 whose features and labels are replaced by anything train the network to the same bits."""
    base = _batches(10, 16, seed=3)
    if kind == "classifier":
        base = [(f, (y > 0).long()) for f, y in base]
    changed = []
    for f, y in base:
        f2, y2 = {k: v.clone() for k, v in f.items()}, y.clone()
        f2["w"][:5] = 0.0
        f2["x"][:5] = torch.randn(5, 3) * 100
        y2[:5] = 1 - y2[:5] if kind == "classifier" else torch.randn(5) * 100
        changed.append((f2, y2))
    base = [({"x": f["x"], "w": c["w"]}, y) for (f, y), (c, _) in zip(base, changed)]
    nets = []
    for name, batches in (("a", base), ("b", changed)):
        cfg = est.RunConfig(tf_random_seed=0, log_step_count_steps=None)
        if kind == "classifier":
            e = est.DNNClassifier([8], _cols(), model_dir=str(tmp_path / name), weight_column="w",
                                  optimizer=lambda: keras.optimizers.SGD(0.05), config=cfg)
        else:
            e = est.DNNRegressor([8], _cols(), model_dir=str(tmp_path / name), weight_column="w",
                                 optimizer=lambda: keras.optimizers.SGD(0.05), config=cfg)
        torch.manual_seed(0)
        e.train(_input(batches), max_steps=10)
        nets.append({n: p.detach() for n, p in e._network.named_parameters()})
    for n in nets[0]:
        assert torch.equal(nets[0][n], nets[1][n]), n


@pytest.mark.parametrize("kind", ["binary", "multiclass", "regressor"])
@pytest.mark.parametrize("scale", [1.0, 0.01])
def test_weighted_evaluate_matches_the_reference(tmp_path, kind, scale):
    """scale 0.01 puts sum(w) below 1: the metrics must divide by sum(w), not by max(sum(w), 1)."""
    g = torch.Generator().manual_seed(11)
    d = 3 if kind == "regressor" else 1
    batches = []
    for b in range(3):
        x = torch.randn(20, 3, generator=g)
        w = torch.rand(20, generator=g) * scale
        w[0] = 0.0
        if kind == "binary":
            y = (torch.rand(20, generator=g) < 0.4).long()
        elif kind == "multiclass":
            y = torch.randint(0, 4, (20,), generator=g)
        else:
            y = torch.randn(20, d, generator=g)
        batches.append(({"x": x, "w": w}, y))
    if kind == "regressor":
        e = est.DNNRegressor([8], _cols(), model_dir=str(tmp_path), weight_column=fc.numeric_column("w"),
                             label_dimension=d)
    else:
        e = est.DNNClassifier([8], _cols(), model_dir=str(tmp_path), weight_column=fc.numeric_column("w"),
                              n_classes=2 if kind == "binary" else 4)
    res = e.evaluate(_input(batches))
    with torch.no_grad():
        z = torch.cat([e._network(f) for f, _ in batches]).double().numpy()
    y = torch.cat([y for _, y in batches]).double().numpy()
    w = torch.cat([f["w"] for f, _ in batches]).double().numpy()
    if kind == "regressor":
        want = ref.regressor_metrics(z, y, w)
        head = ref.REGRESSION
    else:
        want = ref.classifier_metrics(2 if kind == "binary" else 4, z, y, w)
        head = ref.BINARY if kind == "binary" else ref.MULTI_CLASS
    for k, v in want.items():
        assert res[k] == pytest.approx(v, rel=1e-5, abs=1e-7), k
    losses = [ref.loss(head, e._network(f).detach().double().numpy(), yb.double().numpy(), f["w"].double().numpy())
              for f, yb in batches]
    assert res["loss"] == pytest.approx(np.mean(losses), rel=1e-5, abs=1e-9)
    if kind == "binary":
        assert {"auc", "auc_precision_recall", "precision", "recall"} <= set(res)


def test_weight_column_as_a_numeric_column_or_a_key_is_the_same(tmp_path):
    batches = _batches(5, 16, seed=4)
    res = []
    for i, wc in enumerate(("w", fc.numeric_column("w"))):
        e = est.LinearRegressor(_cols(), model_dir=str(tmp_path / str(i)), weight_column=wc,
                                optimizer=lambda: keras.optimizers.SGD(0.05),
                                config=est.RunConfig(tf_random_seed=0, log_step_count_steps=None))
        e.train(_input(batches), max_steps=5)
        res.append(e.evaluate(_input(batches)))
    assert res[0] == res[1]
    unweighted = est.LinearRegressor(_cols(), model_dir=str(tmp_path / "u"),
                                     optimizer=lambda: keras.optimizers.SGD(0.05),
                                     config=est.RunConfig(tf_random_seed=0, log_step_count_steps=None))
    unweighted.train(_input(batches), max_steps=5)
    assert unweighted.evaluate(_input(batches))["average_loss"] != res[0]["average_loss"]


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
        y = x @ torch.tensor([1.0, -2.0, 0.5]) + (cat.float() - 4.5) * 0.5
        w = torch.rand(n, generator=g) * 2
        feats = {"x": x, "cat": cat, "w": w}
        train = lambda: data.Dataset.from_tensor_slices((feats, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa
        evalf = lambda: data.Dataset.from_tensor_slices((feats, y)).batch(1024)  # noqa: E731
        cat_col = fc.categorical_column_with_identity("cat", 10)
        e = est.DNNLinearCombinedRegressor(
            model_dir=model_dir, linear_feature_columns=[cat_col, fc.numeric_column("x", (3,))],
            dnn_feature_columns=[fc.embedding_column(cat_col, 4), fc.numeric_column("x", (3,))],
            dnn_hidden_units=[16], weight_column="w", linear_optimizer=lambda: keras.optimizers.SGD(0.05),
            dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1),
            config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=600),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_trains_a_weighted_wide_and_deep_regressor(tmp_path):
    """chief + 2 workers + 2 ps + evaluator: the weighted regressor learns y (label variance ~7.3)."""
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
    avg = [v for n, v in zip(sc["name"], sc["value"]) if n == "average_loss"]
    assert avg and avg[-1] < 0.5, avg
