"""tfy_canned_head's multi-label, Poisson and logistic heads (codes 3-6) against the float64 reference
(tests/head_kinds_reference.py), their determinism and invalid-label flag; the estimator's ValueError for bad labels;
the HBM and CPU parameter-server planes training MultiLabelHead and PoissonRegressionHead alike; GPU evaluate().

Tolerances (head_kinds_reference.loss_tol / grad_tol), with EPS32 = 2^-23:
  * per element the kernel computes l and dl/dz in fp32 from accurately rounded expf / logf / log1pf (no fast math).
    Sigmoid heads: max(z,0) - z y + log1p(exp(-|z|)) rounds at most four times on values of size |z| (1 + |y|) + 1.
    Poisson: exp(z) (within 2 EPS32 exp(z)), y z and their difference round three times on exp(z) + |y z|; the full
    loss adds y log y - y + log(2 pi y) / 2, whose five roundings (the 2 pi constant, the product inside the log, two
    logs, the products and sums) stay within 8 EPS32 of y |log y| + y + |log(2 pi y)|.  So |l - exact| <= 8 EPS32 S_ij
    with S_ij of element_scale.
  * the batch sum is fp64 (exact enough to ignore); the final (float) rounding adds EPS32 |L|, inside the
    (log2(BC) + 4) EPS32 sum |w l| / (BC) term.
  * gradient: sigmoid(z) - y is off by 4 EPS32 (1 + |y|); exp(z) - y by 4 EPS32 (exp(z) + |y|); the product with
    w / (BC) adds two roundings of the result (4 EPS32 |g|).
A label, indexing or weighting fault is of the order of the values themselves, far above these bounds.

B = 100_003 with C = 1000 (10^8 logits) is left out: the float64 reference would need several GB of host memory.
"""
import numpy as np
import pytest
import torch

import head_kinds_reference as ref
from test_estimator_heads import _kind_batches, _kind_estimator, kinds_inputs
from tf_yarn_b200.ops import head as H

pytestmark = pytest.mark.gpu

BS = [1, 7, 512, 4096, 100_003]
SHAPES = [(ref.MULTI_LABEL, C) for C in (2, 10, 1000)] + \
    [(h, d) for h in (ref.POISSON, ref.POISSON_FULL) for d in (1, 2, 10, 1000)] + [(ref.LOGISTIC, 1)]
LABELS = [torch.int32, torch.int64, torch.float32]


def _cases():
    for head, C in SHAPES:
        for B in BS:
            if B * C > 20_000_000:
                continue
            yield head, C, B


def _run(head, C, z, y, w, with_grad=True):
    h = H.CannedHead(head, C)
    loss, grad = h._launch(z.cuda(), y.cuda(), None if w is None else w.cuda(), with_grad=with_grad)
    torch.cuda.synchronize()
    return h, loss, grad


@pytest.mark.parametrize("label_dtype", LABELS, ids=["i32", "i64", "f32"])
@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "weighted"])
@pytest.mark.parametrize("head,C,B", list(_cases()))
def test_kernel_matches_the_reference(head, C, B, weighted, label_dtype):
    z, y, w = kinds_inputs(head, B, C, seed=B + C + head, weighted=weighted, label_dtype=label_dtype)
    h, loss, grad = _run(head, C, z, y, w)
    wn = None if w is None else w.double().numpy()
    zn, yn = z.double().numpy(), y.double().numpy()
    assert abs(loss.item() - ref.loss(head, zn, yn, wn)) <= ref.loss_tol(head, zn, yn, wn)
    err = np.abs(grad.double().cpu().numpy().reshape(B, C) - ref.dlogits(head, zn, yn, wn))
    bound = ref.grad_tol(head, zn, yn, wn)
    assert (err <= bound).all(), (err.max(), np.unravel_index((err - bound).argmax(), err.shape))
    _, loss_only, none = _run(head, C, z, y, w, with_grad=False)          # dlogits = null: the same loss bits
    assert none is None and torch.equal(loss_only, loss)
    h.check()                                                             # no flag for valid labels


@pytest.mark.parametrize("head,C", SHAPES)
def test_two_runs_and_graph_replay_give_the_same_bits(head, C):
    B = 4096 if C < 1000 else 512
    z, y, w = kinds_inputs(head, B, C, seed=3)
    z, y, w = z.cuda(), y.cuda(), w.cuda()
    h = H.CannedHead(head, C)
    a = h._launch(z, y, w, with_grad=True)
    b = h._launch(z, y, w, with_grad=True)
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            cap = h._launch(z, y, w, with_grad=True)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(cap[0], a[0]) and torch.equal(cap[1], a[1])


@pytest.mark.parametrize("label_dtype", LABELS, ids=["i32", "i64", "f32"])
@pytest.mark.parametrize("head", [ref.POISSON, ref.POISSON_FULL, ref.LOGISTIC], ids=["poisson", "full", "logistic"])
def test_invalid_labels_are_skipped_and_flagged(head, label_dtype):
    B, C = 1029, 1 if head == ref.LOGISTIC else 3
    z, y, w = kinds_inputs(head, B, C, seed=1, label_dtype=label_dtype, bad=True)
    h, loss, grad = _run(head, C, z, y, w)
    zn, yn, wn = z.double().numpy(), y.double().numpy(), w.double().numpy()
    assert abs(loss.item() - ref.loss(head, zn, yn, wn)) <= ref.loss_tol(head, zn, yn, wn)
    bad = ~ref.valid(head, yn.reshape(B, C))
    assert bad.sum() == (3 if label_dtype == torch.float32 else 2)
    assert not grad.cpu().reshape(B, C).numpy()[bad].any()
    rule = "labels must be in \\[0, 1\\]" if head == ref.LOGISTIC else "labels must be counts >= 0"
    with pytest.raises(ValueError, match=rule):
        h.check()
    h.check()                                       # the flag was cleared with the error


def test_multi_label_has_no_invalid_labels():
    z, y, w = kinds_inputs(ref.MULTI_LABEL, 300, 5, seed=2)
    y[0, 0], y[1, 1] = 3.0, -2.0                    # used as the floats they are, as the binary head does
    h, loss, grad = _run(ref.MULTI_LABEL, 5, z, y, w)
    zn, yn, wn = z.double().numpy(), y.double().numpy(), w.double().numpy()
    assert abs(loss.item() - ref.loss(ref.MULTI_LABEL, zn, yn, wn)) <= ref.loss_tol(ref.MULTI_LABEL, zn, yn, wn)
    h.check()


@pytest.mark.parametrize("kind,bad", [("poisson", -1.0), ("logistic", 1.5), ("logistic", float("nan"))])
def test_estimator_raises_on_invalid_labels(tmp_path, kind, bad):
    batches = _kind_batches(kind, 4, 32, seed=0)
    batches[2][1][5] = bad
    e = _kind_estimator(kind, str(tmp_path), "dnn")
    rule = "labels must be in \\[0, 1\\]" if kind == "logistic" else "labels must be counts >= 0"
    with pytest.raises(ValueError, match=rule):
        e.train(lambda: iter(batches), steps=4)
    assert e._device.type == "cuda"
    with pytest.raises(ValueError, match=rule):
        e.evaluate(lambda: iter(batches))
    res = e.evaluate(lambda: iter(batches[:2]))     # valid labels evaluate normally afterwards
    assert np.isfinite(res["average_loss"])


# -------------------------------------------------------------------------------------------- the two planes
@pytest.mark.parametrize("kind", ["multi_label", "poisson"])
def test_hbm_and_cpu_planes_train_the_new_heads_alike(tmp_path, kind):
    """DNNLinearCombinedEstimator's network under MultiLabelHead(8, weight_column=...) or PoissonRegressionHead, one-hot
    hashed columns, weighted examples: still K5 and the fused wide tower; bounds as test_gpu_ps_multihot's."""
    from test_gpu_canned_head import _train_both_weighted
    from test_gpu_ps_multihot import _columns, _multihot_batches
    from tf_yarn_b200 import estimator as est
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = _columns(V, n_cat, n_num, weighted=False)
    spec = est.MultiLabelHead(8, weight_column="weight") if kind == "multi_label" else \
        est.PoissonRegressionHead(weight_column="weight")
    head = spec.canned_head()
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], spec.logits_dimension)
    g = torch.Generator().manual_seed(4)
    batches = []
    for f, _ in _multihot_batches(B, 3, V, n_cat, n_num, 1, seed=2):
        f = {k: (v[:, 0].clamp(min=0) if k.startswith("c") else v) for k, v in f.items() if not k.startswith("w")}
        f["weight"] = torch.tensor([0.0, -0.5, 0.25, 1.0, 2.0, 0.5, 1.5, 3.0]).repeat(B // 8)
        if kind == "multi_label":
            y = torch.stack([(f[f"c{j % n_cat}"] + j) % (2 + j % 3) == 0 for j in range(8)], dim=1).long()
        else:
            y = torch.poisson(torch.exp(0.3 * f["num"][:, 0] + (f["c0"] % 3).float() * 0.2), generator=g)
        batches.append((f, y))
    rels, calls = _train_both_weighted(tmp_path, net_cpu, batches, head)
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert calls.count("tfy_ps_gather_gemm") == 3 and calls.count("tfy_ps_multi_bag") == 3
    assert torch.device("cuda", 0) in head._state             # the HBM plane's loss ran the kernel


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", ["multi_label", "poisson", "logistic"])
def test_evaluate_on_the_gpu_matches_the_reference(tmp_path, kind, weighted):
    batches = _kind_batches(kind, 3, 500, seed=11)
    if weighted:
        batches[0][0]["w"][:7] = 0.0
    e = _kind_estimator(kind, str(tmp_path), "combined", weight_column="w" if weighted else None)
    res = e.evaluate(lambda: iter(batches))
    assert e._device.type == "cuda"
    with torch.no_grad():
        zs = [e._network({k: v.cuda() for k, v in f.items()}).double().cpu().numpy() for f, _ in batches]
    z, y = np.concatenate(zs), torch.cat([y for _, y in batches]).double().numpy()
    w = torch.cat([f["w"] for f, _ in batches]).double().numpy() if weighted else None
    code = {"multi_label": ref.MULTI_LABEL, "poisson": ref.POISSON_FULL, "logistic": ref.LOGISTIC}[kind]
    if kind == "multi_label":
        want = ref.multi_label_metrics(z, y, w, thresholds=(0.3, 0.5), classes=(0, 2))
    else:
        want = ref.regression_metrics(code, z, y, w)
    for k, v in want.items():
        assert res[k] == pytest.approx(v, rel=1e-5, abs=1e-6), k
    losses = [ref.loss(code, zb, yb.double().numpy(), f["w"].double().numpy() if weighted else None)
              for zb, (f, yb) in zip(zs, batches)]
    assert res["loss"] == pytest.approx(np.mean(losses), rel=1e-5, abs=1e-9)
