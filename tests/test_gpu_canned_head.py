"""tfy_canned_head (ops/csrc/tfy_head.cu) against the float64 reference (tests/canned_head_reference.py), its determinism
and its invalid-label flag; weighted canned estimators on the HBM and CPU parameter-server planes; weighted evaluate.

Tolerances (canned_head_reference.loss_tol / grad_tol), with EPS32 = 2^-23:
  * per element the kernel computes l and dl/dz in fp32 from accurately rounded expf / logf / log1pf (no fast math).
    binary: max(z,0) - z y + log1p(exp(-|z|)) rounds at most four times on values of size |z| (1 + |y|) + 1;
    multi-class: m + log(s) - z_y with s a 32-lane fp32 sum of at most C terms <= 1 (relative error <= C EPS32, so
    log(s) is off by at most C EPS32) and two roundings on |m| + |z_y| + log C; regression: (z - y)^2 is off by at
    most 3 EPS32 (|z| + |y|)^2.  So |l - exact| <= 8 EPS32 S_i with S_i the scale of _element_scale.
  * the batch sum is fp64 (exact enough to ignore); the final (float) rounding adds EPS32 |L|, inside the
    (log2(Bc) + 4) EPS32 sum |w l| / (Bc) term that also covers the torch statement's fp32 reduction on the CPU.
  * gradient: sigmoid(z) - y is off by 4 EPS32 (1 + |y|); softmax_j - [j = y] by (C + 8) EPS32 p_j + 2 EPS32; 2 (z - y)
    by 8 EPS32 (|z| + |y|); the product with w / (Bc) adds two roundings of the result (4 EPS32 |g|).
An indexing or weighting fault is of the order of the values themselves, far above these bounds.

B = 100_003 with C = 1000 (10^8 logits) is left out: the float64 reference would need several GB of host memory.
"""
import numpy as np
import pytest
import torch

import canned_head_reference as ref
from test_canned_regressors_and_weights import head_inputs
from tf_yarn_b200.ops import head as H

pytestmark = pytest.mark.gpu

BS = [1, 7, 512, 4096, 100_003]
SHAPES = [(ref.BINARY, 1)] + [(ref.MULTI_CLASS, C) for C in (2, 3, 10, 1000)] + \
    [(ref.REGRESSION, d) for d in (1, 2, 3, 10, 1000)]
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
    z, y, w = head_inputs(head, B, C, seed=B + C, weighted=weighted, label_dtype=label_dtype)
    h, loss, grad = _run(head, C, z, y, w)
    wn = None if w is None else w.double().numpy()
    zn, yn = z.double().numpy(), y.double().numpy()
    assert abs(loss.item() - ref.loss(head, zn, yn, wn)) <= ref.loss_tol(head, zn, yn, wn)
    err = np.abs(grad.double().cpu().numpy() - ref.dlogits(head, zn, yn, wn))
    bound = ref.grad_tol(head, zn, yn, wn)
    assert (err <= bound).all(), (err.max(), np.unravel_index((err - bound).argmax(), err.shape))
    _, loss_only, none = _run(head, C, z, y, w, with_grad=False)          # dlogits = null: the same loss bits
    assert none is None and torch.equal(loss_only, loss)
    h.check()                                                             # no flag for valid labels


@pytest.mark.parametrize("head,C", SHAPES)
def test_two_runs_and_graph_replay_give_the_same_bits(head, C):
    B = 4096 if C < 1000 else 512
    z, y, w = head_inputs(head, B, C, seed=3, label_dtype=torch.float32 if head != ref.MULTI_CLASS else torch.int64)
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


def test_autograd_backward_scales_the_saved_gradient():
    z, y, w = head_inputs(ref.REGRESSION, 300, 3, seed=9, label_dtype=torch.float32)
    zc = z.cuda().requires_grad_(True)
    h = H.CannedHead(H.REGRESSION, 3)
    (h(y.cuda(), zc, w.cuda()) * 2.5).backward()
    _, _, grad = _run(H.REGRESSION, 3, z, y, w)
    assert torch.equal(zc.grad, grad * 2.5)


@pytest.mark.parametrize("label_dtype", LABELS, ids=["i32", "i64", "f32"])
def test_out_of_range_labels_are_skipped_and_flagged(label_dtype):
    B, C = 513, 10
    z, y, w = head_inputs(ref.MULTI_CLASS, B, C, seed=1, label_dtype=label_dtype, bad=True)
    y[7] = 10_000
    if label_dtype == torch.float32:
        y[8] = float("nan")
    h, loss, grad = _run(ref.MULTI_CLASS, C, z, y, w)
    zn, yn, wn = z.double().numpy(), y.double().numpy(), w.double().numpy()
    assert abs(loss.item() - ref.loss(ref.MULTI_CLASS, zn, yn, wn)) <= ref.loss_tol(ref.MULTI_CLASS, zn, yn, wn)
    g = grad.cpu()
    for r in (1, 7, B - 1) + ((8,) if label_dtype == torch.float32 else ()):
        assert not g[r].any(), r
    with pytest.raises(ValueError, match="labels must be class ids"):
        h.check()
    h.check()                                       # the flag was cleared with the error


def test_estimator_raises_on_out_of_range_labels(tmp_path):
    from tf_yarn_b200 import estimator as est
    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import feature_column as fc
    g = torch.Generator().manual_seed(0)
    batches = [({"x": torch.randn(32, 3, generator=g)}, torch.randint(0, 4, (32,), generator=g)) for _ in range(4)]
    batches[2][1][5] = 4
    e = est.DNNClassifier([8], [fc.numeric_column("x", (3,))], n_classes=4, model_dir=str(tmp_path),
                          optimizer=lambda: keras.optimizers.SGD(0.1),
                          config=est.RunConfig(log_step_count_steps=None))
    with pytest.raises(ValueError, match="labels must be class ids"):
        e.train(lambda: iter(batches), steps=4)
    with pytest.raises(ValueError, match="labels must be class ids"):
        e.evaluate(lambda: iter(batches))
    res = e.evaluate(lambda: iter(batches[:2]))     # valid labels evaluate normally afterwards
    assert 0.0 <= res["accuracy"] <= 1.0


# -------------------------------------------------------------------------------------------- the two planes
def _train_both_weighted(tmp_path, net_cpu, batches, head):
    """test_gpu_ps_multihot._train_both with the canned head's weighted loss (kernel on the HBM plane, torch
    statement on the CPU plane)."""
    import copy
    import types

    from test_gpu_ps_multihot import _Spy
    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import ps, ps_hbm
    net = copy.deepcopy(net_cpu).cuda()
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001, l2_regularization_strength=0.01)
    by_name = {n: ftrl for n, _ in named if n.startswith("linear.")}
    layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05), by_name)
    region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
    comm = types.SimpleNamespace(arena=types.SimpleNamespace(peer_base={0: region.data_ptr()}), device=0)
    header = ps.ShmShard(str(tmp_path / "header"), 8, create=True)
    shards = [ps.ShmShard(str(tmp_path / "shard0"), layout.shard_elems[0], create=True)]
    try:
        conn = ps_hbm.HbmConnection(layout, comm, {"ps:0": 0}, 0, [n for n, _ in named], header, net)
        conn.lib = spy = _Spy(conn.lib)
        cpu = ps.WorkerConnection(layout, shards, [n for n, _ in ps._named_trainables(net_cpu)])
        shards[0].data.zero_()
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                conn.remote_tensor(i).copy_(p.detach().reshape(-1))
                cpu._region(i).copy_(p.detach().reshape(-1).cpu())
                if layout.kinds[i] in ("adagrad", "ftrl"):
                    conn.remote_tensor(i, 1).fill_(layout.hypers[i]["init_s1"])
                    cpu._region(i, 1).fill_(layout.hypers[i]["init_s1"])
        conn.refresh_shadows()
        header.set_global_step(0)
        shards[0].set_global_step(0)
        conn.install(net)
        assert conn.fused_first and conn.fused_wide
        w0 = [[cpu._region(i, s).double().clone() for s in range(1 + layout.var_slots[i])] for i in range(len(named))]
        for feats, y in batches:
            for model, plane, dev in ((net, conn, "cuda"), (net_cpu, cpu, "cpu")):
                f = {k: v.to(dev) for k, v in feats.items()}
                plane.pull(model)
                model.zero_grad()
                head(y.to(dev), model(f), f["weight"]).backward()
                plane.push(model)
                plane.increment_global_step()
        torch.cuda.synchronize()
        rels = {}
        for i, (name, _) in enumerate(named):
            for s in range(1 + layout.var_slots[i]):
                hbm = conn.remote_tensor(i, s).double().cpu() - w0[i][s]
                want = cpu._region(i, s).double() - w0[i][s]
                if want.norm() > 0:
                    rels[f"{name}/{s}"] = round(((hbm - want).norm() / want.norm()).item(), 4)
                else:
                    assert hbm.norm() == 0, name
        return rels, spy.calls
    finally:
        header.unlink()
        shards[0].unlink()


@pytest.mark.parametrize("kind", ["regressor", "binary", "multiclass"])
def test_hbm_and_cpu_planes_train_a_weighted_canned_head_alike(tmp_path, kind):
    """One-hot hashed columns, weighted examples (some zero, some negative): the regressor (label_dimension 1) and the
    classifiers still take K5 and the fused wide tower; bounds as test_gpu_ps_multihot's."""
    from test_gpu_ps_multihot import _columns, _multihot_batches
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = _columns(V, n_cat, n_num, weighted=False)
    n_out = {"regressor": 1, "binary": 1, "multiclass": 4}[kind]
    head = {"regressor": H.CannedHead(H.REGRESSION, 1), "binary": H.CannedHead(H.BINARY, 1),
            "multiclass": H.CannedHead(H.MULTI_CLASS, 4)}[kind]
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], n_out)
    g = torch.Generator().manual_seed(4)
    batches = []
    for f, y in _multihot_batches(B, 3, V, n_cat, n_num, 1, seed=2):
        f = {k: (v[:, 0].clamp(min=0) if k.startswith("c") else v) for k, v in f.items() if not k.startswith("w")}
        f["weight"] = torch.tensor([0.0, -0.5, 0.25, 1.0, 2.0, 0.5, 1.5, 3.0]).repeat(B // 8)
        if kind == "regressor":
            y = f["num"][:, 0] * 2 + (f["c0"] % 3).float() + 0.1 * torch.randn(B, generator=g)
        elif kind == "multiclass":
            y = (f["c0"] + f["c1"]) % 4
        batches.append((f, y))
    rels, calls = _train_both_weighted(tmp_path, net_cpu, batches, head)
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert calls.count("tfy_ps_gather_gemm") == 3 and calls.count("tfy_ps_multi_bag") == 3
    assert torch.device("cuda", 0) in head._state             # the HBM plane's loss ran the kernel


@pytest.mark.parametrize("kind", ["binary", "multiclass", "regressor"])
def test_weighted_evaluate_on_the_gpu_matches_the_reference(tmp_path, kind):
    from tf_yarn_b200 import estimator as est
    from tf_yarn_b200.estimator import feature_column as fc
    g = torch.Generator().manual_seed(11)
    d = 3 if kind == "regressor" else 1
    batches = []
    for _ in range(3):
        x = torch.randn(500, 3, generator=g)
        w = torch.rand(500, generator=g) * 0.001                  # sum(w) below 1
        w[:7] = 0.0
        y = {"binary": lambda: (torch.rand(500, generator=g) < 0.4).long(),
             "multiclass": lambda: torch.randint(0, 4, (500,), generator=g, dtype=torch.int32),
             "regressor": lambda: torch.randn(500, d, generator=g)}[kind]()
        batches.append(({"x": x, "w": w}, y))
    cols = [fc.numeric_column("x", (3,))]
    if kind == "regressor":
        e = est.DNNRegressor([16], cols, model_dir=str(tmp_path), weight_column="w", label_dimension=d)
    else:
        e = est.DNNClassifier([16], cols, model_dir=str(tmp_path), weight_column=fc.numeric_column("w"),
                              n_classes=2 if kind == "binary" else 4)
    res = e.evaluate(lambda: iter(batches))
    assert e._device.type == "cuda"
    with torch.no_grad():
        zs = [e._network({k: v.cuda() for k, v in f.items()}).double().cpu().numpy() for f, _ in batches]
    z, y = np.concatenate(zs), torch.cat([y for _, y in batches]).double().numpy()
    w = torch.cat([f["w"] for f, _ in batches]).double().numpy()
    head = {"binary": ref.BINARY, "multiclass": ref.MULTI_CLASS, "regressor": ref.REGRESSION}[kind]
    want = ref.regressor_metrics(z, y, w) if kind == "regressor" else \
        ref.classifier_metrics(2 if kind == "binary" else 4, z, y, w)
    for k, v in want.items():
        assert res[k] == pytest.approx(v, rel=1e-5, abs=1e-7), k
    losses = [ref.loss(head, zb, yb.double().numpy(), f["w"].double().numpy())
              for zb, (f, yb) in zip(zs, batches)]
    assert res["loss"] == pytest.approx(np.mean(losses), rel=1e-5, abs=1e-9)
