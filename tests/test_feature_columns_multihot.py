"""Multi-hot and weighted categorical columns (estimator/feature_column.py) against the float64 statement of TF's
combiner contract (tests/multihot_reference.py): DenseFeatures, LinearModel and indicator_column values and gradients,
the canned estimators and the shared-memory parameter server on a weighted multi-hot task, and the HBM plane's
routing decisions (estimator/ps_hbm.py) on a connection over fake addresses."""
import os
import sys

import numpy as np
import pytest
import torch

import multihot_reference as mh
from hbm_fake import hbm_connection
from tf_yarn_b200 import TaskSpec, data, keras
from tf_yarn_b200 import estimator as est

fc = est.feature_column


def _batch(rng, B, L, V, weighted, raw_max=None):
    """Raw ids [B, L] with -1 padding, zero weights, an all-missing example (0), an all-zero-weight example (1) and an
    example whose present weights cancel (2)."""
    ids = rng.integers(0, raw_max or V, (B, L))
    ids[rng.random((B, L)) < 0.25] = -1
    ids[0] = -1
    w = rng.choice([0.0, 0.25, -0.5, 0.5, 1.0, 2.0], (B, L)) if weighted else None
    if weighted:
        w[1] = 0.0
        if L >= 2:
            ids[2, :2] = [3, 4]
            w[2] = 0.0
            w[2, :2] = [0.5, -0.5]
    return ids, w


def _col(key, V, hashed, weighted):
    c = fc.categorical_column_with_hash_bucket(key, V) if hashed else fc.categorical_column_with_identity(key, V)
    return fc.weighted_categorical_column(c, key + "_w") if weighted else c


def _features(key, ids, w):
    f = {key: torch.from_numpy(ids)}
    if w is not None:
        f[key + "_w"] = torch.from_numpy(w).float()
    return f


def _bucket_ids(col, ids):
    return fc._ids(col, torch.from_numpy(ids)).numpy()


# ---------------------------------------------------------------------------------------------- hand-computed cases
@pytest.mark.parametrize("combiner,den", [("sum", 1.0), ("mean", 2.5), ("sqrtn", np.sqrt(4.25))])
def test_hand_computed_weighted_combiners(combiner, den):
    """ids [[1, 2, -1]], weights [[0.5, 2, 0]]: (0.5 e1 + 2 e2) / den, den = 1, 0.5 + 2, sqrt(0.25 + 4)."""
    col = fc.embedding_column(_col("a", 4, False, True), 3, combiner=combiner)
    df = fc.DenseFeatures([col])
    e = df.embeddings["a"].weight.detach().double()
    out = df(_features("a", np.array([[1, 2, -1]]), np.array([[0.5, 2.0, 0.0]]))).double()
    want = (0.5 * e[1] + 2 * e[2]) / den
    assert torch.allclose(out[0], want, rtol=1e-6, atol=1e-7)


def test_hand_computed_missing_and_cancelling_weights():
    """No present id gives 0 for every combiner; mean over weights summing to 0 is 0 (div_no_nan), sum is not."""
    ids, w = np.array([[-1, -1], [0, 1], [2, -1]]), np.array([[1.0, 1.0], [0.5, -0.5], [0.0, 3.0]])
    for combiner in mh.COMBINERS:
        df = fc.DenseFeatures([fc.embedding_column(_col("a", 4, False, True), 2, combiner=combiner)])
        e = df.embeddings["a"].weight.detach()
        out = df(_features("a", ids, w))
        assert torch.equal(out[0], torch.zeros(2)) and torch.equal(out[2], torch.zeros(2))
        if combiner == "mean":
            assert torch.equal(out[1], torch.zeros(2))
        else:
            assert torch.allclose(out[1], (0.5 * e[0] - 0.5 * e[1]) / (1.0 if combiner == "sum" else np.sqrt(0.5)))


# ---------------------------------------------------------------------------------------------- against the reference
@pytest.mark.parametrize("hashed", [False, True], ids=["identity", "hashed"])
@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "weighted"])
@pytest.mark.parametrize("combiner", mh.COMBINERS)
def test_dense_features_match_reference_values_and_gradients(combiner, weighted, hashed):
    rng = np.random.default_rng(7)
    V, B, L, D = 13, 64, 4, 5
    col = _col("a", V, hashed, weighted)
    df = fc.DenseFeatures([fc.embedding_column(col, D, combiner=combiner), fc.numeric_column("n")])
    df = df.double()
    ids, w = _batch(rng, B, L, V, weighted, raw_max=1000 if hashed else V - 1)
    if not hashed:
        ids[1] = V - 1                     # row V - 1 occurs only in example 1, whose weights are all zero if weighted
    feats = _features("a", ids, w)
    feats["n"] = torch.randn(B, 1, dtype=torch.float64)
    out = df(feats)
    table = df.embeddings["a"].weight.detach().numpy()
    bids = _bucket_ids(col, ids)
    assert np.all(bids[ids < 0] == -1) and np.all((bids[ids >= 0] >= 0) & (bids[ids >= 0] < V))
    want = mh.bag(table, bids, w, combiner)
    np.testing.assert_allclose(out[:, :D].detach().numpy(), want, rtol=1e-12, atol=1e-12)
    dout = torch.randn(B, D + 1, dtype=torch.float64)
    (out * dout).sum().backward()
    g = mh.table_grad(V, bids, w, mh.factors(bids, w, V, combiner), dout[:, :D].numpy())
    np.testing.assert_allclose(df.embeddings["a"].weight.grad.numpy(), g, rtol=1e-12, atol=1e-12)
    untouched = np.bincount(bids[mh.present(bids, w, V)], minlength=V) == 0
    assert untouched[V - 1] == (weighted and not hashed) or hashed
    assert np.all(df.embeddings["a"].weight.grad.numpy()[untouched] == 0)    # rows of absent occurrences only


@pytest.mark.parametrize("combiner", mh.COMBINERS)
def test_linear_model_combines_each_column_then_sums(combiner):
    rng = np.random.default_rng(3)
    V, B, L, units = 11, 50, 3, 2
    ca, cb = _col("a", V, True, True), _col("b", V, False, False)
    lm = fc.LinearModel([ca, fc.indicator_column(cb), fc.numeric_column("n")], units, sparse_combiner=combiner)
    lm = lm.double()
    with torch.no_grad():
        for p in lm.parameters():
            p.normal_()
    ia, wa = _batch(rng, B, L, V, True, raw_max=500)
    ib, _ = _batch(rng, B, L + 2, V, False)                 # a different L per column
    n = torch.randn(B, 1).double()          # LinearModel feeds numeric columns as fp32
    feats = {**_features("a", ia, wa), **_features("b", ib, None), "n": n}
    out = lm(feats)
    ba, bb = _bucket_ids(ca, ia), _bucket_ids(cb, ib)
    ta, tb = lm.tables["a"].weight.detach().numpy(), lm.tables["b"].weight.detach().numpy()
    want = (mh.bag(ta, ba, wa, combiner) + mh.bag(tb, bb, None, combiner) + lm.numeric(feats["n"]).detach().numpy()
            + lm.bias.detach().numpy())
    np.testing.assert_allclose(out.detach().numpy(), want, rtol=1e-12, atol=1e-12)
    dout = torch.randn(B, units, dtype=torch.float64)
    (out * dout).sum().backward()
    np.testing.assert_allclose(lm.tables["a"].weight.grad.numpy(),
                               mh.table_grad(V, ba, wa, mh.factors(ba, wa, V, combiner), dout.numpy()), atol=1e-12)
    np.testing.assert_allclose(lm.tables["b"].weight.grad.numpy(),
                               mh.table_grad(V, bb, None, mh.factors(bb, None, V, combiner), dout.numpy()), atol=1e-12)


@pytest.mark.parametrize("weighted", [False, True], ids=["counts", "weights"])
def test_indicator_column_counts_buckets_or_sums_weights(weighted):
    rng = np.random.default_rng(1)
    V, B, L = 6, 40, 5
    col = _col("a", V, False, weighted)
    ids, w = _batch(rng, B, L, V, weighted)
    ids[3] = [2, 2, 2, -1, 5]
    out = fc.DenseFeatures([fc.indicator_column(col)])(_features("a", ids, w)).double().numpy()
    want = np.zeros((B, V))
    ww = np.ones(ids.shape) if w is None else w
    for b in range(B):
        for j in range(L):
            if ids[b, j] >= 0:
                want[b, ids[b, j]] += ww[b, j]
    np.testing.assert_allclose(out, want, rtol=1e-6, atol=1e-7)
    if not weighted:
        assert out[3, 2] == 3.0 and out[3, 5] == 1.0


# ---------------------------------------------------------------------------------------------- existing inputs
def test_one_hot_and_unpadded_inputs_keep_their_values():
    """What the previous nn.EmbeddingBag-based columns computed: bit for bit for one-hot input and for unpadded
    multi-hot sums; a multi-hot mean divides by sum(w) = L now instead of scaling by 1/L (last bits)."""
    torch.manual_seed(0)
    V, B, D = 30, 64, 8
    for combiner in ("sum", "mean"):
        df = fc.DenseFeatures([fc.embedding_column(fc.categorical_column_with_hash_bucket("a", V), D, combiner)])
        old = torch.nn.EmbeddingBag(V, D, mode=combiner)
        old.weight.data.copy_(df.embeddings["a"].weight.data)
        for shape in [(B,), (B, 1), (B, 4)]:
            raw = torch.randint(0, 10_000, shape)
            ids = fc._ids(fc.categorical_column_with_hash_bucket("a", V), raw).reshape(B, -1)
            got, want = df({"a": raw}), old(ids)
            if combiner == "mean" and len(shape) == 2 and shape[1] > 1:
                assert torch.allclose(got, want, rtol=1e-6, atol=1e-7)
            else:
                assert torch.equal(got, want), (combiner, shape)
    lm = fc.LinearModel([fc.categorical_column_with_identity("a", V)], 1)
    with torch.no_grad():
        lm.tables["a"].weight.normal_()
    old = torch.nn.EmbeddingBag(V, 1, mode="sum")
    old.weight.data.copy_(lm.tables["a"].weight.data)
    ids = torch.randint(0, V, (B, 3))
    assert torch.equal(lm({"a": ids}), old(ids) + lm.bias)


def test_unknown_combiner_and_missing_weight_feature_are_rejected():
    cat = fc.categorical_column_with_identity("a", 5)
    with pytest.raises(ValueError, match="combiner"):
        fc.embedding_column(cat, 4, combiner="max")
    with pytest.raises(ValueError, match="combiner"):
        fc.LinearModel([cat], 1, sparse_combiner="avg")
    with pytest.raises(ValueError, match="combiner"):
        est.LinearClassifier([cat], sparse_combiner="bogus")
    with pytest.raises(ValueError, match="combiner"):
        est.DNNLinearCombinedClassifier(linear_feature_columns=[cat], linear_sparse_combiner="bogus")
    with pytest.raises(ValueError):
        fc.weighted_categorical_column(cat, "w", dtype=torch.int64)
    df = fc.DenseFeatures([fc.embedding_column(fc.weighted_categorical_column(cat, "a_weight"), 4)])
    with pytest.raises(KeyError, match="a_weight"):
        df({"a": torch.zeros(3, 2, dtype=torch.int64)})
    with pytest.raises(ValueError, match="shape"):
        df({"a": torch.zeros(3, 2, dtype=torch.int64), "a_weight": torch.ones(3, 3)})


# ---------------------------------------------------------------------------------------------- training
V_TASK, L_TASK = 20, 3


def _task(n=2048, seed=0):
    """label = 1 iff the weight on ids < 10 outweighs the weight on ids >= 10 (a weighted pair of id sets)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V_TASK, (n, L_TASK), generator=g)
    ids[torch.rand(n, L_TASK, generator=g) < 0.2] = -1
    ids[:, 0] = torch.randint(0, V_TASK, (n,), generator=g)
    w = torch.randint(1, 5, (n, L_TASK), generator=g).float() * 0.5
    w[ids < 0] = 0.0
    score = (w * (ids < 10).float() * (ids >= 0).float()).sum(1) - (w * (ids >= 10).float()).sum(1)
    keep = score != 0
    return {"ids": ids[keep], "ids_w": w[keep]}, (score[keep] > 0).long()


def _task_columns():
    return fc.weighted_categorical_column(fc.categorical_column_with_identity("ids", V_TASK), "ids_w")


def _input_fns():
    x, y = _task()
    train = lambda: data.Dataset.from_tensor_slices((x, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa: E731
    evalf = lambda: data.Dataset.from_tensor_slices((x, y)).batch(512)  # noqa: E731
    return train, evalf


@pytest.mark.parametrize("kind", ["linear", "wide_deep"])
def test_canned_estimators_learn_a_weighted_multihot_task(tmp_path, kind):
    train, evalf = _input_fns()
    cfg = est.RunConfig(save_checkpoints_steps=1000, log_step_count_steps=None)
    col = _task_columns()
    if kind == "linear":
        e = est.LinearClassifier([col], model_dir=str(tmp_path), optimizer=lambda: keras.optimizers.Adagrad(0.3),
                                 sparse_combiner="sum", config=cfg)
    else:
        e = est.DNNLinearCombinedClassifier(
            model_dir=str(tmp_path), linear_feature_columns=[col], linear_sparse_combiner="sqrtn",
            linear_optimizer=lambda: keras.optimizers.Adagrad(0.3),
            dnn_feature_columns=[fc.embedding_column(col, 8, combiner="mean")], dnn_hidden_units=[16],
            dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1), config=cfg)
    e.train(train, max_steps=300)
    assert e.evaluate(evalf)["accuracy"] > 0.9


def _ps_experiment(model_dir):
    def experiment_fn():
        from tf_yarn_b200 import keras
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200.tensorflow import Experiment
        train, evalf = _input_fns()
        col = _task_columns()
        e = est.DNNLinearCombinedClassifier(
            model_dir=model_dir, linear_feature_columns=[col], linear_sparse_combiner="mean",
            linear_optimizer=lambda: keras.optimizers.Adagrad(0.3),
            dnn_feature_columns=[est.feature_column.embedding_column(col, 8, combiner="sqrtn")],
            dnn_hidden_units=[16], dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1),
            config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=300),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_trains_the_weighted_multihot_task(tmp_path):
    """chief + 2 workers + 2 ps + evaluator through the CPU plane's shards, as tests/test_integration.py runs it."""
    import cloudpickle

    from tf_yarn_b200.estimator import summary
    from tf_yarn_b200.tensorflow import run_on_yarn
    cloudpickle.register_pickle_by_value(sys.modules[__name__])
    model_dir = str(tmp_path / "model")
    run_on_yarn(_ps_experiment(model_dir),
                {"chief": TaskSpec("1 GiB", 1), "worker": TaskSpec("1 GiB", 1, instances=2),
                 "ps": TaskSpec("1 GiB", 1, instances=2), "evaluator": TaskSpec("1 GiB", 1)})
    sc = summary.read_scalars(os.path.join(model_dir, "eval"))
    acc = [v for n, v in zip(sc["name"], sc["value"]) if n == "accuracy"]
    assert acc[-1] > 0.85, acc


# ---------------------------------------------------------------------------------------------- HBM routing
def test_hbm_plane_routes_one_hot_to_k5_and_multihot_or_weighted_to_the_weighted_bag():
    from tf_yarn_b200.estimator import canned, ps_hbm
    V = 1000
    cats = [fc.categorical_column_with_hash_bucket(f"c{i}", V) for i in range(3)]
    wcats = [cats[0], fc.weighted_categorical_column(cats[1], "c1_w"), cats[2]]
    num = fc.numeric_column("n", (5,))
    B = 8
    g = torch.Generator().manual_seed(0)
    one_hot = {"c0": torch.randint(0, 99, (B,), generator=g), "c1": torch.randint(0, 99, (B, 1), generator=g),
               "c2": torch.randint(-1, 99, (B,), generator=g), "n": torch.randn(B, 5), "c1_w": torch.ones(B, 1)}
    multi = dict(one_hot, c0=torch.randint(-1, 99, (B, 3), generator=g), c2=torch.randint(-1, 99, (B, 2), generator=g))
    for columns, combiner in ((cats, "sqrtn"), (wcats, "mean")):
        net = canned._WideDeepNet(columns, [fc.embedding_column(c, 64, combiner) for c in columns] + [num], [256, 64],
                                  1, sparse_combiner="sum")
        conn = hbm_connection(net)
        assert ps_hbm._try_fuse_first_layer(conn, net) is True
        assert ps_hbm._try_fuse_wide_tower(conn, net) is True
        weighted = columns is wcats
        for feats, want_one_hot in ((one_hot, not weighted), (multi, False)):
            d = net.dense_features(feats)
            assert d.one_hot is want_one_hot
            if want_one_hot:                                                 # K5: ids [T, B], no weights
                assert d.ids.shape == (3, B) and d.weights is None
            else:                                                            # weighted bag: [T, B, L], padded
                L = 3 if feats is multi else 1
                assert d.ids.shape == (3, B, L)
                assert (d.weights is not None) is weighted
                if feats is multi:
                    assert torch.all(d.ids[2, :, 2] < 0)                     # c2 (L = 2) padded to the group's L
                    if weighted:
                        assert torch.all(d.weights[2, :, 2] == 0) and torch.all(d.weights[0] == 1)
            raw = torch.stack([feats[f"c{t}"].reshape(B, -1)[:, 0] for t in range(3)])
            assert torch.equal(d.ids.reshape(3, B, -1)[:, :, 0] < 0, raw < 0)      # missing survives the hash
            ok = raw >= 0
            want = torch.stack([fc._ids(c, feats[c.key].reshape(B, -1)[:, 0]) for c in columns])
            assert torch.equal(d.ids.reshape(3, B, -1)[:, :, 0][ok], want[ok])   # ids >= 0 mapped as before
    # the wide tower's one-id kernels serve a one-hot unweighted batch only under the sum combiner
    net = canned._WideDeepNet(cats, [], [], 1, sparse_combiner="mean")
    assert ps_hbm._try_fuse_wide_tower(hbm_connection(net), net) is True
    group = ps_hbm._TableGroup(hbm_connection(net), [0, 1, 2], cats)
    assert group.one_hot(one_hot) and not group.one_hot(multi)
    assert not ps_hbm._TableGroup(hbm_connection(net), [0, 1, 2], wcats).one_hot(one_hot)


@pytest.mark.parametrize("hashed", [False, True], ids=["identity", "hashed"])
def test_hbm_bucketing_matches_the_feature_columns_for_large_ids(hashed):
    """The HBM plane's stacked bucketing (_TableGroup.ids_of / multi_of) maps every raw id as feature_column._ids
    does on the CPU plane: 32-bit hashed ids (whose hash product wraps int64 above 2^63 / 2654435761 ~ 3.47e9),
    ids beyond 2^32, and negative ids of any size (missing, -1)."""
    from tf_yarn_b200.estimator import canned, ps_hbm
    V, B = 100_000, 64
    cats = [_col(f"c{i}", V, hashed, i == 1) for i in range(3)]
    net = canned._WideDeepNet(cats, [], [], 1)
    group = ps_hbm._TableGroup(hbm_connection(net), [0, 1, 2], cats)
    g = torch.Generator().manual_seed(0)
    special = torch.tensor([0, 1, V - 1, V, 3_470_000_000, 3_600_000_000, 4_000_000_000, 2 ** 32 - 1, 2 ** 32,
                            2 ** 40 + 7, -1, -2, -V, -(2 ** 32), -(2 ** 40)])
    feats = {}
    for i in range(3):
        raw = torch.randint(0, 2 ** 32, (B, 2 + i), generator=g)
        raw[:special.numel(), 0] = special
        feats[f"c{i}"] = raw
    feats["c1_w"] = torch.rand(B, 3, generator=g)
    ids, w = group.multi_of(feats)
    for i, c in enumerate(cats):
        want = fc._ids(c, feats[c.key])
        assert torch.equal(ids[i, :, :want.shape[1]], want), i
        assert torch.all(ids[i, :, want.shape[1]:] == -1)
    assert torch.equal(w[1, :, :3], feats["c1_w"]) and torch.all(w[1, :, 3:] == 0)        # padded to L = 4
    assert torch.all(w[0, :, :2] == 1) and torch.all(w[0, :, 2:] == 0)
    one = {k: v[:, :1] for k, v in feats.items()}
    assert torch.equal(group.ids_of(one), torch.stack([fc._ids(c, one[c.key]).reshape(-1) for c in cats]))
    assert torch.all(fc._ids(cats[0], special[special < 0]) == -1)
