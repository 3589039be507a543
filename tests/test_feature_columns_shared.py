"""Shared embedding columns (tf.feature_column.shared_embedding_columns): construction, DenseFeatures values and
gradients against tests/shared_embedding_reference.py, checkpoints, and the HBM plane's routing on fake addresses."""
import numpy as np
import pytest
import torch

import shared_embedding_reference as sref
from hbm_fake import hbm_connection
from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import feature_column as fc


def _cats():
    return {"adv": fc.categorical_column_with_identity("adv", 20), "last_adv": fc.categorical_column_with_identity(
        "last_adv", 20), "q": fc.categorical_column_with_hash_bucket("q", 20),
        "wq": fc.weighted_categorical_column(fc.categorical_column_with_identity("tok", 20), "tok_w")}


# ---------------------------------------------------------------------------------------------- construction
def test_names_order_and_alias():
    c = _cats()
    cols = fc.shared_embedding_columns([c["last_adv"], c["adv"]], 8, initializer=None, max_norm=None, trainable=True)
    assert [x.categorical_column.key for x in cols] == ["last_adv", "adv"]
    assert {x.shared_name for x in cols} == {"adv_last_adv_shared_embedding"}
    assert all(x.dimension == 8 and x.combiner == "mean" for x in cols)
    named = fc.shared_embeddings([c["adv"], c["last_adv"]], 4, "sqrtn", shared_embedding_collection_name="advs")
    assert [x.shared_name for x in named] == ["advs", "advs"] and named[0].combiner == "sqrtn"
    # a weighted column counts as its base (identity) column
    w = fc.shared_embedding_columns([c["wq"], c["adv"]], 4)
    assert w[0].shared_name == "adv_tok_shared_embedding"


def test_construction_errors():
    c = _cats()
    b = fc.bucketized_column(fc.numeric_column("x", (4,)), [0.0, 1.0, 2.0, 3.0])          # 20 buckets
    cases = [([], 4, "mean"), ([c["adv"], fc.numeric_column("n")], 4, "mean"),
             ([c["adv"], fc.embedding_column(c["last_adv"], 4)], 4, "mean"),
             ([c["adv"], c["q"]], 4, "mean"), ([c["adv"], b], 4, "mean"),
             ([c["adv"], fc.categorical_column_with_identity("z", 21)], 4, "mean"),
             ([c["adv"], c["adv"]], 4, "mean"), ([c["adv"], c["last_adv"]], 0, "mean"),
             ([c["adv"], c["last_adv"]], 4, "max")]
    for cols, dim, comb in cases:
        with pytest.raises(ValueError):
            fc.shared_embedding_columns(cols, dim, comb)


def test_dense_features_width_parameters_and_name():
    c = _cats()
    sh = fc.shared_embedding_columns([c["adv"], c["last_adv"]], 8)
    df = fc.DenseFeatures([sh[0], fc.numeric_column("n", (3,)), sh[1], fc.embedding_column(c["q"], 5)])
    assert df.width == 8 + 3 + 8 + 5
    assert sum(p.numel() for p in df.parameters()) == 20 * 8 + 20 * 5
    assert set(df.state_dict()) == {"embeddings.adv_last_adv_shared_embedding.weight", "embeddings.q.weight"}
    assert df.shared == {"adv_last_adv_shared_embedding": [0, 2]}


def test_name_collisions_and_linear_model():
    c = _cats()
    sh = fc.shared_embedding_columns([c["adv"], c["last_adv"]], 8, shared_embedding_collection_name="q")
    with pytest.raises(ValueError, match="name"):
        fc.DenseFeatures([fc.embedding_column(c["q"], 8), sh[0]])
    with pytest.raises(ValueError, match="name"):
        fc.DenseFeatures([sh[0], fc.embedding_column(c["q"], 8)])
    other = fc.shared_embedding_columns([c["adv"], c["last_adv"]], 4, shared_embedding_collection_name="q")
    with pytest.raises(ValueError, match="disagree"):
        fc.DenseFeatures([sh[0], other[1]])
    with pytest.raises(ValueError, match="linear model"):
        fc.LinearModel([sh[0]], 1)


# ---------------------------------------------------------------------------------------------- values
@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_values_and_table_gradient_match_the_reference(combiner):
    """Three members (one-hot, multi-hot L = 3, weighted L = 2, with missing ids and zero weights) mixed with a plain
    embedding and a numeric column: each member's values, and the shared table's gradient as the sum over members."""
    g = torch.Generator().manual_seed(1)
    V, B, D = 20, 16, 6
    a, m = fc.categorical_column_with_identity("a", V), fc.categorical_column_with_identity("m", V)
    w = fc.weighted_categorical_column(fc.categorical_column_with_identity("t", V), "tw")
    sh = fc.shared_embedding_columns([a, m, w], D, combiner)
    plain = fc.embedding_column(fc.categorical_column_with_identity("p", V), 4)
    df = fc.DenseFeatures([sh[1], fc.numeric_column("n", (2,)), plain, sh[0], sh[2]]).double()
    f = {"a": torch.randint(0, V, (B, 1), generator=g), "m": torch.randint(-1, V, (B, 3), generator=g),
         "t": torch.randint(-1, V, (B, 2), generator=g), "tw": torch.randint(0, 4, (B, 2), generator=g).double() * 0.5,
         "p": torch.randint(0, V, (B,), generator=g), "n": torch.randn(B, 2, generator=g, dtype=torch.float64)}
    out = df(f)
    table = df.embeddings[sh[0].shared_name].weight
    T = table.detach().numpy()
    ids = [f["a"].numpy(), f["m"].numpy(), f["t"].numpy()]
    wts = [None, None, f["tw"].numpy()]
    want = sref.member_values(T, ids, wts, combiner)
    pos = {0: 6 + 2 + 4, 1: 0, 2: 6 + 2 + 4 + 6}                 # column offsets of the members in the output
    for k in range(3):
        np.testing.assert_allclose(out[:, pos[k]:pos[k] + D].detach().numpy(), want[k], rtol=1e-12, atol=1e-12)
    dout = torch.randn(out.shape, generator=g, dtype=torch.float64)
    (out * dout).sum().backward()
    grad = sref.table_grad(V, ids, wts, combiner, [dout[:, pos[k]:pos[k] + D].numpy() for k in range(3)])
    np.testing.assert_allclose(table.grad.numpy(), grad, rtol=1e-12, atol=1e-12)


def test_shared_sparse_push_reference_folds_each_row_once():
    """The reference push: two columns of one table hitting one row give ONE Adagrad step of (g1 + g2), not two."""
    import ps_reference as ref
    hp = dict(lr=0.1, eps=1e-7, p1=0.0, p2=0.0, p3=0.0)
    w, s1 = [np.zeros((3, 1))], [np.full((3, 1), 0.1)]
    ids = np.array([[[1]], [[1]]])
    sref.sparse_push(ref.ADAGRAD, w, s1, [np.zeros((3, 1))], [0, 0], ids, None, None, np.array([[1.0]]), 1, hp)
    assert s1[0][1, 0] == pytest.approx(0.1 + 4.0)
    assert w[0][1, 0] == pytest.approx(-0.1 * 2.0 / (np.sqrt(4.1) + 1e-7))


# ---------------------------------------------------------------------------------------------- HBM routing
def _net(deep):
    from tf_yarn_b200.estimator import canned
    return canned._WideDeepNet([], deep, [64], 1)


def test_hbm_k5_takes_shared_columns_with_a_column_to_table_map():
    from tf_yarn_b200.estimator import ps_hbm
    cats = [fc.categorical_column_with_hash_bucket(f"c{i}", 50) for i in range(4)]
    s1 = fc.shared_embedding_columns([cats[0], cats[2]], 64)
    s2 = fc.shared_embedding_columns([cats[1], cats[3]], 64)
    net = _net([s1[0], s2[0], s1[1], s2[1], fc.embedding_column(fc.categorical_column_with_hash_bucket("e", 50), 64),
                fc.numeric_column("n")])
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_first_layer(conn, net) is True
    name = {c: conn.names.index(f"dense_features.embeddings.{c}.weight") for c in
            (s1[0].shared_name, s2[0].shared_name, "e")}
    idx = [name[s1[0].shared_name], name[s2[0].shared_name], name[s1[0].shared_name], name[s2[0].shared_name],
           name["e"]]
    group = ps_hbm._TableGroup(conn, idx, [c.categorical_column for c in net.dense_features.columns[:5]])
    # the gather reads one pointer per column, repeats included; the push the distinct tables and table_of
    assert group.tables.tolist() == [conn.master_ptr(i) for i in idx]
    assert group.shared and group.distinct == [idx[0], idx[1], idx[4]]
    assert group.push_tables.tolist() == [conn.master_ptr(i) for i in group.distinct]
    assert group.table_of.dtype == torch.int32 and group.table_of.tolist() == [0, 1, 0, 1, 2]
    assert group.max_members == 2                      # the most columns of any one table
    # mixed-optimizer fallback: one push per distinct table, with its member columns
    parts = group.split()
    assert [m for m, _ in parts] == [[0, 2], [1, 3], [4]]
    assert [sub.shared for _, sub in parts] == [True, True, False]
    assert parts[0][1].table_of.tolist() == [0, 0] and parts[0][1].push_tables.tolist() == [conn.master_ptr(idx[0])]
    # an unshared group keeps the unmapped pushes
    assert not ps_hbm._TableGroup(conn, [idx[0], idx[1]], [cats[0], cats[1]]).shared
    # block sort while max_members * B * L <= 2048, plus the offsets kernel; unshared pushes as before
    assert ps_hbm.push_rows_launches(512, 4) == 4 and ps_hbm.push_rows_launches(512, 5) == 5
    assert ps_hbm.push_rows_launches(1024, 2) == 4 and ps_hbm.push_rows_launches(1024, 3) == 5
    assert ps_hbm.push_rows_launches(512) == 3


def test_hbm_thirteen_shared_pairs_push_with_the_block_sort():
    """26 deep columns as 13 pairs (column i with column i + 13), K5 at B = 512: max_members is 2, not the
    T - n_tables + 1 = 14 a map of 13 tables would allow, so the push counts the block sort's launches."""
    from tf_yarn_b200.estimator import ps_hbm
    cats = [fc.categorical_column_with_hash_bucket(f"c{i}", 50) for i in range(26)]
    pairs = [fc.shared_embedding_columns([cats[i], cats[i + 13]], 64) for i in range(13)]
    net = _net([p[0] for p in pairs] + [p[1] for p in pairs])
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_first_layer(conn, net) is True
    idx = [conn.names.index(f"dense_features.embeddings.{c.shared_name}.weight") for c in net.dense_features.columns]
    group = ps_hbm._TableGroup(conn, idx, [c.categorical_column for c in net.dense_features.columns])
    assert group.table_of.tolist() == list(range(13)) * 2 and group.max_members == 2
    assert ps_hbm.push_rows_launches(512, group.max_members) == 4


def test_hbm_unfused_tower_serves_each_collection_with_one_bag_and_one_group_push(monkeypatch):
    """Without K5 (a 32-wide collection), each collection's members are looked up by one weighted bag (T = members,
    the table repeated, col_stride D) and pushed by one shared push; the lookup returns the members' slices."""
    from tf_yarn_b200.estimator import ps_hbm
    cats = [fc.categorical_column_with_identity(f"c{i}", 30) for i in range(3)]
    sh = fc.shared_embedding_columns(cats, 32, "sqrtn")
    net = _net([sh[2], fc.numeric_column("n"), sh[0], sh[1]])
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_first_layer(conn, net) is False
    bags, pushes = [], []
    monkeypatch.setattr(ps_hbm, "weighted_bag", lambda lib, tables, ids, weights, code, D, V, out, out_ld, cs, f, num:
                        bags.append((tables.tolist(), tuple(ids.shape), code, D, V, out_ld, cs)) or out.zero_())
    monkeypatch.setattr(ps_hbm._TableGroup, "push", lambda self, ids, dout, w, f, code, ld=None: pushes.append(
        (self.table_of.tolist(), self.D, self.out_ld if ld is None else ld, self.col_stride)))
    assert ps_hbm._serve_shared_collections(conn, net) == 1
    df = net.dense_features
    B = 5
    feats = {"c0": torch.randint(0, 30, (B, 2)), "c1": torch.randint(0, 30, (B, 1)), "c2": torch.randint(0, 30, (B,)),
             "n": torch.randn(B, 1)}
    x = df(feats)
    assert x.shape == (B, 32 * 3 + 1)
    ti = conn.names.index(f"dense_features.embeddings.{sh[0].shared_name}.weight")
    # members in column order (c2, c0, c1), padded to the largest L
    assert bags == [([conn.master_ptr(ti)] * 3, (3, B, 2), ps_hbm.COMBINER_CODES["sqrtn"], 32, 30, 96, 32)]
    x.sum().backward()
    assert pushes == [([0, 0, 0], 32, 96, 32)]


# ---------------------------------------------------------------------------------------------- training
def _pair_task(n=4096, seed=0):
    """label = 1 iff the advertiser of the candidate equals the advertiser last clicked: a relation between two ids
    of one id space, which one shared table represents."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(0, 8, (n,), generator=g)
    b = torch.where(torch.rand(n, generator=g) < 0.5, a, torch.randint(0, 8, (n,), generator=g))
    return {"adv": a, "last_adv": b}, (a == b).long()


def _input_fns():
    from tf_yarn_b200 import data
    x, y = _pair_task()
    train = lambda: data.Dataset.from_tensor_slices((x, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa: E731
    evalf = lambda: data.Dataset.from_tensor_slices((x, y)).batch(1024)  # noqa: E731
    return train, evalf


def _shared_pair():
    return fc.shared_embedding_columns([fc.categorical_column_with_identity("adv", 8),
                                        fc.categorical_column_with_identity("last_adv", 8)], 8)


def test_checkpoint_round_trip(tmp_path):
    from tf_yarn_b200 import estimator as est
    train, evalf = _input_fns()
    cfg = est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None)

    def make():
        return est.DNNClassifier([32], _shared_pair(), model_dir=str(tmp_path),
                                 optimizer=lambda: keras.optimizers.Adagrad(0.1), config=cfg)
    e = make()
    e.train(train, max_steps=200)
    first = e.evaluate(evalf)
    payload = torch.load(e.latest_checkpoint(), weights_only=False)
    assert payload["network"]["dense_features.embeddings.adv_last_adv_shared_embedding.weight"].shape == (8, 8)
    again = make().evaluate(evalf)
    assert again["accuracy"] == first["accuracy"] and again["average_loss"] == pytest.approx(first["average_loss"])


def _ps_experiment(model_dir):
    def experiment_fn():
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200 import keras
        from tf_yarn_b200.tensorflow import Experiment
        train, evalf = _input_fns()
        e = est.DNNClassifier([32], _shared_pair(), model_dir=model_dir,
                              optimizer=lambda: keras.optimizers.Adagrad(0.1),
                              config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=600),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_learns_a_shared_id_relation(tmp_path):
    """chief + 2 workers + 2 ps + evaluator through the CPU plane's shards: accuracy above 0.9 on a label that depends
    on both members' ids (their equality; either alone gives 0.5 to 0.56)."""
    import os
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
    acc = [v for n, v in zip(sc["name"], sc["value"]) if n == "accuracy"]
    assert acc[-1] > 0.9, acc
