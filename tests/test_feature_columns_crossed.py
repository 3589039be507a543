"""Bucketized and crossed feature columns (estimator/feature_column.py) against their NumPy statement
(tests/crossed_reference.py): construction rules and names, ids for every kind of key and the special values,
LinearModel / DenseFeatures / indicator_column values and gradients, the per-element math of the tfy_feature_ids kernel
built for the host, the HBM plane's routing on a connection over fake addresses, a checkpoint round trip and the
shared-memory parameter server learning a label that only a cross predicts."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import crossed_reference as ref
import multihot_reference as mh
from hbm_fake import hbm_connection
from tf_yarn_b200 import TaskSpec, data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.ops import features as feature_ids

fc = est.feature_column
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
CUDA_INC = "/usr/local/cuda/include"
BOUNDS = [18.0, 25.0, 30.0, 35.5, 40.0]


def _np(features):
    return {k: v.numpy() for k, v in features.items()}


def _ids(col, features):
    return fc._ids_and_weights(col, features)[0]


# ---------------------------------------------------------------------------------------------- construction
def test_construction_errors_and_names():
    age = fc.numeric_column("age")
    with pytest.raises(ValueError):
        fc.bucketized_column(fc.numeric_column("img", (2, 2)), [1.0])
    with pytest.raises(ValueError):
        fc.bucketized_column(fc.categorical_column_with_identity("a", 3), [1.0])
    for bad in ([], [1.0, 1.0], [2.0, 1.0], (1.0, 3.0, 2.0)):
        with pytest.raises(ValueError, match="boundaries"):
            fc.bucketized_column(age, bad)
    b = fc.bucketized_column(fc.numeric_column("age", (3,)), BOUNDS)
    assert b.key == "age_bucketized" and b.num_buckets == 3 * 6
    ident = fc.categorical_column_with_identity("occ", 7)
    with pytest.raises(ValueError, match="two"):
        fc.crossed_column(["a"], 10)
    with pytest.raises(ValueError, match="hash_bucket_size"):
        fc.crossed_column(["a", "b"], 0)
    with pytest.raises(ValueError, match="hash_bucket_size"):
        fc.crossed_column(["a", "b"], 2 ** 62)                        # the int64 statement of the uint64 modulo
    assert fc.crossed_column(["a", "b"], 2 ** 62 - 1).num_buckets == 2 ** 62 - 1
    with pytest.raises(ValueError, match="hashed"):
        fc.crossed_column(["a", fc.categorical_column_with_hash_bucket("h", 10)], 10)
    with pytest.raises(ValueError, match="weight_tensor"):
        fc.crossed_column(["a", fc.weighted_categorical_column(ident, "w")], 10)
    with pytest.raises(ValueError):
        fc.crossed_column(["a", age], 10)
    x = fc.crossed_column(["education", ident], 1000)
    assert x.key == "education_X_occ" and x.num_buckets == 1000 and x.hash_key == ref.DEFAULT_HASH_KEY
    nested = fc.crossed_column([b, x], 50, hash_key=7)
    assert nested.keys == (b, "education", ident) and nested.key == "age_bucketized_X_education_X_occ"
    assert fc.crossed_column([x], 10).keys == x.keys                  # two leaf keys
    assert fc.crossed_column([x, "z"], 10).keys == ("education", ident, "z")


# ---------------------------------------------------------------------------------------------- ids vs the reference
def _special_batch(B=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    age = torch.randn(B, 3, generator=g) * 15 + 30
    age[0] = torch.tensor([18.0, 25.0, 35.5])                       # exactly on boundaries
    age[1] = torch.tensor([float("nan"), float("inf"), -float("inf")])
    age[2] = torch.tensor([np.nextafter(np.float32(18), np.float32(0)), np.nextafter(np.float32(40), np.float32(99)),
                           35.5000001])                             # the last rounds to 35.5 in float32
    raw = torch.randint(0, 1000, (B, 2), generator=g)
    raw[3] = torch.tensor([2 ** 63 - 1, 2 ** 63 - 2])               # top bit of the uint64 hash input
    raw[4] = torch.tensor([-(2 ** 63), -5])                          # missing
    raw[5, 1] = -1
    occ = torch.randint(-1, 7, (B, 3), generator=g)
    occ[6] = -1                                                      # all missing
    return {"age": age, "edu": raw, "occ": occ, "one": torch.randint(0, 50, (B,), generator=g)}


def _columns():
    b = fc.bucketized_column(fc.numeric_column("age", (3,)), BOUNDS)
    b1 = fc.bucketized_column(fc.numeric_column("one"), [10.0, 20.0])
    ident = fc.categorical_column_with_identity("occ", 7)
    x = fc.crossed_column(["edu", ident], 1000)
    return {"bucketized": b, "bucketized_k1": b1, "raw_x_identity": x,
            "raw_x_bucketized": fc.crossed_column(["edu", b], 997),
            "nested": fc.crossed_column([b, x, "one"], 10_007, hash_key=123),
            "big_v": fc.crossed_column(["edu", "one"], 2 ** 61 - 1),
            "hash_key_top_bit": fc.crossed_column([ident, "edu"], 3, hash_key=2 ** 64 - 1)}


@pytest.mark.parametrize("name", sorted(_columns()))
def test_ids_match_the_reference(name):
    col = _columns()[name]
    f = _special_batch()
    got = _ids(col, f).numpy()
    want = ref.column_ids(col, _np(f))
    np.testing.assert_array_equal(got, want)
    assert np.all((got == -1) | ((got >= 0) & (got < col.num_buckets)))
    if isinstance(col, fc.CrossedColumn):
        assert got.shape[1] == fc._width(col, f)
        assert np.all(got[4, :] == -1)                               # a missing raw value leaves no slot present
        if "occ" in col.key:
            assert np.all(got[6] == -1)


def test_bucketized_special_values_and_offsets():
    col = _columns()["bucketized"]
    f = _special_batch()
    got = _ids(col, f).numpy()
    n = len(BOUNDS) + 1
    assert got[0].tolist() == [1, n + 2, 2 * n + 4]                  # x == boundary counts that boundary
    assert got[1].tolist() == [5, n + 5, 2 * n + 0]                  # NaN and +inf last, -inf first
    assert got[2].tolist() == [0, n + 5, 2 * n + 4]


def test_unsigned_modulo_of_hashes_with_the_top_bit_set():
    col = fc.crossed_column(["a", "b"], 1_000_003)
    g = torch.Generator().manual_seed(1)
    f = {"a": torch.randint(0, 2 ** 62, (4096,), generator=g), "b": torch.randint(0, 2 ** 62, (4096,), generator=g)}
    h = ref.fingerprint_cat64(ref.fingerprint_cat64(np.uint64(col.hash_key), f["a"].numpy().astype(np.uint64)),
                              f["b"].numpy().astype(np.uint64))
    assert (h >> np.uint64(63)).sum() > 1000                          # many hashes read negative as int64
    np.testing.assert_array_equal(_ids(col, f).numpy()[:, 0], (h % np.uint64(1_000_003)).astype(np.int64))


def test_existing_columns_keep_their_ids():
    g = torch.Generator().manual_seed(2)
    raw = torch.randint(-3, 2 ** 40, (32, 3), generator=g)
    for col in (fc.categorical_column_with_identity("a", 17), fc.categorical_column_with_hash_bucket("a", 17)):
        ids, w = fc._ids_and_weights(col, {"a": raw})
        assert w is None and torch.equal(ids, fc._ids(col, raw).reshape(32, -1))
        np.testing.assert_array_equal(ids.numpy(), ref.column_ids(col, {"a": raw.numpy()}))


# ---------------------------------------------------------------------------------------------- the models
@pytest.mark.parametrize("combiner", mh.COMBINERS)
def test_linear_model_dense_features_and_indicator_match_the_reference(combiner):
    cols = _columns()
    b, x, nested = cols["bucketized"], cols["raw_x_identity"], cols["nested"]
    f = _special_batch(B=40, seed=3)
    lm = fc.LinearModel([b, x, nested, fc.numeric_column("one")], 2, sparse_combiner=combiner).double()
    with torch.no_grad():
        for p in lm.parameters():
            p.normal_()
    out = lm(f)
    fn = _np(f)
    ids = {c.key: ref.column_ids(c, fn) for c in (b, x, nested)}
    tables = {k: lm.tables[k].weight.detach().numpy() for k in ids}
    want = sum(mh.bag(tables[k], ids[k], None, combiner) for k in ids)
    want = want + lm.numeric(f["one"].reshape(-1, 1).double()).detach().numpy() + lm.bias.detach().numpy()
    np.testing.assert_allclose(out.detach().numpy(), want, rtol=1e-12, atol=1e-12)
    dout = torch.randn(out.shape, dtype=torch.float64)
    (out * dout).sum().backward()
    for k in ids:
        V = tables[k].shape[0]
        g = mh.table_grad(V, ids[k], None, mh.factors(ids[k], None, V, combiner), dout.numpy())
        np.testing.assert_allclose(lm.tables[k].weight.grad.numpy(), g, atol=1e-12)

    df = fc.DenseFeatures([fc.embedding_column(x, 4, combiner), b, fc.indicator_column(nested),
                           fc.embedding_column(b, 3, combiner)]).double()
    out = df(f)
    ex, eb = df.embeddings[x.key].weight.detach().numpy(), df.embeddings[b.key].weight.detach().numpy()
    onehot = np.zeros((40, b.num_buckets))
    counts = np.zeros((40, nested.num_buckets))
    for r in range(40):
        onehot[r, ids[b.key][r]] = 1.0
        for i in ids[nested.key][r]:
            if i >= 0:
                counts[r, i] += 1.0
    want = np.concatenate([mh.bag(ex, ids[x.key], None, combiner), onehot, counts,
                           mh.bag(eb, ids[b.key], None, combiner)], axis=1)
    assert df.width == want.shape[1]
    np.testing.assert_allclose(out.detach().numpy(), want, rtol=1e-6, atol=1e-6)
    dout = torch.randn(out.shape, dtype=torch.float64)
    (out * dout).sum().backward()
    V = x.num_buckets
    g = mh.table_grad(V, ids[x.key], None, mh.factors(ids[x.key], None, V, combiner), dout[:, :4].numpy())
    np.testing.assert_allclose(df.embeddings[x.key].weight.grad.numpy(), g, atol=1e-12)


# ---------------------------------------------------------------------------------------------- the kernel's math
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("features") / "libfeatures.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "features_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    vp, i = ctypes.c_void_p, ctypes.c_int
    for name, args in (("tfy_host_fingerprint_cat64", [vp, vp, i, vp]), ("tfy_host_bucketize", [vp, i, vp, i, vp]),
                       ("tfy_host_digits", [vp, i, vp]), ("tfy_host_feature_ids", [vp]),
                       ("tfy_host_feature_layout", [vp])):
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = None
    lib.tfy_host_feature_caps.argtypes = [i]
    return lib


def test_ctypes_mirror_matches_the_c_structs(host_lib):
    out = np.zeros(32, np.int64)
    host_lib.tfy_host_feature_layout(out.ctypes.data)
    want = []
    for cls in (feature_ids.FeatComp, feature_ids.FeatCol, feature_ids.FeatureParams):
        want.append(ctypes.sizeof(cls))
        want += [getattr(cls, name).offset for name, _ in cls._fields_]
    assert out[:len(want)].tolist() == want
    assert ctypes.sizeof(feature_ids.FeatureParams) <= 4096           # passed by value in the launch
    assert (host_lib.tfy_host_feature_caps(0), host_lib.tfy_host_feature_caps(1)) == \
        (feature_ids.MAX_COLS, feature_ids.MAX_COMPS)


def test_host_built_fingerprint_bucketize_and_digits(host_lib):
    g = np.random.default_rng(0)
    a = g.integers(0, 2 ** 63, 4096, dtype=np.uint64) * np.uint64(2) + g.integers(0, 2, 4096, dtype=np.uint64)
    b = g.integers(0, 2 ** 63, 4096, dtype=np.uint64)
    out = np.zeros(4096, np.uint64)
    host_lib.tfy_host_fingerprint_cat64(a.ctypes.data, b.ctypes.data, 4096, out.ctypes.data)
    np.testing.assert_array_equal(out, ref.fingerprint_cat64(a, b))
    bounds = np.array(BOUNDS, np.float32)
    x = np.concatenate([bounds, np.nextafter(bounds, -np.inf), np.nextafter(bounds, np.inf),
                        np.array([np.nan, np.inf, -np.inf, 0, 1e30], np.float32),
                        g.normal(30, 15, 1000).astype(np.float32)]).astype(np.float32)
    c = np.zeros(x.size, np.int32)
    host_lib.tfy_host_bucketize(x.ctypes.data, x.size, bounds.ctypes.data, bounds.size, c.ctypes.data)
    np.testing.assert_array_equal(c, ref.bucketize(x[:, None], bounds)[:, 0])
    widths = np.array([3, 1, 4, 2], np.int32)
    d = np.zeros((24, 4), np.int32)
    host_lib.tfy_host_digits(widths.ctypes.data, 4, d.ctypes.data)
    assert d.tolist() == [list(t) for t in np.ndindex(*widths)]       # row-major: the first key slowest


def _host_ids(host_lib, cols, feats):
    fi = feature_ids.FeatureIds(cols, "cpu")
    out, srcs = fi.prepare(feats)
    for p in fi.params:
        host_lib.tfy_host_feature_ids(ctypes.addressof(p))
    return out, fi


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("T", [3, 33, 70])
def test_host_built_kernel_equals_the_torch_path(host_lib, dtype, T):
    """Every column kind in one group, with T below and above one launch's column cap (and component cap)."""
    f = _special_batch(B=17)
    if dtype == torch.int32:
        f["edu"] = torch.where(f["edu"] > 2 ** 31 - 1, 2 ** 31 - 1, f["edu"]).clamp(min=-(2 ** 31)).int()
        f["occ"], f["one"] = f["occ"].int(), f["one"].int()
    kinds = list(_columns().values()) + [fc.categorical_column_with_hash_bucket("edu", 101),
                                         fc.weighted_categorical_column(fc.categorical_column_with_identity("occ", 5),
                                                                        "w")]
    cols = [kinds[t % len(kinds)] for t in range(T)]
    f["w"] = torch.rand(17, 3)
    out, fi = _host_ids(host_lib, cols, f)
    assert (fi.launches == 1) == (T == 3) and fi.launches >= -(-T // feature_ids.MAX_COLS)
    assert all(len(ch) <= feature_ids.MAX_COLS and sum(len(feature_ids._leaves(cols[t])) for t in ch)
               <= feature_ids.MAX_COMPS for ch in fi.chunks)
    fn = _np(f)
    for t, c in enumerate(cols):
        want = _ids(c, f).numpy()
        np.testing.assert_array_equal(want, ref.column_ids(c, fn))
        np.testing.assert_array_equal(out[t, :, :want.shape[1]].numpy(), want)
        assert torch.all(out[t, :, want.shape[1]:] == -1)
        assert torch.all((out[t] == -1) | ((out[t] >= 0) & (out[t] < c.num_buckets)))


def test_a_bucketized_feature_wider_than_its_column_never_leaves_the_column(host_lib, monkeypatch):
    """bucketized_column(numeric_column("x", (3,)), [0, 1]) has V = 9.  A 4-wide "x" would give the id 11 to the
    fourth value, a row past the table that a mixed-V group's bag and push would not reject: FeatureIds refuses the
    batch as the torch path does, and the kernel's own bound writes -1 for it if it ever got such a launch."""
    col = fc.bucketized_column(fc.numeric_column("x", (3,)), [0.0, 1.0])
    other = fc.crossed_column(["a", col], 7)
    f = {"x": torch.tensor([[2.0, 2.0, 2.0, 2.0]]), "a": torch.tensor([[1]])}
    with pytest.raises(ValueError, match="4 values"):
        _ids(col, f)
    for cols in ([col], [other]):
        with pytest.raises(ValueError, match="4 values"):
            feature_ids.FeatureIds(cols, "cpu").prepare(f)
    monkeypatch.setattr(fc, "_check_source_width", lambda c, w: None)          # past the host check
    out, _ = _host_ids(host_lib, [col, other], f)
    assert out[0, 0].tolist() == [2, 5, 8, -1]
    assert torch.all((out[1] >= -1) & (out[1] < 7))


# ---------------------------------------------------------------------------------------------- HBM routing
def test_hbm_wide_tower_with_crosses_of_mixed_v_is_fused_and_padded():
    from tf_yarn_b200.estimator import canned, ps_hbm
    cols = _columns()
    hashed = [fc.categorical_column_with_hash_bucket("edu", 1000), fc.categorical_column_with_identity("occ", 7)]
    wide = hashed + [cols["bucketized"], cols["raw_x_identity"], cols["raw_x_bucketized"]]
    net = canned._WideDeepNet(wide, [], [], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_wide_tower(conn, net) is True
    f = _special_batch(B=9)
    idx = [conn.names.index(f"linear.tables.{c.key}.weight") for c in wide]
    group = ps_hbm._TableGroup(conn, idx, wide)
    assert group.derived and not group.same_v and group.V == max(c.num_buckets for c in wide)
    assert not group.one_hot(f)
    ids, w = group.multi_of(f)
    L = max(fc._width(c, f) for c in wide)
    assert w is None and ids.shape == (5, 9, L) == (5, 9, 6)
    for t, c in enumerate(wide):
        want = _ids(c, f)
        assert torch.equal(ids[t, :, :want.shape[1]], want)
        assert torch.all(ids[t, :, want.shape[1]:] == -1)
    # the push's sort key t * V + id with the group's largest V: distinct per (table, id), below the sentinel T * V,
    # and the block sort's local_bits (from V) hold every id and the local sentinel V
    V = group.V
    local_bits = V.bit_length()                          # tfy_ps.cu: 64 - clz(V)
    assert int(ids.max()) < V < 2 ** local_bits and int((torch.arange(5)[:, None, None] * V + ids).max()) < 5 * V
    pairs = {(t, int(i)) for t in range(5) for i in ids[t][ids[t] >= 0].unique()}
    assert len({t * V + i for t, i in pairs}) == len(pairs)
    # one id per example (k = 1 bucketized, crosses of one-hot keys): the one-id kernels' [T, B] ids
    one = [cols["bucketized_k1"], fc.crossed_column(["one", fc.categorical_column_with_identity("occ", 7)], 100),
           hashed[0]]
    g1 = ps_hbm._TableGroup(hbm_connection(canned._WideDeepNet(one, [], [], 1), "ftrl"), [0, 1, 2], one)
    f1 = dict(f, occ=f["occ"][:, :1], edu=f["edu"][:, :1])
    assert g1.one_hot(f1) and g1.ids_of(f1).shape == (3, 9)
    assert torch.equal(g1.ids_of(f1)[1], _ids(one[1], f1)[:, 0])


def test_hbm_wide_tower_of_mixed_v_without_new_columns_is_still_refused():
    from tf_yarn_b200.estimator import canned, ps_hbm
    wide = [fc.categorical_column_with_hash_bucket("a", 1000), fc.categorical_column_with_hash_bucket("b", 500)]
    net = canned._WideDeepNet(wide, [], [], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_wide_tower(conn, net) is False
    group = ps_hbm._TableGroup(conn, [0, 1], wide)
    assert not group.derived and group.feature_ids is None and group.V == 1000 and not group.same_v


def test_hbm_deep_tower_with_new_columns():
    """K5 keeps its rules (dimension 64, one V): a cross and a bucketized column of the same V take their ids from
    the group; an indicator or bucketized column in DenseFeatures leaves the deep tower unfused."""
    from tf_yarn_b200.estimator import canned, ps_hbm
    b = fc.bucketized_column(fc.numeric_column("age", (3,)), [1.0, 2.0, 3.0, 4.0, 5.0])        # V = 18
    x = fc.crossed_column(["edu", "one"], 18)
    net = canned._WideDeepNet([], [fc.embedding_column(b, 64), fc.embedding_column(x, 64), fc.numeric_column("one")],
                              [64], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_first_layer(conn, net) is True
    f = _special_batch(B=9)
    d = net.dense_features(f)
    assert not d.one_hot and d.ids.shape == (2, 9, 3)
    assert torch.equal(d.ids[0], _ids(b, f)) and torch.equal(d.ids[1, :, :2], _ids(x, f))
    for extra in (b, fc.indicator_column(x)):
        net = canned._WideDeepNet([], [fc.embedding_column(x, 64), extra], [64], 1)
        assert ps_hbm._try_fuse_first_layer(hbm_connection(net, "ftrl"), net) is False


# ---------------------------------------------------------------------------------------------- training
N_A, N_B = 6, 5


def _cross_task(n=4096, seed=0):
    """label = 1 iff (a + b) is even: a and b alone carry no information about it, their cross all of it."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(0, N_A, (n,), generator=g)
    b = torch.randint(0, N_B, (n,), generator=g)
    return {"a": a, "b": b}, ((a + b) % 2 == 0).long()


def _cross_columns():
    ca, cb = fc.categorical_column_with_identity("a", N_A), fc.categorical_column_with_identity("b", N_B)
    return ca, cb, fc.crossed_column([ca, "b"], 10_000)


def test_the_task_needs_the_cross():
    x, y = _cross_task()
    for k in ("a", "b"):
        for v in range(N_A if k == "a" else N_B):
            m = x[k] == v
            assert abs(y[m].float().mean().item() - 0.5) < 0.12
    ids = _ids(_cross_columns()[2], x)[:, 0]
    assert len(set(ids.tolist())) == N_A * N_B                    # no two combinations share a bucket


def _input_fns():
    x, y = _cross_task()
    train = lambda: data.Dataset.from_tensor_slices((x, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa: E731
    evalf = lambda: data.Dataset.from_tensor_slices((x, y)).batch(1024)  # noqa: E731
    return train, evalf


def test_checkpoint_round_trip_and_resume(tmp_path):
    ca, cb, cross = _cross_columns()
    train, evalf = _input_fns()
    cfg = est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None)

    def make():
        return est.LinearClassifier([ca, cb, cross], model_dir=str(tmp_path),
                                    optimizer=lambda: keras.optimizers.Ftrl(0.5), config=cfg)
    e = make()
    e.train(train, max_steps=200)
    first = e.evaluate(evalf)
    payload = torch.load(e.latest_checkpoint(), weights_only=False)
    names = set(payload["network"])
    assert {"linear.tables.a_X_b.weight", "linear.tables.a.weight", "linear.tables.b.weight"} <= names
    assert payload["network"]["linear.tables.a_X_b.weight"].shape == (10_000, 1)
    e2 = make()                                          # a new estimator restores the checkpoint ...
    again = e2.evaluate(evalf)
    assert again["accuracy"] == first["accuracy"] and again["average_loss"] == pytest.approx(first["average_loss"])
    e2.train(train, max_steps=400)                       # ... and resumes from its global step
    assert e2.get_global_step() == 400
    assert e2.evaluate(evalf)["accuracy"] > 0.95


def _ps_experiment(model_dir):
    def experiment_fn():
        from tf_yarn_b200 import keras
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200.tensorflow import Experiment
        train, evalf = _input_fns()
        ca, cb, cross = _cross_columns()
        e = est.DNNLinearCombinedClassifier(
            model_dir=model_dir, linear_feature_columns=[ca, cb, cross],
            linear_optimizer=lambda: keras.optimizers.Ftrl(0.5),
            dnn_feature_columns=[est.feature_column.embedding_column(cross, 8)], dnn_hidden_units=[16],
            dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1),
            config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=300),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_learns_a_crossed_label(tmp_path):
    """chief + 2 workers + 2 ps + evaluator through the CPU plane's shards: accuracy above 0.95 on a label that
    neither column predicts alone (each alone: about 0.5)."""
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
    assert acc[-1] > 0.95, acc
