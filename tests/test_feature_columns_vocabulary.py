"""Vocabulary columns (estimator/feature_column.py VocabularyColumn) against their NumPy statement
(tests/vocabulary_reference.py): construction errors, vocabulary files, ids for int32 and int64 sources and the edge
values, LinearModel / DenseFeatures / indicator / embedding / weighted / shared / crossed values and gradients, pickling,
the per-element lookup of the tfy_vocab_ids kernel built for the host and its struct's layout, the HBM plane's routing
on a connection over fake addresses, a checkpoint round trip and the shared-memory parameter server learning a label
that only the vocabulary ids predict."""
import ctypes
import os
import pickle
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import multihot_reference as mh
import shared_embedding_reference as sref
import vocabulary_reference as ref
from hbm_fake import hbm_connection
from tf_yarn_b200 import TaskSpec, data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.ops import features as feature_ids

fc = est.feature_column
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
TOP = 2 ** 63 - 1
ENTRIES = [907, 0, 2 ** 32 + 5, 13, TOP, 4_000_000_001, 77, 2 ** 31 - 1, 2 ** 31, 12]     # unsorted, 0 and 2^63-1


def _ids(col, features):
    return fc._ids_and_weights(col, features)[0]


def _np(features):
    return {k: v.numpy() for k, v in features.items()}


# ---------------------------------------------------------------------------------------------- construction
class _Huge:
    """A sequence that claims 2^31 entries: the length is checked before any entry is read."""

    def __len__(self):
        return 2 ** 31

    def __iter__(self):
        raise AssertionError("entries read")


def test_construction_errors():
    lst = fc.categorical_column_with_vocabulary_list
    for bad, match in (([], "empty"), ([3, 1, 3], "duplicate"), ([1, -1], r"\[0, 2\^63\)"),
                       ([1, 2 ** 63], r"\[0, 2\^63\)"), ([1, 2.0], r"\[0, 2\^63\)"), (["a", "b"], "string"),
                       ([True, 2], r"\[0, 2\^63\)"), (_Huge(), "2\\^31 - 1"), ("abc", "list"),
                       (np.array([1.0, 2.0]), "integers"), (np.array([[1, 2]]), "1-D"),
                       (np.array([2 ** 63], np.uint64), r"\[0, 2\^63\)")):
        with pytest.raises(ValueError, match=match):
            lst("a", bad)
    with pytest.raises(ValueError, match="num_oov_buckets"):
        lst("a", [1, 2], num_oov_buckets=-1)
    with pytest.raises(ValueError, match="not both"):
        lst("a", [1, 2], num_oov_buckets=2, default_value=0)
    for d in (-2, 2, 5):
        with pytest.raises(ValueError, match="default_value"):
            lst("a", [1, 2], default_value=d)
    for dtype in (torch.float32, "float32", "string", torch.int16, str, float):
        with pytest.raises(ValueError, match="string features"):
            lst("a", [1, 2], dtype=dtype)
    for dtype in (None, torch.int32, torch.int64, "int32", "int64"):
        assert lst("a", [1, 2], dtype=dtype).num_buckets == 2
    c = lst("a", ENTRIES, num_oov_buckets=3)
    assert c.num_buckets == len(ENTRIES) + 3 and c.key == "a" and c.default_value == -1
    assert lst("a", np.array([5, 6], np.uint64)).vocabulary == lst("b", [5, 6]).vocabulary
    assert lst("a", [1, 2], default_value=1).default_value == 1
    assert lst("a", [1, 2], num_oov_buckets=2, default_value=-1).num_buckets == 4
    keys = c.vocabulary.keys
    assert keys.dtype == np.int64 and keys.tolist() == ENTRIES and not keys.flags.writeable
    with pytest.raises(ValueError):
        keys[0] = 1
    for kw in ({"default_value": 0.7}, {"default_value": True}, {"num_oov_buckets": 1.5}, {"num_oov_buckets": "2"}):
        with pytest.raises(ValueError, match="integer"):
            lst("a", [1, 2], **kw)
    assert lst("a", [1, 2], num_oov_buckets=np.int64(2), default_value=np.int32(-1)).num_buckets == 4


def test_vocabulary_keeps_a_private_copy_of_the_entries():
    a = np.array([5, 3, 9], np.int64)
    c = fc.categorical_column_with_vocabulary_list("a", a)
    assert a.flags.writeable                                           # the caller's array is left alone
    a[0] = 4
    assert c.vocabulary.keys.tolist() == [5, 3, 9]
    assert c == fc.categorical_column_with_vocabulary_list("a", [5, 3, 9])
    assert _ids(c, {"a": torch.tensor([5, 4])})[:, 0].tolist() == [0, -1]


def test_weighted_vocabulary_column_is_not_hashed():
    v = fc.categorical_column_with_vocabulary_list("a", [1, 2])
    assert fc.weighted_categorical_column(v, "w").hashed is False
    h = fc.categorical_column_with_hash_bucket("a", 5)
    assert fc.weighted_categorical_column(h, "w").hashed is True


def test_vocabulary_file(tmp_path):
    path = tmp_path / "vocab.txt"
    path.write_text("  907\n0\n\t13 \n+44\r\n9223372036854775807\n")
    c = fc.categorical_column_with_vocabulary_file("a", str(path), num_oov_buckets=2)
    assert c.vocabulary.keys.tolist() == [907, 0, 13, 44, TOP] and c.num_buckets == 7
    assert fc.categorical_column_with_vocabulary_file("a", str(path), 3).vocabulary.keys.tolist() == [907, 0, 13]
    assert fc.categorical_column_with_vocabulary_file("a", str(path), 5, default_value=4).default_value == 4
    assert fc.categorical_column_with_vocabulary_file("a", str(path)).default_value == -1
    for size in (0, 6, -1, 2.5):
        with pytest.raises(ValueError, match="vocabulary_size"):
            fc.categorical_column_with_vocabulary_file("a", str(path), size)
    with pytest.raises(ValueError, match="integer"):
        fc.categorical_column_with_vocabulary_file("a", str(path), num_oov_buckets=0.5, default_value=1)
    with pytest.raises(ValueError, match="not both"):
        fc.categorical_column_with_vocabulary_file("a", str(path), num_oov_buckets=1, default_value=-1)
    with pytest.raises(ValueError, match="string features"):
        fc.categorical_column_with_vocabulary_file("a", str(path), dtype="string")
    path.write_text("1\n2")                                            # no trailing newline
    assert fc.categorical_column_with_vocabulary_file("a", str(path)).vocabulary.keys.tolist() == [1, 2]
    for text, line in (("1\n\n2\n", 2), ("1\n2\n\n", 3), ("1\nabc\n", 2), ("1\n2.5\n", 2), ("1_000\n", 1),
                       ("0x10\n", 1), ("1 2\n", 1), ("\n", 1)):
        path.write_text(text)
        with pytest.raises(ValueError, match=f"line {line}"):
            fc.categorical_column_with_vocabulary_file("a", str(path))
    path.write_text("5\n-1\n")
    with pytest.raises(ValueError, match=r"\[0, 2\^63\)"):
        fc.categorical_column_with_vocabulary_file("a", str(path))
    path.write_text("5\n6\n5\n")
    with pytest.raises(ValueError, match="duplicate"):
        fc.categorical_column_with_vocabulary_file("a", str(path))
    path.write_text("5\n6\nabc\n")                                     # lines past vocabulary_size are not read
    assert fc.categorical_column_with_vocabulary_file("a", str(path), 2).num_buckets == 2


def test_pickle_equality_and_hash():
    import cloudpickle
    c = fc.categorical_column_with_vocabulary_list("a", ENTRIES, num_oov_buckets=2)
    blob = cloudpickle.dumps(c)
    back = pickle.loads(blob)
    assert back == c and hash(back) == hash(c) and back.vocabulary.keys.tolist() == ENTRIES
    assert len(blob) < 8 * len(ENTRIES) + 1000
    c.vocabulary.tables("cpu")                                         # a device cache is not pickled
    assert len(cloudpickle.dumps(c)) == len(blob)
    assert c != fc.categorical_column_with_vocabulary_list("a", ENTRIES[::-1], num_oov_buckets=2)
    assert c != fc.categorical_column_with_vocabulary_list("a", ENTRIES, num_oov_buckets=3)
    assert {c: 1}[back] == 1
    big = fc.categorical_column_with_vocabulary_list("a", np.arange(1_000_000) * 3)
    assert big == pickle.loads(pickle.dumps(big))
    k1 = big.vocabulary.tables("cpu")
    assert big.vocabulary.tables("cpu")[0] is k1[0]                    # built once per device


# ---------------------------------------------------------------------------------------------- ids vs the reference
def _raw_batch(B=48, seed=0, width=3, dtype=torch.int64):
    """Every entry, its neighbours, missing values and random values (mostly out of the vocabulary)."""
    g = torch.Generator().manual_seed(seed)
    near = [v + d for v in ENTRIES for d in (-1, 0, 1) if 0 <= v + d <= TOP]
    vals = near + [-1, -5, -(2 ** 63)] + torch.randint(0, 2 ** 62, (B * width,), generator=g).tolist()
    raw = torch.tensor(vals[:B * width] if len(vals) >= B * width else vals + [1] * (B * width - len(vals)))
    raw = raw[torch.randperm(raw.numel(), generator=g)].reshape(B, width)
    if dtype == torch.int32:
        raw = raw.clamp(-(2 ** 31), 2 ** 31 - 1).int()
    return raw


def _vocab_cols():
    lst = fc.categorical_column_with_vocabulary_list
    n = len(ENTRIES)
    return {"oov0": lst("a", ENTRIES), "oov3": lst("a", ENTRIES, num_oov_buckets=3),
            "oov1": lst("a", ENTRIES, num_oov_buckets=1), "default0": lst("a", ENTRIES, default_value=0),
            "default_last": lst("a", ENTRIES, default_value=n - 1), "one_entry": lst("a", [TOP], num_oov_buckets=2)}


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("name", sorted(_vocab_cols()))
def test_ids_match_the_reference(name, dtype):
    col = _vocab_cols()[name]
    raw = _raw_batch(dtype=dtype)
    got = _ids(col, {"a": raw}).numpy()
    np.testing.assert_array_equal(got, ref.column_ids(col, {"a": raw.numpy()}))
    assert np.all((got == -1) | ((got >= 0) & (got < col.num_buckets)))
    assert np.all(got[raw.numpy() < 0] == -1)
    if dtype == torch.int64:
        for i, v in enumerate(ENTRIES):
            if name != "one_entry":
                assert _ids(col, {"a": torch.tensor([v])}).item() == i
    if name == "oov0":
        assert set(np.unique(got[raw.numpy() >= 0])) - set(range(len(ENTRIES))) == {-1}


def test_oov_buckets_are_the_hash_bucket_hash():
    col = _vocab_cols()["oov3"]
    raw = torch.randint(0, 2 ** 62, (4096,), generator=torch.Generator().manual_seed(5))
    h = fc._ids(fc.categorical_column_with_hash_bucket("a", 3), raw)
    assert torch.equal(_ids(col, {"a": raw})[:, 0], h + len(ENTRIES))


# ---------------------------------------------------------------------------------------------- the models
def _model_batch(B=40, seed=3):
    g = torch.Generator().manual_seed(seed)
    f = {"a": _raw_batch(B, seed, 3), "b": _raw_batch(B, seed + 1, 1)[:, 0],
         "aw": torch.randint(0, 4, (B, 3), generator=g).double() * 0.5, "n": torch.randn(B, 2, generator=g,
                                                                                       dtype=torch.float64)}
    f["b"][::3] = torch.tensor(ENTRIES[4])
    return f


@pytest.mark.parametrize("combiner", mh.COMBINERS)
def test_models_match_the_reference(combiner):
    lst = fc.categorical_column_with_vocabulary_list
    va = lst("a", ENTRIES, num_oov_buckets=3)
    vb = lst("b", ENTRIES[:6], default_value=2)
    wa = fc.weighted_categorical_column(va, "aw")
    x = fc.crossed_column([vb, va], 101)
    f = _model_batch()
    fn = _np(f)
    ids = {k: ref.column_ids(c, fn) for k, c in (("a", va), ("b", vb), ("x", x))}
    assert np.array_equal(ids["x"], _ids(x, f).numpy()) and (ids["x"] >= 0).any()

    # LinearModel: a vocabulary, a weighted vocabulary (other key) and a cross of two vocabularies
    lm = fc.LinearModel([vb, x, fc.numeric_column("n", (2,))], 2, sparse_combiner=combiner).double()
    with torch.no_grad():
        for p in lm.parameters():
            p.normal_()
    out = lm(f)
    tables = {k: lm.tables[c.key].weight.detach().numpy() for k, c in (("b", vb), ("x", x))}
    want = sum(mh.bag(tables[k], ids[k], None, combiner) for k in tables)
    want = want + lm.numeric(f["n"]).detach().numpy() + lm.bias.detach().numpy()
    np.testing.assert_allclose(out.detach().numpy(), want, rtol=1e-6, atol=1e-6)     # numerics enter in float32
    dout = torch.randn(out.shape, dtype=torch.float64)
    (out * dout).sum().backward()
    for k, c in (("b", vb), ("x", x)):
        V = c.num_buckets
        g = mh.table_grad(V, ids[k], None, mh.factors(ids[k], None, V, combiner), dout.numpy())
        np.testing.assert_allclose(lm.tables[c.key].weight.grad.numpy(), g, atol=1e-12)
    lw = fc.LinearModel([wa], 1, sparse_combiner=combiner).double()
    with torch.no_grad():
        lw.tables["a"].weight.normal_()
    np.testing.assert_allclose(lw(f).detach().numpy(),
                               mh.bag(lw.tables["a"].weight.detach().numpy(), ids["a"], fn["aw"], combiner),
                               rtol=1e-12, atol=1e-12)

    # DenseFeatures: embedding (plain and weighted), indicator and a shared collection of two vocabulary columns
    vb2 = lst("b", ENTRIES[:6] + [5, 6, 8], num_oov_buckets=4)
    va2 = lst("a", ENTRIES[:9], num_oov_buckets=4)                     # V = 13 = vb2's
    sh = fc.shared_embedding_columns([vb2, va2], 5, combiner)
    df = fc.DenseFeatures([fc.embedding_column(wa, 4, combiner), fc.indicator_column(va), sh[0],
                           fc.numeric_column("n", (2,)), sh[1]]).double()
    out = df(f)
    ea = df.embeddings["a"].weight.detach().numpy()
    counts = np.zeros((40, va.num_buckets))
    for r in range(40):
        for i in ids["a"][r]:
            if i >= 0:
                counts[r, i] += 1.0
    st = df.embeddings[sh[0].shared_name].weight.detach().numpy()
    sids = [ref.column_ids(vb2, fn), ref.column_ids(va2, fn)]
    mv = sref.member_values(st, sids, [None, None], combiner)
    want = np.concatenate([mh.bag(ea, ids["a"], fn["aw"], combiner), counts, mv[0], fn["n"], mv[1]], axis=1)
    assert df.width == want.shape[1]
    np.testing.assert_allclose(out.detach().numpy(), want, rtol=1e-12, atol=1e-12)
    dout = torch.randn(out.shape, dtype=torch.float64)
    (out * dout).sum().backward()
    V = va.num_buckets
    g = mh.table_grad(V, ids["a"], fn["aw"], mh.factors(ids["a"], fn["aw"], V, combiner), dout[:, :4].numpy())
    np.testing.assert_allclose(df.embeddings["a"].weight.grad.numpy(), g, atol=1e-12)
    o = 4 + va.num_buckets
    g = sref.table_grad(13, sids, [None, None], combiner, [dout[:, o:o + 5].numpy(), dout[:, o + 7:o + 12].numpy()])
    np.testing.assert_allclose(df.embeddings[sh[0].shared_name].weight.grad.numpy(), g, atol=1e-12)


def test_shared_collections_take_vocabulary_as_a_kind():
    lst = fc.categorical_column_with_vocabulary_list
    va, vb = lst("a", [1, 2, 3]), lst("b", [7, 8], num_oov_buckets=1)
    assert fc._kind(va) == fc._kind(fc.weighted_categorical_column(vb, "w")) == "vocabulary"
    assert len(fc.shared_embedding_columns([va, vb], 4)) == 2
    with pytest.raises(ValueError, match="one kind"):
        fc.shared_embedding_columns([va, fc.categorical_column_with_identity("c", 3)], 4)
    with pytest.raises(ValueError, match="num_buckets"):
        fc.shared_embedding_columns([va, lst("b", [7, 8])], 4)
    assert fc.crossed_column([va, "z"], 10).keys == (va, "z")
    with pytest.raises(ValueError, match="weight_tensor"):
        fc.crossed_column([fc.weighted_categorical_column(va, "w"), "z"], 10)


# ---------------------------------------------------------------------------------------------- the kernel's lookup
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("vocab") / "libvocab.so")
    cmd = [cxx, "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC,
           os.path.join(ROOT, "tests", "native", "vocab_host.cpp"),
           os.path.join(ROOT, "tests", "native", "features_host.cpp"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    lib = ctypes.CDLL(out)
    vp, i = ctypes.c_void_p, ctypes.c_int
    for name, args in (("tfy_host_vocab_lower_bound", [vp, i, vp, i, vp]), ("tfy_host_vocab_ids", [vp]),
                       ("tfy_host_vocab_lower_bound_even", [vp, i, i, vp]),
                       ("tfy_host_vocab_layout", [vp]), ("tfy_host_feature_ids", [vp])):
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = None
    return lib


def test_ctypes_mirror_matches_the_c_structs(host_lib):
    out = np.zeros(32, np.int64)
    host_lib.tfy_host_vocab_layout(out.ctypes.data)
    want = []
    for cls in (feature_ids.VocabSrc, feature_ids.VocabParams):
        want.append(ctypes.sizeof(cls))
        want += [getattr(cls, name).offset for name, _ in cls._fields_]
    assert out[:len(want)].tolist() == want
    assert ctypes.sizeof(feature_ids.VocabParams) <= 4096            # passed by value in the launch
    assert host_lib.tfy_host_vocab_cap() == feature_ids.MAX_VOCAB_SRCS


def test_host_built_lower_bound_near_2_to_the_31(host_lib):
    """A vocabulary of up to 2^31 - 1 entries: the search's midpoint must not wrap past INT32_MAX.  The keys are the
    fake sequence key(i) = 2 i, so nothing is stored; (lo + hi) / 2 would wrap once lo + hi > 2^31 - 1."""
    for n in (2 ** 31 - 1, 2 ** 31 - 2, 2 ** 30 + 1, 3):
        idx = np.array(sorted(i for i in {0, 1, n // 2, 2 ** 30, 2 ** 30 + 7, n - 2, n - 1, n} if 0 <= i <= n),
                       np.int64)
        x = np.concatenate([2 * idx, 2 * idx - 1, [-5, 2 * n + 100]]).astype(np.int64)
        out = np.zeros(x.size, np.int32)
        host_lib.tfy_host_vocab_lower_bound_even(x.ctypes.data, x.size, n, out.ctypes.data)
        want = np.clip((x + 1) // 2, 0, n)                          # the number of even keys 2 i < x, i < n
        np.testing.assert_array_equal(out, want)


def test_host_built_lower_bound(host_lib):
    keys = np.array(sorted(ENTRIES), np.int64)
    x = np.array(sorted({min(max(v + d, 0), TOP) for v in ENTRIES for d in (-1, 0, 1)}), np.int64)
    out = np.zeros(x.size, np.int32)
    host_lib.tfy_host_vocab_lower_bound(x.ctypes.data, x.size, keys.ctypes.data, keys.size, out.ctypes.data)
    np.testing.assert_array_equal(out, np.searchsorted(keys, x, side="left"))


def _host_ids(host_lib, cols, feats):
    fi = feature_ids.FeatureIds(cols, "cpu")
    out, srcs = fi.prepare(feats)
    for p in fi.vocab_params:
        host_lib.tfy_host_vocab_ids(ctypes.addressof(p))
    for p in fi.params:
        host_lib.tfy_host_feature_ids(ctypes.addressof(p))
    return out, fi


def _mixed_kinds():
    lst = fc.categorical_column_with_vocabulary_list
    cols = list(_vocab_cols().values())
    va = cols[1]
    return cols + [fc.categorical_column_with_hash_bucket("a", 101), fc.categorical_column_with_identity("c", 9),
                   fc.weighted_categorical_column(lst("c", [3, 1, 4, 5, 9]), "w"),
                   fc.bucketized_column(fc.numeric_column("x", (2,)), [0.0, 1.0]),
                   fc.crossed_column(["a", va], 997), fc.crossed_column([va, fc.categorical_column_with_identity("c", 9)],
                                                                       10_007)]


def _mixed_batch(B, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    f = {"a": _raw_batch(B, seed, 3, dtype), "c": torch.randint(-1, 10, (B, 2), generator=g).to(dtype),
         "w": torch.rand(B, 2, generator=g), "x": torch.randn(B, 2, generator=g)}
    return f


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("T", [3, 12, 40])
def test_host_built_kernels_equal_the_torch_path(host_lib, dtype, T):
    """Vocabulary columns mixed with every other kind, with T vocabulary sources below and above one launch's cap."""
    kinds = _mixed_kinds()
    cols = [kinds[t % len(kinds)] for t in range(T)]
    if T == 40:                                    # 40 distinct vocabulary sources: two vocabulary launches
        lst = fc.categorical_column_with_vocabulary_list
        cols = [lst(f"v{t}", ENTRIES[:1 + t % len(ENTRIES)], num_oov_buckets=t % 3) for t in range(T)]
    f = _mixed_batch(17, dtype)
    for t in range(40):
        f[f"v{t}"] = f["a"]
    out, fi = _host_ids(host_lib, cols, f)
    assert len(fi.vocab_params) == -(-len(fi.vocab_cols) // feature_ids.MAX_VOCAB_SRCS)
    assert fi.launches == len(fi.vocab_params) + len(fi.chunks)
    fn = _np(f)
    for t, c in enumerate(cols):
        want = _ids(c, f).numpy()
        np.testing.assert_array_equal(want, ref.column_ids(c, fn))
        np.testing.assert_array_equal(out[t, :, :want.shape[1]].numpy(), want)
        assert torch.all(out[t, :, want.shape[1]:] == -1)
        assert torch.all((out[t] == -1) | ((out[t] >= 0) & (out[t] < c.num_buckets)))


def test_sources_are_keyed_by_column():
    """A raw cross leaf and a vocabulary column over the same feature, and two vocabulary columns over one feature:
    three sources, with one segment per distinct vocabulary."""
    lst = fc.categorical_column_with_vocabulary_list
    v1 = lst("a", ENTRIES)
    v2 = v1._replace(num_oov_buckets=2)                                # the same Vocabulary object
    fi = feature_ids.FeatureIds([fc.crossed_column(["a", v1], 50), v1, v2, fc.weighted_categorical_column(v2, "w")],
                                "cpu")
    keys, ids = v1.vocabulary.tables("cpu")
    assert fi.vocab_cols == [v1, v2] and keys.numel() == len(ENTRIES) and ids.dtype == torch.int32
    srcs = fi.vocab_params[0].srcs
    assert [s.keys for s in srcs[:2]] == [keys.data_ptr()] * 2 and [s.ids for s in srcs[:2]] == [ids.data_ptr()] * 2
    # one device copy per vocabulary, whichever group or path uses it
    other = feature_ids.FeatureIds([v2], "cpu")
    assert other.vocab_params[0].srcs[0].keys == keys.data_ptr()
    assert [c[0][0] for c in fi._comps] == ["a", 0, 1, 1] and fi._comps[0][1][0] == 0


# ---------------------------------------------------------------------------------------------- HBM routing
def test_hbm_wide_tower_of_vocabulary_columns_is_derived_and_fused():
    from tf_yarn_b200.estimator import canned, ps_hbm
    lst = fc.categorical_column_with_vocabulary_list
    va, vb = lst("a", ENTRIES, num_oov_buckets=3), lst("b", ENTRIES[:4])
    wide = [va, vb, fc.categorical_column_with_hash_bucket("a", 1000)]
    net = canned._WideDeepNet(wide, [], [], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_wide_tower(conn, net) is True
    group = ps_hbm._TableGroup(conn, [0, 1, 2], wide)
    assert group.derived and group.V == 1000 and group.feature_ids.launches == 2     # one vocabulary + one id launch
    f = {"a": _raw_batch(9, 1, 1)[:, 0], "b": _raw_batch(9, 2, 1)}
    assert group.one_hot(f)
    ids = group.ids_of(f)
    for t, c in enumerate(wide):
        assert torch.equal(ids[t], _ids(c, f)[:, 0])
    # each kind of vocabulary use makes a group derived: bare, weighted, a cross's leaf
    for cols in ([va], [fc.weighted_categorical_column(va, "w")], [fc.crossed_column([va, "b"], 10)]):
        g = ps_hbm._TableGroup(conn, [0] * len(cols), cols)
        assert g.derived and g.feature_ids.launches == 2
    g = ps_hbm._TableGroup(conn, [2], [wide[2]])
    assert not g.derived and g.feature_ids is None
    # launches counted per step: 33 vocabulary columns are two vocabulary launches and two id launches
    many = [lst(f"v{t}", [t, t + 1]) for t in range(33)]
    g = ps_hbm._TableGroup(conn, [0] * 33, many)
    assert g.feature_ids.launches == 4


def test_hbm_weighted_vocabulary_column_multi_of():
    from tf_yarn_b200.estimator import canned, ps_hbm
    lst = fc.categorical_column_with_vocabulary_list
    wa = fc.weighted_categorical_column(lst("a", ENTRIES, num_oov_buckets=2), "aw")
    vb = lst("b", ENTRIES[:5], default_value=1)
    net = canned._WideDeepNet([wa, vb], [], [], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_wide_tower(conn, net) is True
    f = _model_batch(B=11)
    group = ps_hbm._TableGroup(conn, [0, 1], [wa, vb])
    assert group.derived and group.weighted and not group.one_hot(f)
    ids, w = group.multi_of(f)
    assert ids.shape == (2, 11, 3) and torch.equal(ids[0], _ids(wa, f)) and torch.equal(ids[1, :, :1], _ids(vb, f))
    assert torch.equal(w[0], f["aw"].float()) and torch.equal(w[1, :, 0], torch.ones(11))


def test_hbm_deep_tower_with_vocabulary_columns():
    """K5 keeps its rules: vocabulary embeddings of one num_buckets take kernel ids; of two sizes, K5 is refused."""
    from tf_yarn_b200.estimator import canned, ps_hbm
    lst = fc.categorical_column_with_vocabulary_list
    va, vb = lst("a", ENTRIES, num_oov_buckets=2), lst("b", ENTRIES[:6], num_oov_buckets=6)       # V = 12 both
    net = canned._WideDeepNet([], [fc.embedding_column(va, 64), fc.embedding_column(vb, 64),
                                   fc.numeric_column("n", (2,))], [64], 1)
    conn = hbm_connection(net, "ftrl")
    assert ps_hbm._try_fuse_first_layer(conn, net) is True
    f = _model_batch(B=9)
    f["a"] = f["a"][:, :1]
    d = net.dense_features(f)
    assert d.one_hot and d.ids.shape == (2, 9)
    assert torch.equal(d.ids[0], _ids(va, f)[:, 0]) and torch.equal(d.ids[1], _ids(vb, f)[:, 0])
    net = canned._WideDeepNet([], [fc.embedding_column(va, 64), fc.embedding_column(lst("b", [1, 2]), 64)], [64], 1)
    assert ps_hbm._try_fuse_first_layer(hbm_connection(net, "ftrl"), net) is False


# ---------------------------------------------------------------------------------------------- training
N_VOCAB = 40


def _vocab_task(n=4096, seed=0):
    """label = the parity of the vocabulary id of a random 32-bit raw value: the raw value's own parity, or any hash
    of it, says nothing about it."""
    g = np.random.default_rng(seed)
    entries = g.choice(2 ** 32, N_VOCAB, replace=False).astype(np.int64)
    idx = torch.from_numpy(g.integers(0, N_VOCAB, n))
    x = torch.from_numpy(entries)[idx]
    return entries, {"v": x}, (idx % 2).long()


def test_the_task_needs_the_vocabulary():
    entries, x, y = _vocab_task()
    assert abs((y == x["v"] % 2).float().mean().item() - 0.5) < 0.1
    col = fc.categorical_column_with_vocabulary_list("v", entries.tolist())
    assert torch.equal(_ids(col, x)[:, 0] % 2, y)


def _input_fns():
    _, x, y = _vocab_task()
    train = lambda: data.Dataset.from_tensor_slices((x, y)).shuffle(500, seed=1).batch(64).repeat()  # noqa: E731
    evalf = lambda: data.Dataset.from_tensor_slices((x, y)).batch(1024)  # noqa: E731
    return train, evalf


def test_checkpoint_round_trip_and_resume(tmp_path):
    entries = _vocab_task()[0]
    col = fc.categorical_column_with_vocabulary_list("v", entries.tolist(), num_oov_buckets=2)
    train, evalf = _input_fns()
    cfg = est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None)

    def make():
        return est.LinearClassifier([col], model_dir=str(tmp_path), optimizer=lambda: keras.optimizers.Ftrl(0.5),
                                    config=cfg)
    e = make()
    e.train(train, max_steps=200)
    first = e.evaluate(evalf)
    payload = torch.load(e.latest_checkpoint(), weights_only=False)
    assert payload["network"]["linear.tables.v.weight"].shape == (N_VOCAB + 2, 1)
    e2 = make()
    again = e2.evaluate(evalf)
    assert again["accuracy"] == first["accuracy"] and again["average_loss"] == pytest.approx(first["average_loss"])
    e2.train(train, max_steps=400)
    assert e2.get_global_step() == 400
    assert e2.evaluate(evalf)["accuracy"] > 0.95


def test_canned_estimators_take_vocabulary_columns(tmp_path):
    entries = _vocab_task()[0]
    col = fc.categorical_column_with_vocabulary_list("v", entries.tolist())
    train, evalf = _input_fns()
    cfg = est.RunConfig(log_step_count_steps=None)
    e = est.DNNClassifier([16], [fc.embedding_column(col, 8)], model_dir=str(tmp_path / "dnn"),
                          optimizer=lambda: keras.optimizers.Adagrad(0.3), config=cfg)
    e.train(train, max_steps=300)
    assert e.evaluate(evalf)["accuracy"] > 0.95


def _ps_experiment(model_dir):
    def experiment_fn():
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200 import keras
        from tf_yarn_b200.tensorflow import Experiment
        train, evalf = _input_fns()
        col = est.feature_column.categorical_column_with_vocabulary_list("v", _vocab_task()[0].tolist(),
                                                                         num_oov_buckets=1)
        e = est.DNNLinearCombinedClassifier(
            model_dir=model_dir, linear_feature_columns=[col], linear_optimizer=lambda: keras.optimizers.Ftrl(0.5),
            dnn_feature_columns=[est.feature_column.embedding_column(col, 8)], dnn_hidden_units=[16],
            dnn_optimizer=lambda: keras.optimizers.Adagrad(0.1),
            config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(train, max_steps=300),
                          est.EvalSpec(evalf, steps=None, start_delay_secs=0, throttle_secs=0))
    return experiment_fn


@pytest.mark.slow
def test_shared_memory_parameter_server_learns_a_vocabulary_label(tmp_path):
    """chief + 2 workers + 2 ps + evaluator through the CPU plane's shards: accuracy above 0.95 on the parity of the
    vocabulary id."""
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
