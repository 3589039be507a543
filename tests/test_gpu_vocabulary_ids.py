"""tfy_vocab_ids (ops/csrc/tfy_features.cu) on the H100, through ops/features.py FeatureIds: bit-equal to the torch
statement of the vocabulary columns (feature_column._vocabulary_ids) for V from 1 to 1,000,000 entries, with and
without OOV buckets, int32 and int64 sources and B from 1 to 100,000, mixed with identity, hashed, bucketized and
crossed columns, below, at and above one launch's source cap; every id inside its column's [0, V) or -1; a launch
captured in a CUDA graph equal to eager; and three training steps of a wide tower of vocabulary columns of different
sizes through the HBM and the CPU parameter-server planes, with the deep tower both through K5 and unfused."""
import copy
import functools
import sys
import types

import numpy as np
import pytest
import torch

from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import features as feature_ids

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


@functools.lru_cache(maxsize=None)
def _entries(V: int) -> np.ndarray:
    """V distinct keys spread over [0, 2^63), 0 and 2^63 - 1 among them, in a shuffled (id) order."""
    g = np.random.default_rng(V)
    keys = np.unique(g.integers(1, 2 ** 63 - 1, V + V // 8 + 8, dtype=np.int64))[:V - 2] if V > 2 \
        else np.zeros(0, np.int64)
    keys = np.concatenate([keys, np.array([0, 2 ** 63 - 1][:V], np.int64)])
    return keys[g.permutation(V)]


@functools.lru_cache(maxsize=None)
def _column(key: str, V: int, oov: int, default: int = -1):
    return fc.categorical_column_with_vocabulary_list(key, _entries(V), num_oov_buckets=oov, default_value=default)


def _raw(B: int, width: int, V: int, dtype, seed: int) -> torch.Tensor:
    """Half hits (every key at least once when B * width allows), a quarter neighbours of keys, the rest random values
    and missing ones."""
    g = np.random.default_rng(seed)
    keys = _entries(V)
    n = B * width
    v = keys[g.integers(0, V, n)]
    v[: min(V, n // 2)] = keys[: min(V, n // 2)]
    near = g.random(n) < 0.25
    v = np.where(near, np.clip(v + g.choice([-1, 1], n), 0, 2 ** 63 - 1), v)
    rnd = g.random(n) < 0.15
    v = np.where(rnd, g.integers(0, 2 ** 63 - 1, n, dtype=np.int64), v)
    v = np.where(g.random(n) < 0.05, -1 - g.integers(0, 5, n), v)
    t = torch.from_numpy(v.reshape(B, width).copy())
    return t.clamp(-(2 ** 31), 2 ** 31 - 1).int() if dtype == torch.int32 else t


def _check(lib, cols, f):
    fi = feature_ids.FeatureIds(cols, "cuda")
    out = fi({k: v.cuda() for k, v in f.items()}, lib).cpu()
    torch.cuda.synchronize()
    for t, c in enumerate(cols):
        want = fc._ids_and_weights(c, f)[0]
        got = out[t, :, :want.shape[1]]
        assert torch.equal(got, want), (t, c.key)
        assert torch.all(out[t, :, want.shape[1]:] == -1)
        assert torch.all((out[t] == -1) | ((out[t] >= 0) & (out[t] < c.num_buckets))), (t, c.key)
        # the CUDA torch path is the CPU torch path
        assert torch.equal(fc._ids_and_weights(c, {k: v.cuda() for k, v in f.items()})[0].cpu(), want)
    return fi


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("B", [1, 24, 1000, 100_000])
@pytest.mark.parametrize("oov", [0, 3])
@pytest.mark.parametrize("V", [1, 7, 1000, 1_000_000])
def test_kernel_is_bit_equal_to_the_torch_path_and_bounded(lib, V, oov, B, dtype):
    """A vocabulary column of width 2, a weighted one (default id V - 1 without OOV buckets), a cross of it with a raw
    feature, and the other kinds over the same features."""
    v = _column("a", V, oov)
    dflt = _column("a", V, 0, V - 1) if oov == 0 else v
    cols = [v, fc.weighted_categorical_column(dflt, "w"), fc.crossed_column([v, "b"], 10_007),
            fc.categorical_column_with_hash_bucket("a", 101), fc.categorical_column_with_identity("b", 50),
            fc.bucketized_column(fc.numeric_column("x", (2,)), [0.0, 1.0]),
            fc.crossed_column([fc.categorical_column_with_identity("b", 50), "a"], 977)]
    g = torch.Generator().manual_seed(B)
    f = {"a": _raw(B, 2, V, dtype, B + V), "b": torch.randint(-1, 50, (B, 1), generator=g).to(dtype),
         "w": torch.rand(B, 2, generator=g), "x": torch.randn(B, 2, generator=g)}
    fi = _check(lib, cols, f)
    assert fi.launches == 2 and len(fi.vocab_cols) == 1 + (oov == 0)


@pytest.mark.parametrize("S", [3, 32, 33, 70])
def test_group_sizes_around_the_source_cap(lib, S):
    cols = [_column(f"v{s}", (1, 7, 1000)[s % 3], s % 2 * 3) for s in range(S)]
    f = {f"v{s}": _raw(1000, 1 + s % 3, (1, 7, 1000)[s % 3], torch.int64 if s % 2 else torch.int32, s)
         for s in range(S)}
    fi = _check(lib, cols, f)
    assert len(fi.vocab_params) == -(-S // feature_ids.MAX_VOCAB_SRCS)
    assert fi.launches == len(fi.vocab_params) + len(fi.chunks)


def test_captured_launch_equals_eager(lib):
    cols = [_column("a", 1000, 3), fc.crossed_column([_column("a", 7, 0), "b"], 101),
            fc.categorical_column_with_hash_bucket("b", 33)]
    f = {"a": _raw(4096, 2, 1000, torch.int64, 0).cuda(), "b": torch.randint(0, 99, (4096, 1), device="cuda")}
    fi = feature_ids.FeatureIds(cols, "cuda")
    eager = fi(f, lib)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fi(f, lib)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = fi(f, lib)
    captured.fill_(-7)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


class _CountingLib:
    """The connection's kernel library, counting the id launches (vocabulary and feature ids) it makes."""

    def __init__(self, lib):
        self._lib, self.launches = lib, 0

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def tfy_feature_ids(self, *args):
        self.launches += 1
        return self._lib.tfy_feature_ids(*args)

    def tfy_vocab_ids(self, *args):
        self.launches += 1
        return self._lib.tfy_vocab_ids(*args)


@pytest.mark.parametrize("deep_kind", ["k5", "unfused"])
def test_hbm_and_cpu_planes_train_vocabulary_towers_alike(tmp_path, deep_kind):
    """The harness and bounds of test_gpu_feature_ids.test_hbm_and_cpu_planes_train_a_wide_tower_with_crosses_alike:
    the wide tower adds three vocabulary columns of different sizes (23, 14 and 38 buckets), one inside a cross, to the
    hashed ones, under FTRL, served by the fused multi-table kernels with ids from tfy_vocab_ids + tfy_feature_ids.
    The deep tower's embeddings are vocabulary columns of 40 buckets each: "k5" runs them through K5 with kernel ids;
    "unfused" adds an indicator of a vocabulary column, which K5 does not take, so the deep tower runs the unfused HBM
    route (torch ids on the device).  Every id launch of a step is in the step's counted launches."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import canned, ps, ps_hbm
    from tf_yarn_b200.models import wide_deep as wdm

    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    lst = fc.categorical_column_with_vocabulary_list
    perm = np.random.default_rng(0).permutation(V)
    wide, _ = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=n_cat, n_num=n_num)
    # over copies u<i> of the features c<i>: a linear model's tables are named by key, as TF's are
    v0 = lst("u0", perm[:20].tolist(), num_oov_buckets=3)                   # 23
    v1 = lst("u1", perm[::3].tolist(), default_value=0)                     # 14
    v2 = lst("u2", list(range(38)))                                         # 38, misses absent
    wide = wide + [v0, v1, fc.crossed_column([v2, "c0"], 500)]
    deep = [fc.embedding_column(lst(f"c{i}", perm[:37 - i].tolist(), num_oov_buckets=3 + i), 64) for i in range(n_cat)]
    deep = deep + [fc.numeric_column("numeric", (n_num,))]
    if deep_kind == "unfused":
        deep = deep + [fc.indicator_column(v1)]
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1)
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
        assert conn.fused_wide and conn.fused_first == (deep_kind == "k5")
        counting = conn.lib = _CountingLib(conn.lib)
        id_launches = []                                  # launches counted by the id path, per step
        account = conn.account

        def counted(pull=0, push=0, launches=1):
            if sys._getframe(1).f_code.co_name == "_derived_ids":
                id_launches[-1] += launches
            account(pull, push, launches)
        conn.account = counted
        w0 = [[cpu._region(i, s).double().clone() for s in range(1 + layout.var_slots[i])] for i in range(len(named))]

        batches = wdm.synthetic_batches(B, 3, vocab=V, seed=1, n_cat=n_cat, n_num=n_num)
        for feats, y in batches:
            feats = dict(feats, **{f"u{i}": feats[f"c{i}"] for i in range(n_cat)})
            before = counting.launches
            id_launches.append(0)
            for model, plane, dev in ((net, conn, "cuda"), (net_cpu, cpu, "cpu")):
                f = {k: v.to(dev) for k, v in feats.items()}
                plane.pull(model)
                model.zero_grad()
                out = model(f).float()
                torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y.to(dev).float()).backward()
                plane.push(model)
                plane.increment_global_step()
            # one vocabulary and one id launch for the wide tower, and as many for K5's group
            assert id_launches[-1] == counting.launches - before == (4 if deep_kind == "k5" else 2)
        torch.cuda.synchronize()
        rels = {}
        for i, (name, _) in enumerate(named):
            for s in range(1 + layout.var_slots[i]):
                hbm = conn.remote_tensor(i, s).double().cpu() - w0[i][s]
                want = cpu._region(i, s).double() - w0[i][s]
                assert want.norm() > 0, (name, s)
                rels[f"{name}/{s}"] = round(((hbm - want).norm() / want.norm()).item(), 4)
        print(rels)
        for k, r in rels.items():
            bound = 1e-2 if k.startswith("linear.") else (0.1 if k.endswith("/0") else 0.35)
            assert r < bound, (k, rels)
    finally:
        header.unlink()
        shards[0].unlink()
