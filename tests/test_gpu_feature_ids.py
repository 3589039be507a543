"""tfy_feature_ids (ops/csrc/tfy_features.cu) on the H100: bit-equal to the torch statement of the columns
(feature_column._ids_and_weights) for every column kind, int32 and int64 sources and the special values, below, at and
above one launch's column cap and from one example to several waves of CTAs; every id inside its column's [0, V) or -1;
a launch captured in a CUDA graph equal to eager; and three training steps of a wide tower with bucketized numerics and
two crosses of different V through the HBM and the CPU parameter-server planes."""
import copy
import sys
import types

import pytest
import torch

from test_feature_columns_crossed import _columns, _ids, _special_batch
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.ops import features as feature_ids

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernel)
    from tf_yarn_b200.ops import native
    return native.load()


def _kinds():
    return list(_columns().values()) + [
        fc.categorical_column_with_hash_bucket("edu", 101),
        fc.weighted_categorical_column(fc.categorical_column_with_identity("occ", 5), "w"),
        fc.crossed_column(["one", fc.categorical_column_with_identity("occ", 7), "edu"], 2 ** 40 + 15)]


def _batch(B, dtype):
    base = _special_batch(B=24)
    reps = -(-B // 24)
    f = {k: v.repeat((reps,) + (1,) * (v.dim() - 1))[:B] for k, v in base.items()}
    g = torch.Generator().manual_seed(B)
    f["age"][24:] = torch.randn(max(B - 24, 0), 3, generator=g) * 15 + 30
    f["edu"][24:] = torch.randint(0, 2 ** 62, (max(B - 24, 0), 2), generator=g)
    if dtype == torch.int32:
        f["edu"] = f["edu"].clamp(-(2 ** 31), 2 ** 31 - 1).int()
        f["occ"], f["one"] = f["occ"].int(), f["one"].int()
    f["w"] = torch.rand(B, 3, generator=g)
    return f


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("B", [1, 24, 1000, 100_000])
@pytest.mark.parametrize("T", [3, 32, 33, 70])
def test_kernel_is_bit_equal_to_the_torch_path_and_bounded(lib, T, B, dtype):
    """B = 100k with L_max = 6: 600k slots per column, several waves of the grid-stride loop."""
    kinds = _kinds()
    cols = [kinds[t % len(kinds)] for t in range(T)]
    f = _batch(B, dtype)
    fi = feature_ids.FeatureIds(cols, "cuda")
    out = fi({k: v.cuda() for k, v in f.items()}, lib)
    torch.cuda.synchronize()
    assert fi.launches == len(fi.chunks) >= -(-T // feature_ids.MAX_COLS) and (fi.launches > 1) == (T > 32)
    out = out.cpu()
    for t, c in enumerate(cols):
        want = _ids(c, f)
        assert torch.equal(out[t, :, :want.shape[1]], want), (t, c)
        assert torch.all(out[t, :, want.shape[1]:] == -1)
        assert torch.all((out[t] == -1) | ((out[t] >= 0) & (out[t] < c.num_buckets))), (t, c)


def test_captured_launch_equals_eager(lib):
    cols = _kinds()
    f = {k: v.cuda() for k, v in _batch(4096, torch.int64).items()}
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
    """The connection's kernel library, counting the tfy_feature_ids launches it makes."""

    def __init__(self, lib):
        self._lib, self.feature_ids = lib, 0

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def tfy_feature_ids(self, *args):
        self.feature_ids += 1
        return self._lib.tfy_feature_ids(*args)


@pytest.mark.parametrize("deep_kind", ["k5", "unfused"])
def test_hbm_and_cpu_planes_train_a_wide_tower_with_crosses_alike(tmp_path, deep_kind):
    """The harness of test_gpu_ps_kernels.test_hbm_and_cpu_planes_train_a_wide_and_deep_network_alike, with the wide
    tower extended by the 5 numerics bucketized at 10 boundaries (V = 55) and two crosses of V = 1000 and 500, under
    FTRL; it must be served by the fused multi-table kernels with ids from tfy_feature_ids.  "unfused" adds the
    bucketized column and an indicator of a cross to DenseFeatures, which K5 does not take: the deep tower then runs
    the unfused HBM route (torch ids, one bag per table, the remote-weight GEMM).

    The wide tower is pushed from fp32 gradients: that test measured its update within 1e-3 of the CPU plane's, and
    this one at most 2e-4 on an H100 80GB HBM3 (700 W), crosses included; what differs comes from the deep tower's bf16
    GEMMs through the shared logits, since the ids are bit-equal.  The bound is 1e-2 for the wide tower's values and
    slots, well below the order-1 differences of a wrong id or table; the deep tower keeps that test's bounds (0.1
    values, 0.35 slots).  Every tfy_feature_ids launch of a step is in the step's counted launches."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import canned, ps, ps_hbm
    from tf_yarn_b200.models import wide_deep as wdm

    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=n_cat, n_num=n_num)
    nb = fc.bucketized_column(fc.numeric_column("numeric", (n_num,)), [-2.0 + 0.4 * i for i in range(10)])
    cross = fc.crossed_column(["c0", "c1"], 1000)
    wide = wide + [nb, cross, fc.crossed_column([nb, "c2"], 500)]
    if deep_kind == "unfused":
        deep = deep + [nb, fc.indicator_column(fc.crossed_column([nb, "c2"], 24))]
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
            before = counting.feature_ids
            id_launches.append(0)
            for model, plane, dev in ((net, conn, "cuda"), (net_cpu, cpu, "cpu")):
                f = {k: v.to(dev) for k, v in feats.items()}
                plane.pull(model)
                model.zero_grad()
                out = model(f).float()
                torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y.to(dev).float()).backward()
                plane.push(model)
                plane.increment_global_step()
            assert id_launches[-1] == counting.feature_ids - before == 1        # the wide tower's 9 tables: one launch
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
