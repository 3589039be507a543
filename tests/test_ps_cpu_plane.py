"""Shared-memory parameter-server plane (estimator/ps.py) in process: the update applied on the ps copy by `push`
must be the optimizer's update -- checked against torch.optim on the same gradient sequence for every optimizer a
variable can carry (what TF's ps runs as ApplyGradientDescent / ApplyAdagrad / ApplyAdam / ApplyFtrl; reference:
tf_yarn/tensorflow/tasks/tf_task_common.py:46-50)."""
import pytest
import torch

from hbm_fake import hbm_connection
from tf_yarn_b200 import keras
from tf_yarn_b200.estimator import ps


def _connection(tmp_path, net, desc, n_ps=2, by_name=None):
    named = ps._named_trainables(net)
    layout = ps.make_layout(named, n_ps, desc, by_name)
    shards = [ps.ShmShard(str(tmp_path / f"shard{i}"), layout.shard_elems[i], create=True) for i in range(n_ps)]
    for s in shards:
        s.data.zero_()
    conn = ps.WorkerConnection(layout, shards, [n for n, _ in named])
    with torch.no_grad():
        for i, (_, p) in enumerate(named):
            conn._region(i).copy_(p.detach().reshape(-1))
            if layout.kinds[i] in ("adagrad", "ftrl"):
                conn._region(i, 1).fill_(layout.hypers[i]["init_s1"])
    shards[0].set_global_step(0)
    return conn, shards


@pytest.mark.parametrize("desc", [keras.optimizers.SGD(0.1), keras.optimizers.Adagrad(0.1), keras.optimizers.Adam(0.01),
                                  keras.optimizers.Adadelta(1.0),
                                  keras.optimizers.Ftrl(0.1, l1_regularization_strength=0.001)],
                         ids=["sgd", "adagrad", "adam", "adadelta", "ftrl"])
def test_push_applies_the_optimizers_update(tmp_path, desc):
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Tanh(), torch.nn.Linear(7, 3))
    ref = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Tanh(), torch.nn.Linear(7, 3))
    ref.load_state_dict(net.state_dict())
    conn, shards = _connection(tmp_path, net, desc)
    opt = desc.to_torch(ref.parameters())
    g = torch.Generator().manual_seed(1)
    for _ in range(6):
        x, y = torch.randn(16, 5, generator=g), torch.randint(0, 3, (16,), generator=g)
        conn.pull(net)
        net.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        conn.push(net)
        conn.increment_global_step()                       # what Estimator.train does after every step
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(x), y).backward()
        opt.step()
    conn.pull(net)
    for (n, a), (_, b) in zip(net.named_parameters(), ref.named_parameters()):
        assert torch.allclose(a, b, atol=2e-6, rtol=1e-5), (n, (a - b).abs().max().item())
    assert conn.global_step() == 6 and set(conn.state_dict_from_ps(net)) == set(ref.state_dict())
    for s in shards:
        s.unlink()


def test_per_variable_optimizers_and_round_robin_placement(tmp_path):
    net = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    by_name = {"0.weight": keras.optimizers.Ftrl(0.05), "0.bias": keras.optimizers.Ftrl(0.05)}
    conn, shards = _connection(tmp_path, net, keras.optimizers.Adagrad(0.1), n_ps=3, by_name=by_name)
    lay = conn.layout
    assert lay.kinds == ["ftrl", "ftrl", "adagrad", "adagrad"] and lay.owner == [0, 1, 2, 0]
    assert lay.var_slots == [2, 2, 1, 1] and lay.shard_elems == [16 * 3 + 8 * 2, 8 * 3, 8 * 2]
    again = ps.Layout.from_json(lay.to_json())
    assert again.offset == lay.offset and again.hypers == lay.hypers
    assert shards[0].add_global_step(5) == 5 and shards[0].global_step() == 5
    for s in shards:
        s.unlink()


def test_hbm_shard_sizing_covers_master_slots_and_row_padded_shadows():
    """estimator/ps_hbm.py: every ps rank reserves `shard_bytes(layout)`; the fp32 area (master + optimizer slots) is
    followed by the bf16 shadows, 2-D ones with rows padded to 8 elements (16 bytes: what a TMA tensor map needs).
    For random layouts: regions never overlap, every shadow starts 16-byte aligned, and the reservation is enough."""
    import random
    from tf_yarn_b200.estimator import ps_hbm
    rnd = random.Random(0)
    hyper = {"lr": 0.1, "p1": 0, "p2": 0, "eps": 1e-7, "wd": 0, "init_s1": 0.1, "flags": 0}
    for trial in range(40):
        n_ps = rnd.choice([1, 2, 3])
        variables, kinds = [], []
        for i in range(rnd.randint(1, 12)):
            if rnd.random() < 0.6:
                shape = [rnd.randint(1, 70), rnd.choice([1, 3, 8, 13, 64, 429, 1024])]
            else:
                shape = [rnd.randint(1, 300)]
            variables.append((f"v{i}", shape))
            kinds.append(rnd.choice(["sgd", "adagrad", "adam", "ftrl"]))
        lay = ps.Layout(variables, n_ps, "adagrad", hyper, kinds=kinds, hypers=[hyper] * len(variables))
        conn = ps_hbm.HbmConnection.__new__(ps_hbm.HbmConnection)
        conn.layout = lay
        conn.ps_base = [0] * n_ps                                   # offsets relative to each rank's region
        reserved = ps_hbm.shard_bytes(lay)
        assert reserved % 4096 == 0
        spans = {p: [] for p in range(n_ps)}
        for i, (_, shape) in enumerate(variables):
            owner = lay.owner[i]
            for slot in range(1 + lay.var_slots[i]):
                a = conn.master_ptr(i, slot)
                spans[owner].append((a, a + 4 * lay.numel[i], f"v{i}/slot{slot}"))
            s0 = conn.shadow_ptr(i)
            ld = conn.shadow_ld(i)
            if len(shape) == 2:
                assert ld % 8 == 0 and ld >= shape[1] and s0 % 16 == 0
                nbytes = 2 * shape[0] * ld
            else:
                assert ld == 0
                nbytes = 2 * lay.numel[i]
            spans[owner].append((s0, s0 + nbytes, f"v{i}/shadow"))
        for p, regions in spans.items():
            regions.sort()
            for (a0, a1, na), (b0, b1, nb) in zip(regions, regions[1:]):
                assert a1 <= b0, (trial, na, nb, a1, b0)
            if regions:
                assert regions[-1][1] <= reserved, (trial, regions[-1], reserved)


def test_hbm_plane_classifies_variables_and_decides_the_fusions():
    """Which variables are served sparsely / streamed by the remote-weight GEMM / pulled, and when the embedding gather
    is fused into the first deep GEMM (K5) and the wide tower into the multi-table kernels -- decided from the network
    structure alone (estimator/ps_hbm.py)."""
    from tf_yarn_b200.estimator import canned, ps_hbm
    from tf_yarn_b200.estimator import feature_column as fc
    from tf_yarn_b200.models import wide_deep as wdm

    wide, deep = wdm.feature_columns(vocab=1000, emb_dim=64, n_cat=3, n_num=13)
    net = canned._WideDeepNet(wide, deep, [256, 64], 1)
    conn = hbm_connection(net)
    names = conn.names
    sparse = sorted(names[i] for i in conn.sparse)
    gemm = sorted(names[i] for i in conn.gemm)
    pulled = sorted(names[i] for i in conn.pull_idx)
    assert len(sparse) == 6 and all("embeddings" in n or "tables" in n for n in sparse)       # 3 deep + 3 wide tables
    assert gemm == ["hidden.0.weight", "hidden.1.weight"]                                      # out_features % 8 == 0
    assert "logits.weight" in pulled and all(n.endswith("bias") or "numeric" in n or n == "logits.weight" for n in pulled)
    assert ps_hbm._try_fuse_first_layer(conn, net) is True                                     # embeddings (64) then numeric
    assert ps_hbm._try_fuse_wide_tower(conn, net) is True

    # numeric columns BEFORE the embeddings: every embedding no longer starts at a multiple of 64 columns
    net2 = canned._WideDeepNet(wide, [deep[-1]] + deep[:-1], [256, 64], 1)
    assert ps_hbm._try_fuse_first_layer(hbm_connection(net2), net2) is False
    # embedding dimension 16: outside the fused kernel's row format
    wide3, deep3 = wdm.feature_columns(vocab=1000, emb_dim=16, n_cat=3, n_num=13)
    net3 = canned._WideDeepNet(wide3, deep3, [256, 64], 1)
    assert ps_hbm._try_fuse_first_layer(hbm_connection(net3), net3) is False
    # first hidden width not a multiple of 8: the layer is not served by the remote-weight GEMM at all
    net4 = canned._WideDeepNet(wide, deep, [100, 64], 1)
    conn4 = hbm_connection(net4)
    assert "hidden.0.weight" not in [conn4.names[i] for i in conn4.gemm]
    assert ps_hbm._try_fuse_first_layer(conn4, net4) is False
    # tables of different vocabulary sizes cannot share one multi-table launch
    cols = [fc.categorical_column_with_hash_bucket("a", 100), fc.categorical_column_with_hash_bucket("b", 200)]
    net5 = canned._WideDeepNet(cols, [], [], 1)
    assert ps_hbm._try_fuse_wide_tower(hbm_connection(net5), net5) is False
