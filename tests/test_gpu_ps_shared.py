"""The shared push tfy_ps_multi_push_rows_shared against the float64 reference (tests/shared_embedding_reference.py),
and the HBM plane's routing of shared embedding columns.

Tolerances are those of tests/test_gpu_ps_kernels.py: a row's error bound grows with the number of terms of its
folded sum, here counted over all the columns of its table.
"""
import numpy as np
import pytest
import torch

import multihot_reference as mh
import ps_reference as ref
import shared_embedding_reference as sref
from test_gpu_ps_kernels import HP, OPT_IDS, OPTS, STEPS, _grad_mag, _ids, _scratch, _stream, _Tables
from test_gpu_ps_multihot import CODES, _Spy, _multihot_batches, _weights

pytestmark = pytest.mark.gpu

MAPS = {"one_table": [0, 0, 0, 0], "pairs": [0, 0, 1, 1, 2, 2], "non_contiguous": [0, 1, 0, 2, 1],
        "identity": [0, 1, 2, 3]}


def _max_members(table_of):
    return max(table_of.count(k) for k in set(table_of))


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _spush(lib, tb, table_of, ids, w, f, combiner, dout, D, dout_ld, col_stride, adam, grad_scale=0.75):
    T, B, L = ids.shape
    sc = _scratch(lib, T * B * L)
    h = HP[tb.opt]
    idt = torch.from_numpy(np.ascontiguousarray(ids)).cuda()
    wt = torch.from_numpy(w).float().cuda() if w is not None else None
    ft = torch.from_numpy(f).float().cuda() if f is not None else None
    tmap = torch.tensor(table_of, dtype=torch.int32, device="cuda")
    rc = lib.tfy_ps_multi_push_rows_shared(
        tb.ptrs[0].data_ptr(), tb.s1.data_ptr() if tb.s1 is not None else None,
        tb.s2.data_ptr() if tb.s2 is not None else None, idt.data_ptr(), dout.data_ptr(),
        int(dout.dtype == torch.bfloat16), B, T, D, tb.state[0][0].shape[0], tb.opt, h["lr"], h["eps"], h["p1"],
        h["p2"], h["p3"], grad_scale, adam.data_ptr(), dout_ld, col_stride, L,
        wt.data_ptr() if wt is not None else None, ft.data_ptr() if ft is not None else None, CODES[combiner],
        max(table_of) + 1, tmap.data_ptr(), _max_members(table_of), sc.data_ptr(), sc.numel(), _stream())
    torch.cuda.current_stream().synchronize()
    return rc


# (D, col_stride, gradient dtype, dout_ld): deep column slices of a bf16 dx; one fp32 gradient for every column
CASES = {"deep_bf16": (64, 64, torch.bfloat16, 64 * 6 + 16), "stride0_fp32": (4, 0, torch.float32, 4),
         "scalar_fp32": (3, 3, torch.float32, 3 * 6 + 1)}


@pytest.mark.parametrize("L", [1, 3], ids=["L1_block_sort", "L3_device_sort"])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mapping", list(MAPS))
@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_shared_push_matches_reference(lib, opt, mapping, case, L):
    """Weighted multi-hot members (zero weights, out-of-range ids, heavy duplicates: runs far above kPsShortRun
    spread over several columns) and unweighted one-hot pushes, every distinct (table, row) folded once."""
    D, col_stride, gdtype, ld = CASES[case]
    table_of = MAPS[mapping]
    T, n, V = len(table_of), max(table_of) + 1, 80
    mm = _max_members(table_of)
    # L = 1: the block sort's limit of max_members * B * L = 2048 reached exactly; L = 3: one example past it
    B = 2048 // mm if L == 1 else 2048 // (mm * L) + 1
    for k, (weighted, combiner) in enumerate([(True, "sqrtn"), (False, "sum")]):
        rng = np.random.default_rng(opt * 1000 + len(mapping) * 10 + L + k)
        tb = _Tables(opt, n, V, D, rng)
        adam = torch.ones(2, dtype=torch.float32, device="cuda")
        counts = [np.zeros(V)] * n
        for step in range(STEPS):
            ids = _ids(rng, (T, B, L), V)
            w = _weights(rng, (T, B, L)) if weighted else None
            f = mh.factors(ids, w, V, combiner).astype(np.float32).astype(np.float64) if weighted else None
            counts = [np.maximum(a, b) for a, b in zip(counts, sref.row_counts(table_of, n, ids, w, V))]
            dout = torch.from_numpy(rng.standard_normal((B, ld)) * _grad_mag(opt)).to(gdtype).cuda()
            sc = tuple(float(np.float32(x)) for x in ref.adam_scale(step + 1, 0.9, 0.999))
            adam.copy_(torch.tensor(sc, dtype=torch.float32))
            sref.sparse_push(tb.opt, [s[0] for s in tb.state], [s[1] for s in tb.state], [s[2] for s in tb.state],
                             table_of, ids, w, f, dout.double().cpu().numpy(), D, HP[opt], grad_scale=0.75,
                             col_stride=col_stride, scale=sc)
            assert _spush(lib, tb, table_of, ids, w, f, combiner, dout, D, ld, col_stride, adam) == 0
        torch.cuda.synchronize()
        tb.check(counts, STEPS, what=(mapping, case, L, weighted))


@pytest.mark.parametrize("weighted", [True, False], ids=["weighted", "unweighted"])
@pytest.mark.parametrize("L", [1, 3])
def test_identity_map_is_bit_equal_to_the_unshared_push(lib, L, weighted):
    rng = np.random.default_rng(7 + L)
    T, V, B, D = 4, 60, 512, 64
    ids = _ids(rng, (T, B, L), V)
    w = _weights(rng, (T, B, L)) if weighted else None
    f = mh.factors(ids, w, V, "mean").astype(np.float32) if weighted else None
    dout = torch.from_numpy(rng.standard_normal((B, D * T)) * 0.5).to(torch.bfloat16).cuda()
    adam = torch.tensor(ref.adam_scale(1, 0.9, 0.999), dtype=torch.float32, device="cuda")
    results = []
    for shared in (True, False):
        tb = _Tables(ref.ADAM, T, V, D, np.random.default_rng(3))
        h = HP[ref.ADAM]
        if shared:
            assert _spush(lib, tb, list(range(T)), ids, w, f, "mean" if weighted else "sum", dout, D, D * T, D,
                          adam) == 0
        else:
            idt = torch.from_numpy(ids).cuda()
            sc = _scratch(lib, T * B * L)
            if weighted or L > 1:
                wt = torch.from_numpy(w).float().cuda() if weighted else None
                ft = torch.from_numpy(f).float().cuda() if weighted else None
                rc = lib.tfy_ps_multi_push_rows_weighted(
                    tb.ptrs[0].data_ptr(), tb.s1.data_ptr(), tb.s2.data_ptr(), idt.data_ptr(), dout.data_ptr(), 1, B, T,
                    D, V, ref.ADAM, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"], 0.75, adam.data_ptr(), D * T, D, L,
                    wt.data_ptr() if weighted else None, ft.data_ptr() if weighted else None, 1 if weighted else 0,
                    sc.data_ptr(), sc.numel(), _stream())
            else:
                rc = lib.tfy_ps_multi_push_rows(
                    tb.ptrs[0].data_ptr(), tb.s1.data_ptr(), tb.s2.data_ptr(), idt.data_ptr(), dout.data_ptr(), 1, B, T,
                    D, V, ref.ADAM, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"], 0.75, adam.data_ptr(), D * T, D,
                    sc.data_ptr(), sc.numel(), _stream())
            torch.cuda.synchronize()
            assert rc == 0
        results.append([b.t.clone() for bb in tb.bufs for b in bb])
    for a, b in zip(*results):
        assert torch.equal(a, b)


@pytest.mark.parametrize("L", [1, 3])
def test_shared_group_push_is_reproducible_and_captures_in_a_cuda_graph(lib, L):
    """_TableGroup.push of a weighted bag's batch in a group whose columns share tables ([0, 1, 0, 2, 1]): twice from
    the same state bit-identical, and a captured CUDA graph's replay equal to eager, on both sort paths."""
    from tf_yarn_b200.estimator import ps_hbm
    import types
    rng = np.random.default_rng(40 + L)
    table_of = MAPS["non_contiguous"]
    T, n, V, B, D = len(table_of), 3, 200, 512, 64
    tb = _Tables(ref.FTRL, n, V, D, rng)
    conn = types.SimpleNamespace(lib=lib, adam_scale=torch.ones(2, device="cuda"), account=lambda **k: None)
    group = ps_hbm._TableGroup.__new__(ps_hbm._TableGroup)
    h = HP[ref.FTRL]
    group.conn, group.hp, group.slots, group.V = conn, (ref.FTRL, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"]), 2, V
    group.D, group.col_stride, group.out_ld, group.one_table, group.parts = D, D, D * T, False, None
    group.idx, group.distinct, group.max_members = table_of, list(range(n)), _max_members(table_of)
    group.push_tables, group.push_s1, group.push_s2 = tb.ptrs
    group.table_of = torch.tensor(table_of, dtype=torch.int32, device="cuda")
    ids = torch.from_numpy(_ids(rng, (T, B, L), V)).cuda()
    w = torch.from_numpy(_weights(rng, (T, B, L))).float().cuda()
    f = torch.from_numpy(mh.factors(ids.cpu().numpy(), w.cpu().numpy(), V, "sqrtn")).float().cuda()
    dout = torch.from_numpy(rng.standard_normal((B, D * T)) * 0.5).to(torch.bfloat16).cuda()
    snap = tb.snapshot()

    def push():
        group.push(ids, dout, w, f, CODES["sqrtn"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        push()
    torch.cuda.current_stream().wait_stream(s)
    results = []
    for _ in range(2):
        tb.restore(snap)
        push()
        torch.cuda.synchronize()
        results.append([b.t.clone() for bb in tb.bufs for b in bb])
    for a, b in zip(*results):
        assert torch.equal(a, b)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        push()
    tb.restore(snap)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(results[0], [b.t for bb in tb.bufs for b in bb]):
        assert torch.equal(a, b)
    tb.restore(snap)
    push()
    torch.cuda.synchronize()
    idn, wn = ids.cpu().numpy(), w.cpu().numpy()
    sref.sparse_push(ref.FTRL, [s[0] for s in tb.state], [s[1] for s in tb.state], [s[2] for s in tb.state], table_of,
                     idn, wn, f.double().cpu().numpy(), dout.double().cpu().numpy(), D, HP[ref.FTRL], col_stride=D)
    tb.check(sref.row_counts(table_of, n, idn, wn, V), 1)


def test_shared_push_error_codes(lib):
    rng = np.random.default_rng(0)
    tb = _Tables(ref.ADAM, 1, 10, 4, rng)
    ids = torch.zeros(2, 8, 1, dtype=torch.int64, device="cuda")
    dout = torch.zeros(8, 8, device="cuda")
    tmap = torch.zeros(2, dtype=torch.int32, device="cuda")
    sc = _scratch(lib, 16)
    p = [x.data_ptr() for x in tb.ptrs]

    def call(n_tables=1, table_of=tmap.data_ptr(), max_members=2, opt=ref.ADAM, s2=p[2], combiner=0):
        return lib.tfy_ps_multi_push_rows_shared(
            p[0], p[1], s2, ids.data_ptr(), dout.data_ptr(), 0, 8, 2, 4, 10, opt, 0.1, 1e-7, 0.9, 0.999, 0.0, 1.0, None,
            8, 4, 1, None, None, combiner, n_tables, table_of, max_members, sc.data_ptr(), sc.numel(), _stream())
    snap = tb.snapshot()
    assert call(n_tables=0) == -2 and call(n_tables=3) == -2 and call(table_of=None) == -2
    assert call(max_members=0) == -2 and call(max_members=3) == -2       # 1 <= max_members <= T - n_tables + 1
    assert call(opt=99) == -3 and call(s2=None) == -4 and call(combiner=1) == -4
    torch.cuda.synchronize()
    for a, b in zip([x for xx in snap for x in xx], [b.t for bb in tb.bufs for b in bb]):
        assert torch.equal(a, b)


def test_thirteen_pairs_at_batch_512_take_the_block_sort(lib):
    """26 deep columns as 13 shared pairs (column i with column i + 13) at B = 512: 2 * 512 occurrences per table,
    so one block sort launch per push, no key kernel and no device radix sort, and the result of the reference."""
    table_of = list(range(13)) * 2
    T, n, V, B, D = 26, 13, 100, 512, 64
    rng = np.random.default_rng(11)
    tb = _Tables(ref.ADAGRAD, n, V, D, rng)
    ids = _ids(rng, (T, B, 1), V)
    dout = torch.from_numpy(rng.standard_normal((B, D * T + 16)) * 0.5).to(torch.bfloat16).cuda()
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    sref.sparse_push(ref.ADAGRAD, [s[0] for s in tb.state], [s[1] for s in tb.state], [s[2] for s in tb.state],
                     table_of, ids, None, None, dout.double().cpu().numpy(), D, HP[ref.ADAGRAD], grad_scale=0.75,
                     col_stride=D)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert _spush(lib, tb, table_of, ids, None, None, "sum", dout, D, D * T + 16, D, adam) == 0
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert sum("tfy_ps_segment_sort_kernel<false, true>" in k for k in names) == 1, names
    assert not any("row_keys" in k or "RadixSort" in k for k in names), names
    from tf_yarn_b200.estimator import ps_hbm
    assert ps_hbm.push_rows_launches(B, _max_members(table_of)) == 4         # block sort, offsets, two applies
    tb.check(sref.row_counts(table_of, n, ids, None, V), 1)


# ---------------------------------------------------------------------------------------------- end to end
def _shared_columns(V, n_num, weighted):
    """Four categorical columns in two shared collections of two (64 wide, as K5 takes them), then a numeric one."""
    from tf_yarn_b200.estimator import feature_column as fc
    cats = [fc.categorical_column_with_hash_bucket(f"c{i}", V) for i in range(4)]
    if weighted:
        cats = [fc.weighted_categorical_column(c, f"w{i}") for i, c in enumerate(cats)]
    deep = fc.shared_embedding_columns([cats[0], cats[2]], 64, combiner="sqrtn")
    deep += fc.shared_embedding_columns([cats[1], cats[3]], 64, combiner="sqrtn")
    deep = [deep[0], deep[2], deep[1], deep[3]] + [fc.numeric_column("num", (n_num,))]   # members not adjacent
    return cats, deep


def _train_both(tmp_path, net_cpu, batches, fused_first, optimizers=None):
    """test_gpu_ps_multihot._train_both, with K5 expected or not and optimizers by variable name: relative errors of
    the HBM plane's updates against the CPU plane's, the native calls of the HBM steps, the HBM plane's launches per
    step, and every launch count the connection accounted with the native call it followed."""
    import copy
    import types

    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import ps, ps_hbm
    net = copy.deepcopy(net_cpu).cuda()
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001, l2_regularization_strength=0.01)
    by_name = {n: ftrl for n, _ in named if n.startswith("linear.")}
    by_name.update(optimizers or {})
    layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05), by_name)
    region = torch.zeros(ps_hbm.shard_bytes(layout) // 4, dtype=torch.float32, device="cuda")
    comm = types.SimpleNamespace(arena=types.SimpleNamespace(peer_base={0: region.data_ptr()}), device=0)
    header = ps.ShmShard(str(tmp_path / "header"), 8, create=True)
    shards = [ps.ShmShard(str(tmp_path / "shard0"), layout.shard_elems[0], create=True)]
    try:
        conn = ps_hbm.HbmConnection(layout, comm, {"ps:0": 0}, 0, [n for n, _ in named], header, net)
        conn.lib = spy = _Spy(conn.lib)
        accounted = []
        account = conn.account

        def attributed(**k):
            accounted.append((spy.calls[-1] if spy.calls else None, k.get("launches", 1)))
            account(**k)
        conn.account = attributed
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
        assert conn.fused_first == fused_first and conn.fused_wide
        assert conn.shared_collections == (0 if fused_first else 2)
        w0 = [[cpu._region(i, s).double().clone() for s in range(1 + layout.var_slots[i])] for i in range(len(named))]
        launches = []
        for feats, y in batches:
            for model, plane, dev in ((net, conn, "cuda"), (net_cpu, cpu, "cpu")):
                f = {k: v.to(dev) for k, v in feats.items()}
                plane.pull(model)
                model.zero_grad()
                out = model(f).float()
                torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y.to(dev).float()).backward()
                plane.push(model)
                plane.increment_global_step()
            launches.append(conn.traffic_per_step()["launches_per_step"])
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
        return rels, spy.calls, launches, accounted
    finally:
        header.unlink()
        shards[0].unlink()


@pytest.mark.parametrize("fuse_first", ["1", "0"], ids=["k5", "unfused"])
@pytest.mark.parametrize("weighted", [False, True], ids=["one_hot", "weighted_multihot"])
def test_hbm_and_cpu_planes_train_a_shared_wide_and_deep_network_alike(tmp_path, monkeypatch, fuse_first, weighted):
    """Three steps of a wide-and-deep network whose deep tower holds two shared collections, on both planes, with the
    bounds and reasoning of test_hbm_and_cpu_planes_train_a_wide_and_deep_network_alike (bf16 GEMMs and a bf16 dx: a
    few 1e-2 relative; pushing a shared table once per member, or an addressing fault, is of order 1).  Each shared
    table is pushed once per step, by K5's backward or by the collection's own bag."""
    from tf_yarn_b200.estimator import canned
    monkeypatch.setenv("TFY_PS_FUSE_FIRST", fuse_first)
    torch.manual_seed(0)
    V, B, n_num = 40, 256, 5
    wide, deep = _shared_columns(V, n_num, weighted)
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1, sparse_combiner="mean")
    batches = _multihot_batches(B, 3, V, 4, n_num, 3 if weighted else 1, seed=5)
    if not weighted:
        batches = [({k: (v[:, 0].clamp(min=0) if k.startswith("c") else v) for k, v in f.items()
                     if not k.startswith("w")}, y) for f, y in batches]
    rels, calls, launches, accounted = _train_both(tmp_path, net_cpu, batches, fused_first=fuse_first == "1")
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    # K5: one push for both shared tables of the first layer; unfused: one bag and one push per collection
    pushes = 1 if fuse_first == "1" else 2
    assert calls.count("tfy_ps_multi_push_rows_shared") == 3 * pushes
    assert "tfy_ps_embedding_bag" not in calls and "tfy_ps_push_rows" not in calls
    if fuse_first == "0":
        assert "tfy_ps_gather_gemm" not in calls
        # the collections' bags plus the wide tower's (its mean combiner takes the weighted bag)
        assert calls.count("tfy_ps_multi_bag_weighted") == 3 * 2 + 3
    # the launches accounted for the shared pushes: each its block sort (2 members * B * L <= 2048), offsets and
    # two applies; every step accounts the same launches
    from tf_yarn_b200.estimator import ps_hbm
    L = 3 if weighted else 1
    shared = [n for c, n in accounted if c == "tfy_ps_multi_push_rows_shared"]
    assert shared == [ps_hbm.push_rows_launches(B * L, 2)] * (3 * pushes) == [4] * (3 * pushes)
    assert launches == [launches[0]] * 3 and launches[0] == sum(n for _, n in accounted) // 3


@pytest.mark.parametrize("weighted", [False, True], ids=["one_hot", "weighted_multihot"])
def test_k5_pushes_shared_tables_of_mixed_optimizers_table_by_table(tmp_path, weighted):
    """K5 over two shared collections whose tables have different optimizers (SGD and Adagrad): the group is not
    uniform, so each shared table is pushed by itself, from its members' dx slices put side by side (members 0 and
    2, 1 and 3 of the first layer), and the HBM plane trains like the CPU plane (bounds as above)."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_num = 40, 256, 5
    wide, deep = _shared_columns(V, n_num, weighted)
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1, sparse_combiner="mean")
    batches = _multihot_batches(B, 3, V, 4, n_num, 3 if weighted else 1, seed=6)
    if not weighted:
        batches = [({k: (v[:, 0].clamp(min=0) if k.startswith("c") else v) for k, v in f.items()
                     if not k.startswith("w")}, y) for f, y in batches]
    sgd = {"dense_features.embeddings.c0_c2_shared_embedding.weight": keras.optimizers.SGD(0.1)}
    rels, calls, _, accounted = _train_both(tmp_path, net_cpu, batches, fused_first=True, optimizers=sgd)
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert "dense_features.embeddings.c0_c2_shared_embedding.weight/0" in rels
    assert calls.count("tfy_ps_multi_push_rows_shared") == 3 * 2                # one push per shared table per step
    assert "tfy_ps_push_rows" not in calls
