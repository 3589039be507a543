"""Weighted multi-hot HBM kernels (tfy_ps_multi_bag_weighted, tfy_ps_multi_push_rows_weighted) against the float64
reference (tests/multihot_reference.py), and the HBM plane's routing of multi-hot / weighted batches.

Tolerances follow tests/test_gpu_ps_kernels.py.  The weights are drawn from small dyadic values (0, +-0.25, 0.5, 1,
1.5, 2), so sum(w) and sum(w^2) are exact in fp32: den is exact for sum and mean and one rounding off for sqrtn, and the
bag's error is that of an fp32 sum of L weighted terms, at most (L + 3) EPS32 sum_j |w_j| |row_j| / |den| per column.
The push adds w f g per occurrence: one more rounding per term than the unweighted fold, covered by the (R + 1) factor.
"""
import types

import numpy as np
import pytest
import torch

import multihot_reference as mh
import ps_reference as ref
from test_gpu_ps_kernels import HP, OPT_IDS, OPTS, STEPS, _Guarded, _grad_mag, _ids, _scratch, _stream, _Tables

pytestmark = pytest.mark.gpu

CODES = {"sum": 0, "mean": 1, "sqrtn": 2}
WVALS = np.array([0.0, 0.25, -0.25, 0.5, 1.0, 1.5, 2.0])


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _weights(rng, shape):
    w = WVALS[rng.integers(0, len(WVALS), size=shape)]
    if shape[-1] >= 2:                 # examples whose weights cancel (sum 0 with present ids: mean gives 0)
        w[..., 2, :] = 0.0
        w[..., 2, 0], w[..., 2, 1] = 0.5, -0.5
    return w


def _special_rows(ids, w):
    """Example 0: every id missing; example 1: every weight zero."""
    ids[..., 0, :] = -1
    if w is not None:
        w[..., 1, :] = 0.0


def _bag(lib, tables, ids, w, combiner, D, V, out, out_ld, col_stride, numeric=None):
    T, B, L = ids.shape
    ptrs = torch.tensor([t.ptr() for t in tables], dtype=torch.int64, device="cuda")
    idt = torch.from_numpy(ids).cuda()
    wt = torch.from_numpy(w).float().cuda() if w is not None else None
    f = torch.full((T, B), -3.0, device="cuda")
    nt = torch.from_numpy(numeric).float().cuda() if numeric is not None else None
    rc = lib.tfy_ps_multi_bag_weighted(ptrs.data_ptr(), idt.data_ptr(), wt.data_ptr() if wt is not None else None,
                                       CODES[combiner], B, L, T, D, V, out.data_ptr(), int(out.dtype == torch.bfloat16),
                                       out_ld, col_stride, nt.data_ptr() if nt is not None else None,
                                       numeric.shape[1] if numeric is not None else 0, f.data_ptr(), _stream())
    torch.cuda.synchronize()
    return rc, f.double().cpu().numpy()


def _check_bag(lib, T, L, D, combiner, weighted, odtype, col_stride, B=40, V=50, seed=0):
    rng = np.random.default_rng(seed)
    host = [rng.standard_normal((V, D)) for _ in range(T)]
    tables = [_Guarded(h) for h in host]
    host = [t.get() for t in tables]
    ids = _ids(rng, (T, B, L), V)
    w = _weights(rng, (T, B, L)) if weighted else None
    _special_rows(ids, w)
    n_num = 3 if col_stride == D else 0
    numeric = rng.standard_normal((B, n_num)) if n_num else None
    width = ((T - 1) * col_stride + D if col_stride else D) + n_num
    out_ld = width + 5                                          # pad columns after the written ones
    out = torch.full((B, out_ld), 7.0, dtype=odtype, device="cuda")
    rc, f = _bag(lib, tables, ids, w, combiner, D, V, out, out_ld, col_stride, numeric)
    assert rc == 0
    got = out.double().cpu().numpy()
    want = mh.multi_bag(host, ids, w, combiner, col_stride)
    fr = mh.factors(ids, w, V, combiner)
    absw = None if w is None else np.abs(w)
    parts = [mh.bag(np.abs(host[t]), ids[t], None if absw is None else absw[t], "sum") * np.abs(fr[t])[:, None]
             for t in range(T)]
    mag = sum(parts) if col_stride == 0 else np.zeros_like(want)
    for t in range(T if col_stride else 0):
        mag[:, t * col_stride:t * col_stride + D] = parts[t]
    nb = want.shape[1]
    tol = (T * L + 4) * ref.EPS32 * mag + (2.0 ** -8 * np.abs(want) if odtype == torch.bfloat16 else 0)
    cols = np.zeros(nb, bool)                    # the written columns: D per table; a wider stride leaves gaps
    for t in range(T if col_stride else 1):
        cols[t * col_stride:t * col_stride + D] = True
    assert np.all(np.abs(got[:, :nb] - want)[:, cols] <= tol[:, cols] + 1e-30), (T, L, D, combiner, weighted,
                                                                                  col_stride)
    assert np.all(got[:, :nb][:, ~cols] == 7.0), "gap columns between table slices written"
    if n_num:
        nw = ref.bf16_round(numeric) if odtype == torch.bfloat16 else numeric.astype(np.float32)
        assert np.array_equal(got[:, T * D:T * D + n_num], nw)
    assert np.all(got[:, width:] == 7.0), "pad columns written"
    assert np.all(got[0, :nb][cols] == 0.0), "an example without a present id must give 0"
    np.testing.assert_allclose(f, fr, rtol=4 * ref.EPS32, atol=0)     # den exact; sqrt and 1/den rounded once


@pytest.mark.parametrize("combiner", mh.COMBINERS)
@pytest.mark.parametrize("D", [1, 3, 4, 64, 65])
@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("T", [1, 3, 26])
def test_weighted_bag_matches_reference(lib, T, L, D, combiner):
    for k, (weighted, odtype, cs) in enumerate([(w, o, c) for w in (False, True)
                                                for o in (torch.float32, torch.bfloat16) for c in (0, D)]):
        _check_bag(lib, T, L, D, combiner, weighted, odtype, cs, seed=T * 1000 + L * 100 + D + k)


def test_weighted_bag_unaligned_output_takes_the_scalar_path(lib):
    """D % 4 == 0 but an odd pitch, or a column stride that breaks 16-byte stores."""
    _check_bag(lib, 3, 3, 64, "sqrtn", True, torch.float32, 67)
    _check_bag(lib, 3, 3, 4, "mean", True, torch.bfloat16, 6)


def test_weighted_bag_grid_stride_wrap(lib):
    """B * T * D / 4 = 960,000 threads' worth of work > 132*8 blocks x 256 threads: the loop wraps."""
    _check_bag(lib, 3, 2, 64, "mean", True, torch.float32, 64, B=20_000, V=1000)


def test_weighted_bag_error_codes(lib):
    t = [_Guarded(np.zeros((10, 4)))]
    ids = np.zeros((1, 8, 2), np.int64)
    out = torch.zeros(8, 64, device="cuda")

    def call(combiner=0, L=2, out_ld=64, cs=0, n_num=0, D=4):
        ptrs = torch.tensor([x.ptr() for x in t], dtype=torch.int64, device="cuda")
        idt = torch.from_numpy(ids).cuda()
        num = torch.zeros(8, 64, device="cuda")
        f = torch.zeros(1, 8, device="cuda")
        return lib.tfy_ps_multi_bag_weighted(ptrs.data_ptr(), idt.data_ptr(), None, combiner, 8, L, 1, D, 10,
                                             out.data_ptr(), 0, out_ld, cs, num.data_ptr(), n_num, f.data_ptr(),
                                             _stream())
    assert call() == 0
    assert call(combiner=3) == -2 and call(combiner=-1) == -2 and call(L=0) == -2
    assert call(out_ld=3) == -2 and call(cs=2) == -2                   # pitch / stride narrower than a row
    assert call(n_num=3) == -2 and call(cs=4, n_num=65) == -2           # numeric needs col_stride == D, n_num <= 64
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- push
def _wpush(lib, tb, ids, w, f, combiner, dout, D, dout_ld, col_stride, adam, grad_scale=0.75):
    T, B, L = ids.shape
    sc = _scratch(lib, T * B * L)
    h = HP[tb.opt]
    idt = torch.from_numpy(np.ascontiguousarray(ids)).cuda()
    wt = torch.from_numpy(w).float().cuda() if w is not None else None
    ft = torch.from_numpy(f).float().cuda() if f is not None else None
    rc = lib.tfy_ps_multi_push_rows_weighted(
        tb.ptrs[0].data_ptr(), tb.s1.data_ptr() if tb.s1 is not None else None,
        tb.s2.data_ptr() if tb.s2 is not None else None, idt.data_ptr(), dout.data_ptr(),
        int(dout.dtype == torch.bfloat16), B, T, D, tb.state[0][0].shape[0], tb.opt, h["lr"], h["eps"], h["p1"],
        h["p2"], h["p3"], grad_scale, adam.data_ptr(), dout_ld, col_stride, L,
        wt.data_ptr() if wt is not None else None, ft.data_ptr() if ft is not None else None, CODES[combiner],
        sc.data_ptr(), sc.numel(), _stream())
    torch.cuda.current_stream().synchronize()       # keep ids, weights and the scratch alive until the push ran
    return rc


def _ref_wpush(tb, ids, w, f, dout, D, col_stride, sc, grad_scale=0.75):
    mh.sparse_push(tb.opt, [s[0] for s in tb.state], [s[1] for s in tb.state], [s[2] for s in tb.state], ids, w, f,
                   dout, D, HP[tb.opt], grad_scale=grad_scale, col_stride=col_stride, scale=sc)


# deep tower: D = 64 column slices of a bf16 dx with pitch Kp; wide tower: [V, 1] tables, one fp32 gradient for all
# (col_stride 0); a scalar-path layout (D = 3)
CASES = {"deep": (64, 64, torch.bfloat16, 64 * 6 + 16), "wide": (1, 0, torch.float32, 1),
         "scalar": (3, 3, torch.float32, 3 * 6 + 1)}
# (weighted, combiner, f given): unweighted sum may pass f = nullptr
VARIANTS = [(True, "sqrtn", True), (True, "mean", True), (False, "sum", False), (False, "mean", True)]


@pytest.mark.parametrize("L", [1, 3, 5], ids=["L1", "L3_block_sort", "L5_device_sort"])     # B*L = 512, 1536, 2560
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_weighted_push_matches_reference(lib, opt, case, L):
    D, col_stride, gdtype, ld = CASES[case]
    T, V, B = 6, 80, 512
    for k, (weighted, combiner, give_f) in enumerate(VARIANTS):
        rng = np.random.default_rng(opt * 100 + D * 10 + L + k)
        tb = _Tables(opt, T, V, D, rng)
        adam = torch.ones(2, dtype=torch.float32, device="cuda")
        counts = np.zeros((T, V))
        for step in range(STEPS):
            ids = _ids(rng, (T, B, L), V)                       # heavy duplicates: runs far above 32
            if L > 1:
                ids[:, ::7, 1] = ids[:, ::7, 0]                 # repeats inside one example, with other weights
            w = _weights(rng, (T, B, L)) if weighted else None
            f = mh.factors(ids, w, V, combiner).astype(np.float32).astype(np.float64) if give_f else None
            counts = np.maximum(counts, mh.row_counts(ids, w, V))
            dout = torch.from_numpy(rng.standard_normal((B, ld)) * _grad_mag(opt)).to(gdtype).cuda()
            sc = tuple(float(np.float32(x)) for x in ref.adam_scale(step + 1, 0.9, 0.999))
            adam.copy_(torch.tensor(sc, dtype=torch.float32))
            _ref_wpush(tb, ids, w, f, dout.double().cpu().numpy(), D, col_stride, sc)
            assert _wpush(lib, tb, ids, w, f, combiner, dout, D, ld, col_stride, adam) == 0
        torch.cuda.synchronize()
        tb.check(counts, STEPS, what=(case, L, weighted, combiner))


def test_weighted_push_run_lengths_around_the_short_run_limit(lib):
    """Runs of 1, 31, 32, 33 and 64 present occurrences, each with different weights, plus zero-weight occurrences
    of the same rows that must not count: the first three are applied by per-run threads, the last two by a warp."""
    V, D = 16, 4
    lengths = {0: 1, 3: 31, 5: 32, 7: 33, 9: 64, 12: 2}
    present = np.concatenate([np.full(n, i) for i, n in lengths.items()])
    rng = np.random.default_rng(0)
    rng.shuffle(present)
    B = present.size
    ids = np.stack([present, rng.integers(0, V, B)], axis=1)[None]        # [1, B, 2]
    w = np.stack([WVALS[rng.integers(3, len(WVALS), B)], np.zeros(B)], axis=1)[None]
    f = mh.factors(ids, w, V, "mean").astype(np.float32).astype(np.float64)
    tb = _Tables(ref.ADAGRAD, 1, V, D, np.random.default_rng(1))
    dout = torch.from_numpy(rng.standard_normal((B, D)) * 0.5).float().cuda()
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    _ref_wpush(tb, ids, w, f, dout.double().cpu().numpy(), D, 0, (1.0, 1.0))
    assert _wpush(lib, tb, ids, w, f, "mean", dout, D, D, 0, adam) == 0
    tb.check(mh.row_counts(ids, w, V), 1)


def test_zero_weight_rows_leave_adam_slots_untouched(lib):
    """Lazy Adam: a row whose every occurrence has weight 0 (or an out-of-range id) keeps w, m and v bit for bit,
    while rows with a present occurrence move."""
    rng = np.random.default_rng(4)
    T, V, B, L, D = 2, 30, 300, 3, 4
    tb = _Tables(ref.ADAM, T, V, D, rng)
    for bb in tb.bufs:                                     # non-zero m, v so that a decay would show
        for k in (1, 2):
            bb[k].t.copy_(torch.rand_like(bb[k].t) * 1e-3)
    before = [[b.t.clone() for b in bb] for bb in tb.bufs]
    ids = rng.integers(0, V, (T, B, L))
    w = _weights(rng, (T, B, L))
    zero_rows = [3, 17]
    for r in zero_rows:
        w[ids == r] = 0.0
    f = mh.factors(ids, w, V, "sqrtn").astype(np.float32)
    dout = torch.from_numpy(rng.standard_normal((B, D * T)) * 1e-4).float().cuda()
    adam = torch.tensor(ref.adam_scale(1, 0.9, 0.999), dtype=torch.float32, device="cuda")
    assert _wpush(lib, tb, ids, w, f.astype(np.float64), "sqrtn", dout, D, D * T, D, adam) == 0
    torch.cuda.synchronize()
    touched = mh.row_counts(ids, w, V)
    for t in range(T):
        for k in range(3):
            a, b = before[t][k], tb.bufs[t][k].t
            for r in zero_rows:
                assert touched[t][r] == 0 and torch.equal(a[r], b[r]), (t, k, r)
            assert not torch.equal(a, b)


def test_weighted_push_error_codes(lib):
    rng = np.random.default_rng(0)
    tb = _Tables(ref.ADAM, 1, 10, 4, rng)
    ids = torch.zeros(8, 2, dtype=torch.int64, device="cuda")
    w = torch.ones(8, 2, device="cuda")
    f = torch.ones(8, device="cuda")
    dout = torch.zeros(8, 4, device="cuda")
    sc = _scratch(lib, 16)
    p = [x.data_ptr() for x in tb.ptrs]

    def call(opt=ref.ADAM, s1=p[1], s2=p[2], L=2, fp=f.data_ptr(), combiner=1, scratch=sc):
        return lib.tfy_ps_multi_push_rows_weighted(
            p[0], s1, s2, ids.data_ptr(), dout.data_ptr(), 0, 8, 1, 4, 10, opt, 0.1, 1e-7, 0.9, 0.999, 0.0, 1.0, None,
            0, 0, L, w.data_ptr(), fp, combiner, scratch.data_ptr() if scratch is not None else None,
            scratch.numel() if scratch is not None else 0, _stream())
    snap = tb.snapshot()
    assert call(L=0) == -2 and call(combiner=3) == -2 and call(combiner=-1) == -2
    assert call(opt=1) == -3 and call(opt=99) == -3
    assert call(s1=None) == -4 and call(s2=None) == -4 and call(opt=ref.FTRL, s2=None) == -4
    assert call(fp=None) == -4 and call(fp=None, combiner=2) == -4           # f may be omitted only for sum
    assert call(scratch=None) == -5
    torch.cuda.synchronize()
    for a, b in zip([x for xx in snap for x in xx], [b.t for bb in tb.bufs for b in bb]):
        assert torch.equal(a, b)                                            # nothing was applied


def _group(lib, tb, T, V, D, opt):
    from tf_yarn_b200.estimator import ps_hbm
    conn = types.SimpleNamespace(lib=lib, adam_scale=torch.ones(2, device="cuda"), account=lambda **k: None)
    group = ps_hbm._TableGroup.__new__(ps_hbm._TableGroup)
    group.conn, group.idx, group.tables, group.s1, group.s2 = conn, list(range(T)), tb.ptrs[0], tb.s1, tb.s2
    h = HP[opt]
    group.V, group.hp, group.slots = V, (opt, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"]), 2
    group.D, group.col_stride, group.one_table, group.parts = D, D, False, None
    group.out_ld = D * T
    return group


@pytest.mark.parametrize("opt", [ref.ADAM, ref.FTRL], ids=["adam", "ftrl"])
def test_weighted_group_push_is_reproducible_and_captures_in_a_cuda_graph(lib, opt):
    """_TableGroup.push of a weighted bag's batch twice from the same state gives bit-identical tables and slots, and
    the same push captured with torch.cuda.graph and replayed matches it bit for bit: no host synchronisation in the fold, on
    both sort paths (B*L = 1536 and 2560)."""
    rng = np.random.default_rng(21 + opt)
    T, V, B, D = 4, 200, 512, 64
    for L in (3, 5):
        tb = _Tables(opt, T, V, D, rng)
        group = _group(lib, tb, T, V, D, opt)
        ids = torch.from_numpy(_ids(rng, (T, B, L), V)).cuda()
        w = torch.from_numpy(_weights(rng, (T, B, L))).float().cuda()
        f = torch.from_numpy(mh.factors(ids.cpu().numpy(), w.cpu().numpy(), V, "sqrtn")).float().cuda()
        dout = torch.from_numpy(rng.standard_normal((B, D * T)) * _grad_mag(opt)).to(torch.bfloat16).cuda()
        snap = tb.snapshot()

        def push():
            group.push(ids, dout, w, f, CODES["sqrtn"])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                          # warm-up off the capture stream, as torch recommends
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
        _ref_wpush(tb, idn, wn, f.double().cpu().numpy(), dout.double().cpu().numpy(), D, D,
                   (1.0, 1.0), grad_scale=1.0)
        tb.check(mh.row_counts(idn, wn, V), 1)


# ---------------------------------------------------------------------------------------------- end to end
class _Spy:
    """The native library, recording which entry points a step called."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name.startswith("tfy_"):
            def rec(*a):
                self.calls.append(name)
                return fn(*a)
            return rec
        return fn


def _multihot_batches(B, n, V, n_cat, n_num, L, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        feats = {}
        for i in range(n_cat):
            ids = torch.randint(0, V, (B, L), generator=g)
            ids[torch.rand(B, L, generator=g) < 0.25] = -1              # ragged lists padded with -1
            feats[f"c{i}"] = ids
            feats[f"w{i}"] = torch.randint(0, 5, (B, L), generator=g).float() * 0.5      # some zero weights
        feats["num"] = torch.randn(B, n_num, generator=g)
        y = ((feats["c0"] % 2 == 0) & (feats["c0"] >= 0)).any(1).long()
        out.append((feats, y))
    return out


def _columns(V, n_cat, n_num, weighted, combiners=("sqrtn",)):
    from tf_yarn_b200.estimator import feature_column as fc
    cats = [fc.categorical_column_with_hash_bucket(f"c{i}", V) for i in range(n_cat)]
    if weighted:
        cats = [fc.weighted_categorical_column(c, f"w{i}") for i, c in enumerate(cats)]
    deep = [fc.embedding_column(c, 64, combiner=combiners[i % len(combiners)]) for i, c in enumerate(cats)]
    deep += [fc.numeric_column("num", (n_num,))]
    return cats, deep


def _train_both(tmp_path, net_cpu, batches):
    import copy

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
                out = model(f).float()
                torch.nn.functional.binary_cross_entropy_with_logits(out[:, 0], y.to(dev).float()).backward()
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


def test_hbm_and_cpu_planes_train_a_multihot_weighted_network_alike(tmp_path):
    """Three steps of a wide-and-deep network whose categorical columns are weighted multi-hot lists (L = 3, padded
    with -1, some zero weights): sqrtn embedding columns in the deep tower, a mean sparse combiner in the wide tower,
    FTRL and Adagrad.  The HBM plane takes the weighted bag + remote-weight GEMM for the first layer and the weighted
    wide tower; the CPU plane computes the contract in torch.  Bounds as in test_gpu_ps_kernels.py's wide-and-deep
    test (bf16 GEMMs and a bf16 dx: a few 1e-2 relative; an addressing or weighting fault is of order 1)."""
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = _columns(V, n_cat, n_num, weighted=True)
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1, sparse_combiner="mean")
    rels, calls = _train_both(tmp_path, net_cpu, _multihot_batches(B, 3, V, n_cat, n_num, 3, seed=1))
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert "tfy_ps_gather_gemm" not in calls and "tfy_ps_multi_bag" not in calls
    assert calls.count("tfy_ps_multi_bag_weighted") == 6 and calls.count("tfy_ps_multi_push_rows_weighted") == 6


def test_one_hot_batches_keep_k5_and_the_multi_table_wide_tower(tmp_path):
    """The same (unweighted) columns fed one id per example still take K5 and tfy_ps_multi_bag / multi_push_rows."""
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = _columns(V, n_cat, n_num, weighted=False)
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1)
    batches = [({k: (v[:, 0].clamp(min=0) if k.startswith("c") else v) for k, v in f.items() if not k.startswith("w")},
                y) for f, y in _multihot_batches(B, 3, V, n_cat, n_num, 1, seed=2)]
    rels, calls = _train_both(tmp_path, net_cpu, batches)
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert calls.count("tfy_ps_gather_gemm") == 3 and calls.count("tfy_ps_multi_bag") == 3
    assert "tfy_ps_multi_bag_weighted" not in calls and "tfy_ps_multi_push_rows_weighted" not in calls


def test_mixed_deep_combiners_are_gathered_table_by_table(tmp_path):
    """Deep embedding columns with different combiners (sqrtn, mean, sum) on weighted multi-hot batches: the first
    layer stays fused, the bag runs once per table (the push once for all, f carrying each table's 1/den), and the
    HBM plane trains like the CPU plane (bounds as above)."""
    from tf_yarn_b200.estimator import canned
    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = _columns(V, n_cat, n_num, weighted=True, combiners=("sqrtn", "mean", "sum"))
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1, sparse_combiner="sqrtn")
    rels, calls = _train_both(tmp_path, net_cpu, _multihot_batches(B, 3, V, n_cat, n_num, 3, seed=3))
    assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    assert calls.count("tfy_ps_multi_bag_weighted") == 3 * (n_cat + 1)          # per deep table, plus the wide tower
    assert calls.count("tfy_ps_multi_push_rows_weighted") == 6
