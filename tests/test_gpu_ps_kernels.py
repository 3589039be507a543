"""HBM parameter-server kernels (ops/csrc/tfy_ps.cu) against the float64 reference (tests/ps_reference.py).

One GPU: local device buffers stand in for the peer shard (the kernels only see addresses).  Every push runs several
times in a row so that the optimizer state builds up.

Tolerances.  The kernels compute in fp32; the reference in float64.  An element's update takes a handful of fp32
roundings per step (relative EPS32 each) on values of order |w| + |the accumulated update|, so after `steps` pushes its
error is below ROUNDINGS * steps * EPS32 * (|w| + |w - w0| + max|w - w0|): the last term is the norm-wise size of
the updates, whose own roundings do not shrink where w passes through 0.  A row that occurs R times in a sparse push gets a gradient
summed from R fp32 terms, which adds at most R * EPS32 * sum|g| to the gradient: the row's bound is scaled by (R + 1),
with R the row's largest count in any one push (the `steps` factor already covers the pushes).
Every defect these tests target -- a duplicate applied once per occurrence, a lost Adam update, epsilon in the wrong
place (|g| ~ 1e-4 with eps = 1e-7 moves the first step by several percent) -- is orders of magnitude above that.
"""
import types

import numpy as np
import pytest
import torch

import ps_reference as ref

pytestmark = pytest.mark.gpu

ROUNDINGS = 16
G = 3                      # guard rows before and after every table, checked to stay untouched
HP = {ref.SGD: dict(lr=0.1, eps=0.0, p1=0.0, p2=0.0, p3=0.0),
      ref.ADAGRAD: dict(lr=0.1, eps=1e-7, p1=0.0, p2=0.0, p3=0.0),
      ref.ADAM: dict(lr=0.01, eps=1e-7, p1=0.9, p2=0.999, p3=0.0),
      ref.FTRL: dict(lr=0.05, eps=0.0, p1=0.02, p2=0.01, p3=0.5)}
OPTS = [ref.SGD, ref.ADAGRAD, ref.ADAM, ref.FTRL]
OPT_IDS = ["sgd", "adagrad", "adam", "ftrl"]
INIT_S1 = 0.1
STEPS = 3


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.estimator import ps_hbm  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _grad_mag(opt):
    return 1e-4 if opt == ref.ADAM else 0.5     # Adam: |g| ~ 1e-4 against eps = 1e-7 makes eps placement visible


def _slots(opt):
    return {ref.SGD: 0, ref.ADAGRAD: 1, ref.ADAM: 2, ref.FTRL: 2}[opt]


def _init_state(opt, shape, rng):
    w = rng.standard_normal(shape) * 0.5
    s1 = np.full(shape, INIT_S1) if opt in (ref.ADAGRAD, ref.FTRL) else np.zeros(shape)
    # Adam starts from zero slots, as after initialisation, so that sqrt(v / (1-b2^t)) ~ |g| stays near epsilon's scale
    s2 = rng.standard_normal(shape) * 0.1 if opt == ref.FTRL else np.zeros(shape)
    if opt == ref.FTRL:     # w must be the function of (z, n) the optimizer maintains
        w = ref.ftrl_w(s2, s1, HP[opt]["lr"], HP[opt]["p1"], HP[opt]["p2"], HP[opt]["p3"])
    return [w.astype(np.float32).astype(np.float64), s1.astype(np.float32).astype(np.float64),
            s2.astype(np.float32).astype(np.float64)]


class _Guarded:
    """fp32 [V, D] device table between guard regions of sentinel values (at least G rows each).  The table starts
    32 bytes into its buffer, as a variable of a shard does (Layout pads every region to 8 elements): the kernels read
    masters and slots with 16-byte vector loads."""

    def __init__(self, x: np.ndarray):
        V, D = x.shape
        self.pad = (G * D + 7) // 8 * 8
        self.full = torch.full((2 * self.pad + V * D,), -777.0, dtype=torch.float32, device="cuda")
        self.t = self.full[self.pad:self.pad + V * D].view(V, D)
        self.t.copy_(torch.from_numpy(x).float())

    def ptr(self):
        return self.t.data_ptr()

    def get(self):
        assert torch.all(self.full[:self.pad] == -777.0) and torch.all(self.full[-self.pad:] == -777.0), "guard written"
        return self.t.double().cpu().numpy()


def _assert_close(got, want, w0, terms=1, steps=STEPS, what="", mag=0.0):
    """|got - want| <= ROUNDINGS * steps * (terms + 1) * EPS32 * (|want| + |want - w0| + mag) (module docstring)."""
    tol = ROUNDINGS * steps * (np.asarray(terms) + 1) * ref.EPS32 * (np.abs(want) + np.abs(want - w0) + mag + 1e-30)
    bad = np.abs(got - want) > tol
    assert not bad.any(), (what, int(bad.sum()), float(np.abs(got - want)[bad].max()), float(tol[bad].min()))


def _slot_mag(opt, state, slot):
    """Size of the terms a slot accumulates.  Its entries are sums of such terms, so their rounding scales with the
    largest entry (norm-wise); FTRL's z also adds (sqrt(n') - sqrt(n)) / lr * w, whose square roots carry roundings
    of sqrt(n) EPS32 each, so its error scales with sqrt(n) / lr * |w| rather than with |z|."""
    mag = float(np.abs(state[slot]).max())
    if opt == ref.FTRL and slot == 2:
        mag += float(np.sqrt(state[1].max()) / HP[opt]["lr"] * np.abs(state[0]).max()) + 1.0
    return mag


def _assert_ftrl_both_branches(w):
    """FTRL's weight is 0 for |z| <= l1.  The weight is continuous there (it goes to 0 as |z| -> l1), so a z that
    rounding puts on the other side of l1 moves w by at most |dz| / ((beta + sqrt(n)) / lr), far inside the tolerance
    of w: no datum can sit "too close" to l1.  What the data must do is exercise both branches."""
    w = np.concatenate([np.ravel(x) for x in w])
    assert (w == 0).any() and (w != 0).any(), "the data never cross l1: pick another l1"


# ---------------------------------------------------------------------------------------------- dense push / pull
def _make_segs(items):
    from tf_yarn_b200.estimator import ps_hbm
    segs = (ps_hbm.PsSeg * len(items))()
    for k, it in enumerate(items):
        for name, val in it.items():
            setattr(segs[k], name, val)
    return torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).cuda()


class _DenseVar:
    """One variable of a dense push: master + slots (guarded), optional row-padded bf16 shadow, local gradient."""

    def __init__(self, opt, n, rng, cols=0, gdtype=torch.float32, wd=0.0):
        self.opt, self.n, self.cols, self.wd = opt, n, cols, wd
        self.state = [x.reshape(-1, 1) for x in _init_state(opt, (n,), rng)]
        self.w0 = self.state[0].copy()
        self.bufs = [_Guarded(x) for x in self.state]
        self.ld = (cols + 7) // 8 * 8 if cols else 0
        rows = n // cols if cols else 0
        self.shadow = torch.zeros(rows * self.ld, dtype=torch.bfloat16, device="cuda") if cols else None
        if cols:     # the non-pad part starts as garbage: the push must overwrite it, and never touch the pad
            self.shadow.view(rows, self.ld)[:, :cols] = 7.0
        self.grad = torch.zeros(n, dtype=gdtype, device="cuda")

    def seg(self, local):
        hp = HP[self.opt]
        ns = _slots(self.opt)
        return dict(remote_w=self.bufs[0].ptr(), remote_s1=self.bufs[1].ptr() if ns >= 1 else 0,
                    remote_s2=self.bufs[2].ptr() if ns >= 2 else 0,
                    remote_shadow=self.shadow.data_ptr() if self.shadow is not None else 0, local=local, n=self.n,
                    opt=self.opt, lr=hp["lr"], eps=hp["eps"], wd=self.wd, p1=hp["p1"], p2=hp["p2"], p3=hp["p3"],
                    cols=self.cols, shadow_ld=self.ld)

    def check(self, steps):
        got = [b.get() for b in self.bufs]
        _assert_close(got[0], self.state[0], self.w0, steps=steps, what=("w", self.opt, self.n),
                      mag=np.abs(self.state[0] - self.w0).max())
        for s in range(1, 1 + _slots(self.opt)):
            _assert_close(got[s], self.state[s], 0.0, steps=steps, what=("slot", s, self.opt, self.n),
                          mag=_slot_mag(self.opt, self.state, s))
        if self.opt == ref.FTRL and self.n > 64:
            _assert_ftrl_both_branches([self.state[0]])
        if self.shadow is not None:
            sh = self.shadow.view(-1, self.ld).double().cpu().numpy()
            assert np.array_equal(sh, ref.shadow(got[0].reshape(-1), self.cols, self.ld)), "shadow != bf16(master)"


def _dense_push(lib, variables, rng, steps, gdtype, grad_scale, max_n=None):
    segs = _make_segs([v.seg(v.grad.data_ptr()) for v in variables])
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    max_n = max_n or max(v.n for v in variables)
    for step in range(steps):
        sc = ref.adam_scale(step + 1, 0.9, 0.999)
        adam.copy_(torch.tensor(sc, dtype=torch.float32))       # changed between launches, as a replayed graph sees it
        sc32 = tuple(float(np.float32(x)) for x in sc)
        for v in variables:
            g = rng.standard_normal(v.n) * _grad_mag(v.opt)
            v.grad.copy_(torch.from_numpy(g))
            g = v.grad.double().cpu().numpy()                     # what the kernel reads (bf16 rounding included)
            hp = dict(HP[v.opt], wd=v.wd)
            ref.dense_push(v.opt, v.state[0][:, 0], v.state[1][:, 0], v.state[2][:, 0], g, hp,
                           grad_scale=grad_scale, scale=sc32)
        rc = lib.tfy_ps_push(segs.data_ptr(), len(variables), max_n, 1 if gdtype == torch.bfloat16 else 0, grad_scale,
                             adam.data_ptr(), _stream())
        assert rc == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16], ids=["g32", "g16"])
@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_dense_push_matches_reference(lib, opt, gdtype):
    rng = np.random.default_rng(10 + opt)
    variables = [_DenseVar(opt, n, rng, gdtype=gdtype, wd=0.01) for n in (1, 3, 4, 5, 1027)]
    variables += [_DenseVar(opt, 37 * 13, rng, cols=13, gdtype=gdtype, wd=0.01),      # cols % 4 != 0, pitch 16
                  _DenseVar(opt, 9 * 24, rng, cols=24, gdtype=gdtype, wd=0.01)]       # cols % 4 == 0, pitch 24
    _dense_push(lib, variables, rng, STEPS, gdtype, grad_scale=0.5)
    for v in variables:
        v.check(STEPS)


def test_dense_push_mixed_segments_and_a_grid_stride_wrap(lib):
    """Different optimizers and sizes in one launch; one segment longer than 540,672 elements (132*4 blocks x 256
    threads x 4) so that the grid-stride loop wraps."""
    rng = np.random.default_rng(3)
    variables = [_DenseVar(ref.SGD, 600_007, rng, wd=0.01), _DenseVar(ref.ADAGRAD, 5, rng),
                 _DenseVar(ref.ADAM, 1027, rng),
                 _DenseVar(ref.FTRL, 11 * 21, rng, cols=21), _DenseVar(ref.ADAGRAD, 560_000, rng, cols=70)]
    _dense_push(lib, variables, rng, 2, torch.float32, grad_scale=1.5)
    for v in variables:
        v.check(2)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1027, 600_001])
def test_pull_and_shadow_refresh_round_to_nearest_even(lib, n):
    rng = np.random.default_rng(n)
    w = torch.from_numpy(rng.standard_normal(n) * 3).float().cuda()
    w[: min(n, 2)] = torch.tensor([1.0 + 2 ** -8, -(1.0 + 3 * 2 ** -8)][: min(n, 2)])      # exact ties
    want = ref.bf16_round(w.cpu().numpy())
    loc32 = torch.zeros(n, device="cuda")
    loc16 = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    for local, bf16 in ((loc32, 0), (loc16, 1)):
        segs = _make_segs([dict(remote_w=w.data_ptr(), local=local.data_ptr(), n=n)])
        assert lib.tfy_ps_pull(segs.data_ptr(), 1, n, bf16, _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(loc32, w)
    assert np.array_equal(loc16.double().cpu().numpy(), want)
    # shadow refresh: flat, and row-padded with cols % 4 != 0 (one row of n, or 1027 = 13 rows of 79), pitch rounded
    # up to 8; the pad columns must stay exactly zero
    for cols in [0] + ([n] if n > 1 and n % 4 else []) + ([79] if n == 1027 else []):
        ld = (cols + 7) // 8 * 8 if cols else 0
        sh = torch.zeros(max(n // cols * ld if cols else n, 1), dtype=torch.bfloat16, device="cuda")
        segs = _make_segs([dict(remote_w=w.data_ptr(), remote_shadow=sh.data_ptr(), n=n, cols=cols, shadow_ld=ld)])
        assert lib.tfy_ps_refresh_shadow(segs.data_ptr(), 1, n, _stream()) == 0
        torch.cuda.synchronize()
        got = sh.double().cpu().numpy()
        assert np.array_equal(got.reshape(ref.shadow(w.cpu().numpy(), cols, ld).shape),
                              ref.shadow(w.cpu().numpy(), cols, ld)), (n, cols)


# ---------------------------------------------------------------------------------------------- sparse pull
def _ids(rng, shape, V, heavy=True, oor=True):
    """Heavy duplicates: half the ids on one row, a quarter on another, the rest uniform; some out of range."""
    ids = rng.integers(0, V, size=shape)
    if heavy and V > 2:
        u = rng.random(shape)
        ids[u < 0.5] = V // 2
        ids[(u >= 0.5) & (u < 0.75)] = 1
    if oor:
        u = rng.random(shape)
        ids[u < 0.03] = -1
        ids[(u >= 0.03) & (u < 0.05)] = V
        ids[(u >= 0.05) & (u < 0.06)] = V + 17
    return ids


@pytest.mark.parametrize("odtype", [torch.float32, torch.bfloat16], ids=["o32", "o16"])
@pytest.mark.parametrize("L,mean", [(1, 0), (3, 0), (3, 1)], ids=["L1", "L3sum", "L3mean"])
@pytest.mark.parametrize("D", [1, 3, 4, 64, 65])
def test_embedding_bag_matches_reference(lib, D, L, mean, odtype):
    rng = np.random.default_rng(D * 10 + L)
    V, B = 50, 300
    table = rng.standard_normal((V, D))
    ids = _ids(rng, (B, L), V)
    t = _Guarded(table)
    idt = torch.from_numpy(ids).cuda()
    out = torch.full((B, D), 5.0, dtype=odtype, device="cuda")
    assert lib.tfy_ps_embedding_bag(t.ptr(), idt.data_ptr(), out.data_ptr(), int(odtype == torch.bfloat16), B, L, D, V,
                                    mean, _stream()) == 0
    torch.cuda.synchronize()
    want = ref.bag(t.get(), ids, bool(mean))
    got = out.double().cpu().numpy()
    if odtype == torch.bfloat16:
        # an fp32 sum of L terms (error <= L EPS32 sum|x|), then one bf16 rounding (relative 2^-8)
        tol = 2.0 ** -8 * np.abs(want) + (L + 1) * ref.EPS32 * ref.bag(np.abs(table), ids, bool(mean))
    else:
        tol = (L + 1) * ref.EPS32 * ref.bag(np.abs(table), ids, bool(mean))
    assert np.all(np.abs(got - want) <= tol + 1e-30)


def test_embedding_bag_grid_stride_wrap(lib):
    """B * D / 4 = 320,000 > 132*8 blocks x 256 threads: the grid-stride loop wraps."""
    rng = np.random.default_rng(5)
    V, B, D, L = 1000, 20_000, 64, 2
    table = rng.standard_normal((V, D)).astype(np.float32)
    ids = _ids(rng, (B, L), V)
    out = torch.zeros(B, D, device="cuda")
    t = torch.from_numpy(table).cuda()
    assert lib.tfy_ps_embedding_bag(t.data_ptr(), torch.from_numpy(ids).cuda().data_ptr(), out.data_ptr(), 0, B, L, D,
                                    V, 0, _stream()) == 0
    torch.cuda.synchronize()
    want = ref.bag(table.astype(np.float64), ids, False)
    assert np.all(np.abs(out.double().cpu().numpy() - want) <= 3 * ref.EPS32 * ref.bag(np.abs(table), ids, False) + 1e-30)


@pytest.mark.parametrize("odtype", [torch.float32, torch.bfloat16], ids=["o32", "o16"])
@pytest.mark.parametrize("D", [1, 3, 64])
def test_multi_bag_matches_reference(lib, D, odtype):
    rng = np.random.default_rng(D)
    V, B, T = 40, 257, 5
    tables = [_Guarded(rng.standard_normal((V, D))) for _ in range(T)]
    ids = _ids(rng, (T, B), V)
    ptrs = torch.tensor([t.ptr() for t in tables], dtype=torch.int64, device="cuda")
    out = torch.zeros(B, D, dtype=odtype, device="cuda")
    assert lib.tfy_ps_multi_bag(ptrs.data_ptr(), torch.from_numpy(ids).cuda().data_ptr(), out.data_ptr(),
                                int(odtype == torch.bfloat16), B, T, D, V, _stream()) == 0
    torch.cuda.synchronize()
    host = [t.get() for t in tables]
    want = ref.multi_bag(host, ids)
    mag = ref.multi_bag([np.abs(h) for h in host], ids)
    tol = (T + 1) * ref.EPS32 * mag + (2.0 ** -8 * np.abs(want) if odtype == torch.bfloat16 else 0)
    assert np.all(np.abs(out.double().cpu().numpy() - want) <= tol + 1e-30)


# ---------------------------------------------------------------------------------------------- sparse push
class _Tables:
    """T guarded tables with their optimizer slots, and the float64 reference state."""

    def __init__(self, opt, T, V, D, rng):
        self.opt, self.T = opt, T
        self.state = [_init_state(opt, (V, D), rng) for _ in range(T)]
        self.w0 = [s[0].copy() for s in self.state]
        self.bufs = [[_Guarded(x) for x in s] for s in self.state]
        ns = _slots(opt)
        self.ptrs = [torch.tensor([b[k].ptr() for b in self.bufs], dtype=torch.int64, device="cuda") for k in range(3)]
        self.s1 = self.ptrs[1] if ns >= 1 else None
        self.s2 = self.ptrs[2] if ns >= 2 else None

    def ref_push(self, ids, dout, D, mean=False, grad_scale=1.0, col_stride=0, scale=(1.0, 1.0)):
        ref.sparse_push(self.opt, [s[0] for s in self.state], [s[1] for s in self.state],
                        [s[2] for s in self.state], ids, dout, D, HP[self.opt], mean=mean, grad_scale=grad_scale,
                        col_stride=col_stride, scale=scale)

    def snapshot(self):
        return [[b.t.clone() for b in bb] for bb in self.bufs]

    def restore(self, snap):
        for bb, ss in zip(self.bufs, snap):
            for b, s in zip(bb, ss):
                b.t.copy_(s)

    def check(self, counts, steps, what=""):
        for t in range(self.T):
            terms = np.asarray(counts[t], np.float64)[:, None]
            got = [b.get() for b in self.bufs[t]]
            _assert_close(got[0], self.state[t][0], self.w0[t], terms, steps, what=("w", t, what),
                          mag=np.abs(self.state[t][0] - self.w0[t]).max())
            for s in range(1, 1 + _slots(self.opt)):
                _assert_close(got[s], self.state[t][s], 0.0, terms, steps, what=("slot", s, t, what),
                              mag=_slot_mag(self.opt, self.state[t], s))
        if self.opt == ref.FTRL and sum(s[0].size for s in self.state) >= 400:
            _assert_ftrl_both_branches([s[0] for s in self.state])


def _scratch(lib, n):
    from tf_yarn_b200.estimator import ps_hbm
    return ps_hbm.push_rows_scratch(lib, n, torch.device("cuda"))


def _push_rows(lib, tb, ids, dout, gdtype, D, L, mean, grad_scale, adam, dout_ld):
    B = ids.shape[1]
    V = tb.state[0][0].shape[0]
    sc = _scratch(lib, B * L)
    ns = _slots(tb.opt)
    idt = torch.from_numpy(np.ascontiguousarray(ids[0])).cuda()
    rc = lib.tfy_ps_push_rows(tb.bufs[0][0].ptr(), tb.bufs[0][1].ptr() if ns >= 1 else None,
                                tb.bufs[0][2].ptr() if ns >= 2 else None, idt.data_ptr(),
                                dout.data_ptr(), int(gdtype == torch.bfloat16), B, L, D, V, mean, tb.opt,
                                HP[tb.opt]["lr"], HP[tb.opt]["eps"], HP[tb.opt]["p1"], HP[tb.opt]["p2"],
                                HP[tb.opt]["p3"], grad_scale, adam.data_ptr(), dout_ld, sc.data_ptr(), sc.numel(),
                                _stream())
    torch.cuda.current_stream().synchronize()       # keep ids and the scratch alive until the push ran
    return rc


def _run_push_rows(lib, opt, D, L, mean, gdtype, dout_ld, B=512, V=60, steps=STEPS, seed=0):
    rng = np.random.default_rng(seed + 100 * opt + D)
    tb = _Tables(opt, 1, V, D, rng)
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    counts = np.zeros((1, V))
    for step in range(steps):
        ids = _ids(rng, (B, L), V)[None]
        if L > 1:
            ids[0, ::7, 1] = ids[0, ::7, 0]               # repeats inside one bag
        counts = np.maximum(counts, ref.row_counts(ids, V))      # per push: the bound already scales with steps
        dout = torch.from_numpy(rng.standard_normal((B, dout_ld)) * _grad_mag(opt)).to(gdtype).cuda()
        sc = ref.adam_scale(step + 1, 0.9, 0.999)
        adam.copy_(torch.tensor(sc, dtype=torch.float32))
        tb.ref_push(ids, dout.double().cpu().numpy(), D, mean=bool(mean), grad_scale=0.5,
                    scale=tuple(float(np.float32(x)) for x in sc))
        assert _push_rows(lib, tb, ids, dout, gdtype, D, L, mean, 0.5, adam, dout_ld) == 0
    torch.cuda.synchronize()
    tb.check(counts, steps, what=(opt, D, L, mean))
    return tb


@pytest.mark.parametrize("L,mean", [(1, 0), (3, 0), (3, 1)], ids=["L1", "L3sum", "L3mean"])
@pytest.mark.parametrize("D", [1, 3, 4, 64, 65])
@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_push_rows_matches_reference(lib, opt, D, L, mean):
    gdtype = torch.bfloat16 if (D + L) % 2 else torch.float32
    _run_push_rows(lib, opt, D, L, mean, gdtype, dout_ld=D + (4 if D % 4 == 0 else 3))


@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_push_rows_odd_pitch_takes_the_scalar_path(lib, opt):
    """D % 4 == 0 but a pitch that breaks 16-byte alignment: the push must not use vector loads."""
    _run_push_rows(lib, opt, 64, 1, 0, torch.float32, dout_ld=67)
    _run_push_rows(lib, opt, 64, 1, 0, torch.bfloat16, dout_ld=66)


def test_push_rows_grid_stride_wrap(lib):
    """B * L = 300,000 sorted positions > 132*8 blocks x 256 threads: the apply kernel's loop wraps."""
    _run_push_rows(lib, ref.ADAGRAD, 4, 3, 1, torch.float32, dout_ld=4, B=100_000, V=5000, steps=2)


def _multi_push(lib, tb, ids, dout, D, dout_ld, col_stride, adam):
    T, B = ids.shape[0], ids.shape[1]
    sc = _scratch(lib, T * B)
    h = HP[tb.opt]
    idt = torch.from_numpy(np.ascontiguousarray(ids[:, :, 0])).cuda()
    rc = lib.tfy_ps_multi_push_rows(tb.ptrs[0].data_ptr(), tb.s1.data_ptr() if tb.s1 is not None else None,
                                      tb.s2.data_ptr() if tb.s2 is not None else None, idt.data_ptr(),
                                      dout.data_ptr(), int(dout.dtype == torch.bfloat16), B, T, D,
                                      tb.state[0][0].shape[0], tb.opt, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"],
                                      0.75, adam.data_ptr(), dout_ld, col_stride, sc.data_ptr(), sc.numel(), _stream())
    torch.cuda.current_stream().synchronize()       # keep ids and the scratch alive until the push ran
    return rc


# wide tower: [V, 1] tables, every table gets the same fp32 gradient (col_stride 0); fused first deep layer: D = 64
# column slices of a bf16 dx with pitch Kp (26*64 + 13 -> 1680) ; a scalar-path layout (D = 3, col_stride 3)
MULTI_CASES = {"wide": (1, 0, torch.float32, 1), "fused_first": (64, 64, torch.bfloat16, 64 * 6 + 16),
               "scalar": (3, 3, torch.float32, 3 * 6 + 1)}


@pytest.mark.parametrize("case", list(MULTI_CASES))
@pytest.mark.parametrize("opt", OPTS, ids=OPT_IDS)
def test_multi_push_rows_matches_reference(lib, opt, case):
    D, col_stride, gdtype, ld = MULTI_CASES[case]
    rng = np.random.default_rng(opt * 7 + D)
    T, V, B = 6, 80, 512
    tb = _Tables(opt, T, V, D, rng)
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    counts = np.zeros((T, V))
    for step in range(STEPS):
        ids = _ids(rng, (T, B, 1), V)
        counts = np.maximum(counts, ref.row_counts(ids, V))      # per push: the bound already scales with steps
        dout = torch.from_numpy(rng.standard_normal((B, ld)) * _grad_mag(opt)).to(gdtype).cuda()
        sc = ref.adam_scale(step + 1, 0.9, 0.999)
        adam.copy_(torch.tensor(sc, dtype=torch.float32))
        tb.ref_push(ids, dout.double().cpu().numpy(), D, grad_scale=0.75, col_stride=col_stride,
                    scale=tuple(float(np.float32(x)) for x in sc))
        assert _multi_push(lib, tb, ids, dout, D, ld, col_stride, adam) == 0
    torch.cuda.synchronize()
    tb.check(counts, STEPS, what=case)


def test_multi_push_rows_grid_stride_wrap(lib):
    rng = np.random.default_rng(11)
    T, V, B, D = 26, 3000, 12_000, 1                       # T * B = 312,000 sorted positions
    tb = _Tables(ref.FTRL, T, V, D, rng)
    ids = _ids(rng, (T, B, 1), V)
    dout = torch.from_numpy(rng.standard_normal((B, 1)) * 0.5).float().cuda()
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    tb.ref_push(ids, dout.double().cpu().numpy(), D, grad_scale=0.75)
    assert _multi_push(lib, tb, ids, dout, D, 1, 0, adam) == 0
    torch.cuda.synchronize()
    tb.check(ref.row_counts(ids, V), 1)


def test_push_rows_error_codes(lib):
    rng = np.random.default_rng(0)
    tb = _Tables(ref.ADAM, 1, 10, 4, rng)
    ids = torch.zeros(8, dtype=torch.int64, device="cuda")
    dout = torch.zeros(8, 4, device="cuda")
    sc = _scratch(lib, 8)
    w, s1, s2 = (b.ptr() for b in tb.bufs[0])

    def call(opt, a, b, scratch=sc):
        return lib.tfy_ps_push_rows(w, a, b, ids.data_ptr(), dout.data_ptr(), 0, 8, 1, 4, 10, 0, opt, 0.1, 1e-7, 0.9,
                                    0.999, 0.0, 1.0, None, 0, scratch.data_ptr() if scratch is not None else None,
                                    scratch.numel() if scratch is not None else 0, _stream())

    def mcall(opt, a, b):
        return lib.tfy_ps_multi_push_rows(tb.ptrs[0].data_ptr(), a, b, ids.data_ptr(), dout.data_ptr(), 0, 8, 1, 4, 10,
                                          opt, 0.1, 1e-7, 0.9, 0.999, 0.0, 1.0, None, 0, 0, sc.data_ptr(), sc.numel(),
                                          _stream())
    assert call(1, s1, s2) == -3 and call(99, s1, s2) == -3                  # Adadelta / unknown: not fused here
    assert mcall(1, tb.ptrs[1].data_ptr(), tb.ptrs[2].data_ptr()) == -3
    assert call(ref.ADAGRAD, None, None) == -4 and call(ref.ADAM, s1, None) == -4 and call(ref.FTRL, s1, None) == -4
    assert mcall(ref.ADAGRAD, None, None) == -4 and mcall(ref.FTRL, tb.ptrs[1].data_ptr(), None) == -4
    assert call(ref.SGD, None, None, scratch=None) == -5                     # the fold needs its scratch
    torch.cuda.synchronize()
    assert np.array_equal(tb.bufs[0][0].get(), tb.state[0][0])               # nothing was applied


@pytest.mark.parametrize("opt", [ref.ADAGRAD, ref.ADAM, ref.FTRL], ids=["adagrad", "adam", "ftrl"])
def test_push_with_heavy_duplicates_is_reproducible(lib, opt):
    """The same push twice from the same state gives bit-identical tables and slots."""
    rng = np.random.default_rng(opt)
    T, V, B, D = 4, 30, 2048, 64
    tb = _Tables(opt, T, V, D, rng)
    ids = _ids(rng, (T, B, 1), V)
    dout = torch.from_numpy(rng.standard_normal((B, D * T)) * _grad_mag(opt)).to(torch.bfloat16).cuda()
    adam = torch.tensor(ref.adam_scale(2, 0.9, 0.999), dtype=torch.float32, device="cuda")
    snap = tb.snapshot()
    results = []
    for _ in range(2):
        tb.restore(snap)
        assert _multi_push(lib, tb, ids, dout, D, D * T, D, adam) == 0
        assert _push_rows(lib, tb, ids[:1, :, :1].reshape(1, B // 4, 4), dout, torch.bfloat16, D, 4, 1, 1.0, adam,
                          D * T) == 0
        torch.cuda.synchronize()
        results.append([b.t.clone() for bb in tb.bufs for b in bb])
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_wide_tower_group_push_captured_in_a_cuda_graph_matches_eager(lib):
    """_TableGroup.push (the wide tower's FTRL push) captured with torch.cuda.graph and replayed from a restored state
    gives the eager result bit for bit: the duplicate fold needs no host synchronisation."""
    from tf_yarn_b200.estimator import ps_hbm
    rng = np.random.default_rng(21)
    T, V, B = 26, 500, 512
    tb = _Tables(ref.FTRL, T, V, 1, rng)
    conn = types.SimpleNamespace(lib=lib, adam_scale=torch.ones(2, device="cuda"), account=lambda **k: None)
    group = ps_hbm._TableGroup.__new__(ps_hbm._TableGroup)
    group.conn, group.idx, group.tables, group.s1, group.s2 = conn, list(range(T)), tb.ptrs[0], tb.s1, tb.s2
    h = HP[ref.FTRL]
    group.V, group.hp, group.slots = V, (ref.FTRL, h["lr"], h["eps"], h["p1"], h["p2"], h["p3"]), 2
    group.D, group.col_stride, group.out_ld, group.one_table, group.parts = 1, 0, 1, False, None
    ids = torch.from_numpy(_ids(rng, (T, B), V, oor=False)).cuda()
    dout = torch.from_numpy(rng.standard_normal((B, 1)) * 0.5).float().cuda()
    snap = tb.snapshot()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                              # warm-up off the capture stream, as torch recommends
        group.push(ids, dout)
    torch.cuda.current_stream().wait_stream(s)
    tb.restore(snap)
    group.push(ids, dout)
    torch.cuda.synchronize()
    eager = [b.t.clone() for bb in tb.bufs for b in bb]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        group.push(ids, dout)
    for _ in range(2):
        tb.restore(snap)
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(eager, [b.t for bb in tb.bufs for b in bb]):
            assert torch.equal(a, b)
    tb.ref_push(ids.cpu().numpy()[:, :, None], dout.double().cpu().numpy(), 1)
    tb.check(ref.row_counts(ids.cpu().numpy()[:, :, None], V), 1)


def test_push_rows_run_lengths_around_the_short_run_limit(lib):
    """Runs of 1, 31, 32, 33 and 64 occurrences: the first three are applied by the per-run threads, the last two by
    the warp kernel.  Every row must still get exactly one update with the sum of its gradients."""
    V, D = 16, 4
    lengths = {0: 1, 3: 31, 5: 32, 7: 33, 9: 64, 12: 2}
    ids = np.concatenate([np.full(n, i) for i, n in lengths.items()])
    np.random.default_rng(0).shuffle(ids)
    tb = _Tables(ref.ADAGRAD, 1, V, D, np.random.default_rng(1))
    B = ids.size
    dout = torch.from_numpy(np.random.default_rng(2).standard_normal((B, D)) * 0.5).float().cuda()
    adam = torch.ones(2, dtype=torch.float32, device="cuda")
    ids3 = ids.reshape(1, B, 1)
    tb.ref_push(ids3, dout.double().cpu().numpy(), D, grad_scale=0.5)
    assert _push_rows(lib, tb, ids3, dout, torch.float32, D, 1, 0, 0.5, adam, D) == 0
    tb.check(ref.row_counts(ids3, V), 1)


def test_hbm_and_cpu_planes_train_a_wide_and_deep_network_alike(tmp_path):
    """Three train steps of a small canned wide-and-deep network through the HBM plane (K5 fused first layer and the
    multi-table wide tower enabled) and through the shared-memory CPU plane, from the same initial values and batches
    with many duplicate buckets.  This checks ps_hbm's addressing and packing -- slot offsets, p3 = beta for FTRL,
    init_s1, the shadow pitch, the dx column slices of the fused first layer -- not precision.  The HBM plane runs its
    GEMMs in bf16: the embedding-row gradients are dx = dy W with dy and W rounded to bf16 (2^-8 relative each) and dx
    itself stored in bf16, about 1.2e-2 per element before any cancellation, and the forward's bf16 activations move
    the loss gradient as well.  So the updates agree to a few 1e-2 relative (the norm of the difference of the updates
    over the norm of the CPU plane's update, per variable and slot).  Measured on an H100 with these seeds: at most
    0.03 for the Dense layers, 0.07 for the deep embedding rows and 0.22 for their Adagrad accumulators, whose
    per-row sums of squared gradients over few occurrences (V = 40) amplify the differences of the bf16 dx and of the
    ReLU gates that the bf16 forward flips; the wide tower, pushed from fp32 gradients, agrees to 1e-3.  The bounds
    are 0.1 for values and 0.35 for slots.  An addressing fault (a wrong slot, row or column slice, p3 or init_s1)
    changes whole updates: a difference of order 1 or more.  FTRL (wide tower) and Adagrad (deep tower) are the canned defaults.  Adam is left out: the HBM
    plane's sparse Adam is lazy (rows outside the batch keep m and v) while the CPU plane's is not."""
    import copy

    from tf_yarn_b200 import keras
    from tf_yarn_b200.estimator import canned, ps, ps_hbm
    from tf_yarn_b200.models import wide_deep as wdm

    torch.manual_seed(0)
    V, B, n_cat, n_num = 40, 256, 3, 5
    wide, deep = wdm.feature_columns(vocab=V, emb_dim=64, n_cat=n_cat, n_num=n_num)
    net_cpu = canned._WideDeepNet(wide, deep, [64, 32], 1)
    net = copy.deepcopy(net_cpu).cuda()
    named = ps._named_trainables(net)
    ftrl = keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001, l2_regularization_strength=0.01)
    by_name = {n: ftrl for n, _ in named if n.startswith("linear.")}
    layout = ps.make_layout(named, 1, keras.optimizers.Adagrad(0.05), by_name)
    assert "ftrl" in layout.kinds and "adagrad" in layout.kinds

    # HBM plane over a local buffer standing in for the ps rank's shard
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
        assert conn.fused_first and conn.fused_wide
        w0 = [[cpu._region(i, s).double().clone() for s in range(1 + layout.var_slots[i])] for i in range(len(named))]

        batches = wdm.synthetic_batches(B, 3, vocab=V, seed=1, n_cat=n_cat, n_num=n_num)   # V = 40: heavy duplicates
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
                assert want.norm() > 0, (name, s)
                rels[f"{name}/{s}"] = round(((hbm - want).norm() / want.norm()).item(), 4)
        assert all(r < (0.1 if k.endswith("/0") else 0.35) for k, r in rels.items()), rels
    finally:
        header.unlink()
        shards[0].unlink()
