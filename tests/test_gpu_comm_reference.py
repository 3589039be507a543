"""The collective kernels (K1 one-shot, K2 two-shot, K3 NVLS all-reduce, broadcast, all-gather) and the fused optimizer
step at several ranks (K4 in P2P and NVLS mode) against tests/comm_reference.py and the float64 optimizer reference.

A module-scoped fixture runs tests/gpu/comm_reference_worker.py once per world size, one process per GPU: 1 (the
multi-GPU kernels at one rank, which any H100 runs), then 2, 3, 5 and 8 as far as the GPUs present allow.  Worlds 3
and 5 cover the partial group of four of the P2P rank loop and a grad_scale / world that fp32 rounds; world 8 has two
full groups.  The worker only launches kernels and saves what they left; every judgement is made here:

* P2P all-reduce: bit for bit the rank-order fp32 sum times the fp32 scale, rounded to nearest even for bf16.
  NVLS: within ``nvls_bound`` of the exact sum, and exact on integer inputs whose sums are representable.
* Every rank holds the same bits; the guard bands around every buffer are intact; one-shot leaves its input alone.
* Fused step: each element of master and states within the per-element bound of tests/fused_step_bounds.py around the
  float64 reference, fed the emulated fp32 rank-order sum (P2P, no error) or the exact sum within the NVLS bound.

NVLS cases skip only when ``Communicator.multicast`` is false, and say so.  ``pytest -s`` prints the largest
error / bound ratio per optimizer variant and mode.
"""
import functools
import json
import math
import os
import shutil
import signal
import subprocess
import sys
import tempfile
from collections import defaultdict

import numpy as np
import pytest
import torch

import comm_reference as cr
import fused_step_reference as ref
from fused_step_bounds import B, _kernel_update

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "gpu", "comm_reference_worker.py")
TIMEOUT_S = 1800
_RATIO = defaultdict(float)
_DIRS = {}


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@functools.lru_cache(maxsize=None)
def _run(world: int):
    """Run the worker at ``world`` ranks (once per module); returns (out_dir, per-rank records) or the failure."""
    out = tempfile.mkdtemp(prefix=f"comm_ref_w{world}_")
    _DIRS[world] = out
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29720 + world), WORKER, out]
    env = dict(os.environ, OMP_NUM_THREADS="4")
    p = subprocess.Popen(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                         start_new_session=True)
    try:
        log, _ = p.communicate(timeout=TIMEOUT_S)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        log, _ = p.communicate()
        return None, f"the worker did not finish in {TIMEOUT_S} s:\n{log[-4000:]}"
    if p.returncode != 0:
        return None, f"the worker failed ({p.returncode}):\n{log[-6000:]}"
    recs = []
    for r in range(world):
        with open(os.path.join(out, f"rank{r}.json")) as f:
            recs.append(json.load(f))
    return out, recs


def _world(world: int):
    need = max(world, 1)
    if _ngpu() < need:
        pytest.skip(f"needs {need} GPUs, {_ngpu()} present")
    out, recs = _run(world)
    assert out is not None, recs
    return out, recs


def _need_multicast(recs):
    if not recs[0]["multicast"]:
        pytest.skip("multicast (NVLS) is not available: Communicator.multicast is False on this machine")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for d in _DIRS.values():
        shutil.rmtree(d, ignore_errors=True)
    if _RATIO:
        print("\nlargest |kernel - reference| / bound per optimizer variant and mode:")
        for w in sorted(_DIRS):
            recs = _run(w)[1]
            if not isinstance(recs, str):
                print(f"  world {w}: multicast {'available' if recs[0]['multicast'] else 'NOT available'}")
        for key in sorted(_RATIO):
            print(f"  {key[0]:28s} {key[1]:5s} {_RATIO[key]:.3f}")


def _sent():
    return {r: cr.sha(cr.sentinel(cr.GUARD, r)) for r in range(16)}


# ---------------------------------------------------------------------------------------------------------------
# all-reduce
# ---------------------------------------------------------------------------------------------------------------
def _judge_allreduce(case, world, got_bits):
    scale = cr.scale_value(case.scale, world)
    xs = lambda: (cr.case_input(case, world, r) for r in range(world))  # noqa: E731
    want = cr.p2p_allreduce(xs(), scale, case.dtype)
    got_f = cr.float_of(got_bits, case.dtype)
    want_f = cr.float_of(want, case.dtype)
    nan = np.isnan(want_f)
    assert np.array_equal(np.isnan(got_f), nan), (case.id, "NaN pattern", np.flatnonzero(np.isnan(got_f) != nan)[:5])
    if case.algo != "nvls" or case.values == "int":
        bad = (got_bits != want) & ~nan
        assert not bad.any(), (case.id, int(bad.sum()), np.flatnonzero(bad)[:5], got_f[bad][:5], want_f[bad][:5])
        return
    s, a = cr.exact_sums(xs())
    centre, radius = cr.nvls_bound(s, a, world, scale, case.dtype)
    inf = np.isinf(want_f)
    assert np.array_equal(got_f[inf], want_f[inf]), (case.id, "overflow")
    fin = ~nan & ~inf
    err = np.abs(got_f[fin].astype(np.float64) - centre[fin])
    bad = ~(err <= radius[fin])
    assert not bad.any(), (case.id, int(bad.sum()), got_f[fin][bad][:5], centre[fin][bad][:5], radius[fin][bad][:5])


@pytest.mark.parametrize("case", cr.CASES, ids=lambda c: c.id)
@pytest.mark.parametrize("world", cr.WORLDS)
def test_allreduce_matches_reference(world, case):
    out, recs = _world(world)
    if case.algo == "nvls":
        _need_multicast(recs)
    got = np.load(os.path.join(out, f"ar_{case.id}.npy"))
    assert got.size == cr.n_elems(case, world)
    rows = [r["allreduce"][case.id] for r in recs]
    assert all(r["rc"] == 0 for r in rows), [r["rc"] for r in rows]
    assert len({r["out"] for r in rows}) == 1, "the ranks hold different results"
    assert rows[0]["out"] == cr.sha(got)
    sent = _sent()
    for rank, r in enumerate(rows):
        assert r["guards"] == [sent[rank]] * 4, (rank, "a store landed outside the buffer")
        if case.algo == "oneshot":
            mine = cr.to_bits(cr.case_input(case, world, rank), case.dtype)
            assert r["input_after"] == cr.sha(mine), (rank, "one-shot changed its input")
        else:
            assert r["input_after"] == r["out"], (rank, "two-shot / NVLS must reduce in place")
    _judge_allreduce(case, world, got)


@pytest.mark.parametrize("world", cr.WORLDS)
def test_launchers_refuse_bad_arguments(world):
    _, recs = _world(world)
    for r in recs:
        want = {"bad_n": -2, "oneshot_no_out": -4, "bcast_bad_bytes": -2, "gather_bad_bytes": -2}
        if world > 1:
            want["shard_not_divisible"] = -3
        if not r["multicast"]:
            want["nvls_without_multicast"] = -5
        assert r["refusals"] == want


@pytest.mark.parametrize("world", cr.WORLDS)
def test_broadcast_and_allgather_are_exact(world):
    _, recs = _world(world)
    sent = _sent()
    modes = [0, 1] if recs[0]["multicast"] else [0]
    for packs in cr.BCAST_PACKS:
        for root in range(world):
            want = cr.sha(cr.payload(packs * 16, f"bcast-{packs}", root))
            for nvls in modes:
                key = f"{packs}-{root}-{nvls}"
                for rank, r in enumerate(recs):
                    row = r["broadcast"][key]
                    assert row["rc"] == 0 and row["out"] == want, (key, rank)
                    assert row["guards"] == [sent[rank]] * 2, (key, rank, "guard band")
    for packs in cr.GATHER_PACKS:
        want = cr.sha(np.concatenate([cr.payload(packs * 16, f"gather-{packs}", r) for r in range(world)]))
        for rank, r in enumerate(recs):
            row = r["allgather"][str(packs)]
            assert row["rc"] == 0 and row["out"] == want, (packs, rank)
            assert row["guards"] == [sent[rank]] * 2, (packs, rank, "guard band")


# ---------------------------------------------------------------------------------------------------------------
# the Communicator's list API
# ---------------------------------------------------------------------------------------------------------------
def _list_bits(v, dtype):
    if dtype == "f16":
        return np.ascontiguousarray(v, np.float16).reshape(-1).view(np.uint16)
    return cr.to_bits(v.reshape(-1), dtype)


@pytest.mark.parametrize("world", cr.WORLDS)
def test_list_api_matches_its_fusion_buffer(world):
    """Communicator.all_reduce of bf16, fp32, fp16, strided, empty and larger-than-the-fusion-buffer tensors, at
    average and sum: the emulation of the P2P reduction of its padded fusion buffer, element by element; broadcast
    of such a list: the root's bits everywhere."""
    out, recs = _world(world)
    for average in (True, False):
        scale = float(np.float32(1.0 / world)) if average else 1.0
        for name, dtype, shape, _ in cr.LIST_TENSORS:
            key = f"reduce-{average}-{name}"
            rows = [r["list"][key] for r in recs]
            assert len({r["out"] for r in rows}) == 1, (key, "ranks differ")
            assert rows[0]["shape"] == list(shape)
            got = np.load(os.path.join(out, f"list_{average}_{name}.npy")).reshape(-1)
            xs = [cr.list_values(name, dtype, shape, r, "reduce").reshape(-1) for r in range(world)]
            if world == 1:
                want = _list_bits(xs[0], dtype)          # one rank: the list API returns at once
            elif dtype == "f16":
                with np.errstate(over="ignore"):
                    want = (cr.p2p_sum([x.astype(np.float32) for x in xs]) * np.float32(scale)).astype(np.float16)
                want = want.view(np.uint16)
            else:
                want = cr.p2p_allreduce(xs, scale, dtype)
            assert got.size == want.size
            bad = got.view(want.dtype) != want
            assert not bad.any(), (key, int(bad.sum()), np.flatnonzero(bad)[:5])
    for name, dtype, shape, _ in cr.LIST_TENSORS:
        want = cr.sha(_list_bits(cr.list_values(name, dtype, shape, world - 1, "bcast"), dtype).view(np.uint8))
        for rank, r in enumerate(recs):
            assert r["list"][f"bcast-{name}"]["out"] == want, (name, rank)


@pytest.mark.parametrize("world", cr.WORLDS)
def test_list_api_sums_float64_and_int64_exactly(world):
    """Horovod-facade dtypes the kernels do not carry: integer-valued float64 and int64 near 2^40, whose every sum is
    exact, give what the CPU plane (gloo) gives: the exact sum, and for float64 averaged, the sum divided by world."""
    out, recs = _world(world)
    f = [cr.wide_values(np.float64, r) for r in range(world)]
    i = [cr.wide_values(np.int64, r) for r in range(world)]
    want = {"wide_False_float64": np.sum(f, axis=0), "wide_False_int64": np.sum(i, axis=0),
            "wide_True_float64": np.sum(f, axis=0) / world}
    for nm, w in want.items():
        got = np.load(os.path.join(out, nm + ".npy")).view(w.dtype)
        assert np.array_equal(got, w), (nm, got[:4], w[:4])
        assert len({r["list"][nm]["out"] for r in recs}) == 1, (nm, "ranks differ")


# ---------------------------------------------------------------------------------------------------------------
# the fused step
# ---------------------------------------------------------------------------------------------------------------
def _split_states(kind, h, S, master, s1, s2):
    s2v = s3v = np.zeros(S)
    if kind == "rmsprop":
        off = 0
        if h.p2 > 0:
            s2v, off = s2[:S], S
        if h.flags & 1:
            s3v = s2[off:off + S]
    elif ref.n_states(kind, h) == 2:
        s2v = s2[:S]
    return master, s1, s2v, s3v


def _gradient(c, world, n, k):
    """The gradient the kernel sees as a bounded value: the rank-order fp32 sum (P2P, exact) or the exact sum within
    the NVLS bound."""
    gs = [cr.as_dtype(cr.case_grads(n, c, r, k), c.pair[0]) for r in range(world)]
    if c.mode == "p2p":
        return B(cr.p2p_sum(gs).astype(np.float64)), gs
    s, a = cr.exact_sums(gs)
    centre, radius = cr.nvls_bound(s, a, world, 1.0, c.pair[0])
    return B(centre, radius), gs


def _check_bound(c, kind, h, k, before, g, got, ratio_key):
    p0, s10, s20, s30 = before
    want = ref.step(kind, p0, g.v, s10, s20, s30, h, k)
    bounds, undecided = _kernel_update(kind, h, k, B(p0), g, B(s10), B(s20), B(s30))
    used = [True, kind != "sgd" or h.p1 != 0.0, ref.n_states(kind, h) >= 2 and (kind != "rmsprop" or h.p2 > 0),
            kind == "rmsprop" and bool(h.flags & 1)]
    for what, on, x, w, b in zip(("p", "s1", "s2", "s3"), used, got, want, bounds):
        if not on:
            continue
        bound = b.e + 2.0 ** -40 * np.abs(w)
        assert np.isfinite(bound).all(), (c.id, what, "no finite bound")
        err = np.abs(x - w)
        if what == "p" and undecided is not None:
            _, _, w_free = ref.ftrl_linear(p0, g.v, s10, s20, h)
            err = np.where(undecided & (x == 0.0), 0.0, np.where(undecided, np.abs(x - w_free), err))
            assert np.array_equal((x == 0.0)[~undecided], (w == 0.0)[~undecided]), (c.id, "FTRL zero pattern")
        bad = ~(err <= bound)
        assert not bad.any(), (c.id, what, k, int(bad.sum()), np.flatnonzero(bad)[:5], x[bad][:5], w[bad][:5],
                               bound[bad][:5])
        ratio = np.divide(err, bound, out=np.zeros_like(err), where=bound > 0)
        _RATIO[ratio_key] = max(_RATIO[ratio_key], float(ratio.max()) if ratio.size else 0.0)


@pytest.mark.parametrize("case", cr.step_cases(8, True), ids=lambda c: c.id)
@pytest.mark.parametrize("world", cr.WORLDS)
def test_fused_step_matches_reference(world, case):
    out, recs = _world(world)
    if case.mode == "nvls":
        _need_multicast(recs)
    c = case
    kind, hp, init = ref.VARIANTS[c.variant]
    shapes = cr.layout_shapes(c.layout, world)
    n = cr.flat_size(shapes, world)
    S = n // world
    pieces = cr.step_pieces(c.split, S, world)
    rows = [r["step"][c.id] for r in recs]
    npz = [np.load(os.path.join(out, "step", f"{c.id}_r{r}.npz")) for r in range(world)]
    pdt = c.pair[1]
    zero_sha = cr.sha(np.zeros(n * cr.ESIZE[c.pair[0]], np.uint8))
    for k, scale in enumerate(cr.STEP_SCALES):
        scale = float(world) if c.solo_grad else scale
        lr = rows[0]["lr"][k]
        assert all(r["lr"][k] == lr for r in rows)
        hk = dict(hp)
        if c.sched:
            from tf_yarn_b200.keras import schedules
            cls, kw = cr.SCHEDULES[c.variant]
            assert math.isclose(lr, getattr(schedules, cls)(**kw)(k), rel_tol=1e-6), (k, lr)
            hk["lr"] = lr
        h = ref.Hyper(grad_scale=scale, world=world, **hk)
        g, gs = _gradient(c, world, n, k)
        for r in range(world):
            assert rows[r]["grads_before"][k] == cr.sha(cr.to_bits(gs[r], c.pair[0])), (r, k, "gradient")
            assert rows[r]["rc"][k] == [0] * len(pieces)
        for r in range(world):
            z = npz[r]
            prev = {nm: z[f"k{k}_before_{nm}"] for nm in ("master", "s1", "s2")}
            for i, piece in enumerate(pieces):
                now = {nm: z[f"k{k}_p{i}_{nm}"] for nm in ("master", "s1", "s2")}
                lo, hi = cr.piece_span(piece, S, r)
                for nm in ("master", "s1", "s2"):
                    for j in range(max(1, now[nm].size // S)):
                        a_, b_ = prev[nm][j * S:(j + 1) * S], now[nm][j * S:(j + 1) * S]
                        keep = np.ones(a_.size, bool)
                        keep[lo:hi] = False
                        assert np.array_equal(a_.view(np.uint32)[keep], b_.view(np.uint32)[keep]), \
                            (r, k, i, nm, "an element outside the launch's range moved")
                prev = now
                after = rows[r]["after"][k][i]
                last = i == len(pieces) - 1
                assert after["step"] == k + (1 if last else 0), (r, k, i, after["step"])
                want_g = zero_sha if c.split == "full" else rows[r]["grads_before"][k]
                assert after["grads"] == want_g, (r, k, i, "gradient buffer")
            before = _split_states(kind, h, S, *(z[f"k{k}_before_{nm}"].astype(np.float64)
                                                 for nm in ("master", "s1", "s2")))
            last = len(pieces) - 1
            got = _split_states(kind, h, S, *(z[f"k{k}_p{last}_{nm}"].astype(np.float64)
                                              for nm in ("master", "s1", "s2")))
            sl = slice(r * S, (r + 1) * S)
            _check_bound(c, kind, h, k, before, B(g.v[sl], g.e[sl] if g.e.ndim else g.e), got, (c.variant, c.mode))
            if c.solo_grad:
                loc = rows[r]["local"][k]
                assert loc["rc"] == 0
                for nm in ("master", "s1", "s2"):
                    if nm in loc:
                        assert loc[nm] == cr.sha(z[f"k{k}_p0_{nm}"].view(np.uint8)), (r, k, nm, "not LOCAL's bits")
        # the replicated parameters: every rank's master shard, rounded to nearest even, bit for bit, on every rank
        for i in range(len(pieces)):
            masters = np.concatenate([npz[r][f"k{k}_p{i}_master"] for r in range(world)])
            params = npz[0][f"k{k}_p{i}_params"]
            want = cr.to_bits(masters, pdt)
            assert np.array_equal(params, want), (k, i, "parameters are not the gathered master")
            assert len({rows[r]["after"][k][i]["params"] for r in range(world)}) == 1, (k, i, "ranks differ")
