"""The HBM parameter server's worker step (estimator/ps_hbm.py), launch for launch, on the CPU.

The kernel library is replaced by a recorder and the connection sits on fake ps base addresses with CPU tensors
(tests/hbm_fake.py), so a step -- pull, the network's forward, a BCE backward, push -- runs here end to end.  Each
step is recorded as the native calls it makes, in order, with their integer and float arguments and, for each
pointer, its role: ``var{i}.w`` / ``.s1`` / ``.s2`` for a master or slot (``+offset`` inside one), ``shadow{i}`` for a
bf16 shadow, the roles held by a device pointer array (a group's tables or slots), the values of an int32 column ->
table map, and ``temp#k`` (``+offset``) for anything else.  Raw addresses are never recorded.  The recorder answers
tfy_ps_push_rows_scratch_bytes and does not record it.  Each step also records traffic_per_step().

The fixture tests/golden/ps_hbm_step_trace.json holds the trace of every case; ``python
tests/test_ps_hbm_step_trace.py`` writes it again.
"""
import ctypes
import json
import os
import sys
import types
from contextlib import ExitStack
from unittest import mock

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hbm_fake import hbm_connection  # noqa: E402
from tf_yarn_b200.estimator import canned  # noqa: E402
from tf_yarn_b200.estimator import feature_column as fc  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ps_hbm_step_trace.json")
SWITCHES = ("TFY_PS_FUSE_FIRST", "TFY_PS_FUSE_WIDE")


def _scratch_bytes(n):
    return 256 + 8 * int(n)


# ------------------------------------------------------------------------------------------------ harness
class _Recorder:
    """Stands in for the kernel library: answers the scratch size query, records every other call."""

    def __init__(self):
        self.calls = []
        self.role = None           # pointer -> role, set per step

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        if name == "tfy_ps_push_rows_scratch_bytes":
            return _scratch_bytes
        argtypes = native._EXTRA_DECLS[name][0]

        def call(*args):
            assert len(args) == len(argtypes), (name, len(args), len(argtypes))
            temps = {}
            out = [name]
            for t, a in zip(argtypes, args):
                if a is None:
                    out.append(None)
                elif t is ctypes.c_void_p and int(a) == 0:          # the stream (stream 0 here)
                    out.append(0)
                elif t is ctypes.c_void_p:
                    out.append(self.role(int(a), temps))
                elif t is ctypes.c_float:
                    out.append(float(a))
                else:
                    assert isinstance(a, int), (name, t, a)
                    out.append(int(a))
            self.calls.append(out)
            return 0
        return call


class _Pointers:
    """Roles of the pointers a step passes: the fake ps regions by address, every other pointer by the tensor whose
    data_ptr() produced it (Tensor.data_ptr is wrapped while a step runs, which also keeps those tensors alive, so
    that no two of them share an address within a step)."""

    def __init__(self, conn):
        self.spans = []
        lay = conn.layout
        for i in range(len(lay.numel)):
            for slot, nm in enumerate(("w", "s1", "s2")[:1 + lay.var_slots[i]]):
                self.spans.append((conn.master_ptr(i, slot), 4 * lay.numel[i], f"var{i}.{nm}"))
        self.shadows = {conn.shadow_ptr(i): f"shadow{i}" for i in conn.gemm}
        self.seen = {}             # data_ptr -> tensor

    def fake(self, ptr):
        if ptr in self.shadows:
            return self.shadows[ptr]
        for start, nbytes, nm in self.spans:
            if start <= ptr < start + nbytes:
                return nm if ptr == start else f"{nm}+{ptr - start}"
        return None

    def __call__(self, ptr, temps):
        role = self.fake(ptr)
        if role is not None:
            return role
        t = self.seen.get(ptr)
        if t is not None and t.dtype == torch.int64 and 0 < t.numel() <= 64 and \
                all(self.fake(int(v)) is not None for v in t.reshape(-1).tolist()):
            return [self.fake(int(v)) for v in t.reshape(-1).tolist()]          # a device pointer array
        if t is not None and t.dtype == torch.int32:
            return {"table_of": t.reshape(-1).tolist()}
        for base, t in self.seen.items():
            nbytes = t.untyped_storage().nbytes()
            start = t.untyped_storage().data_ptr()
            if start <= ptr < start + nbytes:
                k = temps.setdefault(start, len(temps))
                return f"temp#{k}" if ptr == start else f"temp#{k}+{ptr - start}"
        raise AssertionError(f"pointer {ptr:#x} of no tensor")


# ------------------------------------------------------------------------------------------------ cases
V = 50


def _cat(key, v=V):
    return fc.categorical_column_with_hash_bucket(key, v)


def _wide_deep(emb_dim=64, n_cat=3, n_num=5, hidden=(64, 32), **kw):
    cats = [_cat(f"c{i}") for i in range(n_cat)]
    num = fc.numeric_column("numeric", (n_num,))
    return canned._WideDeepNet([num] + cats, [fc.embedding_column(c, emb_dim) for c in cats] + [num], list(hidden), 1,
                               **kw)


def _deep(columns, hidden=(64,)):
    return canned._WideDeepNet([], columns, list(hidden), 1)


def _wide(columns, combiner="sum"):
    return canned._WideDeepNet(columns, [], [], 1, sparse_combiner=combiner)


def _k5_shared_pairs():
    s1 = fc.shared_embedding_columns([_cat("c0"), _cat("c2")], 64)
    s2 = fc.shared_embedding_columns([_cat("c1"), _cat("c3")], 64)
    return _deep([s1[0], s2[0], s1[1], s2[1], fc.embedding_column(_cat("c4"), 64), fc.numeric_column("n")])


def _k5_weighted(combiners):
    cols = [_cat("c0"), fc.weighted_categorical_column(_cat("c1"), "c1_w"), _cat("c2")]
    return _deep([fc.embedding_column(c, 64, k) for c, k in zip(cols, combiners)] + [fc.numeric_column("n", (3,))])


def _k5_mixed_shared():
    sh = fc.shared_embedding_columns([_cat("c0"), _cat("c2")], 64)
    return _deep([sh[0], fc.embedding_column(_cat("c1"), 64), sh[1], fc.embedding_column(_cat("c3"), 64),
                  fc.numeric_column("n")])


def _mixed_v():
    bucket = fc.bucketized_column(fc.numeric_column("age", (2,)), [20.0, 30.0, 40.0])
    cross = fc.crossed_column(["c0", fc.categorical_column_with_identity("c1", 7)], 40)
    vocab = fc.categorical_column_with_vocabulary_list("c2", [3, 5, 7, 11, 13], num_oov_buckets=2)
    return _wide([bucket, cross, vocab, _cat("c3")])


def _unfused(combiner, weighted=False):
    cols = [_cat("c0"), fc.weighted_categorical_column(_cat("c1"), "c1_w") if weighted else _cat("c1")]
    return _deep([fc.embedding_column(c, 16, combiner) for c in cols] + [fc.numeric_column("n", (3,))], (32,))


def _shared_no_k5():
    sh = fc.shared_embedding_columns([_cat("c0"), _cat("c1"), _cat("c2")], 32, "sqrtn")
    return _deep([sh[2], fc.numeric_column("n"), sh[0], sh[1]], (16,))


class _PlainBag(nn.Module):
    """A torch.nn.EmbeddingBag (sum) fed [B, L] ids with per_sample_weights, then a Linear served remotely."""

    def __init__(self):
        super().__init__()
        self.emb = nn.EmbeddingBag(V, 16, mode="sum")
        self.out = nn.Linear(16, 8)
        self.logits = nn.Linear(8, 1)

    def forward(self, f):
        return self.logits(F.relu(self.out(self.emb(f["c0"], per_sample_weights=f.get("c0_w")))))


def _by_name(**opts):
    """Variable names of the tables of the given column keys (deep embeddings) -> optimizer name."""
    return {f"dense_features.embeddings.{k}.weight": o for k, o in opts.items()}


WIDE_FTRL = "linear.tables.{}.weight"


def _case(build, batches, opt="adagrad", by_name=None, env=None):
    return dict(build=build, batches=batches, opt=opt, by_name=by_name, env=env or {})


# a batch: column key -> ids per example (1 = one-hot [B]), "w" weights, "n" numeric width; B examples
ONE = {"L": 1}
MULTI = {"L": 3}
CASES = {
    "k5_one_hot": _case(_wide_deep, [ONE, ONE],
                        by_name={WIDE_FTRL.format(f"c{i}"): "ftrl" for i in range(3)}),
    "k5_multi_hot": _case(_wide_deep, [MULTI, dict(MULTI, ragged=True)]),
    "k5_emb16_unfused": _case(lambda: _wide_deep(emb_dim=16), [ONE, MULTI]),
    "k5_shared_pairs": _case(_k5_shared_pairs, [ONE, MULTI]),
    "k5_mixed_optimizers": _case(lambda: _deep([fc.embedding_column(_cat(f"c{i}"), 64) for i in range(4)] +
                                               [fc.numeric_column("n")]),
                                 [ONE, MULTI], by_name=_by_name(c0="sgd", c1="adam", c2="ftrl")),
    "k5_mixed_optimizers_shared": _case(_k5_mixed_shared, [ONE, MULTI],
                                        by_name=_by_name(c1="ftrl", c3="adam")),
    "k5_weighted_one_combiner": _case(lambda: _k5_weighted(["sqrtn"] * 3), [ONE, MULTI]),
    "k5_weighted_mixed_combiners": _case(lambda: _k5_weighted(["sum", "mean", "sqrtn"]), [ONE, MULTI]),
    "k5_weighted_mixed_optimizers": _case(lambda: _k5_weighted(["sum", "mean", "sqrtn"]), [MULTI],
                                          by_name=_by_name(c0="ftrl", c2="sgd")),
    "k5_big_batch": _case(lambda: _wide_deep(hidden=(32,)), [dict(ONE, B=2100), dict(MULTI, B=700)]),
    "wide_sum": _case(lambda: _wide([_cat(f"c{i}") for i in range(3)]), [ONE, MULTI], opt="ftrl"),
    "wide_mean": _case(lambda: _wide([_cat(f"c{i}") for i in range(3)], "mean"), [ONE, MULTI], opt="ftrl"),
    "wide_weighted": _case(lambda: _wide([_cat("c0"), fc.weighted_categorical_column(_cat("c1"), "c1_w")]),
                           [ONE, MULTI], opt="ftrl"),
    "wide_mixed_v": _case(_mixed_v, [ONE, MULTI], opt="ftrl"),
    "wide_one_table_adam": _case(lambda: _wide([_cat("c0")]), [ONE, MULTI], opt="adam"),
    "unfused_sum": _case(lambda: _unfused("sum"), [ONE, MULTI]),
    "unfused_mean": _case(lambda: _unfused("mean"), [ONE, MULTI], opt="sgd"),
    "unfused_sqrtn": _case(lambda: _unfused("sqrtn"), [ONE, MULTI], opt="adam"),
    "unfused_weighted": _case(lambda: _unfused("mean", weighted=True), [ONE, MULTI], opt="ftrl"),
    "plain_embedding_bag": _case(_PlainBag, [ONE, MULTI, dict(MULTI, psw=True)]),
    "shared_without_k5": _case(_shared_no_k5, [ONE, MULTI], opt="ftrl"),
    "fuse_first_off": _case(_wide_deep, [ONE, MULTI], env={"TFY_PS_FUSE_FIRST": "0"}),
    "fuse_wide_off": _case(_wide_deep, [ONE, MULTI], env={"TFY_PS_FUSE_WIDE": "0"}),
}


def _features(net, spec, seed):
    """One batch for every input the network reads: hashed / identity ids (one per example, or spec["L"] with -1
    missing), weights, numeric values and bucketized sources."""
    B, L = spec.get("B", 16), spec["L"]
    g = torch.Generator().manual_seed(seed)
    f = {}
    for i in range(5):
        ids = torch.randint(0, 7, (B, L), generator=g)
        if L > 1:
            ids[:, -1] = torch.where(torch.rand(B, generator=g) < 0.5, -1, ids[:, -1])
        if spec.get("ragged") and i == 2:
            ids = ids[:, :2]
        f[f"c{i}"] = ids[:, 0] if L == 1 and i % 2 == 0 else ids
        f[f"c{i}_w"] = torch.rand(ids.shape, generator=g)
    f["n"] = torch.randn(B, _num_width(net), generator=g)
    f["numeric"] = torch.randn(B, 5, generator=g)
    f["age"] = torch.rand(B, 2, generator=g) * 50
    if isinstance(net, _PlainBag) and not spec.get("psw"):
        del f["c0_w"]
    return f


def _num_width(net):
    df = getattr(net, "dense_features", None)
    cols = df.columns if df is not None else []
    return next((c.dim for c in cols if isinstance(c, fc.NumericColumn) and c.key == "n"), 3)


def run_case(name):
    """[{calls, traffic} for each step of the case]."""
    case = CASES[name]
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(case["env"])
    rec = _Recorder()
    steps = []
    with ExitStack() as stack:
        stack.enter_context(mock.patch.dict(os.environ, env, clear=True))
        stack.enter_context(mock.patch.object(native, "load", lambda: rec))
        stack.enter_context(mock.patch.object(torch.cuda, "current_stream",
                                              lambda device=None: types.SimpleNamespace(cuda_stream=0)))
        torch.manual_seed(0)
        net = case["build"]()
        conn = hbm_connection(net, case["opt"], by_name=case["by_name"], lib=rec)
        conn.install(net)
        pointers = _Pointers(conn)
        rec.role = pointers
        data_ptr = torch.Tensor.data_ptr

        def recorded_data_ptr(t):
            p = data_ptr(t)
            pointers.seen[p] = t
            return p
        stack.enter_context(mock.patch.object(torch.Tensor, "data_ptr", recorded_data_ptr))
        for k, spec in enumerate(case["batches"]):
            f = _features(net, spec, seed=k)
            y = (torch.arange(f["numeric"].shape[0]) % 2).float()
            rec.calls, pointers.seen = [], {}
            conn.pull(net)
            net.zero_grad()
            out = net(f).float()
            F.binary_cross_entropy_with_logits(out[:, 0], y).backward()
            conn.push(net)
            steps.append({"calls": rec.calls, "traffic": conn.traffic_per_step(),
                          "fused": [bool(conn.fused_first), bool(conn.fused_wide), conn.shared_collections]})
    return steps


def _fmt_arg(a):
    return a if isinstance(a, str) else json.dumps(a)


def fixture_of(steps):
    return [dict(s, calls=[f"{c[0]}({', '.join(_fmt_arg(a) for a in c[1:])})" for c in s["calls"]]) for s in steps]


# ------------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def traces():
    return {}


def _trace(traces, name):
    if name not in traces:
        traces[name] = run_case(name)
    return traces[name]


def test_the_fixture_lists_every_case(golden):
    assert sorted(golden) == sorted(CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_step_trace_matches_the_fixture(golden, traces, name):
    assert fixture_of(_trace(traces, name)) == golden[name]


def test_a_one_hot_wide_and_deep_step_is_k5_and_the_multi_table_kernels(traces):
    step = _trace(traces, "k5_one_hot")[0]
    names = [c[0] for c in step["calls"]]
    assert names == ["tfy_ps_pull", "tfy_ps_multi_bag", "tfy_ps_gather_gemm", "tfy_gemm_bf16", "tfy_dense_bwd",
                     "tfy_dense_bwd", "tfy_ps_multi_push_rows", "tfy_ps_multi_push_rows", "tfy_ps_push"], names
    assert step["traffic"]["launches_per_step"] == 13


def test_every_sparse_entry_point_is_exercised(traces):
    seen = {c[0] for name in CASES for step in _trace(traces, name) for c in step["calls"]}
    assert {"tfy_ps_embedding_bag", "tfy_ps_push_rows", "tfy_ps_multi_bag", "tfy_ps_multi_push_rows",
            "tfy_ps_gather_gemm", "tfy_ps_multi_bag_weighted", "tfy_ps_multi_push_rows_weighted",
            "tfy_ps_multi_push_rows_shared"} <= seen, seen


if __name__ == "__main__":
    out = {name: fixture_of(run_case(name)) for name in sorted(CASES)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {GOLDEN}: {len(out)} cases")
