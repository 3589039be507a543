"""The float64 parameter-server reference (tests/ps_reference.py) pinned on any box: its dense push agrees with the
shared-memory CPU plane (estimator/ps.py ``WorkerConnection.push``), and its duplicate-row handling matches cases
worked out by hand.  The GPU kernels are checked against the same reference in test_gpu_ps_kernels.py."""
import numpy as np
import pytest
import torch

import ps_reference as ref
from tf_yarn_b200.estimator import ps

_KIND = {"sgd": ref.SGD, "adagrad": ref.ADAGRAD, "adam": ref.ADAM, "ftrl": ref.FTRL}


def _cpu_hyper(kind, wd):
    # the CPU plane's layout hypers (OptimizerSpec): FTRL keeps l1, l2 in p1, p2 and beta in eps
    return {"sgd": dict(lr=0.1, p1=0.0, p2=0.0, eps=0.0),
            "adagrad": dict(lr=0.1, p1=0.0, p2=0.0, eps=1e-7),
            "adam": dict(lr=0.01, p1=0.9, p2=0.999, eps=1e-7),
            "ftrl": dict(lr=0.05, p1=0.003, p2=0.01, eps=0.5)}[kind] | {"wd": wd, "init_s1": 0.1, "flags": 0}


@pytest.mark.parametrize("wd", [0.0, 0.02])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam", "ftrl"])
def test_reference_dense_push_matches_the_cpu_plane(tmp_path, kind, wd):
    hyper = _cpu_hyper(kind, wd)
    net = torch.nn.Module()
    net.a = torch.nn.Parameter(torch.randn(5, 7, generator=torch.Generator().manual_seed(0)))
    net.b = torch.nn.Parameter(torch.randn(13, generator=torch.Generator().manual_seed(1)))
    named = ps._named_trainables(net)
    lay = ps.Layout([(n, list(p.shape)) for n, p in named], 1, kind, hyper)
    shard = ps.ShmShard(str(tmp_path / "shard"), lay.shard_elems[0], create=True)
    try:
        shard.data.zero_()
        conn = ps.WorkerConnection(lay, [shard], [n for n, _ in named])
        state = []
        for i, (_, p) in enumerate(named):
            conn._region(i).copy_(p.detach().reshape(-1))
            if kind in ("adagrad", "ftrl"):
                conn._region(i, 1).fill_(hyper["init_s1"])
            n = p.numel()
            state.append([p.detach().reshape(-1).double().numpy().copy(),
                          np.full(n, hyper["init_s1"] if kind in ("adagrad", "ftrl") else 0.0), np.zeros(n)])
        shard.set_global_step(0)
        # the kernels' hyper-parameter convention: FTRL p3 = beta
        khp = dict(lr=hyper["lr"], eps=hyper["eps"], wd=wd, p1=hyper["p1"], p2=hyper["p2"], p3=hyper["eps"])
        rng = np.random.default_rng(2)
        for step in range(5):
            for i, (_, p) in enumerate(named):
                g = rng.standard_normal(p.shape).astype(np.float32) * (1e-4 if kind == "adam" else 0.5)
                p.grad = torch.from_numpy(g)
                w, s1, s2 = state[i]
                ref.dense_push(_KIND[kind], w, s1, s2, g.reshape(-1), khp,
                               scale=ref.adam_scale(step + 1, hyper["p1"], hyper["p2"]))
            conn.push(net)
            conn.increment_global_step()
        for i, (_, p) in enumerate(named):
            w, s1, s2 = state[i]
            # the CPU plane computes in fp32: a handful of roundings per step on values of order |w| + |the updates|
            tol = 5 * 8 * ref.EPS32 * (np.abs(w) + np.abs(w - p.detach().reshape(-1).double().numpy()) + 1e-3)
            got = conn._region(i).double().numpy()
            assert np.all(np.abs(got - w) <= tol), (kind, i, np.abs(got - w).max())
            for slot, want in ((1, s1), (2, s2)):
                if slot <= lay.var_slots[i]:
                    got = conn._region(i, slot).double().numpy()
                    # FTRL's z adds (sqrt(n') - sqrt(n)) / lr * w every step: each square root carries a rounding of
                    # sqrt(n) eps, so the error scales with sqrt(n) / lr * |w|, not with |z|
                    mag = np.sqrt(s1) / hyper["lr"] * np.abs(w).max() + 1.0 if kind == "ftrl" and slot == 2 else 0.0
                    tol = 5 * 8 * ref.EPS32 * (np.abs(want) + mag) + 1e-12
                    assert np.all(np.abs(got - want) <= tol), (kind, i, slot, np.abs(got - want).max())
    finally:
        shard.unlink()


def test_duplicate_rows_are_summed_before_adagrad():
    """Two occurrences of one row: ONE step with g1 + g2 -- acc = init + (g1 + g2)^2, not init + g1^2 + g2^2."""
    hp = dict(lr=0.1, eps=1e-7, p1=0.0, p2=0.0, p3=0.0)
    table, acc = np.array([[1.0, -2.0], [3.0, 4.0]]), np.full((2, 2), 0.1)
    dout = np.array([[0.5, -1.0], [0.25, 3.0], [7.0, 7.0]])
    ids = np.array([[[1], [1], [-1]]])                        # row 1 twice, then an id that is skipped
    ref.sparse_push(ref.ADAGRAD, [table], [acc], None, ids, dout, 2, hp)
    g = np.array([0.75, 2.0])
    assert np.allclose(acc[1], 0.1 + g * g) and np.all(acc[0] == 0.1)
    assert np.allclose(table[1], [3.0, 4.0] - 0.1 * g / (np.sqrt(0.1 + g * g) + 1e-7))
    assert np.all(table[0] == [1.0, -2.0])


def test_duplicate_rows_ftrl_weight_follows_the_final_z():
    hp = dict(lr=0.05, eps=0.0, p1=0.003, p2=0.01, p3=0.5)
    w0 = np.array([[0.2]])
    table, n, z = w0.copy(), np.array([[0.1]]), np.array([[0.0]])
    ids = np.array([[[0, 0, 0]]])                              # one bag, the same id three times, mean
    dout = np.array([[0.6]])
    ref.sparse_push(ref.FTRL, [table], [n], [z], ids, dout, 1, hp, mean=True)
    g = 0.6 * 3 / 3                                            # the sum of three occurrences over L = 3
    n_new = 0.1 + g * g
    z_new = g - (np.sqrt(n_new) - np.sqrt(0.1)) / 0.05 * 0.2
    assert np.isclose(n[0, 0], n_new) and np.isclose(z[0, 0], z_new)
    assert np.isclose(table[0, 0], -(z_new - np.sign(z_new) * 0.003) / ((0.5 + np.sqrt(n_new)) / 0.05 + 0.02))
    assert table[0, 0] == ref.ftrl_w(z, n, 0.05, 0.003, 0.01, 0.5)[0, 0]


def test_lazy_adam_leaves_rows_outside_the_batch_alone():
    hp = dict(lr=0.01, eps=1e-7, p1=0.9, p2=0.999, p3=0.0)
    table, m, v = np.ones((3, 1)), np.full((3, 1), 0.5), np.full((3, 1), 0.25)
    ref.sparse_push(ref.ADAM, [table], [m], [v], np.array([[[2], [5]]]), np.array([[1e-4], [1e-4]]), 1, hp,
                    scale=ref.adam_scale(3, 0.9, 0.999))
    assert np.all(table[:2] == 1.0) and np.all(m[:2] == 0.5) and np.all(v[:2] == 0.25)
    assert table[2, 0] != 1.0


def test_bag_mean_divides_by_l_and_skips_out_of_range_ids():
    table = np.arange(8.0).reshape(4, 2)
    out = ref.bag(table, np.array([[0, 3, 9], [-1, -1, 2]]), mean=True)
    assert np.allclose(out, [[(0 + 6) / 3, (1 + 7) / 3], [4 / 3, 5 / 3]])
    assert np.allclose(ref.multi_bag([table, 2 * table], np.array([[1], [4]])), [[2.0, 3.0]])


def test_bf16_rounding_is_nearest_even():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -1.0 - 2 ** -8, 3.0e38, 1e-40], np.float32)
    want = torch.from_numpy(x).bfloat16().double().numpy()
    assert np.array_equal(ref.bf16_round(x), want)
    sh = ref.shadow(np.arange(6.0), 3, 8)
    assert sh.shape == (2, 8) and np.all(sh[:, 3:] == 0) and np.array_equal(sh[1, :3], [3.0, 4.0, 5.0])
