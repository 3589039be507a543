"""GPU tests of Keras gradient accumulation (``gradient_accumulation_steps``; run with `pytest -m gpu` on an H100).

The accumulate kernel against a torch fp32 sequential sum, bit for bit; the MNIST-CNN fast path and a small
autograd model on the graph engine with N = 4: parameters untouched on three batches and updated on the fourth, the
update against the fp32 CPU-semantics engine, graph replay against eager launches, reproducibility, fresh dropout
masks on every batch, a scheduled Adam, a resume in the middle of an accumulation, and the launches per batch.  With
2+ GPUs, tests/gpu/grad_accum_check.py covers the P2P and NVLS transports.
"""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 4


def _mnist_elems():
    from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn
    m = keras_mnist_cnn()
    m.build((28, 28, 1))
    return sum((p.numel() + 7) // 8 * 8 for p in m.net.parameters())


@pytest.mark.parametrize("clear", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("n", [8, 4096 + 8, "mnist"])
def test_kernel_matches_a_torch_fp32_sequential_sum_bit_for_bit(n, dtype, clear):
    from tf_yarn_b200.ops import native
    from tf_yarn_b200.parallel import comm  # noqa: F401  (declares tfy_grad_accumulate's argument types)
    lib = native.load()
    n = _mnist_elems() if n == "mnist" else n
    g = torch.Generator(device="cuda").manual_seed(11)
    acc = torch.zeros(n, dtype=torch.float32, device="cuda")
    want = torch.zeros(n, dtype=torch.float32, device="cuda")
    for _ in range(3):
        src = (torch.randn(n, device="cuda", generator=g)
               * 10.0 ** torch.randint(-4, 3, (n,), device="cuda", generator=g)).to(dtype)
        keep = src.clone()
        native.check(lib.tfy_grad_accumulate(acc.data_ptr(), src.data_ptr(), native.BF16 if dtype == torch.bfloat16
                                             else native.F32, n, int(clear), None, 0, 0,
                                             torch.cuda.current_stream().cuda_stream), "tfy_grad_accumulate")
        want = want + keep.float()
        torch.cuda.synchronize()
        assert torch.equal(acc.view(torch.int32), want.view(torch.int32))
        assert torch.equal(src, torch.zeros_like(src)) if clear else torch.equal(src, keep)


def _mnist_like(dropout=0.0):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="mnist_cnn_accum")
    m.add(layers.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)))
    m.add(layers.Conv2D(64, (3, 3), activation="relu"))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(dropout))
    m.add(layers.Flatten())
    m.add(layers.Dense(128, activation="relu"))
    m.add(layers.Dropout(dropout))
    m.add(layers.Dense(10))
    return m


def _mlp():
    """Outside the fast-path grammar (a mean-squared-error head): the autograd graph engine."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="mlp_accum")
    m.add(layers.Dense(64, activation="relu", input_shape=(32,)))
    m.add(layers.Dense(10))
    return m


def _batches(kind, n_batches, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_batches):
        if kind == "mnist":
            y = rs.randint(0, 10, 128).astype("int64")
            x = (rs.rand(128, 28, 28, 1) * 0.5 + (y[:, None, None, None] / 20.0)).astype("float32")
        else:
            x = rs.randn(128, 32).astype("float32")
            y = rs.randn(128, 10).astype("float32")
        out.append((torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()))
    return out


def _engine(kind, opt, use_graph=True, dropout=0.0, seed=7):
    from tf_yarn_b200 import keras
    torch.manual_seed(seed)
    m = _mnist_like(dropout) if kind == "mnist" else _mlp()
    loss = keras.losses.SparseCategoricalCrossentropy(from_logits=True) if kind == "mnist" else "mse"
    m.compile(loss=loss, optimizer=opt, use_cuda_graph=use_graph)
    m.build((28, 28, 1) if kind == "mnist" else (32,))
    init = copy.deepcopy(m.net).float()
    x0, y0 = _batches(kind, 1)[0]
    m._ensure_engine(x0, y0)
    return m, m._engine, init


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _adam(**kw):
    from tf_yarn_b200 import keras
    return keras.optimizers.Adam(1e-3, gradient_accumulation_steps=N, **kw)


@pytest.mark.parametrize("kind", ["mnist", "mlp"])
def test_parameters_move_on_every_fourth_batch_and_match_the_fp32_engine(kind):
    from tf_yarn_b200.keras.engine import EagerTrainEngine
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m, eng, init = _engine(kind, _adam())
    assert isinstance(eng, FastSequentialEngine) == (kind == "mnist")
    batches = _batches(kind, 2 * N)
    before = eng.fused.master.clone()
    launches = []
    for s, (x, y) in enumerate(batches):
        k0 = eng.kernel_launches
        eng.train_step(x, y)
        launches.append(eng.kernel_launches - k0)
        assert eng.fused.step_count == s + 1                # the counter counts batches
        moved = not torch.equal(eng.fused.master, before)
        assert moved == ((s + 1) % N == 0), s
        before = eng.fused.master.clone()
        if s == N - 1:
            after_first = [t.clone() for t in eng.master_tensors()]
    if kind == "mnist":      # the fast path's 9 step kernels, + the accumulate kernel, + K4 on an update batch
        assert launches == [10, 10, 10, 11] * 2, launches
    else:
        assert launches == [1, 1, 1, 2] * 2, launches
    # the first update against the fp32 CPU-semantics engine on the same weights and batches
    ref = EagerTrainEngine(init.cuda(), m._loss_fn, _adam(), [], torch.device("cuda"))
    for x, y in batches[:N]:
        ref.train_step(x, y)
    for a, b in zip(after_first, [p.detach() for p in ref.net.parameters()]):
        denom = b.abs().max().clamp_min(2e-2)
        assert ((a - b).abs().max() / denom) < 0.15, ((a - b).abs().max(), denom)


@pytest.mark.parametrize("kind", ["mnist", "mlp"])
def test_graph_replay_equals_eager_launches_and_runs_are_bit_identical(kind):
    batches = _batches(kind, 2 * N + 2)
    runs = []
    for use_graph in (True, True, False):
        m, eng, _ = _engine(kind, _adam(), use_graph=use_graph)
        for x, y in batches:
            eng.train_step(x, y)
        torch.cuda.synchronize()
        runs.append((eng.fused.master.clone(), eng.fused.flat_params.clone(), eng.fused.flat_acc.clone()))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(_bits(a), _bits(b))


def test_dropout_masks_differ_between_the_batches_of_one_update():
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    m, eng, _ = _engine("mnist", _adam(), dropout=0.5)
    x, y = _batches("mnist", 1)[0]
    losses = [float(eng.train_step(x, y)["loss"]) for _ in range(N - 1)]   # the same batch, the same weights
    # the fast path's dropout kernels draw from the device step counter (autograd would draw from torch's RNG)
    assert isinstance(eng, FastSequentialEngine) and eng._launches_per_accum_step == 10
    assert len(set(losses)) == N - 1, losses


@pytest.mark.parametrize("kind", ["mnist", "mlp"])
def test_scheduled_adam_reads_the_schedule_at_the_batch_index(kind):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.engine import EagerTrainEngine
    sch = keras.optimizers.schedules.PiecewiseConstantDecay([2, 5, 9], [1e-3, 5e-4, 2e-4, 1e-4])
    make = lambda: keras.optimizers.Adam(sch, gradient_accumulation_steps=N)  # noqa: E731
    m, eng, init = _engine(kind, make())
    batches = _batches(kind, 3 * N)
    for s, (x, y) in enumerate(batches):
        assert eng.get_learning_rate() == float(np.float32(sch(s)))          # the rate batch s would update with
        eng.train_step(x, y)
    ref = EagerTrainEngine(init.cuda(), m._loss_fn, make(), [], torch.device("cuda"))
    for x, y in batches:
        ref.train_step(x, y)
    for a, b in zip(eng.master_tensors(), [p.detach() for p in ref.net.parameters()]):
        denom = b.abs().max().clamp_min(2e-2)
        assert ((a - b).abs().max() / denom) < 0.15, ((a - b).abs().max(), denom)


@pytest.mark.parametrize("kind", ["mnist", "mlp"])
def test_resume_in_the_middle_of_an_accumulation_is_bit_identical(kind):
    batches = _batches(kind, 2 * N + 1)
    _, straight, _ = _engine(kind, _adam())
    for x, y in batches:
        straight.train_step(x, y)
    _, first, _ = _engine(kind, _adam())
    for x, y in batches[:N + 2]:
        first.train_step(x, y)
    state = first.state_dict()
    assert state["step"] == N + 2 and "grad_accum" in state
    _, resumed, _ = _engine(kind, _adam(), seed=99)            # other initial weights: the state replaces them
    resumed.load_state_dict(state)
    for x, y in batches[N + 2:]:
        resumed.train_step(x, y)
    torch.cuda.synchronize()
    for name in ("master", "flat_params", "flat_acc", "s1", "s2"):
        assert torch.equal(_bits(getattr(resumed.fused, name)), _bits(getattr(straight.fused, name))), name


def test_off_keeps_one_graph_per_slot_and_ten_launches():
    from tf_yarn_b200 import keras
    m, eng, _ = _engine("mnist", keras.optimizers.Adam(1e-3))
    x, y = _batches("mnist", 1)[0]
    k0 = eng.kernel_launches
    eng.train_step(x, y)
    assert eng.kernel_launches - k0 == 10 and eng._launches_per_step == 10
    assert eng.fused.flat_acc is None and eng._acc_graphs == [None, None]


@pytest.mark.parametrize("scheduled", [False, True], ids=["constant", "scheduled"])
def test_local_fused_step_over_the_accumulator_matches_torch_adam_at_the_batch_index(scheduled):
    """LOCAL mode, bf16 gradients and parameters: the accumulate kernel and the fused step over the fp32 accumulator
    against torch Adam fed the same fp32 sums times fl32(1/N), with the rate schedule(s) and the bias correction at
    t = s + 1 for the update's batch index s; the bias correction at the update count k + 1 is shown to differ."""
    from tf_yarn_b200.keras import optimizers as kopt
    from tf_yarn_b200.keras import schedules
    from tf_yarn_b200.keras.engine import _solo_communicator
    from tf_yarn_b200.parallel.comm import FusedShardedOptimizer
    shapes = [(33, 17), (129,), (7, 5, 3)]
    sch = schedules.PiecewiseConstantDecay([4, 9], [1e-2, 5e-3, 2e-3])
    desc = kopt.Adam(sch if scheduled else 1e-2, gradient_accumulation_steps=N)
    fo = FusedShardedOptimizer(_solo_communicator(0), shapes, desc.to_spec(), param_dtype=torch.bfloat16,
                               grad_dtype=torch.bfloat16, accumulation_steps=N)
    g = torch.Generator(device="cuda").manual_seed(5)
    init = [torch.randn(sh, device="cuda", generator=g) * 0.3 for sh in shapes]
    fo.init_from(init, broadcast_root=None)
    refs = {at: [t.clone().requires_grad_(True) for t in init] for at in ("batch", "update")}
    opts = {at: torch.optim.Adam(refs[at], lr=1e-2, eps=1e-7) for at in refs}
    acc = [torch.zeros(sh, device="cuda") for sh in shapes]
    scale = float(np.float32(1.0 / N))
    for s in range(3 * N):
        grads = [(torch.randn(sh, device="cuda", generator=g) * 0.5).to(torch.bfloat16) for sh in shapes]
        for gv, gr in zip(fo.grad_views, grads):
            gv.copy_(gr)
        update = (s + 1) % N == 0
        fo.accumulate(advance=not update)
        if update:
            fo.step_accumulated()
        acc = [a + gr.float() for a, gr in zip(acc, grads)]
        if not update:
            continue
        for at, t in (("batch", s), ("update", s // N)):
            for grp in opts[at].param_groups:
                grp["lr"] = float(np.float32(sch(s))) if scheduled else 1e-2
            for r, a in zip(refs[at], acc):
                r.grad = a * scale
                st = opts[at].state[r]
                if not st:
                    st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(r), torch.zeros_like(r)
                st["step"] = torch.tensor(float(t))
            opts[at].step()
        acc = [torch.zeros_like(a) for a in acc]
    torch.cuda.synchronize()
    assert fo.step_count == 3 * N and float(fo.flat_acc.abs().max()) == 0.0
    master = fo.unflatten(fo.master)
    for t, r in zip(master, refs["batch"]):
        torch.testing.assert_close(t, r.detach(), rtol=1e-4, atol=1e-5)
    assert not all(torch.allclose(t, r.detach(), rtol=1e-4, atol=1e-5) for t, r in zip(master, refs["update"]))


def _ngpu() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_p2p_and_nvls_accumulation_multi_gpu():
    n = min(_ngpu(), 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29631", "tests/gpu/grad_accum_check.py"]
    res = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert res.returncode == 0 and "GRAD ACCUM CHECK OK" in res.stdout, res.stdout[-4000:]
