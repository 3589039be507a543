"""The confusion-histogram kernel (ops/csrc/tfy_confusion.cu) on the H100: against the float64 reference at sizes from
one element to 5M, fp32 / bf16 predictions, fp32 / int64 labels, with and without weights, on bucket edges and at both
threshold limits; bit-identical across runs, between eager and CUDA-graph replay, and for batches accumulated one at a
time in a graph; the error flags; AUC through GraphTrainEngine's captured step; and a GPU-placed canned estimator."""
import numpy as np
import pytest
import torch

import confusion_reference as ref
from tf_yarn_b200 import data, keras
from tf_yarn_b200 import estimator as est
from tf_yarn_b200.estimator import feature_column as fc
from tf_yarn_b200.keras.engine import GraphTrainEngine
from tf_yarn_b200.ops import confusion

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# (prediction dtype, label dtype, weighted)
COMBOS = [(torch.float32, torch.float32, False), (torch.bfloat16, torch.int64, False),
          (torch.float32, torch.int64, True), (torch.bfloat16, torch.float32, True)]


def _batch(n, T, pdt, ldt, weighted, seed, per_sample=1):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(n, generator=g)
    edges = torch.from_numpy(ref.edge_values(T))
    k = min(n // 4, edges.numel())
    if k:
        p[:k] = edges[torch.randint(0, edges.numel(), (k,), generator=g)]      # exactly on / next to bucket edges
    y = (torch.rand(n, generator=g) < p).to(ldt)
    p = p.to(pdt)
    w = None
    if weighted:
        w = torch.rand(n // per_sample, generator=g) * 2
        w[torch.rand(w.numel(), generator=g) < 0.1] = 0.0
    return y, p, w


def _gpu_hist(st, y, p, w=None):
    st.update(y.to(DEV), p.to(DEV), None if w is None else w.to(DEV))
    torch.cuda.synchronize()
    return st.histogram().numpy()


def _ref_hist(y, p, w, T, thresholds=None):
    return ref.histogram(y.numpy(), p.float().numpy(), None if w is None else w.numpy(), T, thresholds)


def _check(h, want, weighted):
    if weighted:
        # fp64 sums of at most 5M terms in another order: |error| <= n * 2^-53 * sum|v|, far inside this bound
        np.testing.assert_allclose(h, want, rtol=1e-9, atol=1e-9)
    else:
        np.testing.assert_array_equal(h, want)                    # counts are exact in fp64


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097, (1 << 20) + 7, 5_000_000])
@pytest.mark.parametrize("pdt,ldt,weighted", COMBOS)
def test_kernel_histogram_matches_the_reference(n, pdt, ldt, weighted):
    T = 200
    y, p, w = _batch(n, T, pdt, ldt, weighted, seed=n)
    st = confusion.ConfusionState(T)
    _check(_gpu_hist(st, y, p, w), _ref_hist(y, p, w, T), weighted)


@pytest.mark.parametrize("T", [2, 3, 1000])
@pytest.mark.parametrize("weighted", [False, True])
def test_threshold_limits_and_explicit_thresholds(T, weighted):
    y, p, w = _batch(100_003, T, torch.float32, torch.float32, weighted, seed=T)
    _check(_gpu_hist(confusion.ConfusionState(T), y, p, w), _ref_hist(y, p, w, T), weighted)
    thr = np.sort(np.random.default_rng(T).random(T).astype(np.float32))
    thr[: T // 3] = ref.edge_values(T)[: T // 3].clip(0, 1) if T > 3 else thr[: T // 3]
    thr = np.sort(thr)
    st = confusion.ConfusionState(T, thr.tolist())
    _check(_gpu_hist(st, y, p, w), _ref_hist(y, p, w, T, thr), weighted)


def test_samples_with_several_elements_share_their_weight():
    y, p, w = _batch(4096 * 3, 200, torch.float32, torch.float32, True, seed=5, per_sample=3)
    st = confusion.ConfusionState(200)
    _check(_gpu_hist(st, y.reshape(-1, 3), p.reshape(-1, 3), w), _ref_hist(y, p, w, 200), True)


def test_from_logits_matches_the_reference_sigmoid():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(200_000, generator=g) * 4
    y = (torch.rand(200_000, generator=g) < torch.sigmoid(x)).float()
    st = confusion.ConfusionState(200, from_logits=True)
    h = _gpu_hist(st, y, x)
    want = ref.histogram(y.numpy(), x.numpy(), None, 200, from_logits=True)
    # expf on the GPU and NumPy's float32 exp may differ in the last bit: an element on a bucket edge may move
    assert np.abs(h - want).sum() <= 4 and h.sum() == want.sum()


def test_one_state_accumulates_batches_of_different_grid_sizes():
    """Large- and small-grid launches share one scratch buffer: every batch must land in the histogram (the ticket
    counter that finds the last CTA sits at the same address whatever the grid)."""
    sizes = [300_000, 1_500, 300_000, 5_000, 1, 1_048_583, 700]
    st = confusion.ConfusionState(200)
    ys, ps, ws = [], [], []
    for i, n in enumerate(sizes):
        g = torch.Generator().manual_seed(500 + i)
        p = torch.rand(n, generator=g)
        y = torch.rand(n, generator=g)                               # soft labels: non-integer slab sums
        w = torch.rand(n, generator=g) * 3
        st.update(y.to(DEV), p.to(DEV), w.to(DEV))
        ys.append(y); ps.append(p); ws.append(w)
    torch.cuda.synchronize()
    want = ref.histogram(torch.cat(ys).numpy(), torch.cat(ps).numpy(), torch.cat(ws).numpy(), 200)
    _check(st.histogram().numpy(), want, True)
    # and the same sequence again gives the same bits
    again = confusion.ConfusionState(200)
    for y, p, w in zip(ys, ps, ws):
        again.update(y.to(DEV), p.to(DEV), w.to(DEV))
    torch.cuda.synchronize()
    assert again.histogram().numpy().tobytes() == st.histogram().numpy().tobytes()


def test_weighted_evaluate_with_a_partial_last_batch():
    torch.manual_seed(1)
    g = np.random.default_rng(1)
    n = 4096 * 3 + 1000                                              # full batches, then a smaller last one
    x = g.standard_normal((n, 8)).astype(np.float32)
    y = (x[:, 0] + 0.5 * g.standard_normal(n) > 0).astype(np.float32)
    w = g.random(n).astype(np.float32)
    model = keras.Sequential([keras.layers.Dense(16, activation="relu", input_shape=(8,)),
                              keras.layers.Dense(1, activation="sigmoid")])
    model.compile(keras.optimizers.SGD(0.0), "binary_crossentropy", weighted_metrics=["AUC"])
    res = model.evaluate(x, y, batch_size=4096, sample_weight=w, return_dict=True)
    p = model.predict(x, batch_size=4096).reshape(-1)
    assert res["auc"] == pytest.approx(ref.auc(y, p, w), rel=1e-9)


def test_two_runs_are_bit_identical():
    y, p, w = _batch((1 << 20) + 7, 200, torch.float32, torch.float32, True, seed=9)
    a = _gpu_hist(confusion.ConfusionState(200), y, p, w)
    b = _gpu_hist(confusion.ConfusionState(200), y, p, w)
    assert a.tobytes() == b.tobytes()


def test_graph_replay_equals_eager_and_accumulates_batch_by_batch():
    T, n = 200, 300_001
    batches = [_batch(n, T, torch.bfloat16, torch.float32, True, seed=100 + i) for i in range(4)]
    eager = confusion.ConfusionState(T)
    for y, p, w in batches:
        eager.update(y.to(DEV), p.to(DEV), w.to(DEV))
    torch.cuda.synchronize()
    sy, sp, sw = (t.to(DEV).clone() for t in batches[0])
    graphed = confusion.ConfusionState(T)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graphed.update(sy, sp, sw)                    # allocates the state; then undone
        graphed.reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.update(sy, sp, sw)
    torch.cuda.synchronize()
    graphed.reset()
    for y, p, w in batches:
        sy.copy_(y.to(DEV)); sp.copy_(p.to(DEV)); sw.copy_(w.to(DEV))
        g.replay()
    torch.cuda.synchronize()
    assert graphed.histogram().numpy().tobytes() == eager.histogram().numpy().tobytes()
    one = confusion.ConfusionState(T)
    y, p, w = batches[0]
    a = _gpu_hist(one, y, p, w)
    graphed.reset()
    sy.copy_(y.to(DEV)); sp.copy_(p.to(DEV)); sw.copy_(w.to(DEV))
    g.replay()
    torch.cuda.synchronize()
    assert graphed.histogram().numpy().tobytes() == a.tobytes()


@pytest.mark.parametrize("y,p,what", [([0.0, 1.0], [0.5, 1.5], "predictions"),
                                       ([0.0, 1.0], [-0.25, 0.5], "predictions"),
                                       ([0.0, 1.0], [0.5, float("nan")], "predictions"),
                                       ([0.0, 2.0], [0.5, 0.5], "labels"),
                                       ([0.0, float("nan")], [0.5, 0.5], "labels")])
def test_invalid_input_sets_its_flag_and_result_raises(y, p, what):
    m = keras.metrics.AUC()
    m.update_state(torch.tensor(y, device=DEV), torch.tensor(p, device=DEV))
    torch.cuda.synchronize()
    bit = confusion.BAD_PREDICTION if what == "predictions" else confusion.BAD_LABEL
    assert int(m._state.flags.item()) == bit
    with pytest.raises(ValueError, match=what):
        m.result()
    m.reset_state()
    m.update_state(torch.tensor([0.0, 1.0], device=DEV), torch.tensor([0.2, 0.7], device=DEV))
    assert m.result() == 1.0


def test_int64_labels_outside_zero_one_are_flagged():
    m = keras.metrics.Precision()
    m.update_state(torch.tensor([0, 3], device=DEV), torch.tensor([0.2, 0.7], device=DEV))
    with pytest.raises(ValueError, match="labels"):
        m.result()


def test_fit_auc_on_the_graph_engine_equals_evaluate_and_skips_warmup_steps():
    torch.manual_seed(0)
    n, bs = 1024, 128
    g = np.random.default_rng(0)
    x = g.standard_normal((n, 16)).astype(np.float32)
    model = keras.Sequential([keras.layers.Dense(32, activation="relu", input_shape=(16,)),
                              keras.layers.Dense(1, activation="sigmoid")])
    model.compile(keras.optimizers.SGD(0.0), "binary_crossentropy", metrics=["AUC"])
    p0 = model.predict(x, batch_size=bs).reshape(-1)
    med = np.median(p0)
    y = (p0 > med).astype(np.float32)
    y[:bs] = 1.0 - y[:bs]                      # the first batch (the warm-up batch) ranks backwards
    hist = model.fit(x, y, batch_size=bs, epochs=2, shuffle=False, verbose=0)
    assert isinstance(model._engine, GraphTrainEngine)
    res = model.evaluate(x, y, batch_size=bs, return_dict=True)
    p = model.predict(x, batch_size=bs).reshape(-1)
    want = ref.auc(y, p)
    warm = ref.auc(np.concatenate([y[:bs]] * 3 + [y]), np.concatenate([p[:bs]] * 3 + [p]))
    assert abs(want - warm) > 0.05
    assert res["auc"] == pytest.approx(want, abs=1e-12)
    for v in hist.history["auc"]:
        assert v == pytest.approx(res["auc"], abs=1e-3)


def test_gpu_placed_canned_estimator_matches_the_reference(tmp_path):
    from test_keras_confusion_metrics import _check_binary_eval, _est_data
    x, y = _est_data(seed=4)
    e = est.LinearClassifier([fc.numeric_column("x", shape=(5,))], model_dir=str(tmp_path), n_classes=2,
                             optimizer=lambda: keras.optimizers.Adam(0.05),
                             config=est.RunConfig(save_checkpoints_steps=20, log_step_count_steps=None))
    e.train(lambda: data.Dataset.from_tensor_slices(({"x": x}, y)).batch(32).repeat(), max_steps=20)
    res = _check_binary_eval(e, x, y)
    assert e._device.type == "cuda" and res["auc"] > 0.5
