"""The fast path's binary cross-entropy head on the CPU: the grammar build_plan accepts and refuses, the target shapes
the engine accepts, the labels fit leaves uncast, and the training step launch for launch.

The step traces use the recorder of tests/test_fastpath_step_trace.py; the fixture
tests/golden/fastpath_binary_step_trace.json holds them, and ``python tests/test_fastpath_binary_plan.py`` writes it
again.
"""
import json
import logging
import os
import sys
import types
from contextlib import ExitStack
from unittest import mock

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import test_fastpath_step_trace as trace  # noqa: E402
from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.keras import fastpath  # noqa: E402
from tf_yarn_b200.keras import layers as L  # noqa: E402
from tf_yarn_b200.keras.engine import GraphTrainEngine  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fastpath_binary_step_trace.json")
BCE = keras.losses.BinaryCrossentropy
SUBSTITUTE = {"tfy_dense_head_fused": "tfy_dense_head_fused_binary"}


def _mnist(units=1, activation="sigmoid"):
    """The headline MNIST CNN with a Dense(units, activation) head."""
    m = keras.Sequential(name="mnist_cnn")
    m.add(L.Conv2D(32, (3, 3), activation="relu", input_shape=(28, 28, 1)))
    m.add(L.Conv2D(64, (3, 3), activation="relu"))
    m.add(L.MaxPooling2D(pool_size=(2, 2)))
    m.add(L.Dropout(0.25))
    m.add(L.Flatten())
    m.add(L.Dense(128, activation="relu"))
    m.add(L.Dropout(0.5))
    m.add(L.Dense(units, activation=activation))
    return m


def _mlp(units=1, activation="sigmoid", hidden=128):
    return keras.Sequential([L.Dense(hidden, activation="relu", input_shape=(4096,)), L.Dropout(0.2),
                             L.Dense(units, activation=activation)])


def _compiled(model, loss, metrics=("accuracy",), weighted=None):
    model.compile(loss=loss, optimizer="sgd", metrics=list(metrics), weighted_metrics=weighted)
    model.build()
    return model


# ------------------------------------------------------------------------------------------------ grammar
@pytest.mark.parametrize("build,loss,metrics,weighted", [
    (lambda: _mnist(), BCE(), ["accuracy"], None),
    (lambda: _mnist(), "binary_crossentropy", ["acc"], None),
    (lambda: _mnist(), BCE(label_smoothing=0.1), ["binary_accuracy"], ["accuracy"]),
    (lambda: _mnist(1, None), BCE(from_logits=True), [], None),
    (lambda: _mlp(10), BCE(label_smoothing=0.2), ["accuracy"], ["binary_accuracy"]),
    (lambda: _mlp(10, None), BCE(from_logits=True, label_smoothing=0.05), ["accuracy"], None),
    (lambda: _mlp(40), "binary_crossentropy", ["accuracy"], None),
], ids=["c1_object", "c1_string", "c1_smoothing_weighted", "c1_logits", "c10_weighted", "c10_logits", "c40_string"])
def test_binary_heads_inside_the_grammar_get_a_plan(build, loss, metrics, weighted):
    m = _compiled(build(), loss, metrics, weighted)
    plan = fastpath.build_plan(m)
    assert plan is not None and plan[-1].kind == "head"


@pytest.mark.parametrize("build", [
    lambda: _compiled(_mnist(), BCE(), ["AUC"]),
    lambda: _compiled(_mnist(), BCE(), ["Precision"]),
    lambda: _compiled(_mnist(), BCE(), ["Recall"]),
    lambda: _compiled(_mnist(), BCE(), ["mae"]),
    lambda: _compiled(_mnist(), BCE(), [lambda y, p: (p - y).abs().mean()]),
    lambda: _compiled(_mnist(), BCE(), ["accuracy"], ["accuracy", "binary_accuracy"]),
    lambda: _compiled(_mnist(), BCE(), ["categorical_accuracy"]),
    lambda: _compiled(_mnist(1, "sigmoid"), BCE(from_logits=True)),
    lambda: _compiled(_mnist(1, None), BCE()),
    lambda: _compiled(_mnist(1, None), "binary_crossentropy"),
    lambda: _compiled(keras.Sequential([L.Dense(64, activation="sigmoid", input_shape=(32,)),
                                        L.Dense(1, activation="sigmoid")]), BCE()),
    lambda: _compiled(_mnist(10, "softmax"), BCE()),
], ids=["auc", "precision", "recall", "mae", "callable", "two_weighted", "categorical_accuracy", "sigmoid_with_logits",
        "linear_with_probabilities", "linear_with_string", "hidden_sigmoid", "softmax_layer"])
def test_binary_heads_outside_the_grammar_get_none(build):
    assert fastpath.build_plan(build()) is None


def test_label_dtype_is_unchanged():
    assert fastpath.label_dtype(BCE()) is None
    assert fastpath.label_dtype("binary_crossentropy") is None
    assert fastpath.head_loss(BCE(from_logits=True)) is None
    assert fastpath.label_dtype(keras.losses.SparseCategoricalCrossentropy()) == torch.int64
    assert fastpath.label_dtype(keras.losses.CategoricalCrossentropy()) == torch.float32
    assert fastpath.binary_head_loss(BCE(label_smoothing=0.3)) == (0.3, "sigmoid")
    assert fastpath.binary_head_loss(BCE(from_logits=True)) == (0.0, "linear")
    assert fastpath.binary_head_loss("binary_crossentropy") == (0.0, "sigmoid")
    assert fastpath.binary_head_loss(keras.losses.CategoricalCrossentropy()) is None


# ------------------------------------------------------------------------------------------------ the engine
def _engine(build, loss):
    """A FastSequentialEngine on the CPU, its library a recorder (tests/test_fastpath_step_trace.py)."""
    rec = trace._Recorder()
    with ExitStack() as stack:
        stack.enter_context(mock.patch.object(native, "load", lambda: rec))
        stack.enter_context(mock.patch.object(GraphTrainEngine, "__init__", trace._stub_engine_init))
        torch.manual_seed(0)
        m = _compiled(build(), loss)
        m._device = torch.device("cpu")
        eng = fastpath.FastSequentialEngine(m, fastpath.build_plan(m), m.net, "sgd")
    return eng, rec


@pytest.mark.parametrize("shape", [(8,), (8, 1)])
def test_single_output_targets_may_be_flat_or_a_column(shape):
    eng, _ = _engine(_mnist, BCE())
    for dtype in (torch.int64, torch.uint8, torch.bool, torch.float64, torch.float32):
        y = torch.zeros(shape, dtype=dtype)
        got = eng._head_targets(y)
        assert got.dtype == torch.float32 and got.shape == shape


@pytest.mark.parametrize("build,shape,want", [
    (_mnist, (8, 3), r"\(8, 3\).*\(batch, 1\).*\(batch,\) or \(batch, 1\)"),
    (_mnist, (8, 1, 1), r"\(8, 1, 1\)"),
    (lambda: _mlp(10), (8,), r"\(8,\).*\(batch, 10\)"),
    (lambda: _mlp(10), (8, 9), r"\(8, 9\).*\(batch, 10\)"),
])
def test_targets_of_the_wrong_shape_raise(build, shape, want):
    eng, _ = _engine(build, BCE())
    with pytest.raises(ValueError, match=want):
        eng._head_targets(torch.zeros(shape))


# ------------------------------------------------------------------------------------------------ step traces
def _case(build, loss=BCE(label_smoothing=0.05), weights=None, env=None, batches=(128, 128)):
    return dict(build=build, loss=loss, weights=weights, env=env or {}, batches=batches)


CASES = {
    "mnist_binary_b128": _case(_mnist),
    "mnist_binary_b128_sample_weight": _case(_mnist, weights="sample"),
    "mnist_binary_b128_class_weight": _case(_mnist, weights="class"),
    "mnist_binary_logits_b128": _case(lambda: _mnist(1, None), loss=BCE(from_logits=True)),
    "mnist_binary_b128_TFY_NO_FUSED_HEAD=1": _case(_mnist, env={"TFY_NO_FUSED_HEAD": "1"}),
    "mnist_binary_b3": _case(_mnist, batches=(3, 3)),
    "mlp_binary_b128": _case(_mlp, loss="binary_crossentropy"),
    "mlp_multilabel_b128": _case(lambda: _mlp(10)),
    "mlp_multilabel_c40_b64": _case(lambda: _mlp(40), batches=(64, 64)),
    "mlp_multilabel_narrow_head_b128": _case(lambda: _mlp(10, hidden=64)),
}


def run_case(name):
    """[{calls, fused_step, launches, warnings} for each step of the case]."""
    case = CASES[name]
    env = {k: v for k, v in os.environ.items() if k not in trace.SWITCHES}
    env.update(case["env"])
    rec = trace._Recorder()
    warn = trace._Warnings()
    logger = logging.getLogger(fastpath.__name__)
    with ExitStack() as stack:
        stack.enter_context(mock.patch.dict(os.environ, env, clear=True))
        stack.enter_context(mock.patch.object(native, "load", lambda: rec))
        stack.enter_context(mock.patch.object(GraphTrainEngine, "__init__", trace._stub_engine_init))
        stack.enter_context(mock.patch.object(torch.cuda, "get_device_properties",
                                              lambda dev=None: types.SimpleNamespace(multi_processor_count=132)))
        stack.enter_context(mock.patch.object(fastpath.FastSequentialEngine, "_s", lambda self: 0))
        logger.addHandler(warn)
        stack.callback(logger.removeHandler, warn)
        torch.manual_seed(0)
        m = _compiled(case["build"](), case["loss"])
        m._device = torch.device("cpu")
        plan = fastpath.build_plan(m)
        assert plan is not None, name
        eng = fastpath.FastSequentialEngine(m, plan, m.net, "adadelta")
        in_shape = tuple(m.layers[0].input_shape_)
        C = plan[-1].layer.units
        if case["weights"] == "class":
            eng._cw, eng._wmode = torch.tensor([0.5, 2.0] + [1.0] * max(C - 2, 0)), (True, False)
        elif case["weights"] == "sample":
            eng._wmode = (False, True)
        steps = []
        for B in case["batches"]:
            g = torch.Generator().manual_seed(B)
            x = torch.rand((B,) + in_shape, generator=g)
            y = torch.randint(0, 2, (B, C), generator=g).float()
            sw = torch.rand(B, generator=g) if case["weights"] == "sample" else None
            rec.calls, rec.roles = [], lambda ptr: trace._roles(eng, x, y, sw)(ptr)
            del warn.msgs[:], eng.fused.steps[:]
            eng._forward_backward(x, y, sw)
            steps.append({"calls": rec.calls, "fused_step": list(eng.fused.steps), "launches": eng._launches_per_step,
                          "warnings": sorted(warn.msgs)})
        return steps


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
    assert trace.fixture_of(_trace(traces, name)) == golden[name]


def test_the_binary_mnist_step_is_the_headline_step_with_its_head_kernel_swapped(traces):
    headline = trace.run_case("mnist_b128")
    for step, ref in zip(_trace(traces, "mnist_binary_b128"), headline):
        assert step["launches"] == 10 and step["warnings"] == [] and step["fused_step"] == [{}]
        assert [c[0] for c in step["calls"]] == [SUBSTITUTE.get(c[0], c[0]) for c in ref["calls"]]
        head = [c for c in step["calls"] if c[0] == "tfy_dense_head_fused_binary"]
        assert len(head) == 1 and head[0][4] == "y" and head[0][5] == pytest.approx(0.05) and head[0][6] == 1


def test_a_logits_head_tells_the_kernel_its_output_is_the_logit(traces):
    for step in _trace(traces, "mnist_binary_logits_b128"):
        head = [c for c in step["calls"] if c[0] == "tfy_dense_head_fused_binary"]
        assert len(head) == 1 and head[0][5] == 0.0 and head[0][6] == 0


@pytest.mark.parametrize("name", ["mnist_binary_b128_TFY_NO_FUSED_HEAD=1", "mlp_multilabel_c40_b64",
                                  "mlp_multilabel_narrow_head_b128"])
def test_heads_outside_the_fused_envelope_use_the_sigmoid_fallback_and_warn_once(traces, name):
    steps = _trace(traces, name)
    for i, step in enumerate(steps):
        names = [c[0] for c in step["calls"]]
        assert "tfy_sigmoid_xent" in names and "tfy_dense_head_fused_binary" not in names
        assert not [n for n in names if "softmax" in n]
        assert bool(step["warnings"]) == (i == 0), step["warnings"]


@pytest.mark.parametrize("name", ["mnist_binary_b128_sample_weight", "mnist_binary_b128_class_weight"])
def test_weighted_binary_steps_keep_ten_launches(traces, name):
    for step in _trace(traces, name):
        assert step["launches"] == 10
        head = [c for c in step["calls"] if c[0] == "tfy_dense_head_fused_binary"]
        want = ("sw", None) if name.endswith("sample_weight") else (None, "eng._cw")
        assert len(head) == 1 and tuple(head[0][-3:-1]) == want


if __name__ == "__main__":
    out = {name: trace.fixture_of(run_case(name)) for name in sorted(CASES)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {GOLDEN}: {len(out)} cases")
