"""The fast path's training step (keras/fastpath.py: FastSequentialEngine._forward_backward), launch for launch, on the
CPU.

The native library is replaced by a recorder and the engine's device state by CPU tensors, so the step runs here
end to end, its cuDNN / cuBLAS fallbacks included (they compute on the CPU).  Each step is recorded as the kernel
launches it makes, in order, with their integer and float arguments and, for each pointer, the tensor it points
into: a named parameter or gradient, the batch (x, y, sw), an engine buffer, or a temporary.  Two pointers of one
launch into the same temporary are marked equal (``temp#0`` twice: an in-place output, a ReLU gate that is the
input).  Raw addresses depend on allocation order and are never recorded.  The size queries the step makes
(scratch sizes, split-K slabs, the dropout keep scale...) are answered by the recorder and not recorded.

The fixture tests/golden/fastpath_step_trace.json holds the trace of every case; ``python
tests/test_fastpath_step_trace.py`` writes it again.
"""
import ctypes
import json
import logging
import os
import sys
import types
from contextlib import ExitStack
from unittest import mock

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tf_yarn_b200 import keras  # noqa: E402
from tf_yarn_b200.keras import fastpath  # noqa: E402
from tf_yarn_b200.keras import layers as L  # noqa: E402
from tf_yarn_b200.keras.engine import GraphTrainEngine  # noqa: E402
from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn  # noqa: E402
from tf_yarn_b200.ops import native  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fastpath_step_trace.json")
SWITCHES = ("TFY_NO_TC_CONV", "TFY_NO_UNPOOL_FUSION", "TFY_NO_TC_DENSE_BWD", "TFY_NO_FUSED_HEAD", "TFY_SPLITK_FUSE",
            "TFY_SPLITK_TILES", "TFY_OVERLAP", "TFY_OVERLAP_GROUPS")
LOGITS = keras.losses.SparseCategoricalCrossentropy(from_logits=True)
N_PART = 5                # what the recorder writes through an int out-pointer (the deferred wgrad's partial count)


def _keep_scale(rate: float) -> float:
    """The recorder's tfy_conv3x3_c32_keep_scale: any value other than 1 / (1 - rate), so the trace shows which of
    the two scales reaches which kernel."""
    return float(np.float32(1.25 + rate))


def _reply_keep_scale(rate, out):
    out._obj.value = _keep_scale(rate)
    return 0


REPLIES = {
    "tfy_conv3x3_c32_keep_scale": _reply_keep_scale,
    "tfy_conv3x3_c32_wgrad_scratch_elems": lambda: 4096,
    "tfy_dense_head_scratch_elems": lambda K, C, B: 1024,
    "tfy_gemm_bf16_splitk_slabs": lambda K, split: split,
    "tfy_nn_max_partial_blocks": lambda: fastpath.PARTIAL_BLOCKS,
    "tfy_conv3x3_c32_wgrad_spare_ctas": lambda B, H, W: 4,
}


# ------------------------------------------------------------------------------------------------ harness
class _Recorder:
    """Stands in for the kernel library: answers the size queries, records every launch."""

    def __init__(self):
        self.calls = []
        self.roles = None          # pointer -> role

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        if name in REPLIES:
            return REPLIES[name]
        argtypes = native._EXTRA_DECLS[name][0]

        def launch(*args):
            assert len(args) == len(argtypes), (name, len(args), len(argtypes))
            self.calls.append([name] + self._args(argtypes, args))
            return 0
        return launch

    def _args(self, argtypes, args):
        out, temps = [], {}
        for t, a in zip(argtypes, args):
            if a is None:
                out.append(None)
            elif type(a).__name__ == "CArgObject":          # ctypes.byref(...)
                obj = a._obj
                if isinstance(obj, ctypes.c_int):
                    obj.value = N_PART
                    out.append("&int")
                else:
                    assert isinstance(obj, native.OverlapStep), type(obj)
                    out.append(f"&overlap(g0={obj.g0}, g1={obj.g1}, n_cta={obj.n_cta})")
            elif t is ctypes.c_void_p and int(a) == 0:   # the stream (the step runs on stream 0 here)
                out.append(0)
            elif t is ctypes.c_void_p:
                role = self.roles(int(a))
                if role == "temp":
                    role = f"temp#{temps.setdefault(int(a), len(temps))}"
                out.append(role)
            elif t is ctypes.c_float:
                out.append(float(a))
            else:
                assert isinstance(a, int), (t, a)
                out.append(int(a))
        return out


class _Fused:
    """The fused optimizer step as the fast path sees it: flat-buffer offsets, the hyper-parameter block, step()."""

    def __init__(self, params, kind):
        self.spec = types.SimpleNamespace(kind=kind)
        self.zero_grads = True
        self.param_dtype = self.grad_dtype = torch.bfloat16
        self.hyper = torch.zeros(ctypes.sizeof(native.HyperBlock), dtype=torch.uint8)
        self.offsets, o = [], 0
        for p in params:
            self.offsets.append(o)
            o += (p.numel() + 7) // 8 * 8
        self.shard_n = o
        self.steps = []

    def overlap_step(self, g0, g1, n_cta):
        ov = native.OverlapStep()
        ov.g0, ov.g1, ov.n_cta = g0, g1, n_cta
        return ov

    def step(self, **kw):
        self.steps.append({k: list(v) if isinstance(v, tuple) else v for k, v in kw.items()})


def _stub_engine_init(self, net, opt_kind):
    """GraphTrainEngine.__init__ on the CPU: bf16 parameters with gradients, conv kernels stored (O, kh, kw, I) as the
    engine's flat buffer stores them."""
    self.device = torch.device("cpu")
    net.to(torch.bfloat16)
    self.params = [p for p in net.parameters() if p.requires_grad]
    for p in self.params:
        if p.dim() == 4:
            p.data = p.data.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        p.grad = torch.zeros_like(p.data)
    self.fused = _Fused(self.params, opt_kind)
    self.metric_fns, self.weighted_metric_fns = [("accuracy", None)], []
    self._loss = torch.zeros((), dtype=torch.float32)
    self._cw, self._wmode = None, (False, False)


def _roles(eng, x, y, sw):
    named = [("x", x), ("y", y), ("sw", sw), ("fused.hyper", eng.fused.hyper)]
    for li, st in enumerate(eng.plan):
        if getattr(st, "layer", None) is not None:
            mod = st.layer.module
            for pn, p in (("w", mod.weight), ("b", mod.bias)):
                named += [(f"{st.kind}{li}.{pn}", p), (f"{st.kind}{li}.{pn}.grad", p.grad)]
    for k, v in vars(eng).items():
        if torch.is_tensor(v):
            named.append((f"eng.{k}", v))
        elif isinstance(v, dict):
            named += [(f"eng.{k}[{kk!r}]", vv) for kk, vv in v.items() if torch.is_tensor(vv)]
    spans = [(t.data_ptr(), t.untyped_storage().nbytes(), n) for n, t in named if t is not None]

    def role(ptr):
        for start, nbytes, n in spans:
            if ptr == start:
                return n
        for start, nbytes, n in spans:
            if start < ptr < start + nbytes:
                return f"{n}+{ptr - start}"
        return "temp"
    return role


class _Warnings(logging.Handler):
    def __init__(self):
        super().__init__()
        self.msgs = []

    def emit(self, record):
        self.msgs.append(record.getMessage())


# ------------------------------------------------------------------------------------------------ cases
def _generic():
    m = keras.Sequential(name="generic_kernels")           # the model of test_gpu_nn_kernels.py
    m.add(L.Conv2D(16, (3, 3), activation="relu", input_shape=(30, 30, 1)))
    m.add(L.MaxPooling2D(pool_size=(2, 2)))
    m.add(L.Dropout(0.25))
    m.add(L.Flatten())
    m.add(L.Dense(96, activation="relu"))
    m.add(L.Dropout(0.5))
    m.add(L.Dense(40))
    return m


def _seq(*layers):
    return lambda: keras.Sequential(list(layers))


def _mlp():                    # Dense-only: split-K Dense, fused head
    return keras.Sequential([L.Dense(128, activation="relu", input_shape=(4096,)), L.Dropout(0.2), L.Dense(10)])


def _narrow_head():            # head K = 64: outside the fused head's envelope
    return keras.Sequential([L.Dense(64, activation="relu", input_shape=(2048,)), L.Dense(10)])


def _softmax_mlp():
    return keras.Sequential([L.Dense(128, activation="relu", input_shape=(4096,)), L.Dense(10, activation="softmax")])


def _conv_dropout():           # C_in = 1 direct kernel, no pool, dropout mask; head after Flatten
    return keras.Sequential([L.Conv2D(8, 3, activation="relu", input_shape=(8, 8, 1)), L.Dropout(0.2), L.Flatten(),
                             L.Dense(3)])


def _head_only():
    return keras.Sequential([L.Dense(8, input_shape=(16,))])


def _case(build, batches=(128, 128), loss=LOGITS, weights=None, env=None, opt="adadelta"):
    return dict(build=build, batches=batches, loss=loss, weights=weights, env=env or {}, opt=opt)


CASES = {
    "mnist_b128": _case(keras_mnist_cnn),
    "mnist_b2": _case(keras_mnist_cnn, (2, 2)),
    "mnist_b3": _case(keras_mnist_cnn, (3, 3)),
    "mnist_b128_b3_b128": _case(keras_mnist_cnn, (128, 3, 128)),
    "mnist_b128_sample_weight": _case(keras_mnist_cnn, weights="sample"),
    "mnist_b128_class_weight": _case(keras_mnist_cnn, weights="class"),
    "generic_b64": _case(_generic, (64, 64)),
    "generic_b64_sample_weight": _case(_generic, (64, 64), weights="sample"),
    "mlp_b128": _case(_mlp),
    "narrow_head_b128": _case(_narrow_head),
    "softmax_string_loss_b128": _case(_softmax_mlp, loss="sparse_categorical_crossentropy"),
    "conv_dropout_b16": _case(_conv_dropout, (16, 16)),
    "head_only_b32": _case(_head_only, (32, 32)),
    "mnist_b128_rmsprop_overlap": _case(keras_mnist_cnn, env={"TFY_OVERLAP": "1"}, opt="rmsprop"),
    "mnist_b128_overlap_groups_100": _case(keras_mnist_cnn, env={"TFY_OVERLAP": "1", "TFY_OVERLAP_GROUPS": "100"}),
}
for _k, _v in {"TFY_NO_TC_CONV": "1", "TFY_NO_UNPOOL_FUSION": "1", "TFY_NO_TC_DENSE_BWD": "1", "TFY_NO_FUSED_HEAD": "1",
               "TFY_SPLITK_FUSE": "1", "TFY_SPLITK_TILES": "4", "TFY_OVERLAP": "1", "TFY_OVERLAP_GROUPS": "100"}.items():
    CASES[f"mnist_b128_{_k}={_v}"] = _case(keras_mnist_cnn, env={_k: _v})


def run_case(name):
    """[{calls, fused_step, launches, warnings} for each step of the case]."""
    case = CASES[name]
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(case["env"])
    rec = _Recorder()
    warn = _Warnings()
    logger = logging.getLogger(fastpath.__name__)
    with ExitStack() as stack:
        stack.enter_context(mock.patch.dict(os.environ, env, clear=True))
        stack.enter_context(mock.patch.object(native, "load", lambda: rec))
        stack.enter_context(mock.patch.object(GraphTrainEngine, "__init__", _stub_engine_init))
        stack.enter_context(mock.patch.object(torch.cuda, "get_device_properties",
                                              lambda dev=None: types.SimpleNamespace(multi_processor_count=132)))
        stack.enter_context(mock.patch.object(fastpath.FastSequentialEngine, "_s", lambda self: 0))
        logger.addHandler(warn)
        stack.callback(logger.removeHandler, warn)
        torch.manual_seed(0)
        m = case["build"]()
        m.compile(loss=case["loss"], optimizer="sgd", metrics=["accuracy"])
        m._device = torch.device("cpu")
        m.build()
        plan = fastpath.build_plan(m)
        assert plan is not None, name
        eng = fastpath.FastSequentialEngine(m, plan, m.net, case["opt"])
        in_shape = tuple(m.layers[0].input_shape_)
        C = plan[-1].layer.units
        if case["weights"] == "class":
            eng._cw, eng._wmode = torch.linspace(0.5, 2.0, C), (True, False)
        elif case["weights"] == "sample":
            eng._wmode = (False, True)
        steps = []
        for B in case["batches"]:
            g = torch.Generator().manual_seed(B)
            x = torch.rand((B,) + in_shape, generator=g)
            y = torch.randint(0, C, (B,), generator=g)
            sw = torch.rand(B, generator=g) if case["weights"] == "sample" else None
            rec.calls, rec.roles = [], lambda ptr: _roles(eng, x, y, sw)(ptr)
            del warn.msgs[:], eng.fused.steps[:]
            eng._forward_backward(x, y, sw)
            steps.append({"calls": rec.calls, "fused_step": list(eng.fused.steps), "launches": eng._launches_per_step,
                          "warnings": sorted(warn.msgs)})
        return steps


def _fmt_call(call):
    return f"{call[0]}({', '.join(json.dumps(a) if a is None or not isinstance(a, str) else a for a in call[1:])})"


def fixture_of(steps):
    return [dict(s, calls=[_fmt_call(c) for c in s["calls"]]) for s in steps]


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


def test_the_mnist_step_is_ten_launches_of_our_kernels(traces):
    for step in _trace(traces, "mnist_b128"):
        assert step["launches"] == 10 and len(step["calls"]) == 9 and step["warnings"] == []
        assert step["fused_step"] == [{}]


def test_no_tc_conv_switch_turns_every_tensor_core_convolution_kernel_off(traces):
    for step in _trace(traces, "mnist_b128_TFY_NO_TC_CONV=1"):
        names = [c[0] for c in step["calls"]]
        assert not [n for n in names if "conv3x3_c32" in n or n.endswith("_tc")], names
        assert {"tfy_conv3x3_c1_fwd", "tfy_bias_relu_pool_drop_fwd", "tfy_conv3x3_c1_wgrad"} <= set(names)


# the kernels that take the dropout scale of a pooled conv stage's backward, and the Dense mask kernels
POOL_BWD = {"tfy_conv3x3_c32_wgrad_unpool_ov", "tfy_conv3x3_c32_wgrad_unpool_deferred", "tfy_conv3x3_c32_wgrad_unpool",
            "tfy_conv3x3_c32_dgrad_unpool_reduce", "tfy_conv3x3_c32_dgrad_unpool", "tfy_pool_drop_relu_bwd"}
DENSE_MASK = {"tfy_act_drop_bwd_bias", "tfy_dense_head_fused", "tfy_dense_head_fused_weighted"}


@pytest.mark.parametrize("name", sorted(n for n in CASES if n.startswith(("mnist", "generic"))))
def test_pooled_conv_backward_scale_is_the_one_its_forward_applied(traces, name):
    """A tensor-core conv stage's backward kernels receive tfy_conv3x3_c32_keep_scale's value; after the general pool
    kernel, the backward pool kernel receives 1 / (1 - rate); 1 / (1 - rate) reaches no other kernel than those and
    the Dense mask kernels (the MNIST / generic models have one pooled conv stage, rate 0.25, Dense rate 0.5)."""
    rate = 0.25
    general = 1.0 / (1.0 - rate)
    for step in _trace(traces, name):
        names = [c[0] for c in step["calls"]]
        tc = "tfy_conv3x3_c32_pool_fwd" in names
        assert tc != ("tfy_bias_relu_pool_drop_fwd" in names)
        want = _keep_scale(rate) if tc else general
        seen = 0
        for call in step["calls"]:
            floats = [a for a in call[1:] if isinstance(a, float)]
            if call[0] in POOL_BWD:
                assert floats == [want], (call, want)
                seen += 1
            elif call[0] not in DENSE_MASK or "conv" in " ".join(a for a in call[1:] if isinstance(a, str)):
                assert general not in floats, call
        assert seen or not tc, names


if __name__ == "__main__":
    out = {name: fixture_of(run_case(name)) for name in sorted(CASES)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {GOLDEN}: {len(out)} cases")
