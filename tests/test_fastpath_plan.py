"""The fast path's layer-pattern grammar (keras/fastpath.py: build_plan), checkable without a GPU: which Sequential
models are served by the fused wgmma kernels, which stages they become, and that anything outside the grammar falls
back to the autograd engine (None) instead of being mis-compiled."""
import pytest
import torch

from tf_yarn_b200 import keras
from tf_yarn_b200.keras import fastpath
from tf_yarn_b200.keras import layers as L
from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn

LOGITS = keras.losses.SparseCategoricalCrossentropy(from_logits=True)


def _plan(layers, loss=LOGITS, metrics=("accuracy",), shape=None):
    m = keras.Sequential(list(layers))
    m.compile(loss=loss, optimizer="sgd", metrics=list(metrics))
    m._device = torch.device("cpu")
    m.build(shape)
    plan = fastpath.build_plan(m)
    return None if plan is None else [(s.kind, getattr(s, "relu", None), getattr(s, "pool", None), getattr(s, "drop", None))
                                      for s in plan]


def test_the_headline_model_maps_onto_five_fused_stages():
    m = keras_mnist_cnn()
    m.compile(loss=LOGITS, optimizer=keras.optimizers.Adadelta(1.0), metrics=["accuracy"])
    m.build()
    plan = fastpath.build_plan(m)
    assert [s.kind for s in plan] == ["conv", "conv", "flatten", "dense", "head"]
    c1, c2, _, d1, head = plan
    assert (c1.relu, c1.pool, c1.drop) == (True, False, 0.0) and c1.layer.filters == 32
    assert (c2.relu, c2.pool, c2.drop) == (True, True, 0.25) and c2.layer.filters == 64     # pool + dropout folded in
    assert (d1.relu, d1.drop) == (True, 0.5) and d1.layer.units == 128 and head.layer.units == 10


def test_softmax_head_with_the_string_loss_and_plain_mlps():
    mlp = [L.Dense(64, activation="relu", input_shape=(32,)), L.Dropout(0.1), L.Dense(16), L.Dense(4, activation="softmax")]
    assert _plan(mlp, loss="sparse_categorical_crossentropy") == [
        ("dense", True, None, 0.1), ("dense", False, None, 0.0), ("head", None, None, None)]
    assert _plan([L.Dense(8, input_shape=(16,))]) == [("head", None, None, None)]
    conv_only_drop = [L.Conv2D(8, 3, activation="relu", input_shape=(8, 8, 1)), L.Dropout(0.2), L.Flatten(), L.Dense(3)]
    assert _plan(conv_only_drop) == [("conv", True, False, 0.2), ("flatten", None, None, None), ("head", None, None, None)]


@pytest.mark.parametrize("layers,loss,metrics", [
    ([L.Dense(8, input_shape=(16,)), L.Dense(4, activation="softmax")], LOGITS, ("accuracy",)),      # softmax + logits loss
    ([L.Dense(8, input_shape=(16,)), L.Dense(4)], "sparse_categorical_crossentropy", ("accuracy",)),  # logits + prob loss
    ([L.Dense(8, input_shape=(16,)), L.Dense(4)], "mse", ()),                                          # other losses
    ([L.Dense(8, input_shape=(16,)), L.Dense(4)], LOGITS, ("mae",)),                                   # other metrics
    ([L.Dense(8, activation="tanh", input_shape=(16,)), L.Dense(4)], LOGITS, ()),                     # other activation
    ([L.Dense(8, use_bias=False, input_shape=(16,)), L.Dense(4)], LOGITS, ()),
    ([L.Dense(12, input_shape=(16,)), L.Dense(4)], LOGITS, ()),                                        # width not % 8
    ([L.Dense(8, input_shape=(16,)), L.BatchNormalization(), L.Dense(4)], LOGITS, ()),                 # unknown layer
    ([L.Dense(8, input_shape=(16,)), L.Dense(2048)], LOGITS, ()),                                      # head too wide
    ([L.Dense(8, activation="relu", input_shape=(16,))], LOGITS, ()),                                  # no linear head
    ([L.Conv2D(8, 5, activation="relu", input_shape=(12, 12, 1)), L.Flatten(), L.Dense(4)], LOGITS, ()),   # 5x5
    ([L.Conv2D(8, 3, strides=2, activation="relu", input_shape=(12, 12, 1)), L.Flatten(), L.Dense(4)], LOGITS, ()),
    ([L.Conv2D(8, 3, padding="same", activation="relu", input_shape=(12, 12, 1)), L.Flatten(), L.Dense(4)], LOGITS, ()),
    ([L.Conv2D(6, 3, activation="relu", input_shape=(12, 12, 1)), L.Flatten(), L.Dense(4)], LOGITS, ()),   # filters % 8
    ([L.Conv2D(8, 3, input_shape=(12, 12, 1)), L.MaxPooling2D(2), L.Flatten(), L.Dense(4)], LOGITS, ()),   # pool w/o relu
    ([L.Conv2D(8, 3, activation="relu", input_shape=(13, 13, 1)), L.MaxPooling2D(2), L.Flatten(), L.Dense(4)], LOGITS, ()),
    ([L.Conv2D(8, 3, activation="relu", input_shape=(12, 12, 1)), L.MaxPooling2D(3), L.Flatten(), L.Dense(4)], LOGITS, ()),
    ([L.Conv2D(8, 3, activation="relu", input_shape=(12, 12, 1)), L.Dropout(0.1), L.MaxPooling2D(2), L.Flatten(),
      L.Dense(4)], LOGITS, ()),                                                                         # dropout BEFORE pool
    ([L.Conv2D(8, 3, activation="relu", input_shape=(12, 12, 1)), L.AveragePooling2D(2), L.Flatten(), L.Dense(4)], LOGITS, ()),
    ([L.Conv2D(8, 3, activation="relu", input_shape=(12, 12, 1)), L.GlobalAveragePooling2D(), L.Dense(4)], LOGITS, ()),
    ([L.Flatten(input_shape=(4, 4, 2)), L.Dropout(0.5), L.Dense(4)], LOGITS, ()),                      # dropout after flatten
])
def test_models_outside_the_grammar_fall_back(layers, loss, metrics):
    assert _plan(layers, loss=loss, metrics=metrics) is None


def test_kernel_envelopes_split_k_and_tensor_core_conv_shapes():
    """Which shapes go to the split-K wgmma GEMM and to the wgmma convolution kernels (everything else is served by
    cuBLAS / cuDNN with a one-time warning)."""
    E = fastpath.FastSequentialEngine
    assert E._split_k(128, 128, 9216) == 24            # the MNIST Dense: 144 k-tiles, 6 per CTA
    assert E._split_k(128, 128, 64 * 31) == 1          # K too short to be worth splitting
    assert E._split_k(128, 128, 9217) == 1             # K not a multiple of 8 (TMA row pitch)
    assert E._split_k(2048, 1024, 9216) == 1           # many output tiles: a plain GEMM fills the machine
    assert 1 < E._split_k(256, 256, 4096) <= 144 // 4  # 4 tiles share the 144 CTAs
    assert E._split_k(128, 128, 9216, 4) == 36         # TFY_SPLITK_TILES=4: 4 k-tiles per CTA
    m = keras_mnist_cnn()
    m.compile(loss=LOGITS, optimizer="sgd")
    m.build()
    plan = fastpath.build_plan(m)
    c1, c2 = plan[0], plan[1]
    assert E._tc_conv(c2, 128) and E._tc_conv(c2, 2)
    assert not E._tc_conv(c2, 3)                       # odd batch: images are processed in pairs
    assert not E._tc_conv(c1, 128)                     # C_in = 1 has its own first-layer kernels
    # the TFY_NO_TC_CONV switch is applied when the step's kernels are chosen, to these and the C_in = 1 kernels:
    # test_fastpath_step_trace.py::test_no_tc_conv_switch_turns_every_tensor_core_convolution_kernel_off
