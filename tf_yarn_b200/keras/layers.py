"""Keras-style layers backed by torch modules.

Only what the reference's examples and BASELINE configs need (reference:
tf_yarn/examples/keras_example.py:55-62, native_keras_with_gloo_example.py:65-69,
README.md:104-109) plus the blocks of the MNIST-CNN and BERT-base configs.

Layout: like Keras, image tensors are NHWC at the API (``input_shape=(28, 28,
1)``).  Internally a 4-D activation is a torch tensor with NCHW *logical*
shape in ``channels_last`` memory format -- the NHWC bytes untouched -- which
is the layout cuDNN's bf16 tensor-core kernels want on H100.
"""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

_ACTIVATIONS: Dict[str, Callable[[torch.Tensor], torch.Tensor]] = {
    "linear": lambda x: x,
    "relu": F.relu,
    "gelu": F.gelu,
    "tanh": torch.tanh,
    "sigmoid": torch.sigmoid,
    "softmax": lambda x: F.softmax(x, dim=-1),
    "elu": F.elu,
    "selu": F.selu,
    "softplus": F.softplus,
    "swish": F.silu,
    "silu": F.silu,
}


def get_activation(name: Union[None, str, Callable]) -> Tuple[str, Callable]:
    if name is None:
        return "linear", _ACTIVATIONS["linear"]
    if callable(name):
        return getattr(name, "__name__", "custom"), name
    if name not in _ACTIVATIONS:
        raise ValueError(f"unknown activation {name!r}")
    return name, _ACTIVATIONS[name]


def _init_(t: torch.Tensor, name, default: str) -> None:
    """Keras initializer names (``kernel_initializer="he_normal"`` ...) on a torch parameter; callables get the tensor."""
    name = default if name is None else name
    if callable(name):
        name(t)
        return
    key = str(name).lower()
    table = {
        "glorot_uniform": nn.init.xavier_uniform_, "xavier_uniform": nn.init.xavier_uniform_,
        "glorot_normal": nn.init.xavier_normal_, "xavier_normal": nn.init.xavier_normal_,
        "he_normal": lambda w: nn.init.kaiming_normal_(w, nonlinearity="relu"),
        "he_uniform": lambda w: nn.init.kaiming_uniform_(w, nonlinearity="relu"),
        "lecun_normal": lambda w: nn.init.kaiming_normal_(w, nonlinearity="linear"),
        "zeros": nn.init.zeros_, "ones": nn.init.ones_,
        "random_normal": lambda w: nn.init.normal_(w, std=0.05),
        "random_uniform": lambda w: nn.init.uniform_(w, -0.05, 0.05),
    }
    if key not in table:
        raise ValueError(f"unknown initializer {name!r}")
    table[key](t)


def _pair(v) -> Tuple[int, int]:
    return (v, v) if isinstance(v, int) else (int(v[0]), int(v[1]))


class Layer:
    """Base class: ``build(input_shape)`` creates the torch module, ``call(x)`` applies it.

    ``input_shape`` / ``output_shape`` exclude the batch dimension and follow the
    Keras (channels-last) convention.
    """

    def __init__(self, name: Optional[str] = None, input_shape: Optional[Sequence[int]] = None, **kwargs):
        if kwargs:
            raise TypeError(f"{type(self).__name__}: unexpected arguments {sorted(kwargs)}")
        self.name = name
        self._declared_input_shape = tuple(input_shape) if input_shape is not None else None
        self.module: Optional[nn.Module] = None
        self.built = False
        self.input_shape_: Optional[Tuple[int, ...]] = None
        self.output_shape_: Optional[Tuple[int, ...]] = None

    # subclasses override -------------------------------------------------------
    def build_module(self, input_shape: Tuple[int, ...]) -> Optional[nn.Module]:
        return None

    def compute_output_shape(self, input_shape: Tuple[int, ...]) -> Tuple[int, ...]:
        return input_shape

    def call(self, x: torch.Tensor, training: bool) -> torch.Tensor:
        return self.module(x) if self.module is not None else x

    def get_config(self) -> Dict[str, Any]:
        return {"name": self.name}

    # -------------------------------------------------------------------------
    def build(self, input_shape: Sequence[int]) -> Tuple[int, ...]:
        input_shape = tuple(int(s) for s in input_shape)
        self.input_shape_ = input_shape
        self.module = self.build_module(input_shape)
        self.output_shape_ = tuple(self.compute_output_shape(input_shape))
        self.built = True
        return self.output_shape_

    def count_params(self) -> int:
        return sum(p.numel() for p in self.module.parameters()) if self.module is not None else 0

    def __call__(self, x: torch.Tensor, training: bool = False) -> torch.Tensor:
        return self.call(x, training)


class InputLayer(Layer):
    def __init__(self, input_shape: Sequence[int], **kw):
        super().__init__(input_shape=input_shape, **kw)

    def get_config(self):
        return {"name": self.name, "input_shape": list(self._declared_input_shape)}


class Dense(Layer):
    def __init__(self, units: int, activation=None, use_bias: bool = True, kernel_initializer=None,
                 bias_initializer=None, **kw):
        super().__init__(**kw)
        self.units = int(units)
        self.use_bias = use_bias
        self.activation_name, self.activation = get_activation(activation)
        self.kernel_initializer, self.bias_initializer = kernel_initializer, bias_initializer

    def build_module(self, input_shape):
        lin = nn.Linear(input_shape[-1], self.units, bias=self.use_bias)
        # Keras defaults: glorot_uniform kernel, zero bias
        _init_(lin.weight, self.kernel_initializer, "glorot_uniform")
        if lin.bias is not None:
            _init_(lin.bias, self.bias_initializer, "zeros")
        return lin

    def compute_output_shape(self, input_shape):
        return input_shape[:-1] + (self.units,)

    def call(self, x, training):
        return self.activation(self.module(x))

    def get_config(self):
        return {"name": self.name, "units": self.units, "activation": self.activation_name,
                "use_bias": self.use_bias, "input_shape": list(self._declared_input_shape)
                if self._declared_input_shape else None}


class Conv2D(Layer):
    def __init__(self, filters: int, kernel_size, strides=(1, 1), padding: str = "valid", activation=None,
                 use_bias: bool = True, kernel_initializer=None, bias_initializer=None, **kw):
        super().__init__(**kw)
        self.kernel_initializer, self.bias_initializer = kernel_initializer, bias_initializer
        self.filters = int(filters)
        self.kernel_size = _pair(kernel_size)
        self.strides = _pair(strides)
        self.padding = padding.lower()
        if self.padding not in ("valid", "same"):
            raise ValueError("padding must be 'valid' or 'same'")
        self.use_bias = use_bias
        self.activation_name, self.activation = get_activation(activation)

    def build_module(self, input_shape):
        h, w, c = input_shape
        pad = "same" if self.padding == "same" else 0
        conv = nn.Conv2d(c, self.filters, self.kernel_size, self.strides, padding=pad, bias=self.use_bias)
        _init_(conv.weight, self.kernel_initializer, "glorot_uniform")
        if conv.bias is not None:
            _init_(conv.bias, self.bias_initializer, "zeros")
        return conv.to(memory_format=torch.channels_last)

    def compute_output_shape(self, input_shape):
        h, w, _ = input_shape
        if self.padding == "same":
            oh, ow = math.ceil(h / self.strides[0]), math.ceil(w / self.strides[1])
        else:
            oh = (h - self.kernel_size[0]) // self.strides[0] + 1
            ow = (w - self.kernel_size[1]) // self.strides[1] + 1
        return (oh, ow, self.filters)

    def call(self, x, training):
        return self.activation(self.module(x))

    def get_config(self):
        return {"name": self.name, "filters": self.filters, "kernel_size": list(self.kernel_size),
                "strides": list(self.strides), "padding": self.padding, "activation": self.activation_name,
                "use_bias": self.use_bias,
                "input_shape": list(self._declared_input_shape) if self._declared_input_shape else None}


class MaxPooling2D(Layer):
    def __init__(self, pool_size=(2, 2), strides=None, padding: str = "valid", **kw):
        super().__init__(**kw)
        self.pool_size = _pair(pool_size)
        self.strides = _pair(strides) if strides is not None else self.pool_size
        self.padding = padding.lower()

    def compute_output_shape(self, input_shape):
        h, w, c = input_shape
        if self.padding == "same":
            return (math.ceil(h / self.strides[0]), math.ceil(w / self.strides[1]), c)
        return ((h - self.pool_size[0]) // self.strides[0] + 1, (w - self.pool_size[1]) // self.strides[1] + 1, c)

    def call(self, x, training):
        if self.padding == "same":
            ph = max(0, (math.ceil(x.shape[2] / self.strides[0]) - 1) * self.strides[0] + self.pool_size[0] - x.shape[2])
            pw = max(0, (math.ceil(x.shape[3] / self.strides[1]) - 1) * self.strides[1] + self.pool_size[1] - x.shape[3])
            x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float("-inf"))
        return F.max_pool2d(x, self.pool_size, self.strides)

    def get_config(self):
        return {"name": self.name, "pool_size": list(self.pool_size), "strides": list(self.strides),
                "padding": self.padding}


class AveragePooling2D(MaxPooling2D):
    def call(self, x, training):
        if self.padding != "same":
            return F.avg_pool2d(x, self.pool_size, self.strides)
        # TF 'same': pad (possibly one more row / column at the end) and average over the REAL elements only
        ph = max(0, (math.ceil(x.shape[2] / self.strides[0]) - 1) * self.strides[0] + self.pool_size[0] - x.shape[2])
        pw = max(0, (math.ceil(x.shape[3] / self.strides[1]) - 1) * self.strides[1] + self.pool_size[1] - x.shape[3])
        pads = (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)
        total = F.avg_pool2d(F.pad(x, pads), self.pool_size, self.strides)
        ones = torch.ones((1, 1) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)
        share = F.avg_pool2d(F.pad(ones, pads), self.pool_size, self.strides)
        return total / share


class GlobalAveragePooling2D(Layer):
    def compute_output_shape(self, input_shape):
        return (input_shape[-1],)

    def call(self, x, training):
        return x.mean(dim=(2, 3))


class Flatten(Layer):
    def compute_output_shape(self, input_shape):
        n = 1
        for s in input_shape:
            n *= s
        return (n,)

    def call(self, x, training):
        if x.dim() == 4:
            # logical NCHW over NHWC bytes: flattening in Keras (H, W, C) order is a free view
            return x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)
        return x.reshape(x.shape[0], -1)


class Dropout(Layer):
    def __init__(self, rate: float, **kw):
        super().__init__(**kw)
        self.rate = float(rate)

    def call(self, x, training):
        return F.dropout(x, self.rate, training) if training and self.rate > 0 else x

    def get_config(self):
        return {"name": self.name, "rate": self.rate}


class Activation(Layer):
    def __init__(self, activation, **kw):
        super().__init__(**kw)
        self.activation_name, self.activation = get_activation(activation)

    def call(self, x, training):
        return self.activation(x)

    def get_config(self):
        return {"name": self.name, "activation": self.activation_name}


class ReLU(Activation):
    def __init__(self, **kw):
        super().__init__("relu", **kw)

    def get_config(self):
        return {"name": self.name}


class Softmax(Activation):
    def __init__(self, **kw):
        super().__init__("softmax", **kw)

    def get_config(self):
        return {"name": self.name}


class BatchNormalization(Layer):
    def __init__(self, momentum: float = 0.99, epsilon: float = 1e-3, **kw):
        super().__init__(**kw)
        self.momentum, self.epsilon = momentum, epsilon

    def build_module(self, input_shape):
        c = input_shape[-1]
        cls = nn.BatchNorm2d if len(input_shape) == 3 else nn.BatchNorm1d
        return cls(c, eps=self.epsilon, momentum=1.0 - self.momentum)

    def get_config(self):
        return {"name": self.name, "momentum": self.momentum, "epsilon": self.epsilon}


class LayerNormalization(Layer):
    def __init__(self, epsilon: float = 1e-3, **kw):
        super().__init__(**kw)
        self.epsilon = epsilon

    def build_module(self, input_shape):
        return nn.LayerNorm(input_shape[-1], eps=self.epsilon)

    def call(self, x, training):
        if x.dim() == 4:          # images are logical NCHW over NHWC bytes: normalise the channel axis, like Keras
            return self.module(x.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
        return self.module(x)

    def get_config(self):
        return {"name": self.name, "epsilon": self.epsilon}


class Embedding(Layer):
    def __init__(self, input_dim: int, output_dim: int, **kw):
        super().__init__(**kw)
        self.input_dim, self.output_dim = int(input_dim), int(output_dim)

    def build_module(self, input_shape):
        emb = nn.Embedding(self.input_dim, self.output_dim)
        nn.init.uniform_(emb.weight, -0.05, 0.05)
        return emb

    def compute_output_shape(self, input_shape):
        return tuple(input_shape) + (self.output_dim,)

    def call(self, x, training):
        return self.module(x.long())

    def get_config(self):
        return {"name": self.name, "input_dim": self.input_dim, "output_dim": self.output_dim}


class TorchModule(Layer):
    """Wrap any ``torch.nn.Module`` as a layer (used for BERT-base and other non-Sequential bodies)."""

    def __init__(self, module: nn.Module, output_shape: Optional[Sequence[int]] = None, **kw):
        super().__init__(**kw)
        self._wrapped = module
        self._out_shape = tuple(output_shape) if output_shape is not None else None

    def build_module(self, input_shape):
        return self._wrapped

    def compute_output_shape(self, input_shape):
        return self._out_shape if self._out_shape is not None else input_shape

    def get_config(self):
        return {"name": self.name, "module": self._wrapped, "output_shape": self._out_shape}


LAYER_CLASSES = {cls.__name__: cls for cls in (
    InputLayer, Dense, Conv2D, MaxPooling2D, AveragePooling2D, GlobalAveragePooling2D, Flatten, Dropout,
    Activation, ReLU, Softmax, BatchNormalization, LayerNormalization, Embedding, TorchModule)}
