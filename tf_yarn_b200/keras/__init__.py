"""mini-Keras: a torch/CUDA-backed subset of the Keras API (TensorFlow is not required).

The reference drives ``tf.keras`` models (``KerasExperiment``); this package
accepts the same user-code patterns and runs them on the H100 train engine
(:mod:`tf_yarn_b200.keras.engine`).
"""
from tf_yarn_b200.keras import callbacks, layers, losses, metrics, optimizers  # noqa: F401
from tf_yarn_b200.keras.models import Model, Sequential, load_model  # noqa: F401


class models:  # namespace parity: keras.models.load_model / keras.models.Sequential
    load_model = staticmethod(load_model)
    Sequential = Sequential
    Model = Model


class estimator:  # namespace parity: tf.keras.estimator.model_to_estimator (reference: examples/keras_example.py:64-65)
    @staticmethod
    def model_to_estimator(keras_model, model_dir=None, config=None, **kwargs):
        from tf_yarn_b200.estimator.canned import model_to_estimator as _impl    # late: estimator imports keras
        return _impl(keras_model, model_dir=model_dir, config=config, **kwargs)
