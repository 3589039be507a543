"""BASELINE config 2: Keras MNIST-CNN on the Horovod all-reduce path, one trainer per H100.

    python -m tf_yarn_b200.examples.baseline.mnist_cnn_allreduce

The model is the canonical Horovod ``keras_mnist`` network the reference's README compiles with
``Adadelta(1.0 * HVD_SIZE)`` (reference: README.md:104-113, examples/native_keras_with_gloo_example.py:65-90).
On H100 the whole step is ten kernels of this repo captured in a CUDA graph; the gradient exchange is the fused
reduce-scatter -> Adadelta -> all-gather kernel over NVSwitch.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch

from tf_yarn_b200 import hvd, keras
from tf_yarn_b200.examples import baseline
from tf_yarn_b200.models.mnist_cnn import keras_mnist_cnn, synthetic_mnist
from tf_yarn_b200.tensorflow import KerasExperiment, NodeLabel, TaskSpec, run_on_yarn

logging.basicConfig(level="INFO")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"mnist_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU
HVD_SIZE = baseline.n_trainers()
N_TRAIN, EPOCHS = (512, 1) if baseline.small() else (60000, int(os.environ.get("EXAMPLE_EPOCHS", "2")))


def experiment_fn() -> KerasExperiment:
    model = keras_mnist_cnn()
    opt = hvd.DistributedOptimizer(keras.optimizers.Adadelta(1.0 * HVD_SIZE))
    model.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True), optimizer=opt, metrics=["accuracy"])
    rank = int(os.environ.get("HOROVOD_RANK", "0"))
    x, y = synthetic_mnist(N_TRAIN, seed=rank)                      # every rank trains on its own shard
    callbacks = [hvd.keras.callbacks.BroadcastGlobalVariablesCallback(0),
                 keras.callbacks.ModelCheckpoint(MODEL_DIR + "/checkpoint-{epoch}")]
    return KerasExperiment(model, MODEL_DIR, {"batch_size": 128, "epochs": EPOCHS, "callbacks": callbacks, "verbose": 1},
                           input_data_fn=lambda: x, target_data_fn=lambda: y,
                           validation_data_fn=lambda: synthetic_mnist(256, seed=99))


def main():
    specs = {"chief": TaskSpec("8 GiB", 4, label=LABEL), "evaluator": TaskSpec("4 GiB", 2)}
    if HVD_SIZE > 1:
        specs["worker"] = TaskSpec("8 GiB", 4, instances=HVD_SIZE - 1, label=LABEL)
    return run_on_yarn(experiment_fn, specs, env={"TFY_KERAS_EVAL_POLL_SECS": "2"},
                       custom_task_module="tf_yarn_b200.tensorflow.tasks.gloo_allred_task")


if __name__ == "__main__":
    print(main())
