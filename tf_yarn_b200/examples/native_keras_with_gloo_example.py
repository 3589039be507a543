"""Keras model trained with the synchronous all-reduce task (the reference's Horovod-gloo example).

(reference: tf_yarn/examples/native_keras_with_gloo_example.py:41-111)

Every trainer is one process on one H100; gradients are averaged by the fused
reduce-scatter -> Adadelta -> all-gather kernel over NVLink (gloo only on CPU-only boxes).
The evaluator picks up the chief's ``ModelCheckpoint`` files.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch

from tf_yarn_b200 import hvd, keras
from tf_yarn_b200.examples import winequality
from tf_yarn_b200.tensorflow import KerasExperiment, NodeLabel, TaskSpec, run_on_yarn

logging.basicConfig(level="INFO")

WINE_QUALITY_FILE = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", "winequality-red.csv")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"hvd_keras_{int(datetime.now().timestamp())}")
HVD_SIZE = 2
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU


def experiment_fn() -> KerasExperiment:
    def convert_to_tensor(x, y):
        return torch.tensor([x[k] for k in winequality.FEATURES]), torch.tensor(y)

    def input_data_fn():
        return (winequality.get_dataset(WINE_QUALITY_FILE, split="train").map(convert_to_tensor)
                .shuffle(1000).batch(128).repeat())

    def validation_data_fn():
        return winequality.get_dataset(WINE_QUALITY_FILE, split="test").map(convert_to_tensor).shuffle(1000).batch(128)

    model = keras.Sequential()
    model.add(keras.layers.Dense(units=300, activation="relu", input_shape=(11,)))
    model.add(keras.layers.Dense(units=100, activation="relu"))
    model.add(keras.layers.Dense(units=10, activation="softmax"))
    model.summary()
    opt = keras.optimizers.Adadelta(1.0 * HVD_SIZE)
    opt = hvd.DistributedOptimizer(opt)
    model.compile(loss="sparse_categorical_crossentropy", optimizer=opt, metrics=["accuracy"])
    my_callbacks = [
        keras.callbacks.ModelCheckpoint(MODEL_DIR + "/checkpoint-{epoch}"),
        hvd.keras.callbacks.BroadcastGlobalVariablesCallback(0),
    ]
    train_params = {"steps_per_epoch": 100, "epochs": 2, "callbacks": my_callbacks}
    return KerasExperiment(model=model, model_dir=MODEL_DIR, train_params=train_params, input_data_fn=input_data_fn,
                           target_data_fn=None, validation_data_fn=validation_data_fn)


def main():
    winequality.ensure_dataset(WINE_QUALITY_FILE)
    return run_on_yarn(
        experiment_fn,
        task_specs={
            "chief": TaskSpec(memory="2 GiB", vcores=4, label=LABEL),
            "worker": TaskSpec(memory="2 GiB", vcores=4, instances=(HVD_SIZE - 1), label=LABEL),
            "evaluator": TaskSpec(memory="2 GiB", vcores=1),
        },
        env={"TFY_KERAS_EVAL_POLL_SECS": "2"},
        custom_task_module="tf_yarn_b200.tensorflow.tasks.gloo_allred_task")


if __name__ == "__main__":
    print(main())
