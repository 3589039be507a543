"""Keras model -> Estimator, trained with the asynchronous parameter-server strategy.

1 chief + 4 workers + 2 ps + evaluator, as in the reference (reference:
tf_yarn/examples/keras_example.py:55-107).  On a H100 box give the trainers / ps tasks
``label=NodeLabel.GPU``: the shards then live in the ps ranks' HBM and are pulled / pushed over
NVLink (K5 / K6 kernels); on a CPU box they live in shared memory.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch

from tf_yarn_b200 import estimator as est
from tf_yarn_b200 import keras
from tf_yarn_b200.examples import winequality
from tf_yarn_b200.tensorflow import Experiment, NodeLabel, TaskSpec, run_on_yarn

logging.basicConfig(level="INFO")

WINE_QUALITY_FILE = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", "winequality-red.csv")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"keras_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU


def experiment_fn() -> Experiment:
    def convert(features, label):
        return {"features": torch.tensor([features[k] for k in winequality.FEATURES])}, label

    def train_input_fn():
        return winequality.get_dataset(WINE_QUALITY_FILE, split="train").map(convert).shuffle(1000).batch(128).repeat()

    def eval_input_fn():
        return winequality.get_dataset(WINE_QUALITY_FILE, split="test").map(convert).shuffle(1000).batch(128)

    model = keras.Sequential()
    model.add(keras.layers.Dense(units=300, activation="relu", input_shape=(11,)))
    model.add(keras.layers.Dense(units=100, activation="relu"))
    model.add(keras.layers.Dense(units=10, activation="softmax"))
    model.summary()
    model.compile(loss="sparse_categorical_crossentropy", optimizer="sgd", metrics=["accuracy"])
    estimator = est.model_to_estimator(model, config=est.RunConfig(model_dir=MODEL_DIR, save_checkpoints_steps=50))
    return Experiment(estimator, est.TrainSpec(train_input_fn, max_steps=100),
                      est.EvalSpec(eval_input_fn, steps=10, start_delay_secs=0, throttle_secs=5))


def main():
    winequality.ensure_dataset(WINE_QUALITY_FILE)
    return run_on_yarn(experiment_fn, task_specs={
        "chief": TaskSpec(memory="2 GiB", vcores=4, label=LABEL),
        "worker": TaskSpec(memory="2 GiB", vcores=4, instances=4, label=LABEL),
        "ps": TaskSpec(memory="2 GiB", vcores=8, instances=2, label=LABEL),
        "evaluator": TaskSpec(memory="2 GiB", vcores=1),
    })


if __name__ == "__main__":
    print(main())
