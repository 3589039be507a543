"""BASELINE config 5: Keras BERT-base pre-training on the Horovod all-reduce path, bf16, one trainer per H100,
with the evaluator and TensorBoard side tasks.

    python -m tf_yarn_b200.examples.baseline.bert_allreduce

The torch module is wrapped as a mini-Keras model (``keras.Model.from_torch``): forward / backward run through the
autograd graph engine (cuBLAS / SDPA kernels captured in a CUDA graph), the 110 M-parameter gradient exchange is the
fused reduce-scatter -> Adam -> all-gather kernel.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch

from tf_yarn_b200 import hvd, keras
from tf_yarn_b200.examples import baseline
from tf_yarn_b200.models import bert
from tf_yarn_b200.tensorflow import KerasExperiment, NodeLabel, TaskSpec, run_on_yarn

logging.basicConfig(level="INFO")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"bert_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU
SMALL = baseline.small()
ARCH = dict(vocab=2000, hidden=32, layers=2, heads=2, intermediate=64, max_pos=32) if SMALL else {}
BATCH, SEQ, STEPS = (4, 16, 6) if SMALL else (32, 128, int(os.environ.get("EXAMPLE_STEPS", "200")))
HVD_SIZE = baseline.n_trainers()


def experiment_fn() -> KerasExperiment:
    model = keras.Model.from_torch(bert.BertForPreTraining(**ARCH), name="bert")
    model.compile(loss=bert.pretraining_loss, optimizer=hvd.DistributedOptimizer(keras.optimizers.Adam(1e-4)))
    rank = int(os.environ.get("HOROVOD_RANK", "0"))
    vocab = ARCH.get("vocab", 30522)
    batches = [bert.synthetic_batch(BATCH, SEQ, vocab=vocab, seed=rank * 100 + i) for i in range(8)]

    def train_batches():
        i = 0
        while True:
            yield batches[i % len(batches)]
            i += 1
    callbacks = [hvd.keras.callbacks.BroadcastGlobalVariablesCallback(0),
                 keras.callbacks.ModelCheckpoint(MODEL_DIR + "/checkpoint-{epoch}")]
    return KerasExperiment(model, MODEL_DIR, {"steps_per_epoch": STEPS, "epochs": 1, "callbacks": callbacks, "verbose": 1},
                           input_data_fn=train_batches, target_data_fn=None,
                           validation_data_fn=lambda: iter(batches[:2]))


def main():
    specs = {"chief": TaskSpec("16 GiB", 8, label=LABEL), "evaluator": TaskSpec("8 GiB", 2),
             "tensorboard": TaskSpec("2 GiB", 1, tb_model_dir=MODEL_DIR, tb_termination_timeout_seconds=2)}
    if HVD_SIZE > 1:
        specs["worker"] = TaskSpec("16 GiB", 8, instances=HVD_SIZE - 1, label=LABEL)
    return run_on_yarn(experiment_fn, specs, env={"TFY_KERAS_EVAL_POLL_SECS": "2"},
                       custom_task_module="tf_yarn_b200.tensorflow.tasks.gloo_allred_task")


if __name__ == "__main__":
    print(main())
