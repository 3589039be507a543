"""BASELINE config 3: Estimator wide & deep on the asynchronous parameter-server path
(1 chief + 5 workers + 2 ps on eight H100s; 1 chief + 1 worker + 1 ps on smaller boxes).

    python -m tf_yarn_b200.examples.baseline.wide_deep_ps

Same task program as the reference's default (reference: tf_yarn/tensorflow/tasks/_independent_workers_task.py:17-43,
examples/keras_example.py:94-107).  On H100 the ps ranks only own HBM: workers gather embedding rows inside the first
GEMM, stream the Dense weights over NVLink and push gradients with the FTRL / Adagrad update fused.
"""
import logging
import os
import tempfile
from datetime import datetime

import torch

from tf_yarn_b200 import estimator as est
from tf_yarn_b200.examples import baseline
from tf_yarn_b200.models import wide_deep
from tf_yarn_b200.tensorflow import Experiment, NodeLabel, TaskSpec, run_on_yarn

logging.basicConfig(level="INFO")
MODEL_DIR = os.path.join(tempfile.gettempdir(), "tf_yarn_b200_test", f"wide_deep_{int(datetime.now().timestamp())}")
LABEL = NodeLabel.GPU if torch.cuda.is_available() else NodeLabel.CPU
SMALL = baseline.small()
VOCAB, EMB, HIDDEN, N_CAT, BATCH, STEPS = (500, 8, (32, 16), 4, 64, 60) if SMALL else \
    (100_000, 64, (1024, 512, 256), 26, 512, int(os.environ.get("EXAMPLE_STEPS", "2000")))


def experiment_fn() -> Experiment:
    config = est.RunConfig(save_checkpoints_steps=max(STEPS // 2, 1), log_step_count_steps=max(STEPS // 4, 1))
    estimator = wide_deep.wide_deep_estimator(MODEL_DIR, vocab=VOCAB, emb_dim=EMB, hidden_units=HIDDEN, config=config,
                                              n_cat=N_CAT)
    train_fn = wide_deep.input_fn_factory(BATCH, 32, VOCAB, seed=int(os.environ.get("TFY_RANK", "0")), n_cat=N_CAT)
    eval_fn = wide_deep.input_fn_factory(BATCH, 4, VOCAB, seed=1234, repeat=False, n_cat=N_CAT)
    return Experiment(estimator, est.TrainSpec(train_fn, max_steps=STEPS),
                      est.EvalSpec(eval_fn, steps=None, start_delay_secs=0, throttle_secs=1))


def main():
    gpus = torch.cuda.device_count() if torch.cuda.is_available() else 0
    workers, ps = (5, 2) if gpus >= 8 else ((2, 1) if gpus >= 4 else (1, 1))
    return run_on_yarn(experiment_fn, {"chief": TaskSpec("8 GiB", 4, label=LABEL),
                                       "worker": TaskSpec("8 GiB", 4, instances=workers, label=LABEL),
                                       "ps": TaskSpec("8 GiB", 2, instances=ps, label=LABEL),
                                       "evaluator": TaskSpec("4 GiB", 2)})


if __name__ == "__main__":
    print(main())
