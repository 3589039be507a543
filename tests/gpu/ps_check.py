"""H100 check of the HBM parameter-server path (K5 pull incl. remote-weight GEMM, K6 push).

Run on a box with >= 2 GPUs:   python tests/gpu/ps_check.py [n_workers]
Topology: 1 chief + n_workers workers + 1 ps (one GPU each) + evaluator on CPU.
Asserts that training through the peer-memory kernels learns (eval accuracy rises).
"""
import json
import logging
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
logging.basicConfig(level=logging.INFO)

from tf_yarn_b200 import NodeLabel, TaskSpec  # noqa: E402
from tf_yarn_b200.tensorflow import Experiment, run_on_yarn  # noqa: E402

model_dir = tempfile.mkdtemp(prefix="tfy_ps_gpu_")
N_WORKERS = int(sys.argv[1]) if len(sys.argv) > 1 else 0
N_PS = int(sys.argv[2]) if len(sys.argv) > 2 else 1
MAX_STEPS = 300


def experiment_fn():
    from tf_yarn_b200 import estimator as est
    from tf_yarn_b200 import keras
    from tf_yarn_b200.models import wide_deep
    vocab = 20_000
    e = wide_deep.wide_deep_estimator(model_dir, vocab=vocab, emb_dim=32, hidden_units=(256, 128),
                                      optimizer=lambda: keras.optimizers.Adagrad(0.05),
                                      config=est.RunConfig(save_checkpoints_steps=100, log_step_count_steps=50),
                                      n_cat=8, n_num=8)
    rank = int(os.environ.get("TFY_RANK", "0"))
    train_fn = wide_deep.input_fn_factory(512, 64, vocab, seed=rank, n_cat=8, n_num=8)
    eval_fn = wide_deep.input_fn_factory(512, 8, vocab, seed=999, repeat=False, n_cat=8, n_num=8)
    return Experiment(e, est.TrainSpec(train_fn, max_steps=MAX_STEPS),
                      est.EvalSpec(eval_fn, steps=None, start_delay_secs=0, throttle_secs=1))


specs = {"chief": TaskSpec("4 GiB", 4, label=NodeLabel.GPU), "ps": TaskSpec("4 GiB", 2, instances=N_PS, label=NodeLabel.GPU),
         "evaluator": TaskSpec("4 GiB", 2)}
if N_WORKERS:
    specs["worker"] = TaskSpec("4 GiB", 4, instances=N_WORKERS, label=NodeLabel.GPU)
metrics = run_on_yarn(experiment_fn, specs, env={"TFY_ARENA_MB": "512", "TFY_FUSION_MB": "16"})
from tf_yarn_b200.estimator import summary  # noqa: E402
sc = summary.read_scalars(os.path.join(model_dir, "eval"))
acc = [(s, v) for s, n, v in zip(sc["step"], sc["name"], sc["value"]) if n == "accuracy"]
print("eval accuracy by step:", acc)
os.makedirs("gpurun_out", exist_ok=True)
json.dump({"accuracy": acc, "training_s": metrics.total_training_duration.total_seconds(), "workers": N_WORKERS,
           "ps": N_PS, "max_steps": MAX_STEPS},
          open(f"gpurun_out/ps_check_w{N_WORKERS}_ps{N_PS}.json", "w"))
assert acc and acc[-1][1] > max(0.6, acc[0][1]), acc
print("PS CHECK OK")
