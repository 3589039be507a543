"""Wall time of Estimator._save on the HBM parameter server, for bench/wide_deep.py's model (26 x 100k x 64 embedding
tables, FTRL wide tower, Adagrad deep tower), with and without the optimizer slots (``ps_state``).

Run on an H100 box:   python tests/gpu/ps_checkpoint_time.py [repeats [out.json]]
Topology: 1 chief + 1 ps, on GPUs 0 and 1 when there are two, else sharing GPU 0.  After a few training steps the
chief saves the checkpoint `repeats` times each way, alternating: weights only (what a checkpoint held before the
slots were saved), then weights and slots.  Prints the result as JSON, and writes it to out.json when given.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from bench import wide_deep as wd  # noqa: E402
from tf_yarn_b200 import NodeLabel, TaskSpec  # noqa: E402
from tf_yarn_b200.tensorflow import Experiment, run_on_yarn  # noqa: E402

REPEATS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
OUT = sys.argv[2] if len(sys.argv) > 2 else None
WARM = 8                 # past the eager steps and the CUDA-graph capture


class SaveTimer:
    def __init__(self, out_dir):
        self.out_dir, self.i = out_dir, 0

    def begin(self):
        pass

    def after_create_session(self, *a):
        pass

    def before_run(self, ctx):
        return None

    def end(self, *a):
        pass

    def after_run(self, ctx, values):
        import torch
        self.i += 1
        if self.i < WARM:
            return
        est = ctx.estimator
        conn = est._ps
        with_slots = conn.optimizer_state
        rows = []
        for _ in range(REPEATS):
            for slots in (False, True):
                conn.optimizer_state = with_slots if slots else (lambda: None)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                path = est._save()
                rows.append({"slots": slots, "save_s": time.perf_counter() - t0, "bytes": os.path.getsize(path)})
            t0 = time.perf_counter()
            state = with_slots()
            rows.append({"optimizer_state_s": time.perf_counter() - t0,
                         "slot_bytes": sum(t.numel() * 4 for e in state.values() for t in e["slots"])})
        conn.optimizer_state = with_slots
        with open(os.path.join(self.out_dir, "rows.json"), "w") as f:
            json.dump(rows, f)
        ctx.request_stop()


def experiment_fn_for(model_dir, out_dir):
    vocab, emb, hidden, n_cat, n_num, batch = wd.VOCAB, wd.EMB, wd.HIDDEN, wd.N_CAT, wd.N_NUM, wd.BATCH

    def experiment_fn():
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200.data import Dataset
        from tf_yarn_b200.models import wide_deep
        e = wide_deep.wide_deep_estimator(model_dir, vocab=vocab, emb_dim=emb, hidden_units=hidden,
                                          config=est.RunConfig(save_checkpoints_steps=None, save_checkpoints_secs=None,
                                                               log_step_count_steps=None, save_summary_steps=None),
                                          n_cat=n_cat, n_num=n_num)
        batches = wide_deep.synthetic_batches(batch, 8, vocab, seed=0, n_cat=n_cat, n_num=n_num)

        def train_fn():
            return Dataset(lambda: iter(batches), len(batches)).repeat()
        return Experiment(e, est.TrainSpec(train_fn, max_steps=None, hooks=[SaveTimer(out_dir)]),
                          est.EvalSpec(train_fn, steps=1, start_delay_secs=10 ** 6, throttle_secs=10 ** 6))
    return experiment_fn


def main():
    out_dir = tempfile.mkdtemp(prefix="tfy_ps_ckpt_time_")
    model_dir = os.path.join(out_dir, "model")
    specs = {"chief": TaskSpec("8 GiB", 4, label=NodeLabel.GPU), "ps": TaskSpec("8 GiB", 2, label=NodeLabel.GPU)}
    run_on_yarn(experiment_fn_for(model_dir, out_dir), specs, env={"TFY_ARENA_MB": "2048", "TFY_FUSION_MB": "16"})
    rows = json.load(open(os.path.join(out_dir, "rows.json")))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    saves = {k: sorted(r["save_s"] for r in rows if r.get("slots") is k) for k in (False, True)}
    out = {"gpus": gpu, "model_dir": model_dir, "repeats": REPEATS, "rows": rows,
           "median_save_s": {"weights_only": saves[False][len(saves[False]) // 2],
                             "weights_and_slots": saves[True][len(saves[True]) // 2]},
           "checkpoint_bytes": {"weights_only": next(r["bytes"] for r in rows if r.get("slots") is False),
                                "weights_and_slots": next(r["bytes"] for r in rows if r.get("slots") is True)}}
    print(json.dumps(out, indent=1))
    if OUT:
        os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
        with open(OUT, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
