"""BASELINE.json config 3 through bench.py: Estimator wide-and-deep on the parameter-server path.

    python bench.py --config wide_deep --gpus 8 [--steps K --warmup W]        (plain python, NOT torchrun:
        the job is launched THROUGH the public API, `run_on_yarn`, which starts its own task processes)

Topology by --gpus (one H100 per cluster task; the BASELINE config is the 8-GPU row):

    8: 1 chief + 5 workers + 2 ps      4: 1 chief + 2 workers + 1 ps      2: 1 chief + 1 ps      1: chief and ps share GPU 0

ours    : DNNLinearCombinedClassifier (FTRL wide tower, Adagrad deep tower; 26 hashed categorical columns of 100k
          buckets, 13 numeric, embedding dim 64, hidden 1024-512-256, batch 512 per trainer) with the HBM parameter
          server: shards in the ps ranks' HBM, embedding rows gathered / pushed over NVLink by the K5/K6 kernels,
          Dense weights streamed by TMA into the wgmma GEMMs, whole step captured in a CUDA graph.
standin : the same model and topology written with stock PyTorch the way a TF-PS job works on an NCCL build:
          every step a worker receives the dense variables and the embedding rows it needs from the ps ranks
          (NCCL send/recv), runs cuBLAS/`embedding_bag`, sends the gradients back; the ps rank applies them
          (`index_add_` + Adagrad/FTRL) -- bench/ps_standin.py.
Every trainer runs W warm-up steps, meets the others on a KV barrier, then times K steps with CUDA events (device
time) and K more with the wall clock and a per-step loss read-back (end to end); value = trainers * batch * K /
max over trainers.  Asynchronous training: no cross-trainer synchronisation inside the region.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import time

from bench import common

BATCH = 512
VOCAB = 100_000
EMB = 64
HIDDEN = (1024, 512, 256)
N_CAT, N_NUM = 26, 13
METRIC = "samples/sec, Estimator wide-and-deep on the parameter-server path (whole job, asynchronous)"


def topology(n_gpus: int):
    return {8: (1, 5, 2), 4: (1, 2, 1), 2: (1, 0, 1), 1: (1, 0, 1)}[n_gpus]


class BenchHook:
    """SessionRunHook: warm-up, KV barrier, device-timed region, end-to-end region, result file, stop."""

    def __init__(self, steps: int, warmup: int, n_trainers: int, out_dir: str):
        self.steps, self.warmup, self.n, self.out_dir = steps, warmup, n_trainers, out_dir
        self.i = 0
        self.ev = None
        self.t0 = 0.0
        self.res = {}

    def begin(self):
        pass

    def after_create_session(self, *a):
        pass

    def before_run(self, ctx):
        return None

    def _barrier(self, tag):
        from tf_yarn_b200 import _task_commons
        kv = _task_commons.TaskClient.from_current().kv
        me = os.environ.get("TFY_TASK_KEY", "chief:0")
        kv[f"bench/{tag}/{me}"] = b"1"
        deadline = time.time() + 600
        while len(kv.keys(f"bench/{tag}/")) < self.n:
            if time.time() > deadline:
                raise TimeoutError("bench barrier")
            time.sleep(0.002)

    def after_run(self, ctx, values):
        import torch
        self.i += 1
        i, W, K = self.i, self.warmup, self.steps
        cuda = torch.cuda.is_available()
        if i == W:
            if cuda:
                torch.cuda.synchronize()
            self._barrier("start")
            if cuda:
                self.ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                self.ev[0].record()
            self.t0 = time.perf_counter()
        elif i == W + K:
            if cuda:
                self.ev[1].record()
                self.ev[1].synchronize()
                self.res["device_ms"] = self.ev[0].elapsed_time(self.ev[1])
            else:                                   # CPU plumbing run (no GPU in the container): wall clock
                self.res["device_ms"] = (time.perf_counter() - self.t0) * 1e3
            self._barrier("e2e")
            self.t0 = time.perf_counter()
        elif W + K < i <= W + 2 * K:
            loss = getattr(ctx.estimator, "_last_loss_t", None)
            if loss is not None:
                self.res["final_loss"] = float(loss)            # D2H read of the step's loss, every step
            if i == W + 2 * K:
                if cuda:
                    torch.cuda.synchronize()
                self.res["e2e_ms"] = (time.perf_counter() - self.t0) * 1e3
                ps = getattr(ctx.estimator, "_ps", None)
                if ps is not None and hasattr(ps, "traffic_per_step"):
                    self.res["traffic"] = ps.traffic_per_step()
                self.res["graph"] = bool(getattr(ctx.estimator, "_ps_graph", None) and
                                         "graph" in ctx.estimator._ps_graph)
                self.res["graph_error"] = (getattr(ctx.estimator, "_ps_graph", None) or {}).get("error")
                self.res["fused_first_layer"] = bool(getattr(ps, "fused_first", False))
                me = os.environ.get("TFY_TASK_KEY", "chief:0").replace(":", "_")
                with open(os.path.join(self.out_dir, f"bench_{me}.json"), "w") as f:
                    json.dump(self.res, f)
                ctx.request_stop()

    def end(self, *a):
        pass


def make_experiment_fn(model_dir, steps, warmup, n_trainers, out_dir):
    def experiment_fn():
        import torch
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200.models import wide_deep
        from tf_yarn_b200.tensorflow import Experiment
        e = wide_deep.wide_deep_estimator(model_dir, vocab=VOCAB, emb_dim=EMB, hidden_units=HIDDEN,
                                          config=est.RunConfig(save_checkpoints_steps=None, save_checkpoints_secs=None,
                                                               log_step_count_steps=None, save_summary_steps=None),
                                          n_cat=N_CAT, n_num=N_NUM)
        rank = int(os.environ.get("TFY_RANK", "0"))
        batches = wide_deep.synthetic_batches(BATCH, 64, VOCAB, seed=rank, n_cat=N_CAT, n_num=N_NUM)
        if torch.cuda.is_available():        # inputs come from pinned host memory every step
            batches = [({k: v.pin_memory() for k, v in f.items()}, y.pin_memory()) for f, y in batches]
        from tf_yarn_b200.data import Dataset

        def train_fn():
            return Dataset(lambda: iter(batches), len(batches)).repeat()
        hook = BenchHook(steps, warmup, n_trainers, out_dir)
        return Experiment(e, est.TrainSpec(train_fn, max_steps=None, hooks=[hook]),
                          est.EvalSpec(train_fn, steps=1, start_delay_secs=10 ** 6, throttle_secs=10 ** 6))
    return experiment_fn


def run(args):
    rank, _, _ = common.dist_env()
    if rank != 0:
        return 0                  # launched under torchrun by mistake: rank 0 alone drives run_on_yarn
    if args.impl == "reference":
        print(json.dumps({"impl": "reference", "unavailable": "the reference's Estimator/ParameterServer path needs "
                          "TensorFlow, which is not installable offline; see --impl standin"}))
        return 0
    if args.impl == "standin":
        from bench import ps_standin
        return ps_standin.run(args)
    n = args.gpus
    n_chief, n_worker, n_ps = topology(n)
    n_trainers = n_chief + n_worker
    steps, warm = args.steps, max(3, args.warmup) + 3          # +3: the eager steps before the graph capture
    out_dir = tempfile.mkdtemp(prefix="tfy_bench_wd_")
    model_dir = os.path.join(out_dir, "model")
    from tf_yarn_b200 import NodeLabel, TaskSpec
    from tf_yarn_b200.tensorflow import run_on_yarn
    specs = {"chief": TaskSpec("8 GiB", 4, label=NodeLabel.GPU),
             "ps": TaskSpec("8 GiB", 2, instances=n_ps, label=NodeLabel.GPU)}
    if n_worker:
        specs["worker"] = TaskSpec("8 GiB", 4, instances=n_worker, label=NodeLabel.GPU)
    sampler = common.ClockSampler(0, period_s=0.05)
    sampler.start()
    sampler.arm(True)
    t0 = time.time()
    # watchdog: a wedged job must not eat the GPU lease -- dump the task logs and give up
    import glob
    import threading

    def _watchdog():
        sys.stderr.write("bench watchdog: the job did not finish in time; task logs follow\n")
        for log in sorted(glob.glob("/tmp/tfy_application_*/logs/*/task.log"), key=os.path.getmtime)[-12:]:
            try:
                tail = open(log, errors="replace").read()[-1500:]
            except OSError:
                continue
            sys.stderr.write(f"==== {log}\n{tail}\n")
        print(json.dumps({"impl": "ours", "config": "wide_deep", "error": "timeout", "n_gpus": n}), flush=True)
        os._exit(1)

    wd_timer = threading.Timer(float(os.environ.get("TFY_BENCH_TIMEOUT", "240")), _watchdog)
    wd_timer.daemon = True
    wd_timer.start()
    run_on_yarn(make_experiment_fn(model_dir, steps, warm, n_trainers, out_dir), specs,
                env={"TFY_ARENA_MB": "2048", "TFY_FUSION_MB": "16"})
    wd_timer.cancel()
    wall = time.time() - t0
    clocks = sampler.stop()
    res = []
    for f in sorted(os.listdir(out_dir)):
        if f.startswith("bench_") and f.endswith(".json"):
            res.append(json.load(open(os.path.join(out_dir, f))))
    if len(res) != n_trainers:
        print(json.dumps({"impl": "ours", "error": f"{len(res)} of {n_trainers} trainers reported", "config": "wide_deep"}))
        return 1
    dev_ms = max(r["device_ms"] for r in res)
    e2e_ms = max(r["e2e_ms"] for r in res)
    value = n_trainers * BATCH * steps / (dev_ms * 1e-3)
    traffic = res[0].get("traffic", {})
    pull_b, push_b = traffic.get("pull_bytes", 0), traffic.get("push_bytes", 0)
    step_s = dev_ms * 1e-3 / steps
    out = {"metric": METRIC, "value": value, "unit": "samples/s", "n_gpus": n, "steps": steps, "warmup": warm,
           "repeats": 1, "ms_per_step": dev_ms / steps, "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "bf16 GEMMs, fp32 master on the ps", "data": "synthetic (Criteo-shaped), "
           "random-init weights", "impl": "ours",
           "config": {"model": f"wide-and-deep: {N_CAT} x {VOCAB} hashed categorical (emb {EMB}) + {N_NUM} numeric, "
                               f"hidden {HIDDEN}, FTRL(wide) + Adagrad(deep)", "topology": f"{n_chief} chief + {n_worker} "
                               f"workers + {n_ps} ps", "global_batch": n_trainers * BATCH, "per_gpu_batch": BATCH,
                      "seq_len": None, "parallelism": f"async-ps {n_trainers} trainers / {n_ps} ps",
                      "l2": "embedding tables (26 x 100k x 64 fp32 x 3 slots = 2 GB) exceed the 50 MB L2",
                      "cuda_graph": all(r.get("graph") for r in res), "graph_error": res[0].get("graph_error"),
                      "k5_gather_fused_into_first_gemm": all(r.get("fused_first_layer") for r in res),
                      "launched_by": "run_on_yarn"},
           "clocks": clocks,
           "e2e": {"value": n_trainers * BATCH * steps / (e2e_ms * 1e-3), "unit": "samples/s",
                   "h2d_bytes_per_step": BATCH * (N_NUM * 4 + N_CAT * 8 + 8), "d2h_bytes_per_step": 4, "steps": steps,
                   "ms_per_step": e2e_ms / steps, "final_loss": res[0].get("final_loss")},
           "gpu_launches": traffic.get("launches_per_step", 0) * steps,
           "nvlink": {"pull_bytes_per_step_per_trainer": pull_b, "push_bytes_per_step_per_trainer": push_b,
                      "pull_GBs_per_trainer": pull_b / step_s / 1e9 if step_s else None,
                      "push_GBs_per_trainer": push_b / step_s / 1e9 if step_s else None,
                      "of_770_GBs_link": (pull_b + push_b) / step_s / 1e9 / 770 if step_s else None},
           "job_wall_s": wall}
    common.emit(out)
    return 0
