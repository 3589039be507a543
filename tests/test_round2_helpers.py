"""Host-side helpers added in round 2: CPU-set planning of the launcher, checkpoint-name parsing of the Keras
evaluator, the bench harness' region arithmetic and the results-table generator."""
import json
import os
import subprocess
import sys

import pytest

from tf_yarn_b200.launcher import local
from tf_yarn_b200.tensorflow.tasks import evaluator_task
from tf_yarn_b200.topologies import NodeLabel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _app(services):
    app = local.LocalApplication.__new__(local.LocalApplication)
    app.spec = local.ApplicationSpec(services=services)
    return app


def _svc(instances, vcores, label):
    return local.ServiceSpec(script="true", instances=instances, nb_proc=1, label=label, memory=64, vcores=vcores, env={},
                             files={})


def test_cpu_plan_gives_disjoint_sets_gpu_tasks_first(monkeypatch):
    monkeypatch.setattr(os, "sched_getaffinity", lambda pid: set(range(16)))
    monkeypatch.delenv("TFY_PIN_CPUS", raising=False)
    plan = _app({"evaluator": _svc(1, 2, NodeLabel.CPU), "chief": _svc(1, 4, NodeLabel.GPU),
                 "worker": _svc(2, 4, NodeLabel.GPU)})._cpu_plan()
    assert plan["chief:0"] == [0, 1, 2, 3] and plan["worker:0"] == [4, 5, 6, 7] and plan["worker:1"] == [8, 9, 10, 11]
    assert plan["evaluator:0"] == [12, 13]
    sets = [set(v) for v in plan.values()]
    assert sum(len(s) for s in sets) == len(set().union(*sets))           # pairwise disjoint


def test_cpu_plan_oversubscribed_box_shares_the_rest_and_can_be_disabled(monkeypatch, caplog):
    monkeypatch.setattr(os, "sched_getaffinity", lambda pid: set(range(6)))
    app = _app({"chief": _svc(1, 4, NodeLabel.GPU), "worker": _svc(1, 4, NodeLabel.GPU),
                "tensorboard": _svc(1, 1, NodeLabel.CPU)})
    plan = app._cpu_plan()
    assert plan["chief:0"] == [0, 1, 2, 3]
    assert plan["worker:0"] == [4, 5] and plan["tensorboard:0"]            # partial, never empty
    monkeypatch.setenv("TFY_PIN_CPUS", "0")
    assert app._cpu_plan() == {}


@pytest.mark.parametrize("name,step", [("x/model.ckpt-123", 123), ("weights.01.h5", 1), ("weights.02.h5", 2),
                                       ("model-7.pt2", 7), ("ckpt_0003.keras", 3), ("dir/checkpoint-7.ckpt", 7),
                                       ("weights.02-0.35.h5", 2), ("run2/epoch-11.weights.h5", 11)])
def test_checkpoint_step_parsing_ignores_extensions_and_metrics(name, step):
    assert evaluator_task._get_step(name) == step


def test_checkpoint_without_a_step_is_rejected_loudly():
    with pytest.raises(ValueError, match="cannot parse a training step"):
        evaluator_task._get_step("best.keras")


def test_bench_region_arithmetic():
    sys.path.insert(0, ROOT)
    from bench import common
    # one timed region of exactly --steps steps unless more regions are requested
    assert common.pick_repeats(20) == 1 and common.pick_repeats(200) == 1 and common.pick_repeats(1000) == 1
    assert common.pick_repeats(20, requested=7) == 7
    assert common.median([3.0, 1.0, 2.0]) == 2.0 and common.median([4.0, 1.0, 2.0, 3.0]) == 2.5


def test_results_table_reads_the_committed_bench_lines():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "results_table.py"),
                          os.path.join(ROOT, "tests", "golden", "bench_lines")], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    assert "| 8 |" in out.stdout and "Scaling efficiency" in out.stdout and "### wide_deep" in out.stdout
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_lines", "bench_mnist_ours_N8_t.json")))
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in d, key
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["params_in_sync"] is True


def test_component_map_paths_exist():
    """docs/ComponentMap.md maps every SURVEY.md §2 row to files of this repo: none of them may be stale."""
    import re
    text = open(os.path.join(ROOT, "docs", "ComponentMap.md")).read()
    paths = set(re.findall(r"`((?:tf_yarn_b200|tests|profiles|docs|tools|bench)/[A-Za-z0-9_./]+|setup\.py|setup\.cfg|"
                           r"requirements\.txt|tests-requirements\.txt|README\.md|__graft_entry__\.py|"
                           r"\.github/workflows/main\.yml)`", text))
    assert len(paths) > 80
    missing = [p for p in sorted(paths) if not os.path.exists(os.path.join(ROOT, p))]
    assert missing == []
    for row in range(1, 34):                                        # every §2.1 row is present
        assert re.search(rf"^\| {row} \|", text, re.M), row
