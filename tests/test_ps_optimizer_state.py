"""The parameter servers' optimizer slots in estimator checkpoints (``ps_state``), on the shared-memory plane
(estimator/ps.py): the matching rule on its own, then whole jobs through ``run_on_yarn`` (chief + ps tasks) that
stop at step 3 and resume from the checkpoint.  A canned wide-and-deep classifier trains on the same batch every
step, with no dropout: a resumed job must end bit for bit where an uninterrupted one does."""
import logging
import os
import shutil
import sys
from types import SimpleNamespace

import pytest
import torch

from tf_yarn_b200.estimator import checkpoint as ckpt
from tf_yarn_b200.estimator import ps

HYPER = {"lr": 0.1, "p1": 0.9, "p2": 0.0, "eps": 1e-7, "wd": 0.0, "init_s1": 0.1, "flags": 0}
INIT_S1 = 0.1       # initial_accumulator_value of keras.optimizers.Adagrad and Ftrl


def _layout(variables, kinds, hypers=None, n_ps=1):
    return ps.Layout(variables, n_ps, kinds[0], HYPER, kinds=kinds, hypers=hypers or [HYPER] * len(variables))


def _regions(layout):
    """region(i, s) over zeroed CPU tensors, as the shards come from the ps tasks."""
    store = {(i, s): torch.zeros(layout.numel[i]) for i in range(len(layout.variables))
             for s in range(1 + layout.var_slots[i])}
    return lambda i, s=0: store[(i, s)]


# ------------------------------------------------------------------------------------------------ the matching rule
def test_slots_are_restored_by_name_when_kind_slots_and_size_match(caplog):
    rms_momentum = dict(HYPER, p2=0.9)                  # mean square, momentum
    rms_centered = dict(HYPER, flags=1)                 # mean square, mean gradient: two slots as well
    saved = _layout([("wide", [10, 1]), ("deep", [10, 4]), ("rms", [3]), ("resized", [5]), ("gone", [2])],
                    ["ftrl", "adagrad", "rmsprop", "adam", "sgd"], [HYPER, HYPER, rms_momentum, HYPER, HYPER])
    src = _regions(saved)
    for i in range(len(saved.variables)):
        for s in range(1, 1 + saved.var_slots[i]):
            src(i, s).copy_(torch.arange(saved.numel[i]) + 100.0 * i + 10.0 * s)
    state = ps.export_slots(saved, src)
    assert state["wide"]["kind"] == "ftrl" and state["wide"]["slot_names"] == ["n", "z"]
    assert state["rms"]["slot_names"] == ["ms", "momentum"] and state["gone"]["slots"] == []
    assert all(t.dtype == torch.float32 and t.device.type == "cpu" for e in state.values() for t in e["slots"])

    # another job: other ps count and order, the wide tower at another learning rate, the deep tower on Adam
    now = _layout([("new", [4]), ("rms", [3]), ("deep", [10, 4]), ("resized", [6]), ("wide", [10, 1])],
                  ["adagrad", "rmsprop", "adam", "adam", "ftrl"], [HYPER, rms_centered, HYPER, HYPER,
                                                                  dict(HYPER, lr=0.5)], n_ps=3)
    with caplog.at_level(logging.WARNING, logger=ps.logger.name):
        got = ps.match_slots(state, now)
    assert [g is not None for g in got] == [False, False, False, False, True]
    assert all(torch.equal(a, b) for a, b in zip(got[4], state["wide"]["slots"]))
    warnings = [r.getMessage() for r in caplog.records if r.levelno == logging.WARNING]
    assert len(warnings) == 1 and all(n in warnings[0] for n in ("new", "rms", "deep", "resized"))
    assert "wide" not in warnings[0]

    dst = _regions(now)
    ps.init_slots(now, dst, state)
    assert torch.equal(dst(4, 1), src(0, 1)) and torch.equal(dst(4, 2), src(0, 2))
    assert torch.all(dst(0, 1) == INIT_S1) and torch.all(dst(2, 1) == 0) and torch.all(dst(1, 2) == 0)
    assert all(torch.all(dst(i, 0) == 0) for i in range(5))             # the values are not the slots' business
    fresh = _regions(now)
    ps.init_slots(now, fresh, None)                                    # no ps_state: every slot starts fresh
    assert torch.all(fresh(0, 1) == INIT_S1) and torch.all(fresh(4, 1) == INIT_S1) and torch.all(fresh(4, 2) == 0)


# ------------------------------------------------------------------------------- whole jobs on the shared-memory plane
def _experiment(model_dir, deep, max_steps):
    def experiment_fn():
        from tf_yarn_b200 import estimator as est
        from tf_yarn_b200 import keras
        from tf_yarn_b200.data import Dataset
        from tf_yarn_b200.estimator import feature_column as fc
        from tf_yarn_b200.tensorflow import Experiment
        g = torch.Generator().manual_seed(0)
        x = torch.randn(64, 3, generator=g)
        cat = torch.randint(0, 10, (64,), generator=g)
        batch = ({"x": x, "cat": cat}, ((x[:, 0] + (cat.float() - 4.5) * 0.3) > 0).long())

        def input_fn():
            torch.manual_seed(1)            # the network is built right after: the same initial values in every job
            return Dataset(lambda: iter([batch]), 1).repeat()
        deep_opt = {"adagrad": lambda: keras.optimizers.Adagrad(0.1), "adam": lambda: keras.optimizers.Adam(0.01),
                    "rmsprop": lambda: keras.optimizers.RMSprop(0.01, momentum=0.9, centered=True)}[deep]
        cat_col = fc.categorical_column_with_identity("cat", 10)
        e = est.DNNLinearCombinedClassifier(
            model_dir=model_dir, linear_feature_columns=[cat_col, fc.numeric_column("x", (3,))],
            linear_optimizer=lambda: keras.optimizers.Ftrl(0.05, l1_regularization_strength=0.001),
            dnn_feature_columns=[fc.embedding_column(cat_col, 4), fc.numeric_column("x", (3,))],
            dnn_hidden_units=[16], dnn_optimizer=deep_opt,
            config=est.RunConfig(save_checkpoints_steps=1, keep_checkpoint_max=10, log_step_count_steps=None))
        return Experiment(e, est.TrainSpec(input_fn, max_steps=max_steps), est.EvalSpec(input_fn, steps=1))
    return experiment_fn


def _train(model_dir, deep="adagrad", max_steps=6, n_ps=1, gpu=False):
    """One job of a chief and n_ps ps tasks; gpu: every task on its own GPU, the HBM plane."""
    import cloudpickle

    from tf_yarn_b200 import NodeLabel
    from tf_yarn_b200.tensorflow import TaskSpec, run_on_yarn
    cloudpickle.register_pickle_by_value(sys.modules[__name__])
    label = NodeLabel.GPU if gpu else NodeLabel.CPU
    run_on_yarn(_experiment(str(model_dir), deep, max_steps),
                {"chief": TaskSpec("1 GiB", 1, label=label), "ps": TaskSpec("1 GiB", 1, instances=n_ps, label=label)},
                env={"TFY_ARENA_MB": "512"} if gpu else {})


def _ckpt(model_dir, step):
    return ckpt.load_checkpoint(os.path.join(str(model_dir), f"{ckpt.PREFIX}{step}"))


def _assert_same(a, b, only=None):
    """Bit-identical checkpoints (of the variables whose names start with `only`, when given)."""
    keep = (lambda n: n.startswith(only)) if only else (lambda n: True)
    assert a["global_step"] == b["global_step"]
    assert a["network"].keys() == b["network"].keys() and a["ps_state"].keys() == b["ps_state"].keys()
    for n, v in a["network"].items():
        if keep(n):
            assert torch.equal(v, b["network"][n]), n
    for n, e in a["ps_state"].items():
        if keep(n):
            f = b["ps_state"][n]
            assert (e["kind"], e["shape"], e["slot_names"]) == (f["kind"], f["shape"], f["slot_names"]), n
            for s, (t, u) in enumerate(zip(e["slots"], f["slots"])):
                assert torch.equal(t, u), (n, s)


@pytest.fixture(scope="module")
def jobs(tmp_path_factory):
    """Per deep-tower optimizer: `straight` trained to step 6 in one job; `resumed` to step 3, then to 6 by a second
    job on the same directory; `at3` a copy of that directory between the two."""
    done = {}

    def get(deep):
        if deep not in done:
            root = tmp_path_factory.mktemp(deep)
            r = SimpleNamespace(straight=root / "straight", resumed=root / "resumed", at3=root / "at3")
            _train(r.straight, deep)
            _train(r.resumed, deep, max_steps=3)
            shutil.copytree(r.resumed, r.at3)
            _train(r.resumed, deep)
            done[deep] = r
        return done[deep]
    return get


@pytest.mark.slow
@pytest.mark.parametrize("deep", ["adagrad", "adam", "rmsprop"])
def test_a_resumed_job_ends_where_an_uninterrupted_one_does(jobs, deep):
    """FTRL on the wide tower; Adagrad, Adam or centered RMSprop with momentum (three slots) on the deep tower."""
    r = jobs(deep)
    a = _ckpt(r.straight, 6)
    _assert_same(_ckpt(r.straight, 3), _ckpt(r.at3, 3))
    _assert_same(a, _ckpt(r.resumed, 6))
    assert {e["kind"] for e in a["ps_state"].values()} == {"ftrl", deep}
    for n, e in a["ps_state"].items():                      # the slots saved are trained ones, not initial values
        assert len(e["slots"]) == {"ftrl": 2, "adagrad": 1, "adam": 2, "rmsprop": 3}[e["kind"]], n
        for s, t in enumerate(e["slots"]):
            assert torch.any(t != (INIT_S1 if s == 0 and e["kind"] in ("ftrl", "adagrad") else 0.0)), (n, s)


@pytest.mark.slow
def test_a_checkpoint_without_ps_state_resumes_with_fresh_slots(jobs, tmp_path):
    """A checkpoint written before the slots were saved: the job resumes from init_s1 and zero slots, exactly as a
    checkpoint holding those values does, and so no longer ends where the uninterrupted job does."""
    r = jobs("adagrad")
    old, fresh = tmp_path / "old", tmp_path / "fresh"
    shutil.copytree(r.at3, old)
    shutil.copytree(r.at3, fresh)
    path = os.path.join(str(old), f"{ckpt.PREFIX}3")
    payload = ckpt.load_checkpoint(path)
    state = payload.pop("ps_state")
    torch.save(payload, path)
    for e in state.values():
        for s, t in enumerate(e["slots"]):
            t.fill_(INIT_S1 if s == 0 and e["kind"] in ("adagrad", "ftrl") else 0.0)
    torch.save(dict(payload, ps_state=state), os.path.join(str(fresh), f"{ckpt.PREFIX}3"))
    _train(old)
    _train(fresh)
    _assert_same(_ckpt(old, 6), _ckpt(fresh, 6))
    straight = _ckpt(r.straight, 6)
    assert any(not torch.equal(v, straight["network"][n]) for n, v in _ckpt(old, 6)["network"].items())


@pytest.mark.slow
def test_a_changed_optimizer_starts_its_variables_fresh(jobs, tmp_path):
    """The deep tower switched from Adagrad to Adam on resuming: its variables start Adam from zero slots while the
    wide tower's FTRL slots are restored.  Step 4 pulls the values of step 3, so its gradients are the uninterrupted
    job's: the wide tower ends step 4 bit for bit where that job does, and one Adam step from zero leaves
    v / (1 - beta2) = (m / (1 - beta1))^2."""
    r = jobs("adagrad")
    d = tmp_path / "adam"
    shutil.copytree(r.at3, d)
    _train(d, deep="adam", max_steps=4)
    got = _ckpt(d, 4)
    _assert_same(_ckpt(r.straight, 4), got, only="linear.")
    deep = {n: e for n, e in got["ps_state"].items() if not n.startswith("linear.")}
    assert deep and all(e["kind"] == "adam" for e in deep.values())
    for n, e in deep.items():
        m, v = e["slots"]
        assert torch.any(m != 0), n
        torch.testing.assert_close(v / (1 - 0.999), (m / (1 - 0.9)) ** 2, rtol=1e-4, atol=1e-12)


@pytest.mark.slow
def test_a_job_resumes_on_another_number_of_ps_tasks(jobs, tmp_path):
    """Written with 1 ps task, resumed on 2: the variables are matched by name and placed round-robin anew; the
    updates do not depend on the placement, so the job ends where the uninterrupted one does."""
    r = jobs("adagrad")
    d = tmp_path / "two_ps"
    shutil.copytree(r.at3, d)
    _train(d, n_ps=2)
    _assert_same(_ckpt(r.straight, 6), _ckpt(d, 6))
