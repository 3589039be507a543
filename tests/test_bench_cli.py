import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_needs_a_gpu_and_says_so():
    """On a CPU box the reference arm exits 0 with an `unavailable` line (its worker wraps the model in NCCL DDP)."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference"], capture_output=True,
                         text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and "unavailable" in line


def test_reference_control_plane_through_the_shims(monkeypatch):
    """The UNMODIFIED reference's control-plane code (event.broadcast / wait, choose_master, _get_experiment,
    TaskSpec) runs against this repo's KV server through bench/shims (what `bench.py --impl reference` relies on)."""
    import pytest
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "tf_yarn")):
        pytest.skip("oracle/_ref is not built: build() installs it when the original project's sources exist")
    code = r"""
import os, sys
sys.path[:0] = [os.path.join(%r, "bench", "shims"), %r, %r]
from tf_yarn_b200.kv import start_server
srv = start_server()
os.environ["TFY_REF_KV_ADDR"] = srv.address
os.environ["SKEIN_CONTAINER_ID"] = "worker_0"
import cloudpickle, skein
from tf_yarn import constants, event
from tf_yarn._task_commons import _get_experiment, choose_master, get_task_key
from tf_yarn.topologies import TaskSpec
from tf_yarn.pytorch.tasks import worker
c = skein.ApplicationClient.from_current()
c.kv[constants.KV_EXPERIMENT_FN] = cloudpickle.dumps(lambda: ("exp", 42))
assert _get_experiment(c) == ("exp", 42)
assert get_task_key().to_kv_str() == "worker:0"
host, port = choose_master(c, 0)
assert event.wait(c, "MASTER_PORT") == str(port)
assert TaskSpec(memory="2 GiB", vcores=4).memory == 2048
assert callable(worker._train)
srv.stop()
print("OK")
""" % (ROOT, ref, ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr


def test_graft_entry_build_is_idempotent():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "__graft_entry__.py")], capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0, out.stderr
    assert os.path.exists(os.path.join(ROOT, "tf_yarn_b200", "ops", "lib", "libtfy_b200.so"))
    assert os.path.exists(os.path.join(ROOT, "tf_yarn_b200", "kv", "libtfy_kv.so"))
