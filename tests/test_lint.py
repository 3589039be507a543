"""Static gate that runs where no linter can be installed: tools/lint_names.py (undefined globals, unused imports)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_no_undefined_names_or_unused_imports():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "lint_names.py"), "tf_yarn_b200", "bench", "tests",
                          "tools", "bench.py", "__graft_entry__.py"], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout


def test_lint_catches_an_undefined_global(tmp_path):
    bad = tmp_path / "bad.py"
    bad.write_text("import os\n\n\ndef f():\n    return dist.get_rank()\n")
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "lint_names.py"), str(bad)], capture_output=True,
                         text=True)
    assert res.returncode == 1
    assert "undefined name 'dist'" in res.stdout and "unused import 'os'" in res.stdout


def test_async_copy_ptx_lives_only_in_the_tma_header():
    """The mbarrier / TMA protocol is written once, in ops/csrc/tfy_tma.cuh; a kernel file that spells the PTX itself
    is a private copy that a fix to the shared helpers would miss (and that the PDL prologue check cannot see)."""
    csrc = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")
    found = {}
    for name in sorted(os.listdir(csrc)):
        with open(os.path.join(csrc, name)) as f:
            code = re.sub(r"//[^\n]*", "", f.read())
        for token in ("mbarrier.", "cp.async.bulk.tensor", "elect.sync", "prefetch.tensormap", "fence.proxy.async",
                      "cuTensorMapEncodeTiled"):
            if token in code:
                found.setdefault(token, []).append(name)
    assert found == {token: ["tfy_tma.cuh"] for token in found} and len(found) == 6, found
