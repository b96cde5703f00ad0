"""Host-side planning of the reduced-camera-system solve (coslam_b200/csrc/ba_plan.h), on CPU:
tests/plan_emul.cpp executes the plan's task list sequentially with plain loops, asserts that every
task's wait conditions already hold when its turn comes (the list is a topological order => the
spinning ticket scheduler of ba_tile_solve cannot deadlock) and compares the solution with a dense
Cholesky solve."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path_factory.mktemp("plan") / "plan_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "plan_emul.cpp")])
    return exe


def _run(exe, *args):
    out = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-2000:]
    return json.loads(out.stdout.splitlines()[-2])


@pytest.mark.parametrize("args", [
    (1, "dense", 0), (7, "band", 2), (12, "dense", 0),       # local BA sizes (one / two blocks)
    (40, "dense", 0), (29, "dense", 0),                      # dense co-visibility, several blocks
    (100, "random", 0.05), (150, "random", 0.01),            # irregular co-visibility
    (200, "band", 20), (200, "band", 20, 0), (200, "band", 20, 2),
    (396, "band", 35), (396, "band", 35, 3),
])
def test_plan_is_topological_and_solves(emul, args):
    st = _run(emul, *args)
    assert st["rel_err"] < 1e-10
    assert st["tiles"] >= st["tiles_orig"] >= st["nb"]


def test_nested_dissection_shortens_the_critical_path(emul):
    """c4 shape: 796 free poses, band 35.  Two-sided elimination alone = 167 dependent tasks;
    the automatic dissection depth must cut that by more than half."""
    flat = _run(emul, 796, "band", 35, 0)
    auto = _run(emul, 796, "band", 35)
    assert flat["nd_depth"] == 0 and auto["nd_depth"] >= 2
    assert auto["critical_cost"] < 0.5 * flat["critical_cost"]
    assert auto["gflop"] < 4 * flat["gflop"]  # bounded fill
    assert auto["diag_sums"] > 0 and auto["bwd_not4"] > 0


def test_band_plans_reach_the_scratch_and_chunk_edges(emul):
    """The band patterns of tests/test_gpu_ba_tile_solve.py reach the SUM of diagonal scratch tiles
    (their rhs parts) and BWD wait lists that end in a partial chunk of 4."""
    st = _run(emul, 121, "band", 29, 1)
    assert st["nd_depth"] == 1 and st["scratch"] > 0
    assert st["diag_sums"] > 0 and st["bwd_not4"] > 0
