"""The selected-inversion plan of coslam_b200/csrc/ba_plan.h (ba_make_selinv_plan), on CPU: tests/selinv_emul.cpp
factors the structures of test_ba_plan.py, runs the plan's steps one task after the other -- asserting that the
factor has no entry outside the tile pattern and that every operand tile of a task is final when its turn
comes -- and writes S and Z; Z must match numpy.linalg.inv(S) on every block of the pattern."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path_factory.mktemp("selinv") / "selinv_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "selinv_emul.cpp")])
    return exe


def block_errors(Z, Sinv, mask):
    """Per pattern block (a, c): |Z_ac - inv_ac|_F / sqrt(|inv_aa|_F |inv_cc|_F) (the scale an SPD inverse's
    off-diagonal block is bounded by)."""
    mf = mask.shape[0]
    B = lambda M, a, c: M[6 * a:6 * a + 6, 6 * c:6 * c + 6]  # noqa: E731
    dn = np.array([np.linalg.norm(B(Sinv, a, a)) for a in range(mf)])
    errs = [np.linalg.norm(B(Z, a, c) - B(Sinv, a, c)) / np.sqrt(dn[a] * dn[c])
            for a, c in zip(*np.nonzero(mask))]
    return np.array(errs)


@pytest.mark.parametrize("args", [
    (1, "dense", 0), (7, "band", 2), (12, "dense", 0),
    (40, "dense", 0), (29, "dense", 0),
    (100, "random", 0.05), (150, "random", 0.01),
    (200, "band", 20), (200, "band", 20, 0), (200, "band", 20, 2),
    (396, "band", 35), (396, "band", 35, 3),
    # block-diagonal S (every step without an operation, separator blocks of 6 rows at mf = 100) and two
    # connected components
    (12, "band", 0), (20, "band", 0), (25, "band", 0), (30, "band", 0), (61, "band", 0), (100, "band", 0),
    (100, "band", 0, 2), (40, "split", 3), (41, "split", 2, 1),
])
def test_selinv_plan_matches_the_dense_inverse(emul, tmp_path, args):
    out = subprocess.run([emul, str(tmp_path), *map(str, args)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-2000:]
    st = json.loads(out.stdout.splitlines()[-2])
    mf = args[0]
    ns = 6 * mf
    S = np.fromfile(tmp_path / "S.bin").reshape(ns, ns)
    Z = np.fromfile(tmp_path / "Z.bin").reshape(ns, ns)
    mask = np.fromfile(tmp_path / "mask.bin", np.uint8).reshape(mf, mf)
    assert st["steps"] == st["nb"] and st["tasks"] >= st["nb"]
    if args[1:3] == ("band", 0):
        assert st["ops"] == 0 and st["tasks"] == st["nb"], st
    assert np.array_equal(mask, mask.T) and mask.diagonal().all()
    err = block_errors(Z, np.linalg.inv(S), mask)
    assert err.max() < 1e-10, (st, float(err.max()))
    # nothing outside the pattern blocks
    outside = np.kron(1 - mask, np.ones((6, 6))).astype(bool)
    assert not Z[outside].any()
