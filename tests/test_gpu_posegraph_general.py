"""CUDA general pose graphs (cosl_posegraph_solve: computeNewCameraRotations +
computeNewCameraTranslations4 on any edge set, normal equations solved by the BA's tile Cholesky) against
the reference-generated vectors tests/golden/posegraph_merge_ref.npz and posegraph_ref.npz, against the
CPU oracle (pinned to the compiled reference by tests/test_posegraph_general.py) and against the chain
kernel.  Floating point: 1e-9 absolute on R and t (O(1) values), 1e-9 relative on scales."""
import os
import subprocess

import numpy as np
import pytest

from coslam_b200.synth import make_merge_graph, make_pose_chains, make_pose_graph, scale_columns
from oracle import orc_pg_general as orc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TOL = 1e-9
KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et")


def _args(g):
    return [g[k] for k in KEYS] + [g["scale_col"], g["n_scale"]]


def _close(a, b, c):
    (R0, t0, s0), (R1, t1, s1) = a, b
    assert np.abs(R0 - R1).max() < TOL, c
    assert np.abs(t0 - t1).max() < TOL, c
    assert np.all(np.abs(s0 - s1) <= TOL * np.maximum(1.0, np.abs(s1))), c


def test_reference_merge_golden(api):
    z = np.load(os.path.join(HERE, "golden", "posegraph_merge_ref.npz"))
    for i in range(int(z["n_cases"])):
        c = {k: z[f"c{i}_{k}"] for k in KEYS + ("scale_id", "newR", "newt", "s")}
        col, ns = scale_columns(c["scale_id"])
        nR, nt, s = api.posegraph_solve(*(c[k] for k in KEYS), col, ns)
        assert np.abs(nR - c["newR"]).max() < TOL, i
        assert np.abs(nt - c["newt"]).max() < TOL, i
        unc = c["scale_id"] >= 0
        assert np.all(np.abs(s[col[unc]] - c["s"][unc]) <= TOL * np.abs(c["s"][unc])), i


def test_reference_general_golden(api):
    """Cases 6 and 7 of posegraph_ref.npz: a skip edge and a loop closure, solved by the reference."""
    z = np.load(os.path.join(HERE, "golden", "posegraph_ref.npz"))
    for i in range(int(z["n_chain_cases"]), int(z["n_cases"])):
        nR, nt, _ = api.posegraph_solve(z[f"c{i}_fixed"], z[f"c{i}_R"], z[f"c{i}_t"], z[f"c{i}_id1"],
                                        z[f"c{i}_id2"], z[f"c{i}_eR_list"], z[f"c{i}_et_list"])
        assert np.abs(nR - z[f"c{i}_newR"]).max() < TOL, i
        assert np.abs(nt - z[f"c{i}_newt"]).max() < TOL, i


@pytest.mark.parametrize("n,kw", [
    (3, dict()),                                                      # one block: ba_tile_two
    (12, dict(loops=2, parallel=1, reverse=1)),
    (40, dict(fixed_every=9, loops=3, fixed_pairs=2, n_scale=1, uncertain=2)),
    (90, dict(components=3, loops=2, reverse=2, n_scale=2, uncertain=3)),
    (300, dict(fixed_every=50, loops=4, parallel=3, reverse=3, fixed_pairs=1, n_scale=2, uncertain=4)),
    (2000, dict(loops=1, n_scale=1, uncertain=2)),                    # long chain + loop closure
])
def test_oracle_parity_general(api, n, kw):
    g = make_pose_graph(n, seed=n, **kw)
    _close(api.posegraph_solve(*_args(g)), orc.posegraph_solve(*_args(g)), (n, kw))


@pytest.mark.parametrize("K,C,nc,ns", [(100, 4, 2, 1), (30, 13, 3, 2), (12, 8, 1, 1)])
def test_oracle_parity_merge(api, K, C, nc, ns):
    g = make_merge_graph(K, C, seed=K * C, n_constraints=nc, n_scale_ids=ns, noise=0.01)
    _close(api.posegraph_solve(*_args(g)), orc.posegraph_solve(*_args(g)), (K, C))


def test_consistent_merge_returns_the_input(api):
    g = make_merge_graph(40, 13, seed=3, n_constraints=3, n_scale_ids=2)
    nR, nt, s = api.posegraph_solve(*_args(g))
    assert np.abs(nR - g["R"]).max() < 1e-10 and np.abs(nt - g["t"]).max() < 1e-10
    assert np.abs(s - g["true_scale"]).max() < 1e-10
    fx = g["fixed"].astype(bool)
    assert np.array_equal(nR[fx], g["R"][fx]) and np.array_equal(nt[fx], g["t"][fx])


def test_chains_match_the_chain_kernel(api):
    g = make_pose_chains([37, 120, 5], key_every=6, seed=4, shift=0.1)
    cR, ct = api.posegraph_spread_chains(g["chain_off"], g["fixed"], g["R"], g["t"], g["eR"], g["et"])
    nR, nt, _ = api.posegraph_solve(g["fixed"], g["R"], g["t"], g["id1"], g["id2"], g["eR_list"], g["et_list"])
    assert np.abs(nR - cR).max() < TOL and np.abs(nt - ct).max() < TOL


def test_bit_reproducible(api):
    g = make_pose_graph(700, seed=8, fixed_every=60, loops=5, parallel=2, n_scale=2, uncertain=3)
    a = api.posegraph_solve(*_args(g))
    b = api.posegraph_solve(*_args(g))
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64))


def test_error_cases(api):
    g = make_pose_graph(10, seed=1, n_scale=1, uncertain=1)
    base = _args(g)

    def call(**over):
        a = dict(zip(KEYS + ("scale_col", "n_scale"), [np.copy(x) if isinstance(x, np.ndarray) else x
                                                        for x in base]))
        a.update(over)
        return api.posegraph_solve(*(a[k] for k in KEYS + ("scale_col", "n_scale")))

    id1 = np.copy(g["id1"])
    id1[0] = 10
    with pytest.raises(api.CoslError, match="error -1"):
        call(id1=id1)
    id2 = np.copy(g["id2"])
    id2[1] = g["id1"][1]
    with pytest.raises(api.CoslError, match="self-loop"):
        call(id2=id2)
    sc = np.copy(g["scale_col"])
    sc[sc >= 0] = 1
    with pytest.raises(api.CoslError, match="error -1"):
        call(scale_col=sc)
    with pytest.raises(api.CoslError, match="scale column 1 gets no row"):
        call(n_scale=2)
    fx = np.zeros_like(g["fixed"])
    with pytest.raises(api.CoslError, match="node 0 .*without a fixed node"):
        call(fixed=fx)
    two = make_pose_graph(20, seed=2, components=2)
    fx = np.copy(two["fixed"])
    fx[10] = 0
    with pytest.raises(api.CoslError, match="node 10 "):
        api.posegraph_solve(fx, *_args(two)[1:])
    et = np.copy(g["et"])
    et[g["scale_col"] >= 0] = 0.0  # the scale column is zero: singular normal matrix
    with pytest.raises(api.CoslError, match="error -4"):
        call(et=et)
    R = np.copy(g["R"])
    R[0, 0, 0] = np.nan
    with pytest.raises(api.CoslError, match="error -4"):
        call(R=R)
    # the device is still usable
    nR, nt, s = call()
    assert np.isfinite(nR).all() and np.isfinite(s).all()


def test_shim_merge_executable(api, tmp_path):
    """A caller compiled with COSL_POSEGRAPH_GENERAL runs a merge-shaped graph through the shim header
    (computeNewCameraRotations + computeNewCameraTranslations4) and matches the oracle."""
    exe = os.path.join(str(tmp_path), "shim_merge_caller")
    lib = os.path.join(ROOT, "coslam_b200")
    subprocess.check_call(["/usr/bin/g++", "-std=c++11", "-Wall", "-Werror", "-DCOSL_POSEGRAPH_GENERAL",
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "coslam_b200", "shim"),
                           os.path.join(HERE, "stubs", "posegraph_merge_caller.cpp"), "-o", exe, "-L" + lib,
                           "-lcoslam_b200", "-Wl,-rpath," + lib])
    g = make_merge_graph(9, 4, seed=12, n_constraints=3, n_scale_ids=2, noise=0.01)
    inp = os.path.join(str(tmp_path), "graph.bin")
    _write_graph(inp, g)
    out = subprocess.run([exe, inp], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    vals = np.array(out.stdout.split()[1:], dtype=np.float64)
    n, ne = len(g["fixed"]), len(g["id1"])
    nR, nt, s = vals[:9 * n].reshape(n, 3, 3), vals[9 * n:12 * n].reshape(n, 3), vals[12 * n:12 * n + ne]
    oR, ot, os_ = orc.posegraph_solve(*_args(g))
    assert np.abs(nR - oR).max() < TOL and np.abs(nt - ot).max() < TOL
    unc = g["scale_id"] >= 0
    assert np.abs(s[unc] - os_[g["scale_col"][unc]]).max() < TOL
    assert np.all(s[~unc] == 0.0)


def _write_graph(path, g):
    n, ne = len(g["fixed"]), len(g["id1"])
    with open(path, "wb") as f:
        np.array([n, ne], np.int32).tofile(f)
        g["fixed"].astype(np.int32).tofile(f)
        g["R"].astype(np.float64).tofile(f)
        g["t"].astype(np.float64).tofile(f)
        g["id1"].astype(np.int32).tofile(f)
        g["id2"].astype(np.int32).tofile(f)
        g["eR"].astype(np.float64).tofile(f)
        g["et"].astype(np.float64).tofile(f)
        g["scale_id"].astype(np.int32).tofile(f)
