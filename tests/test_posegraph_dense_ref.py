"""The dense float64 least-squares reference of the pose-graph solves (tests/posegraph_dense.py), on the CPU,
before any GPU test trusts it: against the compiled reference's vectors (tests/golden/posegraph_ref.npz: 6
chain cases + 2 general graphs; posegraph_merge_ref.npz: 7 merge cases with shared scales) and against
the general-graph oracle (oracle/posegraph_general_oracle.cpp) on graphs with up to 13 scale columns.
Both solve paths of the reference (dense SVD least squares, sparse augmented system) are checked.
Tolerance 1e-9 absolute on R and t (O(1) values), 1e-9 relative on the scales."""
import os

import numpy as np
import pytest

import posegraph_dense as dense
from coslam_b200.synth import make_merge_graph, make_pose_chains, make_pose_graph, scale_columns
from oracle import orc_pg_general as orc

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1e-9
KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et")
METHODS = ("dense", "sparse")


@pytest.mark.parametrize("method", METHODS)
def test_reference_golden_chains_and_general_graphs(method):
    z = np.load(os.path.join(HERE, "golden", "posegraph_ref.npz"))
    assert int(z["n_cases"]) == 8 and int(z["n_chain_cases"]) == 6
    for i in range(int(z["n_cases"])):
        r = dense.solve(z[f"c{i}_fixed"], z[f"c{i}_R"], z[f"c{i}_t"], z[f"c{i}_id1"], z[f"c{i}_id2"],
                        z[f"c{i}_eR_list"], z[f"c{i}_et_list"], method=method)
        assert np.abs(r["newR"] - z[f"c{i}_newR"]).max() < TOL, i
        assert np.abs(r["newt"] - z[f"c{i}_newt"]).max() < TOL, i


@pytest.mark.parametrize("method", METHODS)
def test_reference_golden_merge_graphs(method):
    z = np.load(os.path.join(HERE, "golden", "posegraph_merge_ref.npz"))
    assert int(z["n_cases"]) == 7
    for i in range(int(z["n_cases"])):
        c = {k: z[f"c{i}_{k}"] for k in KEYS + ("scale_id", "newR", "newt", "s")}
        col, ns = scale_columns(c["scale_id"])
        r = dense.solve(*(c[k] for k in KEYS), col, ns, method=method)
        assert np.abs(r["newR"] - c["newR"]).max() < TOL, i
        assert np.abs(r["newt"] - c["newt"]).max() < TOL, i
        unc = col >= 0
        assert np.all(np.abs(r["scale"][col[unc]] - c["s"][unc]) <= TOL * np.abs(c["s"][unc])), i


@pytest.mark.parametrize("kind,kw", [
    ("graph", dict(n_nodes=40, fixed_every=9, loops=3, parallel=2, reverse=2, fixed_pairs=1, n_scale=2, uncertain=3)),
    ("graph", dict(n_nodes=60, fixed_every=10, loops=3, reverse=2, n_scale=7, uncertain=9)),
    ("graph", dict(n_nodes=90, components=3, loops=2, n_scale=13, uncertain=13)),
    ("graph", dict(n_nodes=400, fixed_every=80, loops=4, parallel=3, n_scale=12, uncertain=14)),
    ("merge", dict(n_key=30, n_cams=13, n_constraints=3, n_scale_ids=2, noise=0.01)),
    ("merge", dict(n_key=12, n_cams=8, n_constraints=9, n_scale_ids=9, noise=0.02)),
])
def test_reference_matches_the_general_oracle(kind, kw):
    if kind == "graph":
        g = make_pose_graph(kw.pop("n_nodes"), seed=len(kw) + 17, **kw)
    else:
        g = make_merge_graph(kw.pop("n_key"), kw.pop("n_cams"), seed=5, **kw)
    args = [g[k] for k in KEYS] + [g["scale_col"], g["n_scale"]]
    oR, ot, os_ = orc.posegraph_solve(*args)
    for method in METHODS:
        r = dense.solve(*args, method=method)
        assert np.abs(r["newR"] - oR).max() < TOL and np.abs(r["newt"] - ot).max() < TOL, method
        assert np.all(np.abs(r["scale"] - os_) <= TOL * np.abs(os_)), method


def test_chain_batches_are_solved_chain_by_chain():
    g = make_pose_chains([37, 0, 1, 120, 5], key_every=6, seed=4, shift=0.1)
    r = dense.solve_chains(g["chain_off"], g["fixed"], g["R"], g["t"], g["eR"], g["et"])
    full = dense.solve(g["fixed"], g["R"], g["t"], g["id1"], g["id2"], g["eR_list"], g["et_list"])
    assert np.abs(r["newR"] - full["newR"]).max() < 1e-12 and np.abs(r["newt"] - full["newt"]).max() < 1e-12


def _rx(deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    return np.array([[1.0, 0, 0], [0, c, -s], [0, s, c]])


def test_projection_reports_ties_and_reflections():
    """project() on the degenerate matrices the GPU tests feed the kernels: its rotation is proper and
    as close to M as any rotation, and its signed singular values tell a unique projection from a tie."""
    cases = [(np.diag([0.5, 0.5, 0.0]), True), (np.diag([1.0, 0.0, 0.0]), False), (np.zeros((3, 3)), False),
             (np.diag([1.0, 1.0, -1.0]), False), (0.5 * np.eye(3), True),
             ((np.eye(3) + _rx(175) + np.diag([-1.0, 1, -1]) @ _rx(0)) / 3, True)]
    for M, unique in cases:
        R, sv = dense.project(M)
        assert np.abs(R.T @ R - np.eye(3)).max() < 1e-14 and np.linalg.det(R) > 0
        assert abs(np.linalg.norm(R - M) - dense.min_distance(M, sv)) < 1e-14
        assert (sv[1] + sv[2] > 1e-12) == unique, M
    R, _ = dense.project(np.diag([0.5, 0.5, 0.0]))
    assert np.abs(R - np.eye(3)).max() < 1e-15


def test_rank_deficient_systems_are_refused():
    g = make_pose_chains([6], seed=1, fixed_masks=[[0] * 6])
    for method in METHODS:
        with pytest.raises(ValueError):
            dense.solve(g["fixed"], g["R"], g["t"], g["id1"], g["id2"], g["eR_list"], g["et_list"], method=method)
