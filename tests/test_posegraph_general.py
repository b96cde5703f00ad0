"""General pose graphs with shared unknown scales (the camera-group merge, SURVEY.md 8f-2), on the CPU:
pins the oracle entry orc_posegraph_solve (oracle/posegraph_general_oracle.cpp) to the UNMODIFIED
reference (computeNewCameraRotations + computeNewCameraTranslations4 of slam/SL_GlobalPoseEstimation.cpp)
through tests/golden/posegraph_merge_ref.npz (made by tests/golden/make_posegraph_merge_golden.py) and live where
oracle/_ref/libposegraph_merge_ref.so is built; known answers; the argument checks of cosl_posegraph_solve
(they run before any device work); and the shim header with COSL_POSEGRAPH_GENERAL against a mock ABI
and the merge's call sites.  Tolerance 1e-9 (QR against normal equations, O(1) values)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from coslam_b200.synth import make_merge_graph, make_pose_graph, scale_columns
from oracle import orc_pg_general as orc
from oracle import ref_pg_general as ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TOL = 1e-9
KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et")


def _args(g):
    return [g[k] for k in KEYS] + [g["scale_col"], g["n_scale"]]


def _check_against_reference(oR, ot, os_, rR, rt, rs, scale_id):
    col, _ = scale_columns(scale_id)
    unc = scale_id >= 0
    assert np.abs(oR - rR).max() < TOL and np.abs(ot - rt).max() < TOL
    assert np.all(np.abs(os_[col[unc]] - rs[unc]) <= TOL * np.abs(rs[unc]))


def test_oracle_matches_reference_golden_vectors():
    z = np.load(os.path.join(HERE, "golden", "posegraph_merge_ref.npz"))
    for i in range(int(z["n_cases"])):
        c = {k: z[f"c{i}_{k}"] for k in KEYS + ("scale_id", "newR", "newt", "s")}
        col, ns = scale_columns(c["scale_id"])
        out = orc.posegraph_solve(*(c[k] for k in KEYS), col, ns)
        _check_against_reference(*out, c["newR"], c["newt"], c["s"], c["scale_id"])


@pytest.mark.skipif(not ref.available(), reason="oracle/_ref/libposegraph_merge_ref.so is not built")
@pytest.mark.parametrize("seed", range(10))
def test_oracle_matches_compiled_reference_live(seed):
    g = make_merge_graph(3 + seed, 2 + seed % 5, seed=100 + seed, n_constraints=1 + seed % 3,
                         n_scale_ids=1 + seed % 2, noise=0.01 * (seed % 2))
    out = orc.posegraph_solve(*_args(g))
    _check_against_reference(*out, *ref.posegraph_merge(*(g[k] for k in KEYS), g["scale_id"]), g["scale_id"])


def test_consistent_measurements_return_the_input_and_the_true_scale():
    g = make_merge_graph(12, 4, seed=7, n_constraints=3, n_scale_ids=2)
    nR, nt, s = orc.posegraph_solve(*_args(g))
    assert np.abs(nR - g["R"]).max() < 1e-10 and np.abs(nt - g["t"]).max() < 1e-10
    assert np.abs(s - g["true_scale"]).max() < 1e-10


def test_fixed_nodes_are_copied_and_rotations_are_proper():
    g = make_merge_graph(10, 5, seed=9, n_constraints=2, noise=0.03)
    nR, nt, _ = orc.posegraph_solve(*_args(g))
    fx = g["fixed"].astype(bool)
    assert np.array_equal(nR[fx], g["R"][fx]) and np.array_equal(nt[fx], g["t"][fx])
    assert np.abs(np.einsum("nij,nkj->nik", nR, nR) - np.eye(3)).max() < 1e-12
    assert np.all(np.linalg.det(nR) > 0.999999)


def _abi_error(api, g, **over):
    a = dict(zip(KEYS + ("scale_col", "n_scale"), _args(g)))
    a.update(over)
    with pytest.raises(api.CoslError) as e:
        api.posegraph_solve(*(a[k] for k in KEYS + ("scale_col", "n_scale")))
    return str(e.value)


def test_invalid_arguments_are_reported_before_any_device_work(api):
    g = make_pose_graph(12, seed=3, n_scale=1, uncertain=1)
    id1 = g["id1"].copy()
    id1[2] = 12
    assert "error -1" in _abi_error(api, g, id1=id1) and "edge 2" in _abi_error(api, g, id1=id1)
    id2 = g["id2"].copy()
    id2[0] = g["id1"][0]
    assert "self-loop" in _abi_error(api, g, id2=id2)
    sc = g["scale_col"].copy()
    sc[0] = 1
    assert "error -1" in _abi_error(api, g, scale_col=sc)
    assert "scale column 1 gets no row" in _abi_error(api, g, n_scale=2)
    fx = np.zeros_like(g["fixed"])
    assert "node 0 lies in a connected component without a fixed node" in _abi_error(api, g, fixed=fx)
    two = make_pose_graph(20, seed=4, components=2)
    fx = two["fixed"].copy()
    fx[10] = 0
    assert "node 10 lies" in _abi_error(api, two, fixed=fx)
    # an uncertain edge between two fixed nodes gives no row: its column is empty
    fx = g["fixed"].copy()
    unc = int(np.nonzero(g["scale_col"] >= 0)[0][0])
    fx[g["id1"][unc]] = fx[g["id2"][unc]] = 1
    assert "scale column 0 gets no row" in _abi_error(api, g, fixed=fx)


def test_without_a_device_the_call_returns_cosl_e_cuda(api):
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    g = make_merge_graph(4, 2, seed=1)
    assert "error -2" in _abi_error(api, g)


def test_shim_with_the_definition_against_a_mock_abi(tmp_path):
    """computeNewCameraTranslations4's flattening and scale-id -> column map, the write-back of
    CamPoseEdge::s, one ABI call per rotations + translations, chains on the chain entry, refusals."""
    exe = os.path.join(str(tmp_path), "mock_posegraph_general")
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-DCOSL_POSEGRAPH_GENERAL",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "coslam_b200", "shim"),
                           os.path.join(HERE, "stubs", "mock_posegraph_general.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "MOCK_POSEGRAPH_GENERAL_OK" in out.stdout, out.stdout + out.stderr


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_merge_probe_compiles_against_the_shim_header(tmp_path):
    """MergeCameraGroup's graph construction and both recompute steps compile against the shim header
    with COSL_POSEGRAPH_GENERAL in place of the reference's slam/SL_GlobalPoseEstimation.h."""
    (tmp_path / "slam").mkdir()
    shim = os.path.join(ROOT, "coslam_b200", "shim", "SL_GlobalPoseEstimation.h")
    (tmp_path / "slam" / "SL_GlobalPoseEstimation.h").write_text(f'#include "{shim}"\n')
    cmd = ["g++", "-std=c++11", "-fsyntax-only", "-DCOSL_POSEGRAPH_GENERAL", "-I", os.path.join(HERE, "stubs"),
           "-I", os.path.join(ROOT, "include"), "-I", str(tmp_path),
           os.path.join(HERE, "stubs", "probe_posegraph_merge.cpp")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-4000:]
