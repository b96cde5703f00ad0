"""The pose solver's covariance stage (cosl_pose_solver_set_covariance / _download_covariance): parity with the
float64 reference of tests/pose_cov_dense.py at the device's own R_opt, t_opt, a stage that changes nothing the
solve returns, cameras that do not see each other, singular cameras, the state rules, and a Monte-Carlo check that
the covariance describes the solver's actual error."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_cov_dense as cd
from coslam_b200 import synth
from coslam_b200.ctypes_defs import PoseOpt

pytestmark = pytest.mark.gpu

TAU = 10.0
VAR = 0.25
OPT_FIELDS = [f for f, _ in PoseOpt._fields_]


def _cases(seeds_npts, prev_mask=None, seed=0, W=1280, H=720):
    """(Ks, R0s, t0s, Ms, ms, prev) of synth pose cases; prev_mask[c] False gives camera c no prevErrs."""
    cs = [synth.make_pose_case(n, W, H, seed=s) for s, n in seeds_npts]
    rng = np.random.default_rng(seed)
    prev = [np.abs(rng.normal(0, 4, n)) for _, n in seeds_npts]
    prev = [p if prev_mask is None or prev_mask[c] else None for c, p in enumerate(prev)]
    return [c[0] for c in cs], [c[1] for c in cs], [c[2] for c in cs], [c[3] for c in cs], [c[4].copy() for c in cs], prev


def _beyond_tau():
    """four cameras; camera 2 has 20 points moved 60 px, so beyond tau at any pose near the solution"""
    case = _cases([(120 + c, 150) for c in range(4)], seed=5)
    case[4][2][::7, 0] += 60.0
    return case


CASES = {
    # bench.py's pose workload: 4 cameras x 192 points, no prevErrs
    "bench_4x192": _cases([(100 + c, 192) for c in range(4)], [False] * 4),
    "c13_mixed": _cases([(50 + c, 60 + 11 * c) for c in range(13)], [c % 3 != 1 for c in range(13)], seed=1),
    "beyond_tau": _beyond_tau(),
}


def _take(case, idx):
    return tuple([x[c] for c in idx] for x in case)


def _solver(api, case, armed=True):
    s = api.PoseSolver(0, len(case[3]), max(1, sum(len(a) for a in case[3])))
    if armed:
        s.set_covariance(VAR)
    return s


def _solve(s, case):
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev)
    return s.collect()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _same_solve(a, b):
    ok_a, R_a, t_a, op_a = a[:4]
    ok_b, R_b, t_b, op_b = b[:4]
    assert np.array_equal(ok_a, ok_b)
    assert np.array_equal(_bits(R_a), _bits(R_b)) and np.array_equal(_bits(t_a), _bits(t_b))
    for c in range(len(op_a)):
        for f in OPT_FIELDS:
            assert np.array(getattr(op_a[c], f)).tobytes() == np.array(getattr(op_b[c], f)).tobytes(), (c, f)


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_the_dense_reference(api, name):
    case = CASES[name]
    s = _solver(api, case)
    ok, R, t, _, dms = _solve(s, case)
    cov, err, st = s.download_covariance()
    s.close()
    assert dms > 0
    n_beyond = 0
    for c in range(len(case[3])):
        ref = cd.cov_stage(case[0][c], R[c], t[c], case[3][c], case[4][c], TAU, VAR)
        assert len(err[c]) == len(case[3][c])
        assert cd.residual_error(err[c], ref["e"]) <= 1e-9, c
        assert st[c, 1] == ref["dof"], c
        assert st[c, 0] == pytest.approx(ref["sigma2_hat"], rel=1e-10), c
        assert st[c, 3] == 1.0 and ref["valid"], c
        assert st[c, 2] == pytest.approx(ref["min_pivot"], rel=1e-6), c
        rel = np.linalg.norm(cov[c] - ref["cov"]) / np.linalg.norm(ref["cov"])
        assert rel <= 1e-9, (c, rel)
        assert np.array_equal(_bits(cov[c]), _bits(cov[c].T))
        n_beyond += int((ref["w"] == 0).sum())
    if name == "beyond_tau":
        assert n_beyond >= 20


@pytest.mark.parametrize("name", ["bench_4x192", "c13_mixed"])
def test_arming_changes_nothing(api, name):
    case = CASES[name]
    ref = api.pose_intracam_batch(*case[:5], TAU, case[5])
    armed, plain = _solver(api, case), _solver(api, case, armed=False)
    _same_solve(_solve(armed, case), ref)
    _same_solve(_solve(plain, case), ref)
    armed.close()
    plain.close()


def test_cameras_are_independent(api):
    case = CASES["c13_mixed"]
    s = _solver(api, case)
    all_res = _solve(s, case)
    all_cov = s.download_covariance()
    for c in range(len(case[3])):
        one = _solve(s, _take(case, [c]))
        cov, err, st = s.download_covariance()
        assert np.array_equal(_bits(one[1][0]), _bits(all_res[1][c])) and np.array_equal(_bits(one[2][0]),
                                                                                          _bits(all_res[2][c]))
        assert np.array_equal(_bits(cov[0]), _bits(all_cov[0][c]))
        assert np.array_equal(_bits(err[0]), _bits(all_cov[1][c]))
        assert np.array_equal(_bits(st[0]), _bits(all_cov[2][c]))
    s.close()


def test_singular_cameras(api):
    """camera 1 has 2 points, camera 2 every point beyond tau (zero prevErrs weights, then 200 px off): both get
    NaN and valid = 0; cameras 0 and 3 come out as when they are solved without them."""
    Ks, R0s, t0s, Ms, ms, prev = _cases([(140 + c, 120) for c in range(4)], seed=6)
    Ms[1], ms[1], prev[1] = Ms[1][:2], ms[1][:2], prev[1][:2]
    ms[2] = ms[2] + 200.0
    prev[2] = np.full(len(Ms[2]), 1e3)
    case = (Ks, R0s, t0s, Ms, ms, prev)
    s = _solver(api, case)
    res = _solve(s, case)
    cov, err, st = s.download_covariance()
    for c in (1, 2):
        assert np.isnan(cov[c]).all() and st[c, 3] == 0.0, c
        ref = cd.cov_stage(Ks[c], res[1][c], res[2][c], Ms[c], ms[c], TAU, VAR)
        assert not ref["valid"] and st[c, 1] == ref["dof"] and np.isnan(st[c, 0])
        assert cd.residual_error(err[c], ref["e"]) <= 1e-9
    assert st[1, 2] < 1e-12
    assert st[2, 1] == -6 and st[2, 2] == 0.0 and (err[2] > TAU).all()
    pair = _solve(s, _take(case, [0, 3]))
    cov2, err2, st2 = s.download_covariance()
    for i, c in enumerate((0, 3)):
        assert st[c, 3] == 1.0
        assert np.array_equal(_bits(pair[1][i]), _bits(res[1][c])) and np.array_equal(_bits(pair[2][i]),
                                                                                      _bits(res[2][c]))
        assert np.array_equal(_bits(cov2[i]), _bits(cov[c])) and np.array_equal(_bits(st2[i]), _bits(st[c]))
        assert np.array_equal(_bits(err2[i]), _bits(err[c]))
    s.close()


def test_state_rules(api):
    case = CASES["bench_4x192"]
    L = api.LIB
    s = _solver(api, case, armed=False)
    with pytest.raises(api.CoslError, match="error -6"):  # no armed solve yet
        s.download_covariance()
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(api.CoslError, match="error -1"):
            s.set_covariance(bad)
    _solve(s, case)
    with pytest.raises(api.CoslError, match="error -6"):  # an unarmed solve
        s.download_covariance()
    s.set_covariance(VAR)
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev)
    with pytest.raises(api.CoslError, match="error -6"):  # in flight
        s.download_covariance()
    with pytest.raises(api.CoslError, match="error -6"):
        s.set_covariance(0.0)
    s.collect()
    first = s.download_covariance()
    out = np.empty((4, 4))
    assert L.cosl_pose_solver_download_covariance(s.h, None, None, out.ctypes.data) == 0  # cov and err nullable
    assert np.array_equal(_bits(out), _bits(first[2]))
    assert L.cosl_pose_solver_download_covariance(s.h, None, None, None) == -1
    s.set_covariance(0.0)  # disarmed: the last armed result stays until the next submit
    assert np.array_equal(_bits(s.download_covariance()[0]), _bits(first[0]))
    _solve(s, case)
    with pytest.raises(api.CoslError, match="error -6"):
        s.download_covariance()
    s.set_covariance(2 * VAR)  # re-armed: the buffers of the first arming, the new variance
    _solve(s, case)
    again = s.download_covariance()
    assert np.allclose(again[0], 2 * first[0], rtol=1e-15, atol=0)
    assert np.array_equal(_bits(again[2]), _bits(first[2]))
    s.close()


def test_monte_carlo_nees(api):
    """200 solves of one camera, 192 points, 0.5 px noise and no outliers: the mean NEES of
    (log(R_true^T R_opt), t_opt - t_true) under cov is chi-square with 6 dof, mean 6 (std of the mean 0.245)."""
    s = api.PoseSolver(0, 1, 192)
    s.set_covariance(VAR)
    nees = []
    for k in range(200):
        K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(192, seed=5000 + k, noise_px=0.5, outlier_frac=0.0)
        s.submit([K], [R0], [t0], [Ms], [ms], TAU)
        ok, R, t, _, _ = s.collect()
        cov, _, st = s.download_covariance()
        assert ok[0] and st[0, 3] == 1.0
        x = np.concatenate([Rotation.from_matrix(Rt.T @ R[0]).as_rotvec(), t[0] - tt])
        nees.append(float(x @ np.linalg.solve(cov[0], x)))
    s.close()
    m = float(np.mean(nees))
    assert 5.2 <= m <= 6.8, m
