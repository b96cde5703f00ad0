"""The pose solver with 2x2 measurement covariances (cosl_pose_solver_submit_cov, DESIGN.md 5.2): identity
covariances are the plain submit bit for bit, Sigma = 4I quarters the first cost exactly, anisotropic covariances
match the float64 restatement of tests/pose_obscov_dense.py in the solve and in the armed stage, cameras stay
independent, bad covariances are refused with their camera and point, and a Monte-Carlo check that the whitened
covariance describes the solver's error and that the whitened solve beats the unweighted one."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_cov_dense as cd
import pose_obscov_dense as od
from coslam_b200 import synth
from coslam_b200.ctypes_defs import PoseOpt
from test_gpu_pose_covariance import CASES, OPT_FIELDS, TAU, _bits, _same_solve

pytestmark = pytest.mark.gpu

ERR_KEYS = ("err0", "err", "errRW")
# err0, err and errRW are whitened costs at poses that agree with the restatement only to summation-order noise
# (~1e-10 here).  Factors of up to 1 / 0.15 px^-1 make the cost of a later round up to ~7 times more sensitive to
# the pose than the unweighted one (1e-9 relative, tests/test_gpu_pose_edges.py): on an H100 they moved by up to
# 7.6e-9 relative (beyond_tau, bench_4x192)
ERR_REL = 3e-8


def _covx(case, seed, lo=0.15, hi=1.5):
    rng = np.random.default_rng(seed)
    return [od.random_covx(len(m), rng, lo, hi)[0] for m in case[3]]


def _solver(api, case, pixel_var=1.0):
    s = api.PoseSolver(0, len(case[3]), max(1, sum(len(a) for a in case[3])))
    s.set_covariance(pixel_var)
    return s


def _run(s, case, covx=None, opts=None):
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, opts=opts, covx=covx)
    res = s.collect()
    return res, s.download_covariance()


def _same_stage(a, b):
    assert np.array_equal(_bits(a[0]), _bits(b[0]))
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(a[1], b[1]))
    assert np.array_equal(_bits(a[2]), _bits(b[2]))


def _opts(n, **kw):
    opts = (PoseOpt * n)(*[PoseOpt.defaults() for _ in range(n)])
    for o in opts:
        for k, v in kw.items():
            setattr(o, k, v)
    return opts


@pytest.mark.parametrize("name", sorted(CASES))
def test_identity_covariances_are_the_plain_submit(api, name):
    case = CASES[name]
    C = len(case[3])
    s = _solver(api, case)
    plain = _run(s, case)
    eye = [np.tile(np.eye(2), (len(m), 1, 1)) for m in case[3]]
    half = [e if c % 2 else None for c, e in enumerate(eye)]
    for covx in ([None] * C, eye, half):
        got = _run(s, case, covx)
        _same_solve(got[0], plain[0])
        _same_stage(got[1], plain[1])
    # covx == NULL through cosl_pose_solver_submit_cov
    args, opts, _keep = api._pose_batch_args(*case[:5], TAU, case[5], None)
    api._ck(api.LIB.cosl_pose_solver_submit_cov(s.h, *args[:7], None, *args[7:], opts))
    s._opts = opts
    _same_solve(s.collect(), plain[0])
    _same_stage(s.download_covariance(), plain[1])
    s.close()


@pytest.mark.parametrize("name", ["bench_4x192", "c13_mixed"])
def test_four_identity_quarters_the_first_cost(api, name):
    """One re-weighting round: err0 is the cost at R0, t0 under the prevErrs weights, the same for both solves."""
    case = CASES[name]
    C = len(case[3])
    s = _solver(api, case)
    one = _run(s, case, opts=_opts(C, maxIterRW=1))[0]
    four = _run(s, case, [4 * np.tile(np.eye(2), (len(m), 1, 1)) for m in case[3]], _opts(C, maxIterRW=1))[0]
    for c in range(C):
        assert four[3][c].err0 == one[3][c].err0 / 4, c
    s.close()


def _check_camera(c, ok, R, t, o, case, covx):
    K, R0, t0, Ms, ms, prev = (x[c] for x in case)
    ok_d, R_d, t_d, f = od.estimate(K, R0, t0, Ms, ms, TAU, prev, covx=covx)
    margin = min((m for _, m in od.margins(K, R0, t0, Ms, ms, TAU, prev, covx=covx)), default=np.inf)
    assert ok == ok_d and o.retTypeLM == f["retTypeLM"], c
    dR, dt = np.abs(R - R_d).max(), np.abs(t - t_d).max()
    assert dR <= 1e-8 and dt <= 1e-8, (c, dR, dt)
    if margin < 1e-7:  # a decision at the rounding floor: the path may differ, the pose may not
        return margin
    assert (o.npts, o.nIterLM, o.nIterRW) == (f["npts"], f["nIterLM"], f["nIterRW"]), c
    assert o.lambda_ == f["lambda_"] and o.lambda0 == f["lambda0"], c
    for k in ERR_KEYS:
        a, b = getattr(o, k), f[k]
        assert a == b or abs(a - b) <= ERR_REL * abs(b) + 1e-12, (c, k, a, b)
    print(f"camera {c}: |pose - dense| {max(dR, dt):.1e}, costs "
          + " ".join(f"{k} {abs(getattr(o, k) - f[k]) / abs(f[k]):.1e}" for k in ERR_KEYS))
    return margin


@pytest.mark.parametrize("name", sorted(CASES))
def test_anisotropic_covariances_match_the_dense_restatement(api, name):
    case = CASES[name]
    covx = _covx(case, 11)
    s = _solver(api, case)
    (ok, R, t, opts, dms), (cov, err, st) = _run(s, case, covx)
    s.close()
    assert dms > 0
    worst = np.inf
    for c in range(len(case[3])):
        worst = min(worst, _check_camera(c, ok[c], R[c], t[c], opts[c], case, covx[c]))
        ref = od.cov_stage(case[0][c], R[c], t[c], case[3][c], case[4][c], TAU, 1.0, covx[c])
        assert cd.residual_error(err[c], ref["e"]) <= 1e-9, c
        assert st[c, 1] == ref["dof"] and st[c, 3] == 1.0 and ref["valid"], c
        assert st[c, 0] == pytest.approx(ref["sigma2_hat"], rel=1e-10), c
        assert st[c, 2] == pytest.approx(ref["min_pivot"], rel=1e-6), c
        rel = np.linalg.norm(cov[c] - ref["cov"]) / np.linalg.norm(ref["cov"])
        assert rel <= 1e-9, (c, rel)
        assert np.array_equal(_bits(cov[c]), _bits(cov[c].T))
    print(f"{name}: smallest decision margin {worst:.1e}")


def test_cameras_are_independent(api):
    case = CASES["c13_mixed"]
    covx = _covx(case, 12)
    s = _solver(api, case)
    a = _run(s, case, covx)
    covx2 = list(covx)
    covx2[0] = _covx(case, 13)[0]
    b = _run(s, case, covx2)
    s.close()
    assert not np.array_equal(_bits(a[0][1][0]), _bits(b[0][1][0]))
    for c in range(1, len(case[3])):
        assert a[0][0][c] == b[0][0][c]
        assert np.array_equal(_bits(a[0][1][c]), _bits(b[0][1][c])) and np.array_equal(_bits(a[0][2][c]),
                                                                                      _bits(b[0][2][c])), c
        for f in OPT_FIELDS:
            assert np.array(getattr(a[0][3][c], f)).tobytes() == np.array(getattr(b[0][3][c], f)).tobytes(), (c, f)
        assert np.array_equal(_bits(a[1][0][c]), _bits(b[1][0][c])) and np.array_equal(_bits(a[1][2][c]),
                                                                                      _bits(b[1][2][c])), c
        assert np.array_equal(_bits(a[1][1][c]), _bits(b[1][1][c])), c


BAD = {
    "nan": [np.nan, 0.0, 0.0, 1.0],
    "asymmetric": [1.0, 0.2, 0.2 + 1e-16, 1.0],
    "zero": [0.0, 0.0, 0.0, 0.0],
    "indefinite": [1.0, 2.0, 2.0, 1.0],
}


@pytest.mark.parametrize("bad", sorted(BAD))
def test_bad_covariances_are_refused(api, bad):
    case = CASES["c13_mixed"]
    covx = _covx(case, 14)
    covx[2] = covx[2].reshape(-1, 4).copy()
    covx[2][5] = BAD[bad]
    s = _solver(api, case)
    Ks, R0s, t0s, Ms, ms, prev = case
    with pytest.raises(api.CoslError, match=r"error -1: cosl_pose_solver_submit_cov: .*camera 2 point 5"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, covx=covx)
    covx[2][5] = [1.0, 0.0, 0.0, 1.0]
    ok = _run(s, case, covx)[0][0]
    assert ok.any()
    s.close()


def test_submit_cov_while_in_flight(api):
    case = CASES["bench_4x192"]
    s = _solver(api, case)
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, covx=_covx(case, 15))
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, covx=_covx(case, 16))
    s.collect()
    s.close()


def test_monte_carlo_nees_and_pose_error(api):
    """200 solves of one camera, 192 points, no outliers, noise drawn from covariances with standard deviations of
    0.15 to 1.5 px along random axes: the mean NEES of (log(R_true^T R_opt), t_opt - t_true) under the whitened
    covariance is chi-square with 6 dof, mean 6 (std of the mean 0.245), and on the same draws the whitened solve's
    mean pose error is below the unweighted solve's."""
    s = api.PoseSolver(0, 1, 192)
    s.set_covariance(1.0)
    nees, err_w, err_u = [], [], []
    for k in range(200):
        K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(192, seed=7000 + k, noise_px=0.0, outlier_frac=0.0)
        rng = np.random.default_rng(7000 + k)
        covx, S = od.random_covx(len(Ms), rng)
        ms = ms + od.draw_noise(S, rng)
        s.submit([K], [R0], [t0], [Ms], [ms], TAU, covx=[covx])
        ok, R, t, _, _ = s.collect()
        cov, _, st = s.download_covariance()
        assert ok[0] and st[0, 3] == 1.0
        x = np.concatenate([Rotation.from_matrix(Rt.T @ R[0]).as_rotvec(), t[0] - tt])
        nees.append(float(x @ np.linalg.solve(cov[0], x)))
        err_w.append(x)
        s.submit([K], [R0], [t0], [Ms], [ms], TAU)
        ok, R, t, _, _ = s.collect()
        assert ok[0]
        err_u.append(np.concatenate([Rotation.from_matrix(Rt.T @ R[0]).as_rotvec(), t[0] - tt]))
    s.close()
    m = float(np.mean(nees))
    ew, eu = np.array(err_w), np.array(err_u)
    rot_w, rot_u = np.linalg.norm(ew[:, :3], axis=1).mean(), np.linalg.norm(eu[:, :3], axis=1).mean()
    tr_w, tr_u = np.linalg.norm(ew[:, 3:], axis=1).mean(), np.linalg.norm(eu[:, 3:], axis=1).mean()
    print(f"mean NEES {m:.2f}; mean rotation error {rot_w:.2e} vs {rot_u:.2e} rad, translation {tr_w:.2e} vs "
          f"{tr_u:.2e}")
    assert 5.2 <= m <= 6.8, m
    assert rot_w < rot_u and tr_w < tr_u
