"""The pose solver with Gaussian pose priors (cosl_pose_solver_submit_prior, DESIGN.md 5.3): no prior, or a camera
without one, is the plain and the covariance submit bit for bit; random priors match the float64 restatement of
tests/pose_prior_dense.py in the solve and in the armed stage, with and without measurement covariances; cameras with
no, one or two points are regular with a prior; a loose prior is the solve without one; cameras stay independent; bad
priors are refused with their camera; and a Monte-Carlo check that chains each frame's posterior into the next
frame's prior."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_cov_dense as cd
import pose_dense as pd
import pose_prior_dense as ppd
from test_gpu_pose_covariance import CASES, OPT_FIELDS, TAU, VAR, _bits, _same_solve
from test_gpu_pose_obscov import ERR_KEYS, ERR_REL, _covx, _same_stage

pytestmark = pytest.mark.gpu


def _solver(api, case, pixel_var=1.0):
    s = api.PoseSolver(0, len(case[3]), max(1, sum(len(a) for a in case[3])))
    s.set_covariance(pixel_var)
    return s


def _run(s, case, covx=None, prior=None):
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, covx=covx, prior=prior)
    return s.collect(), s.download_covariance()


def _priors(case, seed, max_deg=30.0, cond=1e4, scale=1e-3, every=1):
    """A random prior on every `every`-th camera (None elsewhere), its mean up to max_deg from the start pose."""
    rng = np.random.default_rng(seed)
    return [ppd.random_prior(R0, t0, rng, max_deg, cond, scale) if c % every == 0 else None
            for c, (R0, t0) in enumerate(zip(case[1], case[2]))]


def _drawn_priors(case, seed, max_deg=30.0, cond=1e4, scale=0.04):
    """A prior on every camera that its start pose is a draw of: rotations up to max_deg from the mean, largest
    standard deviation sqrt(scale) = 0.2 rad or units.  A mean far outside P would pull against 192 points with a
    stiff prior, and the pose would then follow summation-order noise far more than the solve without a prior does."""
    rng = np.random.default_rng(seed)
    return [ppd.drawn_prior(R0, t0, rng, max_deg, cond, scale) for R0, t0 in zip(case[1], case[2])]


def _same_camera(a, b, c):
    """collect and stage outputs of camera c bit-identical"""
    assert a[0][0][c] == b[0][0][c], c
    assert np.array_equal(_bits(a[0][1][c]), _bits(b[0][1][c])) and np.array_equal(_bits(a[0][2][c]),
                                                                                  _bits(b[0][2][c])), c
    for f in OPT_FIELDS:
        assert np.array(getattr(a[0][3][c], f)).tobytes() == np.array(getattr(b[0][3][c], f)).tobytes(), (c, f)
    assert np.array_equal(_bits(a[1][0][c]), _bits(b[1][0][c])) and np.array_equal(_bits(a[1][2][c]),
                                                                                  _bits(b[1][2][c])), c
    assert np.array_equal(_bits(a[1][1][c]), _bits(b[1][1][c])), c


@pytest.mark.parametrize("with_covx", [False, True])
@pytest.mark.parametrize("name", sorted(CASES))
def test_cameras_without_a_prior_are_bit_identical(api, name, with_covx):
    case = CASES[name]
    C = len(case[3])
    covx = _covx(case, 21) if with_covx else None
    s = _solver(api, case)
    plain = _run(s, case, covx)
    got = _run(s, case, covx, [None] * C)
    _same_solve(got[0], plain[0])
    _same_stage(got[1], plain[1])
    mixed = _priors(case, 22, every=2)
    got = _run(s, case, covx, mixed)
    s.close()
    for c in range(C):
        if mixed[c] is None:
            _same_camera(got, plain, c)
        else:
            assert not np.array_equal(_bits(got[0][2][c]), _bits(plain[0][2][c])), c


def _check_camera(c, ok, R, t, o, case, covx, prior):
    K, R0, t0, Ms, ms, prev = (x[c] for x in case)
    ok_d, R_d, t_d, f = ppd.estimate(K, R0, t0, Ms, ms, TAU, prev, pd.DEFAULT_OPT, covx, prior)
    margin = min((m for _, m in ppd.margins(K, R0, t0, Ms, ms, TAU, prev, pd.DEFAULT_OPT, covx, prior)),
                 default=np.inf)
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
    return margin


def _check_stage(c, R, t, cov, err, st, case, covx, prior, pixel_var=1.0):
    ref = ppd.cov_stage(case[0][c], R, t, case[3][c], case[4][c], TAU, pixel_var, covx, prior)
    assert cd.residual_error(err, ref["e"]) <= 1e-9, c
    assert st[1] == ref["dof"] and st[3] == 1.0 and ref["valid"], c
    if ref["dof"] > 0:
        assert st[0] == pytest.approx(ref["sigma2_hat"], rel=1e-9), c
    assert st[2] == pytest.approx(ref["min_pivot"], rel=1e-6), c
    rel = np.linalg.norm(cov - ref["cov"]) / np.linalg.norm(ref["cov"])
    assert rel <= 1e-9, (c, rel)


@pytest.mark.parametrize("with_covx", [False, True])
@pytest.mark.parametrize("name", sorted(CASES))
def test_random_priors_match_the_dense_restatement(api, name, with_covx):
    case = CASES[name]
    C = len(case[3])
    covx = _covx(case, 31) if with_covx else [None] * C
    prior = _drawn_priors(case, 32)
    s = _solver(api, case)
    (ok, R, t, opts, dms), (cov, err, st) = _run(s, case, covx if with_covx else None, prior)
    s.close()
    assert dms > 0
    worst = np.inf
    for c in range(C):
        worst = min(worst, _check_camera(c, ok[c], R[c], t[c], opts[c], case, covx[c], prior[c]))
        _check_stage(c, R[c], t[c], cov[c], err[c], st[c], case, covx[c], prior[c])
    print(f"{name}: smallest decision margin {worst:.1e}")


def _few_points_case(npts, seed=40):
    """four cameras of bench_4x192 cut to npts points each"""
    Ks, R0s, t0s, Ms, ms, _ = CASES["bench_4x192"]
    rng = np.random.default_rng(seed)
    idx = [np.sort(rng.choice(len(m), npts, replace=False)) for m in Ms]
    return (Ks, R0s, t0s, [m[i] for m, i in zip(Ms, idx)], [m[i] for m, i in zip(ms, idx)], [None] * len(Ms))


def test_unobserved_cameras_go_to_their_mean_with_cov_p(api):
    case = _few_points_case(0)
    prior = _priors(case, 41, max_deg=25.0, cond=1e3, scale=1e-3)
    s = api.PoseSolver(0, 4, 1)
    s.set_covariance(VAR)
    (ok, R, t, opts, _), (cov, err, st) = _run(s, case, None, prior)
    s.close()
    for c, (Rp, tp, P) in enumerate(prior):
        assert ok[c], c
        assert np.abs(R[c] - Rp).max() <= 1e-12 and np.abs(t[c] - tp).max() <= 1e-12, c
        assert np.linalg.norm(cov[c] - VAR * P) <= 1e-9 * np.linalg.norm(VAR * P), c
        assert st[c, 3] == 1.0 and st[c, 1] == 0 and len(err[c]) == 0, c


@pytest.mark.parametrize("npts", [1, 2])
def test_one_or_two_points_are_regular_with_a_prior(api, npts):
    case = _few_points_case(npts)
    prior = _priors(case, 42, max_deg=2.0, cond=1e3, scale=1e-3)
    s = _solver(api, case)
    plain = _run(s, case)
    got = _run(s, case, None, prior)
    s.close()
    assert (plain[1][2][:, 3] == 0.0).all()
    for c in range(4):
        assert got[1][2][c, 3] == 1.0 and np.isfinite(got[1][0][c]).all(), c
        _check_camera(c, got[0][0][c], got[0][1][c], got[0][2][c], got[0][3][c], case, None, prior[c])
        _check_stage(c, got[0][1][c], got[0][2][c], got[1][0][c], got[1][1][c], got[1][2][c], case, None, prior[c])


@pytest.mark.parametrize("name", sorted(CASES))
def test_loose_prior_is_the_plain_submit(api, name):
    case = CASES[name]
    C = len(case[3])
    prior = [(Rp, tp, 1e12 * np.eye(6)) for Rp, tp, _ in _priors(case, 51, max_deg=10.0)]
    s = _solver(api, case)
    (ok0, R0, t0, o0, _), _ = _run(s, case)
    (ok, R, t, o, _), _ = _run(s, case, None, prior)
    s.close()
    assert np.array_equal(ok, ok0)
    assert np.abs(R - R0).max() <= 1e-8 and np.abs(t - t0).max() <= 1e-8
    for c in range(C):
        for k in ERR_KEYS:
            a, b = getattr(o[c], k), getattr(o0[c], k)
            assert a == b or abs(a - b) <= ERR_REL * abs(b) + 1e-12, (c, k, a, b)


def test_cameras_are_independent(api):
    case = CASES["c13_mixed"]
    covx = _covx(case, 61)
    prior = _priors(case, 62)
    s = _solver(api, case)
    a = _run(s, case, covx, prior)
    prior2 = list(prior)
    prior2[0] = _priors(case, 63)[0]
    b = _run(s, case, covx, prior2)
    s.close()
    assert not np.array_equal(_bits(a[0][1][0]), _bits(b[0][1][0]))
    for c in range(1, len(case[3])):
        _same_camera(a, b, c)


def _bad(kind, rec):
    R, t, P = (np.array(x, np.float64) for x in rec)
    if kind == "not_rotation":
        R[0, 0] += 1e-6
    elif kind == "reflection":
        R = -R
    elif kind == "nan":
        t[1] = np.nan
    elif kind == "asymmetric":
        P[0, 4] += 1e-9 * np.abs(np.diag(P)).max()
    elif kind == "indefinite":
        w, V = np.linalg.eigh(P)
        w[2] = -w[2]
        P = (V * w) @ V.T
    return R, t, P


BAD = {"not_rotation": "not a rotation", "reflection": "not a rotation", "nan": "not finite",
       "asymmetric": "not symmetric", "indefinite": "not positive definite"}


@pytest.mark.parametrize("kind", sorted(BAD))
def test_bad_priors_are_refused(api, kind):
    case = CASES["c13_mixed"]
    prior = _priors(case, 71)
    good = prior[2]
    prior[2] = _bad(kind, good)
    s = _solver(api, case)
    Ks, R0s, t0s, Ms, ms, prev = case
    with pytest.raises(api.CoslError, match=rf"error -1: cosl_pose_solver_submit_prior: .*camera 2.*{BAD[kind]}"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, prior=prior)
    prior[2] = good
    ok = _run(s, case, None, prior)[0][0]
    assert ok.any()
    s.close()


def test_submit_prior_while_in_flight(api):
    case = CASES["bench_4x192"]
    s = _solver(api, case)
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, prior=_priors(case, 81))
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, prior=_priors(case, 82))
    s.collect()
    s.close()


# ---------------------------------------------------------------- Monte-Carlo filter check
W_IMG, H_IMG = 640, 480
K_MC = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
Q = np.diag([1e-4] * 3 + [4e-4] * 3)     # the true step: 0.01 rad and 0.02 units per axis
P0 = np.diag([4e-4] * 3 + [2.5e-3] * 3)  # the first frame's prior: 0.02 rad and 0.05 units per axis
TAU_MC = 1e3                             # far beyond 1 px noise: every weight is 1 to 1e-6


def _err(R, t, Rt, tt):
    """(Log(R^T R_true), t_true - t): the truth in the estimate's chart R_true = R exp([e]x)"""
    return np.concatenate([Rotation.from_matrix(R.T @ Rt).as_rotvec(), tt - t])


def _frame_points(Rt, tt, rng, n=6):
    """n world points in front of the true camera (pixels uniform over the image, depth 4 to 8) and their
    observations with 1 px noise"""
    uv = rng.uniform([0.0, 0.0], [W_IMG, H_IMG], (n, 2))
    z = rng.uniform(4.0, 8.0, n)
    Xc = np.linalg.solve(K_MC, np.column_stack([uv, np.ones(n)]).T).T * z[:, None]
    M = (Xc - tt) @ Rt  # R^T (Xc - t), row-wise
    return M, uv + rng.normal(0.0, 1.0, (n, 2))


def test_monte_carlo_filter_chain(api):
    """20 random-walk cameras, 10 frames each, 6 points per frame at 1 px: each frame's prior is the previous frame's
    posterior (mean and download_covariance block) plus the true step covariance Q; the first frame's prior is the
    true pose displaced by a draw from P0, with covariance P0.  The posterior NEES is chi-square with 6 dof, mean 6;
    the chain correlates consecutive frames of one camera, so the mean of the 200 is less tight than 200 independent
    draws (std 0.245).  On the same draws, the solve without a prior has larger mean errors."""
    ncam, nfr = 20, 10
    rng = np.random.default_rng(9100)
    Rt = [Rotation.from_rotvec(rng.normal(0, 0.1, 3)).as_matrix() for _ in range(ncam)]
    tt = [rng.normal(0, 0.5, 3) for _ in range(ncam)]
    mean = []
    for c in range(ncam):
        e = rng.multivariate_normal(np.zeros(6), P0)
        mean.append(ppd.apply(Rt[c], tt[c], -e))
    Pk = [P0] * ncam
    s = api.PoseSolver(0, ncam, ncam * 6)
    s.set_covariance(1.0)
    nees, err_p, err_u = [], [], []
    for k in range(nfr):
        if k:  # the true step, in the chart
            for c in range(ncam):
                Rt[c], tt[c] = ppd.apply(Rt[c], tt[c], rng.multivariate_normal(np.zeros(6), Q))
        pts = [_frame_points(Rt[c], tt[c], rng) for c in range(ncam)]
        args = ([K_MC] * ncam, [m[0] for m in mean], [m[1] for m in mean], [p[0] for p in pts], [p[1] for p in pts])
        s.submit(*args, TAU_MC, prior=[(mean[c][0], mean[c][1], Pk[c]) for c in range(ncam)])
        ok, R, t, _, _ = s.collect()
        cov, _, st = s.download_covariance()
        assert ok.all() and (st[:, 3] == 1.0).all()
        s.submit(*args, TAU_MC)
        ok_u, R_u, t_u, _, _ = s.collect()
        assert ok_u.all()
        for c in range(ncam):
            x = _err(R[c], t[c], Rt[c], tt[c])
            nees.append(float(x @ np.linalg.solve(cov[c], x)))
            err_p.append(x)
            err_u.append(_err(R_u[c], t_u[c], Rt[c], tt[c]))
        mean = [(R[c], t[c]) for c in range(ncam)]
        Pk = [0.5 * (cov[c] + cov[c].T) + Q for c in range(ncam)]
    s.close()
    m = float(np.mean(nees))
    ep, eu = np.array(err_p), np.array(err_u)
    rot_p, rot_u = np.linalg.norm(ep[:, :3], axis=1).mean(), np.linalg.norm(eu[:, :3], axis=1).mean()
    tr_p, tr_u = np.linalg.norm(ep[:, 3:], axis=1).mean(), np.linalg.norm(eu[:, 3:], axis=1).mean()
    print(f"mean NEES {m:.2f} over {len(nees)}; mean rotation error {rot_p:.2e} vs {rot_u:.2e} rad without a prior, "
          f"translation {tr_p:.2e} vs {tr_u:.2e}")
    assert 5.2 <= m <= 6.8, m
    assert rot_p < rot_u and tr_p < tr_u
