"""The pose-prior references of tests/pose_prior_dense.py without a GPU, before any GPU test trusts them: the prior
Jacobian against central differences up to 179 degrees, Log exact near pi, P = 1e12 I reproduces the solve without a
prior, the solve lands on the minimiser scipy.optimize.least_squares finds for the augmented residuals and the stage
on its covariance, an unobserved camera goes to its mean with cov = P, and the BA's camera covariance converts to the
pose solver's chart as diag(R^T, I) Sigma diag(R, I)."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares

import ba_cov_dense as bcd
import pose_dense as pd
import pose_obscov_dense as od
import pose_prior_dense as ppd
from coslam_b200 import synth
from coslam_b200.problem import BAProblem

TAU = 10.0


def _unit(rng):
    a = rng.normal(size=3)
    return a / np.linalg.norm(a)


@pytest.mark.parametrize("deg", [0.0, 1e-6, 0.01, 1.0, 30.0, 90.0, 119.0, 121.0, 150.0, 175.0, 179.0])
def test_prior_jacobian_matches_central_differences(deg):
    """d r / d(dw, dt) for R' = R exp([dw]x), t' = t + dt, at a pose deg degrees from the prior mean."""
    rng = np.random.default_rng(int(deg * 100) + 1)
    Rp = pd.exp_map(rng.normal(size=3))
    tp = rng.normal(size=3)
    R = Rp @ pd.exp_map(math.radians(deg) * _unit(rng))
    t = tp + rng.normal(size=3)
    rec = ppd.prior_record(Rp, tp, np.eye(6))
    J, _ = ppd.rows(R, t, rec)
    h = 1e-6
    Jfd = np.empty((6, 6))
    for k in range(6):
        x = np.zeros(6)
        x[k] = h
        Jfd[:, k] = (ppd.residual(*ppd.apply(R, t, x), rec) - ppd.residual(*ppd.apply(R, t, -x), rec)) / (2 * h)
    assert np.abs(J - Jfd).max() <= 1e-7 * max(1.0, np.abs(J).max()), np.abs(J - Jfd).max()
    assert abs(np.linalg.norm(ppd.residual(R, t, rec)[:3]) - math.radians(deg)) <= 1e-12


@pytest.mark.parametrize("eps", [1e-3, 1e-6, 1e-9])
def test_log_is_exact_near_pi(eps):
    rng = np.random.default_rng(5)
    for _ in range(20):
        a = _unit(rng)
        th = math.pi - eps
        w = ppd.log_so3(pd.exp_map(th * a))
        assert np.abs(w - th * a).max() <= 4e-15 * math.pi / eps + 1e-14, (eps, np.abs(w - th * a).max())


def _case(seed, n=192, **kw):
    K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(n_pts=n, seed=seed, **kw)
    return K, R0, t0, Ms, ms, Rt, tt


@pytest.mark.parametrize("seed,covx", [(3, False), (17, True)])
def test_loose_prior_is_the_solve_without_one(seed, covx):
    K, R0, t0, Ms, ms, _, _ = _case(seed)
    rng = np.random.default_rng(seed)
    cov = od.random_covx(len(Ms), rng)[0] if covx else None
    Rp, tp, _ = ppd.random_prior(R0, t0, rng, max_deg=10.0)
    ok, R, t, _ = od.estimate(K, R0, t0, Ms, ms, TAU, None, pd.DEFAULT_OPT, cov)
    ok_p, R_p, t_p, _ = ppd.estimate(K, R0, t0, Ms, ms, TAU, None, pd.DEFAULT_OPT, cov, (Rp, tp, 1e12 * np.eye(6)))
    assert ok and ok_p
    assert np.abs(R - R_p).max() <= 1e-9 and np.abs(t - t_p).max() <= 1e-9


def _augmented(K, Rc, tc, Ms, ms, rec, Lf=None):
    """The residuals of the prior-augmented objective in the chart around (Rc, tc)."""
    def res(x):
        R, t = ppd.apply(Rc, tc, x)
        u, v = pd.project(K, R, t, Ms)
        r0, r1 = ms[:, 0] - u, ms[:, 1] - v
        if Lf is not None:
            r0, r1 = od.whiten(Lf, r0, r1)
        return np.concatenate([r0, r1, ppd.rows(R, t, rec)[1]])
    return res


@pytest.mark.parametrize("seed,n,covx", [(7, 192, False), (23, 12, True), (41, 4, False)])
def test_solve_and_stage_reach_the_least_squares_minimum(seed, n, covx):
    """prevErrs None and maxIterRW = 1: every weight is 1, so the solve minimises the augmented sum of squares; scipy's
    trust-region solver on the same residuals finds the same pose, and the stage's covariance (tau far beyond every
    residual, so every weight is 1 to roundoff) is scipy's (J^T J)^-1 there."""
    rng = np.random.default_rng(seed)
    K, R0, t0, Ms, ms, Rt, tt = _case(seed, n, noise_px=1.0, outlier_frac=0.0)
    cov = od.random_covx(len(Ms), rng)[0] if covx else None
    Lf = None if cov is None else od.factors(cov)
    prior = ppd.random_prior(Rt, tt, rng, max_deg=2.0, cond=1e4, scale=1e-2)
    rec = ppd.prior_record(*prior)
    tau = 1e6
    opt = (100, 1) + pd.DEFAULT_OPT[2:]
    ok, R, t, f = ppd.estimate(K, R0, t0, Ms, ms, tau, None, opt, cov, prior)
    sol = least_squares(_augmented(K, R0, t0, Ms, ms, rec, Lf), np.zeros(6), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    R_ls, t_ls = ppd.apply(R0, t0, sol.x)
    assert ok and f["nIterRW"] == 1
    assert np.abs(R - R_ls).max() < 1e-6 and np.abs(t - t_ls).max() < 1e-6, (np.abs(R - R_ls).max(),
                                                                              np.abs(t - t_ls).max())
    L = od.factors(od.identity(len(Ms)) if cov is None else cov)
    assert ppd.cost(K, R, t, np.ones(len(Ms)), Ms, ms, L, rec) == pytest.approx(2 * sol.cost, rel=1e-9)
    # the stage at the scipy minimum against (J^T J)^-1 of the residuals in the chart there
    st = ppd.cov_stage(K, R_ls, t_ls, Ms, ms, tau, 1.0, cov, prior)
    at = least_squares(_augmented(K, R_ls, t_ls, Ms, ms, rec, Lf), np.zeros(6), jac="3-point", max_nfev=1)
    want = np.linalg.inv(at.jac.T @ at.jac)
    assert st["valid"] and st["dof"] == 2 * n
    rel = np.linalg.norm(st["cov"] - want) / np.linalg.norm(want)
    assert rel <= 1e-6, rel


def test_unobserved_camera_goes_to_its_mean_with_cov_p():
    rng = np.random.default_rng(9)
    K, R0, t0, _, _, _, _ = _case(9)
    Rp, tp, P = ppd.random_prior(R0, t0, rng, max_deg=25.0, cond=1e3, scale=1e-2)
    none3, none2 = np.zeros((0, 3)), np.zeros((0, 2))
    ok, R, t, f = ppd.estimate(K, R0, t0, none3, none2, TAU, None, pd.DEFAULT_OPT, None, (Rp, tp, P))
    assert ok
    assert np.abs(R - Rp).max() <= 1e-12 and np.abs(t - tp).max() <= 1e-12
    st = ppd.cov_stage(K, R, t, none3, none2, TAU, 1.0, None, (Rp, tp, P))
    assert st["valid"] and st["dof"] == 0
    assert np.linalg.norm(st["cov"] - P) <= 1e-9 * np.linalg.norm(P)


@pytest.mark.parametrize("seed", [2, 13])
def test_ba_camera_covariance_converts_to_the_pose_chart(seed):
    """One camera whose points are all fixed: the BA's camCov, in R' = exp([w]x) R, converted by
    diag(R^T, I) Sigma diag(R, I), is the pose stage's covariance in R' = R exp([w]x) at the same pose and threshold."""
    K, _, _, Ms, ms, Rt, tt = _case(seed, 60, noise_px=1.0, outlier_frac=0.1)
    n = len(Ms)
    prob = BAProblem(K, Rt, tt, Ms, np.arange(n + 1), np.zeros(n, np.int32), ms, 0, n)
    camCov, _, _, _ = bcd.cov_full(prob, TAU, 1.0)
    D = np.eye(6)
    D[:3, :3] = Rt
    conv = D.T @ camCov[0] @ D
    st = ppd.cov_stage(K, Rt, tt, Ms, ms, TAU, 1.0)
    assert st["valid"]
    rel = np.linalg.norm(conv - st["cov"]) / np.linalg.norm(st["cov"])
    assert rel <= 1e-9, rel
