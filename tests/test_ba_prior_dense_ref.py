"""Pins tests/ba_prior_dense.py, the float64 restatement of a bundle adjustment with camera priors, on the CPU:
  - the analytic prior Jacobian in the solver's chart against central differences, at v != 0 and prior angles up to
    30 degrees (and the Log near pi);
  - with P -> infinity the trial and the covariance reduce to ba_obscov_dense's;
  - with the estimate at the prior mean, r = 0: the gradient is the observations' and only H changes;
  - cov_full against scipy.optimize.least_squares' (J^T J)^-1 at a converged fit."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
import ba_prior_dense as pd
from coslam_b200.problem import BAProblem


def _unit(rng):
    a = rng.normal(size=3)
    return a / np.linalg.norm(a)


@pytest.mark.parametrize("deg", [0.0, 1e-3, 0.5, 5.0, 30.0])
def test_prior_jacobian_against_central_differences(deg):
    rng = np.random.default_rng(int(deg * 100) + 1)
    for _ in range(5):
        R0 = pd.so3_exp(rng.normal(size=3))
        v = 0.05 * rng.normal(size=3)  # the solver's local rotation, away from 0
        t = rng.normal(size=3)
        Rp = pd.so3_exp(np.deg2rad(deg) * _unit(rng)) @ pd.chart_R(R0, v)
        tp = t + 0.1 * rng.normal(size=3)
        J = pd.prior_jacobian(R0, v, t, Rp, tp)
        h = 1e-6
        Jn = np.empty((6, 6))
        for k in range(6):
            dv, dt = np.zeros(3), np.zeros(3)
            (dv if k < 3 else dt)[k % 3] = h
            Jn[:, k] = (pd.prior_residual(R0, v + dv, t + dt, Rp, tp) -
                        pd.prior_residual(R0, v - dv, t - dt, Rp, tp)) / (2 * h)
        assert np.abs(J - Jn).max() <= 1e-8 * max(1.0, np.abs(J).max()), (deg, np.abs(J - Jn).max())
        r = pd.prior_residual(R0, v, t, Rp, tp)
        assert abs(np.linalg.norm(r[:3]) - np.deg2rad(deg)) <= 1e-12


@pytest.mark.parametrize("deg", [100.0, 150.0, 179.0, 179.999])
def test_log_is_the_inverse_of_exp_up_to_pi(deg):
    rng = np.random.default_rng(int(deg))
    for _ in range(5):
        w = np.deg2rad(deg) * _unit(rng)
        assert np.abs(pd.so3_log(pd.so3_exp(w)) - w).max() <= 1e-12 / max(np.pi - np.deg2rad(deg), 1e-3)


def _priors(prob, cams, seed, scale=1.0, deg=3.0):
    rng = np.random.default_rng(seed)
    cov = pd.random_cov(len(cams), rng) * scale
    R, t = pd.offset_means(prob, cams, rng, deg=deg)
    return pd.Priors(cams, R, t, cov)


@pytest.mark.parametrize("name", ["rig_intrinsics", "unobserved_points", "tukey_mixed"])
def test_infinite_prior_covariance_is_the_obscov_reference(name):
    prob, opt = bd.make(name)
    covx = od.random_covx(prob.nobs, np.random.default_rng(3))[0]
    cams = np.arange(prob.m_con, prob.m)
    pr = _priors(prob, cams, 4, scale=1e30)
    T = pd.PTrial(prob, opt, covx, pr)
    W = od.WTrial(prob, opt, covx)
    assert abs(T.mu - W.mu) <= 1e-12 * W.mu
    assert np.abs(T.d - W.d).max() <= 1e-9 * np.abs(W.d).max()
    assert abs(T.cost0 - W.cost0) <= 1e-12 * W.cost0
    c = cd.make("rig_intrinsics")[0]
    cam, pt, inf, _ = pd.cov_full(c, bd.MAX_ERR, 2.0, None, _priors(c, np.arange(c.m_con, c.m), 5, scale=1e30))
    wcam, wpt, winf, _ = od.cov_full(c, bd.MAX_ERR, 2.0, pd.identity_covx(c))
    assert np.abs(cam - wcam).max() <= 1e-9 * np.abs(wcam).max()
    assert np.abs(pt - wpt).max() <= 1e-9 * np.abs(wpt).max()
    assert inf["dof"] == winf["dof"] + 6 * (c.m - c.m_con) and inf["priors"] == c.m - c.m_con


def test_prior_at_the_estimate_changes_only_h():
    prob, _ = bd.make("rig_intrinsics")
    cams = np.arange(prob.m_con, prob.m)
    cov = pd.random_cov(len(cams), np.random.default_rng(6))
    pr = pd.Priors(cams, prob.R.reshape(-1, 3, 3)[cams], prob.t[cams], cov)
    assert np.abs(pd.residuals(prob, pr)).max() == 0.0
    H0, g0 = od.normal_equations(prob, bd.MAX_ERR, pd.identity_covx(prob))
    H1, g1 = pd.normal_equations(prob, bd.MAX_ERR, None, pr)
    assert np.array_equal(g0, g1)
    D = np.diag([2.0, 2.0, 2.0, 1.0, 1.0, 1.0])  # J at r = 0 and v = 0: Jl^-1 = I, J_q = 2 I
    for k, j in enumerate(cams):
        c = 6 * (j - prob.m_con) + np.arange(6)
        want = D @ np.linalg.inv(cov[k]) @ D
        assert np.abs((H1 - H0)[np.ix_(c, c)] - want).max() <= 1e-9 * np.abs(want).max()
    dH = H1 - H0
    for k, j in enumerate(cams):
        c = 6 * (j - prob.m_con) + np.arange(6)
        dH[np.ix_(c, c)] = 0
    assert np.abs(dH).max() <= 1e-9 * np.abs(H0).max()


# ---------------------------------------------------------------- against scipy's minimiser
def _pack(prob, base, x):
    """prob with the free cameras at exp([w]x) R_base, t and the free points at X, from x = [w, t per free camera |
    X per free point]"""
    p = bd.fresh(base)
    mf = prob.m - prob.m_con
    R = base.R.reshape(-1, 3, 3).copy()
    t = base.t.copy()
    X = base.X.copy()
    cx = x[:6 * mf].reshape(mf, 6)
    for q, j in enumerate(range(prob.m_con, prob.m)):
        R[j] = pd.so3_exp(cx[q, :3]) @ R[j]
        t[j] = cx[q, 3:]
    X[prob.n_con:] = x[6 * mf:].reshape(-1, 3)
    return BAProblem(base.K.copy(), R, t, X, base.ptr.copy(), base.cam.copy(), base.xy.copy(), base.m_con,
                     base.n_con)


def _fun(prob, base, pr, Lp):
    def f(x):
        p = _pack(prob, base, x)
        return np.concatenate([bd.residuals(p).ravel(), np.einsum("kab,kb->ka", Lp, pd.residuals(p, pr)).ravel()])
    return f


def _x0(prob):
    mf = prob.m - prob.m_con
    return np.concatenate([np.concatenate([np.zeros((mf, 3)), prob.t[prob.m_con:]], 1).ravel(),
                           prob.X[prob.n_con:].ravel()])


def test_cov_full_is_scipy_inverse_at_the_optimum():
    truth = cd.small_nonrobust()
    rng = np.random.default_rng(8)
    prob = bd.fresh(truth)
    prob.xy = truth.xy + rng.normal(0, 0.5, truth.xy.shape)
    cams = np.array([2, 4, 5])
    cov = pd.random_cov(3, rng)
    R, t = pd.draw_means(truth, cams, cov, rng)
    pr = pd.Priors(cams, R, t, cov)
    Lp = pr.factors()
    sol = least_squares(_fun(prob, prob, pr, Lp), _x0(prob), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    fit = _pack(prob, prob, sol.x)
    # J at the optimum in the chart anchored there (w = 0), by central differences
    again = least_squares(_fun(fit, fit, pr, Lp), _x0(fit), jac="3-point", method="lm", max_nfev=1)
    J = again.jac
    C = np.linalg.inv(J.T @ J)
    cam, pt, info, H = pd.cov_full(fit, 0.0, 1.0, None, pr)
    mf = fit.m - fit.m_con
    for q, j in enumerate(range(fit.m_con, fit.m)):
        want = C[6 * q:6 * q + 6, 6 * q:6 * q + 6]
        assert np.abs(cam[j] - want).max() <= 1e-5 * np.abs(want).max(), j
    for i in range(fit.n_con, fit.n):
        c = 6 * mf + 3 * (i - fit.n_con)
        want = C[c:c + 3, c:c + 3]
        assert np.abs(pt[i] - want).max() <= 1e-5 * np.abs(want).max(), i
    assert info["dof"] == 2 * fit.nobs - 6 * mf - 3 * (fit.n - fit.n_con) + 18
    assert abs(info["sigma2_hat"] - float(again.fun @ again.fun) / info["dof"]) <= 1e-9 * info["sigma2_hat"]
