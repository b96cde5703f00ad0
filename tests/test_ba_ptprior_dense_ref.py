"""Pins tests/ba_ptprior_dense.py, the float64 restatement of a bundle adjustment with point priors, on the CPU:
  - with P -> infinity the trial, the normal equations and the covariance reduce to the references without point
    priors (ba_obscov_dense, and ba_prior_dense with camera priors set as well);
  - with the estimate at the prior mean, r = 0: the gradient is unchanged and only the point blocks of H change;
  - cov_full against scipy.optimize.least_squares' (J^T J)^-1 at a converged fit, with 0- and 1-observation points;
  - priors on three non-collinear points make the gauge of a problem without fixed cameras or points regular (two
    leave the rotation about their line free)."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
import ba_prior_dense as pd
import ba_ptprior_dense as ppd
from coslam_b200.problem import BAProblem


def _observed(prob, k):
    """k free points seen by at least two observations"""
    cnt = np.bincount(bd.point_of(prob), minlength=prob.n)
    return np.array([i for i in range(prob.n_con, prob.n) if cnt[i] >= 2][:k])


def _loose(prob, pts, seed):
    rng = np.random.default_rng(seed)
    return ppd.PtPriors(pts, ppd.offset_pt_means(prob, pts, rng), np.tile(1e30 * np.eye(3), (len(pts), 1, 1)))


@pytest.mark.parametrize("cams", [False, True], ids=["points", "points_and_cameras"])
@pytest.mark.parametrize("name", ["rig_intrinsics", "unobserved_points", "tukey_mixed"])
def test_infinite_point_prior_covariance_is_the_reference(name, cams):
    prob, opt = bd.make(name)
    covx = od.random_covx(prob.nobs, np.random.default_rng(3))[0]
    pp = _loose(prob, _observed(prob, 12), 4)
    pr = None
    if cams:
        c = np.arange(prob.m_con, prob.m)
        rng = np.random.default_rng(5)
        R, t = pd.offset_means(prob, c, rng)
        pr = pd.Priors(c, R, t, pd.random_cov(len(c), rng))
    T = ppd.PPTrial(prob, opt, covx, pr, pp)
    W = pd.PTrial(prob, opt, covx, pr) if cams else od.WTrial(prob, opt, covx)
    assert abs(T.mu - W.mu) <= 1e-12 * W.mu
    assert np.abs(T.d - W.d).max() <= 1e-9 * np.abs(W.d).max()
    assert abs(T.cost0 - W.cost0) <= 1e-12 * W.cost0
    H1, g1 = ppd.normal_equations(prob, opt.max_err, covx, pr, pp)
    H0, g0 = pd.normal_equations(prob, opt.max_err, covx, pr or ppd.no_cam_priors())
    assert np.abs(H1 - H0).max() <= 1e-12 * np.abs(H0).max() and np.abs(g1 - g0).max() <= 1e-12 * np.abs(g0).max()
    c = cd.make("rig_intrinsics")[0]
    cpp = _loose(c, _observed(c, 12), 6)
    cam, pt, inf, _ = ppd.cov_full(c, bd.MAX_ERR, 2.0, None, None, cpp)
    wcam, wpt, winf, _ = od.cov_full(c, bd.MAX_ERR, 2.0, pd.identity_covx(c))
    assert np.abs(cam - wcam).max() <= 1e-9 * np.abs(wcam).max()
    assert np.abs(pt - wpt).max() <= 1e-9 * np.abs(wpt).max()
    assert inf["dof"] == winf["dof"] + 3 * len(cpp) and inf["pt_priors"] == len(cpp)


def test_point_prior_at_the_estimate_changes_only_h():
    prob, _ = bd.make("rig_intrinsics")
    pts = _observed(prob, 20)
    cov = ppd.random_pt_cov(len(pts), np.random.default_rng(6))
    pp = ppd.PtPriors(pts, prob.X[pts], cov)
    assert np.abs(ppd.residuals(prob, pp)).max() == 0.0
    H0, g0 = od.normal_equations(prob, bd.MAX_ERR, pd.identity_covx(prob))
    H1, g1 = ppd.normal_equations(prob, bd.MAX_ERR, None, None, pp)
    assert np.array_equal(g0, g1)
    dH = H1 - H0
    mf = prob.m - prob.m_con
    for k, i in enumerate(pts):
        c = 6 * mf + 3 * (i - prob.n_con) + np.arange(3)
        want = np.linalg.inv(cov[k])
        assert np.abs(dH[np.ix_(c, c)] - want).max() <= 1e-9 * np.abs(want).max()
        dH[np.ix_(c, c)] = 0
    assert np.abs(dH).max() <= 1e-9 * np.abs(H0).max()
    assert ppd.total_cost(prob, None, None, pp) == pd.total_cost(prob, None, ppd.no_cam_priors())


# ---------------------------------------------------------------- against scipy's minimiser
def _pack(prob, base, x):
    """prob with the free cameras at exp([w]x) R_base, t and the free points at X, from x = [w, t per free camera |
    X per free point]"""
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


def _fun(prob, base, pp, Lp):
    def f(x):
        p = _pack(prob, base, x)
        return np.concatenate([bd.residuals(p).ravel(), np.einsum("kab,kb->ka", Lp, ppd.residuals(p, pp)).ravel()])
    return f


def _x0(prob):
    mf = prob.m - prob.m_con
    return np.concatenate([np.concatenate([np.zeros((mf, 3)), prob.t[prob.m_con:]], 1).ravel(),
                           prob.X[prob.n_con:].ravel()])


def _with_sparse_points(base, rng):
    """base with two more free points: one that no observation sees, one seen once"""
    X = np.concatenate([base.X, base.X[-1:] + [0.3, -0.2, 0.1], base.X[-1:] + [-0.2, 0.25, 0.05]])
    o = int(np.flatnonzero(base.cam == base.cam[-1])[0])
    K = base.K.reshape(base.m, -1).copy()
    R = base.R.reshape(-1, 3, 3)
    # the single observation of the last point by the camera of observation o, with noise
    j = int(base.cam[o])
    u = K[j].reshape(3, 3) @ (R[j] @ X[-1] + base.t[j])
    xy = np.concatenate([base.xy, (u[:2] / u[2] + rng.normal(0, 0.5, 2))[None]])
    ptr = np.concatenate([base.ptr, [base.ptr[-1], base.ptr[-1] + 1]])
    cam = np.concatenate([base.cam, [j]])
    return BAProblem(base.K.copy(), base.R.copy(), base.t.copy(), X, ptr, cam, xy, base.m_con, base.n_con)


def test_cov_full_is_scipy_inverse_at_the_optimum():
    truth = cd.small_nonrobust()
    rng = np.random.default_rng(8)
    prob = bd.fresh(truth)
    prob.xy = truth.xy + rng.normal(0, 0.5, truth.xy.shape)
    prob = _with_sparse_points(prob, rng)
    pts = np.concatenate([_observed(prob, 5), [prob.n - 2, prob.n - 1]])
    cov = ppd.random_pt_cov(len(pts), rng)
    pp = ppd.PtPriors(pts, ppd.draw_pt_means(prob, pts, cov, rng), cov)
    Lp = pp.factors()
    sol = least_squares(_fun(prob, prob, pp, Lp), _x0(prob), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    fit = _pack(prob, prob, sol.x)
    again = least_squares(_fun(fit, fit, pp, Lp), _x0(fit), jac="3-point", method="lm", max_nfev=1)
    J = again.jac
    C = np.linalg.inv(J.T @ J)
    cam, pt, info, H = ppd.cov_full(fit, 0.0, 1.0, None, None, pp)
    assert info["unconstrained"] == 0 and not info["singular"]
    mf = fit.m - fit.m_con
    for q, j in enumerate(range(fit.m_con, fit.m)):
        want = C[6 * q:6 * q + 6, 6 * q:6 * q + 6]
        assert np.abs(cam[j] - want).max() <= 1e-5 * np.abs(want).max(), j
    for i in range(fit.n_con, fit.n):
        c = 6 * mf + 3 * (i - fit.n_con)
        want = C[c:c + 3, c:c + 3]
        assert np.abs(pt[i] - want).max() <= 1e-5 * np.abs(want).max(), i
    # the unobserved prior point sits at its mean with its prior covariance
    assert np.abs(fit.X[-2] - pp.X[-2]).max() <= 1e-9
    assert np.abs(pt[-2] - cov[-2]).max() <= 1e-9 * np.abs(cov[-2]).max()
    assert info["dof"] == 2 * fit.nobs - 6 * mf - 3 * (fit.n - fit.n_con) + 3 * len(pp)
    assert abs(info["sigma2_hat"] - float(again.fun @ again.fun) / info["dof"]) <= 1e-9 * info["sigma2_hat"]


def gauge_free():
    """small_nonrobust with noise and nothing fixed"""
    p = cd.small_nonrobust()
    rng = np.random.default_rng(40)
    xy = p.xy + rng.normal(0, 0.3, p.xy.shape)
    return BAProblem(p.K.copy(), p.R, p.t, p.X, p.ptr.copy(), p.cam.copy(), xy, 0, 0)


def gauge_points(prob, k):
    """k free points far apart and not on one line (the first and last point, then the farthest from their line)"""
    X = prob.X
    a, b = 0, prob.n - 1
    d = (X[b] - X[a]) / np.linalg.norm(X[b] - X[a])
    off = X - X[a]
    dist = np.linalg.norm(off - np.outer(off @ d, d), axis=1)
    return np.array([a, b, int(np.argmax(dist))][:k])


@pytest.mark.parametrize("k", [2, 3])
def test_three_prior_points_fix_the_gauge(k):
    prob = gauge_free()
    _, _, info0, _ = ppd.cov_full(prob, 0.0, 1.0, None, None, ppd.no_pt_priors())
    assert info0["singular"]
    pts = gauge_points(prob, k)
    cov = ppd.random_pt_cov(k, np.random.default_rng(9))
    pp = ppd.PtPriors(pts, ppd.draw_pt_means(prob, pts, cov, np.random.default_rng(10)), cov)
    cam, pt, info, H = ppd.cov_full(prob, 0.0, 1.0, None, None, pp)
    assert info["singular"] == (k < 3)
    if k == 3:
        assert np.isfinite(cam).all() and np.isfinite(pt).all()
        assert cd.min_relative_pivot(H) >= 1e-9
