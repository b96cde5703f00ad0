"""The pose covariance reference of tests/pose_cov_dense.py without a GPU, so that it is pinned before it judges the
device: its analytic Jacobian against central differences of the projection under the solver's right-multiplied
chart, its covariance against scipy.optimize.least_squares' (J^T W J)^-1 at a converged robust solution, and its
statistics and singular cameras."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares

import pose_cov_dense as cd
import pose_dense as pd
from coslam_b200 import synth

TAU = 10.0


def _case(seed, n=192, **kw):
    K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(n_pts=n, seed=seed, **kw)
    return K, R0, t0, Ms, ms


def _moved(R, t, x):
    return R @ pd.exp_map(x[:3]), t + x[3:]


@pytest.mark.parametrize("seed", [3, 17, 29])
def test_analytic_jacobian_matches_central_differences(seed):
    K, R, t, Ms, _ = _case(seed, 64)
    J = cd.jacobian(K, R, t, Ms)
    h = 1e-6
    num = np.empty_like(J)
    for k in range(6):
        dx = np.zeros(6)
        dx[k] = h
        up = np.stack(pd.project(K, *_moved(R, t, dx), Ms), 1)
        dn = np.stack(pd.project(K, *_moved(R, t, -dx), Ms), 1)
        num[:, :, k] = (up - dn) / (2 * h)
    assert np.abs(J - num).max() <= 1e-6 * np.abs(J).max()


def _robust_fit(K, R, t, Ms, ms, rounds=8):
    """Tukey-IRLS with least_squares inner solves in the chart around the current pose, unit weights in the
    first round as the solver without prevErrs; returns the pose and the last least_squares result, taken
    around that pose's predecessor."""
    sw = np.ones(len(Ms))
    for k in range(rounds):
        if k:
            sw = np.sqrt(pd.weights(cd.residuals(K, R, t, Ms, ms), TAU))

        def f(x, R=R, t=t, sw=sw):
            u, v = pd.project(K, *_moved(R, t, x), Ms)
            return np.concatenate([sw * (u - ms[:, 0]), sw * (v - ms[:, 1])])

        sol = least_squares(f, np.zeros(6), jac="3-point", xtol=1e-15, ftol=1e-15, gtol=1e-15)
        R, t = _moved(R, t, sol.x)
    return R, t, sol


@pytest.mark.parametrize("seed", [5, 11])
def test_covariance_matches_least_squares(seed):
    K, R0, t0, Ms, ms = _case(seed)
    var = 0.25
    R, t, sol = _robust_fit(K, R0, t0, Ms, ms)
    assert np.abs(sol.x).max() < 1e-9  # the last round started at its own solution
    ref = cd.cov_stage(K, R, t, Ms, ms, TAU, var)
    assert ref["valid"] and (ref["w"] == 0).any()  # the outliers of the case are beyond tau
    cov_ls = var * np.linalg.inv(sol.jac.T @ sol.jac)
    assert np.linalg.norm(ref["cov"] - cov_ls) <= 1e-8 * np.linalg.norm(cov_ls)
    assert np.allclose(ref["cov"], ref["cov"].T, rtol=0, atol=1e-12 * np.abs(ref["cov"]).max())
    assert np.all(np.linalg.eigvalsh(ref["cov"]) > 0)


def test_statistics():
    K, R, t, Ms, ms = _case(7, 100, outlier_frac=0.0)
    ms = ms.copy()
    ms[:15, 0] += 50.0  # beyond tau
    ref = cd.cov_stage(K, R, t, Ms, ms, TAU, 1.0)
    e, w = ref["e"], ref["w"]
    assert np.array_equal(w == 0, e >= TAU) and (w == 0).sum() >= 15
    assert ref["dof"] == 2 * int((w > 0).sum()) - 6
    assert ref["sigma2_hat"] == pytest.approx(float(np.sum(w * e * e)) / ref["dof"], rel=1e-13)
    H = sum(w[i] * ref["J"][i].T @ ref["J"][i] for i in range(len(w)))
    assert np.allclose(ref["H"], H, rtol=1e-13, atol=0)
    assert ref["valid"] and 1e-12 <= ref["min_pivot"] <= 1.0


def test_points_with_non_finite_residuals_are_left_out():
    """x_depth0 of tests/pose_edge_cases.py at R0: its last point has depth 0, e = inf and weight 0.  The
    covariance is the one of the other 128 points alone (0 * inf must not make H NaN), and e stays inf.  A NaN
    residual (a point at the camera centre) likewise has a NaN weight and is left out."""
    import pose_edge_cases as pc
    K, R0, t0, Ms, ms, tau, _, _ = pc.case_inputs(pc.row("x_depth0"))
    ref = cd.cov_stage(K, R0, t0, Ms, ms, tau, 1.0)
    rest = cd.cov_stage(K, R0, t0, Ms[:-1], ms[:-1], tau, 1.0)
    assert np.isinf(ref["e"][-1]) and ref["w"][-1] == 0 and np.isfinite(ref["e"][:-1]).all()
    assert rest["valid"] and ref["valid"]
    assert np.array_equal(ref["H"], rest["H"]) and np.array_equal(ref["cov"], rest["cov"])
    assert ref["dof"] == rest["dof"] and ref["sigma2_hat"] == rest["sigma2_hat"]
    assert cd.residual_error(ref["e"], rest["e"].tolist() + [np.inf]) == 0.0
    assert cd.residual_error(ref["e"], rest["e"].tolist() + [np.nan]) == np.inf
    Mn = Ms.copy()
    Mn[-1] = -R0.T @ t0  # the camera centre: 0 / 0
    with np.errstate(invalid="ignore", divide="ignore"):
        nan = cd.cov_stage(K, R0, t0, Mn, ms, tau, 1.0)
    assert np.isnan(nan["e"][-1]) and np.array_equal(nan["cov"], rest["cov"])


def test_singular_cameras():
    K, R, t, Ms, ms = _case(9, 40)
    two = cd.cov_stage(K, R, t, Ms[:2], ms[:2], TAU, 1.0)
    assert not two["valid"] and np.isnan(two["cov"]).all()
    assert two["dof"] <= -2 and math.isnan(two["sigma2_hat"])
    far = cd.cov_stage(K, R, t, Ms, ms + 200.0, TAU, 1.0)
    assert not far["valid"] and far["min_pivot"] == 0.0 and np.isnan(far["cov"]).all()
    assert far["dof"] == -6 and math.isnan(far["sigma2_hat"])
    none = cd.cov_stage(K, R, t, Ms[:0], ms[:0], TAU, 1.0)
    assert not none["valid"] and none["dof"] == -6
