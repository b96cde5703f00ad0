"""The float64 references of a BA with measurement covariances (tests/ba_obscov_dense.py) on the CPU, before any GPU
test trusts them: Sigma = I reduces every one of them to the unweighted reference of ba_dense / ba_cov_dense, and
Sigma = s^2 I scales the normal equations, the gradient and the costs by 1 / s^2 (the step stays) and the covariance
by s^2.  Anisotropic covariances are whitened by an upper-triangular L with L^T L = Sigma^-1."""
import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od

ROWS = ["rig_intrinsics", "unobserved_points", "tukey_mixed", "unsorted_observations"]


def _eye(N, s2=1.0):
    return np.tile(s2 * np.eye(2), (N, 1, 1))


def test_factors_whiten():
    rng = np.random.default_rng(1)
    covx, S = od.random_covx(500, rng)
    L = od.factors(covx)
    assert np.all(L[:, 1, 0] == 0) and np.all(L[:, 0, 0] > 0) and np.all(L[:, 1, 1] > 0)
    lam = np.linalg.inv(covx)
    assert np.abs(L.transpose(0, 2, 1) @ L - lam).max() <= 1e-12 * np.abs(lam).max()
    sd = np.sqrt(np.linalg.eigvalsh(covx))
    assert sd.min() >= 0.3 - 1e-12 and sd.max() <= 1.5 + 1e-12
    # noise drawn through S has covariance S S^T = covx: whitened it is standard
    z = np.stack([od.draw_noise(S, rng) for _ in range(400)])
    zw = np.einsum("nab,knb->kna", L, z)
    assert abs(zw.var() - 1.0) < 0.02
    # the closed form the device uses: l00 = sqrt(s11 / det), l01 = -s01 / sqrt(s11 det), l11 = 1 / sqrt(s11)
    a, b, c = covx[:, 0, 0], covx[:, 0, 1], covx[:, 1, 1]
    det = a * c - b * b
    closed = np.stack([np.sqrt(c / det), -b / np.sqrt(c * det), 1 / np.sqrt(c)], 1)
    assert np.abs(closed - L[:, [0, 0, 1], [0, 1, 1]]).max() <= 1e-12 * np.abs(closed).max()


@pytest.mark.parametrize("name", ROWS)
def test_identity_is_the_unweighted_trial(name):
    prob, opt = bd.make(name)
    T, W = bd.Trial(prob, opt), od.WTrial(prob, opt, _eye(prob.nobs))
    assert np.array_equal(T.A, W.A) and np.array_equal(T.g, W.g) and np.array_equal(T.d, W.d)
    assert T.cost0 == W.cost0 and T.mu == W.mu


@pytest.mark.parametrize("name", ROWS)
def test_scaled_identity_scales_the_trial(name):
    prob, opt = bd.make(name)
    s2 = 4.0  # a power of two: every scaled quantity is exact
    T, W = bd.Trial(prob, opt), od.WTrial(prob, opt, _eye(prob.nobs, s2))
    assert np.array_equal(W.A, T.A / s2) and np.array_equal(W.g, T.g / s2) and np.array_equal(W.d, T.d)
    assert W.cost0 == T.cost0 / s2
    W9 = od.WTrial(prob, opt, _eye(prob.nobs, 9.0))
    assert np.abs(W9.A - T.A / 9).max() <= 1e-14 * np.abs(T.A).max()
    assert np.abs(W9.d - T.d).max() <= 1e-9 * np.abs(T.d).max()
    H, g = od.normal_equations(prob, opt.max_err, _eye(prob.nobs, 9.0))
    assert np.abs(H - (T.A - T.mu * np.eye(T.np)) / 9).max() <= 1e-14 * np.abs(H).max() * 9
    assert np.abs(g - T.g / 9).max() <= 1e-14 * np.abs(T.g).max()


@pytest.mark.parametrize("name", ["rig_intrinsics", "tukey_mixed"])
def test_covariance_reduces_and_scales(name):
    prob, opt = bd.make(name)
    N = prob.nobs
    cam, pt, inf, H = cd.cov_full(prob, opt.max_err, 2.5)
    wcam, wpt, winf, wH = od.cov_full(prob, opt.max_err, 2.5, _eye(N))
    assert np.array_equal(H, wH)
    for a, b in ((cam, wcam), (pt, wpt)):
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a, b, rtol=1e-12, atol=0, equal_nan=True)
    assert winf["dof"] == inf["dof"] and abs(winf["sigma2_hat"] - inf["sigma2_hat"]) <= 1e-14 * inf["sigma2_hat"]
    # Sigma = s^2 I with pixel_var 1 is the unweighted covariance with pixel_var s^2; sigma2_hat scales by 1 / s^2
    scam, spt, sinf, _ = od.cov_full(prob, opt.max_err, 1.0, _eye(N, 2.5))
    for a, b in ((cam, scam), (pt, spt)):
        assert np.allclose(a, b, rtol=1e-9, atol=0, equal_nan=True)
    assert abs(sinf["sigma2_hat"] * 2.5 - inf["sigma2_hat"]) <= 1e-12 * inf["sigma2_hat"]


def test_anisotropic_weights_change_the_step():
    prob, opt = bd.make("rig_intrinsics")
    covx, _ = od.random_covx(prob.nobs, np.random.default_rng(3))
    T, W = bd.Trial(prob, opt), od.WTrial(prob, opt, covx)
    assert np.abs(W.d - T.d).max() > 1e-3 * np.abs(T.d).max()
    # the whitened gradient is J^T W Lambda e, written out
    H, g = od.normal_equations(prob, opt.max_err, covx)
    assert np.abs(g - W.g).max() <= 1e-12 * np.abs(W.g).max()
    assert np.abs(H + W.mu * np.eye(W.np) - W.A).max() <= 1e-12 * np.abs(W.A).max()
