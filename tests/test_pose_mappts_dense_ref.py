"""The map-point update restatement of tests/pose_mappts_dense.py without a GPU, before any GPU test trusts it: H_X and
H_c against central differences (H_c in the pose solver's chart), the first Gauss-Newton step is the Kalman update and
the information-form covariance the Joseph form, the converged update is the minimiser scipy.optimize.least_squares
finds with P+ its (J^T J)^-1, P_c = 0 leaves R_eff = Sigma_m, every status, and a Monte-Carlo run whose statistics
fix the bounds of the GPU test."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.stats import chi2

import pose_cov_dense as cd
import pose_dense as pd
import pose_mappts_dense as md

# the Monte-Carlo bounds tests/test_gpu_pose_mappts.py uses, fixed from test_monte_carlo below
MC_NEES = (2.75, 3.25)
MC_D2 = (1.85, 2.15)
MC_REJECT = (0.035, 0.065)


def _scene(seed, n=8, p0=(1e-4, 1e-2), sm=(0.25, 2.25)):
    """A camera at a random pose, a random pose covariance and n map points in view with random P0 and Sigma_m."""
    rng = np.random.default_rng(seed)
    K = md.K_MC
    R, t = pd.exp_map(rng.normal(0.0, 0.3, 3)), rng.normal(0.0, 0.5, 3)
    Pc = md.random_spd(rng, 6, 1e-8, 1e-5)
    Xt = md.view_points(K, R, t, rng, n, md.W_MC, md.H_MC, 3.0, 10.0)
    P0 = np.array([md.random_spd(rng, 3, *p0) for _ in range(n)])
    X0 = np.array([rng.multivariate_normal(Xt[i], P0[i]) for i in range(n)])
    Sm = np.array([md.random_spd(rng, 2, *sm) for _ in range(n)])
    u, v = pd.project(K, R, t, Xt)
    m = np.column_stack([u, v]) + rng.normal(0.0, 1.0, (n, 2))
    return K, R, t, Pc, X0, P0, m, Sm


def test_jacobians_match_central_differences():
    K, R, t, _, X0, _, _, _ = _scene(1)
    h = 1e-6
    for X in X0:
        _, HX, Hc, _ = md.jacobians(K, R, t, X)
        fd = np.empty((2, 3))
        for k in range(3):
            dx = np.zeros(3)
            dx[k] = h
            fd[:, k] = (md.jacobians(K, R, t, X + dx)[0] - md.jacobians(K, R, t, X - dx)[0]) / (2 * h)
        assert np.abs(HX - fd).max() <= 1e-6 * np.abs(HX).max(), np.abs(HX - fd).max()
        fdc = np.empty((2, 6))
        for k in range(6):
            x = np.zeros(6)
            x[k] = h
            plus = md.jacobians(K, R @ pd.exp_map(x[:3]), t + x[3:], X)[0]
            minus = md.jacobians(K, R @ pd.exp_map(-x[:3]), t - x[3:], X)[0]
            fdc[:, k] = (plus - minus) / (2 * h)
        assert np.abs(Hc - fdc).max() <= 1e-6 * np.abs(Hc).max(), np.abs(Hc - fdc).max()


@pytest.mark.parametrize("seed", [2, 3, 4])
def test_first_step_is_the_kalman_update(seed):
    K, R, t, Pc, X0, P0, m, Sm = _scene(seed)
    for i in range(len(X0)):
        r = md.update(K, R, t, Pc, X0[i], P0[i], m[i], Sm[i], 1e9)
        assert r["status"] == 0
        m0, H, _, _ = md.jacobians(K, R, t, X0[i])
        Reff = md.r_eff(K, R, t, X0[i], Pc, Sm[i])
        S = H @ P0[i] @ H.T + Reff
        G = P0[i] @ H.T @ np.linalg.inv(S)
        X1 = X0[i] + G @ (m[i] - m0)
        assert np.abs(r["X1"] - X1).max() <= 1e-12 * np.abs(X1).max()
        A = np.eye(3) - G @ H
        joseph = A @ P0[i] @ A.T + G @ Reff @ G.T
        info = md.posterior_cov(H, P0[i], Reff)
        assert np.linalg.norm(info - joseph) <= 1e-12 * np.linalg.norm(joseph)
        # the step test's objective change, formed from differences, is the difference of the objectives
        df = md.objective(K, R, t, X1, X0[i], P0[i], m[i], Reff) - md.objective(K, R, t, X0[i], X0[i], P0[i], m[i], Reff)
        got = md.descent(K, R, t, X0[i], X0[i], P0[i], Reff, m[i] - m0, X1 - X0[i])
        assert got == pytest.approx(df, rel=1e-9, abs=1e-12)


def _whitened(K, R, t, X0, P0, m, Reff):
    Lp = np.linalg.cholesky(np.linalg.inv(P0)).T  # Lp^T Lp = P0^-1
    Lr = np.linalg.cholesky(np.linalg.inv(Reff)).T
    return lambda X: np.concatenate([Lp @ (X - X0), Lr @ (m - md.jacobians(K, R, t, X)[0])])


@pytest.mark.parametrize("seed", [5, 6, 7])
def test_converged_update_is_the_least_squares_minimiser(seed):
    """weak priors (10 to 30 cm) so that the update takes several Gauss-Newton steps"""
    K, R, t, Pc, X0, P0, m, Sm = _scene(seed, p0=(1e-2, 9e-2))
    multi = 0
    for i in range(len(X0)):
        r = md.update(K, R, t, Pc, X0[i], P0[i], m[i], Sm[i], 1e9)
        assert r["status"] == 0
        multi += r["steps"] > 1
        Reff = md.r_eff(K, R, t, X0[i], Pc, Sm[i])
        f = _whitened(K, R, t, X0[i], P0[i], m[i], Reff)
        # Levenberg-Marquardt: the trust-region default stalls 1e-9 short of the minimum on these badly scaled
        # problems (depth is known from the prior alone)
        ls = least_squares(f, X0[i], method="lm", jac="3-point", ftol=1e-15, xtol=1e-15, gtol=1e-15)
        assert np.abs(r["X"] - ls.x).max() <= 1e-9 * np.abs(ls.x).max(), np.abs(r["X"] - ls.x).max()
        cov = np.linalg.inv(ls.jac.T @ ls.jac)
        assert np.linalg.norm(r["P"] - cov) <= 1e-8 * np.linalg.norm(cov)
        assert md.objective(K, R, t, r["X"], X0[i], P0[i], m[i], Reff) <= 2 * float(ls.cost) * (1 + 1e-9)
    assert multi > 0


def test_zero_pose_covariance_leaves_sigma_m():
    K, R, t, _, X0, P0, m, Sm = _scene(8)
    for i in range(len(X0)):
        assert np.array_equal(md.r_eff(K, R, t, X0[i], np.zeros((6, 6)), Sm[i]), Sm[i])
        r = md.update(K, R, t, np.zeros((6, 6)), X0[i], P0[i], m[i], Sm[i], 1e9)
        m0, H, _, _ = md.jacobians(K, R, t, X0[i])
        nu = m[i] - m0
        assert r["d2_0"] == pytest.approx(float(nu @ np.linalg.solve(H @ P0[i] @ H.T + Sm[i], nu)), rel=1e-12)


def test_statuses():
    K, R, t, Pc, X0, P0, m, Sm = _scene(9, n=4)
    centre = md.centre_point(R, t)
    ahead = R.T @ (np.array([0.0, 0.0, 5.0]) - t)
    behind = R.T @ (np.array([0.0, 0.0, -5.0]) - t)
    assert md.update(K, R, t, Pc, centre, P0[0], m[0], Sm[0], 5.99)["status"] == 2
    zero = md.update(K, np.eye(3), np.array([1.0, 2.0, 3.0]), Pc, [-1.0, -2.0, -3.0], P0[0], m[0], Sm[0], 5.99)
    assert zero["status"] == 2 and math.isnan(zero["e0"])
    r = md.update(K, R, t, Pc, behind, P0[0], m[0], Sm[0], 5.99)
    assert r["status"] == 2 and math.isnan(r["d2_0"]) and np.array_equal(r["X"], behind)
    far = md.update(K, R, t, Pc, ahead, P0[1], md.jacobians(K, R, t, ahead)[0] + 200.0, Sm[1], 5.99)
    assert far["status"] == 1 and far["d2_0"] >= 5.99 and math.isnan(far["d2_1"])
    assert np.array_equal(far["X"], ahead) and far["e0"] == pytest.approx(200.0 * math.sqrt(2.0))
    r = md.update(K, R, t, Pc, X0[2], P0[2], m[2], Sm[2], 5.99, pose_valid=False)
    assert r["status"] == 3 and math.isnan(r["d2_0"]) and np.array_equal(r["X"], X0[2])
    r = md.update(K, R, t, Pc, X0[3], P0[3], m[3], Sm[3], 1e9)
    assert r["status"] == 0 and r["d2_1"] < r["d2_0"] and np.linalg.det(r["P"]) < np.linalg.det(P0[3])


def mc_stats(frames):
    """(mean NEES of the updated points, mean d2_0, rejection rate at the 95 % gate) over the frames' updates."""
    ne, d2, rej = [], [], []
    for fr, res in frames:
        ok = res["status"] == 0
        assert ((res["status"] == 0) | (res["status"] == 1)).all()
        ne.append(md.nees(res["X"][ok], res["P"][ok], fr["Xt"][ok]))
        d2.append(res["d2_0"])
        rej.append(res["status"] == 1)
    return float(np.mean(np.concatenate(ne))), float(np.mean(np.concatenate(d2))), float(np.mean(np.concatenate(rej)))


def test_monte_carlo():
    """300 frames of 20 map points: the pose from a separate noisy solve (30 points at 1 px) with its stage
    covariance, prior means drawn from P0 and observations from Sigma_m.  NEES of X+ has 3 dof, d2_0 is chi-square
    with 2 dof and the 95 % gate rejects 5 %; the gating leaves out the largest innovations, so the NEES of the
    updated points sits slightly below 3.  The means of 6000 points are correlated within a frame by its pose error."""
    rng = np.random.default_rng(7300)
    frames = []
    for _ in range(300):
        fr = md.mc_frame(rng)
        R, t = md.pose_gn(md.K_MC, fr["R0"], fr["t0"], fr["Ms"], fr["ms"])
        Pc = cd.cov_stage(md.K_MC, R, t, fr["Ms"], fr["ms"], md.TAU_MC, 1.0)["cov"]
        frames.append((fr, md.update_all(md.K_MC, R, t, Pc, fr["X0"], fr["P0"], fr["m"], fr["Sm"], md.GATE_95)))
    m_nees, m_d2, rej = mc_stats(frames)
    print(f"mean NEES {m_nees:.3f}, mean d2_0 {m_d2:.3f}, rejected {rej:.4f}")
    assert md.GATE_95 == pytest.approx(chi2.ppf(0.95, 2), rel=1e-15)
    assert MC_NEES[0] <= m_nees <= MC_NEES[1]
    assert MC_D2[0] <= m_d2 <= MC_D2[1]
    assert MC_REJECT[0] <= rej <= MC_REJECT[1]
