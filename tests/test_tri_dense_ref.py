"""The triangulation restatement of tests/tri_dense.py without a GPU, before any GPU test trusts it: X_lin is the true
point for noise-free views, H_X and H_c match central differences, X+ is the minimiser scipy.optimize.least_squares
finds with P its (J^T J)^-1, P_c = 0 leaves R_v = Sigma_m, the BA's camera covariance converts to the pose chart,
every status is reached in its order, and a Monte-Carlo run whose statistics fix the bounds of the GPU test."""
import math

import numpy as np
import pytest
from scipy.optimize import least_squares

import pose_dense as pd
import pose_mappts_dense as md
import tri_dense as td

# the Monte-Carlo bounds tests/test_gpu_tri.py uses, fixed from test_monte_carlo below
MC_NEES = (2.5, 3.5)
MC_REJECT = (0.0, 0.02)
MC_MAX_ERR = 8.0


def _scene(seed, n_views, n_pts=10, sm=(0.25, 2.25), pc=(1e-8, 1e-6)):
    """A rig of n_views camera entries, true points in front of all of them, Sigma_m per view and a pose covariance
    per camera; the observations are the true projections plus noise from Sigma_m."""
    rng = np.random.default_rng(seed)
    R, t = td.rig(rng, n_views)
    K = np.array([td.K_TRI] * n_views)
    Pc = [md.random_spd(rng, 6, *pc) for _ in range(n_views)]
    Xt = td.scene_points(rng, n_pts)
    Sm = np.array([[md.random_spd(rng, 2, *sm) for _ in range(n_views)] for _ in range(n_pts)])
    m = np.array([td.observe(td.K_TRI, R, t, X, S, rng) for X, S in zip(Xt, Sm)])
    return rng, K, R, t, Pc, Xt, Sm, m


@pytest.mark.parametrize("n_views", [2, 3, 8])
def test_linear_estimate_is_the_true_point_without_noise(n_views):
    _, K, R, t, _, Xt, _, _ = _scene(n_views, n_views)
    for X in Xt:
        m = np.array([md.jacobians(td.K_TRI, Ri, ti, X)[0] for Ri, ti in zip(R, t)])
        X_lin = td.linear(K, R, t, m)
        assert np.linalg.norm(X_lin - X) <= 1e-12 * np.linalg.norm(X), np.linalg.norm(X_lin - X)


def test_jacobians_match_central_differences():
    _, _, R, t, _, Xt, _, _ = _scene(11, 3)
    h = 1e-6
    for X in Xt[:4]:
        for Ri, ti in zip(R, t):
            _, HX, Hc, _ = md.jacobians(td.K_TRI, Ri, ti, X)
            fd = np.empty((2, 3))
            for k in range(3):
                dx = np.zeros(3)
                dx[k] = h
                fd[:, k] = (md.jacobians(td.K_TRI, Ri, ti, X + dx)[0] - md.jacobians(td.K_TRI, Ri, ti, X - dx)[0]) / (2 * h)
            assert np.abs(HX - fd).max() <= 1e-6 * np.abs(HX).max()
            fdc = np.empty((2, 6))
            for k in range(6):
                x = np.zeros(6)
                x[k] = h
                plus = md.jacobians(td.K_TRI, Ri @ pd.exp_map(x[:3]), ti + x[3:], X)[0]
                minus = md.jacobians(td.K_TRI, Ri @ pd.exp_map(-x[:3]), ti - x[3:], X)[0]
                fdc[:, k] = (plus - minus) / (2 * h)
            assert np.abs(Hc - fdc).max() <= 1e-6 * np.abs(Hc).max()


@pytest.mark.parametrize("seed,n_views", [(21, 2), (22, 3), (23, 8), (24, 32)])
def test_converged_point_is_the_least_squares_minimiser(seed, n_views):
    rng, K, R, t, Pc, Xt, Sm, m = _scene(seed, n_views, n_pts=6)
    for j in range(len(Xt)):
        r = td.triangulate(K, R, t, Pc, m[j], Sm[j])
        assert r["status"] == 0 and r["steps"] >= 1
        Rv = td.noise(K, R, t, Pc, r["X_lin"], Sm[j])
        Ls = [np.linalg.cholesky(np.linalg.inv(S)).T for S in Rv]  # L^T L = R_v^-1
        f = lambda X: np.concatenate([L @ (mv - md.jacobians(td.K_TRI, Ri, ti, X)[0])  # noqa: E731
                                      for L, mv, Ri, ti in zip(Ls, m[j], R, t)])
        # Levenberg-Marquardt from X_lin, restarted once from where it stops: its xtol test can end it while the
        # gradient is still 1e-5 on these depth-dominated problems
        ls = least_squares(f, r["X_lin"], method="lm", jac="3-point", ftol=1e-15, xtol=1e-15, gtol=1e-15)
        ls = least_squares(f, ls.x, method="lm", jac="3-point", ftol=1e-15, xtol=1e-15, gtol=1e-15)
        assert np.linalg.norm(r["X"] - ls.x) <= 1e-9 * np.linalg.norm(ls.x), np.linalg.norm(r["X"] - ls.x)
        cov = np.linalg.inv(ls.jac.T @ ls.jac)
        assert np.linalg.norm(r["P"] - cov) <= 1e-8 * np.linalg.norm(cov), np.linalg.norm(r["P"] - cov)
        assert r["stat"][0] == pytest.approx(2 * float(ls.cost), rel=1e-9, abs=1e-12)
        assert np.array_equal(r["P"], r["P"].T)


def test_zero_pose_covariance_leaves_sigma_m():
    _, K, R, t, _, Xt, Sm, m = _scene(31, 3)
    zeros = [np.zeros((6, 6))] * 3
    for j in range(len(Xt)):
        assert np.array_equal(td.noise(K, R, t, zeros, Xt[j], Sm[j]), Sm[j])
        a, b = td.triangulate(K, R, t, zeros, m[j], Sm[j]), td.triangulate(K, R, t, [None] * 3, m[j], Sm[j])
        assert np.array_equal(a["X"], b["X"]) and np.array_equal(a["P"], b["P"])


@pytest.mark.parametrize("seed", [41, 42])
def test_ba_camera_covariance_converts_to_the_pose_chart(seed):
    """H_BA, the central-difference Jacobian of the projection in the BA's chart exp([w]x) R, t + dt, gives the same
    projected pose noise with the BA covariance as H_c with blockdiag(R^T, I) P blockdiag(R, I)."""
    rng, _, R, t, _, Xt, _, _ = _scene(seed, 2)
    h = 1e-6
    for Ri, ti in zip(R, t):
        P_ba = md.random_spd(rng, 6, 1e-7, 1e-4)
        P_pose = td.ba_to_pose_chart(Ri, P_ba)
        for X in Xt[:3]:
            Hba = np.empty((2, 6))
            for k in range(6):
                x = np.zeros(6)
                x[k] = h
                plus = md.jacobians(td.K_TRI, pd.exp_map(x[:3]) @ Ri, ti + x[3:], X)[0]
                minus = md.jacobians(td.K_TRI, pd.exp_map(-x[:3]) @ Ri, ti - x[3:], X)[0]
                Hba[:, k] = (plus - minus) / (2 * h)
            Hc = md.jacobians(td.K_TRI, Ri, ti, X)[2]
            want, got = Hba @ P_ba @ Hba.T, Hc @ P_pose @ Hc.T
            assert np.linalg.norm(got - want) <= 1e-6 * np.linalg.norm(want)
            assert np.linalg.norm(got - Hc @ P_ba @ Hc.T) > 1e-3 * np.linalg.norm(want)  # the chart matters


def status_cases():
    """Purpose-built points, each (name, Ks, Rs, ts, m, max_err, status): two side-by-side cameras 1 m apart looking
    along +z, and two 1 cm apart for a far point."""
    K = td.K_TRI
    R = np.eye(3)
    t2 = [np.array([0.5, 0.0, 0.0]), np.array([-0.5, 0.0, 0.0])]  # centres at x = -0.5 and +0.5
    X = np.array([0.1, 0.2, 5.0])
    m_good = np.array([md.jacobians(K, R, t, X)[0] for t in t2])
    far = np.array([0.3, 0.1, 60.0])
    t_far = [np.array([0.005, 0.0, 0.0]), np.array([-0.005, 0.0, 0.0])]
    m_far = np.array([md.jacobians(K, R, t, far)[0] for t in t_far])
    same = [np.zeros(3), np.zeros(3)]  # one centre: parallel rays
    m_same = np.array([md.jacobians(K, R, np.zeros(3), X)[0]] * 2)
    diverge = np.array([[640.0 - 80.0, 360.0], [640.0 + 80.0, 360.0]])  # rays that meet behind the cameras
    off = np.array([[0.0, 0.3], [0.0, -0.3]])  # across the (horizontal) epipolar lines: no point explains it
    Ks, Rs = [K, K], [R, R]
    return [
        ("good", Ks, Rs, t2, m_good + off, math.inf, 0),
        ("too far off", Ks, Rs, t2, m_good + off, 0.1, 3),
        ("too uncertain", Ks, Rs, t_far, m_far, math.inf, 2),
        ("too uncertain beats too far off", Ks, Rs, t_far, m_far + off, 0.1, 2),
        ("behind", Ks, Rs, t2, diverge, math.inf, 1),
        ("behind beats too far off", Ks, Rs, t2, diverge, 1e-9, 1),
        ("parallel", Ks, Rs, same, m_same, math.inf, 4),
        ("singular K", [K, np.diag([700.0, 700.0, 0.0])], Rs, t2, m_good, math.inf, 4),
    ]


@pytest.mark.parametrize("case", status_cases(), ids=lambda c: c[0])
def test_statuses_and_their_order(case):
    _, Ks, Rs, ts, m, max_err, want = case
    Sm = [np.eye(2)] * 2
    r = td.triangulate(Ks, Rs, ts, [None, None], m, Sm, max_err)
    assert r["status"] == want, (r["status"], r["stat"])
    if want in (1, 4):
        assert np.isnan(r["X"]).all() and np.isnan(r["P"]).all() and np.isnan(r["stat"]).all()
    else:
        assert np.isfinite(r["X"]).all() and np.isfinite(r["P"]).all() and np.isfinite(r["stat"]).all()
    if want == 2:
        assert r["stat"][3] > 1.0
    if want == 3:
        assert r["stat"][1] >= max_err


def mc_trial(rng, n_views, n_pts=20, with_pc=True):
    """One rig: true poses, estimated poses drawn from each camera's P_c (in the pose chart), true points observed
    through the true poses with noise from Sigma_m (0.5 to 1.5 px); the triangulation sees the estimated poses.
    Returns (K, R, t, Pc, off, cam, m, covm, Xt) in cosl_tri_solver_submit's form, one view per camera per point."""
    Rt, tt = td.rig(rng, n_views)
    Pc = [md.random_spd(rng, 6, 1e-8, 1e-6) for _ in range(n_views)]
    R, t = [], []
    for Ri, ti, P in zip(Rt, tt, Pc):
        d = rng.multivariate_normal(np.zeros(6), P)
        R.append(Ri @ pd.exp_map(d[:3]))
        t.append(ti + d[3:])
    Xt = td.scene_points(rng, n_pts)
    Sm = np.array([[md.random_spd(rng, 2, 0.25, 2.25) for _ in range(n_views)] for _ in range(n_pts)])
    m = np.array([td.observe(td.K_TRI, Rt, tt, X, S, rng) for X, S in zip(Xt, Sm)])
    off = np.arange(n_pts + 1) * n_views
    cam = np.tile(np.arange(n_views), n_pts)
    K = np.array([td.K_TRI] * n_views)
    return K, np.array(R), np.array(t), Pc if with_pc else None, off, cam, m.reshape(-1, 2), Sm.reshape(-1, 2, 2), Xt


def mc_stats(results):
    """(mean NEES of the status-0 points, rejection rate) over a list of (triangulate_all output, Xt)."""
    ne, rej = [], []
    for r, Xt in results:
        ok = r["status"] == 0
        ne.append(md.nees(r["X"][ok], r["P"][ok], Xt[ok]))
        rej.append(~ok)
    return float(np.mean(np.concatenate(ne))), float(np.mean(np.concatenate(rej)))


MC_TRIALS = {2: 60, 3: 40, 8: 20}


def test_monte_carlo():
    """Per view count, rigs of 20 points: the mean NEES of X+ (3 dof) with P_c in R_v sits near 3, and the rejection
    rate at max_err = MC_MAX_ERR px is small.  Dropping P_c from the same draws inflates the NEES: the pose error is
    then unaccounted noise."""
    rng = np.random.default_rng(5500)
    for n_views, trials in MC_TRIALS.items():
        with_pc, without = [], []
        for _ in range(trials):
            K, R, t, Pc, off, cam, m, covm, Xt = mc_trial(rng, n_views)
            with_pc.append((td.triangulate_all(K, R, t, Pc, off, cam, m, covm, max_err=MC_MAX_ERR), Xt))
            without.append((td.triangulate_all(K, R, t, None, off, cam, m, covm, max_err=MC_MAX_ERR), Xt))
        nees, rej = mc_stats(with_pc)
        nees0, rej0 = mc_stats(without)
        print(f"{n_views} views: mean NEES {nees:.3f} (without P_c {nees0:.3f}), rejected {rej:.4f} ({rej0:.4f})")
        assert MC_NEES[0] <= nees <= MC_NEES[1]
        assert MC_REJECT[0] <= rej <= MC_REJECT[1]
        assert nees0 > 1.2 * nees
