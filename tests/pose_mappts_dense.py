"""A float64 restatement of the map-point update of cosl_pose_solver_submit_mappts (DESIGN.md 5.4), on top of
pose_dense and pose_cov_dense.

Per camera: (R, t) the refined pose and P_c its 6x6 stage covariance in the chart R' = R exp([w]x), t' = t + dt.  Per
map point: mean X0, 3x3 covariance P0 (world), observation m (px) and 2x2 covariance Sigma_m (px^2).

    H_X(X) = d pi / dX = (a; b) R,  H_c(X) = pose_cov_dense's analytic 2x6 Jacobian,
    R_eff = Sigma_m + H_c(X0) P_c H_c(X0)^T,
    gate:   nu0 = m - pi(X0), S0 = H_X P0 H_X^T + R_eff, d2_0 = nu0^T S0^-1 nu0, e0 = |nu0|; updated when d2_0 < gate;
    update: at most 8 Gauss-Newton steps on f(X) = (X - X0)^T P0^-1 (X - X0) + (m - pi(X))^T R_eff^-1 (m - pi(X)) in
            Kalman form, X' = X0 + P0 H^T (H P0 H^T + R_eff)^-1 (m - pi(X) + H (X - X0)), taken only when f drops
            (descent, the change formed from differences) and the depth stays > 0, stopped at |X' - X| <= 1e-12
            max(1, |X'|);
            P+ = (P0^-1 + H_X(X+)^T R_eff^-1 H_X(X+))^-1, symmetrised;
    re-gate: d2_1 = nu1^T (H_X P+ H_X^T + R_eff)^-1 nu1 at X+.

    status 0 updated, 1 gated out, 2 not updatable (depth <= 0 at X0, a non-finite value, S0 not positive definite),
    3 the camera's pose covariance is invalid.

The inverses are numpy.linalg's, so they share no arithmetic with the kernel's closed forms.

    jacobians(K, R, t, X)                     -> (pi(X), H_X, H_c, depth)
    r_eff(K, R, t, X0, Pc, Sm)                -> R_eff
    objective(K, R, t, X, X0, P0, m, Reff)    -> f(X)
    update(K, R, t, Pc, X0, P0, m, Sm, gate)  -> dict of X, P, d2_0, d2_1, e0, status, X1 (the first step), steps
    update_all(...)                           -> update over arrays of points, as the device returns them
    mc_frame(rng), nees(X, P, Xt)             -> one Monte-Carlo frame (truth, solve points, map points), NEES"""
import math

import numpy as np

import pose_cov_dense as cd
import pose_dense as pd

MAX_ITER = 8


def jacobians(K, R, t, X):
    """(pi(X) [2], H_X [2, 3], H_c [2, 6], depth (R X + t)_z)."""
    K, R = np.asarray(K, np.float64).reshape(3, 3), np.asarray(R, np.float64).reshape(3, 3)
    t, X = np.asarray(t, np.float64).reshape(3), np.asarray(X, np.float64).reshape(3)
    c = camera_point(R, t, X)
    x = K @ c
    m = x[:2] / x[2]
    a = (K[0] - m[0] * K[2]) / x[2]
    b = (K[1] - m[1] * K[2]) / x[2]
    HX = np.stack([a, b]) @ R
    Hc = cd.jacobian(K, R, t, X.reshape(1, 3))[0]
    return m, HX, Hc, c[2]


def camera_point(R, t, X):
    """c = R X + t in the kernel's operation order, so that the sign of the depth c_2 is the kernel's."""
    R = np.asarray(R, np.float64).reshape(3, 3)
    return np.array([float(R[i, 0]) * float(X[0]) + float(R[i, 1]) * float(X[1]) + float(R[i, 2]) * float(X[2])
                     + float(t[i]) for i in range(3)])


def centre_point(R, t):
    """A point at the camera centre -R^T t, moved by roundoff until its depth computes to 0 or below."""
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)
    X = -R.T @ t
    for _ in range(64):
        z = camera_point(R, t, X)[2]
        if z <= 0:
            return X
        X = X - R[2] * (2.0 * z)
    raise AssertionError("no point of non-positive depth found at the camera centre")


def r_eff(K, R, t, X0, Pc, Sm):
    _, _, Hc, _ = jacobians(K, R, t, X0)
    return np.asarray(Sm, np.float64).reshape(2, 2) + Hc @ np.asarray(Pc, np.float64).reshape(6, 6) @ Hc.T


def objective(K, R, t, X, X0, P0, m, Reff):
    mX, _, _, _ = jacobians(K, R, t, X)
    d, r = np.asarray(X) - X0, np.asarray(m) - mX
    return float(d @ np.linalg.solve(P0, d) + r @ np.linalg.solve(Reff, r))


def descent(K, R, t, X, X0, P0, Reff, nu, s):
    """f(X + s) - f(X) of the update's objective, from differences: s^T P0^-1 (2 (X - X0) + s) - dpi^T Reff^-1 (2 nu -
    dpi), nu = m - pi(X) and dpi = pi(X + s) - pi(X) = (dx_{0,1} - pi(X) dx_2) / (x_2 + dx_2), dx = K R s.  Near the
    minimum the two objectives agree to their roundoff and their difference would decide a step by noise."""
    K, R = np.asarray(K, np.float64).reshape(3, 3), np.asarray(R, np.float64).reshape(3, 3)
    x = K @ camera_point(R, t, X)
    dx = K @ (R @ s)
    dpi = (dx[:2] - x[:2] / x[2] * dx[2]) / (x[2] + dx[2])
    return float(s @ np.linalg.solve(P0, 2.0 * (X - X0) + s) - dpi @ np.linalg.solve(Reff, 2.0 * nu - dpi))


def posterior_cov(HX, P0, Reff):
    """(P0^-1 + H_X^T R_eff^-1 H_X)^-1, symmetrised."""
    P = np.linalg.inv(np.linalg.inv(P0) + HX.T @ np.linalg.solve(Reff, HX))
    return 0.5 * (P + P.T)


def _unchanged(X0, P0, status, d0, e0):
    return dict(X=np.array(X0, np.float64), P=np.array(P0, np.float64), d2_0=d0, d2_1=math.nan, e0=e0,
                status=status, X1=None, steps=0)


def update(K, R, t, Pc, X0, P0, m, Sm, gate, pose_valid=True):
    """The update of one map point; P0 is symmetrised first, as the device stages it."""
    X0 = np.asarray(X0, np.float64).reshape(3)
    P0 = np.asarray(P0, np.float64).reshape(3, 3)
    P0 = 0.5 * (P0 + P0.T)
    m = np.asarray(m, np.float64).reshape(2)
    m0, HX, Hc, z0 = jacobians(K, R, t, X0)
    nu = m - m0
    e0 = math.sqrt(nu @ nu)
    if not pose_valid:
        return _unchanged(X0, P0, 3, math.nan, e0)
    if not (z0 > 0) or not np.isfinite(m0).all():
        return _unchanged(X0, P0, 2, math.nan, e0)
    Reff = np.asarray(Sm, np.float64).reshape(2, 2) + Hc @ np.asarray(Pc, np.float64).reshape(6, 6) @ Hc.T
    S0 = HX @ P0 @ HX.T + Reff
    try:
        np.linalg.cholesky(S0)
        np.linalg.cholesky(Reff)
        np.linalg.cholesky(P0)
    except np.linalg.LinAlgError:
        return _unchanged(X0, P0, 2, math.nan, e0)
    d0 = float(nu @ np.linalg.solve(S0, nu))
    if not math.isfinite(d0):
        return _unchanged(X0, P0, 2, math.nan, e0)
    if not d0 < gate:
        return _unchanged(X0, P0, 1, d0, e0)
    X, H, r = X0.copy(), HX, nu
    X1, steps = None, 0
    for _ in range(MAX_ITER):
        U = P0 @ H.T
        Xn = X0 + U @ np.linalg.solve(H @ U + Reff, r + H @ (X - X0))
        if X1 is None:
            X1 = Xn.copy()
        mn, Hn, _, zn = jacobians(K, R, t, Xn)
        if not zn > 0:
            break
        step = Xn - X
        if not descent(K, R, t, X, X0, P0, Reff, r, step) < 0:
            break
        X, H, r = Xn, Hn, m - mn
        steps += 1
        if math.sqrt(step @ step) <= 1e-12 * max(1.0, math.sqrt(X @ X)):
            break
    P = posterior_cov(H, P0, Reff)
    d1 = float(r @ np.linalg.solve(H @ P @ H.T + Reff, r))
    if not (np.isfinite(X).all() and np.isfinite(P).all() and math.isfinite(d1)):
        return _unchanged(X0, P0, 2, math.nan, e0)
    return dict(X=X, P=P, d2_0=d0, d2_1=d1, e0=e0, status=0, X1=X1, steps=steps)


def update_all(K, R, t, Pc, X0, P0, m, Sm, gate, pose_valid=True):
    """update over n points: X0 [n, 3], P0 [n, 3, 3], m [n, 2], Sm [n, 2, 2]; a dict of stacked arrays."""
    rs = [update(K, R, t, Pc, X0[i], P0[i], m[i], Sm[i], gate, pose_valid) for i in range(len(X0))]
    return dict(X=np.array([r["X"] for r in rs]).reshape(-1, 3), P=np.array([r["P"] for r in rs]).reshape(-1, 3, 3),
                d2_0=np.array([r["d2_0"] for r in rs]), d2_1=np.array([r["d2_1"] for r in rs]),
                e0=np.array([r["e0"] for r in rs]), status=np.array([r["status"] for r in rs], np.int32))


def random_spd(rng, n, lo, hi):
    """A random n x n covariance with eigenvalues spread geometrically over [lo, hi]."""
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    P = (Q * np.geomspace(hi, lo, n)) @ Q.T
    return 0.5 * (P + P.T)


def view_points(K, R, t, rng, n, W=1280, H=720, zmin=3.0, zmax=10.0):
    """n world points whose projections are uniform over a W x H image at depths zmin to zmax."""
    K, R = np.asarray(K, np.float64).reshape(3, 3), np.asarray(R, np.float64).reshape(3, 3)
    uv = rng.uniform([0.0, 0.0], [W, H], (n, 2))
    z = rng.uniform(zmin, zmax, n)
    Xc = np.linalg.solve(K, np.column_stack([uv, np.ones(n)]).T).T * z[:, None]
    return (Xc - np.asarray(t)) @ R


def pose_gn(K, R, t, Ms, ms, iters=6):
    """Gauss-Newton on the unweighted reprojection error in the solver's chart: the pose of a noisy solve."""
    R, t = np.array(R, np.float64).reshape(3, 3), np.array(t, np.float64).reshape(3)
    K = np.asarray(K, np.float64).reshape(3, 3)
    for _ in range(iters):
        u, v = pd.project(K, R, t, Ms)
        r = np.column_stack([ms[:, 0] - u, ms[:, 1] - v]).ravel()
        J = cd.jacobian(K, R, t, Ms).reshape(-1, 6)
        x = np.linalg.lstsq(J, r, rcond=None)[0]
        R, t = R @ pd.exp_map(x[:3]), t + x[3:]
    return R, t


# ---------------------------------------------------------------- Monte-Carlo frames
K_MC = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
W_MC, H_MC = 640, 480
TAU_MC = 1e3  # far beyond 1 px noise: every weight of the solve is 1 to 1e-6
GATE_95 = 5.991464547107979  # the 95 % quantile of chi-square with 2 dof


def mc_frame(rng, n_solve=30, n_map=20):
    """One frame: a random true pose (Rt, tt) and a start pose near it; n_solve points observed with 1 px noise for
    the pose solve; n_map true map points Xt with a prior mean X0 drawn from a random P0 (standard deviations 1 to 10
    cm), and their observations m drawn from a random Sigma_m (standard deviations 0.5 to 1.5 px)."""
    Rt = pd.exp_map(rng.normal(0.0, 0.2, 3))
    tt = rng.normal(0.0, 0.5, 3)
    R0, t0 = Rt @ pd.exp_map(rng.normal(0.0, 0.01, 3)), tt + rng.normal(0.0, 0.02, 3)
    Ms = view_points(K_MC, Rt, tt, rng, n_solve, W_MC, H_MC, 3.0, 10.0)
    u, v = pd.project(K_MC, Rt, tt, Ms)
    ms = np.column_stack([u, v]) + rng.normal(0.0, 1.0, (n_solve, 2))
    Xt = view_points(K_MC, Rt, tt, rng, n_map, W_MC, H_MC, 3.0, 10.0)
    P0 = np.array([random_spd(rng, 3, 1e-4, 1e-2) for _ in range(n_map)])
    X0 = np.array([rng.multivariate_normal(Xt[i], P0[i]) for i in range(n_map)])
    Sm = np.array([random_spd(rng, 2, 0.25, 2.25) for _ in range(n_map)])
    u, v = pd.project(K_MC, Rt, tt, Xt)
    m = np.column_stack([u, v]) + np.array([rng.multivariate_normal(np.zeros(2), Sm[i]) for i in range(n_map)])
    return dict(Rt=Rt, tt=tt, R0=R0, t0=t0, Ms=Ms, ms=ms, Xt=Xt, X0=X0, P0=P0, m=m, Sm=Sm)


def nees(X, P, Xt):
    """(X - Xt)^T P^-1 (X - Xt) per point."""
    d = np.asarray(X) - np.asarray(Xt)
    return np.einsum("ni,ni->n", d, np.linalg.solve(P, d[..., None])[..., 0])
