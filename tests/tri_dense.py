"""A float64 restatement of the multi-view triangulation of cosl_tri_solver_submit (DESIGN.md 5.5), on top of
pose_mappts_dense's jacobians and camera_point.

Per view v: a camera entry (K, R, t) with an optional 6x6 pose covariance P_c in the chart R' = R exp([w]x),
t' = t + dt, an observation m (px) and its 2x2 covariance Sigma_m (px^2).

    1. X_lin = A^-1 b, A = sum (I - d d^T), b = sum (I - d d^T) C, d = normalize(R^T K^-1 [m; 1]), C = -R^T t;
       parallel rays (smallest relative Cholesky pivot L_kk^2 / A_kk < 1e-12): status 4;
    2. R_v = Sigma_m + H_c(X_lin) P_c H_c(X_lin)^T, fixed; not positive definite: status 4;
    3. from X_lin in front of every camera, at most 10 Gauss-Newton steps s = N^-1 sum H_X^T R_v^-1 nu_v on
       f(X) = sum nu_v^T R_v^-1 nu_v, each taken when f drops (the change formed from differences) and every depth
       stays > 0, else halved at most 4 times, stopped at |s| <= 1e-12 max(1, |X|) or when N is not positive
       definite (a smallest relative Cholesky pivot below 1e-12, as for A);
    4. P = N(X+)^-1; N not positive definite: status 4;
    5. stat = f(X+), e_max = max |nu_v|, parallax = the largest angle between two rays X+ -> C_v, and
       rho = sqrt(trace P) / |X+ - C_last|;
    6. status 4 degenerate, 1 behind a camera at X_lin or X+, 2 rho > 1, 3 e_max >= max_err, else 0; X, P, stat NaN
       for 1 and 4.

The inverses are numpy.linalg's, so they share no arithmetic with the kernel's closed forms.

    linear(Ks, Rs, ts, m)                                   -> X_lin or None (parallel rays)
    noise(Ks, Rs, ts, Pcs, X, Sm)                           -> [n, 2, 2] R_v
    triangulate(Ks, Rs, ts, Pcs, m, Sm, max_err)            -> dict of X, P, stat, status, X_lin, steps
    triangulate_all(K, R, t, cam_cov, off, cam, m, covm, pixel_var, max_err) -> the device's outputs over every point
    ba_to_pose_chart(R, P)                                  -> blockdiag(R^T, I) P blockdiag(R, I)"""
import math

import numpy as np

import pose_mappts_dense as md

MAX_ITER = 10
HALVINGS = 4
MIN_PIVOT = 1e-12


def centre(R, t):
    return -np.asarray(R, np.float64).reshape(3, 3).T @ np.asarray(t, np.float64).reshape(3)


def positive_definite(A):
    """Cholesky succeeds with a smallest relative pivot L_kk^2 / A_kk of at least MIN_PIVOT: the test of every 3x3 the
    stage factors.  A point running off to infinity leaves N singular to roundoff, where a plain Cholesky may pass."""
    try:
        L = np.linalg.cholesky(A)
    except np.linalg.LinAlgError:
        return False
    return bool(np.min(np.diag(L) ** 2 / np.diag(A)) >= MIN_PIVOT)


def linear(Ks, Rs, ts, m):
    """The point closest to every ray, or None when the rays are parallel (or a K is singular)."""
    A, b = np.zeros((3, 3)), np.zeros(3)
    for K, R, t, mv in zip(Ks, Rs, ts, m):
        R = np.asarray(R, np.float64).reshape(3, 3)
        try:
            x = np.linalg.solve(np.asarray(K, np.float64).reshape(3, 3), np.array([mv[0], mv[1], 1.0]))
        except np.linalg.LinAlgError:
            return None
        d = R.T @ x
        d = d / np.linalg.norm(d)
        Q = np.eye(3) - np.outer(d, d)
        A += Q
        b += Q @ centre(R, t)
    if not positive_definite(A):
        return None
    return np.linalg.solve(A, b)


def noise(Ks, Rs, ts, Pcs, X, Sm):
    """R_v = Sigma_m + H_c(X) P_c H_c(X)^T per view (Sigma_m where P_c is None)."""
    out = []
    for K, R, t, Pc, S in zip(Ks, Rs, ts, Pcs, Sm):
        Rv = np.array(S, np.float64).reshape(2, 2)
        if Pc is not None:
            Hc = md.jacobians(K, R, t, X)[2]
            Rv = Rv + Hc @ np.asarray(Pc, np.float64).reshape(6, 6) @ Hc.T
        out.append(Rv)
    return np.array(out)


def _views(Ks, Rs, ts, X):
    """(pi [n, 2], H_X [n, 2, 3], depth [n]) at X."""
    js = [md.jacobians(K, R, t, X) for K, R, t in zip(Ks, Rs, ts)]
    return np.array([j[0] for j in js]), np.array([j[1] for j in js]), np.array([j[3] for j in js])


def descent(Ks, Rs, ts, Wi, m, X, s):
    """f(X + s) - f(X) = -sum dpi^T R_v^-1 (2 nu - dpi), dpi = (dx_{0,1} - pi dx_2) / (x_2 + dx_2), dx = K R s."""
    df = 0.0
    for K, R, t, W, mv in zip(Ks, Rs, ts, Wi, m):
        K, R = np.asarray(K, np.float64).reshape(3, 3), np.asarray(R, np.float64).reshape(3, 3)
        x = K @ md.camera_point(R, t, X)
        dx = K @ (R @ s)
        p = x[:2] / x[2]
        dpi = (dx[:2] - p * dx[2]) / (x[2] + dx[2])
        df -= float(dpi @ W @ (2.0 * (mv - p) - dpi))
    return df


def _nan(status, X_lin=None, steps=0):
    return dict(X=np.full(3, math.nan), P=np.full((3, 3), math.nan), stat=np.full(4, math.nan), status=status,
                X_lin=X_lin, steps=steps)


def triangulate(Ks, Rs, ts, Pcs, m, Sm, max_err=math.inf):
    """One point from its n views; the last view is the one rho measures the distance to."""
    m = np.asarray(m, np.float64).reshape(-1, 2)
    with np.errstate(all="ignore"):
        X = linear(Ks, Rs, ts, m)
        if X is None or not np.isfinite(X).all():
            return _nan(4)
        X_lin = X.copy()
        Rv = noise(Ks, Rs, ts, Pcs, X, Sm)
        try:
            for S in Rv:
                if not np.isfinite(S).all():
                    return _nan(4, X_lin)
                np.linalg.cholesky(S)
        except np.linalg.LinAlgError:
            return _nan(4, X_lin)
        Wi = np.linalg.inv(Rv)
        behind = not (_views(Ks, Rs, ts, X)[2] > 0).all()
        steps = 0
        for _ in range(0 if behind else MAX_ITER):
            p, H, _ = _views(Ks, Rs, ts, X)
            nu = m - p
            N = np.einsum("via,vij,vjb->ab", H, Wi, H)
            g = np.einsum("via,vij,vj->a", H, Wi, nu)
            if not positive_definite(N):
                break
            s = np.linalg.solve(N, g)
            taken = False
            for h in range(HALVINGS + 1):
                if h:
                    s = s * 0.5
                Xn = X + s
                front = all(md.camera_point(R, t, Xn)[2] > 0 for R, t in zip(Rs, ts))
                if front and descent(Ks, Rs, ts, Wi, m, X, s) < 0:
                    taken = True
                    break
            if not taken:
                break
            X = Xn
            steps += 1
            if math.sqrt(s @ s) <= 1e-12 * max(1.0, math.sqrt(X @ X)):
                break
        p, H, z = _views(Ks, Rs, ts, X)
        behind = behind or not (z > 0).all()
        nu = m - p
        f = float(np.einsum("vi,vij,vj->", nu, Wi, nu))
        e_max = float(np.max(np.linalg.norm(nu, axis=1)))
        N = np.einsum("via,vij,vjb->ab", H, Wi, H)
        if not positive_definite(N):
            return _nan(4, X_lin, steps)
        P = np.linalg.inv(N)
        P = 0.5 * (P + P.T)
        u = np.array([centre(R, t) - X for R, t in zip(Rs, ts)])
        dist = np.linalg.norm(u, axis=1)
        u = u / dist[:, None]
        par = 0.0
        for a in range(len(u)):
            for b in range(a):
                par = max(par, math.atan2(np.linalg.norm(np.cross(u[a], u[b])), float(u[a] @ u[b])))
        rho = math.sqrt(np.trace(P)) / dist[-1]
        stat = np.array([f, e_max, par, rho])
        if not (np.isfinite(X).all() and np.isfinite(P).all() and np.isfinite(stat).all()):
            return _nan(4, X_lin, steps)
        if behind:
            return _nan(1, X_lin, steps)
        status = 2 if rho > 1.0 else 3 if e_max >= max_err else 0
        return dict(X=X, P=P, stat=stat, status=status, X_lin=X_lin, steps=steps)


def triangulate_all(K, R, t, cam_cov, off, cam, m, covm=None, pixel_var=1.0, max_err=math.inf):
    """triangulate over every point of a submit in cosl_tri_solver_submit's form; a dict of stacked arrays."""
    K, R = np.asarray(K, np.float64).reshape(-1, 3, 3), np.asarray(R, np.float64).reshape(-1, 3, 3)
    t = np.asarray(t, np.float64).reshape(-1, 3)
    m = np.asarray(m, np.float64).reshape(-1, 2)
    Sm = (np.broadcast_to(pixel_var * np.eye(2), (len(m), 2, 2)) if covm is None
          else np.asarray(covm, np.float64).reshape(-1, 2, 2))
    Pc = [None] * len(K) if cam_cov is None else [None if P is None else 0.5 * (np.reshape(P, (6, 6)) +
                                                                             np.reshape(P, (6, 6)).T)
                                                   for P in cam_cov]
    rs = []
    for j in range(len(off) - 1):
        v = np.arange(off[j], off[j + 1])
        c = np.asarray(cam)[v]
        rs.append(triangulate(K[c], R[c], t[c], [Pc[i] for i in c], m[v], Sm[v], max_err))
    return dict(X=np.array([r["X"] for r in rs]).reshape(-1, 3), P=np.array([r["P"] for r in rs]).reshape(-1, 3, 3),
                stat=np.array([r["stat"] for r in rs]).reshape(-1, 4),
                status=np.array([r["status"] for r in rs], np.int32))


def ba_to_pose_chart(R, P):
    """A BA camCov (chart exp([w]x) R) in the pose solver's chart R exp([w]x): blockdiag(R^T, I) P blockdiag(R, I)."""
    D = np.eye(6)
    D[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    return D.T @ np.asarray(P, np.float64).reshape(6, 6) @ D


# ---------------------------------------------------------------- scenes
K_TRI = np.array([[700.0, 0.0, 640.0], [0.0, 700.0, 360.0], [0.0, 0.0, 1.0]])
W_TRI, H_TRI = 1280, 720


def look_at(C, target, rng=None, roll=0.0):
    """(R, t) of a camera at centre C looking at target (world to camera)."""
    C, target = np.asarray(C, np.float64), np.asarray(target, np.float64)
    z = target - C
    z = z / np.linalg.norm(z)
    up = np.array([0.0, -1.0, 0.0]) + (rng.normal(0.0, 0.05, 3) if rng is not None else 0.0)
    x = np.cross(up, z)
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    if roll:
        c, s = math.cos(roll), math.sin(roll)
        R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]) @ R
    return R, -R @ C


def rig(rng, n_cams, spread=1.0, centre_at=(0.0, 0.0, 6.0)):
    """n_cams camera entries spread over a spread-wide patch around the origin, looking at centre_at."""
    Cs = np.column_stack([rng.uniform(-spread, spread, n_cams), rng.uniform(-0.3 * spread, 0.3 * spread, n_cams),
                          rng.uniform(-0.2, 0.2, n_cams)])
    Rt = [look_at(C, np.asarray(centre_at) + rng.normal(0.0, 0.3, 3), rng) for C in Cs]
    return np.array([r[0] for r in Rt]), np.array([r[1] for r in Rt])


def scene_points(rng, n, lo=(-2.0, -1.2, 4.0), hi=(2.0, 1.2, 9.0)):
    return rng.uniform(lo, hi, (n, 3))


def observe(K, R, t, X, Sm, rng):
    """The projection of X in each camera plus noise drawn from Sm [n, 2, 2]."""
    p = np.array([md.jacobians(K, Ri, ti, X)[0] for Ri, ti in zip(R, t)])
    return p + np.array([rng.multivariate_normal(np.zeros(2), S) for S in Sm])


def chain_trial(rng, n_solve=30, n_map=20, n_frames=4):
    """One camera over n_frames frames for the chain of triangulation and map-point update: frames 0 and 1 are the
    key frames the points are triangulated from, the later ones update them.  The camera moves sideways 0.4 m per
    frame and turns a little.  Per frame: the true pose, a start pose near it, n_solve points observed at 1 px for the
    pose solve, and the n_map true map points observed with noise from Sigma_m (0.5 to 1.5 px)."""
    R1, t1 = md.pd.exp_map(rng.normal(0.0, 0.2, 3)), rng.normal(0.0, 0.5, 3)
    C1 = centre(R1, t1)
    Xt = md.view_points(md.K_MC, R1, t1, rng, n_map, md.W_MC, md.H_MC, 3.0, 10.0)
    frames = []
    for k in range(n_frames):
        Rk = R1 @ md.pd.exp_map(rng.normal(0.0, 0.02, 3))
        tk = -Rk @ (C1 + R1.T @ np.array([0.4 * k, 0.05 * k, 0.0]))
        R0, t0 = Rk @ md.pd.exp_map(rng.normal(0.0, 0.01, 3)), tk + rng.normal(0.0, 0.02, 3)
        Ms = md.view_points(md.K_MC, Rk, tk, rng, n_solve, md.W_MC, md.H_MC, 3.0, 10.0)
        u, v = md.pd.project(md.K_MC, Rk, tk, Ms)
        ms = np.column_stack([u, v]) + rng.normal(0.0, 1.0, (n_solve, 2))
        Sm = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in range(n_map)])
        u, v = md.pd.project(md.K_MC, Rk, tk, Xt)
        m = np.column_stack([u, v]) + np.array([rng.multivariate_normal(np.zeros(2), S) for S in Sm])
        frames.append(dict(Rt=Rk, tt=tk, R0=R0, t0=t0, Ms=Ms, ms=ms, m=m, Sm=Sm))
    return Xt, frames


def chain_views(n_map):
    """view_off and view_cam of n_map points seen by camera entries 0 (the first key frame) and 1 (the current)."""
    return np.arange(n_map + 1) * 2, np.tile([0, 1], n_map)
