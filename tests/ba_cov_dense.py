"""float64 references for the marginal covariances of a bundle adjustment (cosl_ba_solver_download_covariance).

At the parameters of a problem, with Tukey weights w evaluated there (free points with fewer than two observations
of non-zero weight are left out, their weights set to 0), H = sum w J^T J over the free parameters, and the
covariance is pixel_var H^-1.  The camera chart is (w, t): R' = exp([w]x) R, t' = t + dt.

Three restatements that must agree with each other:
  - cov_full: the inverse of the whole H, J from ba_dense.local_jacobian (complex steps in the solver's local
    rotation v at v = 0, where R(q(v)) = exp([2 v]x) to first order: dx/dw = dx/dv / 2, so Sigma_w = 4 Sigma_v);
  - cov_full(jac=expmap_jacobian): the same with J by complex steps straight through exp([w]x) (Rodrigues);
  - cov_schur: the Schur form the device computes (reduced camera system S = U - W V^-1 W^T, Z = S^-1, point blocks
    V^-1 + V^-1 (sum W^T Z W) V^-1), with S dense and the points one by one."""
import numpy as np

from ba_dense import (H_CS, K_of, _finish, cancellation, layout, local_jacobian, point_of, residuals, rot,
                      tukey_weights)


def weights(prob, max_err):
    """(residuals e [N, 2], effective weights w [N], unconstrained-point mask [n])."""
    e = residuals(prob)
    w = tukey_weights(np.sqrt((e * e).sum(1)), max_err)
    pt = point_of(prob)
    cnt = np.bincount(pt[w > 0], minlength=prob.n)
    unc = (np.arange(prob.n) >= prob.n_con) & (cnt < 2)
    return e, np.where(unc[pt], 0.0, w), unc


def omega_jacobian(prob):
    """d xhat / d (w, t, X) [N, 2, 9] from the solver-chart Jacobian at v = 0."""
    J = local_jacobian(prob)
    J[:, :, :3] *= 0.5
    return J


def expmap_jacobian(prob):
    """d xhat / d (w, t, X) [N, 2, 9] by complex steps through R' = exp([w]x) R, t + dt, X + dX."""
    pt, cam = point_of(prob), prob.cam
    R = prob.R.reshape(-1, 3, 3)[cam]
    K = prob.K.reshape(-1, 3, 3)[cam]
    N = prob.nobs
    J = np.empty((N, 2, 9))
    for k in range(9):
        d = np.zeros((N, 3), np.complex128)
        d[:, k % 3] = 1j * H_CS
        Rk = R.astype(np.complex128)
        if k < 3:  # exp([w]x) = I + A [w]x + B [w]x^2, A = sin th / th, B = (1 - cos th) / th^2 (series: th ~ 1e-30)
            th2 = (d * d).sum(1)
            A = 1 - th2 / 6 + th2 * th2 / 120
            B = 0.5 - th2 / 24 + th2 * th2 / 720
            W = np.zeros((N, 3, 3), np.complex128)
            W[:, 0, 1], W[:, 0, 2], W[:, 1, 2] = -d[:, 2], d[:, 1], -d[:, 0]
            W[:, 1, 0], W[:, 2, 0], W[:, 2, 1] = d[:, 2], -d[:, 1], d[:, 0]
            E = np.eye(3)[None] + A[:, None, None] * W + B[:, None, None] * (W @ W)
            Rk = E @ Rk
        X = prob.X[pt] + (d if k >= 6 else 0)
        P = np.einsum("nij,nj->ni", Rk, X) + prob.t[cam] + (d if 3 <= k < 6 else 0)
        u = np.einsum("nij,nj->ni", K, P)
        J[:, :, k] = (u[:, :2] / u[:, 2:3]).imag / H_CS
    return J


def _blocks(prob, C, cols_cam, cols_pt, unc):
    m, n, mcon, ncon = prob.m, prob.n, prob.m_con, prob.n_con
    cam = np.zeros((m, 6, 6))
    pt = np.zeros((n, 3, 3))
    for j in range(mcon, m):
        c = cols_cam[j]
        cam[j] = C[np.ix_(c, c)]
    for i in range(ncon, n):
        if unc[i]:
            pt[i] = np.nan
        else:
            c = cols_pt[i]
            pt[i] = C[np.ix_(c, c)]
    return cam, pt


def _info(prob, e, w, unc, pixel_var):
    mf = prob.m - prob.m_con
    npts = int(((np.arange(prob.n) >= prob.n_con) & ~unc).sum())
    dof = 2 * int((w > 0).sum()) - 6 * mf - 3 * npts
    s2 = float((w * (e * e).sum(1)).sum()) / dof if dof > 0 else np.nan
    return {"pixel_var": pixel_var, "sigma2_hat": s2, "dof": dof, "unconstrained": int(unc.sum())}


def cov_full(prob, max_err, pixel_var, jac=omega_jacobian):
    """(camCov [m, 6, 6], ptCov [n, 3, 3], info, H) from the inverse of the whole information matrix."""
    e, w, unc = weights(prob, max_err)
    J = jac(prob) * np.sqrt(w)[:, None, None]
    cols, _ = layout(prob)
    mf = prob.m - prob.m_con
    # parameters: free cameras, then the free points that stay in H
    keep_pts = [i for i in range(prob.n_con, prob.n) if not unc[i]]
    pos = {i: 6 * mf + 3 * k for k, i in enumerate(keep_pts)}
    npar = 6 * mf + 3 * len(keep_pts)
    pt_of = point_of(prob)
    c9 = np.full((prob.nobs, 9), -1, np.int64)
    c9[:, :6] = cols[:, :6]
    for o in range(prob.nobs):
        i = pt_of[o]
        if i in pos:
            c9[o, 6:] = pos[i] + np.arange(3)
    H = np.zeros((npar, npar))
    for o in range(prob.nobs):
        c = c9[o]
        ok = c >= 0
        Jo = J[o][:, ok]
        H[np.ix_(c[ok], c[ok])] += Jo.T @ Jo
    C = pixel_var * np.linalg.inv(H)
    cols_cam = {j: 6 * (j - prob.m_con) + np.arange(6) for j in range(prob.m_con, prob.m)}
    cols_pt = {i: pos[i] + np.arange(3) for i in keep_pts}
    cam, pt = _blocks(prob, C, cols_cam, cols_pt, unc)
    return cam, pt, _info(prob, e, w, unc, pixel_var), H


def cov_schur(prob, max_err, pixel_var):
    """(camCov, ptCov, info) by the Schur form: S dense, points one at a time."""
    e, w, unc = weights(prob, max_err)
    J = omega_jacobian(prob) * np.sqrt(w)[:, None, None]
    A, B = J[:, :, :6], J[:, :, 6:]
    m, n, mcon, ncon = prob.m, prob.n, prob.m_con, prob.n_con
    mf = m - mcon
    pt_of, cam_of = point_of(prob), prob.cam
    S = np.zeros((6 * mf, 6 * mf))
    for o in range(prob.nobs):
        j = cam_of[o] - mcon
        if j >= 0:
            S[6 * j:6 * j + 6, 6 * j:6 * j + 6] += A[o].T @ A[o]
    Vinv, Ws = {}, {}
    for i in range(ncon, n):
        if unc[i]:
            continue
        obs = np.arange(prob.ptr[i], prob.ptr[i + 1])
        V = sum(B[o].T @ B[o] for o in obs)
        Vinv[i] = np.linalg.inv(V)
        Ws[i] = [(cam_of[o] - mcon, A[o].T @ B[o]) for o in obs if cam_of[o] >= mcon]
        for ja, Wa in Ws[i]:
            for jb, Wb in Ws[i]:
                S[6 * ja:6 * ja + 6, 6 * jb:6 * jb + 6] -= Wa @ Vinv[i] @ Wb.T
    Z = np.linalg.inv(S) if mf else np.zeros((0, 0))
    cam = np.zeros((m, 6, 6))
    for j in range(mf):
        cam[mcon + j] = pixel_var * Z[6 * j:6 * j + 6, 6 * j:6 * j + 6]
    pt = np.zeros((n, 3, 3))
    for i in range(ncon, n):
        if unc[i]:
            pt[i] = np.nan
            continue
        T = np.zeros((3, 3))
        for ja, Wa in Ws[i]:
            for jb, Wb in Ws[i]:
                T += Wa.T @ Z[6 * ja:6 * ja + 6, 6 * jb:6 * jb + 6] @ Wb
        pt[i] = pixel_var * (Vinv[i] + Vinv[i] @ T @ Vinv[i])
    return cam, pt, _info(prob, e, w, unc, pixel_var)


def block_errors(got, want):
    """Per block |got - want|_F / |want|_F over the blocks with a non-zero finite reference; the NaN and zero
    blocks must match exactly (returned as a bool)."""
    got, want = np.asarray(got), np.asarray(want)
    nan_w = np.isnan(want).all(axis=(1, 2))
    zero_w = (want == 0).all(axis=(1, 2))
    same = bool(np.array_equal(np.isnan(got).all(axis=(1, 2)), nan_w) and (got[zero_w] == 0).all()
                and not np.isnan(got[~nan_w]).any())
    live = ~nan_w & ~zero_w
    nw = np.linalg.norm(want[live], axis=(1, 2))
    err = np.linalg.norm(got[live] - want[live], axis=(1, 2)) / nw
    return err, same


def far_tolerance(prob, H, base=1e-8):
    """base, widened on scenes whose camera-frame points cancel in float64 (ba_dense.cancellation): the device's
    J carries a relative error up to rho per entry, H then 2 rho, and H^-1 kappa(H) times that."""
    rho, _ = cancellation(prob)
    return base + 2.0 * float(np.linalg.cond(H)) * float(rho.max())


# ---------------------------------------------------------------- scenes
def banded(seed=21, m=84, span=4, per_start=10):
    """m cameras 0.25 m apart along x (looking along z); every point is seen by `span` consecutive cameras, so
    the reduced camera system is banded: the plan dissects it (ND depth >= 1) into more than two blocks.  The two
    fixed cameras (indices 0 and 1) sit at the two ends of the row, so that the chain between them is pinned at
    both ends; the free cameras 2 .. m-1 follow each other along it."""
    rng = np.random.default_rng(seed)
    at = [0, m - 1] + list(range(1, m - 1))  # camera index -> position along the row
    cam_at = np.argsort(at)
    K = np.tile(K_of(500.0, 1.0, 0.0, 320.0, 240.0), (m, 1))
    R = np.array([rot([0, 1, 0], 3.0 * np.sin(0.2 * at[j])) @ rot([1, 0, 0], 1.0 * np.cos(0.3 * at[j]))
                  for j in range(m)])
    C = np.array([[0.25 * at[j], 0.02 * np.sin(at[j]), 0.0] for j in range(m)])
    t = -np.einsum("jab,jb->ja", R, C)
    X, vis = [], []
    for j0 in range(m - span + 1):
        for _ in range(per_start):
            X.append([0.25 * (j0 + (span - 1) / 2) + rng.uniform(-0.3, 0.3), rng.uniform(-1.0, 1.0),
                      rng.uniform(4.0, 7.0)])
            vis.append(sorted(int(c) for c in cam_at[j0:j0 + span]))
    return _finish(K, R, t, np.array(X), vis, 2, 3, rng, sizes=[(640, 480)] * m)


def small_nonrobust(seed=31):
    """6 cameras (2 fixed: they pin the scale), 60 points seen by 3-6 cameras, noise-free observations: the
    truth for a Monte-Carlo check of the covariance."""
    rng = np.random.default_rng(seed)
    m = 6
    K = np.tile(K_of(600.0, 1.0, 0.0, 320.0, 240.0), (m, 1))
    R = np.array([rot([0, 1, 0], -6.0 + 2.5 * j) for j in range(m)])
    C = np.array([[0.3 * j - 0.75, 0.05 * (j % 2), 0.0] for j in range(m)])
    t = -np.einsum("jab,jb->ja", R, C)
    X, vis = [], []
    while len(X) < 60:
        x = np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.0, 1.0), rng.uniform(4.0, 7.0)])
        v = sorted(rng.choice(m, size=int(rng.integers(3, m + 1)), replace=False).tolist())
        X.append(x)
        vis.append(v)
    return _finish(K, R, t, np.array(X), vis, 2, 0, rng, noise=0.0, dR=0.0, dt=0.0, dX=0.0)


def long_tracks_seen(seed=14):
    """ba_dense.long_tracks, whose last camera has a single observation (its H is singular: 2 equations for 6
    parameters), with four more points that the last camera and its two neighbours see: well posed."""
    from ba_dense import long_tracks, project
    from coslam_b200.problem import BAProblem
    base = long_tracks(seed)
    rng = np.random.default_rng(seed + 100)
    m, last = base.m, base.m - 1
    R = base.R.reshape(-1, 3, 3)[last]
    Cl = -R.T @ base.t[last]
    newX = [Cl + R.T @ np.array([rng.uniform(-1, 1), rng.uniform(-0.7, 0.7), rng.uniform(6, 8)]) for _ in range(4)]
    vis = [[last - 2, last - 1, last]] * 4
    cam = np.concatenate([base.cam] + [np.asarray(v, np.int32) for v in vis])
    X = np.concatenate([base.X, np.array(newX)])
    ptr = np.concatenate([base.ptr, base.ptr[-1] + 3 * np.arange(1, 5)])
    tmp = BAProblem(base.K.copy(), base.R, base.t, X, ptr, cam, np.zeros((len(cam), 2)), base.m_con, base.n_con)
    xy = project(tmp)[0]
    xy[:base.nobs] = base.xy
    xy[base.nobs:] += rng.normal(0, 0.3, (12, 2))
    assert m == tmp.m
    return BAProblem(base.K.copy(), base.R, base.t, X, ptr, cam, xy, base.m_con, base.n_con)


# the scenes of ba_dense.ROWS that have a covariance (long_tracks replaced by its well-posed variant)
def cov_rows():
    import ba_dense as bd
    rows = {k: v for k, v in bd.ROWS.items() if k != "long_tracks"}
    rows["long_tracks_seen"] = (long_tracks_seen, bd.MAX_ERR)
    return rows


def make(name):
    import ba_dense as bd
    f, max_err = cov_rows()[name]
    return f(), bd.options(max_err)
