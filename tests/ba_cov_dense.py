"""float64 references for the marginal covariances of a bundle adjustment (cosl_ba_solver_download_covariance).

At the parameters of a problem, with Tukey weights w evaluated there (free points with fewer than two observations
of non-zero weight are left out, their weights set to 0), H = sum w J^T J over the free parameters, and the
covariance is pixel_var H^-1.  The camera chart is (w, t): R' = exp([w]x) R, t' = t + dt.

Three restatements that must agree with each other:
  - cov_full: the inverse of the whole H, J from ba_dense.local_jacobian (complex steps in the solver's local
    rotation v at v = 0, where R(q(v)) = exp([2 v]x) to first order: dx/dw = dx/dv / 2, so Sigma_w = 4 Sigma_v);
  - cov_full(jac=expmap_jacobian): the same with J by complex steps straight through exp([w]x) (Rodrigues);
  - cov_schur: the Schur form the device computes (reduced camera system S = U - W V^-1 W^T, Z = S^-1, point blocks
    V^-1 + V^-1 (sum W^T Z W) V^-1), with S dense and the points' terms batched over observations."""
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


def _pairs(prob, keep):
    """(oa, ob): every ordered pair of observations of one point that has keep[point], both by free cameras."""
    cnt = np.diff(prob.ptr)
    oa, ob = [], []
    for da in range(int(cnt.max(initial=0))):
        for db in range(int(cnt.max(initial=0))):
            i = np.nonzero(keep & (cnt > max(da, db)))[0]
            a, b = prob.ptr[i] + da, prob.ptr[i] + db
            free = (prob.cam[a] >= prob.m_con) & (prob.cam[b] >= prob.m_con)
            oa.append(a[free])
            ob.append(b[free])
    return np.concatenate(oa).astype(np.int64), np.concatenate(ob).astype(np.int64)


def cov_schur(prob, max_err, pixel_var):
    """(camCov, ptCov, info) by the Schur form: S dense, the points' V, W and T batched over observations."""
    e, w, unc = weights(prob, max_err)
    J = omega_jacobian(prob) * np.sqrt(w)[:, None, None]
    A, B = J[:, :, :6], J[:, :, 6:]
    m, n, mcon, ncon = prob.m, prob.n, prob.m_con, prob.n_con
    mf = m - mcon
    pt_of, cam_of = point_of(prob), prob.cam
    keep = (np.arange(n) >= ncon) & ~unc
    Sb = np.zeros((mf, mf, 6, 6))
    fo = np.nonzero(cam_of >= mcon)[0]
    np.add.at(Sb, (cam_of[fo] - mcon, cam_of[fo] - mcon), np.einsum("nia,nib->nab", A[fo], A[fo]))
    V = np.zeros((n, 3, 3))
    np.add.at(V, pt_of, np.einsum("nia,nib->nab", B, B))
    Vinv = np.zeros((n, 3, 3))
    Vinv[keep] = np.linalg.inv(V[keep])
    W = np.einsum("nia,nib->nab", A, B)  # A^T B per observation
    oa, ob = _pairs(prob, keep)
    ja, jb, Vi = cam_of[oa] - mcon, cam_of[ob] - mcon, Vinv[pt_of[oa]]
    np.add.at(Sb, (ja, jb), -np.einsum("nab,nbc,ndc->nad", W[oa], Vi, W[ob]))
    S = Sb.transpose(0, 2, 1, 3).reshape(6 * mf, 6 * mf)
    Z = np.linalg.inv(S) if mf else np.zeros((0, 0))
    Zb = Z.reshape(mf, 6, mf, 6).transpose(0, 2, 1, 3)
    cam = np.zeros((m, 6, 6))
    cam[mcon:] = pixel_var * Zb[np.arange(mf), np.arange(mf)]
    T = np.zeros((n, 3, 3))
    np.add.at(T, pt_of[oa], np.einsum("nba,nbc,ncd->nad", W[oa], Zb[ja, jb], W[ob]))
    pt = np.zeros((n, 3, 3))
    pt[keep] = pixel_var * (Vinv[keep] + Vinv[keep] @ T[keep] @ Vinv[keep])
    pt[(np.arange(n) >= ncon) & unc] = np.nan
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


# ---------------------------------------------------------------- edge scenes of the covariance stage
# Built with the scene() / random_vis() of tests/test_gpu_ba_edges.py (camera 0 at the origin, cameras 0.25 apart
# along x, points 4-7 in front).  One fixed camera and no fixed point leave the scale free, so every regular row
# fixes it with a second fixed camera or with fixed points.
def groups(k, g, blind_group=None, seed=7):
    """Camera 0 fixed, then k groups of g free cameras that share no point; every third point of a group is also
    seen by camera 0, and the first three points of every group are fixed: they fix its scale.  The reduced camera
    system is block-diagonal over the groups.  In `blind_group` the middle camera sees no point: its rows of S are
    exactly zero, a singular block.  (A group without fixed points is singular in its scale too, but only through
    the cancellation of S = U - W V^-1 W^T, which leaves that pivot at rounding noise, 1e-13 to 1e-8 relative:
    not a reliable singular case.)"""
    import test_gpu_ba_edges as te
    rng = np.random.default_rng(seed)
    fixed, rest = [], []
    for q in range(k):
        cams = [c for c in range(1 + q * g, 1 + (q + 1) * g) if q != blind_group or c != 1 + q * g + g // 2]
        vis = te.random_vis(rng, 6 * g, cams, 2, 5)
        vis = [v + [0] if i % 3 == 0 else v for i, v in enumerate(vis)]
        fixed += vis[:3]
        rest += vis[3:]
    return te.scene(fixed + rest, k * g + 1, 1, len(fixed), seed)


def _edge(name):
    import test_gpu_ba_edges as te
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in ("structure_only", "motion_only", "free_camera_sees_only_fixed_points",
                "points_seen_only_by_fixed_cameras"):
        return te.make(name)
    if name == "single_observation_points_fixed":  # 10 points seen once, 8 of them by free cameras
        return te.scene(te.random_vis(rng, 50, range(6)) + [[1 + k % 5] for k in range(10)], 6, 2, 0, 6)
    if name == "weight_dropped_points":  # 10 two-observation points: one observation 5 max_err off in y (across
        # the epipolar lines of cameras displaced along x), the other 0.3 px off at the start
        from ba_dense import project
        prob = te.scene(te.random_vis(rng, 50, range(6)) + [[2 + k % 4, 2 + (k + 1) % 4] for k in range(10)],
                        6, 2, 0, 9)
        o = prob.ptr[50:60]
        xy = project(prob)[0]
        prob.xy[o] = xy[o] + [0.0, 5.0 * te.MAX_ERR]
        prob.xy[o + 1] = xy[o + 1] + rng.normal(0, 0.3, (10, 2))
        return prob
    if name == "one_long_pair_fixed":  # free cameras 2 and 3 share 532 = 4 x 128 + 20 free points
        return te.scene([[0, 1, 2, 3]] * 532, 4, 2, 0, 8)
    if name.startswith("groups_"):  # groups_<k>x<g>[_blind<q>]
        f = name.split("_")
        k, g = map(int, f[1].split("x"))
        return groups(k, g, int(f[2][5:]) if len(f) > 2 else None)
    if name == "points_fix_gauge":  # m_con = 0: four fixed points fix the gauge
        return te.scene(te.random_vis(rng, 60, range(5), 2, 4), 5, 0, 4, 10)
    if name == "many_points":  # 6n > 1024 x 256: ba_cov_begin clears T in more than one grid-stride pass
        return te.scene(te.random_vis(rng, 50000, range(8), 2, 4), 8, 2, 0, 11)
    raise KeyError(name)


# name -> max_err.  motion_only takes 30 px: at 6 px its cameras 3 and 5 have no observation of non-zero weight
# at the start, so they never move and stay singular.
EDGE_ROWS = {
    "structure_only": 6.0, "motion_only": 30.0, "free_camera_sees_only_fixed_points": 6.0,
    "points_seen_only_by_fixed_cameras": 6.0, "single_observation_points_fixed": 6.0,
    "weight_dropped_points": 6.0, "one_long_pair_fixed": 6.0,
    "groups_2x6": 6.0, "groups_2x10": 6.0, "groups_3x10": 6.0, "groups_5x5": 6.0,
    "points_fix_gauge": 6.0, "many_points": 6.0,
}
# the singular block first, in the middle, last
SINGULAR_EDGE_ROWS = {"groups_3x10_blind0": 6.0, "groups_3x10_blind1": 6.0, "groups_3x10_blind2": 6.0}
LARGE = ("many_points",)  # beyond cov_full: H has 150 000 rows


def make_edge(name):
    import ba_dense as bd
    return _edge(name), bd.options({**EDGE_ROWS, **SINGULAR_EDGE_ROWS}[name])


def reference(prob, max_err, pixel_var):
    """(camCov, ptCov, info, H or None): cov_full, or cov_schur where H is too large to invert whole."""
    if prob.nobs > 20000:
        return (*cov_schur(prob, max_err, pixel_var), None)
    return cov_full(prob, max_err, pixel_var)


def decision_margin(prob, max_err):
    """min over the observations of ||e| - max_err| / max_err: how far every Tukey decision is from its tie."""
    e = residuals(prob)
    return float((np.abs(np.sqrt((e * e).sum(1)) - max_err) / max_err).min())


def min_relative_pivot(H):
    """smallest L_kk^2 / H_kk of the Cholesky factor of H, 0 when the factorisation breaks down"""
    try:
        L = np.linalg.cholesky(H)
    except np.linalg.LinAlgError:
        return 0.0
    return float((np.diag(L) ** 2 / np.diag(H)).min())
