"""A float64 restatement of one bundle-adjustment LM trial, and the scenes the BA tests run it on.

The reference works on the whole problem at once:
  - residuals x - pi(K (R(dq(v)) R0 X + t)) with each camera's full 3x3 K (fx, fy, skew, cx, cy);
  - the Jacobian by a complex step over each observation's 9 local parameters (v and t of its camera,
    X of its point): 9 vectorised residual evaluations whatever the problem size, exact to roundoff,
    assembled as a scipy.sparse matrix;
  - Tukey weights frozen at the start of the round, mu = tau max diag(J^T W J), and the damped normal
    equations (J^T W J + mu I) d = J^T W e solved densely.

check_trial() compares a solver's first trial with it through scale-free measures whose tolerances come
from float64 error bounds, not from measured values:
  1. the backward error of the damped normal equations at the solver's step,
     |(H + mu I) d - g|_inf / (|H + mu I|_inf |d|_inf + |g|_inf);
  2. the forward error against the reference step, bounded by kappa_inf(H + mu I) times the backward bound;
  3. the costs before and after the trial, relative to 1e-12 plus the cancellation bound of the scene.
The forward bound is weak: the LM damping leaves kappa near 1 / tau = 1e7, so it sits near 1e-5 on the plain
rows and above 1 on far_offset, while the measured forward errors are 1e-12 or less (1e-8 on far_offset).
It is a sanity bound only; the backward error and the two costs are the checks that catch a wrong step.
The solver's step is recovered from its state: v = vec(quat(R R0^T)) with w > 0, dt, dX.

Every scene is built from fresh arrays: BAProblem.copy() shares K, ptr, cam and xy with the original, so a
scene that edits those on a copy would edit its parent too."""
import numpy as np
import scipy.sparse as sp

from coslam_b200.ctypes_defs import BaOptions
from coslam_b200.problem import BAProblem

EPS = np.finfo(np.float64).eps
MAX_ERR = 6.0
H_CS = 1e-30  # complex step

# backward error of a Cholesky / Schur solve of order n in float64: c n eps with a modest c; the
# reduced systems here have n <= 2500, so 64 n^(1/2) eps (the usual random-walk growth of the
# roundoff of n-term sums) is far above what a correct solve leaves and far below a wrong term
BWD_C = 64.0


def quat_to_R(w, x, y, z):
    """Rotation matrices of (possibly complex) unit quaternions, batched over the leading axis."""
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def R_to_quat(R):
    """Unit quaternions (w > 0) [.., 4] of rotation matrices [.., 3, 3] (Shepperd's branch by the largest
    diagonal term, so small and large rotations are both exact to roundoff)."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    q = np.empty((len(R), 4))
    for k, M in enumerate(R):
        tr = np.trace(M)
        c = int(np.argmax([tr, M[0, 0], M[1, 1], M[2, 2]]))
        if c == 0:
            s = 2 * np.sqrt(1 + tr)
            q[k] = [s / 4, (M[2, 1] - M[1, 2]) / s, (M[0, 2] - M[2, 0]) / s, (M[1, 0] - M[0, 1]) / s]
        else:
            i = c - 1
            j, l = (i + 1) % 3, (i + 2) % 3
            s = 2 * np.sqrt(1 + M[i, i] - M[j, j] - M[l, l])
            v = np.empty(3)
            v[i], v[j], v[l] = s / 4, (M[j, i] + M[i, j]) / s, (M[l, i] + M[i, l]) / s
            q[k] = [(M[l, j] - M[j, l]) / s, *v]
        if q[k, 0] < 0:
            q[k] = -q[k]
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def quat_mul(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.stack([a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2] - a[..., 3] * b[..., 3],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0] + a[..., 2] * b[..., 3] - a[..., 3] * b[..., 2],
                     a[..., 0] * b[..., 2] - a[..., 1] * b[..., 3] + a[..., 2] * b[..., 0] + a[..., 3] * b[..., 1],
                     a[..., 0] * b[..., 3] + a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1] + a[..., 3] * b[..., 0]], -1)


def fresh(prob):
    """A copy of `prob` that shares no array with it (BAProblem.copy() shares K, ptr, cam and xy)."""
    p = BAProblem(prob.K.copy(), prob.R, prob.t, prob.X, prob.ptr.copy(), prob.cam.copy(), prob.xy.copy(),
                  prob.m_con, prob.n_con)
    p.outlier[:] = prob.outlier
    return p


def point_of(prob):
    return np.repeat(np.arange(prob.n), np.diff(prob.ptr))


def options(max_err=MAX_ERR):
    opt = BaOptions.defaults()
    opt.max_err = max_err
    return opt


# ---------------------------------------------------------------- residuals and Jacobian
def project(prob, dv=None, dt=None, dX=None):
    """Projections [nobs, 2] of every observation at the local parameters (v, t + dt, X + dX) of its camera and
    point (per observation, possibly complex; None = 0), and the camera-frame points [nobs, 3]."""
    pt, cam = point_of(prob), prob.cam
    R0 = prob.R.reshape(-1, 3, 3)[cam]
    X = prob.X[pt] + (0 if dX is None else dX)
    Y = np.einsum("nij,nj->ni", R0, X)
    if dv is not None:
        w = np.sqrt(1.0 - (dv * dv).sum(1))
        Y = np.einsum("nij,nj->ni", quat_to_R(w, dv[:, 0], dv[:, 1], dv[:, 2]), Y)
    P = Y + prob.t[cam] + (0 if dt is None else dt)
    u = np.einsum("nij,nj->ni", prob.K.reshape(-1, 3, 3)[cam], P)
    return u[:, :2] / u[:, 2:3], P


def residuals(prob):
    return prob.xy - project(prob)[0]


def local_jacobian(prob):
    """d xhat / d (v, t, X) [nobs, 2, 9] of every observation at v = 0, by complex steps."""
    N = prob.nobs
    J = np.empty((N, 2, 9))
    for k in range(9):
        z = np.zeros((N, 3), np.complex128)
        z[:, k % 3] = 1j * H_CS
        args = {0: dict(dv=z), 1: dict(dt=z), 2: dict(dX=z)}[k // 3]
        J[:, :, k] = project(prob, **args)[0].imag / H_CS
    return J


def layout(prob):
    """Column of every observation's 9 local parameters in the free-parameter vector [free cameras (v, t) |
    free points X], -1 where the camera or point is fixed."""
    mf = prob.m - prob.m_con
    pt, cam = point_of(prob), prob.cam.astype(np.int64)
    cols = np.full((prob.nobs, 9), -1, np.int64)
    fc = cam >= prob.m_con
    cols[fc, :6] = 6 * (cam[fc, None] - prob.m_con) + np.arange(6)
    fp = pt >= prob.n_con
    cols[fp, 6:] = 6 * mf + 3 * (pt[fp, None] - prob.n_con) + np.arange(3)
    return cols, 6 * mf + 3 * (prob.n - prob.n_con)


def tukey_weights(e, max_err):
    if max_err <= 0:
        return np.ones_like(e)
    q = 1 - (e / max_err) ** 2
    return np.where(e >= max_err, 0.0, q * q)


def cancellation(prob):
    """Per observation: rho, a bound on the relative error of the camera-frame point R X + t in float64
    (it cancels when the world is far from the origin: |R X| + |t| >> |R X + t|), and delta, the pixel error
    that follows from it (and from forming K P / z)."""
    pt, cam = point_of(prob), prob.cam
    _, P = project(prob)
    # R X + t: each component a sum of 4 terms of size <= |X|_1 + |t|_1, a few roundings of eps / 2 each
    mag = np.abs(prob.X[pt]).sum(1) + np.abs(prob.t[cam]).sum(1) + np.abs(P).sum(1)
    rho = 2 * EPS * mag / np.abs(P[:, 2])
    K = prob.K.reshape(-1, 3, 3)[cam]
    kscale = np.abs(K[:, 0, 0]) + np.abs(K[:, 0, 1]) + np.abs(K[:, 1, 1])
    delta = rho * kscale * np.abs(P).sum(1) / np.abs(P[:, 2])
    return rho, delta


class Trial:
    """The dense first LM trial of a round: J, weights, H + mu I, g, the reference step, its costs."""

    def __init__(self, prob, opt):
        self.prob = prob
        e = residuals(prob)
        self.w = tukey_weights(np.sqrt((e * e).sum(1)), opt.max_err)
        cols, self.np = layout(prob)
        Jl = local_jacobian(prob)
        rows = np.arange(2 * prob.nobs).reshape(-1, 2)
        sw = np.sqrt(self.w)
        keep = np.broadcast_to(cols[:, None, :] >= 0, Jl.shape)
        r = np.broadcast_to(rows[:, :, None], Jl.shape)[keep]
        c = np.broadcast_to(cols[:, None, :], Jl.shape)[keep]
        self.Jl = Jl
        self.J = sp.csr_matrix(((Jl * sw[:, None, None])[keep], (r, c)), shape=(2 * prob.nobs, self.np))
        self.Jabs = sp.csr_matrix((np.abs(Jl * sw[:, None, None])[keep], (r, c)), shape=self.J.shape)
        self.e = (e * sw[:, None]).ravel()
        H = (self.J.T @ self.J).toarray()
        self.mu = opt.opts[0] * H.diagonal().max()
        self.A = H + self.mu * np.eye(self.np)
        self.g = self.J.T @ self.e
        self.d = np.linalg.solve(self.A, self.g)
        self.cost0 = float((self.w * (e * e).sum(1)).sum())
        self.rho, self.delta = cancellation(prob)
        self.Anorm = np.abs(self.A).sum(1).max()
        self.kappa = self.Anorm * np.abs(np.linalg.inv(self.A)).sum(1).max()

    # -------- costs
    def cost(self, state):
        e = state.xy - project(state)[0]
        return float((self.w * (e * e).sum(1)).sum())

    def cost_tol(self, state):
        """1e-12 plus the first-order effect of the cancellation error delta on sum w |e|^2."""
        e = state.xy - project(state)[0]
        _, delta = cancellation(state)
        c = (self.w * (e * e).sum(1)).sum()
        return 1e-12 + float((self.w * (2 * np.sqrt((e * e).sum(1)) * delta + 2 * delta * delta)).sum() / c)

    # -------- steps
    def step_of(self, state):
        """The step (v, t, X of the free parameters) that takes the start to `state`, and a bound on the
        error of recovering it from rounded states (|t|, |X| eps from the subtractions; v from R R0^T)."""
        p, mf = self.prob, self.prob.m - self.prob.m_con
        d = np.empty(self.np)
        err = np.empty(self.np)
        if mf:
            R0 = p.R.reshape(-1, 3, 3)[p.m_con:]
            R1 = state.R.reshape(-1, 3, 3)[p.m_con:]
            q = R_to_quat(R1 @ R0.transpose(0, 2, 1))
            cams = np.concatenate([q[:, 1:], state.t[p.m_con:] - p.t[p.m_con:]], 1)
            d[:6 * mf] = cams.ravel()
            cerr = np.concatenate([np.full((mf, 3), 8 * EPS),
                                   EPS * (np.abs(state.t[p.m_con:]) + np.abs(p.t[p.m_con:]))], 1)
            err[:6 * mf] = cerr.ravel()
        d[6 * mf:] = (state.X[p.n_con:] - p.X[p.n_con:]).ravel()
        err[6 * mf:] = (EPS * (np.abs(state.X[p.n_con:]) + np.abs(p.X[p.n_con:]))).ravel()
        return d, err

    def backward(self, d):
        return float(np.abs(self.A @ d - self.g).max() / (self.Anorm * np.abs(d).max() + np.abs(self.g).max()))

    def backward_tol(self, d, derr):
        """BWD_C sqrt(n) eps for the solve, plus what float64 cannot resolve in this scene: the error of the
        solver's own J (analytic, from a cancelling R X + t: |dJ| <= rho |J|) and e (delta), propagated
        through H and g, and the error of recovering d from rounded states."""
        rw = np.repeat(self.rho, 2)
        ew = np.repeat(self.delta * np.sqrt(self.w), 2)
        dHd = 2 * (self.Jabs.T @ (rw * (self.Jabs @ np.abs(d))))
        dg = self.Jabs.T @ (rw * np.abs(self.e) + ew)
        den = self.Anorm * np.abs(d).max() + np.abs(self.g).max()
        return float(BWD_C * np.sqrt(self.np) * EPS + (dHd.max() + dg.max() + self.Anorm * derr.max()) / den)

    def forward(self, d):
        return float(np.abs(d - self.d).max() / np.abs(self.d).max())

    def forward_tol(self, bwd_tol, derr):
        """kappa_inf 2 b for a solve with normwise backward error b (Higham, Thm 7.2), plus the recovery error
        of d and the reference's own solve (LAPACK, backward error n eps).  With kappa ~ 1e7 this is a sanity
        bound only (see the module docstring): a step that passes the backward check passes it as well."""
        b = bwd_tol + self.np * EPS
        return float(2 * self.kappa * b + derr.max() / np.abs(self.d).max())


def check_trial(prob, info, after, opt):
    """One trial that ran on `prob` and left `after` with info: measured (bwd, fwd, cost) errors and their
    tolerances.  The trial must be accepted, as the first trial of these scenes is a descent step."""
    T = Trial(prob, opt)
    assert int(info[9]) == 1
    d, derr = T.step_of(after)
    bwd, fwd = T.backward(d), T.forward(d)
    btol = T.backward_tol(d, derr)
    ftol = T.forward_tol(btol, derr)
    c0 = abs(info[0] - T.cost0) / T.cost0
    c0tol = T.cost_tol(prob)
    c1_ref = T.cost(after)
    c1 = abs(info[1] - c1_ref) / c1_ref
    c1tol = T.cost_tol(after)
    assert info[1] < info[0]
    out = dict(bwd=bwd, bwd_tol=btol, fwd=fwd, fwd_tol=ftol, cost0=c0, cost0_tol=c0tol, cost1=c1, cost1_tol=c1tol,
               kappa=T.kappa)
    assert bwd <= btol, out
    assert fwd <= ftol, out
    assert c0 <= c0tol and c1 <= c1tol, out
    return out


# ---------------------------------------------------------------- sba's parameter block
def pack_sba(prob, dq=None):
    """cosl_sba_motstr_levmar_x's p = [m x (fx, cx, cy, ar, s, v1, v2, v3, t1, t2, t3) | n x 3], rot0 [m, 4]
    and vmask [n, m] of `prob`.  dq [m, 3] is the initial local rotation v of every camera: rot0 is chosen
    so that quat(sqrt(1 - |v|^2), v) (x) rot0 is the rotation of prob.R."""
    m, n = prob.m, prob.n
    dq = np.zeros((m, 3)) if dq is None else np.asarray(dq, np.float64)
    K = prob.K
    p = np.zeros(11 * m + 3 * n)
    c = p[:11 * m].reshape(m, 11)
    c[:, 0], c[:, 1], c[:, 2], c[:, 3], c[:, 4] = K[:, 0], K[:, 2], K[:, 5], K[:, 4] / K[:, 0], K[:, 1]
    c[:, 5:8] = dq
    c[:, 8:11] = prob.t
    p[11 * m:] = prob.X.ravel()
    w = np.sqrt(1.0 - (dq * dq).sum(1))
    dq_conj = np.concatenate([w[:, None], -dq], 1)
    rot0 = quat_mul(dq_conj, R_to_quat(prob.R))
    vmask = np.zeros((n, m), np.int8)
    vmask[point_of(prob), prob.cam] = 1
    return p, rot0, vmask


def unpack_sba(p, rot0, vmask, xy, m_con, n_con):
    """The BAProblem that cosl_sba_motstr_levmar_x solves for (p, rot0, vmask): K = [[fx, s, cx], [0, ar fx,
    cy], [0, 0, 1]], R = R(quat(sqrt(1 - |v|^2), v) (x) rot0); observations point-major by ascending camera."""
    n, m = vmask.shape
    c = p[:11 * m].reshape(m, 11)
    K = np.zeros((m, 9))
    K[:, 0], K[:, 1], K[:, 2], K[:, 4], K[:, 5], K[:, 8] = c[:, 0], c[:, 4], c[:, 1], c[:, 3] * c[:, 0], c[:, 2], 1.0
    v = c[:, 5:8]
    q = quat_mul(np.concatenate([np.sqrt(1.0 - (v * v).sum(1))[:, None], v], 1), rot0)
    R = quat_to_R(q[:, 0], q[:, 1], q[:, 2], q[:, 3])
    pt, cam = np.nonzero(vmask)
    ptr = np.concatenate([[0], np.cumsum(np.bincount(pt, minlength=n))])
    return BAProblem(K, R, c[:, 8:11].copy(), p[11 * m:].reshape(n, 3).copy(), ptr, cam, np.array(xy).reshape(-1, 2),
                     m_con, n_con)


# ---------------------------------------------------------------- scenes
def K_of(fx, ar, s, cx, cy):
    return np.array([fx, s, cx, 0.0, ar * fx, cy, 0.0, 0.0, 1.0])


# the three cameras of a rig of different image sizes, each with its own K
RIG_SIZES = [(640, 480), (1280, 720), (1920, 1080)]
RIG_K = np.array([K_of(350.0, 0.92, -4.0, 331.5, 229.0),
                  K_of(800.0, 1.0, 0.0, 622.0, 371.25),
                  K_of(1400.0, 1.07, 3.5, 985.0, 527.5)])


def rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    h = np.radians(deg) / 2
    return quat_to_R(np.cos(h), *(np.sin(h) * a))


def _finish(K, R, t, X, vis, m_con, n_con, rng, noise=0.3, dR=0.0003, dt=0.002, dX=0.001, sizes=None):
    """Observations = projections of (R, t, X) + noise (inside each camera's image when sizes is given,
    vis[i] = the cameras that see point i, in the order listed); free cameras and points then start off
    by rotations of about dR rad, dt m and dX times their depth."""
    m, n = len(R), len(X)
    cam = np.concatenate([np.asarray(v, np.int32) for v in vis]) if n else np.zeros(0, np.int32)
    ptr = np.concatenate([[0], np.cumsum([len(v) for v in vis])]).astype(np.int64)
    truth = BAProblem(K, R, t, X, ptr, cam, np.zeros((len(cam), 2)), m_con, n_con)
    xy, P = project(truth)
    assert np.all(P[:, 2] > 0)
    if sizes is not None:
        for j, (W, Hh) in enumerate(sizes):
            o = cam == j
            assert np.all((xy[o] >= 0) & (xy[o] < [W, Hh])), j
    xy = xy + rng.normal(0, noise, xy.shape)
    prob = BAProblem(K.copy(), R, t, X, ptr.copy(), cam.copy(), xy, m_con, n_con)
    Rr = prob.R.reshape(-1, 3, 3)
    for j in range(m_con, m):
        v = rng.normal(size=3) * dR
        Rr[j] = quat_to_R(np.sqrt(1 - v @ v), *v) @ Rr[j]
        prob.t[j] += rng.normal(0, dt, 3)
    depth = np.minimum.reduceat(P[:, 2], ptr[:-1])[n_con:, None]  # nearest camera's depth of each point
    prob.X[n_con:] += rng.normal(0, 1, (n - n_con, 3)) * dX * np.maximum(depth, 1.0) / 5
    return prob


def _rig_poses(n_kf, yaws=(-25.0, 0.0, 25.0), step=0.3):
    """3 cameras on a rig (yawed apart) x n_kf key frames moving along x; pose index = 3 kf + camera."""
    R, C = [], []
    for k in range(n_kf):
        Rk = rot([0, 1, 0], 2.0 * k) @ rot([1, 0, 0], 1.0 * (k % 2))
        for c, yaw in enumerate(yaws):
            R.append(rot([0, 1, 0], yaw) @ Rk)
            C.append(np.array([step * k + 0.1 * c, 0.05 * (k % 2), 0.02 * c]))
    R = np.array(R)
    C = np.array(C)
    return R, -np.einsum("jab,jb->ja", R, C)


def _visible(K, R, t, X, sizes, margin=2.0):
    P = np.einsum("jab,nb->nja", R, X) + t[None]
    u = np.einsum("jab,njb->nja", K.reshape(-1, 3, 3), P)
    xy = u[..., :2] / u[..., 2:3]
    W = np.array([s[0] for s in sizes])[None, :]
    Hh = np.array([s[1] for s in sizes])[None, :]
    return ((P[..., 2] > 0.2) & (xy[..., 0] > margin) & (xy[..., 0] < W - margin) & (xy[..., 1] > margin)
            & (xy[..., 1] < Hh - margin))


def rig_intrinsics(offset=None, seed=11, n=160, n_kf=4, dR=0.0003):
    rng = np.random.default_rng(seed)
    R, t = _rig_poses(n_kf)
    m = len(R)
    K = np.tile(RIG_K, (n_kf, 1))
    sizes = RIG_SIZES * n_kf
    X, vis = [], []
    while len(X) < n:
        x = np.array([rng.uniform(-4, 5), rng.uniform(-2, 2), rng.uniform(3, 9)])
        v = np.nonzero(_visible(K, R, t, x[None], sizes)[0])[0]
        if len(v) >= 2:
            X.append(x)
            vis.append(list(v))
    prob = _finish(K, R, t, np.array(X), vis, 3, 2, rng, dR=dR, sizes=sizes)
    if offset is not None:  # X' = X + c, t' = t - R c: the same scene in world coordinates far from the origin
        c = np.asarray(offset, np.float64)
        prob.X[:] += c
        prob.t[:] -= np.einsum("jab,b->ja", prob.R.reshape(-1, 3, 3), c)
    return prob


def wide_and_deep(seed=12):
    """Depths from 0.3 m to 800 m (log-uniform), |x/z| up to 2, the far points with under 0.05 deg of
    parallax over the whole 0.5 m baseline."""
    rng = np.random.default_rng(seed)
    n_kf = 3
    R, t = _rig_poses(n_kf, yaws=(-40.0, 0.0, 40.0), step=0.2)
    K = np.tile(RIG_K, (n_kf, 1))
    X, vis = [], []
    depths = np.concatenate([[0.3, 0.31, 800.0, 790.0, 650.0], np.exp(rng.uniform(np.log(0.3), np.log(800), 200))])
    for z in depths:
        for _ in range(200):
            x = np.array([rng.uniform(-2, 2) * z + 0.2, rng.uniform(-1.2, 1.2) * z, z])
            P = np.einsum("jab,b->ja", R, x) + t
            ok = (P[:, 2] > 0.1) & (np.abs(P[:, 0] / P[:, 2]) <= 2.0) & (np.abs(P[:, 1] / P[:, 2]) <= 1.5)
            v = np.nonzero(ok)[0]
            if len(v) >= 2:
                X.append(x)
                vis.append(list(v))
                break
    X = np.array(X)
    return _finish(K, R, t, X, vis, 3, 2, rng, dX=0.0005)


def far_offset():
    return rig_intrinsics(offset=(1e4, -5e3, 3e3))


def rotated_start(seed=13):
    """rig_intrinsics with every free camera started 3-8 degrees off (|v| up to about 0.07)."""
    rng = np.random.default_rng(seed)
    prob = rig_intrinsics(seed=seed, dR=0.0)
    Rr = prob.R.reshape(-1, 3, 3)
    for j in range(prob.m_con, prob.m):
        a = rng.normal(size=3)
        Rr[j] = rot(a, rng.uniform(3.0, 8.0)) @ Rr[j]
    return prob


LONG = (33, 64, 100)


def long_tracks(seed=14):
    """104 cameras on an arc around the points (2 fixed); points seen by 33, 64 and 100 cameras whose runs in
    the point-major list start at offsets 250 (mod 256), 30 (mod 32) and 250 (mod 256), so that they cross warp
    and 256-thread block boundaries; the last camera has a single observation at a multiple of 128 of the
    camera-major list (the order of the 128-thread camera kernel)."""
    rng = np.random.default_rng(seed)
    m, m_con = 104, 2
    K = np.tile(K_of(600.0, 1.03, 1.5, 640.0, 360.0), (m, 1))
    R, C = [], []
    for j in range(m):
        a = np.radians(-40 + 80 * j / (m - 1))
        Cj = np.array([10 * np.sin(a), 0.3 * np.sin(5 * a), 8 - 10 * np.cos(a)])
        R.append(rot([0, 1, 0], np.degrees(a)))
        C.append(Cj)
    R, C = np.array(R), np.array(C)
    t = -np.einsum("jab,jb->ja", R, C)
    last = m - 1
    others = np.arange(m - 1)
    vis = []

    def filler(k):
        return sorted(rng.choice(others, size=k, replace=False).tolist())

    size = 0
    for k, mod, off in ((LONG[0], 256, 250), (LONG[1], 32, 30), (LONG[2], 256, 250)):
        while (off - size) % mod or size < 300:
            g = (off - size) % mod or mod
            kk = g if g in (2, 3, 4) else (2 if g == 5 else (3 if g == 1 else 4))
            vis.append(filler(kk))
            size += kk
        vis.append(filler(k))
        size += k
    for _ in range(40):
        vis.append(filler(int(rng.integers(2, 5))))
    # the last camera's single observation comes after every free observation of the other cameras in the
    # camera-major list, one past those of the point that shares it: make that position 0 (mod 128)
    nfree = lambda: sum(sum(1 for j in v if j >= m_con) for v in vis)  # noqa: E731
    while (nfree() + 1) % 128:
        need = 128 - (nfree() + 1) % 128
        vis.append([0, int(rng.integers(m_con, m - 1))] if need == 1 else filler(2 if need == 2 else 3))
    vis.append([int(rng.integers(m_con, m - 1)), last])
    n = len(vis)
    X = np.column_stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.0, 1.0, n), rng.uniform(7.0, 9.0, n)])
    return _finish(K, R, t, X, vis, m_con, 3, rng)


def long_track_layout(prob):
    """(start offsets of the 33-, 64- and 100-camera runs in the point-major list, the position of the last
    camera's observations in the camera-major list of the free cameras)."""
    k = np.diff(prob.ptr)
    starts = [int(prob.ptr[np.nonzero(k == L)[0][0]]) for L in LONG]
    free = prob.cam[prob.cam >= prob.m_con]
    order = np.argsort(free, kind="stable")
    pos = np.nonzero(free[order] == prob.m - 1)[0]
    return starts, pos


def unobserved_points(seed=15):
    """rig_intrinsics with points nobody observes: the first fixed point, the first free point, one in the
    middle and the last one."""
    base = rig_intrinsics(seed=seed, n=120)
    n = base.n
    k = np.diff(base.ptr)
    lists = [list(base.cam[base.ptr[i]:base.ptr[i + 1]]) for i in range(n)]
    xys = [base.xy[base.ptr[i]:base.ptr[i + 1]] for i in range(n)]
    X = list(base.X)
    rng = np.random.default_rng(seed)
    mid = n // 2
    new = []
    for i in range(n):
        if i in (0, base.n_con, mid):
            new.append((rng.normal(size=3) + [0, 0, 6], [], np.zeros((0, 2))))
        new.append((X[i], lists[i], xys[i]))
    new.append((rng.normal(size=3) + [0, 0, 6], [], np.zeros((0, 2))))
    Xn = np.array([a for a, _, _ in new])
    cam = np.concatenate([np.asarray(b, np.int32) for _, b, _ in new])
    xy = np.concatenate([c for _, _, c in new])
    ptr = np.concatenate([[0], np.cumsum([len(b) for _, b, _ in new])])
    assert k.min() >= 2
    return BAProblem(base.K.copy(), base.R, base.t, Xn, ptr, cam, xy, base.m_con, base.n_con + 1)


def unobserved_indices(prob):
    return np.nonzero(np.diff(prob.ptr) == 0)[0]


def tukey_mixed(seed=16):
    """rig_intrinsics with 25 % outliers (10-60 px off), and residuals placed 1e-9 relative inside and just
    outside max_err at the start."""
    rng = np.random.default_rng(seed)
    prob = rig_intrinsics(seed=seed)
    N = prob.nobs
    idx = rng.permutation(N)
    out = idx[:N // 4]
    d = rng.normal(size=(len(out), 2))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    prob.xy[out] += d * rng.uniform(10, 60, (len(out), 1))
    xhat = project(prob)[0]
    edge = idx[N // 4:N // 4 + 16]
    for k, o in enumerate(edge):
        r = prob.xy[o] - xhat[o]
        r = r / np.linalg.norm(r) if np.linalg.norm(r) > 0 else np.array([1.0, 0.0])
        prob.xy[o] = xhat[o] + r * MAX_ERR * (1 - 1e-9 if k % 2 == 0 else 1 + 1e-9)
    return prob


def unsorted_observations(seed=17):
    """rig_intrinsics with every third point listing its cameras in descending order."""
    base = rig_intrinsics(seed=seed)
    cam, xy = base.cam.copy(), base.xy.copy()
    for i in range(0, base.n, 3):
        a, b = base.ptr[i], base.ptr[i + 1]
        cam[a:b] = cam[a:b][::-1]
        xy[a:b] = xy[a:b][::-1]
    return BAProblem(base.K.copy(), base.R, base.t, base.X, base.ptr.copy(), cam, xy, base.m_con, base.n_con)


def sorted_permutation(prob):
    """The same problem with every point's observations sorted by camera, and the permutation used."""
    perm = np.concatenate([prob.ptr[i] + np.argsort(prob.cam[prob.ptr[i]:prob.ptr[i + 1]], kind="stable")
                           for i in range(prob.n)]).astype(np.int64)
    return BAProblem(prob.K.copy(), prob.R, prob.t, prob.X, prob.ptr.copy(), prob.cam[perm], prob.xy[perm],
                     prob.m_con, prob.n_con), perm


ROWS = {
    "rig_intrinsics": (rig_intrinsics, MAX_ERR),
    "wide_and_deep": (wide_and_deep, MAX_ERR),
    "far_offset": (far_offset, MAX_ERR),
    # 3-8 degrees off puts residuals at tens to hundreds of px: the plain (non-robust) trial
    "rotated_start": (rotated_start, 0.0),
    "long_tracks": (long_tracks, MAX_ERR),
    "unobserved_points": (unobserved_points, MAX_ERR),
    "tukey_mixed": (tukey_mixed, MAX_ERR),
    "unsorted_observations": (unsorted_observations, MAX_ERR),
}


def make(name):
    """(problem, options) of a scene row"""
    f, max_err = ROWS[name]
    return f(), options(max_err)
