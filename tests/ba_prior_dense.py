"""float64 references of a bundle adjustment with Gaussian pose priors on free cameras (cosl_ba_solver_set_cam_prior;
DESIGN.md 4.8), on top of ba_dense, ba_cov_dense and ba_obscov_dense.

A prior on free camera j has a mean (R_p, t_p) and a 6x6 covariance P for (w, dt) in the chart of camCov.  Its residual
is r = [Log(R_j R_p^T); t_j - t_p] and its term of the objective r^T P^-1 r = |L r|^2 with L = chol(P^-1)^T (upper
triangular).  The normal equations gain, per prior, the whitened rows L J with J = dr / d(v, t) in the solver's chart
R = R(q(v)) R0:
  dr_w / dv = Jl^-1(r_w) J_q(v),  J_q = 2 (w_q I + [v]x + v v^T / w_q),  dr_t / dt = I,
where Jl^-1 is the inverse left Jacobian of SO(3).  In the (w, t) chart of the covariance stage dr_w / dw = Jl^-1(r_w).

  - prior_residual / prior_jacobian: r and J at any v (pinned against central differences by the CPU tests);
  - PTrial: the dense first LM trial with the prior rows appended to ba_obscov_dense.WTrial's system, check_ptrial
    its check_trial;
  - normal_equations: the undamped H and g (observations plus priors) at a problem's parameters, v = 0;
  - cov_full: pixel_var (J^T W Lambda J + sum J_p^T P^-1 J_p)^-1 over the free parameters, sigma2_hat and dof with six
    measurements per prior;
  - random_cov / draw_means: priors for the tests."""
import numpy as np
import scipy.sparse as sp

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od

EPS = np.finfo(np.float64).eps


class Priors:
    """cams [k], R [k, 3, 3], t [k, 3], cov [k, 6, 6]"""

    def __init__(self, cams, R, t, cov):
        self.cams = np.asarray(cams, np.int64).reshape(-1)
        self.R = np.asarray(R, np.float64).reshape(-1, 3, 3)
        self.t = np.asarray(t, np.float64).reshape(-1, 3)
        self.cov = np.asarray(cov, np.float64).reshape(-1, 6, 6)

    def __len__(self):
        return len(self.cams)

    def factors(self):
        """L [k, 6, 6] upper triangular with L^T L = P^-1"""
        return np.linalg.cholesky(np.linalg.inv(self.cov)).transpose(0, 2, 1)

    def subset(self, keep):
        return Priors(self.cams[keep], self.R[keep], self.t[keep], self.cov[keep])


def hat(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def so3_exp(w):
    th = float(np.linalg.norm(w))
    W = hat(w)
    if th < 1e-8:
        return np.eye(3) + W + 0.5 * W @ W
    return np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th ** 2 * W @ W


def so3_log(M):
    """w with exp([w]x) = M, |w| <= pi"""
    s = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    c = 0.5 * (np.trace(M) - 1.0)
    th = np.arctan2(np.linalg.norm(s), c)
    if c > -0.5:
        return (1.0 + th * th / 6.0 if th < 1e-4 else th / np.linalg.norm(s)) * s
    S = 0.5 * (M + M.T) - c * np.eye(3)
    k = int(np.argmax(np.diag(S)))
    a = S[:, k] / np.sqrt((1.0 - c) * S[k, k])
    return th * (a if a @ s >= 0 else -a)


def jl_inv(w):
    th = float(np.linalg.norm(w))
    W = hat(w)
    c2 = 1 / 12 + th * th / 720 if th < 1e-4 else (1 - 0.5 * th / np.tan(0.5 * th)) / th ** 2
    return np.eye(3) - 0.5 * W + c2 * W @ W


def chart_R(R0, v):
    w = np.sqrt(1.0 - v @ v)
    return bd.quat_to_R(w, v[0], v[1], v[2]) @ R0


def chart_factor(v):
    """J_q: w = J_q dv for R(q(v + dv)) R(q(v))^T = exp([w]x)"""
    wq = np.sqrt(1.0 - v @ v)
    return 2.0 * (wq * np.eye(3) + hat(v) + np.outer(v, v) / wq)


def prior_residual(R0, v, t, Rp, tp):
    return np.concatenate([so3_log(chart_R(R0, v) @ Rp.T), t - tp])


def prior_jacobian(R0, v, t, Rp, tp):
    """dr / d(v, t) [6, 6] in the solver's chart"""
    r = prior_residual(R0, v, t, Rp, tp)
    J = np.zeros((6, 6))
    J[:3, :3] = jl_inv(r[:3]) @ chart_factor(v)
    J[3:, 3:] = np.eye(3)
    return J


def omega_jacobian(R, t, Rp, tp):
    """dr / d(w, t) [6, 6] in the chart of camCov"""
    r = prior_residual(R, np.zeros(3), t, Rp, tp)
    J = np.eye(6)
    J[:3, :3] = jl_inv(r[:3])
    return J


def residuals(prob, pr):
    """r [k, 6] of every prior at prob's parameters"""
    Rs = prob.R.reshape(-1, 3, 3)
    return np.array([prior_residual(Rs[j], np.zeros(3), prob.t[j], pr.R[k], pr.t[k])
                     for k, j in enumerate(pr.cams)]).reshape(-1, 6)


def prior_cost(prob, pr):
    rw = np.einsum("kab,kb->ka", pr.factors(), residuals(prob, pr))
    return float((rw * rw).sum())


def _rows(prob, pr, jac):
    """whitened prior rows: (Jw [k, 6, 6], rw [k, 6], columns [k, 6])"""
    L = pr.factors()
    Rs = prob.R.reshape(-1, 3, 3)
    J = np.array([jac(Rs[j], prob.t[j], pr.R[k], pr.t[k]) for k, j in enumerate(pr.cams)]).reshape(-1, 6, 6)
    rw = np.einsum("kab,kb->ka", L, residuals(prob, pr))
    cols = 6 * (pr.cams[:, None] - prob.m_con) + np.arange(6)
    return np.einsum("kab,kbc->kac", L, J), rw, cols


def _solver_jac(R, t, Rp, tp):
    return prior_jacobian(R, np.zeros(3), t, Rp, tp)


class PTrial(od.WTrial):
    """The dense first LM trial of a round with the prior rows L J and residuals -L r (the system's e is x - h, and
    a prior's "x - h" is -r) appended to the whitened observation rows.  The error bounds of ba_dense carry over;
    the prior rows are formed from exact inputs, so they add no cancellation term."""

    def __init__(self, prob, opt, covx, pr):
        super().__init__(prob, opt, np.tile(np.eye(2), (prob.nobs, 1, 1)) if covx is None else covx)
        self.pr = pr
        self.w_obs = self.w
        Jp, rw, cols = _rows(prob, pr, _solver_jac)
        k = len(pr)
        r = np.repeat(np.arange(6 * k).reshape(k, 6, 1), 6, 2) + 2 * prob.nobs
        c = np.repeat(cols[:, None, :], 6, 1)
        shape = (2 * prob.nobs + 6 * k, self.np)
        extra = sp.csr_matrix((Jp.ravel(), (r.ravel(), c.ravel())), shape=shape)
        extra_abs = sp.csr_matrix((np.abs(Jp).ravel(), (r.ravel(), c.ravel())), shape=shape)
        self.J = sp.vstack([self.J, sp.csr_matrix((6 * k, self.np))]).tocsr() + extra
        self.Jabs = sp.vstack([self.Jabs, sp.csr_matrix((6 * k, self.np))]).tocsr() + extra_abs
        self.e = np.concatenate([self.e, -rw.ravel()])
        # backward_tol's per-row error terms: none on the prior rows (three pseudo-observations of two rows each)
        self.rho = np.concatenate([self.rho, np.zeros(3 * k)])
        self.delta = np.concatenate([self.delta, np.zeros(3 * k)])
        self.w = np.concatenate([self.w_obs, np.ones(3 * k)])
        H = (self.J.T @ self.J).toarray()
        self.mu = opt.opts[0] * H.diagonal().max()
        self.A = H + self.mu * np.eye(self.np)
        self.g = self.J.T @ self.e
        self.d = np.linalg.solve(self.A, self.g)
        self.cost_obs0 = self.cost0
        self.cost0 = self.cost_obs0 + float((rw * rw).sum())
        self.Anorm = np.abs(self.A).sum(1).max()
        self.kappa = self.Anorm * np.abs(np.linalg.inv(self.A)).sum(1).max()

    def cost(self, state):
        return od.whitened_cost(state, self.w_obs, self.L) + prior_cost(state, self.pr)

    def cost_tol(self, state):
        """WTrial's bound on the observation part, relative to the whole cost, plus 1e-12 for the priors"""
        w, self.w = self.w, self.w_obs
        try:
            c_obs = od.whitened_cost(state, self.w_obs, self.L)
            err = (super().cost_tol(state) - 1e-12) * c_obs
        finally:
            self.w = w
        return 1e-12 + err / (c_obs + prior_cost(state, self.pr))


def check_ptrial(prob, covx, pr, info, after, opt):
    """ba_dense.check_trial on the prior-augmented system."""
    T = PTrial(prob, opt, covx, pr)
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


def identity_covx(prob):
    return np.tile(np.eye(2), (prob.nobs, 1, 1))


def normal_equations(prob, max_err, covx, pr):
    """(H, g) of the observations (ba_obscov_dense.normal_equations) plus the priors' J^T P^-1 J and -J^T P^-1 r,
    over the free parameters in the solver's chart at v = 0."""
    H, g = od.normal_equations(prob, max_err, identity_covx(prob) if covx is None else covx)
    Jp, rw, cols = _rows(prob, pr, _solver_jac)
    for k in range(len(pr)):
        H[np.ix_(cols[k], cols[k])] += Jp[k].T @ Jp[k]
        g[cols[k]] -= Jp[k].T @ rw[k]
    return H, g


def total_cost(prob, covx, pr, max_err=0.0):
    e = bd.residuals(prob)
    w = bd.tukey_weights(np.sqrt((e * e).sum(1)), max_err)
    return od.whitened_cost(prob, w, od.factors(identity_covx(prob) if covx is None else covx)) + prior_cost(prob, pr)


def cov_full(prob, max_err, pixel_var, covx, pr):
    """(camCov [m, 6, 6], ptCov [n, 3, 3], info, H) of ba_cov_dense.cov_full on the whitened system with the priors'
    information J_w^T P^-1 J_w (J_w = diag(Jl^-1(r_w), I)) added to the camera blocks.  sigma2_hat = (sum w e^T Lambda
    e + sum r^T P^-1 r) / (dof + 6 #priors); info["singular"] when H is not invertible."""
    covx = identity_covx(prob) if covx is None else covx
    Lx = od.factors(covx)
    e, w, unc = cd.weights(prob, max_err)
    J = np.einsum("nab,nbk->nak", Lx, cd.omega_jacobian(prob)) * np.sqrt(w)[:, None, None]
    cols, _ = bd.layout(prob)
    mf = prob.m - prob.m_con
    keep_pts = [i for i in range(prob.n_con, prob.n) if not unc[i]]
    pos = {i: 6 * mf + 3 * k for k, i in enumerate(keep_pts)}
    npar = 6 * mf + 3 * len(keep_pts)
    pt_of = bd.point_of(prob)
    H = np.zeros((npar, npar))
    for o in range(prob.nobs):
        c = np.full(9, -1, np.int64)
        c[:6] = cols[o, :6]
        if pt_of[o] in pos:
            c[6:] = pos[pt_of[o]] + np.arange(3)
        ok = c >= 0
        Jo = J[o][:, ok]
        H[np.ix_(c[ok], c[ok])] += Jo.T @ Jo
    Jp, rw, pcols = _rows(prob, pr, omega_jacobian)
    for k in range(len(pr)):
        H[np.ix_(pcols[k], pcols[k])] += Jp[k].T @ Jp[k]
    info = cd._info(prob, e, w, unc, pixel_var)
    info["dof"] += 6 * len(pr)
    ew = np.einsum("nab,nb->na", Lx, e)
    num = float((w * (ew * ew).sum(1)).sum()) + float((rw * rw).sum())
    info["sigma2_hat"] = num / info["dof"] if info["dof"] > 0 else np.nan
    info["priors"] = len(pr)
    info["singular"] = bool(npar and cd.min_relative_pivot(H) < 1e-12)
    C = pixel_var * np.linalg.inv(H) if npar and not info["singular"] else np.full((npar, npar), np.nan)
    cols_cam = {j: 6 * (j - prob.m_con) + np.arange(6) for j in range(prob.m_con, prob.m)}
    cols_pt = {i: pos[i] + np.arange(3) for i in keep_pts}
    cam, pt = cd._blocks(prob, C, cols_cam, cols_pt, unc)
    return cam, pt, info, H


# ---------------------------------------------------------------- priors for the tests
def random_cov(k, rng, sig_w=(0.002, 0.01), sig_t=(0.005, 0.03)):
    """k covariances for (w, dt): standard deviations uniform in the given ranges (rad, m), and a random correlation
    matrix (G G^T + 6 I scaled to a unit diagonal) that couples rotation and translation"""
    out = np.empty((k, 6, 6))
    for q in range(k):
        s = np.concatenate([rng.uniform(*sig_w, 3), rng.uniform(*sig_t, 3)])
        G = rng.normal(size=(6, 6))
        C = G @ G.T + 6 * np.eye(6)
        d = 1 / np.sqrt(np.diag(C))
        C = C * d[:, None] * d[None, :]
        out[q] = s[:, None] * C * s[None, :]
        out[q] = 0.5 * (out[q] + out[q].T)
    return out


def draw_means(prob, cams, cov, rng):
    """(R_p, t_p) with r at prob's parameters drawn from N(0, P): R = exp([r_w]x) R_p, t = t_p + r_t"""
    Rs = prob.R.reshape(-1, 3, 3)
    Rp, tp = [], []
    for k, j in enumerate(cams):
        r = np.linalg.cholesky(cov[k]) @ rng.normal(size=6)
        Rp.append(so3_exp(-r[:3]) @ Rs[j])
        tp.append(prob.t[j] - r[3:])
    return np.array(Rp), np.array(tp)


def offset_means(prob, cams, rng, deg=5.0, dist=0.05):
    """means a fixed distance away from prob's cameras (deg degrees about a random axis, dist along a random
    direction), re-orthonormalised to roundoff"""
    Rs = prob.R.reshape(-1, 3, 3)
    Rp, tp = [], []
    for j in cams:
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        b = rng.normal(size=3)
        b /= np.linalg.norm(b)
        Rp.append(so3_exp(np.deg2rad(deg) * a) @ Rs[j])
        tp.append(prob.t[j] + dist * b)
    Rp = np.array(Rp)
    U, _, Vt = np.linalg.svd(Rp)
    return U @ Vt, np.array(tp)
