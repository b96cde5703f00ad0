"""float64 references of a bundle adjustment with Gaussian position priors on free points (cosl_ba_solver_set_pt_prior;
DESIGN.md 4.9), on top of ba_prior_dense (camera priors) and ba_obscov_dense.

A prior on free point i has a mean mu and a 3x3 covariance P in world coordinates.  Its residual is r = X_i - mu and
its term of the objective r^T P^-1 r = |L r|^2 with L = chol(P^-1)^T (upper triangular).  Its Jacobian is the
identity in every chart, so the normal equations gain L^T L on the point block and -L^T L r in the gradient.

  - PPTrial: the dense first LM trial with the point-prior rows (and camera-prior rows when those are set too)
    appended to the whitened observation rows, check_pptrial its check_trial;
  - normal_equations: the undamped H and g (observations plus both kinds of priors) at a problem's parameters;
  - cov_full: pixel_var H^-1 over the free parameters, where a free point with a prior always stays in H, sigma2_hat
    and dof with three measurements per point prior (six per camera prior);
  - no_cam_priors / random_pt_cov / draw_pt_means: priors for the tests."""
import numpy as np
import scipy.sparse as sp

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
import ba_prior_dense as pd


class PtPriors:
    """pts [k], X [k, 3], cov [k, 3, 3]"""

    def __init__(self, pts, X, cov):
        self.pts = np.asarray(pts, np.int64).reshape(-1)
        self.X = np.asarray(X, np.float64).reshape(-1, 3)
        self.cov = np.asarray(cov, np.float64).reshape(-1, 3, 3)

    def __len__(self):
        return len(self.pts)

    def factors(self):
        """L [k, 3, 3] upper triangular with L^T L = P^-1"""
        if not len(self):
            return np.zeros((0, 3, 3))
        return np.linalg.cholesky(np.linalg.inv(self.cov)).transpose(0, 2, 1)

    def subset(self, keep):
        return PtPriors(self.pts[keep], self.X[keep], self.cov[keep])


def no_cam_priors():
    return pd.Priors(np.zeros(0), np.zeros((0, 3, 3)), np.zeros((0, 3)), np.zeros((0, 6, 6)))


def no_pt_priors():
    return PtPriors(np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3, 3)))


def _cam(pr):
    return no_cam_priors() if pr is None else pr


def residuals(prob, pp):
    """r [k, 3] of every point prior at prob's parameters"""
    return (prob.X[pp.pts] - pp.X).reshape(-1, 3)


def pt_prior_cost(prob, pp):
    rw = np.einsum("kab,kb->ka", pp.factors(), residuals(prob, pp))
    return float((rw * rw).sum())


def _cam_prior_cost(prob, pr):
    return pd.prior_cost(prob, pr) if len(pr) else 0.0


def _pt_cols(prob, pp):
    mf = prob.m - prob.m_con
    return 6 * mf + 3 * (pp.pts[:, None] - prob.n_con) + np.arange(3)


class PPTrial(pd.PTrial):
    """The dense first LM trial of a round with each point prior's rows L and residuals -L r appended to PTrial's
    system (observations, then camera priors).  Each point prior takes four rows, the last one zero, so that it is
    two pseudo-observations of two rows for the per-row error terms, which are zero on prior rows."""

    def __init__(self, prob, opt, covx, pr, pp):
        pr = _cam(pr)
        if len(pr):
            super().__init__(prob, opt, covx, pr)
        else:  # PTrial's system without camera rows
            od.WTrial.__init__(self, prob, opt, pd.identity_covx(prob) if covx is None else covx)
            self.pr = pr
            self.w_obs = self.w
            self.cost_obs0 = self.cost0
        self.pp = pp
        k = len(pp)
        L = pp.factors()
        rw = np.einsum("kab,kb->ka", L, residuals(prob, pp))
        J4 = np.zeros((k, 4, 3))
        J4[:, :3] = L
        rows = self.J.shape[0] + np.arange(4 * k).reshape(k, 4, 1).repeat(3, 2)
        cols = np.repeat(_pt_cols(prob, pp)[:, None, :], 4, 1)
        shape = (self.J.shape[0] + 4 * k, self.np)
        extra = sp.csr_matrix((J4.ravel(), (rows.ravel(), cols.ravel())), shape=shape)
        extra_abs = sp.csr_matrix((np.abs(J4).ravel(), (rows.ravel(), cols.ravel())), shape=shape)
        self.J = sp.vstack([self.J, sp.csr_matrix((4 * k, self.np))]).tocsr() + extra
        self.Jabs = sp.vstack([self.Jabs, sp.csr_matrix((4 * k, self.np))]).tocsr() + extra_abs
        e4 = np.zeros((k, 4))
        e4[:, :3] = -rw
        self.e = np.concatenate([self.e, e4.ravel()])
        self.rho = np.concatenate([self.rho, np.zeros(2 * k)])
        self.delta = np.concatenate([self.delta, np.zeros(2 * k)])
        self.w = np.concatenate([self.w, np.ones(2 * k)])
        H = (self.J.T @ self.J).toarray()
        self.mu = opt.opts[0] * H.diagonal().max()
        self.A = H + self.mu * np.eye(self.np)
        self.g = self.J.T @ self.e
        self.d = np.linalg.solve(self.A, self.g)
        self.cost0 = self.cost_obs0 + _cam_prior_cost(prob, self.pr) + float((rw * rw).sum())
        self.Anorm = np.abs(self.A).sum(1).max()
        self.kappa = self.Anorm * np.abs(np.linalg.inv(self.A)).sum(1).max()

    def cost(self, state):
        return (od.whitened_cost(state, self.w_obs, self.L) + _cam_prior_cost(state, self.pr) +
                pt_prior_cost(state, self.pp))

    def cost_tol(self, state):
        """WTrial's bound on the observation part, relative to the whole cost, plus 1e-12 for the priors"""
        w, self.w = self.w, self.w_obs
        try:
            c_obs = od.whitened_cost(state, self.w_obs, self.L)
            err = (od.WTrial.cost_tol(self, state) - 1e-12) * c_obs
        finally:
            self.w = w
        return 1e-12 + err / (c_obs + _cam_prior_cost(state, self.pr) + pt_prior_cost(state, self.pp))


def check_pptrial(prob, covx, pr, pp, info, after, opt):
    """ba_dense.check_trial on the prior-augmented system."""
    T = PPTrial(prob, opt, covx, pr, pp)
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


def normal_equations(prob, max_err, covx, pr, pp):
    """(H, g) of ba_prior_dense.normal_equations (observations and camera priors) plus the point priors' L^T L and
    -L^T L r, over the free parameters in the solver's chart at v = 0."""
    H, g = pd.normal_equations(prob, max_err, covx, _cam(pr))
    L = pp.factors()
    rw = np.einsum("kab,kb->ka", L, residuals(prob, pp))
    for k, c in enumerate(_pt_cols(prob, pp)):
        H[np.ix_(c, c)] += L[k].T @ L[k]
        g[c] -= L[k].T @ rw[k]
    return H, g


def total_cost(prob, covx, pr, pp, max_err=0.0):
    return pd.total_cost(prob, covx, _cam(pr), max_err) + pt_prior_cost(prob, pp)


def weights(prob, max_err, pp):
    """cd.weights where a free point with a prior is never left out of H"""
    e = bd.residuals(prob)
    w = bd.tukey_weights(np.sqrt((e * e).sum(1)), max_err)
    pt = bd.point_of(prob)
    cnt = np.bincount(pt[w > 0], minlength=prob.n)
    has = np.zeros(prob.n, bool)
    has[pp.pts] = True
    unc = (np.arange(prob.n) >= prob.n_con) & (cnt < 2) & ~has
    return e, np.where(unc[pt], 0.0, w), unc


def cov_full(prob, max_err, pixel_var, covx, pr, pp):
    """(camCov [m, 6, 6], ptCov [n, 3, 3], info, H) of ba_prior_dense.cov_full with the point priors' P^-1 added to
    their point blocks; a point with a prior stays in H whatever its observations.  sigma2_hat = (sum w e^T Lambda e
    + sum of both kinds of r^T P^-1 r) / (dof + 6 #camera priors + 3 #point priors); info["singular"] when H is not
    invertible."""
    pr = _cam(pr)
    covx = pd.identity_covx(prob) if covx is None else covx
    Lx = od.factors(covx)
    e, w, unc = weights(prob, max_err, pp)
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
    num = 0.0
    if len(pr):
        Jp, rwc, pcols = pd._rows(prob, pr, pd.omega_jacobian)
        for k in range(len(pr)):
            H[np.ix_(pcols[k], pcols[k])] += Jp[k].T @ Jp[k]
        num += float((rwc * rwc).sum())
    Lp = pp.factors()
    rwp = np.einsum("kab,kb->ka", Lp, residuals(prob, pp))
    for k, i in enumerate(pp.pts):
        c = pos[int(i)] + np.arange(3)
        H[np.ix_(c, c)] += Lp[k].T @ Lp[k]
    num += float((rwp * rwp).sum())
    info = cd._info(prob, e, w, unc, pixel_var)
    info["dof"] += 6 * len(pr) + 3 * len(pp)
    ew = np.einsum("nab,nb->na", Lx, e)
    num += float((w * (ew * ew).sum(1)).sum())
    info["sigma2_hat"] = num / info["dof"] if info["dof"] > 0 else np.nan
    info["priors"] = len(pr)
    info["pt_priors"] = len(pp)
    info["singular"] = bool(npar and cd.min_relative_pivot(H) < 1e-12)
    C = pixel_var * np.linalg.inv(H) if npar and not info["singular"] else np.full((npar, npar), np.nan)
    cols_cam = {j: 6 * (j - prob.m_con) + np.arange(6) for j in range(prob.m_con, prob.m)}
    cols_pt = {i: pos[i] + np.arange(3) for i in keep_pts}
    cam, pt = cd._blocks(prob, C, cols_cam, cols_pt, unc)
    return cam, pt, info, H


# ---------------------------------------------------------------- priors for the tests
def random_pt_cov(k, rng, sig=(0.005, 0.05)):
    """k 3x3 covariances: standard deviations uniform in sig (m) and a random correlation matrix"""
    out = np.empty((k, 3, 3))
    for q in range(k):
        s = rng.uniform(*sig, 3)
        G = rng.normal(size=(3, 3))
        C = G @ G.T + 3 * np.eye(3)
        d = 1 / np.sqrt(np.diag(C))
        C = C * d[:, None] * d[None, :]
        out[q] = s[:, None] * C * s[None, :]
        out[q] = 0.5 * (out[q] + out[q].T)
    return out


def draw_pt_means(prob, pts, cov, rng):
    """mu with r = X - mu at prob's points drawn from N(0, P)"""
    return np.array([prob.X[i] - np.linalg.cholesky(cov[k]) @ rng.normal(size=3) for k, i in enumerate(pts)])


def offset_pt_means(prob, pts, rng, dist=0.05):
    """means dist away from prob's points along random directions"""
    out = []
    for i in pts:
        b = rng.normal(size=3)
        out.append(prob.X[i] + dist * b / np.linalg.norm(b))
    return np.array(out).reshape(-1, 3)
