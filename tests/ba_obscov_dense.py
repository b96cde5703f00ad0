"""float64 references of a bundle adjustment whose observations carry 2x2 measurement covariances
(cosl_ba_solver_set_obs_cov, cosl_sba_motstr_levmar_x_cov; DESIGN.md 4.7).

With Lambda_k = Sigma_k^-1 = L_k^T L_k (L_k upper triangular) the least-squares term of observation k is
w_k e_k^T Lambda_k e_k: the residual and the Jacobian rows of observation k are whitened, e' = L e and J' = L J, and the
normal equations are those of ba_dense on (e', J').  The Tukey weights w stay on the pixel distance |e_k|.

  - WTrial: ba_dense.Trial on the whitened system (one damped LM trial), check_wtrial its check_trial;
  - normal_equations: the undamped H = J^T W Lambda J and g = J^T W Lambda e at a problem's parameters;
  - cov_full: pixel_var (J^T W Lambda J)^-1 over the free parameters, as ba_cov_dense.cov_full, and sigma2_hat =
    sum w e^T Lambda e / dof;
  - random_covx / draw_noise: heteroscedastic, anisotropic covariances and noise drawn from them."""
import numpy as np
import scipy.sparse as sp

import ba_cov_dense as cd
import ba_dense as bd


def factors(covx):
    """L [N, 2, 2], upper triangular, with L^T L = covx^-1."""
    lam = np.linalg.inv(np.asarray(covx, np.float64).reshape(-1, 2, 2))
    return np.linalg.cholesky(lam).transpose(0, 2, 1)


def random_covx(N, rng, lo=0.3, hi=1.5):
    """N covariances with standard deviations uniform in [lo, hi] px along two random orthogonal axes:
    [N, 2, 2] and the square roots (R diag(s)) [N, 2, 2] that draw_noise uses."""
    th = rng.uniform(0, np.pi, N)
    s = rng.uniform(lo, hi, (N, 2))
    R = np.stack([np.stack([np.cos(th), -np.sin(th)], -1), np.stack([np.sin(th), np.cos(th)], -1)], -2)
    S = R * s[:, None, :]
    return S @ S.transpose(0, 2, 1), S


def draw_noise(S, rng):
    return np.einsum("nab,nb->na", S, rng.normal(size=(len(S), 2)))


def whitened_cost(prob, w, L):
    e = np.einsum("nab,nb->na", L, bd.residuals(prob))
    return float((w * (e * e).sum(1)).sum())


class WTrial(bd.Trial):
    """The dense first LM trial of a round on the whitened system.  The error bounds of ba_dense carry over with the
    whitening's entries: |L| |J| bounds the entries of J', and the rows of |L| the pixel error delta of e'."""

    def __init__(self, prob, opt, covx):
        self.prob = prob
        self.L = factors(covx)
        Labs = np.abs(self.L)
        e = bd.residuals(prob)
        self.w = bd.tukey_weights(np.sqrt((e * e).sum(1)), opt.max_err)
        cols, self.np = bd.layout(prob)
        Jr = bd.local_jacobian(prob)
        Jl = np.einsum("nab,nbk->nak", self.L, Jr)
        Ja = np.einsum("nab,nbk->nak", Labs, np.abs(Jr))
        rows = np.arange(2 * prob.nobs).reshape(-1, 2)
        sw = np.sqrt(self.w)
        keep = np.broadcast_to(cols[:, None, :] >= 0, Jl.shape)
        r = np.broadcast_to(rows[:, :, None], Jl.shape)[keep]
        c = np.broadcast_to(cols[:, None, :], Jl.shape)[keep]
        self.Jl = Jl
        self.J = sp.csr_matrix(((Jl * sw[:, None, None])[keep], (r, c)), shape=(2 * prob.nobs, self.np))
        self.Jabs = sp.csr_matrix(((Ja * sw[:, None, None])[keep], (r, c)), shape=self.J.shape)
        ew = np.einsum("nab,nb->na", self.L, e)
        self.e = (ew * sw[:, None]).ravel()
        H = (self.J.T @ self.J).toarray()
        self.mu = opt.opts[0] * H.diagonal().max()
        self.A = H + self.mu * np.eye(self.np)
        self.g = self.J.T @ self.e
        self.d = np.linalg.solve(self.A, self.g)
        self.cost0 = float((self.w * (ew * ew).sum(1)).sum())
        self.rho, delta = bd.cancellation(prob)
        self.lrow = Labs.sum(2).max(1)  # per observation: the largest row sum of |L|
        self.delta = delta * self.lrow
        self.Anorm = np.abs(self.A).sum(1).max()
        self.kappa = self.Anorm * np.abs(np.linalg.inv(self.A)).sum(1).max()

    def cost(self, state):
        return whitened_cost(state, self.w, self.L)

    def cost_tol(self, state):
        e = np.einsum("nab,nb->na", self.L, bd.residuals(state))
        _, delta = bd.cancellation(state)
        delta = delta * self.lrow
        c = (self.w * (e * e).sum(1)).sum()
        return 1e-12 + float((self.w * (2 * np.sqrt((e * e).sum(1)) * delta + 2 * delta * delta)).sum() / c)


def check_wtrial(prob, covx, info, after, opt):
    """ba_dense.check_trial on the whitened system."""
    T = WTrial(prob, opt, covx)
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


def normal_equations(prob, max_err, covx):
    """(H, g) = (J^T W Lambda J, J^T W Lambda e) over the free parameters in the solver's chart at v = 0, with the
    Tukey weights of the pixel distances at prob's parameters (all 1 for max_err <= 0)."""
    e = bd.residuals(prob)
    w = bd.tukey_weights(np.sqrt((e * e).sum(1)), max_err)
    L = factors(covx)
    J = np.einsum("nab,nbk->nak", L, bd.local_jacobian(prob)) * np.sqrt(w)[:, None, None]
    ew = np.einsum("nab,nb->na", L, e) * np.sqrt(w)[:, None]
    cols, npar = bd.layout(prob)
    H = np.zeros((npar, npar))
    g = np.zeros(npar)
    for o in range(prob.nobs):
        c = cols[o]
        ok = c >= 0
        Jo = J[o][:, ok]
        H[np.ix_(c[ok], c[ok])] += Jo.T @ Jo
        g[c[ok]] += Jo.T @ ew[o]
    return H, g


def cov_full(prob, max_err, pixel_var, covx):
    """(camCov, ptCov, info, H) of ba_cov_dense.cov_full on the whitened system; sigma2_hat = sum w e^T Lambda e / dof
    over the observations that enter H."""
    L = factors(covx)
    cam, pt, info, H = cd.cov_full(prob, max_err, pixel_var,
                                   jac=lambda p: np.einsum("nab,nbk->nak", L, cd.omega_jacobian(p)))
    _, w, _ = cd.weights(prob, max_err)
    info["sigma2_hat"] = whitened_cost(prob, w, L) / info["dof"] if info["dof"] > 0 else np.nan
    return cam, pt, info, H
