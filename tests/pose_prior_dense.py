"""float64 references of the pose solve and its covariance stage with Gaussian pose priors
(cosl_pose_solver_submit_prior; DESIGN.md 5.3), built on pose_dense, pose_obscov_dense and pose_cov_dense.

A prior on a camera has a mean (R_p, t_p) and a 6x6 covariance P for (w, dt) in the solver's chart R = R_p exp([w]x),
t = t_p + dt.  With the upper-triangular L, L^T L = P^-1, its residual and rows are

    r = [Log(R_p^T R); t - t_p],  rows L J_p, residual L r,  J_p = diag(Jr^-1(r_w), I)

for the solver's update R' = R exp([dw]x), t' = t + dt, with Jr^-1 the inverse right Jacobian of SO(3).  Every cost
gains |L r|^2; the LM step adds (L J_p)^T (L J_p) to the system and -(L J_p)^T (L r) to its right-hand side before
lambda, without a Tukey weight; the weights stay on the pixel distance.  The stage adds J_p^T P^-1 J_p to H, 6 to dof
and r^T P^-1 r to sigma2_hat's numerator.

    prior_record(R, t, P)        -> (L, R_p, t_p)
    log_so3(M), jr_inv(phi)      -> the rotation log (exact to pi) and Jr^-1
    residual(R, t, rec)          -> r
    rows(R, t, rec)              -> (L J_p, L r)
    estimate(..., prior)         -> (ok, R, t, fields) as pose_obscov_dense.estimate
    cov_stage(..., prior)        -> pose_obscov_dense.cov_stage's dict with the prior in H, dof and sigma2_hat
    apply(R, t, x)               -> (R exp([x_w]x), t + x_t): the chart
    random_prior / drawn_prior   -> random test priors: a mean at a chosen distance, or drawn from P itself"""
import math

import numpy as np

import pose_cov_dense as cd
import pose_dense as pd
import pose_obscov_dense as od


def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def prior_record(R, t, P):
    """(L, R_p, t_p) with L upper triangular, L^T L = P^-1."""
    P = np.asarray(P, np.float64).reshape(6, 6)
    C = np.linalg.cholesky(np.linalg.inv(0.5 * (P + P.T)))
    return C.T, np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)


def log_so3(M):
    """Log of the rotation M by atan2, the axis from the skew part below 120 degrees and from the symmetric part
    above: exact to roundoff all the way to pi."""
    s = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    sn = math.sqrt(s @ s)
    cs = 0.5 * (M[0, 0] + M[1, 1] + M[2, 2] - 1.0)
    th = math.atan2(sn, cs)
    if cs > -0.5:
        return (1.0 + th * th / 6.0 if th < 1e-4 else th / sn) * s
    S = 0.5 * (M + M.T) - cs * np.eye(3)  # (1 - cos th) a a^T
    c = int(np.argmax(np.diag(S)))
    a = S[:, c] / math.sqrt((1.0 - cs) * S[c, c])
    return th * (-a if a @ s < 0 else a)


def jr_inv(phi):
    """Jr^-1(phi) = I + [phi]x / 2 + (1 / th^2 - (1 + cos th) / (2 th sin th)) [phi]x^2."""
    th = math.sqrt(phi @ phi)
    W = skew(phi)
    c2 = (1.0 / 12.0 + th * th / 720.0 if th < 1e-2
          else 1.0 / (th * th) - (1.0 + math.cos(th)) / (2.0 * th * math.sin(th)))
    return np.eye(3) + 0.5 * W + c2 * (W @ W)


def apply(R, t, x):
    """The solver's chart: (R exp([x_w]x), t + x_t)."""
    return np.asarray(R) @ pd.exp_map(x[:3]), np.asarray(t) + x[3:]


def residual(R, t, rec):
    _, Rp, tp = rec
    return np.concatenate([log_so3(Rp.T @ np.asarray(R)), np.asarray(t) - tp])


def rows(R, t, rec):
    """(L J_p, L r) at (R, t)."""
    L = rec[0]
    r = residual(R, t, rec)
    J = np.eye(6)
    J[:3, :3] = jr_inv(r[:3])
    return L @ J, L @ r


def prior_cost(R, t, rec):
    _, Lr = rows(R, t, rec)
    return float(Lr @ Lr)


def cost(K, R, t, W, Ms, ms, L, rec):
    c = od.cost(K, R, t, W, Ms, ms, L)
    return c if rec is None else c + prior_cost(R, t, rec)


def one_step(K, R, t, Ms, ms, W, lam, L, rec):
    """One LM step at (R, t): the whitened observation rows of pose_obscov_dense plus the prior's, then lambda."""
    u0, v0 = pd.project(K, R, t, Ms)
    Ju, Jv = pd._jacobian_fd(K, R, t, Ms, u0, v0)
    Ju, Jv = L[:, 0:1] * Ju + L[:, 1:2] * Jv, L[:, 2:3] * Jv
    r0, r1 = od.whiten(L, ms[:, 0] - u0, ms[:, 1] - v0)
    A, b = pd._normal(Ju, Jv, W, r0, r1)
    if rec is not None:
        LJ, Lr = rows(R, t, rec)
        A = A + LJ.T @ LJ
        b = b - LJ.T @ Lr
    S, d = pd._solve(A, b, lam)
    return S, b, d


def estimate(K, R0, t0, Ms, ms, tau, prev=None, opt=pd.DEFAULT_OPT, covx=None, prior=None, trace=None):
    """pose_obscov_dense.estimate with the prior (R, t, P) or None in every cost and step."""
    rec = None if prior is None else prior_record(*prior)
    maxIterLM, maxIterRW, epsErr, epsParam, epsRW, lambda0 = opt
    K = np.asarray(K, np.float64).reshape(3, 3)
    Ms = np.asarray(Ms, np.float64).reshape(-1, 3)
    ms = np.asarray(ms, np.float64).reshape(-1, 2)
    n = len(Ms)
    L = od.factors(od.identity(n) if covx is None else covx)
    W = pd.prev_weights(n, tau, prev)
    R, t = np.array(R0, np.float64).reshape(3, 3), np.array(t0, np.float64)
    R_opt, t_opt = R.copy(), t.copy()
    f = dict(lambda_=lambda0, lambda0=lambda0, err0=0.0, err=0.0, errRW=-1.0, retTypeLM=1, npts=n,
             nIterLM=0, nIterRW=0)
    note = trace.append if trace is not None else (lambda m: None)
    ok = True
    k = 0
    while k < maxIterRW:
        lam = f["lambda0"]
        err0 = cost(K, R, t, W, Ms, ms, L, rec)
        errLM = err = err0
        Rl, tl, R_tmp, t_tmp = R, t, R, t
        ret, i = 1, 0
        while i < maxIterLM:
            _, _, p = one_step(K, Rl, tl, Ms, ms, W, lam, L, rec)
            R_opt, t_opt = pd.mat33(Rl, pd.exp_map(p[:3])), tl + p[3:]
            p2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] + p[4] * p[4] + p[5] * p[5]
            note((f"rw{k} lm{i} p2", pd._rel(p2, epsParam)))
            if p2 < epsParam:
                Rl, tl, ret = R_opt, t_opt, 0
                break
            err = cost(K, R_opt, t_opt, W, Ms, ms, L, rec)
            note((f"rw{k} lm{i} |derr|", pd._rel(abs(err - errLM), epsErr)))
            if abs(err - errLM) < epsErr:
                ret = 0
                break
            big = max(abs(err), abs(errLM))
            note((f"rw{k} lm{i} accept", abs(err - errLM) / big if big > 0 else math.inf))
            if err <= errLM:
                Rl, tl, R_tmp, t_tmp, errLM = R_opt, t_opt, R_opt, t_opt, err
                lam /= 10
            else:
                lam *= 10
                if lam > 1e18:
                    ret = -1
                    break
            i += 1
        if ret == -1:
            R_opt, t_opt = R_tmp, t_tmp
        f.update(lambda_=lam, err0=err0, err=err, retTypeLM=ret, nIterLM=i)
        if ret < 0:
            ok = False
            break
        f["lambda0"] = lam
        if f["errRW"] < 0:
            f["errRW"] = err
        else:
            note((f"rw{k} |derrRW|", pd._rel(abs(err - f["errRW"]), epsRW)))
            if abs(err - f["errRW"]) < epsRW:
                break
            f["errRW"] = err
        R, t = R_opt, t_opt
        e = cd.residuals(K, R, t, Ms, ms)  # the Tukey weights stay on the pixel distance
        if n:
            note((f"rw{k} tukey", float(np.min(np.abs(e - tau))) / tau))
        W = pd.weights(e, tau)
        k += 1
    f["nIterRW"] = k
    return ok, R_opt, t_opt, f


def margins(K, R0, t0, Ms, ms, tau, prev=None, opt=pd.DEFAULT_OPT, covx=None, prior=None):
    """(label, relative distance from its threshold) of every decision on estimate's trajectory."""
    trace = []
    estimate(K, R0, t0, Ms, ms, tau, prev, opt, covx, prior, trace)
    return trace


def cov_stage(K, R, t, Ms, ms, tau, pixel_var, covx=None, prior=None):
    """pose_obscov_dense.cov_stage with the prior: H += (L J_p)^T (L J_p), dof += 6, sigma2_hat's numerator +=
    |L r|^2, all at (R, t)."""
    d = od.cov_stage(K, R, t, Ms, ms, tau, pixel_var, covx)
    if prior is None:
        return d
    LJ, Lr = rows(np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64), prior_record(*prior))
    live = d["w"] > 0
    H = d["H"] + LJ.T @ LJ
    dof = d["dof"] + 6
    if covx is None:
        ew = d["e"]
    else:
        u, v = pd.project(np.asarray(K, np.float64).reshape(3, 3), np.asarray(R, np.float64).reshape(3, 3),
                          np.asarray(t, np.float64), np.asarray(Ms, np.float64).reshape(-1, 3))
        ms = np.asarray(ms, np.float64).reshape(-1, 2)
        r0, r1 = od.whiten(od.factors(covx), u - ms[:, 0], v - ms[:, 1])
        ew = np.sqrt(r0 * r0 + r1 * r1)
    num = pd.fsum(np.concatenate([d["w"][live] * (ew * ew)[live], [float(Lr @ Lr)]]))
    sigma2_hat = num / dof if dof > 0 else math.nan
    try:
        C = np.linalg.cholesky(H)
        min_pivot = float(np.min(np.diag(C) ** 2 / np.diag(H)))
    except np.linalg.LinAlgError:
        min_pivot = 0.0
    valid = min_pivot >= cd.MIN_PIVOT
    cov = pixel_var * np.linalg.inv(H) if valid else np.full((6, 6), math.nan)
    return dict(d, H=H, cov=cov, dof=dof, sigma2_hat=sigma2_hat, min_pivot=min_pivot, valid=valid)


def random_prior(R, t, rng, max_deg=30.0, cond=1e4, scale=1e-3):
    """A prior whose mean lies up to max_deg degrees and about 0.1 units from (R, t), with a random covariance of
    condition number cond and largest eigenvalue scale."""
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = math.radians(rng.uniform(0.0, max_deg))
    Rp = np.asarray(R) @ pd.exp_map(ang * ax)
    tp = np.asarray(t) + rng.normal(0.0, 0.1 / math.sqrt(3.0), 3)
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    ev = scale * np.geomspace(1.0, 1.0 / cond, 6)
    P = (Q * ev) @ Q.T
    return Rp, tp, 0.5 * (P + P.T)


def drawn_prior(R, t, rng, max_deg=30.0, cond=1e4, scale=0.04):
    """A prior (R_p, t_p, P) that (R, t) is a draw of: P random with condition number cond and largest eigenvalue
    scale, (R, t) = apply(R_p, t_p, x) with x ~ N(0, P), redrawn until the rotation part is below max_deg degrees."""
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    ev = scale * np.geomspace(1.0, 1.0 / cond, 6)
    P = (Q * ev) @ Q.T
    P = 0.5 * (P + P.T)
    while True:
        x = rng.multivariate_normal(np.zeros(6), P)
        if np.linalg.norm(x[:3]) < math.radians(max_deg):
            break
    Rp = np.asarray(R) @ pd.exp_map(-x[:3])
    return Rp, np.asarray(t) - x[3:], P
