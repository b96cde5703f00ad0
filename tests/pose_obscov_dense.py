"""float64 references of the pose solve and its covariance stage with 2x2 measurement covariances
(cosl_pose_solver_submit_cov; DESIGN.md 5.2), built on pose_dense and pose_cov_dense.

With Sigma_i = [a b; b c] and det = ac - b^2 the whitening factor of point i is the upper-triangular
L_i = [sqrt(c/det), -b/sqrt(c det); 0, 1/sqrt(c)], L_i^T L_i = Sigma_i^-1, computed in the host's operation order.
The residual m_i - project and both forward-difference Jacobian rows are whitened by L_i before the Tukey weight,
so the cost is sum w |L (m - project)|^2 and the LM step pose_dense's on the whitened rows; the Tukey weights stay
on the pixel distance.  With Sigma = I, L = [1, -0; 0, 1] and every whitened value is the unwhitened one bit for
bit, so estimate(..., covx=identity) is pose_dense.estimate exactly.

    factors(covx)          -> [n, 3] (l00, l01, l11)
    estimate(..., covx)    -> (ok, R, t, fields) as pose_dense.estimate
    one_step(..., L)       -> (A + lam I, b, delta): one whitened forward-difference LM step
    cov_stage(..., covx)   -> pose_cov_dense.cov_stage with H = sum w (L J)^T (L J), sigma2_hat from |L e|^2
    random_covx / draw_noise: anisotropic covariances and noise drawn from them (ba_obscov_dense's)"""
import math

import numpy as np

import ba_obscov_dense as bod
import pose_cov_dense as cd
import pose_dense as pd

draw_noise = bod.draw_noise


def random_covx(n, rng, lo=0.15, hi=1.5):
    """n covariances with standard deviations uniform in [lo, hi] px along two random orthogonal axes (condition
    numbers up to (hi / lo)^2 = 100 by default): [n, 2, 2] and the square roots draw_noise uses."""
    return bod.random_covx(n, rng, lo, hi)


def factors(covx):
    """[n, 3] = (l00, l01, l11) of every covariance (None stays None)."""
    if covx is None:
        return None
    c = np.asarray(covx, np.float64).reshape(-1, 4)
    a, b, cc = c[:, 0], c[:, 1], c[:, 3]
    det = a * cc - b * b
    return np.stack([np.sqrt(cc / det), -b / np.sqrt(cc * det), 1.0 / np.sqrt(cc)], 1)


def identity(n):
    return np.tile(np.array([1.0, 0.0, 0.0, 1.0]), (n, 1))


def whiten(L, r0, r1):
    """(l00 r0 + l01 r1, l11 r1), each operation rounded once, as the kernel's whiten."""
    return L[:, 0] * r0 + L[:, 1] * r1, L[:, 2] * r1


def cost(K, R, t, W, Ms, ms, L):
    u, v = pd.project(K, R, t, Ms)
    dx, dy = whiten(L, ms[:, 0] - u, ms[:, 1] - v)
    return pd.fsum((dx * dx + dy * dy) * W)


def one_step(K, R, t, Ms, ms, W, lam, L):
    """One whitened forward-difference LM step at (R, t) with weights W: (A + lam I, b, delta)."""
    u0, v0 = pd.project(K, R, t, Ms)
    Ju, Jv = pd._jacobian_fd(K, R, t, Ms, u0, v0)
    Ju, Jv = L[:, 0:1] * Ju + L[:, 1:2] * Jv, L[:, 2:3] * Jv
    r0, r1 = whiten(L, ms[:, 0] - u0, ms[:, 1] - v0)
    A, b = pd._normal(Ju, Jv, W, r0, r1)
    S, d = pd._solve(A, b, lam)
    return S, b, d


def estimate(K, R0, t0, Ms, ms, tau, prev=None, opt=pd.DEFAULT_OPT, covx=None, trace=None):
    """pose_dense.estimate on the whitened residuals (covx [n, 2, 2] or [n, 4]; None = identity).  The LM control,
    the re-weighting and the option block are pose_dense's; trace receives (label, margin) of every decision."""
    maxIterLM, maxIterRW, epsErr, epsParam, epsRW, lambda0 = opt
    Ms = np.asarray(Ms, np.float64).reshape(-1, 3)
    ms = np.asarray(ms, np.float64).reshape(-1, 2)
    n = len(Ms)
    L = factors(identity(n) if covx is None else covx)
    W = pd.prev_weights(n, tau, prev)
    R, t = np.array(R0, np.float64), np.array(t0, np.float64)
    R_opt, t_opt = R.copy(), t.copy()
    f = dict(lambda_=lambda0, lambda0=lambda0, err0=0.0, err=0.0, errRW=-1.0, retTypeLM=1, npts=n,
             nIterLM=0, nIterRW=0)
    note = trace.append if trace is not None else (lambda m: None)
    ok = True
    k = 0
    while k < maxIterRW:
        lam = f["lambda0"]
        err0 = cost(K, R, t, W, Ms, ms, L)
        errLM = err = err0
        Rl, tl, R_tmp, t_tmp = R, t, R, t
        ret, i = 1, 0
        while i < maxIterLM:
            _, _, p = one_step(K, Rl, tl, Ms, ms, W, lam, L)
            R_opt, t_opt = pd.mat33(Rl, pd.exp_map(p[:3])), tl + p[3:]
            p2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] + p[4] * p[4] + p[5] * p[5]
            note((f"rw{k} lm{i} p2", pd._rel(p2, epsParam)))
            if p2 < epsParam:
                Rl, tl, ret = R_opt, t_opt, 0
                break
            err = cost(K, R_opt, t_opt, W, Ms, ms, L)
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


def margins(K, R0, t0, Ms, ms, tau, prev=None, opt=pd.DEFAULT_OPT, covx=None):
    """(label, relative distance from its threshold) of every decision on estimate's trajectory."""
    trace = []
    estimate(K, R0, t0, Ms, ms, tau, prev, opt, covx, trace)
    return trace


def cov_stage(K, R, t, Ms, ms, tau, pixel_var, covx=None):
    """pose_cov_dense.cov_stage with the points' covariances: H = sum w (L J)^T (L J), sigma2_hat = sum w |L e|^2 /
    dof; e and w stay on the pixel distance.  Returns its dict (J unwhitened)."""
    K, R, t = (np.asarray(a, np.float64) for a in (K, R, t))
    K, R = K.reshape(3, 3), R.reshape(3, 3)
    Ms = np.asarray(Ms, np.float64).reshape(-1, 3)
    ms = np.asarray(ms, np.float64).reshape(-1, 2)
    if covx is None:
        return cd.cov_stage(K, R, t, Ms, ms, tau, pixel_var)
    Lf = factors(covx)
    L = np.zeros((len(Ms), 2, 2))
    L[:, 0, 0], L[:, 0, 1], L[:, 1, 1] = Lf[:, 0], Lf[:, 1], Lf[:, 2]
    e = cd.residuals(K, R, t, Ms, ms)
    w = pd.weights(e, tau)
    J = cd.jacobian(K, R, t, Ms)
    LJ = np.einsum("nab,nbk->nak", L, J)
    u, v = pd.project(K, R, t, Ms)
    r0, r1 = whiten(Lf, u - ms[:, 0], v - ms[:, 1])
    live = w > 0
    H = np.einsum("n,nia,nib->ab", w[live], LJ[live], LJ[live])
    dof = 2 * int(np.count_nonzero(live)) - 6
    ew = np.sqrt(r0 * r0 + r1 * r1)
    sigma2_hat = pd.fsum(w[live] * (ew * ew)[live]) / dof if dof > 0 else math.nan
    try:
        C = np.linalg.cholesky(H)
        min_pivot = float(np.min(np.diag(C) ** 2 / np.diag(H)))
    except np.linalg.LinAlgError:
        min_pivot = 0.0
    valid = min_pivot >= cd.MIN_PIVOT
    cov = pixel_var * np.linalg.inv(H) if valid else np.full((6, 6), math.nan)
    return dict(J=J, H=H, cov=cov, e=e, w=w, dof=dof, sigma2_hat=sigma2_hat, min_pivot=min_pivot, valid=valid)
