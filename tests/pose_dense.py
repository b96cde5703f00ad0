"""A vectorized float64 restatement of intraCamEstimate, written from the reference text
(slam/SL_IntraCamPose.cpp: :10-39 exp map, :43-117 forward differences, :259-303 step, :439-456 cost,
:475-549 LM procedure, :626-709 re-weighting).  It is the CPU yardstick of the pose kernel at frame-sized
point counts: the per-point arithmetic runs over all points at once in the reference's operation order,
every sum over points is exactly rounded (math.fsum) and the 6x6 system is solved by LAPACK, so it shares
no summation order and no inverse with the oracle or the kernel.

    estimate(...)    -> (ok, R, t, fields): the solve, fields = the option block it hands back
    one_step(...)    -> (A, b, delta): one forward-difference LM step
    exact_step(...)  -> (A, b, delta): the same step with the analytic Jacobian
    margins(...)     -> [(label, relative distance from the threshold)] of every decision

Where the reference leaves R_opt / t_opt unwritten (maxIterRW = 0, maxIterLM = 0, a first LM procedure
that accepts nothing) they start at R0 / t0, the project's choice (pose.cu, oracle/pose_oracle.cpp)."""
import math

import numpy as np

EPS = 1e-8
DEFAULT_OPT = (100, 5, 1e-7, 1e-6, 1e-6, 1e-3)


def exp_map(w):  # :10-39
    th = math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    if th == 0:
        return np.eye(3)
    a0, a1, a2 = w[0] / th, w[1] / th, w[2] / th
    s, c1 = math.sin(th), 1 - math.cos(th)
    a00, a01, a02, a11, a12, a22 = a0 * a0, a0 * a1, a0 * a2, a1 * a1, a1 * a2, a2 * a2
    return np.array([[-c1 * a11 - c1 * a22 + 1, c1 * a01 - s * a2, s * a1 + c1 * a02],
                     [s * a2 + c1 * a01, -c1 * a00 - c1 * a22 + 1, c1 * a12 - s * a0],
                     [c1 * a02 - s * a1, s * a0 + c1 * a12, -c1 * a00 - c1 * a11 + 1]])


def mat33(A, B):
    return np.array([[A[i, 0] * B[0, j] + A[i, 1] * B[1, j] + A[i, 2] * B[2, j] for j in range(3)]
                     for i in range(3)])


def project(K, R, t, Ms):
    """x = K (R M + t), m = x_{1,2} / x_3 for every row of Ms, each operation rounded once."""
    M0, M1, M2 = Ms[:, 0], Ms[:, 1], Ms[:, 2]
    c0 = R[0, 0] * M0 + R[0, 1] * M1 + R[0, 2] * M2 + t[0]
    c1 = R[1, 0] * M0 + R[1, 1] * M1 + R[1, 2] * M2 + t[1]
    c2 = R[2, 0] * M0 + R[2, 1] * M1 + R[2, 2] * M2 + t[2]
    u = K[0, 0] * c0 + K[0, 1] * c1 + K[0, 2] * c2
    v = K[1, 0] * c0 + K[1, 1] * c1 + K[1, 2] * c2
    w = K[2, 0] * c0 + K[2, 1] * c1 + K[2, 2] * c2
    return u / w, v / w


def weights(e, tau):
    """Tukey weights of the non-negative errors e: 0 at e >= tau, else (1 - (e/tau)^2)^2."""
    e = np.asarray(e, np.float64)
    q = e / tau
    q = 1 - q * q
    return np.where(e >= tau, 0.0, q * q)


def fsum(a):
    return math.fsum(np.asarray(a, np.float64).tolist())


def cost(K, R, t, W, Ms, ms):  # :439-456
    u, v = project(K, R, t, Ms)
    dx, dy = ms[:, 0] - u, ms[:, 1] - v
    return fsum((dx * dx + dy * dy) * W)


def _normal(Ju, Jv, W, r0, r1):
    """A = sum (W J)^T (W J), b = sum (W J)^T (W r), each entry an exactly rounded sum over points."""
    Ju, Jv = Ju * W[:, None], Jv * W[:, None]
    r0, r1 = r0 * W, r1 * W
    A = np.empty((6, 6))
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = fsum(Ju[:, a] * Ju[:, b] + Jv[:, a] * Jv[:, b])
    b = np.array([fsum(Ju[:, a] * r0 + Jv[:, a] * r1) for a in range(6)])
    return A, b


def _jacobian_fd(K, R, t, Ms, u0, v0):  # :43-117
    n = len(Ms)
    Ju, Jv = np.empty((n, 6)), np.empty((n, 6))
    for k in range(3):
        w = [0.0, 0.0, 0.0]
        w[k] = EPS
        u, v = project(K, mat33(R, exp_map(w)), t, Ms)
        Ju[:, k], Jv[:, k] = (u - u0) / EPS, (v - v0) / EPS
    for k in range(3):
        t1 = np.array(t, np.float64)
        t1[k] = t[k] + EPS
        u, v = project(K, R, t1, Ms)
        Ju[:, 3 + k], Jv[:, 3 + k] = (u - u0) / EPS, (v - v0) / EPS
    return Ju, Jv


def _jacobian_exact(K, R, t, Ms):
    """d m / d(w, t) of m(R exp(w), t + dt) at 0: dc/dw = -R [M]x, dc/dt = I, c = R M + t."""
    c = Ms @ R.T + t
    x = c @ K.T
    Mx = np.zeros((len(Ms), 3, 3))
    Mx[:, 0, 1], Mx[:, 0, 2], Mx[:, 1, 2] = -Ms[:, 2], Ms[:, 1], -Ms[:, 0]
    Mx[:, 1, 0], Mx[:, 2, 0], Mx[:, 2, 1] = Ms[:, 2], -Ms[:, 1], Ms[:, 0]
    dc = np.concatenate([-np.einsum("ij,njk->nik", R, Mx), np.broadcast_to(np.eye(3), (len(Ms), 3, 3))], 2)
    dx = np.einsum("ij,njk->nik", K, dc)
    Ju = (dx[:, 0] - x[:, 0:1] / x[:, 2:3] * dx[:, 2]) / x[:, 2:3]
    Jv = (dx[:, 1] - x[:, 1:2] / x[:, 2:3] * dx[:, 2]) / x[:, 2:3]
    return Ju, Jv


def _solve(A, b, lam):  # :293-302
    S = A + lam * np.eye(6)
    try:
        return S, np.linalg.solve(S, b)
    except np.linalg.LinAlgError:  # the oracle's and the kernel's inverse report failure with a zero step
        return S, np.zeros(6)


def prev_weights(n, tau, prev):  # :637-651
    return np.ones(n) if prev is None else weights(np.abs(prev), tau)


def one_step(K, R, t, Ms, ms, W, lam):
    """One forward-difference LM step at (R, t) with weights W: (A + lam I, b, delta)."""
    u0, v0 = project(K, R, t, Ms)
    Ju, Jv = _jacobian_fd(K, R, t, Ms, u0, v0)
    A, b = _normal(Ju, Jv, W, ms[:, 0] - u0, ms[:, 1] - v0)
    S, d = _solve(A, b, lam)
    return S, b, d


def exact_step(K, R, t, Ms, ms, W, lam):
    """one_step with the exact Jacobian of the right-multiplied rotation update."""
    u0, v0 = project(K, R, t, Ms)
    Ju, Jv = _jacobian_exact(K, R, t, Ms)
    A, b = _normal(Ju, Jv, W, ms[:, 0] - u0, ms[:, 1] - v0)
    S, d = _solve(A, b, lam)
    return S, b, d


def _rel(x, thr):
    """Relative distance of x from the threshold of `x < thr`; a zero threshold cannot be crossed."""
    return abs(x - thr) / thr if thr > 0 else math.inf


def estimate(K, R0, t0, Ms, ms, tau, prev=None, opt=DEFAULT_OPT, trace=None):
    """intraCamEstimate.  Returns ok, R, t and the option block (lambda, lambda0, err0, err, errRW,
    retTypeLM, npts, nIterLM, nIterRW).  trace, a list, receives (label, margin) of every decision."""
    maxIterLM, maxIterRW, epsErr, epsParam, epsRW, lambda0 = opt
    Ms = np.asarray(Ms, np.float64).reshape(-1, 3)
    ms = np.asarray(ms, np.float64).reshape(-1, 2)
    n = len(Ms)
    W = prev_weights(n, tau, prev)
    R, t = np.array(R0, np.float64), np.array(t0, np.float64)
    R_opt, t_opt = R.copy(), t.copy()
    f = dict(lambda_=lambda0, lambda0=lambda0, err0=0.0, err=0.0, errRW=-1.0, retTypeLM=1, npts=n,
             nIterLM=0, nIterRW=0)
    note = trace.append if trace is not None else (lambda m: None)
    ok = True
    k = 0
    while k < maxIterRW:
        # ---- intraCamWeightedLMProc (:475-549) from (R, t)
        lam = f["lambda0"]
        err0 = cost(K, R, t, W, Ms, ms)
        errLM = err = err0
        Rl, tl, R_tmp, t_tmp = R, t, R, t
        ret, i = 1, 0
        while i < maxIterLM:
            _, _, p = one_step(K, Rl, tl, Ms, ms, W, lam)
            R_opt, t_opt = mat33(Rl, exp_map(p[:3])), tl + p[3:]
            p2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] + p[4] * p[4] + p[5] * p[5]
            note((f"rw{k} lm{i} p2", _rel(p2, epsParam)))
            if p2 < epsParam:
                Rl, tl, ret = R_opt, t_opt, 0
                break
            err = cost(K, R_opt, t_opt, W, Ms, ms)
            note((f"rw{k} lm{i} |derr|", _rel(abs(err - errLM), epsErr)))
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
        # ---- re-weighting (:664-702)
        f["lambda0"] = lam
        if f["errRW"] < 0:
            f["errRW"] = err
        else:
            note((f"rw{k} |derrRW|", _rel(abs(err - f["errRW"]), epsRW)))
            if abs(err - f["errRW"]) < epsRW:
                break
            f["errRW"] = err
        R, t = R_opt, t_opt
        u, v = project(K, R, t, Ms)
        du, dv = u - ms[:, 0], v - ms[:, 1]
        e = np.sqrt(du * du + dv * dv)
        if n:
            note((f"rw{k} tukey", float(np.min(np.abs(e - tau))) / tau))
        W = weights(e, tau)
        k += 1
    f["nIterRW"] = k
    return ok, R_opt, t_opt, f


def margins(K, R0, t0, Ms, ms, tau, prev=None, opt=DEFAULT_OPT):
    """(label, relative distance from its threshold) of every decision on estimate's trajectory: p2 vs
    epsParamChangeLM, |err - errLM| vs epsErrorChangeLM, the accept test err <= errLM, |errLM - errRW|
    vs epsErrorChangeRW and each point's residual vs tau at every re-weighting."""
    trace = []
    estimate(K, R0, t0, Ms, ms, tau, prev, opt, trace)
    return trace
