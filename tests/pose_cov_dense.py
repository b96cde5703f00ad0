"""A float64 reference of the pose solver's covariance stage (cosl_pose_solver_set_covariance): per camera, at a
given (R, t), in the solver's chart R' = R exp([w]x), t' = t + dt, order (w, dt):

    e_i = |project(K, R, t, M_i) - m_i|,  w_i = tukey(e_i, tau),  H = sum_i w_i J_i^T J_i,
    cov = pixel_var H^-1,  dof = 2 #(w_i > 0) - 6,  sigma2_hat = sum w_i e_i^2 / dof (NaN for dof <= 0)

with the analytic 2x6 Jacobian J_i of the projection.  The sums run over the points with w_i > 0 only: a point
with a non-finite residual (depth 0 gives e_i = inf, 0 / 0 gives NaN) has weight 0 or NaN and is left out, where
0 * inf would make H NaN; its e_i is still reported as computed.  The camera is singular when the Cholesky
factorisation of H breaks down or its smallest relative pivot L_kk^2 / H_kk is below 1e-12; its covariance is
then NaN.  The inverse is numpy.linalg's, so it shares no arithmetic with the kernel's Cholesky."""
import math

import numpy as np

import pose_dense as pd

MIN_PIVOT = 1e-12


def jacobian(K, R, t, Ms):
    """[n, 2, 6]: d project(K, R exp([w]x), t + dt, M_i) / d(w, dt) at 0."""
    Ju, Jv = pd._jacobian_exact(np.asarray(K, np.float64), np.asarray(R, np.float64), np.asarray(t, np.float64),
                                np.asarray(Ms, np.float64).reshape(-1, 3))
    return np.stack([Ju, Jv], 1)


def residuals(K, R, t, Ms, ms):
    """e_i in pixels, in the operation order of the pose kernel's re-weighting."""
    u, v = pd.project(K, R, t, Ms)
    du, dv = u - ms[:, 0], v - ms[:, 1]
    return np.sqrt(du * du + dv * dv)


def cov_stage(K, R, t, Ms, ms, tau, pixel_var):
    """dict of J, H, cov, e, w, dof, sigma2_hat, min_pivot (0 on a break-down), valid."""
    K, R, t = (np.asarray(a, np.float64) for a in (K, R, t))
    K, R = K.reshape(3, 3), R.reshape(3, 3)
    Ms = np.asarray(Ms, np.float64).reshape(-1, 3)
    ms = np.asarray(ms, np.float64).reshape(-1, 2)
    e = residuals(K, R, t, Ms, ms)
    w = pd.weights(e, tau)
    J = jacobian(K, R, t, Ms)
    live = w > 0  # False for NaN
    H = np.einsum("n,nia,nib->ab", w[live], J[live], J[live])
    dof = 2 * int(np.count_nonzero(live)) - 6
    sigma2_hat = pd.fsum(w[live] * e[live] ** 2) / dof if dof > 0 else math.nan
    try:
        L = np.linalg.cholesky(H)
        min_pivot = float(np.min(np.diag(L) ** 2 / np.diag(H)))
    except np.linalg.LinAlgError:
        min_pivot = 0.0
    valid = min_pivot >= MIN_PIVOT
    cov = pixel_var * np.linalg.inv(H) if valid else np.full((6, 6), math.nan)
    return dict(J=J, H=H, cov=cov, e=e, w=w, dof=dof, sigma2_hat=sigma2_hat, min_pivot=min_pivot, valid=valid)


def residual_error(got, want):
    """max |got - want| over the finite e_i, or inf when a non-finite e_i differs in class (inf vs NaN vs
    finite): |inf - inf| would be NaN and fail any bound."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    fin = np.isfinite(want)
    if not (np.array_equal(np.isfinite(got), fin) and np.array_equal(np.isnan(got), np.isnan(want))
            and np.array_equal(got[np.isinf(want)], want[np.isinf(want)])):
        return math.inf
    return float(np.abs(got[fin] - want[fin]).max(initial=0.0))
