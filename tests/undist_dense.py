"""numpy float64 restatement of the KLT undistortion stage (DESIGN.md section 3.5, klt_undist.cuh):
Bouguet's / OpenCV's forward model with skew, its Newton inverse with the stage's schedule and stopping rule,
the NaN rules, and the covariance map A = K2 J(x*)^-1 K2^-1.  Everything is vectorised over points."""
import numpy as np

MAX_STEPS, TOL_PX = 20, 1e-9


def intrinsics(K):
    """(fx, s, cx, fy, cy) of a row-major 3x3 camera matrix"""
    K = np.asarray(K, np.float64).reshape(3, 3)
    return K[0, 0], K[0, 1], K[0, 2], K[1, 1], K[1, 2]


def distort(x, y, kc):
    """d(x) and J = dd/dx at normalised points (x, y): (dx, dy, j00, j01, j10, j11)"""
    k1, k2, p1, p2, k3 = (float(v) for v in kc)
    r2 = x * x + y * y
    a = 1.0 + r2 * (k1 + r2 * (k2 + r2 * k3))
    b = k1 + r2 * (2.0 * k2 + 3.0 * r2 * k3)
    dx = a * x + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x)
    dy = a * y + p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y
    c = 2.0 * x * y * b + 2.0 * p1 * x + 2.0 * p2 * y
    j00 = a + 2.0 * x * x * b + 2.0 * p1 * y + 6.0 * p2 * x
    j11 = a + 2.0 * y * y * b + 6.0 * p1 * y + 2.0 * p2 * x
    return dx, dy, j00, c, c, j11


def project(K, kc, x, y):
    """pixels of normalised undistorted points: K2 d(x) + (cx, cy)"""
    fx, s, cx, fy, cy = intrinsics(K)
    dx, dy = distort(np.asarray(x, np.float64), np.asarray(y, np.float64), kc)[:2]
    return fx * dx + s * dy + cx, fy * dy + cy


def normalise(K, u, v):
    """K2^-1 (u - cx, v - cy)"""
    fx, s, cx, fy, cy = intrinsics(K)
    y = (np.asarray(v, np.float64) - cy) / fy
    return (np.asarray(u, np.float64) - cx - s * y) / fx, y


def undistort(K, kc, ud, vd):
    """The stage's inverse at distorted pixels (ud, vd): (u, v, J at x*, ok).  Newton from x_d, at most 20
    steps, stopping once |K2 (d(x) - x_d)|_inf <= 1e-9 px; a point fails when that is not met, when det J <= 0
    at an iterate or at the answer, or on a non-finite value (u, v NaN there)."""
    fx, s, cx, fy, cy = intrinsics(K)
    xd, yd = normalise(K, ud, vd)
    xd, yd = np.atleast_1d(xd).astype(np.float64), np.atleast_1d(yd).astype(np.float64)
    x, y = xd.copy(), yd.copy()
    J = np.zeros(xd.shape + (2, 2))
    active = np.isfinite(xd) & np.isfinite(yd)
    ok = np.zeros(xd.shape, bool)
    with np.errstate(all="ignore"):
        for it in range(MAX_STEPS + 1):
            if not active.any():
                break
            dx, dy, j00, j01, j10, j11 = distort(x, y, kc)
            det = j00 * j11 - j01 * j10
            r0, r1 = dx - xd, dy - yd
            J[active] = np.stack([np.stack([j00, j01], -1), np.stack([j10, j11], -1)], -2)[active]
            bad = active & ~((det > 0) & np.isfinite(det) & np.isfinite(r0) & np.isfinite(r1))
            active &= ~bad
            done = active & (np.maximum(np.abs(fx * r0 + s * r1), np.abs(fy * r1)) <= TOL_PX)
            ok |= done
            active &= ~done
            if it == MAX_STEPS:
                break
            step = active
            x = np.where(step, x - (j11 * r0 - j01 * r1) / det, x)
            y = np.where(step, y - (j00 * r1 - j10 * r0) / det, y)
        u, v = fx * x + s * y + cx, fy * y + cy
        ok &= np.isfinite(u) & np.isfinite(v)
    return np.where(ok, u, np.nan), np.where(ok, v, np.nan), J, ok


def cov_map(K, J):
    """A = K2 J^-1 K2^-1 for every J (n, 2, 2)"""
    fx, s, _, fy, _ = intrinsics(K)
    K2 = np.array([[fx, s], [0.0, fy]])
    with np.errstate(all="ignore"):
        return K2 @ np.linalg.inv(J) @ np.linalg.inv(K2)


def stage(K, kc, W, H, feats, cov=None):
    """The stage on one camera's handed-out table (FEAT_DTYPE, n slots) and its position covariances (n, 3)
    float32 or None: (pos (n, 2) float64, ucov (n, 3) float64 or None), NaN as the device gives it."""
    pos32 = feats["pos"].astype(np.float32)
    ud = pos32[:, 0].astype(np.float64) * W
    vd = pos32[:, 1].astype(np.float64) * H
    u, v, J, ok = undistort(K, kc, ud, vd)
    ok &= feats["status"] >= 0
    pos = np.where(ok[:, None], np.stack([u, v], 1), np.nan)
    if cov is None:
        return pos, None
    c = np.asarray(cov, np.float64)
    S = np.stack([np.stack([c[:, 0], c[:, 1]], -1), np.stack([c[:, 1], c[:, 2]], -1)], -2)
    J = np.where(ok[:, None, None], J, np.eye(2))
    A = cov_map(K, J)
    with np.errstate(all="ignore"):
        Su = A @ S @ A.transpose(0, 2, 1)
    out = np.stack([Su[:, 0, 0], Su[:, 0, 1], Su[:, 1, 1]], 1)
    good = ok & np.isfinite(out).all(1)
    return pos, np.where(good[:, None], out, np.nan)


def camera(fx, fy, cx, cy, s=0.0):
    return np.array([[fx, s, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


# The calibrations the tests use: (K, kc, W, H)
CALIBS = {
    "mild_barrel": (camera(900.0, 905.0, 640.3, 358.7), np.array([-0.08, 0.02, 0.0, 0.0, 0.0]), 1280, 720),
    "strong_barrel_k3": (camera(760.0, 760.0, 641.0, 361.0), np.array([-0.30, 0.10, 0.0, 0.0, -0.01]), 1280, 720),
    "pincushion_tangential": (camera(520.0, 515.0, 322.0, 243.5), np.array([0.12, -0.05, 0.0015, -0.001, 0.01]),
                              640, 480),
    "skew": (camera(610.0, 600.0, 318.0, 245.0, s=2.5), np.array([-0.15, 0.05, 0.0008, 0.0006, 0.0]), 640, 480),
}
