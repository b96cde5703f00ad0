"""Float64 numpy restatement of the reference's KLT front end and trackers, written from the shaders
and the host loops of V3D_GPU::KLT_SequenceTracker, not from the oracle:

  level0, reduce1331      pyramid_with_derivative_pass1v/1h.cg, pass2.cg ([1 3 3 1] / 8, size >> 1)
  cornerness              klt_detector_pass1/2.cg (Shi-Tomasi, 7x7 box, margin mask)
  nonmax_survivors        klt_detector_nonmax.cg
  tracker_levels          the level loops of klt_tracker.cg and v3d_gpuklt.cpp:254 with the
                          KLT_TrackerBase rule levelSkip <= 0 -> nLevels - 1 (v3d_gpuklt.h:14)
  track_2x2               klt_tracker.cg (window half-width, iterations per level, 5 with ITER5)
  gain_neighbours         klt_tracker_with_gain.cg:64-75: NEAREST, CLAMP_TO_EDGE lookups of the slot
                          texture at st0 +- ds0.x (the scalar added to both coordinates), st0 +- ds0.y
                          and the four axis neighbours, computed exactly with fractions
  track_gain              klt_tracker_with_gain.cg:42-148 and the pass loop v3d_gpuklt.cpp:243-287
                          (lax thresholds on iteration 1, strict on the last iteration of a level,
                          so never armed when nIterations == 1)

CLAMP_TO_EDGE is np.pad(mode="edge") / index clamping; GL_LINEAR is the exact two-stage lerp.  The
trackers run over all slots at once (one row per slot)."""
import math
from fractions import Fraction

import numpy as np


def _tap_v(a, taps, lo):
    """out[y] = sum_k taps[k] * a[clamp(y + lo + k)] along axis 0."""
    n = len(taps)
    hi = lo + n - 1
    p = np.pad(a, ((max(0, -lo), max(0, hi)), (0, 0)), mode="edge")
    off = max(0, -lo)
    H = a.shape[0]
    return sum(t * p[off + lo + k: off + lo + k + H] for k, t in enumerate(taps))


def _tap_h(a, taps, lo):
    return _tap_v(a.T, taps, lo).T


def level0(img):
    g = img.astype(np.float64)
    v = _tap_v(g, [0.25, 0.5, 0.25], -1)                    # pass1v.cg:63-83
    dv = _tap_v(g, [-0.125, -0.25, 0.0, 0.25, 0.125], -2)
    I = _tap_h(v, [0.25, 0.5, 0.25], -1)                    # pass1h.cg:96-128
    Ix = _tap_h(v, [-0.125, -0.25, 0.0, 0.25, 0.125], -2)
    Iy = _tap_h(dv, [0.25, 0.5, 0.25], -1)
    return np.stack([I, Ix, Iy], -1)


def reduce1331(P):
    """pass2.cg: rows 2j-1..2j+2 then columns 2i-1..2i+2, weights [1 3 3 1] / 8, size >> 1."""
    H, W, _ = P.shape
    h, w = H >> 1, W >> 1
    out = np.empty((h, w, 3))
    for c in range(3):
        a = P[..., c]
        t = _tap_v(a, [0.125, 0.375, 0.375, 0.125], -1)[0:2 * h:2]      # row 2j: taps 2j-1..2j+2
        out[..., c] = _tap_h(t, [0.125, 0.375, 0.375, 0.125], -1)[:, 0:2 * w:2]
    return out


def cornerness(P0, min_c, margin, W, H):
    gx, gy = P0[..., 1], P0[..., 2]
    box = lambda a: _tap_h(_tap_v(a, [1.0] * 7, -3), [1.0] * 7, -3)     # detector_pass1/2.cg
    a, b, c = box(gx * gx), box(gx * gy), box(gy * gy)
    cs = np.maximum(0.5 * (a + c - np.sqrt((a - c) ** 2 + 4 * b * b)) - min_c, 0.0)
    sx = (np.arange(W) + 0.5) / W
    sy = (np.arange(H) + 0.5) / H
    inside = ((sx >= margin / W) & (sx <= 1 - margin / W))[None, :] & \
             ((sy >= margin / H) & (sy <= 1 - margin / H))[:, None]
    return np.where(inside, cs, 0.0)


def nonmax_survivors(c, r):
    """klt_detector_nonmax.cg: strictly greatest |.| in the clamped (2r+1)^2 window, ties kill."""
    H, W = c.shape
    a = np.abs(c)
    p = np.pad(a, r, mode="edge")
    best = np.zeros_like(a)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            if dx == 0 and dy == 0:
                continue
            best = np.maximum(best, p[r + dy: r + dy + H, r + dx: r + dx + W])
    return (c > 0) & (a > best)


# --------------------------------------------------------------------------------------------
# Trackers
# --------------------------------------------------------------------------------------------
def tracker_levels(n_levels, level_skip):
    """Levels the trackers visit: nLevels-1, nLevels-1-levelSkip, ... >= 0; levelSkip <= 0 means
    nLevels - 1 (coarsest level and base level).  A single level (nLevels = 1) is level 0."""
    skip = level_skip if level_skip > 0 else n_levels - 1
    skip = max(skip, 1)
    return list(range(n_levels - 1, -1, -skip))


def iterations_2x2(n_iterations, iter5):
    """klt_tracker.cg runs N_ITERATIONS, which the host never defines (it passes -DNITERATIONS):
    always 5, unless the ITER5 compat bit is cleared."""
    return 5 if iter5 else n_iterations


def _sample(P, s, t):
    """Bilinear sample of level array P[h][w][3] at normalised (s, t), clamp-to-edge (A.3)."""
    h, w, _ = P.shape
    u = np.clip(s * w - 0.5, -2.0, w + 1.0)
    v = np.clip(t * h - 0.5, -2.0, h + 1.0)
    x0 = np.floor(u).astype(int)
    y0 = np.floor(v).astype(int)
    ax, ay = (u - x0)[..., None], (v - y0)[..., None]
    cx0, cx1 = np.clip(x0, 0, w - 1), np.clip(x0 + 1, 0, w - 1)
    cy0, cy1 = np.clip(y0, 0, h - 1), np.clip(y0 + 1, 0, h - 1)
    top = P[cy0, cx0] + ax * (P[cy0, cx1] - P[cy0, cx0])
    bot = P[cy1, cx0] + ax * (P[cy1, cx1] - P[cy1, cx0])
    return top + ay * (bot - top)


def _window(hw):
    """Window offsets (dx, dy), row-major, as (1, (2hw+1)^2) rows that broadcast against slots."""
    d = np.arange(-hw, hw + 1, dtype=np.float64)
    dx, dy = np.meshgrid(d, d)
    return dx.reshape(1, -1), dy.reshape(1, -1)


def track_2x2(P0, P1, X0, W, H, levels, n_iter, hw, conv, ssd_thr, margin):
    """klt_tracker.cg.  P0/P1: dict level -> array; X0: (F, 2) normalised, x < 0 = dead.  The window
    step at level l is 2^l / W (ds * multiplier); the convergence and SSD tests follow each level,
    the valid region the last one.  Returns (F, 3): (x1, y1, x0), -1 where invalid."""
    dx, dy = _window(hw)
    X0 = np.asarray(X0, np.float64)
    x0, y0 = X0[:, :1], X0[:, 1:2]
    x1, y1 = x0.copy(), y0.copy()
    invalid = X0[:, 0] < 0
    for lv in levels:
        sx, sy = (2.0 ** lv) / W, (2.0 ** lv) / H
        a0 = _sample(P0[lv], x0 + dx * sx, y0 + dy * sy)
        len2 = ssd = np.zeros(len(X0))
        for _ in range(n_iter):
            a1 = _sample(P1[lv], x1 + dx * sx, y1 + dy * sy)
            e = a0[..., 0] - a1[..., 0]
            jx = (a0[..., 1] + a1[..., 1]) * W / 2
            jy = (a0[..., 2] + a1[..., 2]) * H / 2
            a, b, c = (jx * jx).sum(1), (jx * jy).sum(1), (jy * jy).sum(1)
            r0, r1, ssd = (e * jx).sum(1), (e * jy).sum(1), (e * e).sum(1)
            det = a * c - b * b
            invalid |= det < 1e-5
            dd = np.where(invalid, 1.0, det)          # an invalid slot's iterate is never read
            ux = np.where(invalid, 0.0, (c * r0 - b * r1) / dd)
            uy = np.where(invalid, 0.0, (-b * r0 + a * r1) / dd)
            x1, y1 = x1 + ux[:, None], y1 + uy[:, None]
            len2 = (ux * W) ** 2 + (uy * H) ** 2
        invalid |= (len2 > conv * conv) | (ssd > ssd_thr)
    x1, y1 = x1[:, 0], y1[:, 0]
    invalid |= (x1 < margin / W) | (y1 < margin / H) | (x1 > 1 - margin / W) | (y1 > 1 - margin / H)
    out = np.column_stack([x1, y1, X0[:, 0]])
    out[invalid] = -1.0
    return out


def _nearest(s, n, lower_on_tie=False):
    """NEAREST + CLAMP_TO_EDGE texel of the exact normalised coordinate s in n texels: floor(s n),
    clamped.  A coordinate exactly on a texel boundary takes the texel that starts there (GL's
    floor(u) rule); lower_on_tie takes the one that ends there instead."""
    u = s * n
    i = math.ceil(u) - 1 if lower_on_tie else math.floor(u)
    return min(max(i, 0), n - 1)


def _gain_lookups(fw, fh):
    """The eight lookup offsets of klt_tracker_with_gain.cg:64-71 for ds0 = (1/fw, 1/fh): betaN1 adds
    the scalar ds0.x (resp. ds0.y) to both coordinates, betaN2 steps along one axis."""
    dx, dy = Fraction(1, fw), Fraction(1, fh)
    z = Fraction(0)
    return [(dx, dx), (-dx, -dx), (dy, dy), (-dy, -dy), (dx, z), (-dx, z), (z, dy), (z, -dy)]


def gain_neighbours(fw, fh, lower_on_tie=False):
    """(fw * fh, 8) slot index of each lookup of each slot, exact."""
    offs = _gain_lookups(fw, fh)
    nbr = np.empty((fw * fh, 8), np.int64)
    for sy in range(fh):
        t = Fraction(2 * sy + 1, 2 * fh)
        for sx in range(fw):
            s = Fraction(2 * sx + 1, 2 * fw)
            for k, (ox, oy) in enumerate(offs):
                nbr[sy * fw + sx, k] = (_nearest(t + oy, fh, lower_on_tie) * fw +
                                        _nearest(s + ox, fw, lower_on_tie))
    return nbr


def gain_lookup_ties(fw, fh):
    """Lookups that land exactly on a boundary between two slots (inside the grid): (slot, k)."""
    ties = []
    for sy in range(fh):
        t = Fraction(2 * sy + 1, 2 * fh)
        for sx in range(fw):
            s = Fraction(2 * sx + 1, 2 * fw)
            for k, (ox, oy) in enumerate(_gain_lookups(fw, fh)):
                u, v = (s + ox) * fw, (t + oy) * fh
                if (u.denominator == 1 and 0 < u < fw) or (v.denominator == 1 and 0 < v < fh):
                    ties.append((sy * fw + sx, k))
    return ties


def track_gain(P0, P1, X0, W, H, fw, fh, levels, n_iter, hw, conv, ssd_thr, margin, lam=1.0, delta=200.0,
               nbr=None):
    """klt_tracker_with_gain.cg: one pass over all slots per (level, iteration); the neighbours'
    gains come from the previous pass.  nbr: the neighbour table (default gain_neighbours).
    Returns (F, 3): (x1, y1, gain), -1 where invalid."""
    dx, dy = _window(hw)
    npx = dx.shape[1]
    F = fw * fh
    X0 = np.asarray(X0, np.float64)
    nbr = gain_neighbours(fw, fh) if nbr is None else nbr
    cur = np.column_stack([X0[:, 0], X0[:, 1], np.ones(F)])      # X1 <- X0, beta <- 1
    for lv in levels:
        w, h = W >> lv, H >> lv
        a0 = _sample(P0[lv], X0[:, :1] + dx / w, X0[:, 1:2] + dy / h)
        I0, g0 = a0[..., 0], np.hypot(a0[..., 1], a0[..., 2])
        for it in range(1, n_iter + 1):
            strict = (it == n_iter) and (it != 1)
            conv2, ssd_t = (conv * conv, ssd_thr) if strict else (1e6, 1e6)
            vr = (margin / W, margin / H, 1 - margin / W, 1 - margin / H) if strict else (-1, -1, 2, 2)
            x1, y1, beta = cur[:, :1], cur[:, 1:2], cur[:, 2:3]
            g = cur[nbr, 2]
            nb = np.where(g < 0, beta, g).sum(1)
            a1 = _sample(P1[lv], x1 + dx / w, y1 + dy / h)
            e = beta * I0 - a1[..., 0]
            jx = (beta * a0[..., 1] + a1[..., 1]) * W / 2
            jy = (beta * a0[..., 2] + a1[..., 2]) * H / 2
            g1 = np.hypot(a1[..., 1], a1[..., 2])
            J = np.stack([jx, jy, -I0], 1)                          # (F, 3, npx)
            M = J @ J.transpose(0, 2, 1)
            M[:, 2, 2] = (I0 * I0 + lam * g0 * g0).sum(1) + 8 * delta * npx
            r = (J @ e[..., None])[..., 0]
            r[:, 2] = (-e * I0 + lam * g0 * (g1 - beta * g0)).sum(1) + npx * delta * (nb - 8 * beta[:, 0])
            dead = (cur[:, 0] < 0) | (X0[:, 0] < 0)
            det = np.linalg.det(M)
            ok = ~dead & (det != 0)
            u = np.zeros((F, 3))
            if ok.any():
                u[ok] = np.linalg.solve(M[ok], r[ok][..., None])[..., 0]
            nx, ny, nbeta = x1[:, 0] + u[:, 0], y1[:, 0] + u[:, 1], beta[:, 0] + u[:, 2]
            bad = ~ok | (det < 1e-5) | ((e * e).sum(1) > ssd_t) | ((u[:, 0] * W) ** 2 + (u[:, 1] * H) ** 2 > conv2)
            bad |= (nx < vr[0]) | (ny < vr[1]) | (nx > vr[2]) | (ny > vr[3])
            cur = np.column_stack([nx, ny, nbeta])
            cur[bad] = -1.0
    return cur
