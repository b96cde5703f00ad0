"""A numpy float64 restatement of the pose solver's PnP RANSAC (cosl_pose_solver_set_ransac, DESIGN.md 5.7): the
counter-based sampler, the 5-point EPnP with its cyclic Jacobi eigensolvers and Householder least squares, the scoring
and the deterministic selection.  Every stage is vectorised over the hypotheses of one camera and performs the
kernel's operations in the kernel's order."""
import numpy as np

MASK64 = (1 << 64) - 1
NDRAW = 256  # draws per hypothesis before a sample is degenerate
JACOBI_TOL = 1e-30  # a sweep starts only while sum_{p<q} a_pq^2 > JACOBI_TOL * sum_p a_pp^2
SWEEPS3, SWEEPS12 = 12, 16
PCA_MIN = 1e-12  # smallest / largest PCA eigenvalue of a usable sample
GN_ITERS = 5

# Monte-Carlo bounds (DESIGN.md 5.7), fixed by `python tests/test_pnp_dense_ref.py`: a start pose is a success within
# MC_ANGLE_DEG and MC_CENTRE_REL of the mean depth.  The full campaign (1 002 cameras per outlier share, 200 points,
# 0.5 px, 30 % and 50 % outliers, R0 20-40 degrees off, three depth ranges, MC_HYP hypotheses, MC_THR px) found such a
# start for at least 99.4 % of the cameras in every setting; MC_MIN_SUCCESS leaves room for the smaller runs.  The
# Tukey solve that follows without prevErrs often leaves a good start under gross outliers (the solve's behaviour,
# which RANSAC does not change); a second solve with prevErrs from the start's inlier flags (prev_errs) keeps it.
MC_ANGLE_DEG = 2.0
MC_CENTRE_REL = 0.05
MC_MIN_SUCCESS = 0.97
MC_HYP, MC_THR = 256, 2.0
DEPTHS = [(2.0, 6.0), (4.0, 20.0), (15.0, 60.0)]

# status of download_ransac
REPLACED, TOO_FEW, FEW_INLIERS, NOT_SELECTED, KEPT = 0, 1, 2, 3, 4


def splitmix64(x):
    """The SplitMix64 output for state x (uint64 array or int): z = x + 0x9e3779b97f4a7c15, then the finaliser."""
    with np.errstate(over="ignore"):  # arithmetic modulo 2^64
        z = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def samples(seed, c, n, n_hyp):
    """[n_hyp, 5] indices of camera c's hypotheses, -1 rows for a hypothesis without 5 distinct indices in NDRAW
    draws: u_j = splitmix64(seed ^ ((c << 40) | (h << 8) | j)), idx = u_j mod n, duplicates skipped."""
    h = np.arange(n_hyp, dtype=np.uint64)[:, None]
    j = np.arange(NDRAW, dtype=np.uint64)[None, :]
    key = np.uint64((int(c) << 40) & MASK64) | (h << np.uint64(8)) | j
    idx = (splitmix64(np.uint64(int(seed) & MASK64) ^ key) % np.uint64(n)).astype(np.int64)
    out = np.full((n_hyp, 5), -1, np.int64)
    cnt = np.zeros(n_hyp, np.int64)
    rows = np.arange(n_hyp)
    for k in range(NDRAW):
        v = idx[:, k]
        dup = ((out == v[:, None]) & (np.arange(5)[None, :] < cnt[:, None])).any(1)
        take = ~dup & (cnt < 5)
        out[rows[take], cnt[take]] = v[take]
        cnt += take
        if (cnt == 5).all():
            break
    out[cnt < 5] = -1
    return out


def jacobi(A, sweeps):
    """Cyclic Jacobi on a batch [B, n, n] of symmetric matrices: sweeps over (p, q), p < q, row by row, each a
    rotation with theta = (a_qq - a_pp) / (2 a_pq), t = sign(theta) / (|theta| + sqrt(theta^2 + 1)), c = 1 / sqrt(t^2
    + 1), s = t c, applied to the columns p, q, then the rows p, q, then a_pq = a_qp = 0, and to the columns of V; a_pq
    = 0 skips.  Before each sweep a matrix stops when sum_{p<q} a_pq^2 <= JACOBI_TOL sum_p a_pp^2.  Returns (diag,
    V): A = V diag(d) V^T."""
    A = np.array(A, np.float64)
    B, n = A.shape[0], A.shape[1]
    V = np.broadcast_to(np.eye(n), (B, n, n)).copy()
    active = np.ones(B, bool)
    for _ in range(sweeps):
        off = np.zeros(B)
        dia = np.zeros(B)
        for p in range(n):
            dia = dia + A[:, p, p] * A[:, p, p]
            for q in range(p + 1, n):
                off = off + A[:, p, q] * A[:, p, q]
        active &= ~(off <= JACOBI_TOL * dia)
        if not active.any():
            break
        for p in range(n - 1):
            for q in range(p + 1, n):
                apq = A[:, p, q]
                rot = active & (apq != 0)
                if not rot.any():
                    continue
                with np.errstate(all="ignore"):
                    theta = (A[:, q, q] - A[:, p, p]) / (2.0 * apq)
                    t = 1.0 / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
                    t = np.where(theta < 0, -t, t)
                    c = 1.0 / np.sqrt(t * t + 1.0)
                    s = t * c
                r = rot[:, None]
                c, s = c[:, None], s[:, None]
                for X in (A, V):
                    xp, xq = X[:, :, p].copy(), X[:, :, q].copy()
                    X[:, :, p] = np.where(r, c * xp - s * xq, xp)
                    X[:, :, q] = np.where(r, s * xp + c * xq, xq)
                    if X is A:
                        xp, xq = A[:, p, :].copy(), A[:, q, :].copy()
                        A[:, p, :] = np.where(r, c * xp - s * xq, xp)
                        A[:, q, :] = np.where(r, s * xp + c * xq, xq)
                        A[:, p, q] = np.where(rot, 0.0, A[:, p, q])
                        A[:, q, p] = np.where(rot, 0.0, A[:, q, p])
    return np.einsum("bii->bi", A).copy(), V


def lstsq_hh(A, b):
    """Least squares min |A x - b| for a batch A [B, 6, n], b [B, 6] by Householder QR in the kernel's order."""
    A, b = np.array(A, np.float64), np.array(b, np.float64)
    m, n = A.shape[1], A.shape[2]
    with np.errstate(all="ignore"):
        for k in range(n):
            nrm2 = np.zeros(A.shape[0])
            for i in range(k, m):
                nrm2 = nrm2 + A[:, i, k] * A[:, i, k]
            alpha = np.where(A[:, k, k] > 0, -np.sqrt(nrm2), np.sqrt(nrm2))
            v = A[:, k:, k].copy()
            v[:, 0] = v[:, 0] - alpha
            vv = np.zeros(A.shape[0])
            for i in range(m - k):
                vv = vv + v[:, i] * v[:, i]
            for j in range(k, n):
                f = np.zeros(A.shape[0])
                for i in range(m - k):
                    f = f + v[:, i] * A[:, k + i, j]
                f = 2.0 * f / vv
                for i in range(m - k):
                    A[:, k + i, j] = A[:, k + i, j] - f * v[:, i]
            f = np.zeros(A.shape[0])
            for i in range(m - k):
                f = f + v[:, i] * b[:, k + i]
            f = 2.0 * f / vv
            for i in range(m - k):
                b[:, k + i] = b[:, k + i] - f * v[:, i]
        x = np.zeros((A.shape[0], n))
        for k in range(n - 1, -1, -1):
            a = b[:, k].copy()
            for j in range(k + 1, n):
                a = a - A[:, k, j] * x[:, j]
            x[:, k] = a / A[:, k, k]
    return x


def project(K, R, t, M):
    """(u, v, depth) of world points M [B, N, 3] at poses R [B, 3, 3], t [B, 3]: the solver's projection."""
    c = [R[:, i, 0, None] * M[..., 0] + R[:, i, 1, None] * M[..., 1] + R[:, i, 2, None] * M[..., 2] + t[:, i, None]
         for i in range(3)]
    u = K[0, 0] * c[0] + K[0, 1] * c[1] + K[0, 2] * c[2]
    v = K[1, 0] * c[0] + K[1, 1] * c[1] + K[1, 2] * c[2]
    w = K[2, 0] * c[0] + K[2, 1] * c[1] + K[2, 2] * c[2]
    with np.errstate(all="ignore"):
        return u / w, v / w, c[2]


def _mean(P):
    """(p_0 + p_1 + ... ) / n over axis 1, summed in order"""
    s = P[:, 0].copy()
    for i in range(1, P.shape[1]):
        s = s + P[:, i]
    return s / P.shape[1]


def _pairs():
    return [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def epnp(K, Mw, mp):
    """EPnP on a batch of 5-point samples: Mw [B, 5, 3] world points, mp [B, 5, 2] pixels.  Returns (R [B, 3, 3],
    t [B, 3], ok [B]); ok False is a degenerate sample (PCA ratio below PCA_MIN or a non-finite value)."""
    B, n = Mw.shape[0], Mw.shape[1]
    K = np.asarray(K, np.float64)
    with np.errstate(all="ignore"):
        # control points: centroid and PCA
        c0 = _mean(Mw)
        D = Mw - c0[:, None, :]
        Cv = np.zeros((B, 3, 3))
        for i in range(n):
            Cv += D[:, i, :, None] * D[:, i, None, :]
        lam, E = jacobi(Cv, SWEEPS3)
        order = np.argsort(-lam, axis=1, kind="stable")
        lam = np.take_along_axis(lam, order, 1)
        E = np.take_along_axis(E, order[:, None, :], 2)
        ok = np.isfinite(lam).all(1) & (lam[:, 2] >= PCA_MIN * lam[:, 0]) & (lam[:, 0] > 0)
        sc = np.sqrt(lam / n)  # [B, 3]
        cw = np.zeros((B, 4, 3))
        cw[:, 0] = c0
        for j in range(3):
            cw[:, j + 1] = c0 + sc[:, j, None] * E[:, :, j]
        # barycentric coordinates: alpha_j = (D . e_j) / sc_j
        al = np.zeros((B, n, 4))
        for j in range(3):
            al[:, :, j + 1] = (D[..., 0] * E[:, None, 0, j] + D[..., 1] * E[:, None, 1, j] +
                               D[..., 2] * E[:, None, 2, j]) / sc[:, None, j]
        al[:, :, 0] = 1.0 - al[:, :, 1] - al[:, :, 2] - al[:, :, 3]
        # M (2n x 12) and MtM, rows accumulated in order
        MtM = np.zeros((B, 12, 12))
        for i in range(n):
            for r in range(2):
                x = mp[:, i, r]
                row = np.zeros((B, 12))
                for j in range(4):
                    for k in range(3):
                        row[:, 3 * j + k] = al[:, i, j] * (K[r, k] - x * K[2, k])
                MtM += row[:, :, None] * row[:, None, :]
        d, V = jacobi(MtM, SWEEPS12)
        ok &= np.isfinite(d).all(1)
        order = np.argsort(d, axis=1, kind="stable")[:, :4]
        v = np.stack([np.take_along_axis(V, order[:, None, k:k + 1], 2)[:, :, 0] for k in range(4)], 1)  # [B, 4, 12]
        # L_6x10 and rho
        L = np.zeros((B, 6, 10))
        rho = np.zeros((B, 6))
        for r, (a, b) in enumerate(_pairs()):
            dv = [v[:, i, 3 * a:3 * a + 3] - v[:, i, 3 * b:3 * b + 3] for i in range(4)]

            def dot(x, y):
                return x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1] + x[:, 2] * y[:, 2]
            L[:, r, 0] = dot(dv[0], dv[0])
            L[:, r, 1] = 2.0 * dot(dv[0], dv[1])
            L[:, r, 2] = dot(dv[1], dv[1])
            L[:, r, 3] = 2.0 * dot(dv[0], dv[2])
            L[:, r, 4] = 2.0 * dot(dv[1], dv[2])
            L[:, r, 5] = dot(dv[2], dv[2])
            L[:, r, 6] = 2.0 * dot(dv[0], dv[3])
            L[:, r, 7] = 2.0 * dot(dv[1], dv[3])
            L[:, r, 8] = 2.0 * dot(dv[2], dv[3])
            L[:, r, 9] = dot(dv[3], dv[3])
            dw = cw[:, a] - cw[:, b]
            rho[:, r] = dot(dw, dw)
        best_err = np.full(B, np.inf)
        best_R = np.full((B, 3, 3), np.nan)
        best_t = np.full((B, 3), np.nan)
        for N in (1, 2, 3):
            bet = np.zeros((B, 4))
            if N == 1:
                x = lstsq_hh(L[:, :, [0, 1, 3, 6]], rho)
                neg = x[:, 0] < 0
                b0 = np.sqrt(np.where(neg, -x[:, 0], x[:, 0]))
                bet[:, 0] = b0
                for k in range(1, 4):
                    bet[:, k] = np.where(neg, -x[:, k], x[:, k]) / b0
            elif N == 2:
                x = lstsq_hh(L[:, :, [0, 1, 2]], rho)
                neg = x[:, 0] < 0
                bet[:, 0] = np.sqrt(np.where(neg, -x[:, 0], x[:, 0]))
                bet[:, 1] = np.where(neg, np.where(x[:, 2] < 0, np.sqrt(-x[:, 2]), 0.0),
                                     np.where(x[:, 2] > 0, np.sqrt(x[:, 2]), 0.0))
                bet[:, 0] = np.where(x[:, 1] < 0, -bet[:, 0], bet[:, 0])
            else:
                x = lstsq_hh(L[:, :, [0, 1, 2, 3, 4]], rho)
                neg = x[:, 0] < 0
                bet[:, 0] = np.sqrt(np.where(neg, -x[:, 0], x[:, 0]))
                bet[:, 1] = np.where(neg, np.where(x[:, 2] < 0, np.sqrt(-x[:, 2]), 0.0),
                                     np.where(x[:, 2] > 0, np.sqrt(x[:, 2]), 0.0))
                bet[:, 0] = np.where(x[:, 1] < 0, -bet[:, 0], bet[:, 0])
                bet[:, 2] = x[:, 3] / bet[:, 0]
            bet = gauss_newton(L, rho, bet)
            R, t = pose_from_betas(v, bet, al, Mw)
            u, w_, _ = project(K, R, t, Mw)
            du, dv_ = mp[..., 0] - u, mp[..., 1] - w_
            err = np.zeros(B)
            for i in range(n):
                err = err + np.sqrt(du[:, i] * du[:, i] + dv_[:, i] * dv_[:, i])
            fin = np.isfinite(err) & np.isfinite(R).all((1, 2)) & np.isfinite(t).all(1)
            better = fin & (err < best_err)
            best_err = np.where(better, err, best_err)
            best_R = np.where(better[:, None, None], R, best_R)
            best_t = np.where(better[:, None], t, best_t)
        ok &= np.isfinite(best_err)
    return best_R, best_t, ok


def gauss_newton(L, rho, bet):
    """GN_ITERS Gauss-Newton steps on the 4 betas: A dx = b by Householder least squares, beta += dx."""
    bet = bet.copy()
    for _ in range(GN_ITERS):
        A = np.zeros((L.shape[0], 6, 4))
        b = np.zeros((L.shape[0], 6))
        b0, b1, b2, b3 = bet[:, 0], bet[:, 1], bet[:, 2], bet[:, 3]
        with np.errstate(all="ignore"):
            for i in range(6):
                l = L[:, i]
                A[:, i, 0] = 2 * l[:, 0] * b0 + l[:, 1] * b1 + l[:, 3] * b2 + l[:, 6] * b3
                A[:, i, 1] = l[:, 1] * b0 + 2 * l[:, 2] * b1 + l[:, 4] * b2 + l[:, 7] * b3
                A[:, i, 2] = l[:, 3] * b0 + l[:, 4] * b1 + 2 * l[:, 5] * b2 + l[:, 8] * b3
                A[:, i, 3] = l[:, 6] * b0 + l[:, 7] * b1 + l[:, 8] * b2 + 2 * l[:, 9] * b3
                b[:, i] = rho[:, i] - (l[:, 0] * b0 * b0 + l[:, 1] * b0 * b1 + l[:, 2] * b1 * b1 + l[:, 3] * b0 * b2 +
                                       l[:, 4] * b1 * b2 + l[:, 5] * b2 * b2 + l[:, 6] * b0 * b3 + l[:, 7] * b1 * b3 +
                                       l[:, 8] * b2 * b3 + l[:, 9] * b3 * b3)
        dx = lstsq_hh(A, b)
        bet = bet + dx
    return bet


def pose_from_betas(v, bet, al, Mw):
    """Camera-frame control points sum_k beta_k v_k, the sample's camera points, the sign fix and the absolute
    orientation: R = u1 v1^T + u2 v2^T + det(V) (u1 x u2) v3^T from the eigenvectors V of A^T A, A = sum (pc -
    pc0)(pw - pw0)^T, u1 = A v1 normalised, u2 = A v2 orthogonalised against u1 and normalised; t = pc0 - R pw0."""
    B, n = Mw.shape[0], Mw.shape[1]
    with np.errstate(all="ignore"):
        cc = np.zeros((B, 4, 3))
        for j in range(4):
            for k in range(3):
                cc[:, j, k] = (bet[:, 0] * v[:, 0, 3 * j + k] + bet[:, 1] * v[:, 1, 3 * j + k] +
                               bet[:, 2] * v[:, 2, 3 * j + k] + bet[:, 3] * v[:, 3, 3 * j + k])
        pc = np.zeros((B, n, 3))
        for k in range(3):
            pc[:, :, k] = (al[:, :, 0] * cc[:, None, 0, k] + al[:, :, 1] * cc[:, None, 1, k] +
                           al[:, :, 2] * cc[:, None, 2, k] + al[:, :, 3] * cc[:, None, 3, k])
        flip = pc[:, 0, 2] < 0
        pc = np.where(flip[:, None, None], -pc, pc)
        pc0 = _mean(pc)
        pw0 = _mean(Mw)
        A = np.zeros((B, 3, 3))
        for i in range(n):
            A += (pc[:, i] - pc0)[:, :, None] * (Mw[:, i] - pw0)[:, None, :]
        S = np.zeros((B, 3, 3))
        for a in range(3):
            for b in range(3):
                S[:, a, b] = A[:, 0, a] * A[:, 0, b] + A[:, 1, a] * A[:, 1, b] + A[:, 2, a] * A[:, 2, b]
        lam, V = jacobi(S, SWEEPS3)
        order = np.argsort(-lam, axis=1, kind="stable")
        V = np.take_along_axis(V, order[:, None, :], 2)
        v1, v2, v3 = V[:, :, 0], V[:, :, 1], V[:, :, 2]

        def mv(x):
            return np.stack([A[:, i, 0] * x[:, 0] + A[:, i, 1] * x[:, 1] + A[:, i, 2] * x[:, 2] for i in range(3)], 1)

        def dot(x, y):
            return x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1] + x[:, 2] * y[:, 2]
        u1 = mv(v1)
        u1 = u1 / np.sqrt(dot(u1, u1))[:, None]
        u2 = mv(v2)
        u2 = u2 - dot(u1, u2)[:, None] * u1
        u2 = u2 / np.sqrt(dot(u2, u2))[:, None]
        u3 = np.stack([u1[:, 1] * u2[:, 2] - u1[:, 2] * u2[:, 1], u1[:, 2] * u2[:, 0] - u1[:, 0] * u2[:, 2],
                       u1[:, 0] * u2[:, 1] - u1[:, 1] * u2[:, 0]], 1)
        detV = (v1[:, 0] * (v2[:, 1] * v3[:, 2] - v2[:, 2] * v3[:, 1]) -
                v2[:, 0] * (v1[:, 1] * v3[:, 2] - v1[:, 2] * v3[:, 1]) +
                v3[:, 0] * (v1[:, 1] * v2[:, 2] - v1[:, 2] * v2[:, 1]))
        sgn = np.where(detV < 0, -1.0, 1.0)
        R = np.zeros((B, 3, 3))
        for i in range(3):
            for j in range(3):
                R[:, i, j] = u1[:, i] * v1[:, j] + u2[:, i] * v2[:, j] + sgn * u3[:, i] * v3[:, j]
        t = np.stack([pc0[:, i] - (R[:, i, 0] * pw0[:, 0] + R[:, i, 1] * pw0[:, 1] + R[:, i, 2] * pw0[:, 2])
                      for i in range(3)], 1)
    return R, t


def score(K, R, t, M, m, thr):
    """(inliers [B], sse [B], flags [B, N]) of poses R [B, 3, 3], t [B, 3] over points M [N, 3], m [N, 2]: point i
    is an inlier when its depth is > 0 and e_i = sqrt(du^2 + dv^2) < thr; sse sums du^2 + dv^2 over the inliers in
    point order."""
    u, v, z = project(np.asarray(K, np.float64), R, t, np.broadcast_to(M, (R.shape[0],) + M.shape))
    with np.errstate(all="ignore"):
        du, dv = m[None, :, 0] - u, m[None, :, 1] - v
        e2 = du * du + dv * dv
        flag = (z > 0) & (np.sqrt(e2) < thr)
    sse = np.zeros(R.shape[0])
    for i in range(M.shape[0]):
        sse = sse + np.where(flag[:, i], e2[:, i], 0.0)
    return flag.sum(1), sse, flag


def better(a, b):
    """True when score a = (inliers, sse, h) ranks before b: more inliers, then less sse, then lower h."""
    if a[0] != b[0]:
        return a[0] > b[0]
    if a[1] != b[1]:
        return a[1] < b[1]
    return a[2] < b[2]


def ransac_camera(K, R0, t0, M, m, c, selected, n_hyp, thr, min_inl, seed):
    """One camera's RANSAC.  Returns a dict: R, t (the start pose), status, inliers, sse, h (the selection's winner;
    for status 1 and 3 R0's), flags (of the start pose), and per hypothesis idx [n_hyp, 5], hR, ht, ok, cnt (-1 when
    degenerate), hsse."""
    K, R0, t0 = (np.asarray(a, np.float64) for a in (K, R0, t0))
    M, m = np.asarray(M, np.float64).reshape(-1, 3), np.asarray(m, np.float64).reshape(-1, 2)
    n = len(M)
    c0, s0, f0 = score(K, R0[None], t0[None], M, m, thr)
    out = dict(R=R0.copy(), t=t0.copy(), inliers=int(c0[0]), sse=float(s0[0]), h=-1, flags=f0[0])
    if not selected:
        return dict(out, status=NOT_SELECTED)
    if n < 5:
        return dict(out, status=TOO_FEW)
    idx = samples(seed, c, n, n_hyp)
    good = (idx >= 0).all(1)
    sel = np.where(good[:, None], idx, 0)
    hR, ht, ok = epnp(K, M[sel], m[sel])
    ok &= good
    cnt, hsse, _ = score(K, np.where(ok[:, None, None], hR, np.eye(3)), np.where(ok[:, None], ht, 0.0), M, m, thr)
    cnt = np.where(ok, cnt, -1)
    hsse = np.where(ok, hsse, 0.0)
    out.update(idx=idx, hR=hR, ht=ht, ok=ok, cnt=cnt, hsse=hsse)
    best = (out["inliers"], out["sse"], -1)
    # order by inliers, then sse, then h: lexsort's last key is the primary one
    h = int(np.lexsort((np.arange(n_hyp), hsse, -cnt))[0])
    if better((int(cnt[h]), float(hsse[h]), h), best):
        best = (int(cnt[h]), float(hsse[h]), h)
    if best[2] < 0:
        return dict(out, status=KEPT)
    out.update(inliers=best[0], sse=best[1], h=best[2])
    if best[0] < min_inl:
        return dict(out, status=FEW_INLIERS)
    _, _, f = score(K, hR[h][None], ht[h][None], M, m, thr)
    out.update(R=hR[h].copy(), t=ht[h].copy(), flags=f[0])
    return dict(out, status=REPLACED)


def rodrigues(w):
    w = np.asarray(w, np.float64)
    th = float(np.linalg.norm(w))
    if th < 1e-300:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


def unit(rng):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v)


def scene(rng, n, out_frac, rot_deg, depth=(4.0, 20.0), noise=0.5, shift=0.3, W=1280, H=720):
    """One camera of the RANSAC tests: (K, R0, t0, M [n, 3], m [n, 2], Rt, tt, outlier mask).  Points at depths in
    `depth` over the image, observed with Gaussian noise of `noise` px; a share out_frac of them replaced by pixels drawn
    uniformly over the image (gross outliers); R0 rot_deg off the true rotation about a random axis and the start
    camera centre shift x the mean depth away from the true one."""
    f = 0.9 * W
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1.0]])
    Rt = rodrigues(rng.normal(0, 0.3, 3))
    Ct = rng.normal(0, 1.0, 3)
    tt = -Rt @ Ct
    z = rng.uniform(depth[0], depth[1], n)
    u, v = rng.uniform(20, W - 20, n), rng.uniform(20, H - 20, n)
    Pc = np.stack([(u - W / 2) / f * z, (v - H / 2) / f * z, z], 1)
    M = (Pc - tt) @ Rt
    m = np.stack([u, v], 1) + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < out_frac
    m[out] = np.stack([rng.uniform(0, W, out.sum()), rng.uniform(0, H, out.sum())], 1)
    R0 = rodrigues(unit(rng) * np.deg2rad(rot_deg)) @ Rt
    C0 = Ct + shift * z.mean() * unit(rng)
    return K, R0, -R0 @ C0, M, m, Rt, tt, out


def pose_error(R, t, Rt, tt):
    """(rotation error in degrees, camera-centre distance) of (R, t) against (Rt, tt)"""
    c = np.clip((np.trace(np.asarray(R) @ np.asarray(Rt).T) - 1) / 2, -1.0, 1.0)
    return float(np.degrees(np.arccos(c))), float(np.linalg.norm(-np.asarray(R).T @ t + np.asarray(Rt).T @ tt))


def prev_errs(flags, out_px=1e3):
    """prevErrs for a second solve from a RANSAC start: 0 for the start's inliers, out_px for the rest, so that the
    solve's first Tukey weights drop the points RANSAC found to be outliers."""
    return np.where(np.asarray(flags, bool), 0.0, out_px)
