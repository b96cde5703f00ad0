"""A float64 restatement of the map-point registration of cosl_assoc_solver_submit (DESIGN.md 5.6), on top of
pose_mappts_dense's jacobians and camera_point.  It scans every feature of an entry (no grid) and resolves claims in a
plain loop.

Per query pair (j, c): m_hat = pi_c(X_j), S = H_X P_X H_X^T + H_c P_c H_c^T (the second term with the entry's P_c only);

    status 7 unless the depth, m_hat and S are finite; 1 depth <= 0; 2 m_hat outside [0, W) x [0, H);
    d2_f = (m_f - m_hat)^T (S + Sigma_f)^-1 (m_f - m_hat) over the features of entry c; f* the least (d2, f) with
    d2 < gate, d2_2 the second least such d2 (+inf without); 3 without f*; 4 f* owned;
    5 (finite track_gate only) an earlier observation k of f* with depth <= 0 or not d2_k < track_gate,
      d2_k = nu_k^T (H_X P_X H_X^T + H_c P_c H_c^T + pixel_var I)^-1 nu_k;
    6 another pair at 0 holds f* with a smaller (d2, point index); else 0.

The quadratic forms are the adjugate form (c nu0^2 - 2 b nu0 nu1 + a nu1^2) / det, not the kernel's |L^-1 nu|^2, so
the two share no arithmetic; a Sigma_f + S that is not positive definite takes no part.

    predict(K, R, t, Pc, X, PX, add)             -> (depth, m_hat [2], S [2, 2] + add I)
    quad(A, nu)                                  -> nu^T A^-1 nu over stacked 2x2 A, NaN where A is not PD
    associate(...)                               -> dict of status, feat, d2 [Q, 2], pred [Q, 5], as the device
    search_maha_nearest(m, var, max_dist, mf)    -> the reference's searchMahaNearestFeatPt argmin
    scene(...), mc_trial(...), mc_stats(...)     -> the shapes the tests draw and the Monte-Carlo chain"""
import math

import numpy as np

import pose_dense as pd
import pose_mappts_dense as md
import tri_dense as td

GATE_99 = 9.21034037197618  # the 99 % quantile of chi-square with 2 dof


def predict(K, R, t, Pc, X, PX, add=0.0):
    """(depth, m_hat, S) of X with covariance PX in camera (K, R, t), Pc the entry's pose covariance or None."""
    m, HX, Hc, z = md.jacobians(K, R, t, X)
    S = HX @ np.asarray(PX, np.float64).reshape(3, 3) @ HX.T + add * np.eye(2)
    if Pc is not None:
        S = S + Hc @ np.asarray(Pc, np.float64).reshape(6, 6) @ Hc.T
    return z, m, S


def quad(A, nu):
    """nu^T A^-1 nu for A [..., 2, 2], nu [..., 2]; NaN where A is not positive definite."""
    a, b, c = A[..., 0, 0], 0.5 * (A[..., 0, 1] + A[..., 1, 0]), A[..., 1, 1]
    with np.errstate(all="ignore"):
        det = a * c - b * b
        q = (c * nu[..., 0] ** 2 - 2.0 * b * nu[..., 0] * nu[..., 1] + a * nu[..., 1] ** 2) / det
    return np.where((a > 0) & (det > 0), q, np.nan)


def _sym(P, n):
    P = np.asarray(P, np.float64).reshape(n, n)
    return 0.5 * (P + P.T)


def associate(K, R, t, cam_cov, wh, feat_off, mf, X, P, q_off, q_cam, covf=None, owned=None, trk_off=None,
              trk_cam=None, trk_m=None, pixel_var=1.0, gate=GATE_99, track_gate=math.inf, chunk=256):
    """Every query pair of one submit in cosl_assoc_solver_submit's form; a dict of the device's outputs."""
    K, R = np.asarray(K, np.float64).reshape(-1, 3, 3), np.asarray(R, np.float64).reshape(-1, 3, 3)
    t = np.asarray(t, np.float64).reshape(-1, 3)
    wh = np.asarray(wh).reshape(-1, 2)
    fo = np.asarray(feat_off, np.int64)
    mf = np.asarray(mf, np.float64).reshape(-1, 2)
    nF = len(mf)
    Sf = (np.broadcast_to(pixel_var * np.eye(2), (nF, 2, 2)) if covf is None
          else np.asarray(covf, np.float64).reshape(-1, 2, 2))
    own = np.zeros(nF, bool) if owned is None else np.asarray(owned).astype(bool)
    to = np.zeros(nF + 1, np.int64) if trk_off is None else np.asarray(trk_off, np.int64)
    Pc = [None] * len(K) if cam_cov is None else [None if p is None else _sym(p, 6) for p in cam_cov]
    X = np.asarray(X, np.float64).reshape(-1, 3)
    P = [_sym(p, 3) for p in np.asarray(P, np.float64).reshape(-1, 9)]
    qo, qc = np.asarray(q_off, np.int64), np.asarray(q_cam, np.int64)
    nQ = int(qo[-1])
    qpt = np.repeat(np.arange(len(X)), np.diff(qo))
    status = np.zeros(nQ, np.int32)
    feat = np.full(nQ, -1, np.int32)
    d2 = np.full((nQ, 2), math.nan)
    pred = np.full((nQ, 5), math.nan)
    S_all = np.zeros((nQ, 2, 2))
    with np.errstate(all="ignore"):
        for q in range(nQ):
            j, c = qpt[q], qc[q]
            z, m, S = predict(K[c], R[c], t[c], Pc[c], X[j], P[j])
            S_all[q] = S
            if not (np.isfinite(z) and np.isfinite(m).all() and np.isfinite(S).all()):
                status[q] = 7
                continue
            pred[q] = [m[0], m[1], S[0, 0], S[0, 1], S[1, 1]]
            if not z > 0:
                status[q], pred[q] = 1, math.nan
            elif not (0 <= m[0] < wh[c, 0] and 0 <= m[1] < wh[c, 1]):
                status[q] = 2
        # the search, one entry at a time over every one of its features
        for c in range(len(K)):
            qs = np.flatnonzero((qc == c) & (status == 0))
            f0, f1 = fo[c], fo[c + 1]
            for k in range(0, len(qs), chunk):
                qq = qs[k:k + chunk]
                if f1 == f0:
                    status[qq] = 3
                    d2[qq] = math.inf
                    continue
                nu = mf[None, f0:f1] - pred[qq, None, :2]
                dd = quad(S_all[qq, None] + Sf[None, f0:f1], nu)
                inside = np.where(dd < gate, dd, math.inf)
                best = np.argmin(inside, axis=1)  # the first of equal values: the least feature index
                b = inside[np.arange(len(qq)), best]
                second = np.partition(inside, 1, axis=1)[:, 1] if f1 - f0 > 1 else np.full(len(qq), math.inf)
                d2[qq, 0], d2[qq, 1] = b, second
                found = np.isfinite(b)
                status[qq[~found]] = 3
                feat[qq[found]] = f0 + best[found]
        for q in np.flatnonzero(status == 0):
            f = feat[q]
            if own[f]:
                status[q] = 4
            elif track_gate < math.inf:
                j = qpt[q]
                for k in range(to[f], to[f + 1]):
                    e = int(trk_cam[k])
                    z, m, S = predict(K[e], R[e], t[e], Pc[e], X[j], P[j], pixel_var)
                    dk = quad(S, np.asarray(trk_m[k], np.float64) - m)
                    if not (z > 0 and dk < track_gate):
                        status[q] = 5
                        break
    # claims: the least (d2, point index) among the pairs at 0 that hold a feature keeps it
    holders = {}
    for q in np.flatnonzero(status == 0):
        holders.setdefault(int(feat[q]), []).append(q)
    for qs in holders.values():
        win = min(qs, key=lambda q: (d2[q, 0], qpt[q]))
        for q in qs:
            if q != win:
                status[q] = 6
    return dict(status=status, feat=feat, d2=d2, pred=pred)


def search_maha_nearest(m, var, max_dist, mf):
    """searchMahaNearestFeatPt (app/SL_SingleSLAM.cpp:1141-1166) restated: ivar = var^-1 / max_dist, then the first
    feature of the list with the least mahaDist2 under ivar (a strict < over the list); None without features."""
    ivar = np.linalg.inv(np.asarray(var, np.float64).reshape(2, 2)) / max_dist
    d_min, p_min = math.inf, None
    for i, p in enumerate(np.asarray(mf, np.float64).reshape(-1, 2)):
        r = p - np.asarray(m, np.float64)
        d = float(r @ ivar @ r)
        if d < d_min:
            d_min, p_min = d, i
    return p_min


# ---------------------------------------------------------------- scenes
def scene(rng, n_entries, n_feats, n_pts, q_lo=1, q_hi=4, half=True, owned_share=0.1, trk_hi=3, n_empty=0,
          sigma_x=(1e-4, 1e-2)):
    """A submit over n_entries entries of td.rig with K_TRI (1280 x 720), n_pts points of td.scene_points with a prior
    mean drawn from a random P (standard deviations sigma_x, m^2), each querying q_lo to q_hi distinct entries.  Entry c
    has n_feats features (the last n_empty entries none): the projections of a random share of the points plus noise,
    the rest uniform clutter.  With half, covf holds a random 2x2 (0.25 to 2.25 px^2) on half the features and
    pixel_var I on the others, and half the entries have a pose covariance.  owned_share of the features are owned, and
    each has 0 to trk_hi earlier observations on other entries.  Returns the keyword arguments of associate and
    AssocSolver.submit."""
    R, t = td.rig(rng, n_entries, spread=1.5)
    K = np.array([td.K_TRI] * n_entries)
    wh = np.tile([td.W_TRI, td.H_TRI], (n_entries, 1)).astype(np.int32)
    cc = [md.random_spd(rng, 6, 1e-8, 1e-6) if half and c % 2 == 0 else None for c in range(n_entries)]
    Xt = td.scene_points(rng, n_pts)
    Pj = np.array([md.random_spd(rng, 3, *sigma_x) for _ in range(n_pts)])
    X = Xt + np.array([rng.multivariate_normal(np.zeros(3), p) for p in Pj])
    counts = [0 if c >= n_entries - n_empty else n_feats for c in range(n_entries)]
    fo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    mf = np.empty((fo[-1], 2))
    for c in range(n_entries):
        n = counts[c]
        if not n:
            continue
        src = rng.choice(n_pts, min(n_pts, int(0.7 * n)), replace=False)
        u, v = pd.project(td.K_TRI, R[c], t[c], Xt[src])
        true = np.column_stack([u, v]) + rng.normal(0.0, 1.0, (len(src), 2))
        clutter = rng.uniform([0.0, 0.0], [td.W_TRI, td.H_TRI], (n - len(src), 2))
        mf[fo[c]:fo[c + 1]] = rng.permutation(np.concatenate([true, clutter]))
    nF = int(fo[-1])
    covf = np.broadcast_to(np.eye(2), (nF, 2, 2)).copy()
    if half:
        some = rng.random(nF) < 0.5
        covf[some] = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in range(int(some.sum()))])
    owned = (rng.random(nF) < owned_share).astype(np.int32)
    tl = rng.integers(0, trk_hi + 1, nF)
    to = np.concatenate([[0], np.cumsum(tl)]).astype(np.int32)
    tc = rng.integers(0, n_entries, int(to[-1])).astype(np.int32)
    tm = mf[np.repeat(np.arange(nF), tl)] + rng.normal(0.0, 30.0, (int(to[-1]), 2))
    qn = rng.integers(q_lo, q_hi + 1, n_pts)
    qo = np.concatenate([[0], np.cumsum(qn)]).astype(np.int32)
    qc = np.concatenate([rng.choice(n_entries, k, replace=False) for k in qn]).astype(np.int32)
    return dict(K=K, R=R, t=t, cam_cov=cc, wh=wh, feat_off=fo, mf=mf, X=X, P=Pj, q_off=qo, q_cam=qc, covf=covf,
                owned=owned, trk_off=to, trk_cam=tc, trk_m=tm)


def mc_trial(rng, n_pts=100, miss=0.3, clutter=0.5, owned_share=0.1, pixel_var=1.0):
    """One Monte-Carlo rig for the chain: two key frames (entries 0 and 1) observe n_pts true points with pixel_var I
    noise and td.triangulate_all gives each point X and P; a later frame (entry 2, its estimate drawn from the pose
    covariance P_c it carries) has a feature for each point with probability 1 - miss, drawn from the true projection
    with a random Sigma_f (0.25 to 2.25 px^2), plus clutter * n_pts uniform features; owned_share of all features are
    owned.  A point's feature has its two key-frame observations as its track, a clutter feature two uniform ones.
    Returns (the keyword arguments of associate, truth: the feature of each point or -1, the status-0 points)."""
    Rt, tt = td.rig(rng, 3)
    Xt = np.array([X for X in td.scene_points(rng, 4 * n_pts)
                   if all(md.camera_point(Ri, ti, X)[2] > 0.5 for Ri, ti in zip(Rt, tt))][:n_pts])
    n_pts = len(Xt)
    Pc2 = md.random_spd(rng, 6, 1e-8, 1e-6)
    d = rng.multivariate_normal(np.zeros(6), Pc2)
    R = np.array([Rt[0], Rt[1], Rt[2] @ pd.exp_map(d[:3])])
    t = np.array([tt[0], tt[1], tt[2] + d[3:]])
    K = np.array([td.K_TRI] * 3)
    Sm = np.broadcast_to(pixel_var * np.eye(2), (n_pts * 2, 2, 2))
    mk = np.array([td.observe(td.K_TRI, Rt[:2], tt[:2], X, Sm[:2], rng) for X in Xt])  # [n, 2, 2]
    tri = td.triangulate_all(K[:2], Rt[:2], tt[:2], None, np.arange(n_pts + 1) * 2, np.tile([0, 1], n_pts),
                             mk.reshape(-1, 2), None, pixel_var)
    good = np.flatnonzero(tri["status"] == 0)
    u, v = pd.project(td.K_TRI, Rt[2], tt[2], Xt)
    seen = np.flatnonzero(rng.random(n_pts) >= miss)
    Sf_true = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in seen])
    m_true = np.column_stack([u, v])[seen] + np.array([rng.multivariate_normal(np.zeros(2), S) for S in Sf_true])
    n_cl = int(clutter * n_pts)
    m_cl = rng.uniform([0.0, 0.0], [td.W_TRI, td.H_TRI], (n_cl, 2))
    Sf_cl = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in range(n_cl)])
    order = rng.permutation(len(seen) + n_cl)
    mf = np.concatenate([m_true, m_cl])[order]
    covf = np.concatenate([Sf_true, Sf_cl])[order]
    src = np.concatenate([seen, np.full(n_cl, -1)])[order]
    owned = (rng.random(len(mf)) < owned_share).astype(np.int32)
    trk_m = np.array([mk[s] if s >= 0 else rng.uniform([0.0, 0.0], [td.W_TRI, td.H_TRI], (2, 2)) for s in src])
    truth = np.full(n_pts, -1)
    truth[src[src >= 0]] = np.flatnonzero(src >= 0)
    kw = dict(K=K, R=R, t=t, cam_cov=[None, None, Pc2], wh=np.tile([td.W_TRI, td.H_TRI], (3, 1)).astype(np.int32),
              feat_off=np.array([0, 0, 0, len(mf)], np.int32), mf=mf, covf=covf, owned=owned,
              trk_off=np.arange(len(mf) + 1, dtype=np.int32) * 2, trk_cam=np.tile([0, 1], len(mf)).astype(np.int32),
              trk_m=trk_m.reshape(-1, 2), X=tri["X"][good], P=tri["P"][good],
              q_off=np.arange(len(good) + 1, dtype=np.int32), q_cam=np.full(len(good), 2, np.int32))
    return kw, truth[good], owned


def mc_stats(results, wh=(td.W_TRI, td.H_TRI)):
    """(mean d2 of the registered true matches, precision, recall) over (output, truth, owned) triples: a registered
    pair is a true match when its feature is its point's own; recall counts the points whose own feature exists, is
    not owned and whose prediction lies in the wh[0] x wh[1] image."""
    d2, reg, right, can = [], 0, 0, 0
    for r, truth, owned in results:
        ok = r["status"] == 0
        hit = ok & (r["feat"] == truth) & (truth >= 0)
        d2.append(r["d2"][hit, 0])
        reg += int(ok.sum())
        right += int(hit.sum())
        inside = (r["pred"][:, 0] >= 0) & (r["pred"][:, 0] < wh[0]) & (r["pred"][:, 1] >= 0) & (r["pred"][:, 1] < wh[1])
        can += int(((truth >= 0) & inside & (owned[np.maximum(truth, 0)] == 0)).sum())
    return float(np.mean(np.concatenate(d2))), right / max(reg, 1), right / max(can, 1)
