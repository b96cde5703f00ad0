"""Seeded synthetic inputs for the two hot paths (SURVEY.md 8d).  numpy/scipy only.

* images: static texture (band-limited noise octaves + Gaussian blobs) warped by a smooth
  per-camera similarity; ground-truth flow known in closed form.
* BA scenes: camera rigs along a smooth trajectory, points in a slab in front of it, windowed
  visibility, Gaussian pixel noise + gross outliers, perturbed initial values.
"""
import numpy as np
from scipy import ndimage

from .problem import BAProblem

BASE_SEED = 20130901


def make_texture(h, w, seed, n_blobs=None, pad=32):
    """Float32 texture of size (h+2*pad, w+2*pad) in 0..255 with plenty of Shi-Tomasi corners."""
    rng = np.random.default_rng(seed)
    H, W = h + 2 * pad, w + 2 * pad
    img = np.zeros((H, W), np.float64)
    for o, (sigma, amp) in enumerate([(24.0, 30.0), (10.0, 22.0), (4.0, 16.0), (1.6, 10.0)]):
        n = rng.standard_normal((H, W))
        g = ndimage.gaussian_filter(n, sigma, mode="wrap")
        img += amp * g / (g.std() + 1e-12)
    if n_blobs is None:
        n_blobs = max(500, (h * w) // 140)
    blobs = np.zeros((H, W), np.float64)
    ys = rng.integers(0, H, n_blobs)
    xs = rng.integers(0, W, n_blobs)
    amps = rng.uniform(40, 110, n_blobs) * rng.choice([-1.0, 1.0], n_blobs)
    np.add.at(blobs, (ys, xs), amps)
    # two blob scales (sigma 1.5 and 2.5 px), normalised so a single blob peaks at ~amp
    b1 = ndimage.gaussian_filter(blobs, 1.5, mode="wrap") * (2 * np.pi * 1.5 ** 2)
    rng2 = np.random.default_rng(seed + 7)
    blobs2 = np.zeros((H, W), np.float64)
    ys = rng2.integers(0, H, n_blobs // 2)
    xs = rng2.integers(0, W, n_blobs // 2)
    np.add.at(blobs2, (ys, xs), rng2.uniform(40, 110, n_blobs // 2) * rng2.choice([-1.0, 1.0], n_blobs // 2))
    b2 = ndimage.gaussian_filter(blobs2, 2.5, mode="wrap") * (2 * np.pi * 2.5 ** 2)
    img = 128.0 + img + b1 + b2
    return np.clip(img, 0, 255).astype(np.float32)


class ImageSequence:
    """Frames of one camera: frame k = texture warped by the similarity S_k (about the image
    centre): p_tex = c + s_k R(a_k) (p - c) + d_k, with smooth (a, s, d) trajectories."""

    def __init__(self, h, w, seed, n_frames=8, max_shift=3.0, max_rot_deg=0.2, max_scale=0.001,
                 noise_sigma=1.0, pad=32):
        self.h, self.w, self.pad = h, w, pad
        self.seed = seed
        self.rng = np.random.default_rng(seed + 1)
        self.tex = make_texture(h, w, seed, pad=pad)
        # cubic prefilter once
        self.coef = ndimage.spline_filter(self.tex.astype(np.float64), order=3, mode="mirror")
        vel = self.rng.uniform(-1, 1, 2)
        vel = vel / np.linalg.norm(vel) * max_shift * self.rng.uniform(0.5, 1.0)
        self.vel = vel
        self.rot = np.deg2rad(max_rot_deg) * self.rng.uniform(-1, 1)
        self.scl = max_scale * self.rng.uniform(-1, 1)
        self.noise_sigma = noise_sigma
        self.n_frames = n_frames
        self.frames = [self.render(k) for k in range(n_frames)]

    def params(self, k):
        # smooth, bounded excursion so that the padded texture always covers the frame
        ph = 2 * np.pi * k / 64.0
        d = self.vel * k * (1.0 if k < 9 else 9.0 / k)  # <= 9 frames of drift
        d = np.clip(d, -(self.pad - 6), self.pad - 6)
        a = self.rot * k * (1.0 if k < 9 else 9.0 / k)
        s = 1.0 + self.scl * k * (1.0 if k < 9 else 9.0 / k)
        return a, s, d

    def tex_coords(self, k, x, y):
        """Texture (x, y) coordinates (pixel-centre convention, padded frame) of frame-k pixel
        coordinates (x, y) given in the half-integer-centre convention of the tracker."""
        a, s, d = self.params(k)
        cx, cy = self.w / 2.0, self.h / 2.0
        ca, sa = np.cos(a) * s, np.sin(a) * s
        xt = cx + ca * (x - cx) - sa * (y - cy) + d[0]
        yt = cy + sa * (x - cx) + ca * (y - cy) + d[1]
        return xt + self.pad, yt + self.pad

    def render(self, k):
        ys, xs = np.mgrid[0:self.h, 0:self.w]
        xt, yt = self.tex_coords(k, xs + 0.5, ys + 0.5)
        # map_coordinates uses integer-centre indices
        v = ndimage.map_coordinates(self.coef, [yt - 0.5, xt - 0.5], order=3, mode="mirror",
                                    prefilter=False)
        if self.noise_sigma > 0:
            v = v + np.random.default_rng(self.seed * 1000 + 17 + k).normal(
                0, self.noise_sigma, v.shape)
        return np.clip(np.rint(v), 0, 255).astype(np.uint8)

    def flow_truth(self, k0, k1, x, y):
        """Where does the scene point seen at (x, y) in frame k0 appear in frame k1?"""
        xt, yt = self.tex_coords(k0, x, y)
        xt, yt = xt - self.pad, yt - self.pad
        a, s, d = self.params(k1)
        cx, cy = self.w / 2.0, self.h / 2.0
        ux, uy = xt - cx - d[0], yt - cy - d[1]
        ca, sa = np.cos(a) / s, np.sin(a) / s
        return cx + ca * ux + sa * uy, cy - sa * ux + ca * uy

    def frame(self, i):
        """Ping-pong access so that arbitrarily long runs stay temporally smooth."""
        n = self.n_frames
        if n == 1:
            return self.frames[0]
        period = 2 * (n - 1)
        j = i % period
        return self.frames[j if j < n else period - j]

    def frame_index(self, i):
        n = self.n_frames
        if n == 1:
            return 0
        period = 2 * (n - 1)
        j = i % period
        return j if j < n else period - j


def _rodrigues(w):
    th = np.linalg.norm(w)
    if th < 1e-15:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def make_ba_scene(n_cams=4, n_kf=5, n_pts=20000, width=1280, height=720, seed=BASE_SEED,
                  m_con=None, n_con=2, window=4, p_vis=0.55, noise_px=0.5, outlier_frac=0.02,
                  pose_rot_deg=0.1, pose_trans_frac=0.002, point_frac=0.002, min_obs=2,
                  sort_by_home=False):
    """Synthetic multi-camera BA problem (SURVEY.md 8d).  Returns (BAProblem with perturbed
    initial values, dict of ground truth).  sort_by_home: number the points in the order of their
    home key frame (map-creation order of a real SLAM run), so that contiguous point shards see
    DIFFERENT camera pairs -- the realistic case for the multi-GPU structure exchange."""
    rng = np.random.default_rng(seed)
    f = 0.9 * width
    K1 = np.array([f, 0, width / 2.0, 0, f, height / 2.0, 0, 0, 1.0])
    step = 0.35  # metres between key frames
    # rig: cameras side by side with small yaw offsets
    rig_off = np.array([[(c - (n_cams - 1) / 2.0) * 0.6, 0.0, 0.0] for c in range(n_cams)])
    rig_yaw = np.array([np.deg2rad((c - (n_cams - 1) / 2.0) * 8.0) for c in range(n_cams)])
    Rs, ts, Cs = [], [], []
    for kf in range(n_kf):
        s = kf * step
        centre = np.array([s, 0.15 * np.sin(0.05 * s * 2 * np.pi), 0.1 * np.cos(0.03 * s * 2 * np.pi)])
        heading = np.deg2rad(3.0) * np.sin(0.02 * s * 2 * np.pi)
        for c in range(n_cams):
            # world: x along the trajectory, cameras look along +z
            Rwc = _rodrigues(np.array([0.0, heading + rig_yaw[c], 0.0]))
            C = centre + rig_off[c]
            R = Rwc.T
            Rs.append(R)
            ts.append(-R @ C)
            Cs.append(C)
    Rs, ts, Cs = np.array(Rs), np.array(ts), np.array(Cs)
    m = n_kf * n_cams
    # points: slab 4..20 m in front of the trajectory, home key frame uniform
    home = rng.integers(0, n_kf, n_pts)
    if sort_by_home:
        home = np.sort(home)
    depth = rng.uniform(4.0, 20.0, n_pts)
    lat = rng.uniform(-1.0, 1.0, n_pts) * depth * (width / 2.0 / f) * 1.3
    vert = rng.uniform(-1.0, 1.0, n_pts) * depth * (height / 2.0 / f) * 1.1
    X = np.stack([home * step + lat, vert, depth], 1)
    # visibility
    cam_kf = np.repeat(np.arange(n_kf), n_cams)
    obs_pt, obs_cam, obs_xy = [], [], []
    chunk = 4096
    for a in range(0, n_pts, chunk):
        b = min(n_pts, a + chunk)
        Xc = np.einsum("jab,ib->ija", Rs, X[a:b]) + ts[None]  # [pts, cams, 3]
        z = Xc[..., 2]
        u = f * Xc[..., 0] / z + width / 2.0
        v = f * Xc[..., 1] / z + height / 2.0
        ok = (z > 0.5) & (u >= 0) & (u < width) & (v >= 0) & (v < height)
        ok &= np.abs(cam_kf[None, :] - home[a:b, None]) <= window
        ok &= rng.random(ok.shape) < p_vis
        pi, ci = np.nonzero(ok)
        obs_pt.append(pi + a)
        obs_cam.append(ci)
        obs_xy.append(np.stack([u[pi, ci], v[pi, ci]], 1))
    obs_pt = np.concatenate(obs_pt)
    obs_cam = np.concatenate(obs_cam)
    obs_xy = np.concatenate(obs_xy)
    # keep points with >= min_obs observations (parseInputs keeps nfpts > 1)
    cnt = np.bincount(obs_pt, minlength=n_pts)
    keep = cnt >= min_obs
    remap = -np.ones(n_pts, np.int64)
    remap[keep] = np.arange(keep.sum())
    sel = keep[obs_pt]
    obs_pt, obs_cam, obs_xy = remap[obs_pt[sel]], obs_cam[sel], obs_xy[sel]
    X = X[keep]
    n = len(X)
    order = np.lexsort((obs_cam, obs_pt))
    obs_pt, obs_cam, obs_xy = obs_pt[order], obs_cam[order], obs_xy[order]
    ptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(obs_pt, minlength=n), out=ptr[1:])
    xy_true = obs_xy.copy()
    xy = obs_xy + rng.normal(0, noise_px, obs_xy.shape)
    is_out = rng.random(len(xy)) < outlier_frac
    xy[is_out] += rng.uniform(-30, 30, (is_out.sum(), 2))
    # perturbed start
    if m_con is None:
        m_con = n_cams
    R0 = Rs.copy()
    t0 = ts.copy()
    base = step  # inter-key-frame baseline
    for j in range(m_con, m):
        dR = _rodrigues(rng.normal(0, np.deg2rad(pose_rot_deg) / np.sqrt(3), 3))
        Cj = Cs[j] + rng.normal(0, pose_trans_frac * max(base, 1.0) / np.sqrt(3), 3)
        R0[j] = dR @ Rs[j]
        t0[j] = -R0[j] @ Cj
    X0 = X.copy()
    zc = np.maximum(X[:, 2], 1.0)
    X0[n_con:] += rng.normal(0, 1, (n - n_con, 3)) * (point_frac * zc[n_con:, None])
    prob = BAProblem(np.tile(K1, (m, 1)), R0.reshape(m, 9), t0, X0, ptr, obs_cam.astype(np.int32),
                     xy, m_con, n_con)
    truth = dict(R=Rs.reshape(m, 9), t=ts, X=X, xy_true=xy_true, is_outlier=is_out,
                 n_cams=n_cams, n_kf=n_kf)
    return prob, truth


def make_pose_case(n_pts=192, width=1280, height=720, seed=BASE_SEED, noise_px=0.5,
                   outlier_frac=0.05, rot_deg=0.6, trans=0.03):
    """One intraCamEstimate input: (K, R0, t0, Ms, ms, R_true, t_true)."""
    rng = np.random.default_rng(seed)
    f = 0.9 * width
    K = np.array([[f, 0, width / 2.0], [0, f, height / 2.0], [0, 0, 1.0]])
    Rt = _rodrigues(rng.normal(0, 0.2, 3))
    C = rng.normal(0, 0.5, 3)
    tt = -Rt @ C
    depth = rng.uniform(4.0, 20.0, n_pts)
    u = rng.uniform(20, width - 20, n_pts)
    v = rng.uniform(20, height - 20, n_pts)
    Pc = np.stack([(u - width / 2) / f * depth, (v - height / 2) / f * depth, depth], 1)
    Ms = (Pc - tt) @ Rt  # Rt^T (Pc - t)
    ms = np.stack([u, v], 1) + rng.normal(0, noise_px, (n_pts, 2))
    out = rng.random(n_pts) < outlier_frac
    ms[out] += rng.uniform(-40, 40, (out.sum(), 2))
    R0 = _rodrigues(rng.normal(0, np.deg2rad(rot_deg) / np.sqrt(3), 3)) @ Rt
    t0 = tt + rng.normal(0, trans / np.sqrt(3), 3)
    return K, R0, t0, Ms, ms, Rt, tt


def _rodrigues(w):
    th = float(np.linalg.norm(w))
    if th < 1e-300:
        return np.eye(3)
    k = np.asarray(w, np.float64) / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def make_pose_chains(lengths, key_every=8, seed=0, shift=0.03, lead_free=0, fixed_masks=None):
    """Synthetic input of the post-BA pose-graph spreading (RobustBundleRTS::constructCameraGraphs,
    reference app/SL_CoSLAMRobustBA.cpp:182-232): one chain of camera poses per camera, a smooth
    trajectory; edge k = rigid transform from pose k to pose k+1 measured BEFORE bundle adjustment;
    every `key_every`-th node is a key frame (fixed) and has then been moved by BA (rotation ~shift rad,
    translation ~shift).  lead_free > 0 leaves that many free nodes before the first key frame.
    Returns dict(chain_off, fixed, R, t, eR, et, id1, id2, eR_list, et_list): eR/et have one slot per
    node (slot of a chain's last node zero), eR_list/et_list + id1/id2 are the same edges as a list."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    N = int(off[-1])
    R, t = np.zeros((N, 3, 3)), np.zeros((N, 3))
    eR, et = np.zeros((N, 3, 3)), np.zeros((N, 3))
    fixed = np.zeros(N, np.uint8)
    id1, id2 = [], []
    for c, n in enumerate(lengths):
        a = int(off[c])
        if n == 0:
            continue
        R[a] = _rodrigues(rng.normal(size=3))
        t[a] = rng.normal(size=3)
        for k in range(1, n):
            R[a + k] = _rodrigues(rng.normal(size=3) * 0.05) @ R[a + k - 1]
            t[a + k] = t[a + k - 1] + rng.normal(size=3) * 0.1
        for k in range(n - 1):
            eR[a + k] = R[a + k + 1] @ R[a + k].T
            et[a + k] = t[a + k + 1] - eR[a + k] @ t[a + k]
            id1.append(a + k)
            id2.append(a + k + 1)
        if fixed_masks is not None:
            fixed[a:a + n] = np.asarray(fixed_masks[c], np.uint8)
        else:
            fixed[a + lead_free:a + n:key_every] = 1
        for k in np.nonzero(fixed[a:a + n])[0]:
            R[a + k] = _rodrigues(rng.normal(size=3) * shift) @ R[a + k]
            t[a + k] += rng.normal(size=3) * shift
    id1 = np.asarray(id1, np.int32)
    id2 = np.asarray(id2, np.int32)
    return dict(chain_off=off, fixed=fixed, R=R, t=t, eR=eR, et=et, id1=id1, id2=id2,
                eR_list=eR[id1] if len(id1) else np.zeros((0, 3, 3)),
                et_list=et[id1] if len(id1) else np.zeros((0, 3)))


def _rel(Ra, ta, Rb, tb):
    """Rigid transform from pose a to pose b (getRigidTransFromTo): x_b = R x_a + t."""
    R = Rb @ Ra.T
    return R, tb - R @ ta


def scale_columns(scale_id):
    """Scale column of every edge the way computeNewCameraTranslations4 numbers them
    (slam/SL_GlobalPoseEstimation.cpp:383-403): the distinct scale ids of the constraint edges in
    increasing order; -1 for an edge without one.  Returns (columns, number of columns)."""
    sid = np.asarray(scale_id, np.int64)
    ids = np.unique(sid[sid >= 0])
    col = np.full(sid.shape, -1, np.int32)
    for c, s in enumerate(ids):
        col[sid == s] = c
    return col, len(ids)


def _trajectories(rng, n_frames, n_cams):
    R, t = np.zeros((n_frames, n_cams, 3, 3)), np.zeros((n_frames, n_cams, 3))
    for c in range(n_cams):
        R[0, c] = _rodrigues(rng.normal(size=3))
        t[0, c] = rng.normal(size=3)
        for k in range(1, n_frames):
            R[k, c] = _rodrigues(rng.normal(size=3) * 0.05) @ R[k - 1, c]
            t[k, c] = t[k - 1, c] + rng.normal(size=3) * 0.1
    return R, t


def _noisy(rng, R, t, noise):
    if noise <= 0:
        return R, t
    return _rodrigues(rng.normal(size=3) * noise) @ R, t + rng.normal(size=3) * noise


def make_merge_graph(n_key, n_cams, seed=0, groups=None, merge_frame=None, n_constraints=1, n_scale_ids=1,
                     noise=0.0):
    """Synthetic key-frame graph of a camera-group merge, shaped as MergeCameraGroup::
    _constructGraphForKeyFrms builds it (reference app/SL_MergeCameraGroup.cpp:907-1035): node
    k * n_cams + c = camera c at key frame k, the first key frame's nodes fixed; up to the merge frame,
    edges between the cameras of each group (a ring when a group has more than 2); per camera, edges
    between successive key frames; n_constraints merge edges between the groups near the merge frame,
    uncertain scale, scale id = edge index % n_scale_ids.  A constraint edge's t is the true translation
    divided by the true scale of its id, so with noise = 0 every edge is consistent with the input poses
    and the solution is the input with those scales.  noise > 0 perturbs every edge measurement.
    Returns dict(fixed, R, t, id1, id2, eR, et, scale_id, scale_col, n_scale, true_scale)."""
    rng = np.random.default_rng(seed)
    if groups is None:
        h = (n_cams + 1) // 2
        groups = [list(range(h)), list(range(h, n_cams))]
    if merge_frame is None:
        merge_frame = max(1, (2 * n_key) // 3)
    Rt, tt = _trajectories(rng, n_key, n_cams)
    node = lambda k, c: k * n_cams + c  # noqa: E731
    fixed = np.zeros(n_key * n_cams, np.uint8)
    fixed[:n_cams] = 1
    id1, id2, eR, et, sid = [], [], [], [], []

    def edge(a, b, R, t, s=-1):
        R, t = _noisy(rng, R, t, noise)
        id1.append(a)
        id2.append(b)
        eR.append(R)
        et.append(t)
        sid.append(s)

    for k in range(n_key):
        if k <= merge_frame:
            for g in groups:
                if len(g) < 2:
                    continue
                ring = list(zip(g[:-1], g[1:])) + ([(g[-1], g[0])] if len(g) > 2 else [])
                for c1, c2 in ring:
                    edge(node(k, c1), node(k, c2), *_rel(Rt[k, c1], tt[k, c1], Rt[k, c2], tt[k, c2]))
        if k > 0:
            for c in range(n_cams):
                edge(node(k - 1, c), node(k, c), *_rel(Rt[k - 1, c], tt[k - 1, c], Rt[k, c], tt[k, c]))
    true_scale = 0.5 + rng.uniform(size=n_scale_ids)
    for q in range(n_constraints):
        ga, gb = groups[0], groups[-1]
        c1, c2 = ga[q % len(ga)], gb[(q * 7 + 1) % len(gb)]
        f1 = merge_frame
        f2 = max(1, merge_frame - (q % 3))
        R, t = _rel(Rt[f1, c1], tt[f1, c1], Rt[f2, c2], tt[f2, c2])
        s = q % n_scale_ids
        edge(node(f1, c1), node(f2, c2), R, t / true_scale[s], s)
    sid = np.asarray(sid, np.int32)
    col, ns = scale_columns(sid)
    return dict(fixed=fixed, R=Rt.reshape(-1, 3, 3).copy(), t=tt.reshape(-1, 3).copy(),
                id1=np.asarray(id1, np.int32), id2=np.asarray(id2, np.int32), eR=np.asarray(eR).reshape(-1, 3, 3),
                et=np.asarray(et).reshape(-1, 3), scale_id=sid, scale_col=col, n_scale=ns,
                true_scale=true_scale[:ns])


def make_pose_graph(n_nodes, seed=0, components=1, fixed_every=0, loops=0, parallel=0, reverse=0,
                    fixed_pairs=0, n_scale=0, uncertain=0, noise=0.02):
    """A general pose graph: `components` disjoint chains over n_nodes (each with its first node fixed,
    and every fixed_every-th when > 0), plus per component `loops` random loop closures, `parallel`
    duplicated edges, `reverse` edges in the opposite direction, `fixed_pairs` edges between two fixed
    nodes, and `uncertain` extra edges with scale columns 0 .. n_scale-1 (each column used at least once).
    Edges are measured from the true poses with `noise`; the fixed nodes are then moved by ~noise.
    Returns dict(fixed, R, t, id1, id2, eR, et, scale_col, n_scale)."""
    rng = np.random.default_rng(seed)
    Rt, tt = _trajectories(rng, n_nodes, 1)
    Rt, tt = Rt[:, 0], tt[:, 0]
    bounds = np.linspace(0, n_nodes, components + 1).astype(int)
    fixed = np.zeros(n_nodes, np.uint8)
    id1, id2, eR, et, col = [], [], [], [], []

    def edge(a, b, c=-1):
        R, t = _rel(Rt[a], tt[a], Rt[b], tt[b])
        s = 1.0
        if c >= 0:
            s = 0.5 + 0.25 * c
            t = t / s
        R, t = _noisy(rng, R, t, noise)
        id1.append(a)
        id2.append(b)
        eR.append(R)
        et.append(t)
        col.append(c)

    n_unc = max(uncertain, n_scale)
    for q in range(components):
        a, b = int(bounds[q]), int(bounds[q + 1])
        if b <= a:
            continue
        fixed[a] = 1
        if fixed_every > 0:
            fixed[a:b:fixed_every] = 1
        for k in range(a, b - 1):
            edge(k, k + 1)
        n = b - a
        if n < 3:
            continue
        for _ in range(loops):
            i, j = sorted(rng.choice(n, 2, replace=False) + a)
            edge(int(i), int(j))
        for _ in range(parallel):
            k = int(rng.integers(a, b - 1))
            edge(k, k + 1)
        for _ in range(reverse):
            k = int(rng.integers(a, b - 1))
            edge(k + 1, k)
        fx = np.nonzero(fixed[a:b])[0] + a
        if len(fx) >= 2:
            for _ in range(fixed_pairs):
                i, j = rng.choice(fx, 2, replace=False)
                edge(int(i), int(j))
        if q == 0:
            for u in range(n_unc):
                i, j = rng.choice(n, 2, replace=False) + a
                if fixed[i] and fixed[j]:
                    j = a + 1 + (j - a) % (n - 1) if not fixed[a + 1] else i
                edge(int(i), int(j), u % n_scale if n_scale else -1)
    R, t = Rt.copy(), tt.copy()
    for k in np.nonzero(fixed)[0]:
        R[k] = _rodrigues(rng.normal(size=3) * noise) @ R[k]
        t[k] += rng.normal(size=3) * noise
    return dict(fixed=fixed, R=R, t=t, id1=np.asarray(id1, np.int32), id2=np.asarray(id2, np.int32),
                eR=np.asarray(eR).reshape(-1, 3, 3), et=np.asarray(et).reshape(-1, 3),
                scale_col=np.asarray(col, np.int32), n_scale=n_scale)
