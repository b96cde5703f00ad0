"""Position covariances of the tracked KLT slots (cosl_klt_set_covariance / cosl_klt_group_download_covariance):
every slot against a float64 numpy restatement built on the pyramids, start table and returned table of the
frame; NaN where no slot was tracked; armed groups return bit-identical tables on every path and launch one
kernel more per tracked frame; submitted frames hand out the covariances of the synchronous calls; and the
predicted variance has the scale of the empirical error of a known sub-pixel shift (needs a GPU)."""
import numpy as np
import pytest
from scipy import ndimage

import klt_numpy as K
from coslam_b200 import synth
from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

S, F1, T, N = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT


def cov_ref(P0, P1, x0, x1, beta, W, H, level, hw, gain, noise_var, lam=1.0, delta=200.0):
    """float64 restatement of klt_cov: P0, P1 the tracker's level `level` of camera W x H ((h, w, 3)), x0 the
    start and x1 the returned positions (n, 2, normalised), beta the returned gains.  Returns ((n, 3) (xx, xy,
    yy) in level-0 pixels^2, condition number of M)."""
    dx, dy = K._window(hw)
    npx = dx.shape[1]
    if gain:  # taps one texel of the level apart (klt_track_gain)
        sx, sy = 1.0 / (W >> level), 1.0 / (H >> level)
    else:     # taps 2^level / W apart (klt_track_2x2)
        sx, sy = 2.0 ** level / W, 2.0 ** level / H
    a0 = K._sample(np.asarray(P0, np.float64), x0[:, :1] + dx * sx, x0[:, 1:2] + dy * sy)
    a1 = K._sample(np.asarray(P1, np.float64), x1[:, :1] + dx * sx, x1[:, 1:2] + dy * sy)
    b = beta[:, None] if gain else 1.0
    I0 = a0[..., 0]
    e = b * I0 - a1[..., 0]
    jx = (b * a0[..., 1] + a1[..., 1]) * W / 2
    jy = (b * a0[..., 2] + a1[..., 2]) * H / 2
    if gain:  # klt_numpy.track_gain's M, the neighbour gains held fixed
        J = np.stack([jx, jy, -I0], 1)
        M = J @ J.transpose(0, 2, 1)
        M[:, 2, 2] = (I0 * I0 + lam * (a0[..., 1] ** 2 + a0[..., 2] ** 2)).sum(1) + 8 * delta * npx
    else:
        J = np.stack([jx, jy], 1)
        M = J @ J.transpose(0, 2, 1)
    k = M.shape[1]
    var = np.full(len(x0), float(noise_var)) if noise_var > 0 else (e * e).sum(1) / (npx - k)
    Sg = np.linalg.inv(M)[:, :2, :2] * var[:, None, None] * np.outer([W, H], [W, H])
    return np.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 1, 1]], 1), np.linalg.cond(M)


def _group(api, cfg, sizes, L, fw, fh):
    ws, hs = [w for w, _ in sizes], [h for _, h in sizes]
    if len(set(sizes)) == 1:
        return api.KltGroup(cfg, len(sizes), ws[0], hs[0], L, fw, fh)
    return api.KltGroup(cfg, len(sizes), ws, hs, L, fw, fh)


def _check_frame(g, cfg, start, feats, cov, noise_var, what, rel=1e-3):
    """Every camera's status-0 slots of `feats` against cov_ref on the pyramids the frame's tracker read (after
    the frame's advance: which 1 = its previous frame, which 0 = its current one); the rest NaN.  start[c]:
    the start table (n, 2) the tracker read.  Returns (slots compared, largest relative error)."""
    levels = K.tracker_levels(cfg.nLevels, cfg.levelSkip)
    lv = levels[-1]
    hw, gain = cfg.windowWidth // 2, bool(cfg.trackWithGain)
    n, worst = 0, 0.0
    for c, (W, H) in enumerate(g.sizes):
        live = feats[c]["status"] == 0
        assert np.isnan(cov[c][~live]).all(), (what, c)
        if not live.any():
            continue
        ref, cond = cov_ref(g.pyramid(c, 1, lv), g.pyramid(c, 0, lv), start[c][live].astype(np.float64),
                            feats[c]["pos"][live].astype(np.float64), feats[c]["gain"][live].astype(np.float64),
                            W, H, lv, hw, gain, noise_var)
        got = cov[c][live].astype(np.float64)
        well = cond < 1e4
        assert well.mean() > 0.8, (what, c, "too few well-conditioned slots to test")
        scale = np.maximum(np.abs(ref[:, 0]), np.abs(ref[:, 2]))[:, None]
        err = np.abs(got - ref)[well] / scale[well]
        assert np.isfinite(got[well]).all(), (what, c)
        worst = max(worst, float(err.max()))
        assert err.max() <= rel, (what, c, float(err.max()), int(np.argmax(err.max(1))))
        assert (ref[well, 0] > 0).all() and (ref[well, 2] > 0).all()
        n += int(well.sum())
    return n, worst


def _points(rng, n):
    """n fed points (x, y, 0) inside the frame"""
    return np.stack([rng.uniform(0.1, 0.9, n), rng.uniform(0.1, 0.9, n), np.zeros(n)], 1).astype(np.float32)


def _start(feats):
    """the start table the next frame's tracker reads: the positions of the slots with status >= 0"""
    s = feats["pos"].astype(np.float64).copy()
    s[feats["status"] < 0] = -1.0
    return s


# id: camera sizes, levels, levelSkip, windowWidth, gain, noise_var, feed
CASES = {
    "gain_hw3_live": ([(320, 240)] * 2, 6, 2, 6, True, 0.0, False),        # levels 5, 3, 1
    "2x2_hw3_live": ([(320, 240)] * 2, 6, 2, 6, False, 0.0, False),
    "gain_hw2_level0": ([(320, 240)] * 2, 3, 2, 5, True, 25.0, True),      # levels 2, 0; runtime width
    "2x2_hw4_level0": ([(320, 240)] * 2, 5, 2, 9, False, 0.0, True),       # levels 4, 2, 0
    "gain_mixed": ([(320, 240), (333, 251), (256, 200)], 5, 2, 6, True, 16.0, True),
    "2x2_mixed_hw2": ([(320, 240), (333, 251)], 4, 2, 5, False, 0.0, False),  # levels 3, 1
}


@pytest.mark.parametrize("case", list(CASES))
def test_against_float64(api, case):
    sizes, L, skip, ww, gain, noise_var, feed = CASES[case]
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    cfg.nLevels, cfg.levelSkip, cfg.windowWidth = L, skip, ww
    seqs = [seq(h, w, 500 + 7 * c + len(case), n=5, max_shift=2.5) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    g = _group(api, cfg, sizes, L, 16, 16)
    g.set_covariance(noise_var)
    feats, _ = g.first(frames(0))
    assert np.isnan(g.download_covariance()).all()
    rng = np.random.default_rng(len(case))
    total, fed_checked, worst = 0, 0, 0.0
    for k in range(1, 5):
        start = [_start(feats[c]) for c in range(g.C)]
        fed_slots = []
        if feed and k == 2:
            pts = [_points(rng, 30) for _ in range(g.C)]
            ids, nfed = g.feed(pts)
            g.advance()
            for c in range(g.C):
                for j, slot in enumerate(ids[c]):
                    if slot >= 0:
                        start[c][slot] = pts[c][j, :2]
                        fed_slots.append((c, slot))
            assert sum(nfed) > 0
        feats, _ = g.next(frames(k))
        feats = feats.copy()
        n, w = _check_frame(g, cfg, start, feats, g.download_covariance(), noise_var, f"{case} frame {k}")
        total += n
        worst = max(worst, w)
        fed_checked += sum(1 for c, s in fed_slots if feats[c]["status"][s] == 0)
    assert total > 200, total
    if feed:
        assert fed_checked > 5, fed_checked
    print(f"{case}: {total} slots, largest relative error {worst:.2e}")
    g.close()


def test_nan_pattern_and_skipped_cameras(api):
    """a step NEXT / FIRST / SKIP / TRACK: the FIRST camera is all NaN, the skipped one keeps the previous
    frame's entries, the tracked ones are NaN exactly where status != 0; a detect frame is all NaN"""
    sizes = [(320, 240)] * 4
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(h, w, 610 + c, n=4) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    g = _group(api, cfg, sizes, 5, 16, 16)
    with pytest.raises(api.CoslError):
        g.download_covariance()                       # nothing armed handed out
    with pytest.raises(api.CoslError):
        g.set_covariance(float("nan"))
    with pytest.raises(api.CoslError):
        g.set_covariance(float("inf"))
    g.first(frames(0))
    g.set_covariance(0.0)
    with pytest.raises(api.CoslError):
        g.download_covariance()                       # the frame handed out was not armed
    feats, _ = g.next(frames(1))
    before = g.download_covariance()
    for c in range(4):
        live = feats[c]["status"] == 0
        assert live.sum() > 50 and np.isfinite(before[c][live]).mean() > 0.99
        assert np.isnan(before[c][~live]).all()
    tables, _ = g.step([N, F1, S, T], [frames(2)[0], frames(2)[1], None, frames(2)[3]])
    cov = g.download_covariance()
    for c in (0, 3):
        live = tables[c]["status"] == 0
        assert live.sum() > 50 and np.isnan(cov[c][~live]).all() and np.isfinite(cov[c][live]).mean() > 0.99
    assert np.isnan(cov[1]).all()
    assert cov[2].tobytes() == before[2].tobytes()
    g.first(frames(3))
    assert np.isnan(g.download_covariance()).all()
    g.set_covariance(-1.0)
    g.next(frames(0))
    with pytest.raises(api.CoslError):
        g.download_covariance()
    g.close()


def _copy(res):
    tables, counts = res
    return [None if t is None else np.array(t).copy() for t in tables], [None if n is None else int(n) for n in counts]


def _same(want, got, what):
    (wt, wn), (gt, gn) = want, got
    assert wn == gn, (what, wn, gn)
    for c, (x, y) in enumerate(zip(wt, gt)):
        assert (x is None) == (y is None), (what, c)
        assert x is None or x.tobytes() == y.tobytes(), (what, c)


@pytest.mark.parametrize("gain", [True, False])
def test_armed_changes_nothing_else(api, gain):
    """an armed and an unarmed twin fed the same calls return bit-identical tables and counts on next, mixed
    steps, two submitted frames in flight, and prefetch + feed + advance + run_prefetched / submit_prefetched"""
    sizes = [(320, 240)] * 3
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    seqs = [seq(h, w, 640 + c, n=6) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[s.frame_index(k)] for s in seqs]  # noqa: E731
    a, b = _group(api, cfg, sizes, 5, 16, 16), _group(api, cfg, sizes, 5, 16, 16)
    b.set_covariance(0.0)
    rng = np.random.default_rng(3)
    _same(_copy(a.first(frames(0))), _copy(b.first(frames(0))), "first")
    _same(_copy(a.next(frames(1))), _copy(b.next(frames(1))), "next")
    ops = [N, T, S]
    _same(_copy(a.step(ops, [*frames(2)[:2], None])), _copy(b.step(ops, [*frames(2)[:2], None])), "step")
    ops = [T, N, F1]
    _same(_copy(a.step(ops, frames(3))), _copy(b.step(ops, frames(3))), "step 2")
    for g in (a, b):
        g.submit(frames(4))
        g.submit_step([N, S, T], [frames(5)[0], None, frames(5)[2]])
    for what in ("collect 1", "collect 2"):
        _same(_copy(a.collect()), _copy(b.collect()), what)
    pts = [_points(rng, 20) for _ in range(3)]
    for k, submit in ((6, False), (7, True)):
        for g in (a, b):
            g.prefetch(frames(k))
        fa, fb = a.feed(pts), b.feed(pts)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(fa[0], fb[0]))
        a.advance()
        b.advance()
        if submit:
            a.submit_prefetched()
            b.submit_prefetched()
            _same(_copy(a.collect()), _copy(b.collect()), "submit_prefetched")
        else:
            _same(_copy(a.run_prefetched()), _copy(b.run_prefetched()), "run_prefetched")
    for which in (0, 1):
        assert a.pyramid(0, which, 1).tobytes() == b.pyramid(0, which, 1).tobytes()
    a.close()
    b.close()


def test_launch_count(api):
    """an armed tracked frame launches one kernel more; disarming restores the unarmed count"""
    sizes = [(320, 240)] * 2
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(h, w, 660 + c, n=6) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[s.frame_index(k)] for s in seqs]  # noqa: E731
    g = _group(api, cfg, sizes, 5, 16, 16)
    g.first(frames(0))

    def count(k):
        n0 = api.kernel_launch_count()
        g.next(frames(k))
        return api.kernel_launch_count() - n0

    plain = count(1)
    g.set_covariance(0.0)
    armed = count(2)
    g.set_covariance(-1.0)
    assert (plain, armed, count(3)) == (plain, plain + 1, plain)
    g.close()


@pytest.mark.parametrize("gain", [True, False])
def test_submitted_frames_hand_out_their_own_covariances(api, gain):
    """two submitted frames in flight: after each collect the covariances are those the synchronous calls
    returned for the same frame, bit for bit"""
    sizes = [(320, 240), (256, 200)]
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    seqs = [seq(h, w, 680 + c, n=6) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[s.frame_index(k)] for s in seqs]  # noqa: E731
    a, b = _group(api, cfg, sizes, 5, 16, 16), _group(api, cfg, sizes, 5, 16, 16)
    for g in (a, b):
        g.set_covariance(0.0)
        g.first(frames(0))
    want = []
    for k in range(1, 5):
        a.next(frames(k))
        want.append(a.download_covariance())
    b.submit(frames(1))
    for k in range(2, 5):
        b.submit(frames(k))
        b.collect()
        assert b.download_covariance().tobytes() == want[k - 2].tobytes(), k - 1
    b.collect()
    assert b.download_covariance().tobytes() == want[3].tobytes()
    assert np.isfinite(want[3]).any()
    a.close()
    b.close()


# Known answer.  A seeded texture and the same texture shifted by D pixels with Gaussian noise of SIGMA grey
# levels added, tracked from a 40 x 30 grid of start points (present points of first(); no corners detected).
# On the float64 restatement (klt_numpy.track_gain / track_2x2 and cov_ref, live settings, 640 x 480) the
# empirical variance of (x1 - truth) over the slots is 2.7 - 3.0 times the mean predicted xx and yy for both
# trackers: the pyramid's smoothing correlates the residual of neighbouring window samples, which the
# independent-residual model does not see.  The bound admits half to twice that ratio, so a predicted
# variance 4x too large or too small fails.
D, SIGMA, RATIO = (0.37, -0.21), 8.0, 2.8


def _shifted_pair(h, w, seed, pad=32):
    tex = synth.make_texture(h, w, seed, pad=pad)
    coef = ndimage.spline_filter(tex.astype(np.float64), order=3, mode="mirror")
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)

    def render(dx, dy, sigma):
        v = ndimage.map_coordinates(coef, [ys + pad - dy, xs + pad - dx], order=3, mode="mirror", prefilter=False)
        if sigma > 0:
            v = v + np.random.default_rng(seed + 1).normal(0, sigma, v.shape)
        return np.clip(np.rint(v), 0, 255).astype(np.uint8)

    return render(0.0, 0.0, 0.0), render(D[0], D[1], SIGMA)


@pytest.mark.parametrize("gain", [True, False])
def test_known_answer_scale(api, gain):
    W, H, fw, fh = 640, 480, 40, 30
    f0, f1 = _shifted_pair(H, W, 4242)
    cfg = live_cfg(gain=gain, min_corner=1e30)
    g = api.KltGroup(cfg, 1, W, H, cfg.nLevels, fw, fh)
    g.set_covariance(0.0)
    gx, gy = np.meshgrid((np.arange(fw) + 0.5) / fw, (np.arange(fh) + 0.5) / fh)
    X0 = np.column_stack([0.08 + 0.84 * gx.ravel(), 0.08 + 0.84 * gy.ravel(), np.zeros(fw * fh)]).astype(np.float32)
    feats, n = g.first([f0], present=[X0])
    assert n[0] == fw * fh
    feats, _ = g.next([f1])
    cov = g.download_covariance()[0]
    live = feats[0]["status"] == 0
    assert live.mean() > 0.95
    err = (feats[0]["pos"][live].astype(np.float64) - X0[live, :2]) * [W, H] - D
    emp = (err ** 2).mean(0)
    pred = cov[live][:, [0, 2]].astype(np.float64).mean(0)
    ratio = emp / pred
    assert ((ratio > RATIO / 2) & (ratio < RATIO * 2)).all(), (emp, pred, ratio)
    g.close()
