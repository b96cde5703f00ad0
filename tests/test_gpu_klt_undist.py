"""Undistorted positions and covariances of the KLT slots (cosl_klt_set_undistortion /
cosl_klt_group_download_undistorted): every path against the float64 restatement (undist_dense.py) applied to
the tables the group handed out and to its position covariances; arming changes nothing else and adds one
launch per frame; skipped cameras keep their entries; a setting applies from the next enqueued frame; every
refusal; and, end to end, a strong-barrel sequence whose undistorted tracks move by the known shift (needs a
GPU)."""
import ctypes as C

import numpy as np
import pytest
from scipy import ndimage

import undist_dense as U
from coslam_b200 import synth
from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

S, F1, T, N = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT
COSL_E_INVALID, COSL_E_STATE = -1, -6
POS_TOL, COV_TOL = 1e-8, 1e-6


def _lenses(sizes):
    """a different calibration per camera: the restatement's calibrations in turn, scaled to each camera"""
    names = list(U.CALIBS)
    Ks, kcs = [], []
    for c, (W, H) in enumerate(sizes):
        K0, kc, W0, H0 = U.CALIBS[names[c % len(names)]]
        Ks.append(np.diag([W / W0, H / H0, 1.0]) @ K0)
        kcs.append(kc)
    return np.array(Ks), np.array(kcs)


def _group(api, cfg, sizes, L, fw, fh):
    ws, hs = [w for w, _ in sizes], [h for _, h in sizes]
    if len(set(sizes)) == 1:
        return api.KltGroup(cfg, len(sizes), ws[0], hs[0], L, fw, fh)
    return api.KltGroup(cfg, len(sizes), ws, hs, L, fw, fh)


def _copy(tables):
    return [None if t is None else np.array(t).copy() for t in tables]


def check(sizes, Ks, kcs, tables, pos, ucov, cov, what):
    """pos / ucov (download_undistorted) against the restatement on the handed-out tables (None: camera
    skipped, not compared) and the position covariances cov (None: not armed).  Returns the slots compared."""
    assert (ucov is None) == (cov is None), what
    n = 0
    for c, t in enumerate(tables):
        if t is None:
            continue
        W, H = sizes[c]
        rp, rc = U.stage(Ks[c], kcs[c], W, H, t, None if cov is None else cov[c])
        assert np.array_equal(np.isnan(pos[c]), np.isnan(rp)), (what, c)
        live = ~np.isnan(rp[:, 0])
        assert np.array_equal(live, t["status"] >= 0), (what, c)
        if live.any():
            err = np.abs(pos[c][live] - rp[live]).max()
            assert err <= POS_TOL, (what, c, err)
        n += int(live.sum())
        if rc is None:
            continue
        assert np.array_equal(np.isnan(ucov[c]), np.isnan(rc)), (what, c)
        ok = ~np.isnan(rc[:, 0])
        if ok.any():
            # within COV_TOL of the larger variance (a slot whose window residual is exactly zero has Sigma = 0)
            scale = np.maximum(np.abs(rc[ok, 0]), np.abs(rc[ok, 2]))
            err = np.abs(ucov[c][ok].astype(np.float64) - rc[ok]).max(1)
            assert (err <= COV_TOL * scale).all(), (what, c, float((err / np.maximum(scale, 1e-300)).max()))
    return n


class Rig:
    """a group armed with a lens per camera and (optionally) position covariances"""

    def __init__(self, api, gain, sizes, fw, fh, n_frames=8, seed=0, with_cov=True):
        self.api, self.sizes = api, sizes
        self.cfg = live_cfg(gain=gain, min_corner=1500.0)
        self.g = _group(api, self.cfg, sizes, self.cfg.nLevels, fw, fh)
        self.Ks, self.kcs = _lenses(sizes)
        self.g.set_undistortion(self.Ks, self.kcs)
        self.with_cov = with_cov
        if with_cov:
            self.g.set_covariance(0.0)
        self.seqs = [seq(h, w, 900 + 11 * c + seed, n=n_frames) for c, (w, h) in enumerate(sizes)]
        self.last = [None] * len(sizes)

    def frames(self, k):
        return [s.frames[s.frame_index(k)] for s in self.seqs]

    def check(self, tables, what):
        pos, ucov = self.g.download_undistorted()
        cov = self.g.download_covariance() if self.with_cov else None
        n = check(self.sizes, self.Ks, self.kcs, tables, pos, ucov, cov, what)
        for c, t in enumerate(tables):
            if t is None and self.last[c] is not None:  # a skipped camera keeps its entries
                assert pos[c].tobytes() == self.last[c][0].tobytes(), (what, c)
                assert ucov is None or ucov[c].tobytes() == self.last[c][1].tobytes(), (what, c)
            elif t is not None:
                self.last[c] = (pos[c].copy(), None if ucov is None else ucov[c].copy())
        return n


def _all_paths(r, dev):
    """every group path of the rig r: returns the slots compared"""
    g, C_ = r.g, len(r.sizes)
    n = 0
    feats, _ = g.first(r.frames(0))
    n += r.check(_copy(feats), "first")
    pos, ucov = g.download_undistorted()
    if r.with_cov:
        assert np.isnan(ucov).all()  # nothing was tracked
    for k in (1, 2):
        feats, _ = g.next(r.frames(k))
        n += r.check(_copy(feats), f"next {k}")
    if dev:
        import torch
        d = [torch.from_numpy(f).cuda() for f in r.frames(3)]
        torch.cuda.synchronize()
        pitch = r.sizes[0][0] if len(set(r.sizes)) == 1 else 0
        g.next_dev([t.data_ptr() for t in d], pitch)
        n += r.check(_copy(g.fetch()[0]), "next_dev + fetch")
    ops = ([N, F1, S, T] * C_)[:C_]
    fr = r.frames(4)
    tables, _ = g.step(ops, [None if o == S else f for o, f in zip(ops, fr)])
    n += r.check(_copy(tables), "step N F S T")
    ops = ([T, N, N, S] * C_)[:C_]
    fr = r.frames(5)
    if dev:
        d = [torch.from_numpy(f).cuda() for f in fr]
        torch.cuda.synchronize()
        g.step_dev(ops, [0 if o == S else t.data_ptr() for o, t in zip(ops, d)], pitch)
        feats, _ = g.fetch()
        tables = [None if o == S else feats[c] for c, o in enumerate(ops)]
    else:
        tables, _ = g.step(ops, [None if o == S else f for o, f in zip(ops, fr)])
    n += r.check(_copy(tables), "step T N N S")
    # two frames in flight: each collect hands out its own frame's results
    g.submit(r.frames(6))
    ops = ([N, S, T, N] * C_)[:C_]
    g.submit_step(ops, [None if o == S else f for o, f in zip(ops, r.frames(7))])
    feats, _ = g.collect()
    n += r.check(_copy(feats), "submit / collect")
    tables, _ = g.collect()
    n += r.check(_copy(tables), "submit_step / collect")
    g.prefetch(r.frames(8))
    feats, _ = g.run_prefetched()
    n += r.check(_copy(feats), "prefetch + run_prefetched")
    g.prefetch(r.frames(9), ops=[N] * C_)
    g.submit_prefetched()
    tables, _ = g.collect()
    n += r.check(_copy(tables), "prefetch + submit_prefetched")
    return n


@pytest.mark.parametrize("gain", [True, False])
def test_c3_group_every_path(api, gain):
    """4 x 1280x720, 2 000 slots, live settings, a different lens per camera"""
    r = Rig(api, gain, [(1280, 720)] * 4, 50, 40)
    n = _all_paths(r, dev=True)
    assert n > 40000, n
    print(f"c3 gain={gain}: {n} slots compared")
    r.g.close()


@pytest.mark.parametrize("gain", [True, False])
def test_mixed_size_group_every_path(api, gain):
    r = Rig(api, gain, [(640, 480), (800, 600), (512, 384)], 24, 24, seed=3)
    n = _all_paths(r, dev=False)
    assert n > 3000, n
    r.g.close()


def test_without_position_covariances(api):
    """armed without set_covariance: positions on every path, cov None"""
    r = Rig(api, True, [(640, 480)] * 2, 24, 24, seed=5, with_cov=False)
    _all_paths(r, dev=False)
    h = r.g.h
    pos = np.zeros((2, r.g.F, 2))
    cov = np.zeros((2, r.g.F, 3), np.float32)
    pp = (C.c_void_p * 2)(pos[0].ctypes.data, pos[1].ctypes.data)
    cp = (C.c_void_p * 2)(cov[0].ctypes.data, cov[1].ctypes.data)
    assert api.LIB.cosl_klt_group_download_undistorted(h, pp, cp) == COSL_E_STATE
    assert api.LIB.cosl_klt_group_download_undistorted(h, pp, None) == 0
    assert api.LIB.cosl_klt_group_download_undistorted(h, None, None) == 0
    r.g.close()


def _single_download(api, t, with_cov):
    pos = np.empty((t.F, 2))
    cov = np.empty((t.F, 3), np.float32)
    pp = (C.c_void_p * 1)(pos.ctypes.data)
    cp = (C.c_void_p * 1)(cov.ctypes.data)
    assert api.LIB.cosl_klt_group_download_undistorted(t.h, pp, cp if with_cov else None) == 0
    if not with_cov:
        return pos, None, None
    sc = np.empty((t.F, 3), np.float32)
    assert api.LIB.cosl_klt_group_download_covariance(t.h, (C.c_void_p * 1)(sc.ctypes.data)) == 0
    return pos, cov, sc


@pytest.mark.parametrize("gain", [True, False])
def test_single_camera_paths(api, gain):
    """cosl_klt_detect / redetect / track on a one-camera tracker"""
    W, H = 640, 480
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    t = api.KltTracker(cfg, W, H, cfg.nLevels, 24, 24)
    K, kc = _lenses([(W, H)] * 2)
    K, kc = K[1:], kc[1:]  # the strong barrel
    assert api.LIB.cosl_klt_set_undistortion(t.h, np.ascontiguousarray(K).ctypes.data,
                                             np.ascontiguousarray(kc).ctypes.data) == 0
    assert api.LIB.cosl_klt_set_covariance(t.h, 0.0) == 0
    s = seq(H, W, 950, n=5)
    n = 0
    for k, call in enumerate(["detect", "advance", "redetect", "advance", "track", "advance", "redetect"]):
        if call == "advance":
            t.advance()
            continue
        feats, _ = getattr(t, call)(s.frames[k // 2 + (k > 0)])
        pos, ucov, cov = _single_download(api, t, True)
        n += check([(W, H)], K, kc, [feats], pos[None], ucov[None], cov[None], call)
    assert n > 1000, n
    t.close()


def _same_tables(a, b, what):
    (ta, na), (tb, nb) = a, b
    for c, (x, y) in enumerate(zip(ta, tb)):
        assert (x is None) == (y is None), (what, c)
        assert x is None or np.asarray(x).tobytes() == np.asarray(y).tobytes(), (what, c)
    assert [None if v is None else int(v) for v in na] == [None if v is None else int(v) for v in nb], what


@pytest.mark.parametrize("gain", [True, False])
def test_armed_changes_nothing_else(api, gain):
    """twins with position covariances, one of them also undistorting: bit-identical tables, counts and
    position covariances on next, steps, submitted frames and prefetched frames"""
    sizes = [(640, 480)] * 3
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    seqs = [seq(h, w, 970 + c, n=6) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[s.frame_index(k)] for s in seqs]  # noqa: E731
    a, b = _group(api, cfg, sizes, 5, 24, 24), _group(api, cfg, sizes, 5, 24, 24)
    for g in (a, b):
        g.set_covariance(0.0)
    b.set_undistortion(*_lenses(sizes))

    def same(fa, fb, what):
        ca = (_copy(fa[0]), list(fa[1]))
        cb = (_copy(fb[0]), list(fb[1]))
        _same_tables(ca, cb, what)
        assert a.download_covariance().tobytes() == b.download_covariance().tobytes(), what

    same(a.first(frames(0)), b.first(frames(0)), "first")
    same(a.next(frames(1)), b.next(frames(1)), "next")
    ops = [N, T, S]
    same(a.step(ops, [*frames(2)[:2], None]), b.step(ops, [*frames(2)[:2], None]), "step")
    ops = [T, N, F1]
    same(a.step(ops, frames(3)), b.step(ops, frames(3)), "step 2")
    for g in (a, b):
        g.submit(frames(4))
        g.submit_step([N, S, T], [frames(5)[0], None, frames(5)[2]])
    for what in ("collect 1", "collect 2"):
        same(a.collect(), b.collect(), what)
    for g in (a, b):
        g.prefetch(frames(6))
        g.advance()
    same(a.run_prefetched(), b.run_prefetched(), "run_prefetched")
    for which in (0, 1):
        assert a.pyramid(0, which, 1).tobytes() == b.pyramid(0, which, 1).tobytes()
    a.close()
    b.close()


def test_launch_count(api):
    """one launch more per armed frame, on tracked and detect frames; none once disarmed"""
    sizes = [(640, 480)] * 2
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(h, w, 990 + c, n=6) for c, (w, h) in enumerate(sizes)]
    frames = lambda k: [s.frames[s.frame_index(k)] for s in seqs]  # noqa: E731
    g = _group(api, cfg, sizes, 5, 16, 16)

    def count(fn, k):
        n0 = api.kernel_launch_count()
        fn(frames(k))
        return api.kernel_launch_count() - n0

    first0 = count(g.first, 0)
    plain = count(g.next, 1)
    g.set_undistortion(*_lenses(sizes))
    assert count(g.next, 2) == plain + 1
    g.set_covariance(0.0)
    assert count(g.next, 3) == plain + 2
    assert count(g.first, 4) == first0 + 1  # a detect frame's position covariances are a memset
    g.set_undistortion(None, None)
    assert count(g.next, 5) == plain + 1
    g.set_covariance(-1.0)
    assert count(g.next, 6) == plain
    g.close()


def test_setting_applies_to_the_next_enqueued_frame(api):
    """frames already submitted keep the setting they were enqueued with"""
    sizes = [(640, 480)] * 2
    r = Rig(api, True, sizes, 16, 16, seed=9)
    g = r.g
    g.set_undistortion(None, None)
    g.first(r.frames(0))
    g.submit(r.frames(1))                      # unarmed
    g.set_undistortion(r.Ks, r.kcs)
    g.submit(r.frames(2))                      # lens A
    feats, _ = g.collect()
    with pytest.raises(api.CoslError):
        g.download_undistorted()
    Kb = r.Ks.copy()
    Kb[:, 0, 0] *= 1.1
    g.set_undistortion(Kb, r.kcs[::-1].copy())  # lens B for the frame after
    g.submit(r.frames(3))
    feats, _ = g.collect()
    r.check(_copy(feats), "lens A")
    feats, _ = g.collect()
    r.Ks, r.kcs = Kb, r.kcs[::-1].copy()
    r.check(_copy(feats), "lens B")
    # a pending prefetch takes the setting when it is consumed
    g.prefetch(r.frames(4))
    g.set_undistortion(None, None)
    g.run_prefetched()
    with pytest.raises(api.CoslError):
        g.download_undistorted()
    g.close()


def test_refusals_name_their_camera(api):
    sizes = [(640, 480)] * 4
    cfg = live_cfg(gain=True, min_corner=1500.0)
    g = _group(api, cfg, sizes, 5, 16, 16)
    Ks, kcs = _lenses(sizes)
    with pytest.raises(api.CoslError, match="not armed"):
        g.download_undistorted()                     # nothing handed out
    cases = []
    K = Ks.copy(); K[2, 1, 2] = np.nan; cases.append((K, kcs, "camera 2"))            # noqa: E702
    k = kcs.copy(); k[1, 4] = np.inf; cases.append((Ks, k, "camera 1"))               # noqa: E702
    K = Ks.copy(); K[3, 0, 0] = 0.0; cases.append((K, kcs, "camera 3"))               # noqa: E702
    K = Ks.copy(); K[1, 1, 1] = -5.0; cases.append((K, kcs, "camera 1"))              # noqa: E702
    K = Ks.copy(); K[0, 1, 0] = 1e-3; cases.append((K, kcs, "camera 0"))              # noqa: E702
    K = Ks.copy(); K[2, 2, 2] = 2.0; cases.append((K, kcs, "camera 2"))               # noqa: E702
    K = Ks.copy(); K[3, 2, 0] = 0.1; cases.append((K, kcs, "camera 3"))               # noqa: E702
    for K, k, name in cases:
        with pytest.raises(api.CoslError, match=name):
            g.set_undistortion(K, k)
    assert api.LIB.cosl_klt_set_undistortion(g.h, np.ascontiguousarray(Ks).ctypes.data, None) == COSL_E_INVALID
    seqs = [seq(h, w, 1000 + c, n=3) for c, (w, h) in enumerate(sizes)]
    g.first([s.frames[0] for s in seqs])
    with pytest.raises(api.CoslError, match="not armed"):
        g.download_undistorted()                     # the frame handed out was not armed
    g.set_undistortion(Ks, kcs)
    with pytest.raises(api.CoslError):
        g.set_undistortion(cases[2][0], kcs)         # refused: the group stays armed with Ks
    feats, _ = g.next([s.frames[1] for s in seqs])
    pos, ucov = g.download_undistorted()
    assert ucov is None
    check(sizes, Ks, kcs, _copy(feats), pos, None, None, "after a refusal")
    g.close()


# End to end.  Frame k is a texture plane translated by k * SHIFT undistorted pixels and seen through the
# strong-barrel lens: its pixel u_d samples the plane at inverse(u_d) - k * SHIFT.  The undistorted
# displacement of every track is SHIFT; the distorted one is not, most of all near the image border.
SHIFT = np.array([2.3, -1.7])


def _barrel_sequence(W, H, n, seed=4242, pad=40, sigma=0.5):
    K, kc = _lenses([(W, H)] * 2)
    K, kc = K[1], kc[1]
    tex = synth.make_texture(H, W, seed, pad=pad)
    coef = ndimage.spline_filter(tex.astype(np.float64), order=3, mode="mirror")
    ud, vd = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    u, v, _, ok = U.undistort(K, kc, ud.ravel(), vd.ravel())
    assert ok.all()
    u, v = u.reshape(H, W), v.reshape(H, W)
    rng = np.random.default_rng(seed + 1)
    frames = []
    for k in range(n):
        x, y = u - k * SHIFT[0] + pad, v - k * SHIFT[1] + pad
        img = ndimage.map_coordinates(coef, [y - 0.5, x - 0.5], order=3, mode="mirror", prefilter=False)
        frames.append(np.clip(np.rint(img + rng.normal(0, sigma, img.shape)), 0, 255).astype(np.uint8))
    return K, kc, frames


def test_end_to_end_known_shift(api):
    W, H = 1280, 720
    K, kc, frames = _barrel_sequence(W, H, 4)
    cfg = live_cfg(gain=True, min_corner=1000.0)
    g = api.KltGroup(cfg, 1, W, H, cfg.nLevels, 50, 40)
    g.set_undistortion(K[None], kc[None])
    feats, _ = g.first([frames[0]])
    prev_pos, _ = g.download_undistorted()
    prev_raw = feats[0]["pos"].astype(np.float64) * [W, H]
    und_err, raw_err = [], []
    outer = []
    for k in range(1, 4):
        feats, _ = g.next([frames[k]])
        pos, _ = g.download_undistorted()
        live = feats[0]["status"] == 0
        raw = feats[0]["pos"].astype(np.float64) * [W, H]
        du = pos[0][live] - prev_pos[0][live]
        dd = raw[live] - prev_raw[live]
        und_err.append(np.hypot(*(du - SHIFT).T))
        raw_err.append(np.hypot(*(dd - SHIFT).T))
        rel = np.maximum(np.abs(raw[live, 0] - W / 2) / (W / 2), np.abs(raw[live, 1] - H / 2) / (H / 2))
        outer.append(rel > 2.0 / 3.0)
        prev_pos, prev_raw = pos, raw
    und_err, raw_err, outer = np.concatenate(und_err), np.concatenate(raw_err), np.concatenate(outer)
    assert outer.sum() > 500, int(outer.sum())
    mu, mr = float(np.median(und_err[outer])), float(np.median(raw_err[outer]))
    print(f"end to end: {int(outer.sum())} outer tracks, median |du - s| {mu:.4f} px, raw {mr:.4f} px, "
          f"all tracks {float(np.median(und_err)):.4f} px")
    # first H100 run: 0.095 px undistorted against 0.826 px raw over 3 268 outer tracks
    assert mu < 0.2 and mu < mr / 4, (mu, mr)
    g.close()
