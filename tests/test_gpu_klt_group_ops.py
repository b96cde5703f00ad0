"""Per-camera feed, advance and seeded first on a KLT camera group (cosl_klt_group_feed,
cosl_klt_group_advance_cams, cosl_klt_group_first_present): every camera of the group must behave bit
for bit like a single-camera tracker that receives the same calls, and cameras a call does not
address keep their state (needs a GPU)."""
import ctypes as C

import numpy as np
import pytest

from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

W, H, L, FW, FH = 640, 480, 6, 32, 32
COSL_E_INVALID, COSL_E_STATE = -1, -6


def _pts(rng, n):
    p = np.zeros((n, 3), np.float32)
    p[:, 0] = rng.uniform(0.05, 0.95, n)
    p[:, 1] = rng.uniform(0.05, 0.95, n)
    return p


def _rig(api, cfg, n_cams=3):
    return api.KltGroup(cfg, n_cams, W, H, L, FW, FH), [api.KltTracker(cfg, W, H, L, FW, FH)
                                                         for _ in range(n_cams)]


def _check(f, n, outs, what):
    for c, (fs, ns) in enumerate(outs):
        assert ns == n[c], (what, c, ns, n[c])
        assert fs.tobytes() == f[c].tobytes(), (what, c)


def _feed_both(grp, singles, lists):
    ids, fed = grp.feed(lists)
    for c, p in enumerate(lists):
        if p is None:
            assert ids[c] is None and fed[c] == 0
            continue
        i1, n1 = singles[c].feed(p)
        assert fed[c] == n1 and np.array_equal(ids[c], i1), c
    return fed


@pytest.mark.parametrize("compat_bit", [0, 4])  # 4 = COSL_KLT_COMPAT_FEED_STRIDE2
def test_rig_cadence_matches_single_trackers(api, compat_bit):
    """The CoSLAM rig cadence: seeded first (different list sizes, one camera empty), next, next,
    feed + advance on cameras {0, 2} (one list kills a live track), next, feed + advance on {0, 2}
    again (the reference's double swap of the pyramids), next.  Camera 1 never receives a feed or an
    advance of its own and must match a single tracker that did not either."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    cfg.compat |= compat_bit
    seqs = [seq(H, W, 70 + c, n=6) for c in range(3)]
    grp, singles = _rig(api, cfg)
    rng = np.random.default_rng(11)
    present = [_pts(rng, 40), np.zeros((0, 3), np.float32), _pts(rng, 90)]
    f, n = grp.first([s.frames[0] for s in seqs], present=present)
    outs = []
    for c in range(3):
        outs.append(singles[c].detect(seqs[c].frames[0], present[c]))
        singles[c].advance()
    _check(f, n, outs, "first_present")
    assert (f[0]["fed"] >= 0).sum() == 40 and (f[1]["fed"] >= 0).sum() == 0
    k = 1
    for step in ("next", "next", "feed", "next", "feed", "next"):
        if step == "next":
            f, n = grp.next([s.frames[k] for s in seqs])
            _check(f, n, [singles[c].next(seqs[c].frames[k]) for c in range(3)], f"next frame {k}")
            k += 1
            continue
        p0 = np.zeros((7, 3), np.float32)
        p0[:, 0] = np.linspace(0.2, 0.8, 7)
        p0[:, 1] = 0.5
        p0[0, :2] = f[0]["pos"][f[0]["status"] >= 0][0]  # forces one KLT point to be killed and replaced
        fed = _feed_both(grp, singles, [p0, None, _pts(rng, 12)])
        assert fed[0] > 0 and fed[2] > 0
        grp.advance([0, 2])
        singles[0].advance()
        singles[2].advance()


def test_first_present_without_points_equals_group_first(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 80 + c, n=2) for c in range(3)]
    a = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    b = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    fa, na = a.first([s.frames[0] for s in seqs])
    fb, nb = b.first([s.frames[0] for s in seqs], present=[np.zeros((0, 3), np.float32)] * 3)
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()
    fa, na = a.next([s.frames[1] for s in seqs])
    fb, nb = b.next([s.frames[1] for s in seqs])
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()


def test_advance_of_every_camera_equals_advance(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 90 + c, n=3) for c in range(3)]
    a = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    b = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    rng = np.random.default_rng(3)
    pts = [_pts(rng, 20), None, _pts(rng, 5)]
    for g in (a, b):
        g.first([s.frames[0] for s in seqs])
        g.next([s.frames[1] for s in seqs])
        g.feed(pts)
    a.advance()
    b.advance([0, 1, 2])
    fa, na = a.next([s.frames[2] for s in seqs])
    fb, nb = b.next([s.frames[2] for s in seqs])
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()


def test_pyramids_after_a_subset_advance(api):
    """After first + next the previous-frame buffer holds a tracked frame (level 0 not stored, the
    live tracker visits levels 5/3/1) and the current one the detected frame (every level stored).
    advance {0, 2} exchanges those two cameras' slices: each camera returns its own levels and
    refuses exactly the level 0 its single-camera twin refuses."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 100 + c, n=3) for c in range(3)]
    grp, singles = _rig(api, cfg)
    grp.first([s.frames[0] for s in seqs])
    grp.next([s.frames[1] for s in seqs])
    grp.advance([0, 2])
    for c in range(3):
        singles[c].first(seqs[c].frames[0])
        singles[c].next(seqs[c].frames[1])
        if c != 1:
            singles[c].advance()
    for c in range(3):
        for which in (0, 1):
            refused = which == (1 if c != 1 else 0)
            for level in range(L):
                if level == 0 and refused:
                    with pytest.raises(api.CoslError, match="not stored"):
                        grp.pyramid(c, which, 0)
                    with pytest.raises(api.CoslError, match="not stored"):
                        singles[c].pyramid(which, 0)
                    continue
                a, b = grp.pyramid(c, which, level), singles[c].pyramid(which, level)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (c, which, level)
    f, n = grp.next([s.frames[2] for s in seqs])
    _check(f, n, [singles[c].next(seqs[c].frames[2]) for c in range(3)], "next after the exchange")


def test_bad_arguments_and_frames_in_flight(api):
    from coslam_b200.api import _ptr
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 110 + c, n=3) for c in range(3)]
    grp = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    imgs, pitch = grp.host_ptrs([s.frames[0] for s in seqs])
    lib, F = api.LIB, FW * FH
    pts = np.zeros((4, 3), np.float32)
    ids = np.zeros(4, np.int32)
    fed = np.zeros(3, np.int32)
    cams = np.ones(3, np.uint8)

    def ptrs(*arrs):
        return (C.c_void_p * 3)(*[None if a is None else a.ctypes.data for a in arrs])

    def first_present(npres, pres):
        return lib.cosl_klt_group_first_present(grp.h, imgs, pitch, _ptr(np.asarray(npres, np.int32)), pres,
                                                grp._dest, _ptr(grp.counts))

    def feed(npts, p, i):
        return lib.cosl_klt_group_feed(grp.h, _ptr(np.asarray(npts, np.int32)), p, i, _ptr(fed))

    assert first_present([0, F + 1, 0], None) == COSL_E_INVALID
    assert first_present([0, -1, 0], None) == COSL_E_INVALID
    assert first_present([0, 4, 0], ptrs(pts, None, pts)) == COSL_E_INVALID
    assert lib.cosl_klt_group_first_present(grp.h, imgs, pitch, None, None, grp._dest, None) == COSL_E_INVALID
    full = np.zeros((F, 3), np.float32)
    assert first_present([0, F, 4], ptrs(None, full, pts)) == 0
    assert feed([4, -1, 0], None, None) == COSL_E_INVALID
    assert feed([4, -1, 0], ptrs(None, None, None), ptrs(ids, None, None)) == COSL_E_INVALID
    assert feed([4, -1, 0], ptrs(pts, None, None), ptrs(None, None, None)) == COSL_E_INVALID
    assert lib.cosl_klt_group_feed(grp.h, None, None, None, _ptr(fed)) == COSL_E_INVALID
    assert lib.cosl_klt_group_advance_cams(grp.h, None) == COSL_E_INVALID
    # cosl_klt_feed stays single-camera only
    assert lib.cosl_klt_feed(grp.h, 4, _ptr(pts), _ptr(ids), C.byref(C.c_int(0))) == COSL_E_STATE
    grp.submit([s.frames[1] for s in seqs])
    assert first_present([0, 0, 0], ptrs(None, None, None)) == COSL_E_STATE
    assert feed([4, -1, -1], ptrs(pts, None, None), ptrs(ids, None, None)) == COSL_E_STATE
    assert lib.cosl_klt_group_advance_cams(grp.h, _ptr(cams)) == COSL_E_STATE
    with pytest.raises(api.CoslError, match="not yet collected"):
        grp.advance([0])
    grp.collect()
    assert feed([4, -1, -1], ptrs(pts, None, None), ptrs(ids, None, None)) == 0
    assert lib.cosl_klt_group_advance_cams(grp.h, _ptr(cams)) == 0
