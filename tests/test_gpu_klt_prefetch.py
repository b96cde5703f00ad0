"""Prefetched KLT frames (cosl_klt_group_prefetch / _run_prefetched / _submit_prefetched /
_discard_prefetch): a group that enqueues the image half of frame n+1 before the host's feeds and
advances, and the rest after them, is bit-identical to a twin group made from the same config and
driven by the synchronous calls in the same order -- tables, counts, fed slots, both pyramids at every
stored level and the cornerness maps -- and the prefetch keeps its state rules (needs a GPU)."""
import ctypes as C
import time

import numpy as np
import pytest

from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

COSL_E_INVALID, COSL_E_STATE = -1, -6
S, F, T, N = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT
# camera sizes, levels, slot grid
GEOMS = {
    "c3": ([(1280, 720)] * 4, 6, 50, 40),
    "small": ([(320, 240)] * 3, 4, 16, 16),
    "single": ([(320, 240)], 4, 16, 16),
    "mixed": ([(1280, 720), (640, 480), (640, 480), (320, 240)], 5, 24, 24),
}


class Rig:
    """One geometry's groups, frames and feed points: frame k of camera c cycles through n_frames."""

    def __init__(self, api, geom, seed, n_frames=6, gain=True):
        self.api, self.geom = api, geom
        self.sizes, self.L, self.fw, self.fh = GEOMS[geom]
        self.C = len(self.sizes)
        self.cfg = live_cfg(gain=gain, min_corner=1500.0)
        self.seqs = [seq(h, w, seed + c, n=n_frames) for c, (w, h) in enumerate(self.sizes)]
        self.rng = np.random.default_rng(seed)

    def group(self):
        ws, hs = [w for w, _ in self.sizes], [h for _, h in self.sizes]
        if len(set(self.sizes)) == 1:
            return self.api.KltGroup(self.cfg, self.C, ws[0], hs[0], self.L, self.fw, self.fh)
        return self.api.KltGroup(self.cfg, self.C, ws, hs, self.L, self.fw, self.fh)

    def frames(self, k):
        return [s.frames[s.frame_index(k)] for s in self.seqs]

    def pts(self, n):
        r = self.rng
        return np.stack([r.uniform(0.02, 0.98, n), r.uniform(0.02, 0.98, n), np.zeros(n)], 1).astype(np.float32)

    def feed_list(self, cams, n=100):
        return [self.pts(n) if c in cams else None for c in range(self.C)]


def _copy(res):
    tables, counts = res
    return [None if t is None else np.array(t).copy() for t in tables], [None if n is None else int(n) for n in counts]


def _check(want, got, what):
    (wt, wn), (gt, gn) = want, got
    assert wn == gn, (what, wn, gn)
    for c, (x, y) in enumerate(zip(wt, gt)):
        assert (x is None) == (y is None), (what, c)
        if x is not None:
            assert x.tobytes() == y.tobytes(), (what, c)


def _feed(g, pts):
    """group_feed, or cosl_klt_feed on a one-camera group: (trackIds, nFed) per camera"""
    if g.C == 1 and pts[0] is not None:
        p = np.ascontiguousarray(pts[0], np.float32)
        ids, n = np.full(len(p), -1, np.int32), C.c_int(0)
        g.api_ck(g.LIB.cosl_klt_feed(g.h, len(p), p.ctypes.data, ids.ctypes.data, C.byref(n)))
        return [ids], np.array([n.value], np.int32)
    return g.feed(pts)


def _same_feed(fa, fb, what):
    (ia, na), (ib, nb) = fa, fb
    assert list(na) == list(nb), (what, na, nb)
    for x, y in zip(ia, ib):
        assert (x is None) == (y is None) and (x is None or x.tobytes() == y.tobytes()), what


def _same_state(api, rig, a, b, what, corn_cams):
    """both pyramids at every level (and which levels are readable) of every camera, and the
    cornerness maps of corn_cams"""
    for c in range(rig.C):
        for which in (0, 1):
            for level in range(rig.L):
                got = []
                for g in (a, b):
                    try:
                        got.append(g.pyramid(c, which, level).tobytes())
                    except api.CoslError:
                        got.append(None)
                assert got[0] == got[1], (what, c, which, level)
    for c in corn_cams:
        assert a.cornerness(c).tobytes() == b.cornerness(c).tobytes(), (what, c)


def _with_lib(api, g):
    g.LIB, g.api_ck = api.LIB, api._ck
    return g


@pytest.mark.parametrize("geom", ["c3", "small"])
def test_coslam_cadence(api, geom):
    """first with 100 present points per camera, then next on every frame; after every 4th frame
    100 points are fed to cameras {0, 1} and those two advance -- between the prefetch of the next
    frame and its consume.  Twin group and one single-camera tracker per camera alongside."""
    rig = Rig(api, geom, 700 + len(geom))
    n_frames, every = 12, 4
    a, b = rig.group(), rig.group()
    singles = [api.KltTracker(rig.cfg, w, h, rig.L, rig.fw, rig.fh) for w, h in rig.sizes]
    present = [rig.pts(100) for _ in range(rig.C)]
    feeds = [rig.feed_list({0, 1}) for _ in range(n_frames // every)]
    want = _copy(a.first(rig.frames(0), present=present))
    _check(want, _copy(b.first(rig.frames(0), present=present)), "first")
    for c, s in enumerate(singles):
        f, n = s.detect(rig.frames(0)[c], present[c])
        s.advance()
        assert f.tobytes() == want[0][c].tobytes() and n == want[1][c], ("first single", c)
    b.prefetch(rig.frames(1))
    for k in range(1, n_frames + 1):
        want = _copy(a.next(rig.frames(k)))
        got = _copy(b.run_prefetched())
        _check(want, got, f"{geom} frame {k}")
        for c, s in enumerate(singles):
            f, n = s.next(rig.frames(k)[c])
            assert f.tobytes() == got[0][c].tobytes() and n == got[1][c], (f"{geom} frame {k} single", c)
        if k < n_frames:
            b.prefetch(rig.frames(k + 1))
        if k % every == 0:
            pts = feeds[k // every - 1]
            fa, fb = a.feed(pts), b.feed(pts)
            _same_feed(fa, fb, f"{geom} feed after {k}")
            for c in (0, 1):
                ids, n = singles[c].feed(pts[c])
                assert ids.tobytes() == fb[0][c].tobytes() and n == fb[1][c], (f"{geom} feed single", c)
                singles[c].advance()
            a.advance([0, 1])
            b.advance([0, 1])
    _same_state(api, rig, a, b, f"{geom} after the last frame", range(rig.C))
    for g in [a, b, *singles]:
        g.close()


@pytest.mark.parametrize("gain", [True, False])
def test_submitted_cadence(api, gain):
    """submit_prefetched(k), prefetch(k+1) while k is in flight, collect(k), feed + advance,
    submit_prefetched(k+1)"""
    rig = Rig(api, "small", 740, gain=gain)
    n_frames, every = 12, 4
    a, b = rig.group(), rig.group()
    present = [rig.pts(100) for _ in range(rig.C)]
    _check(_copy(a.first(rig.frames(0), present=present)), _copy(b.first(rig.frames(0), present=present)), "first")
    b.prefetch(rig.frames(1))
    b.submit_prefetched()
    for k in range(1, n_frames + 1):
        if k < n_frames:
            b.prefetch(rig.frames(k + 1))
        want = _copy(a.next(rig.frames(k)))
        _check(want, _copy(b.collect()), f"frame {k}")
        if k % every == 0:
            pts = rig.feed_list({0, 1})
            _same_feed(a.feed(pts), b.feed(pts), f"feed after {k}")
            a.advance([0, 1])
            b.advance([0, 1])
        if k < n_frames:
            b.submit_prefetched()
    _same_state(api, rig, a, b, "after the last collect", range(rig.C))
    a.close()
    b.close()


@pytest.mark.parametrize("geom", ["small", "single"])
def test_full_advance_between_prefetch_and_consume(api, geom):
    """cosl_klt_advance (the reference's double swap after next), with and without a feed before it,
    between the prefetch and the consume; the twin runs next + [feed +] advance + next"""
    rig = Rig(api, geom, 760)
    a, b = _with_lib(api, rig.group()), _with_lib(api, rig.group())
    _check(_copy(a.first(rig.frames(0))), _copy(b.first(rig.frames(0))), "first")
    b.prefetch(rig.frames(1))
    for k in range(1, 10):
        _check(_copy(a.next(rig.frames(k))), _copy(b.run_prefetched()), f"{geom} frame {k}")
        if k < 9:
            b.prefetch(rig.frames(k + 1))
        if k % 3 == 2:
            pts = rig.feed_list({0}, n=60)
            _same_feed(_feed(a, pts), _feed(b, pts), f"{geom} feed after {k}")
        if k % 3 != 0:
            a.advance()
            b.advance()
    _same_state(api, rig, a, b, f"{geom} after the last frame", range(rig.C))
    a.close()
    b.close()


SCHEDULES = {
    # 4 x TRACK + 1 x NEXT on every camera (frames of one kind)
    "cadence": [[F] * 4] + [[T] * 4 if k % 5 < 4 else [N] * 4 for k in range(10)],
    # the same cadence, each camera re-detecting on a step of its own
    "staggered": [[F] * 4] + [[N if (k + c) % 5 == 4 else T for c in range(4)] for k in range(10)],
    # one camera restarts mid-sequence
    "first_mid": [[F] * 4, [N] * 4, [T, N, T, N], [T, F, T, N], [N, T, N, T], [T, N, F, T], [N] * 4, [T] * 4],
    # synchronous steps with skipped cameras (which build into p1) before prefetched ones
    "after_skip": [[F] * 4, [N, N, N, S], [N] * 4, [T, S, N, T], [T, N, T, N], [S, F, S, S], [N] * 4, [T] * 4],
}
CASES = [(name, "c3") for name in SCHEDULES] + [("first_mid", "mixed"), ("after_skip", "mixed")]


def _corn_cams(sched):
    """the cameras that detect in the last entry with a detecting camera: the cornerness map the
    debug hook shows is theirs"""
    for ops in reversed(sched):
        cams = [c for c, o in enumerate(ops) if o in (F, N)]
        if cams:
            return cams
    return []


@pytest.mark.parametrize("name,geom", CASES)
def test_per_camera_ops(api, name, geom):
    """Every entry without a skipped camera is prefetched (the first one included) and consumed after
    a feed to cameras {0, 1} + their advance on every third entry; the twin runs group_step."""
    sched = SCHEDULES[name]
    rig = Rig(api, geom, 780 + 7 * len(name), n_frames=5)
    a, b = rig.group(), rig.group()
    imgs = lambda ops, k: [None if o == S else im for o, im in zip(ops, rig.frames(k))]  # noqa: E731
    for k, ops in enumerate(sched):
        if S in ops:
            want = _copy(a.step(ops, imgs(ops, k)))
            got = _copy(b.step(ops, imgs(ops, k)))
        else:
            b.prefetch(rig.frames(k), ops=ops)
            if k % 3 == 2:
                pts = rig.feed_list({0, 1}, n=50)
                _same_feed(a.feed(pts), b.feed(pts), f"{name} feed before {k}")
                a.advance([0, 1])
                b.advance([0, 1])
            want = _copy(a.step(ops, imgs(ops, k)))
            got = _copy(b.run_prefetched())
        _check(want, got, f"{name} {geom} step {k} {ops}")
    _same_state(api, rig, a, b, f"{name} {geom} after the last step", _corn_cams(sched))
    a.close()
    b.close()


@pytest.mark.parametrize("n_cams", [1, 3])
def test_state_rules(api, n_cams):
    rig = Rig(api, "single" if n_cams == 1 else "small", 820 + n_cams)
    a, b = _with_lib(api, rig.group()), _with_lib(api, rig.group())
    lib, Cn, W = api.LIB, rig.C, rig.sizes[0][0]
    _check(_copy(a.first(rig.frames(0))), _copy(b.first(rig.frames(0))), "first")
    fr = rig.frames(1)
    imgs = (C.c_void_p * Cn)(*[im.ctypes.data for im in fr])
    dest = (C.c_void_p * Cn)(*[b.feats[c].ctypes.data for c in range(Cn)])
    n = np.zeros(Cn, np.int32)
    keep = []  # the arrays whose addresses the calls below are given

    def arr(v, dtype):
        keep.append(np.array(v, dtype))
        return keep[-1].ctypes.data

    def ops(*v):
        return arr(v[:Cn], np.uint8)

    def prefetch(o, ptrs=imgs, pitch=W):
        return lib.cosl_klt_group_prefetch(b.h, o, ptrs, pitch)

    # nothing pending
    assert lib.cosl_klt_group_run_prefetched(b.h, dest, n.ctypes.data) == COSL_E_STATE
    assert lib.cosl_klt_group_submit_prefetched(b.h) == COSL_E_STATE
    assert lib.cosl_klt_group_discard_prefetch(b.h) == COSL_E_STATE
    # bad arguments: nothing enqueued
    assert prefetch(ops(S, N, N)) == COSL_E_INVALID
    assert prefetch(ops(N, S, N) if Cn > 1 else ops(S)) == COSL_E_INVALID
    assert prefetch(ops(4, N, N)) == COSL_E_INVALID
    assert prefetch(None, None) == COSL_E_INVALID
    assert prefetch(None, imgs, W - 1) == COSL_E_INVALID
    missing = (C.c_void_p * Cn)(*([None] + [im.ctypes.data for im in fr[1:]]))
    assert prefetch(None, missing) == COSL_E_INVALID
    assert lib.cosl_klt_group_prefetch(None, None, imgs, W) == COSL_E_INVALID

    # pending: every call that processes a frame of its own, set_margin and a second prefetch refuse
    b.prefetch(fr)
    assert prefetch(None) == COSL_E_STATE
    refused = {
        "next": lambda: lib.cosl_klt_group_next(b.h, imgs, W, dest, n.ctypes.data),
        "next_dev": lambda: lib.cosl_klt_group_next_dev(b.h, imgs, W),
        "first": lambda: lib.cosl_klt_group_first(b.h, imgs, W, dest, n.ctypes.data),
        "first_present": lambda: lib.cosl_klt_group_first_present(b.h, imgs, W, arr([0] * Cn, np.int32), None,
                                                                  dest, n.ctypes.data),
        "step": lambda: lib.cosl_klt_group_step(b.h, ops(N, N, N), imgs, W, dest, n.ctypes.data),
        "step_dev": lambda: lib.cosl_klt_group_step_dev(b.h, ops(N, N, N), imgs, W),
        "submit": lambda: lib.cosl_klt_group_submit(b.h, imgs, W),
        "submit_step": lambda: lib.cosl_klt_group_submit_step(b.h, ops(N, N, N), imgs, W),
        "set_margin": lambda: lib.cosl_klt_set_margin(b.h, 4.0),
    }
    if Cn == 1:
        f1, n1 = C.c_void_p(b.feats[0].ctypes.data), C.c_int(0)
        refused["detect"] = lambda: lib.cosl_klt_detect(b.h, imgs[0], W, 0, None, f1, C.byref(n1))
        refused["redetect"] = lambda: lib.cosl_klt_redetect(b.h, imgs[0], W, f1, C.byref(n1))
        refused["track"] = lambda: lib.cosl_klt_track(b.h, imgs[0], W, f1, C.byref(n1))
    for name, call in refused.items():
        assert call() == COSL_E_STATE, name
    # allowed: the tracker thresholds (same values on the twin) and sync
    for g in (a, b):
        api._ck(lib.cosl_klt_set_conv(g.h, rig.cfg.convergenceThreshold * 0.5))
        api._ck(lib.cosl_klt_set_ssd(g.h, rig.cfg.SSD_Threshold * 0.5))
    b.sync()
    _check(_copy(a.next(fr)), _copy(b.run_prefetched()), "consumed after the refusals")

    # with a submitted frame in flight and a prefetch pending, feeds and advances still refuse; the
    # prefetched frame runs behind the submitted one
    b.prefetch(rig.frames(2))
    b.submit_prefetched()
    b.prefetch(rig.frames(3))
    mask = np.ones(Cn, np.uint8)
    assert lib.cosl_klt_group_advance_cams(b.h, mask.ctypes.data) == COSL_E_STATE
    npts = np.full(Cn, -1, np.int32)
    assert lib.cosl_klt_group_feed(b.h, npts.ctypes.data, None, None, n.ctypes.data) == COSL_E_STATE
    assert lib.cosl_klt_group_run_prefetched(b.h, dest, n.ctypes.data) == 0
    b._prefetched = None
    got3 = _copy((b.feats, n))
    _check(_copy(a.next(rig.frames(2))), _copy(b.collect()), "submitted frame 2")
    _check(_copy(a.next(rig.frames(3))), got3, "frame 3 consumed with frame 2 in flight")

    # a step prefetch with a frame in flight: run_prefetched refuses as group_step does, and a third
    # frame in flight is refused with the prefetch left pending
    b.prefetch(rig.frames(4), ops=[N] * Cn)
    b.submit_prefetched()
    b.prefetch(rig.frames(5), ops=[T] * Cn)
    assert lib.cosl_klt_group_run_prefetched(b.h, dest, n.ctypes.data) == COSL_E_STATE
    b.submit_prefetched()
    b.prefetch(rig.frames(6), ops=[N] * Cn)
    assert lib.cosl_klt_group_submit_prefetched(b.h) == COSL_E_STATE
    _check(_copy(a.step([N] * Cn, rig.frames(4))), _copy(b.collect()), "step 4")
    _check(_copy(a.step([T] * Cn, rig.frames(5))), _copy(b.collect()), "step 5")
    _check(_copy(a.step([N] * Cn, rig.frames(6))), _copy(b.run_prefetched()), "step 6")

    # discard: the group is as if nothing had been prefetched, before and after the next frame
    b.prefetch(rig.frames(7))
    pts = rig.feed_list({0}, n=40)
    _same_feed(_feed(a, pts), _feed(b, pts), "feed with a prefetch pending")
    a.advance([0])
    b.advance([0])
    b.discard_prefetch()
    _same_state(api, rig, a, b, "after discard", range(Cn))
    _check(_copy(a.next(rig.frames(8))), _copy(b.next(rig.frames(8))), "next after discard")
    _same_state(api, rig, a, b, "next after discard", range(Cn))
    # a camera restarting with FIRST after a discard
    b.prefetch(rig.frames(9), ops=[T] * Cn)
    b.discard_prefetch()
    _check(_copy(a.first(rig.frames(9))), _copy(b.first(rig.frames(9))), "first after discard")
    b.prefetch(rig.frames(10))
    _check(_copy(a.next(rig.frames(10))), _copy(b.run_prefetched()), "prefetch after discard")
    _same_state(api, rig, a, b, "the end", range(Cn))
    a.close()

    # destroy with a prefetch pending, also with a frame in flight
    b.prefetch(rig.frames(11))
    b.close()
    c = rig.group()
    c.first(rig.frames(0))
    c.prefetch(rig.frames(1))
    c.submit_prefetched()
    c.prefetch(rig.frames(2))
    c.close()
    d = rig.group()
    d.first(rig.frames(0))
    d.close()


def test_fetch_and_debug_reads_see_the_last_consumed_frame(api):
    """group_fetch, the pyramids and the cornerness maps show the last consumed frame while a
    prefetch is pending and after it is discarded, for every kind of prefetch; a TRACK-only frame
    keeps the last frame's counter set, whose counts must survive until the frame is consumed"""
    rig = Rig(api, "small", 900)
    a, b = rig.group(), rig.group()
    _check(_copy(a.first(rig.frames(0))), _copy(b.first(rig.frames(0))), "first")
    _check(_copy(a.step([N] * 3, rig.frames(1))), _copy(b.step([N] * 3, rig.frames(1))), "step")
    want = _copy(a.fetch())
    assert all(n > 0 for n in want[1]), want[1]
    for ops in ([T] * 3, None, [T, N, F]):
        b.prefetch(rig.frames(2), ops=ops)
        b.sync()
        _check(want, _copy(b.fetch()), f"fetch with {ops} pending")
        _same_state(api, rig, a, b, f"{ops} pending", range(3))
        b.discard_prefetch()
        _check(want, _copy(b.fetch()), f"fetch after {ops} discarded")
        _same_state(api, rig, a, b, f"{ops} discarded", range(3))
    b.prefetch(rig.frames(2), ops=[T] * 3)
    _check(want, _copy(b.fetch()), "fetch with TRACK pending")
    _check(_copy(a.step([T] * 3, rig.frames(2))), _copy(b.run_prefetched()), "TRACK consumed")
    _check(_copy(a.fetch()), _copy(b.fetch()), "fetch after the TRACK frame")
    _check(_copy(a.next(rig.frames(3))), _copy(b.next(rig.frames(3))), "next after")
    a.close()
    b.close()


def _count(api, fn):
    n0 = api.kernel_launch_count()
    fn()
    return api.kernel_launch_count() - n0


@pytest.mark.parametrize("gain", [True, False])
def test_launches(api, gain):
    """prefetch + consume launch what the synchronous frame of the same ops launches"""
    rig = Rig(api, "small", 860, gain=gain)
    a, b = rig.group(), rig.group()
    a.first(rig.frames(0))
    b.first(rig.frames(0))
    kinds = [None, [F] * 3, [T] * 3, [N] * 3, [T, N, F], [N, T, T], None]
    for k, ops in enumerate(kinds, start=1):
        fr = rig.frames(k)
        n_sync = _count(api, lambda: a.next(fr) if ops is None else a.step(ops, fr))
        n_pre = _count(api, lambda: b.prefetch(fr, ops=ops))
        n_run = _count(api, lambda: b.run_prefetched())
        assert n_pre + n_run == n_sync, (ops, n_pre, n_run, n_sync)
        assert n_pre > 0 and n_run > 0, ops
    # submitted: prefetch + submit_prefetched launch what submit launches
    n_sub = _count(api, lambda: a.submit(rig.frames(9)))
    a.collect()
    n_pre = _count(api, lambda: b.prefetch(rig.frames(9)))
    n_run = _count(api, lambda: b.submit_prefetched())
    b.collect()
    assert n_pre + n_run == n_sub, (n_pre, n_run, n_sub)
    a.close()
    b.close()


def test_prefetch_does_not_wait_for_the_device(api):
    import torch

    rig = Rig(api, "small", 880)
    a, b = rig.group(), rig.group()
    _check(_copy(a.first(rig.frames(0))), _copy(b.first(rig.frames(0))), "first")
    pinned = [torch.from_numpy(f).pin_memory().numpy() for f in rig.frames(1)]
    with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
        t0 = time.perf_counter()
        torch.cuda._sleep(int(1.5e9))  # about a second at H100 clocks
    b.prefetch(pinned)
    dt = time.perf_counter() - t0
    assert dt < 0.25, dt
    _check(_copy(a.next(rig.frames(1))), _copy(b.run_prefetched()), "frame 1")
    a.close()
    b.close()
    torch.cuda.synchronize()
