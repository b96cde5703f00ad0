"""Back-to-back KLT frames overlap: frame n+1's image copies, front pass and pyramid tail run on a side
stream next to frame n's detector, with the cornerness map, prelim list and counters double-buffered
(DESIGN.md §3.2 "Streams").  A group driven through calls that return without synchronising must
end in the same state, bit for bit, as a second group driven through the synchronous next(): feature
tables, counts, every pyramid level of both buffers, the cornerness map and the candidate count.
Each case runs once; the event graph in run_frame is the argument for correctness (needs a GPU)."""
import ctypes as C

import numpy as np
import pytest

from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

W, H, L = 640, 480, 6
MIXED = [(640, 480), (320, 240), (752, 480), (333, 251)]


def _pts(rng, n):
    p = np.zeros((n, 3), np.float32)
    p[:, 0] = rng.uniform(0.05, 0.95, n)
    p[:, 1] = rng.uniform(0.05, 0.95, n)
    return p


def _group(api, cfg, sizes, fw, fh):
    if len(set(sizes)) == 1:
        return api.KltGroup(cfg, len(sizes), sizes[0][0], sizes[0][1], L, fw, fh)
    return api.KltGroup(cfg, len(sizes), [w for w, _ in sizes], [h for _, h in sizes], L, fw, fh)


def _dev_frames(seqs, k):
    """Camera frames k on the device, each contiguous (rows of its own width), and synchronised:
    next_dev takes images that hold the frame when it is called."""
    import torch
    out = [torch.from_numpy(np.ascontiguousarray(s.frame(k))).cuda() for s in seqs]
    torch.cuda.synchronize()
    return out


def _next_dev(g, frames):
    g.next_dev([t.data_ptr() for t in frames], 0 if g.mixed else g.W)


def _cornerness(api, g, cam):
    w, h = g.sizes[cam]
    out = np.empty((h, w), np.float32)
    assert api.LIB.cosl_klt_debug_cornerness(g.h, cam, out.ctypes.data_as(C.c_void_p)) == 0
    return out


def _same_pyramids(api, a, b, what):
    for c in range(a.C):
        for which in (0, 1):
            for level in range(L):
                try:
                    pa = a.pyramid(c, which, level)
                except api.CoslError:
                    with pytest.raises(api.CoslError, match="not stored"):
                        b.pyramid(c, which, level)
                    continue
                pb = b.pyramid(c, which, level)
                assert pa.tobytes() == pb.tobytes(), (what, c, which, level)


def _same_state(api, a, b, what):
    """a: the group driven asynchronously (fetched here), b: the synchronous one after its last call."""
    fb, nb = b.feats.copy(), b.counts.copy()
    fa, na = a.fetch()
    assert np.array_equal(na, nb), (what, na, nb)
    assert fa.tobytes() == fb.tobytes(), what
    for c in range(a.C):
        assert api.LIB.cosl_klt_debug_num_candidates(a.h, c) == api.LIB.cosl_klt_debug_num_candidates(b.h, c), \
            (what, c)
        assert _cornerness(api, a, c).tobytes() == _cornerness(api, b, c).tobytes(), (what, c)
    _same_pyramids(api, a, b, what)


@pytest.mark.parametrize("case", [
    ("gain", [(W, H)] * 4, 32, 32),
    ("gain", [(W, H)] * 3, 25, 15),   # F = 375: F % 4 != 0
    ("2x2", [(W, H)] * 4, 32, 32),
    ("gain", MIXED, 20, 20),          # cameras of different sizes
], ids=["gain-F1024", "gain-F375", "2x2-F1024", "gain-mixed"])
def test_next_dev_run_equals_next(api, case):
    """20 next_dev calls in a row with no synchronise in between, against next()."""
    kind, sizes, fw, fh = case
    cfg = live_cfg(gain=kind == "gain", min_corner=1500.0)
    seqs = [seq(h, w, 300 + c, n=6) for c, (w, h) in enumerate(sizes)]
    a, b = _group(api, cfg, sizes, fw, fh), _group(api, cfg, sizes, fw, fh)
    dev = {k: _dev_frames(seqs, k) for k in range(1, 21)}
    host = [s.frame(0) for s in seqs]
    a.first(host)
    b.first(host)
    for k in range(1, 21):
        _next_dev(a, dev[k])
    for k in range(1, 21):
        b.next([s.frame(k) for s in seqs])
    _same_state(api, a, b, "after 20 next_dev")
    a.close()
    b.close()


def test_calls_between_asynchronous_frames(api):
    """feed + advance of a camera subset, first with present lists, a margin change (the front pass of a
    mixed group reads the per-camera table it rewrites) and debug reads placed between next_dev calls
    that are not synchronised."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(h, w, 400 + c, n=6) for c, (w, h) in enumerate(MIXED)]
    a, b = _group(api, cfg, MIXED, 32, 32), _group(api, cfg, MIXED, 32, 32)
    dev = {k: _dev_frames(seqs, k) for k in range(1, 16)}
    rng = np.random.default_rng(17)
    present = [_pts(rng, 40), np.zeros((0, 3), np.float32), _pts(rng, 90), _pts(rng, 5)]
    for g in (a, b):
        g.first([s.frame(0) for s in seqs], present=present)
    k = 1

    def step(n):
        nonlocal k
        for _ in range(n):
            _next_dev(a, dev[k])
            b.next([s.frame(k) for s in seqs])
            k += 1

    step(3)
    # a debug read of the previous-frame pyramid and the map between two asynchronous calls
    assert a.pyramid(1, 0, 3).tobytes() == b.pyramid(1, 0, 3).tobytes()
    assert _cornerness(api, a, 2).tobytes() == _cornerness(api, b, 2).tobytes()
    step(2)
    lists = [_pts(rng, 12), None, _pts(rng, 7), None]
    ia, na = a.feed(lists)
    ib, nb = b.feed(lists)
    assert np.array_equal(na, nb) and all(x is None or np.array_equal(x, y) for x, y in zip(ia, ib))
    a.advance([0, 2])
    b.advance([0, 2])
    step(2)
    for g in (a, b):
        g.advance([1, 3])
    step(1)
    _same_state(api, a, b, "after feed / advance")
    for g in (a, b):
        api._ck(api.LIB.cosl_klt_set_margin(g.h, 12.0))
    step(2)
    present = [_pts(rng, 0), _pts(rng, 60), _pts(rng, 25), _pts(rng, 3)]
    fa, cnt_a = a.first([s.frame(k) for s in seqs], present=present)
    fa, cnt_a = fa.copy(), cnt_a.copy()
    fb, cnt_b = b.first([s.frame(k) for s in seqs], present=present)
    assert np.array_equal(cnt_a, cnt_b) and fa.tobytes() == fb.tobytes()
    k += 1
    step(3)
    _same_state(api, a, b, "after margin change, first with present lists and next_dev")
    a.close()
    b.close()


def test_two_frames_in_flight_equal_next(api):
    """submit(n+1) before collect(n): both frames' pyramids and detectors overlap."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    sizes = [(W, H)] * 4
    seqs = [seq(H, W, 500 + c, n=6) for c in range(4)]
    a, b = _group(api, cfg, sizes, 32, 32), _group(api, cfg, sizes, 32, 32)
    frames = lambda k: [s.frame(k) for s in seqs]  # noqa: E731
    a.first(frames(0))
    b.first(frames(0))
    a.submit(frames(1))
    for k in range(2, 12):
        a.submit(frames(k))
        fa, na = a.collect()
        fb, nb = b.next(frames(k - 1))
        assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes(), k - 1
    fa, na = a.collect()
    fb, nb = b.next(frames(11))
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes(), 11
    _same_state(api, a, b, "after submit / collect")
    a.close()
    b.close()


def test_track_keeps_the_last_cornerness_map(api):
    """A tracked frame produces no cornerness map: the debug read still shows the last detector's, and
    every call matches a second tracker that reads the map after each call."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    s = seq(H, W, 600, n=6)
    a, b = api.KltTracker(cfg, W, H, L, 32, 32), api.KltTracker(cfg, W, H, L, 32, 32)
    a.detect(s.frame(0))
    a.advance()
    m0 = a.cornerness().copy()
    fa, _ = a.track(s.frame(1))
    assert a.cornerness().tobytes() == m0.tobytes()
    a.advance()
    a.redetect(s.frame(2))
    a.advance()
    m2 = a.cornerness().copy()
    a.track(s.frame(3))
    a.track(s.frame(4))
    assert a.cornerness().tobytes() == m2.tobytes()
    # the same calls on b, with nothing read in between, end in the same tables and pyramids
    b.detect(s.frame(0))
    b.advance()
    fb, _ = b.track(s.frame(1))
    assert fa.tobytes() == fb.tobytes()
    b.advance()
    b.redetect(s.frame(2))
    b.advance()
    b.track(s.frame(3))
    fb, _ = b.track(s.frame(4))
    assert a._out().tobytes() == fb.tobytes()
    assert b.cornerness().tobytes() == m2.tobytes()
    for which in (0, 1):
        for level in (1, 3, 5):
            assert a.pyramid(which, level).tobytes() == b.pyramid(which, level).tobytes(), (which, level)
    a.close()
    b.close()
