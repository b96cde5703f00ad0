"""Frame-pipelined per-camera steps (cosl_klt_group_submit_step / _collect): a group driven with step
n+1 submitted before step n is collected is bit-identical to a group driven by the synchronous
cosl_klt_group_step on the same frames and ops -- tables, counts, the frames after, pyramids and
cornerness -- and the pipelined calls keep the state rules of submit and step (needs a GPU)."""
import ctypes as C

import numpy as np
import pytest

from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

W, H, L, FW, FH = 640, 480, 6, 32, 32
MIXED_SIZES = [(1280, 720), (1280, 720), (640, 480), (640, 480)]
COSL_E_INVALID, COSL_E_STATE = -1, -6
S, F, T, N = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT
PLAIN = "submit"  # a schedule entry run by group_next / submit instead of a step

SCHEDULES = {
    # 4 x TRACK + 1 x NEXT on every camera (uniform steps)
    "cadence": [[F] * 4] + [[T] * 4 if k % 5 < 4 else [N] * 4 for k in range(10)],
    # the same cadence, each camera re-detecting on a step of its own
    "cadence_staggered": [[F] * 4] + [[N if (k + c) % 5 == 4 else T for c in range(4)] for k in range(10)],
    # camera 3 skipped on every other step
    "skip3": [[F] * 4] + [[N, N, N, S] if k % 2 == 0 else [N] * 4 for k in range(10)],
    # one camera restarts mid-sequence
    "first_mid": [[F] * 4, [N] * 4, [T, N, T, N], [T, F, T, N], [N, T, N, T], [T, N, F, T], [N] * 4, [T] * 4],
    # all-SKIP steps, alone and back to back
    "all_skip": [[F] * 4, [N, T, N, T], [S] * 4, [T, N, S, N], [S] * 4, [S] * 4, [N] * 4, [S] * 4, [T, T, N, S]],
    # submit and submit_step interleaved
    "interleaved": [[F] * 4, PLAIN, [T, T, N, S], PLAIN, [S, N, T, T], [T] * 4, PLAIN, [N, S, N, S], PLAIN],
}
# (schedule, mixed sizes): the mixed-size group runs a schedule with every op and SKIP
CASES = [(name, False) for name in SCHEDULES] + [("first_mid", True), ("all_skip", True)]


def _group(api, cfg, mixed):
    if mixed:
        return api.KltGroup(cfg, 4, [w for w, _ in MIXED_SIZES], [h for _, h in MIXED_SIZES], L, FW, FH)
    return api.KltGroup(cfg, 4, W, H, L, FW, FH)


def _seqs(mixed, seed, n):
    sizes = MIXED_SIZES if mixed else [(W, H)] * 4
    return [seq(h, w, seed + c, n=n) for c, (w, h) in enumerate(sizes)]


def _imgs(ops, frames):
    return [None if o == S else im for o, im in zip(ops, frames)]


def _sync(a, entry, frames):
    """the synchronous call of a schedule entry: per-camera (table copy or None, count or None)"""
    if entry is PLAIN:
        f, n = a.next(frames)
        return [f[c].copy() for c in range(a.C)], [int(v) for v in n]
    tables, counts = a.step(entry, _imgs(entry, frames))
    return [None if t is None else t.copy() for t in tables], counts


def _submit(b, entry, frames):
    if entry is PLAIN:
        b.submit(frames)
    else:
        b.submit_step(entry, _imgs(entry, frames))


SENTINEL = 0x5A


def _collect(b, entry):
    """collect, after filling the result buffers with a sentinel: a skipped camera's must survive"""
    b.feats.view(np.uint8)[:] = SENTINEL
    b.counts[:] = -7
    tables, counts = b.collect()
    skipped = [] if entry is PLAIN else [c for c, o in enumerate(entry) if o == S]
    for c in skipped:
        assert tables[c] is None and counts[c] is None
        assert (b.feats[c].view(np.uint8) == SENTINEL).all() and b.counts[c] == -7, c
    return [None if t is None else t.copy() for t in tables], [None if n is None else int(n) for n in counts]


def _detected_last(sched):
    """the cameras that detect in the last entry with a detecting camera: the cornerness map the
    debug hook shows is theirs"""
    for entry in reversed(sched):
        cams = list(range(4)) if entry is PLAIN else [c for c, o in enumerate(entry) if o in (F, N)]
        if cams:
            return cams
    return []


def _same_state(api, a, b, what, corn_cams):
    """pyramids (both buffers, every level, which levels are readable) of every camera, and the
    cornerness map of corn_cams"""
    for c in range(a.C):
        for which in (0, 1):
            for level in range(L):
                got = []
                for g in (a, b):
                    try:
                        got.append(g.pyramid(c, which, level).tobytes())
                    except api.CoslError:
                        got.append(None)
                assert got[0] == got[1], (what, c, which, level)
    for c in corn_cams:
        assert a.cornerness(c).tobytes() == b.cornerness(c).tobytes(), (what, c)


def _check(want, got, what):
    wt, wn = want
    gt, gn = got
    assert wn == gn, (what, wn, gn)
    for c, (x, y) in enumerate(zip(wt, gt)):
        assert (x is None) == (y is None), (what, c)
        if x is not None:
            assert x.tobytes() == y.tobytes(), (what, c)


@pytest.mark.parametrize("gain", [True, False])
@pytest.mark.parametrize("name,mixed", CASES)
def test_pipelined_steps_equal_synchronous_steps(api, name, mixed, gain):
    """Every step submitted before the previous one is collected (two in flight); then two more
    synchronous steps on both groups, and their pyramids and cornerness maps."""
    sched = SCHEDULES[name]
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    seqs = _seqs(mixed, 500 + 10 * mixed, len(sched) + 2)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    a, b = _group(api, cfg, mixed), _group(api, cfg, mixed)
    want = [_sync(a, entry, frames(k)) for k, entry in enumerate(sched)]
    pending = []
    for k, entry in enumerate(sched):
        _submit(b, entry, frames(k))
        pending.append(k)
        if len(pending) == 2:
            j = pending.pop(0)
            _check(want[j], _collect(b, sched[j]), f"{name} step {j}")
    j = pending.pop(0)
    _check(want[j], _collect(b, sched[j]), f"{name} step {j}")
    _same_state(api, a, b, f"{name} after the last collect", _detected_last(sched))
    later = [[T, N, T, N], [N] * 4]
    for k, ops in enumerate(later, start=len(sched)):
        _check(_sync(a, ops, frames(k)), _sync(b, ops, frames(k)), f"{name} later step {k}")
    _same_state(api, a, b, f"{name} after the later steps", range(4))
    a.close()
    b.close()


def test_pipelined_step_launches_what_the_step_launches(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = _seqs(False, 560, 6)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    a, b = _group(api, cfg, False), _group(api, cfg, False)

    def count(fn):
        n0 = api.kernel_launch_count()
        fn()
        return api.kernel_launch_count() - n0

    for k, ops in enumerate([[F] * 4, [T, N, S, T], [S] * 4, [T] * 4, [N, N, N, S], [N] * 4]):
        n_sync = count(lambda: a.step(ops, _imgs(ops, frames(k))))
        n_pipe = count(lambda: b.submit_step(ops, _imgs(ops, frames(k))))
        b.collect()
        assert n_sync == n_pipe, (ops, n_sync, n_pipe)
        assert (n_pipe == 0) == (ops == [S] * 4), ops


def test_state_rules_and_bad_arguments(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = _seqs(False, 580, 4)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    g = _group(api, cfg, False)
    lib = api.LIB
    imgs = (C.c_void_p * 4)(*[im.ctypes.data for im in frames(1)])
    one_missing = (C.c_void_p * 4)(imgs[0], imgs[1], None, imgs[3])
    dest = (C.c_void_p * 4)(*[g.feats[c].ctypes.data for c in range(4)])
    n = np.zeros(4, np.int32)
    ops_ok = np.array([T, N, S, T], np.uint8)

    def submit_step(ops, ptrs=imgs):
        ops = None if ops is None else np.asarray(ops, np.uint8)
        return lib.cosl_klt_group_submit_step(g.h, None if ops is None else ops.ctypes.data, ptrs, W)

    assert lib.cosl_klt_group_collect(g.h, dest, n.ctypes.data) == COSL_E_STATE
    g.step([F] * 4, frames(0))
    # bad ops, a missing image of an addressed camera, bad pointers and pitch: nothing enqueued
    assert submit_step([T, 4, N, N]) == COSL_E_INVALID
    assert submit_step([255, N, N, N]) == COSL_E_INVALID
    assert submit_step([N, N, T, N], one_missing) == COSL_E_INVALID
    assert submit_step(None) == COSL_E_INVALID
    assert submit_step(ops_ok, None) == COSL_E_INVALID
    assert lib.cosl_klt_group_submit_step(g.h, ops_ok.ctypes.data, imgs, W - 1) == COSL_E_INVALID
    assert lib.cosl_klt_group_submit_step(None, ops_ok.ctypes.data, imgs, W) == COSL_E_INVALID
    assert lib.cosl_klt_group_collect(g.h, dest, n.ctypes.data) == COSL_E_STATE
    # a skipped camera's image may be NULL
    g.submit_step([N, N, S, N], [*frames(1)[:2], None, frames(1)[3]])
    g.submit_step([S] * 4, [None] * 4)
    # a third frame in flight, by either call
    assert submit_step(ops_ok) == COSL_E_STATE
    assert lib.cosl_klt_group_submit(g.h, imgs, W) == COSL_E_STATE
    # the calls that refuse to run while frames are in flight
    ops_all = np.array([N] * 4, np.uint8)
    assert lib.cosl_klt_group_step(g.h, ops_all.ctypes.data, imgs, W, dest, n.ctypes.data) == COSL_E_STATE
    assert lib.cosl_klt_group_step_dev(g.h, ops_all.ctypes.data, imgs, W) == COSL_E_STATE
    npts = np.full(4, -1, np.int32)
    assert lib.cosl_klt_group_feed(g.h, npts.ctypes.data, None, None, n.ctypes.data) == COSL_E_STATE
    mask = np.ones(4, np.uint8)
    assert lib.cosl_klt_group_advance_cams(g.h, mask.ctypes.data) == COSL_E_STATE
    npres = np.zeros(4, np.int32)
    assert lib.cosl_klt_group_first_present(g.h, imgs, W, npres.ctypes.data, None, dest,
                                            n.ctypes.data) == COSL_E_STATE
    tables, counts = g.collect()
    assert tables[2] is None and counts[2] is None and all(t is not None for t in tables[:2])
    assert g.collect() == ([None] * 4, [None] * 4)  # the all-SKIP step
    with pytest.raises(api.CoslError, match="nothing submitted"):
        g.collect()
    # nothing in flight: the synchronous calls run again
    g.step([T, T, N, N], frames(2))
    g.submit_step(ops_ok, frames(3))
    g.collect()
    g.close()
