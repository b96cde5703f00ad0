"""Per-camera frame ops on a KLT camera group (cosl_klt_group_step): a camera addressed with an op
behaves bit for bit like a single-camera tracker that receives the matching call followed by
advance, and a skipped camera keeps all of its state (needs a GPU)."""
import numpy as np
import pytest

from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import compare_features, live_cfg, seq

pytestmark = pytest.mark.gpu

W, H, L, FW, FH = 640, 480, 6, 32, 32
SIZES = [(640, 480), (328, 250), (512, 384), (400, 300)]
COSL_E_INVALID, COSL_E_STATE = -1, -6
SKIP, FIRST, TRACK, NEXT = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT


def _single_op(t, op, img):
    """the single tracker's call for `op` followed by advance: (table, count)"""
    if op == FIRST:
        out = t.detect(img)
    elif op == TRACK:
        out = t.track(img)
    else:
        out = t.redetect(img)
    t.advance()
    return out


def _step_both(grp, singles, ops, frames, what):
    imgs = [None if o == SKIP else im for o, im in zip(ops, frames)]
    tables, counts = grp.step(ops, imgs)
    for c, o in enumerate(ops):
        if o == SKIP:
            assert tables[c] is None and counts[c] is None
            continue
        f1, n1 = _single_op(singles[c], o, frames[c])
        assert counts[c] == n1, (what, c, o, counts[c], n1)
        assert tables[c].tobytes() == f1.tobytes(), (what, c, o)
    return tables, counts


def _schedule(rng, n_cams, n_steps):
    """random ops with every camera detected first and all four ops present"""
    sched = [np.full(n_cams, FIRST, np.uint8)]
    sched[0][0] = SKIP  # camera 0 comes in late: its first op is FIRST below
    for k in range(1, n_steps):
        ops = rng.choice([SKIP, FIRST, TRACK, NEXT], size=n_cams, p=[0.25, 0.1, 0.35, 0.3]).astype(np.uint8)
        if k == 1:
            ops[0] = FIRST
        sched.append(ops)
    return sched


def _mixed_rig(api, cfg, sizes, n_levels=L):
    ws, hs = [w for w, _ in sizes], [h for _, h in sizes]
    grp = api.KltGroup(cfg, len(sizes), ws, hs, n_levels, FW, FH)
    return grp, [api.KltTracker(cfg, w, h, n_levels, FW, FH) for w, h in sizes]


# 2 = COSL_KLT_PASS_KERNELS (one gain-tracker launch per pass; with trackWithGain 0 the untiled 2x2
# tracker), 8 = COSL_KLT_COMPAT_HISTOPYR (the reference's candidate list in klt_select_refill)
@pytest.mark.parametrize("compat_bit", [0, 2, 8])
@pytest.mark.parametrize("gain", [True, False])
@pytest.mark.parametrize("mixed", [False, True])
def test_random_schedule_matches_single_trackers(api, gain, mixed, compat_bit):
    """12 steps of random ops (all four, SKIP included) on 4 cameras against 4 single trackers."""
    sizes = SIZES if mixed else [(W, H)] * 4
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    cfg.compat |= compat_bit
    grp, singles = _mixed_rig(api, cfg, sizes)
    seqs = [seq(h, w, 300 + c, n=12) for c, (w, h) in enumerate(sizes)]
    rng = np.random.default_rng(7 + 2 * gain + mixed)
    sched = _schedule(rng, 4, 12)
    seen = set()
    for k, ops in enumerate(sched):
        seen.update(int(o) for o in ops)
        _step_both(grp, singles, ops, [s.frames[k] for s in seqs], f"step {k} ops {list(ops)}")
    assert seen == {SKIP, FIRST, TRACK, NEXT}


def test_all_next_and_all_first_equal_the_group_calls(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 320 + c, n=4) for c in range(3)]
    a = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    b = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    fa, na = a.first(frames(0))
    tb, nb = b.step([FIRST] * 3, frames(0))
    assert list(na) == nb and all(fa[c].tobytes() == tb[c].tobytes() for c in range(3))
    for k in range(1, 4):
        fa, na = a.next(frames(k))
        tb, nb = b.step([NEXT] * 3, frames(k))
        assert list(na) == nb and all(fa[c].tobytes() == tb[c].tobytes() for c in range(3)), k


def test_skipped_camera_keeps_its_state(api):
    """Camera 1 skips two mixed steps (one that exchanges the skipped cameras' pyramids, one that
    exchanges the addressed camera's): its pyramids (both buffers, every level and which levels are
    readable) are unchanged and equal a single tracker that did not get the frames; its next frame
    continues as that tracker."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 340 + c, n=5) for c in range(3)]
    grp, singles = _mixed_rig(api, cfg, [(W, H)] * 3)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    _step_both(grp, singles, [FIRST] * 3, frames(0), "first")
    _step_both(grp, singles, [TRACK, TRACK, NEXT], frames(1), "track")

    def snapshot(get):
        out = {}
        for which in (0, 1):
            for level in range(L):
                try:
                    out[which, level] = get(which, level).tobytes()
                except api.CoslError:
                    out[which, level] = None
        return out

    before = snapshot(lambda w, lv: grp.pyramid(1, w, lv))
    assert before == snapshot(lambda w, lv: singles[1].pyramid(w, lv))
    for ops, k in (([NEXT, SKIP, TRACK], 2), ([SKIP, SKIP, FIRST], 3)):  # flip + exchange, then exchange
        _step_both(grp, singles, ops, frames(k), f"skip {ops}")
        assert snapshot(lambda w, lv: grp.pyramid(1, w, lv)) == before
        assert snapshot(lambda w, lv: singles[1].pyramid(w, lv)) == before
    _step_both(grp, singles, [NEXT, TRACK, NEXT], frames(4), "after skip")


def test_step_composes_with_feed_and_advance(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 360 + c, n=5) for c in range(3)]
    grp, singles = _mixed_rig(api, cfg, [(W, H)] * 3)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    rng = np.random.default_rng(5)
    _step_both(grp, singles, [FIRST] * 3, frames(0), "first")
    _step_both(grp, singles, [TRACK, SKIP, NEXT], frames(1), "step 1")
    pts = np.zeros((6, 3), np.float32)
    pts[:, 0] = rng.uniform(0.1, 0.9, 6)
    pts[:, 1] = rng.uniform(0.1, 0.9, 6)
    ids, fed = grp.feed([pts, None, pts])
    for c in (0, 2):
        i1, n1 = singles[c].feed(pts)
        assert fed[c] == n1 and np.array_equal(ids[c], i1)
    grp.advance([0, 2])
    singles[0].advance()
    singles[2].advance()
    _step_both(grp, singles, [NEXT, TRACK, TRACK], frames(2), "step 2")
    _step_both(grp, singles, [SKIP, NEXT, NEXT], frames(3), "step 3")
    _step_both(grp, singles, [TRACK, TRACK, NEXT], frames(4), "step 4")


def test_step_dev_then_fetch_equals_step(api):
    import torch

    cfg = live_cfg(gain=True, min_corner=1500.0)
    sizes = SIZES[:3]
    seqs = [seq(h, w, 380 + c, n=4) for c, (w, h) in enumerate(sizes)]
    a, _ = _mixed_rig(api, cfg, sizes)
    b, _ = _mixed_rig(api, cfg, sizes)
    sched = [[FIRST] * 3, [TRACK, SKIP, NEXT], [NEXT, TRACK, SKIP], [SKIP, NEXT, TRACK]]
    for k, ops in enumerate(sched):
        frames = [s.frames[k] for s in seqs]
        ta, na = a.step(ops, [None if o == SKIP else im for o, im in zip(ops, frames)])
        dev = [torch.from_numpy(np.ascontiguousarray(im)).cuda() for im in frames]
        torch.cuda.synchronize()
        b.step_dev(ops, [0 if o == SKIP else t.data_ptr() for o, t in zip(ops, dev)], 0)
        fb, nb = b.fetch()
        for c, o in enumerate(ops):
            if o != SKIP:
                assert na[c] == nb[c] and ta[c].tobytes() == fb[c].tobytes(), (k, c)


def test_bad_arguments_and_frames_in_flight(api):
    import ctypes as C

    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 400 + c, n=3) for c in range(2)]
    g = api.KltGroup(cfg, 2, W, H, L, FW, FH)
    frames = [s.frames[0] for s in seqs]
    imgs = (C.c_void_p * 2)(*[im.ctypes.data for im in frames])
    dest = (C.c_void_p * 2)(*[g.feats[c].ctypes.data for c in range(2)])
    n = np.zeros(2, np.int32)

    def call(ops, ptrs=imgs):
        ops = np.asarray(ops, np.uint8)
        return api.LIB.cosl_klt_group_step(g.h, ops.ctypes.data, ptrs, W, dest, n.ctypes.data)

    assert call([FIRST, 4]) == COSL_E_INVALID
    assert call([255, FIRST]) == COSL_E_INVALID
    assert call([FIRST, TRACK], (C.c_void_p * 2)(imgs[0], None)) == COSL_E_INVALID
    assert call([FIRST, SKIP], (C.c_void_p * 2)(imgs[0], None)) == 0
    assert api.LIB.cosl_klt_group_step_dev(g.h, np.array([1, 9], np.uint8).ctypes.data, imgs, W) == COSL_E_INVALID
    g.submit([s.frames[1] for s in seqs])
    assert call([NEXT, NEXT]) == COSL_E_STATE
    g.collect()
    assert call([NEXT, SKIP], (C.c_void_p * 2)(imgs[0], None)) == 0


def test_all_skip_launches_nothing_and_one_camera_no_more_than_next(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 420 + c, n=4) for c in range(4)]
    g = api.KltGroup(cfg, 4, W, H, L, FW, FH)
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    g.first(frames(0))

    def count(fn):
        n0 = api.kernel_launch_count()
        fn()
        return api.kernel_launch_count() - n0

    assert count(lambda: g.step([SKIP] * 4, [None] * 4)) == 0
    n_next = count(lambda: g.next(frames(1)))
    one = count(lambda: g.step([SKIP, TRACK, SKIP, SKIP], [None, frames(2)[1], None, None]))
    assert 0 < one <= n_next, (one, n_next)


def test_track_cadence_on_one_camera_matches_the_oracle(api, orc):
    """Camera 1 of a 3-camera group runs first, 3 x TRACK, NEXT, TRACK while the others re-detect
    or skip: its tables follow the CPU restatement within the tolerances of test_gpu_klt.py."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 440 + c, n=6) for c in range(3)]
    g = api.KltGroup(cfg, 3, W, H, L, FW, FH)
    o = orc.OracleKlt(cfg, W, H, L, FW, FH)
    cadence = [FIRST, TRACK, TRACK, TRACK, NEXT, TRACK]
    others = [[FIRST, FIRST], [NEXT, SKIP], [SKIP, NEXT], [NEXT, NEXT], [TRACK, SKIP], [NEXT, TRACK]]
    for k, op in enumerate(cadence):
        ops = [others[k][0], op, others[k][1]]
        frames = [s.frames[k] for s in seqs]
        tables, counts = g.step(ops, [None if x == SKIP else im for x, im in zip(ops, frames)])
        if op == FIRST:
            fo, no = o.first(frames[1])
            assert counts[1] == no
            assert np.array_equal(tables[1]["pos"].view(np.uint32), fo["pos"].view(np.uint32))
            continue
        if op == TRACK:
            fo, no = o.track(frames[1])
            o.advance()
        else:
            fo, no = o.next(frames[1])
        st = compare_features(fo, tables[1], W, H, max_flip_frac=0.005)
        assert abs(counts[1] - no) <= max(2, st["flips"] * 2), (k, counts[1], no, st)


def test_track_and_next_before_any_detect(api):
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 460 + c, n=2) for c in range(3)]
    grp, singles = _mixed_rig(api, cfg, [(W, H)] * 3)
    _step_both(grp, singles, [TRACK, NEXT, FIRST], [s.frames[0] for s in seqs], "undetected")
    _step_both(grp, singles, [NEXT, TRACK, TRACK], [s.frames[1] for s in seqs], "after")


def test_mixed_group_steps_cameras_narrower_than_the_widest(api):
    """A step that addresses only cameras narrower than the widest one: frames whose rows are their
    own camera's width apart (pitch 0 through the binding), and frames sharing one pitch that holds
    the widest camera."""
    cfg = live_cfg(gain=True, min_corner=1500.0)
    grp, singles = _mixed_rig(api, cfg, SIZES)
    seqs = [seq(h, w, 480 + c, n=4) for c, (w, h) in enumerate(SIZES)]
    _step_both(grp, singles, [FIRST] * 4, [s.frames[0] for s in seqs], "first")
    _step_both(grp, singles, [SKIP, TRACK, SKIP, SKIP], [s.frames[1] for s in seqs], "one small camera")
    _step_both(grp, singles, [SKIP, SKIP, NEXT, TRACK], [s.frames[2] for s in seqs], "two small cameras")
    padded = []
    for c, s in enumerate(seqs):  # rows 640 bytes apart, the widest camera's width
        buf = np.zeros((SIZES[c][1], SIZES[0][0]), np.uint8)
        buf[:, :SIZES[c][0]] = s.frames[3]
        padded.append(buf[:, :SIZES[c][0]])
    _step_both(grp, singles, [SKIP, NEXT, SKIP, TRACK], padded, "shared pitch")
