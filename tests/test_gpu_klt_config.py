"""The CUDA KLT path against the oracle beyond the live CoSLAM settings (needs a GPU): every row of
KLT_CONFIG_ROWS (window half-widths 1 to 15, level lists with and without level 0, 1 to 12
iterations, ITER5 on and off, slot grids whose gain-tracker wait sets overflow), InitMap's detector
call, a level-0-reading configuration through per-camera group steps, the run-time setters, and the
detector past the shared-memory sort's capacity.  The oracle is held to a float64 restatement on
the same rows by tests/test_oracle_klt_config.py.

LK tolerances are what an H100 measured plus a margin (ROW_TOL); each row prints its worst."""
import ctypes as C

import numpy as np
import pytest

import klt_numpy as kn
from coslam_b200.ctypes_defs import (COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK,
                                     KltConfig)
from helpers import KLT_CONFIG_ROWS, compare_features, live_cfg, row_cfg, seq

pytestmark = pytest.mark.gpu

W, H = 640, 480
PASS_KERNELS = 2  # COSL_KLT_PASS_KERNELS: gain tracker one launch per pass, 2x2 tracker untiled
SKIP, FIRST, TRACK, NEXT = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT
LOOSE = dict(pos_tol_px=1.0, gain_tol=1.0, max_flip_frac=1.0)  # statistics only; asserted below
# (max |dpos| px, max |dgain|, max status flips) per row against the oracle, over 3 x next + track.
# Measured on an H100 80GB HBM3 (700 W): <= 2.3e-4 px, <= 1.4e-5 in gain and no flips on every row
# but single_level_2x2, which reaches 3.6e-3 px at one slot (a 5x5 window tracking the whole motion
# at level 0 leaves some tracks unconverged, where rounding differences grow; the row also reports
# which of GPU and oracle lies closer to the float64 restatement there).  The gain limit sits below
# what a wrong gain-neighbour table does on the elongated grids (3.8e-4 and more).  The file takes
# about 40 s there.
ROW_TOL = {r.id: (5e-4, 5e-5, 1) for r in KLT_CONFIG_ROWS}
ROW_TOL["single_level_2x2"] = (6e-3, 5e-5, 1)
POS_TOL_DEFAULT_PX = 2e-3  # compare_features' default: larger differences are checked against float64
MARK = -1e29  # the detector's suppression marks (-1e30 at the pixel of each live track)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same_table(fa, fb):
    return fa.tobytes() == fb.tobytes()


def _pyramids_equal(g, o, L, levels, which=0):
    """every level of the GPU's pyramid `which` bit for bit with the oracle's; level 0 whenever the
    tracker reads it (a tracked frame may leave it unstored otherwise)"""
    for l in range(L):
        if l == 0 and 0 not in levels:
            continue
        assert np.array_equal(_bits(g.pyramid(which, l)), _bits(o.pyramid(which, l))), f"level {l}"


def _cornerness_equal(a, b):
    """bit for bit outside the suppression marks of the live tracks (a track's pixel follows its
    position, which is LK-tolerance parity)"""
    m = (a > MARK) & (b > MARK)
    assert np.array_equal(_bits(a[m]), _bits(b[m]))
    assert m.mean() > 0.99


class Worst:
    def __init__(self):
        self.pos = self.gain = 0.0
        self.flips = 0

    def add(self, st):
        self.pos = max(self.pos, st["pos_max_px"])
        self.gain = max(self.gain, st["gain_max"])
        self.flips = max(self.flips, st["flips"])

    def check(self, name, tol):
        print(f"{name}: worst max |dpos| {self.pos:.2e} px, max |dgain| {self.gain:.2e}, flips {self.flips}")
        assert self.pos <= tol[0] and self.gain <= tol[1] and self.flips <= tol[2], (name, vars(self), tol)


def _closer_to_float64(row, o, prev, fo, fg, tol):
    """The slots where GPU and oracle differ by more than POS_TOL_DEFAULT_PX, against the float64
    restatement of the frame just tracked (the oracle's pyramids of the two frames, which the GPU's
    equal bit for bit, and the provided table `prev`): prints how far each lies from it and asserts
    that the GPU is no farther than the oracle plus the row's tolerance."""
    levels = kn.tracker_levels(row.n_levels, row.level_skip)
    P0 = {l: o.pyramid(1, l).astype(np.float64) for l in levels}
    P1 = {l: o.pyramid(0, l).astype(np.float64) for l in levels}
    X0 = np.where((prev["status"] >= 0)[:, None], prev["pos"].astype(np.float64), -1.0)
    cfg = o.cfg
    args = dict(levels=levels, hw=row.window // 2, conv=cfg.convergenceThreshold, ssd_thr=cfg.SSD_Threshold,
                margin=cfg.trackBorderMargin)
    if row.gain:
        ref = kn.track_gain(P0, P1, X0, W, H, row.fw, row.fh, n_iter=row.n_iter, **args)
    else:
        ref = kn.track_2x2(P0, P1, X0, W, H, n_iter=kn.iterations_2x2(row.n_iter, row.iter5), **args)
    live = (fo["status"] == 0) & (fg["status"] == 0) & (ref[:, 0] >= 0)
    px = np.array([W, H])
    far = live & ((np.abs(fo["pos"] - fg["pos"]) * px).max(1) > POS_TOL_DEFAULT_PX)
    e_gpu = float((np.abs(fg["pos"][far] - ref[far, :2]) * px).max(initial=0))
    e_orc = float((np.abs(fo["pos"][far] - ref[far, :2]) * px).max(initial=0))
    print(f"{row.id}: {int(far.sum())} slots differ by > {POS_TOL_DEFAULT_PX} px; from float64 there: "
          f"GPU {e_gpu:.2e} px, oracle {e_orc:.2e} px")
    assert e_gpu <= e_orc + tol, (e_gpu, e_orc)


@pytest.mark.parametrize("row", KLT_CONFIG_ROWS, ids=[r.id for r in KLT_CONFIG_ROWS])
def test_config_row_against_oracle(api, orc, row):
    """first + 3 x next + track/advance: pyramids, cornerness and first-frame slots bit-exact, LK
    frames within ROW_TOL; the per-pass gain kernels equal the fused tracker bit for bit, the
    untiled 2x2 tracker equals the tiled one within ROW_TOL."""
    orc.set_threads(orc.max_threads())
    L, levels = row.n_levels, kn.tracker_levels(row.n_levels, row.level_skip)
    cfg = row_cfg(row, 1500.0)
    cfg_p = row_cfg(row, 1500.0)
    cfg_p.compat |= PASS_KERNELS
    s = seq(H, W, 71, n=5)
    g = api.KltTracker(cfg, W, H, L, row.fw, row.fh)
    p = api.KltTracker(cfg_p, W, H, L, row.fw, row.fh)
    o = orc.OracleKlt(cfg, W, H, L, row.fw, row.fh)
    fg, ng = g.first(s.frames[0])
    fp, _ = p.first(s.frames[0])
    fo, no = o.first(s.frames[0])
    assert ng == no and g.num_candidates() == o.num_candidates()
    assert _same_table(fg, fo) and _same_table(fp, fo)
    assert np.array_equal(_bits(g.cornerness()), _bits(o.cornerness()))
    _pyramids_equal(g, o, L, range(L))
    worst, other = Worst(), Worst()
    tiled = not row.gain and row.window // 2 <= 3
    for k in range(1, 5):
        prev = fo
        if k < 4:
            fg, ng = g.next(s.frames[k])
            fp, np_ = p.next(s.frames[k])
            fo, no = o.next(s.frames[k])
        else:
            fg, ng = g.track(s.frames[k])
            fp, np_ = p.track(s.frames[k])
            fo, no = o.track(s.frames[k])
            for t in (g, p, o):
                t.advance()
        st = compare_features(fo, fg, W, H, **LOOSE)
        worst.add(st)
        assert abs(ng - no) <= max(2, 2 * st["flips"]), (k, ng, no, st)
        assert (fo["status"] == 0).sum() >= min(20, row.fw * row.fh // 2), (k, (fo["status"] == 0).sum())
        if st["pos_max_px"] > POS_TOL_DEFAULT_PX:
            _closer_to_float64(row, o, prev, fo, fg, ROW_TOL[row.id][0])
        _pyramids_equal(g, o, L, levels if k < 4 else range(L))
        if k < 4:
            _cornerness_equal(g.cornerness(), o.cornerness())
        if tiled:
            other.add(compare_features(fg, fp, W, H, **LOOSE))
            assert abs(ng - np_) <= max(2, 2 * other.flips)
        else:
            assert _same_table(fg, fp) and ng == np_, f"frame {k}: per-pass / untiled tracker differs"
    worst.check(f"{row.id} vs oracle", ROW_TOL[row.id])
    if tiled:
        other.check(f"{row.id} tiled vs untiled 2x2", ROW_TOL[row.id])


@pytest.mark.parametrize("fw,fh", [(32, 4), (4, 64), (1, 16)])
def test_wait_set_overflow_runs_pass_kernels(api, fw, fh):
    """A slot read by more than 8 slots outside its neighbours overflows the persistent gain
    tracker's wait set: the group runs one launch per (level, iteration) pass instead, as
    COSL_KLT_PASS_KERNELS does.  A 32x32 grid keeps the single launch."""
    row = next(r for r in KLT_CONFIG_ROWS if r.id == f"wait_set_{fw}x{fh}")
    n_pass = len(kn.tracker_levels(row.n_levels, row.level_skip)) * row.n_iter
    s = seq(H, W, 72, n=2)

    def launches(grid, compat=0):
        cfg = row_cfg(row, 1500.0)
        cfg.compat |= compat
        t = api.KltTracker(cfg, W, H, row.n_levels, *grid)
        t.first(s.frames[0])
        n0 = api.kernel_launch_count()
        t.next(s.frames[1])
        return api.kernel_launch_count() - n0

    over, forced, square = launches((fw, fh)), launches((fw, fh), PASS_KERNELS), launches((32, 32))
    assert over == forced, (over, forced)
    assert over - square >= n_pass - 1, (over, square, n_pass)


def test_initmap_detector_call(api, orc):
    """InitMap::detectCorners -> GPUKLT::detectCorners (tracking/GPUKLT.cpp:196-210): the default
    config with nLevels = 1, minCornerness 500, minDistance 5 and 32x32 slots, first() on 1280x720."""
    orc.set_threads(orc.max_threads())
    Wi, Hi = 1280, 720
    cfg = KltConfig.reference_defaults()
    cfg.nLevels, cfg.minCornerness, cfg.minDistance = 1, 500.0, 5
    s = seq(Hi, Wi, 73, n=1)
    g = api.KltTracker(cfg, Wi, Hi, 1, 32, 32)
    o = orc.OracleKlt(cfg, Wi, Hi, 1, 32, 32)
    fg, ng = g.first(s.frames[0])
    fo, no = o.first(s.frames[0])
    assert np.array_equal(_bits(g.cornerness()), _bits(o.cornerness()))
    assert ng == no == 1024 and g.num_candidates() == o.num_candidates()
    assert _same_table(fg, fo)
    assert np.array_equal(_bits(g.pyramid(0, 0)), _bits(o.pyramid(0, 0)))


@pytest.mark.parametrize("min_distance,min_corner", [(1, 50.0), (32, 1500.0)])
def test_detector_capacity(api, orc, min_distance, min_corner):
    """minDistance 1 on a textured 1920x1080 frame: more candidates than klt_select_refill sorts in
    shared memory (16 384), so the global-memory sort runs; minDistance 32 is the largest accepted.
    Cornerness, candidate count and slots bit-exact, then one re-detect frame."""
    orc.set_threads(orc.max_threads())
    Wc, Hc = 1920, 1080
    cfg = live_cfg(gain=True, min_corner=min_corner)
    cfg.minDistance = min_distance
    s = seq(Hc, Wc, 91, n=2)
    g = api.KltTracker(cfg, Wc, Hc, 4, 64, 64)
    o = orc.OracleKlt(cfg, Wc, Hc, 4, 64, 64)
    fg, ng = g.first(s.frames[0])
    fo, no = o.first(s.frames[0])
    if min_distance == 1:
        assert o.num_candidates() > 16384, o.num_candidates()
    assert np.array_equal(_bits(g.cornerness()), _bits(o.cornerness()))
    assert ng == no and g.num_candidates() == o.num_candidates()
    assert _same_table(fg, fo)
    fg, ng = g.next(s.frames[1])
    fo, no = o.next(s.frames[1])
    st = compare_features(fo, fg, Wc, Hc, pos_tol_px=5e-4, gain_tol=5e-4, max_flip_frac=0.001)
    assert abs(ng - no) <= max(2, 2 * st["flips"]), (ng, no, st)
    print(f"minDistance {min_distance}: {o.num_candidates()} candidates, next {st}")


def _single_op(t, op, img):
    if op == FIRST:
        out = t.detect(img)
    elif op == TRACK:
        out = t.track(img)
    else:
        out = t.redetect(img)
    t.advance()
    return out


def test_group_steps_level0_config(api, orc):
    """ref_defaults_gain (levels 2,0: the tracker reads level 0) through per-camera group steps that
    mix TRACK / NEXT / SKIP / FIRST, then two pipelined submit_step / collect frames: every addressed
    camera bit for bit with a single tracker and within ROW_TOL of the oracle, and every camera's
    pyramid, level 0 included, bit for bit with the oracle's after every step."""
    orc.set_threads(orc.max_threads())
    row = next(r for r in KLT_CONFIG_ROWS if r.id == "ref_defaults_gain")
    cfg = row_cfg(row, 1500.0)
    n_cams, L = 3, row.n_levels
    seqs = [seq(H, W, 400 + c, n=8) for c in range(n_cams)]
    grp = api.KltGroup(cfg, n_cams, W, H, L, row.fw, row.fh)
    singles = [api.KltTracker(cfg, W, H, L, row.fw, row.fh) for _ in range(n_cams)]
    oracles = [orc.OracleKlt(cfg, W, H, L, row.fw, row.fh) for _ in range(n_cams)]
    sched = [[FIRST, FIRST, FIRST], [NEXT, TRACK, SKIP], [TRACK, NEXT, FIRST], [NEXT, SKIP, NEXT],
             [NEXT, NEXT, TRACK], [NEXT, TRACK, NEXT], [SKIP, NEXT, NEXT]]
    worst = Worst()

    def check(k, ops, tables, counts, pyramids=True):
        for c, op in enumerate(ops):
            if op != SKIP:
                fs, ns = _single_op(singles[c], op, seqs[c].frames[k])
                fo, no = _single_op(oracles[c], op, seqs[c].frames[k])
                assert counts[c] == ns and _same_table(tables[c], fs), (k, c, op)
                if op == FIRST:
                    assert _same_table(fs, fo) and ns == no, (k, c)
                else:
                    worst.add(compare_features(fo, fs, W, H, **LOOSE))
            for l in range(L if pyramids else 0):
                assert np.array_equal(_bits(grp.pyramid(c, 0, l)), _bits(oracles[c].pyramid(0, l))), (k, c, l)

    for k, ops in enumerate(sched[:5]):
        ops = np.array(ops, np.uint8)
        tables, counts = grp.step(ops, [s.frames[k] for s in seqs])
        check(k, ops, [None if t is None else t.copy() for t in tables], counts)
    # pipelined: step 6 is submitted before step 5 is collected
    ops5, ops6 = np.array(sched[5], np.uint8), np.array(sched[6], np.uint8)
    grp.submit_step(ops5, [s.frames[5] for s in seqs])
    grp.submit_step(ops6, [None if o == SKIP else s.frames[6] for s, o in zip(seqs, ops6)])
    t5, c5 = grp.collect()
    t5 = [None if t is None else t.copy() for t in t5]
    t6, c6 = grp.collect()
    t6 = [None if t is None else t.copy() for t in t6]
    check(5, ops5, t5, c5, pyramids=False)  # the group's pyramids are step 6's by now
    check(6, ops6, t6, c6)
    worst.check("group steps (ref_defaults_gain) vs oracle", ROW_TOL[row.id])


@pytest.mark.parametrize("gain", [True, False])
@pytest.mark.parametrize("setter,value,default", [("set_conv", 0.002, 1.0), ("set_ssd", 1000.0, 20000.0),
                                                  ("set_margin", 40.0, 4.0)])
def test_setters_against_oracle(api, orc, gain, setter, value, default):
    """set_conv / set_ssd / set_margin between frames, on the GPU and the oracle alike, with values
    that change the outcome (a convergence threshold that kills most tracks, an SSD threshold that
    kills some, a 40 px margin for tracker and detector), then set back before a re-detect frame."""
    orc.set_threads(orc.max_threads())
    cfg = live_cfg(gain=gain, min_corner=1500.0)
    s = seq(H, W, 81, n=4)
    g = api.KltTracker(cfg, W, H, 6, 32, 32)
    ctl = api.KltTracker(cfg, W, H, 6, 32, 32)  # the same frames without the setter calls
    o = orc.OracleKlt(cfg, W, H, 6, 32, 32)
    for t in (g, ctl, o):
        t.first(s.frames[0])
        t.next(s.frames[1])
    getattr(g, setter)(value)
    getattr(o, setter)(value)
    fg, ng = g.track(s.frames[2])
    fc, _ = ctl.track(s.frames[2])
    fo, no = o.track(s.frames[2])
    st = compare_features(fo, fg, W, H)
    assert abs(ng - no) <= st["flips"], (ng, no, st)
    assert (fc["status"] == 0).sum() - (fg["status"] == 0).sum() >= 10, (setter, ng, (fc["status"] == 0).sum())
    for t in (g, o):
        t.advance()
        getattr(t, setter)(default)
    fg, ng = g.next(s.frames[3])
    fo, no = o.next(s.frames[3])
    st = compare_features(fo, fg, W, H)
    assert abs(ng - no) <= max(2, 2 * st["flips"]), (ng, no, st)
    _cornerness_equal(g.cornerness(), o.cornerness())


def _set(api, grp, name, v):
    fn = getattr(api.LIB, "cosl_klt_" + name)
    fn.argtypes = [C.c_void_p, C.c_float]
    assert fn(grp.h, v) == 0


def test_setter_applies_to_next_submitted_frame(api, orc):
    """On the pipelined path a setter call between submit(n) and submit(n + 1) applies to frame
    n + 1, the first one enqueued after the call, and not to frame n, which is still in flight."""
    orc.set_threads(orc.max_threads())
    cfg = live_cfg(gain=True, min_corner=1500.0)
    n_cams = 2
    seqs = [seq(H, W, 500 + c, n=3) for c in range(n_cams)]
    a = api.KltGroup(cfg, n_cams, W, H, 6, 32, 32)    # pipelined, setter between the two submits
    b = api.KltGroup(cfg, n_cams, W, H, 6, 32, 32)    # synchronous, setter before frame 2
    ctl = api.KltGroup(cfg, n_cams, W, H, 6, 32, 32)  # no setter
    ors = [orc.OracleKlt(cfg, W, H, 6, 32, 32) for _ in range(n_cams)]
    frames = [[s.frames[k] for s in seqs] for k in range(3)]
    for grp in (a, b, ctl):
        grp.first(frames[0])
    for c in range(n_cams):
        ors[c].first(frames[0][c])
    a.submit(frames[1])
    _set(api, a, "set_conv", 0.002)
    a.submit(frames[2])
    r1 = a.collect()[0].copy()
    r2 = a.collect()[0].copy()
    want1 = b.next(frames[1])[0].copy()
    _set(api, b, "set_conv", 0.002)
    want2 = b.next(frames[2])[0].copy()
    ctl1 = ctl.next(frames[1])[0].copy()
    ctl2 = ctl.next(frames[2])[0].copy()
    assert _same_table(r1, want1) and _same_table(r1, ctl1), "frame 1 was enqueued before the call"
    assert _same_table(r2, want2), "frame 2 is the first frame enqueued after the call"
    assert (r2["status"] == 0).sum() < (ctl2["status"] == 0).sum() - 20
    for c in range(n_cams):
        ors[c].next(frames[1][c])
        ors[c].set_conv(0.002)
        fo, _ = ors[c].next(frames[2][c])
        compare_features(fo, r2[c], W, H)
