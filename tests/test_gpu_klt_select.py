"""klt_select_refill against a numpy restatement of the slot logic (needs a GPU).

The restatement takes the candidate keys (~cornerness | y | x) from the detector's cornerness map
(debug_cornerness, suppression marks included), sorts all of them, takes the first
nSel = min(nCand, plCap, free slots) and places them: on a detect frame into slots [0, nSel) ahead
of the present points, on a re-detect frame into the dead slots in increasing index.  The table,
the returned count and the raw candidate count must match bit for bit.  The cases cover fewer,
exactly as many and more free slots than candidates, detect with present lists, a per-camera step
of a mixed-size group (select mode 2), more candidates than the 16 384 keys shared memory holds,
and the HistoPyramid compat list (against the oracle, which restates its Morton order)."""
import ctypes as C

import numpy as np
import pytest

from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

HISTOPYR = 8  # COSL_KLT_COMPAT_HISTOPYR


def candidate_keys(corn, r):
    """sorted uint64 keys of the pixels with c > 0 that are strictly larger than |v| of every other
    texel of their clamped (2r+1)^2 window"""
    a = np.abs(corn)
    p = np.pad(a, r, mode="edge")
    Hc, Wc = corn.shape
    others = np.zeros_like(a)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            if dy or dx:
                np.maximum(others, p[r + dy:r + dy + Hc, r + dx:r + dx + Wc], out=others)
    ys, xs = np.nonzero((corn > 0) & (corn > others))
    cb = (~corn[ys, xs].view(np.uint32)).astype(np.uint64)
    return np.sort((cb << np.uint64(32)) | (ys.astype(np.uint64) << np.uint64(16)) | xs.astype(np.uint64))


def placed(keys, W, H):
    """(pos x, pos y, cornerness) of the first len(keys) keys as klt_select_refill writes them"""
    x = (keys & np.uint64(0xffff)).astype(np.float32)
    y = ((keys >> np.uint64(16)) & np.uint64(0xffff)).astype(np.float32)
    c = (~(keys >> np.uint64(32)).astype(np.uint32)).view(np.float32)
    return (x + np.float32(0.5)) / np.float32(W), (y + np.float32(0.5)) / np.float32(H), c


def check_detect(feats, n, corn, r, W, H, F, pl_cap, present=None, with_gain=True):
    keys = candidate_keys(corn, r)
    n_pres = 0 if present is None else len(present)
    n_sel = max(0, min(len(keys), pl_cap, F - n_pres))
    px, py, c = placed(keys[:n_sel], W, H)
    assert n == n_sel + n_pres
    assert np.array_equal(feats["status"][:n_sel + n_pres], np.ones(n_sel + n_pres, np.int32))
    assert np.array_equal(feats["status"][n_sel + n_pres:], -np.ones(F - n_sel - n_pres, np.int32))
    assert np.array_equal(feats["pos"][:n_sel, 0].view(np.uint32), px.view(np.uint32))
    assert np.array_equal(feats["pos"][:n_sel, 1].view(np.uint32), py.view(np.uint32))
    gain = np.ones(n_sel, np.float32) if with_gain else c
    assert np.array_equal(feats["gain"][:n_sel].view(np.uint32), gain.view(np.uint32))
    if n_pres:
        assert np.array_equal(feats["pos"][n_sel:n_sel + n_pres], np.asarray(present, np.float32)[:, :2])
        assert np.array_equal(feats["fed"][n_sel:n_sel + n_pres], np.arange(n_pres, dtype=np.int32))
    return len(keys), n_sel


def check_redetect(feats, n, corn, r, W, H, F, pl_cap):
    """the slots with status 1 are the first nSel dead slots, in increasing index"""
    keys = candidate_keys(corn, r)
    st = feats["status"]
    n_present = int((st == 0).sum())
    dead = np.nonzero(st != 0)[0]
    n_sel = max(0, min(len(keys), pl_cap, F - n_present))
    new = dead[:n_sel]
    px, py, c = placed(keys[:n_sel], W, H)
    assert n == n_sel + n_present
    assert np.array_equal(np.nonzero(st == 1)[0], new)
    assert np.array_equal(feats["pos"][new, 0].view(np.uint32), px.view(np.uint32))
    assert np.array_equal(feats["pos"][new, 1].view(np.uint32), py.view(np.uint32))
    assert np.array_equal(feats["gain"][new].view(np.uint32), c.view(np.uint32))
    return len(keys), n_sel


@pytest.mark.parametrize("min_corner,fw,fh", [(1500.0, 16, 16), (8000.0, 48, 48)])
def test_detect_then_redetect(api, min_corner, fw, fh):
    """first(): fewer free slots than candidates (1500) or more (8000); then re-detect frames, where
    the dead slots are few against the candidates"""
    W, H = 640, 480
    cfg = live_cfg(gain=True, min_corner=min_corner)
    r = max(1, cfg.minDistance)
    s = seq(H, W, 17, n=4)
    g = api.KltTracker(cfg, W, H, 4, fw, fh)
    F, pl_cap = fw * fh, 4 * fw * fh
    f, n = g.first(s.frames[0])
    nc, ns = check_detect(f, n, g.cornerness(), r, W, H, F, pl_cap)
    assert g.num_candidates() == nc
    assert (ns < nc) == (min_corner == 1500.0), (ns, nc)
    for k in (1, 2, 3):
        f, n = g.next(s.frames[k])
        nc, ns = check_redetect(f, n, g.cornerness(), r, W, H, F, pl_cap)
        assert g.num_candidates() == nc


def test_free_slots_equal_to_candidates(api):
    """nSel == nCand: a tracker with exactly as many slots as the frame has candidates"""
    W, H = 640, 480
    cfg = live_cfg(gain=False, min_corner=3000.0)
    s = seq(H, W, 23, n=1)
    probe = api.KltTracker(cfg, W, H, 4, 64, 64)
    probe.first(s.frames[0])
    n_cand = probe.num_candidates()
    probe.close()
    assert 0 < n_cand < 4096
    g = api.KltTracker(cfg, W, H, 4, n_cand, 1)
    f, n = g.first(s.frames[0])
    nc, ns = check_detect(f, n, g.cornerness(), max(1, cfg.minDistance), W, H, n_cand, 4 * n_cand,
                          with_gain=False)
    assert nc == ns == n_cand


def test_detect_with_present_points(api):
    W, H = 640, 480
    cfg = live_cfg(gain=True, min_corner=1500.0)
    s = seq(H, W, 29, n=1)
    g = api.KltTracker(cfg, W, H, 4, 32, 32)
    rng = np.random.default_rng(3)
    present = np.column_stack([rng.uniform(0.05, 0.95, (300, 2)), np.zeros(300)]).astype(np.float32)
    f, n = g.detect(s.frames[0], present)
    check_detect(f, n, g.cornerness(), max(1, cfg.minDistance), W, H, 1024, 4096, present=present)


def test_many_candidates(api):
    """minDistance 1 on a textured 1920x1080 frame: more candidates than 16 384, 4096 slots"""
    W, H = 1920, 1080
    cfg = live_cfg(gain=True, min_corner=50.0)
    cfg.minDistance = 1
    s = seq(H, W, 91, n=2)
    g = api.KltTracker(cfg, W, H, 4, 64, 64)
    f, n = g.first(s.frames[0])
    nc, ns = check_detect(f, n, g.cornerness(), 1, W, H, 4096, 16384)
    assert nc > 16384 and ns == 4096
    f, n = g.next(s.frames[1])
    check_redetect(f, n, g.cornerness(), 1, W, H, 4096, 16384)


def test_mixed_size_group_step(api):
    """a per-camera step of a mixed-size group: FIRST, NEXT and SKIP cameras in one select launch"""
    sizes = [(640, 480), (320, 240), (512, 384)]
    cfg = live_cfg(gain=True, min_corner=1500.0)
    r = max(1, cfg.minDistance)
    seqs = [seq(h, w, 41 + c, n=3) for c, (w, h) in enumerate(sizes)]
    grp = api.KltGroup(cfg, len(sizes), [w for w, _ in sizes], [h for _, h in sizes], 4, 32, 32)
    grp.first([q.frames[0] for q in seqs])
    for k, ops in ((1, [COSL_KLT_OP_NEXT, COSL_KLT_OP_FIRST, COSL_KLT_OP_SKIP]),
                   (2, [COSL_KLT_OP_NEXT, COSL_KLT_OP_NEXT, COSL_KLT_OP_FIRST])):
        ops = np.array(ops, np.uint8)
        tables, counts = grp.step(ops, [None if o == COSL_KLT_OP_SKIP else q.frames[k] for o, q in zip(ops, seqs)])
        for c, ((w, h), o) in enumerate(zip(sizes, ops)):
            if o == COSL_KLT_OP_SKIP:
                continue
            corn = np.empty((h, w), np.float32)
            assert api.LIB.cosl_klt_debug_cornerness(grp.h, c, corn.ctypes.data_as(C.c_void_p)) == 0
            f = np.array(tables[c])
            if o == COSL_KLT_OP_FIRST:
                nc, _ = check_detect(f, counts[c], corn, r, w, h, 1024, 4096)
            else:
                nc, _ = check_redetect(f, counts[c], corn, r, w, h, 1024, 4096)
            assert api.LIB.cosl_klt_debug_num_candidates(grp.h, c) == nc


@pytest.mark.parametrize("min_corner", [1500.0, 8000.0])
def test_histopyr_compat(api, orc, min_corner):
    """COSL_KLT_COMPAT_HISTOPYR keeps the whole Morton-ordered list: against the oracle"""
    W, H = 640, 480
    cfg = live_cfg(gain=True, min_corner=min_corner)
    cfg.compat |= HISTOPYR
    s = seq(H, W, 53, n=3)
    g = api.KltTracker(cfg, W, H, 4, 32, 32)
    o = orc.OracleKlt(cfg, W, H, 4, 32, 32)
    fg, ng = g.first(s.frames[0])
    fo, no = o.first(s.frames[0])
    assert ng == no and fg.tobytes() == fo.tobytes()
    assert g.num_candidates() == o.num_candidates()
