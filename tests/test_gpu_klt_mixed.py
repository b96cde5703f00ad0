"""KLT camera groups whose cameras differ in image size (cosl_klt_group_create_sizes): every camera of
a mixed group must behave bit for bit like a single-camera tracker of its own size that receives the
same calls.  The sizes include odd ones, widths that are not multiples of 4, 16 or 64, and a small
camera whose level 5 is 10 x 7 texels; every buffer slice is laid out at the largest camera, so these
comparisons also show that no kernel reads a smaller camera's padding.  GPU tests are marked; the
last two tests run without a GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from helpers import live_cfg, seq

SIZES = [(640, 480), (320, 240), (752, 480), (333, 251)]
L = 6
COSL_E_INVALID, COSL_E_CUDA, COSL_E_STATE = -1, -2, -6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coslam_b200", "libcoslam_b200.so")


def _cfg(gain, live_window):
    c = live_cfg(gain=gain, min_corner=1500.0)
    if not live_window:
        c.windowWidth = 5  # half-width 2: the trackers' generic (run-time width) instantiation
    return c


def _seqs(seed, n, sizes=SIZES):
    return [seq(h, w, seed + c, n=n) for c, (w, h) in enumerate(sizes)]


def _pts(rng, n):
    p = np.zeros((n, 3), np.float32)
    p[:, 0] = rng.uniform(0.05, 0.95, n)
    p[:, 1] = rng.uniform(0.05, 0.95, n)
    return p


def _rig(api, cfg, fw, fh, sizes=SIZES):
    grp = api.KltGroup(cfg, len(sizes), [w for w, _ in sizes], [h for _, h in sizes], L, fw, fh)
    return grp, [api.KltTracker(cfg, w, h, L, fw, fh) for w, h in sizes]


def _check(f, n, outs, what):
    for c, (fs, ns) in enumerate(outs):
        assert ns == n[c], (what, c, ns, n[c])
        assert fs.tobytes() == f[c].tobytes(), (what, c)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [(32, 32), (10, 15)], ids=["F1024", "F150"])
@pytest.mark.parametrize("live_window", [True, False], ids=["hw3", "hw2"])
@pytest.mark.parametrize("gain", [True, False], ids=["gain", "2x2"])
def test_rig_cadence_matches_single_trackers(api, gain, live_window, grid):
    """Seeded first (camera 1 without present points), next x3, feed + advance of cameras {0, 2},
    next, two frames through submit / collect, then next_dev + fetch."""
    import torch

    fw, fh = grid
    cfg = _cfg(gain, live_window)
    seqs = _seqs(200, 8)
    grp, singles = _rig(api, cfg, fw, fh)
    rng = np.random.default_rng(17)
    present = [_pts(rng, 30), np.zeros((0, 3), np.float32), _pts(rng, 20), _pts(rng, 9)]
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    f, n = grp.first(frames(0), present=present)
    outs = []
    for c in range(4):
        outs.append(singles[c].detect(seqs[c].frames[0], present[c]))
        singles[c].advance()
    _check(f, n, outs, "first_present")
    assert (f[1]["fed"] >= 0).sum() == 0
    for k in (1, 2, 3):
        f, n = grp.next(frames(k))
        _check(f, n, [singles[c].next(seqs[c].frames[k]) for c in range(4)], f"next frame {k}")
    # feed + advance of a subset; the first point of camera 0 sits on a live track, which dies
    p0 = _pts(rng, 7)
    p0[0, :2] = f[0]["pos"][f[0]["status"] >= 0][0]
    lists = [p0, None, _pts(rng, 11), None]
    ids, fed = grp.feed(lists)
    for c in (0, 2):
        i1, n1 = singles[c].feed(lists[c])
        assert fed[c] == n1 and np.array_equal(ids[c], i1), c
        singles[c].advance()
    grp.advance([0, 2])
    f, n = grp.next(frames(4))
    _check(f, n, [singles[c].next(seqs[c].frames[4]) for c in range(4)], "next after the subset advance")
    # two frames in flight
    grp.submit(frames(5))
    grp.submit(frames(6))
    for k in (5, 6):
        f, n = grp.collect()
        _check(f, n, [singles[c].next(seqs[c].frames[k]) for c in range(4)], f"collect frame {k}")
    # device-resident frames, each camera's rows its own width apart (pitch 0)
    dev = [torch.from_numpy(im).cuda() for im in frames(7)]
    torch.cuda.synchronize()
    grp.next_dev([t.data_ptr() for t in dev], 0)
    f, n = grp.fetch()
    _check(f, n, [singles[c].next(seqs[c].frames[7]) for c in range(4)], "next_dev")
    assert all(n[c] > 0 for c in range(4))


@pytest.mark.gpu
@pytest.mark.parametrize("gain", [True, False], ids=["gain", "2x2"])
def test_pyramids_and_cornerness_match_single_trackers(api, gain):
    """After first + next + advance of cameras {0, 2}, every camera returns its own pyramid levels
    from both buffers and refuses exactly the level 0 its single-camera twin refuses; the cornerness
    map of each camera equals its twin's after every frame."""
    cfg = _cfg(gain, True)
    seqs = _seqs(300, 3)
    grp, singles = _rig(api, cfg, 32, 32)
    grp.first([s.frames[0] for s in seqs])
    for c in range(4):
        singles[c].first(seqs[c].frames[0])
        assert np.array_equal(grp.cornerness(c).view(np.uint32), singles[c].cornerness().view(np.uint32)), c
    grp.next([s.frames[1] for s in seqs])
    for c in range(4):
        singles[c].next(seqs[c].frames[1])
        assert np.array_equal(grp.cornerness(c).view(np.uint32), singles[c].cornerness().view(np.uint32)), c
    grp.advance([0, 2])
    for c in (0, 2):
        singles[c].advance()
    for c, (w, h) in enumerate(SIZES):
        for which in (0, 1):
            for level in range(L):
                try:
                    b = singles[c].pyramid(which, level)
                except api.CoslError as e:
                    assert level == 0 and "not stored" in str(e)
                    with pytest.raises(api.CoslError, match="not stored"):
                        grp.pyramid(c, which, 0)
                    continue
                a = grp.pyramid(c, which, level)
                assert a.shape == (h >> level, w >> level, 3)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (c, which, level)
    f, n = grp.next([s.frames[2] for s in seqs])
    _check(f, n, [singles[c].next(seqs[c].frames[2]) for c in range(4)], "next after the exchange")
    for c in range(4):
        assert np.array_equal(grp.cornerness(c).view(np.uint32), singles[c].cornerness().view(np.uint32)), c


@pytest.mark.gpu
def test_equal_sizes_equal_group_create(api):
    cfg = _cfg(True, True)
    seqs = _seqs(400, 4, sizes=[(640, 480)] * 4)
    a = api.KltGroup(cfg, 4, 640, 480, L, 32, 32)
    b = api.KltGroup(cfg, 4, [640] * 4, [480] * 4, L, 32, 32)
    assert b.mixed and not a.mixed
    rng = np.random.default_rng(4)
    present = [_pts(rng, 10), None, _pts(rng, 3), None]
    fa, na = a.first([s.frames[0] for s in seqs], present=present)
    fb, nb = b.first([s.frames[0] for s in seqs], present=present)
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()
    for k in (1, 2):
        fa, na = a.next([s.frames[k] for s in seqs])
        fb, nb = b.next([s.frames[k] for s in seqs])
        assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes(), k
    pts = [_pts(rng, 5), None, None, _pts(rng, 8)]
    ia, da = a.feed(pts)
    ib, db = b.feed(pts)
    assert np.array_equal(da, db) and all(x is None and y is None or np.array_equal(x, y) for x, y in zip(ia, ib))
    a.advance([0, 3])
    b.advance([0, 3])
    fa, na = a.next([s.frames[3] for s in seqs])
    fb, nb = b.next([s.frames[3] for s in seqs])
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()


def _count(api, fn):
    n0 = api.kernel_launch_count()
    fn()
    return api.kernel_launch_count() - n0


@pytest.mark.gpu
def test_mixed_group_launches_equal_a_uniform_group(api):
    import torch

    cfg = _cfg(True, True)
    got = []
    for sizes in (SIZES, [(640, 480)] * 4):
        seqs = _seqs(500, 5, sizes=sizes)
        frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
        dev = [torch.from_numpy(im).cuda() for im in frames(3)]
        torch.cuda.synchronize()
        g = api.KltGroup(cfg, 4, [w for w, _ in sizes], [h for _, h in sizes], L, 32, 32)
        rng = np.random.default_rng(5)
        n = {"first": _count(api, lambda: g.first(frames(0), present=[_pts(rng, 9), None, None, _pts(rng, 4)]))}
        n["next"] = _count(api, lambda: g.next(frames(1)))
        n["submit"] = _count(api, lambda: g.submit(frames(2)))
        g.collect()
        n["next_dev"] = _count(api, lambda: g.next_dev([t.data_ptr() for t in dev], 0))
        g.fetch()
        n["feed"] = _count(api, lambda: g.feed([_pts(rng, 20), None, _pts(rng, 30), None]))
        n["advance_subset"] = _count(api, lambda: g.advance([0, 2]))
        n["advance_all"] = _count(api, lambda: g.advance())
        n["first_plain"] = _count(api, lambda: g.first(frames(4)))
        g.close()
        got.append(n)
    assert got[0] == got[1], got


@pytest.mark.gpu
def test_bad_arguments(api):
    from coslam_b200.api import _ptr
    lib = api.LIB
    cfg = _cfg(True, True)
    ws, hs = np.array([w for w, _ in SIZES], np.int32), np.array([h for _, h in SIZES], np.int32)
    h = C.c_void_p()

    def create(w, hh, n_levels=L):
        return lib.cosl_klt_group_create_sizes(C.byref(cfg), len(ws), _ptr(w), _ptr(hh), n_levels, 32, 32, 0, 0,
                                               0, C.byref(h))

    assert create(None, hs) == COSL_E_INVALID
    assert create(ws, None) == COSL_E_INVALID
    # the smallest camera decides the depth: 240 >> 7 = 1
    assert create(ws, hs, 8) == COSL_E_INVALID and b"camera 1" in lib.cosl_last_error()
    small = ws.copy()
    small[3] = 60  # 60 >> 5 = 1
    assert create(small, hs) == COSL_E_INVALID and b"camera 3" in lib.cosl_last_error()
    seqs = _seqs(600, 2)
    grp = api.KltGroup(cfg, 4, ws, hs, L, 32, 32)
    frames = [np.ascontiguousarray(s.frames[0]) for s in seqs]
    ptrs = (C.c_void_p * 4)(*[f.ctypes.data for f in frames])
    dest, cnt = grp._dest, _ptr(grp.counts)
    # a pitch > 0 must hold the widest camera
    assert lib.cosl_klt_group_first(grp.h, ptrs, 751, dest, cnt) == COSL_E_INVALID
    assert lib.cosl_klt_group_next(grp.h, ptrs, 640, dest, cnt) == COSL_E_INVALID
    assert lib.cosl_klt_group_submit(grp.h, ptrs, 333) == COSL_E_INVALID
    assert lib.cosl_klt_group_first(grp.h, ptrs, 0, dest, cnt) == 0
    padded = [np.zeros((h_, 752), np.uint8) for _, h_ in SIZES]
    for p, f in zip(padded, frames):
        p[:, :f.shape[1]] = f
    pp = (C.c_void_p * 4)(*[p.ctypes.data for p in padded])
    assert lib.cosl_klt_group_next(grp.h, pp, 752, dest, cnt) == 0
    # single-camera calls stay single-camera only
    pts, ids = np.zeros((4, 3), np.float32), np.zeros(4, np.int32)
    assert lib.cosl_klt_feed(grp.h, 4, _ptr(pts), _ptr(ids), C.byref(C.c_int(0))) == COSL_E_STATE
    grp.close()
    # pitch 0 stays invalid on a group made with cosl_klt_group_create
    uni = api.KltGroup(cfg, 4, 640, 480, L, 32, 32)
    same = [np.ascontiguousarray(s.frames[0]) for s in _seqs(610, 1, sizes=[(640, 480)] * 4)]
    up = (C.c_void_p * 4)(*[f.ctypes.data for f in same])
    assert lib.cosl_klt_group_first(uni.h, up, 0, uni._dest, _ptr(uni.counts)) == COSL_E_INVALID
    assert lib.cosl_klt_group_next_dev(uni.h, up, 0) == COSL_E_INVALID
    assert lib.cosl_klt_group_first(uni.h, up, 640, uni._dest, _ptr(uni.counts)) == 0
    uni.close()


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_create_sizes_is_exported_and_needs_a_device(api):
    from coslam_b200.api import _ptr
    assert hasattr(C.CDLL(api.LIB_PATH), "cosl_klt_group_create_sizes")
    cfg = _cfg(True, True)
    ws, hs = np.array([w for w, _ in SIZES], np.int32), np.array([h for _, h in SIZES], np.int32)
    h = C.c_void_p()
    rc = api.LIB.cosl_klt_group_create_sizes(C.byref(cfg), 4, _ptr(ws), _ptr(hs), L, 32, 32, 0, 0, 0, C.byref(h))
    assert rc == COSL_E_CUDA and not h.value
    with pytest.raises(api.CoslError):
        api.KltGroup(cfg, 4, ws, hs, L, 32, 32)


def _tool(name):
    exe = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    if not os.path.exists(exe):
        pytest.skip(f"{name} not found")
    if not os.path.exists(LIB):
        pytest.skip(f"{LIB} is not built")
    return exe


def test_every_gain_tracker_instantiation_keeps_its_budget():
    """The per-camera extents are read from global memory, never selected between kernel
    parameters: every gain-tracker instantiation in the library (whatever its name) has no predicated
    32-bit constant load, no spill and at most 128 registers (the checks of test_klt_sass.py)."""
    exe = _tool("cuobjdump")
    pat = re.compile(r"klt_gain_(?:fused|pass)I")
    sass = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    bodies = {p.split(None, 1)[0]: p for p in re.split(r"\n\s*Function : ", sass)[1:] if pat.search(p.split(None, 1)[0])}
    assert len(bodies) >= 4, sorted(bodies)
    for name, body in bodies.items():
        loads = re.findall(r"@!?U?P[0-6T]\s+LDC(?:\.(?:U8|S8|U16|S16|32))?\s+[^;]*;", body)
        assert not loads, (name, loads[:4])
    res = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    seen = 0
    for part in re.split(r"\n\s*Function ", res)[1:]:
        name = part.split(None, 1)[0].rstrip(":")
        if not pat.search(name):
            continue
        seen += 1
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:\d+\s+LOCAL:(\d+)", part)
        assert m, name
        regs, stack, local = map(int, m.groups())
        assert regs <= 128 and stack == 0 and local == 0, (name, regs, stack, local)
    assert seen == len(bodies)
