"""The hw = 3 gain tracker walks a window one column per lane (klt_track.cuh).  Every path of both
drivers -- the staged tile, the re-centred tile, the fused kernel's items without a tile and the
per-pass kernel -- must take the same lane assignment and summation order, so the persistent
tracker equals the per-pass launches bit for bit, and both stay within the oracle tolerance.  The
sequences are built for those paths: windows across the borders of tiny coarse levels, motion
large enough to carry windows out of their tiles, slot grids with F % 4 != 0 (lane groups of one
warp on two cameras), dead slots, more items than resident lane groups, and a group of cameras of
different sizes."""
import numpy as np
import pytest

from helpers import compare_features, live_cfg, seq

pytestmark = pytest.mark.gpu

# id: camera sizes, pyramid levels, slot grid, pixels of motion per frame, minCornerness
CASES = {
    # level 5 is 7 x 4 texels: every coarse window straddles the level borders; F = 143
    "coarse_borders": ([(224, 136)] * 2, 6, (13, 11), 3.0, 800.0),
    # 14 px per frame carries the level-1 windows several texels: tiles are re-centred
    "large_motion": ([(640, 480)] * 2, 6, (32, 32), 14.0, 1500.0),
    # 40 x 225 = 9 000 items, more than an H100 keeps resident (132 SMs x 4 CTAs x 16 lane groups):
    # the last cameras' slots take the fused kernel's path without a tile
    "non_resident": ([(320, 240)] * 40, 4, (15, 15), 3.0, 300.0),
    # three image sizes in one group, F = 195
    "mixed": ([(640, 480), (333, 251), (752, 480)], 6, (15, 13), 8.0, 3000.0),
}


def _seqs(sizes, shift, seed):
    return [seq(h, w, seed + c, n=4, max_shift=shift, pad=48) for c, (w, h) in enumerate(sizes)]


def _group(api, cfg, sizes, L, fw, fh):
    ws, hs = [w for w, _ in sizes], [h for _, h in sizes]
    if len(set(sizes)) == 1:
        return api.KltGroup(cfg, len(sizes), ws[0], hs[0], L, fw, fh)
    return api.KltGroup(cfg, len(sizes), ws, hs, L, fw, fh)


@pytest.mark.parametrize("case", list(CASES))
def test_fused_equals_pass_kernels_and_oracle(api, orc, case):
    sizes, L, (fw, fh), shift, corner = CASES[case]
    orc.set_threads(orc.max_threads())
    seqs = _seqs(sizes, shift, 900 + 10 * list(CASES).index(case))
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    cfg_f = live_cfg(gain=True, min_corner=corner)
    cfg_p = live_cfg(gain=True, min_corner=corner)
    cfg_p.compat |= 2  # COSL_KLT_PASS_KERNELS
    a = _group(api, cfg_f, sizes, L, fw, fh)
    b = _group(api, cfg_p, sizes, L, fw, fh)
    ors = [orc.OracleKlt(cfg_f, w, h, L, fw, fh) for w, h in sizes]
    fa, na = a.first(frames(0))
    fb, nb = b.first(frames(0))
    assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes()
    for c, (w, h) in enumerate(sizes):
        fo, no = ors[c].first(seqs[c].frames[0])
        assert na[c] == no and np.array_equal(fa[c]["pos"].view(np.uint32), fo["pos"].view(np.uint32))
    dead = 0
    for k in range(1, 4):
        fa, na = a.next(frames(k))
        fb, nb = b.next(frames(k))
        assert np.array_equal(na, nb) and fa.tobytes() == fb.tobytes(), f"frame {k}"
        for c, (w, h) in enumerate(sizes):
            fo, _ = ors[c].next(seqs[c].frames[k])
            compare_features(fo, fa[c], w, h)
        dead += int((fa["status"] < 0).sum())
        assert (fa["status"] == 0).sum() > 0.2 * fa.size, f"frame {k}: too few tracks to test"
    assert dead > 0, "the sequence should leave dead slots"
    if case == "non_resident":
        assert (fa.reshape(-1)["status"][8448:] >= 0).sum() > 100, "too few live items without a tile"
    a.close()
    b.close()
