"""The pyramid chain klt_front -> klt_pyr_down_tma x (L - 2) runs as programmatic dependent launches:
each level's CTAs may start while the kernel that writes its source level still runs, and wait for
it in the kernel (DESIGN.md §3.2).  Every level of both pyramid buffers must come out bit for bit
as the CPU oracle builds it from the same image, for groups driven by unsynchronised next_dev calls
and by the synchronous next() (host uploads: two front launches per frame), at L = 3, 4, 6 and 8
and in a group of cameras of different sizes (needs a GPU)."""
import numpy as np
import pytest

from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

FRAMES = 8
MIXED = [(640, 480), (320, 240), (752, 480), (333, 251)]


def _group(api, cfg, sizes, L):
    if len(set(sizes)) == 1:
        return api.KltGroup(cfg, len(sizes), sizes[0][0], sizes[0][1], L, 16, 16)
    return api.KltGroup(cfg, len(sizes), [w for w, _ in sizes], [h for _, h in sizes], L, 16, 16)


def _oracle_pyramids(orc, cfg, sizes, seqs, L, k):
    """[camera][level] of the oracle's pyramid of frame k (None where the group does not keep it)"""
    out = []
    for (w, h), s in zip(sizes, seqs):
        o = orc.OracleKlt(cfg, w, h, L, 16, 16)
        o.detect(s.frame(k))
        out.append([o.pyramid(1, level).copy() for level in range(L)])
        o.close()
    return out


@pytest.mark.parametrize("sizes,L", [
    ([(320, 240)] * 2, 3),
    ([(328, 250)] * 3, 4),
    ([(640, 480)] * 4, 6),
    ([(1280, 720)] * 2, 8),
    (MIXED, 6),
], ids=["L3", "L4", "L6", "L8", "mixed-L6"])
def test_pyramid_chain_equals_oracle(api, orc, sizes, L):
    import torch

    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(h, w, 700 + c, n=5) for c, (w, h) in enumerate(sizes)]
    a, b = _group(api, cfg, sizes, L), _group(api, cfg, sizes, L)
    dev = [[torch.from_numpy(np.ascontiguousarray(s.frame(k))).cuda() for s in seqs]
           for k in range(FRAMES + 1)]
    torch.cuda.synchronize()
    a.first([s.frame(0) for s in seqs])
    b.first([s.frame(0) for s in seqs])
    for k in range(1, FRAMES + 1):  # no synchronise between the calls
        a.next_dev([t.data_ptr() for t in dev[k]], 0 if a.mixed else a.W)
    for k in range(1, FRAMES + 1):
        b.next([s.frame(k) for s in seqs])
    # after next(k) the previous-frame buffer (which = 0) holds frame k, the current one frame k - 1
    want = {0: _oracle_pyramids(orc, cfg, sizes, seqs, L, FRAMES),
            1: _oracle_pyramids(orc, cfg, sizes, seqs, L, FRAMES - 1)}
    for g, what in ((a, "next_dev"), (b, "next")):
        for c in range(len(sizes)):
            for which in (0, 1):
                for level in range(L):
                    try:
                        got = g.pyramid(c, which, level)
                    except api.CoslError:
                        assert level == 0, (what, c, which, level)  # a tracked frame may skip level 0
                        continue
                    ref = want[which][c][level]
                    assert got.shape == ref.shape, (what, c, which, level)
                    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (what, c, which, level)
    a.close()
    b.close()
