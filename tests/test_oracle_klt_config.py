"""The oracle's trackers against the float64 restatement (tests/klt_numpy.py) across the tracker
configurations of KLT_CONFIG_ROWS: window half-widths 1 to 15, level lists with and without level
0, 1 to 12 iterations, ITER5 on and off, elongated slot grids and a grid whose gain-neighbour
lookups land on slot boundaries.  CPU only; the GPU is held to the oracle on the same rows by
tests/test_gpu_klt_config.py.

Tolerances: measured, the oracle agrees with the restatement to <= 1.5e-5 px and <= 6e-7 in gain
with no status difference on every row.  They are set far below what the gain-neighbour table
changes: the table of a square grid applied to the 1x16 grid moves positions by 3.6e-4 px and gains
by 6.5e-5, so the usual 5e-3 px would not notice a wrong table."""
import numpy as np
import pytest

import klt_numpy as kn
from helpers import KLT_CONFIG_ROWS, row_cfg, seq

W, H = 192, 144
POS_TOL_PX, GAIN_TOL, MIN_AGREE = 1e-4, 1e-5, 0.99


def _two_frames(orc, row):
    """first + track on a seeded pair: the oracle's tracked table, its two pyramids (float64) and
    the first frame's positions (-1 for empty slots)."""
    s = seq(H, W, 29, n=2)
    cfg = row_cfg(row, 800.0)
    L = row.n_levels
    k = orc.OracleKlt(cfg, W, H, L, row.fw, row.fh)
    f0, _ = k.first(s.frames[0])
    f1, _ = k.track(s.frames[1])
    P0 = {l: k.pyramid(0, l).astype(np.float64) for l in range(L)}
    P1 = {l: k.pyramid(1, l).astype(np.float64) for l in range(L)}
    X0 = np.where((f0["status"] >= 0)[:, None], f0["pos"].astype(np.float64), -1.0)
    return cfg, f1, P0, P1, X0


def _restate(row, cfg, P0, P1, X0, nbr=None):
    args = dict(levels=kn.tracker_levels(row.n_levels, row.level_skip), hw=row.window // 2,
                conv=cfg.convergenceThreshold, ssd_thr=cfg.SSD_Threshold, margin=cfg.trackBorderMargin)
    if row.gain:
        return kn.track_gain(P0, P1, X0, W, H, row.fw, row.fh, n_iter=row.n_iter, nbr=nbr, **args)
    return kn.track_2x2(P0, P1, X0, W, H, n_iter=kn.iterations_2x2(row.n_iter, row.iter5), **args)


def _diff(f1, ref):
    """(status agreement, slots tracked by both, max |dpos| px, max |dgain|)"""
    o_ok, r_ok = f1["status"] == 0, ref[:, 0] >= 0
    both = o_ok & r_ok
    d = np.abs(f1["pos"][both].astype(np.float64) - ref[both, :2]) * [W, H]
    g = np.abs(f1["gain"][both].astype(np.float64) - ref[both, 2])
    return (o_ok == r_ok).mean(), int(both.sum()), float(d.max(initial=0)), float(g.max(initial=0))


def test_tracker_levels():
    """The level list, from the loops of klt_tracker.cg / v3d_gpuklt.cpp:254 and levelSkip <= 0 ->
    nLevels - 1 (v3d_gpuklt.h:14)."""
    assert kn.tracker_levels(6, 2) == [5, 3, 1]
    assert kn.tracker_levels(3, 2) == [2, 0]
    assert kn.tracker_levels(4, 1) == [3, 2, 1, 0]
    assert kn.tracker_levels(4, 3) == [3, 0]
    assert kn.tracker_levels(4, 5) == [3]
    assert kn.tracker_levels(5, 0) == [4, 0]
    assert kn.tracker_levels(1, 2) == [0]


def test_gain_neighbour_lookups():
    """klt_tracker_with_gain.cg:64-75 on the slot grids: square grids get the 8-neighbourhood with
    (+1, +1) twice; on elongated grids the diagonal lookups st0 +- ds0.x / ds0.y move one slot along
    one axis and a fraction of a slot along the other.  10x15 (fh / fw = 1.5) and 32x16 (0.5) put
    lookups exactly on slot boundaries; no other grid used in the tests does."""
    sq = kn.gain_neighbours(8, 8)
    i = 3 * 8 + 4
    assert list(sq[i]) == [i + 9, i - 9, i + 9, i - 9, i + 1, i - 1, i + 8, i - 8]
    wide = kn.gain_neighbours(32, 4)   # ds0.x = 1/32: a quarter of a row; ds0.y = 1/4: 8 columns
    i = 1 * 32 + 10
    assert list(wide[i]) == [i + 1, i - 1, 2 * 32 + 18, 0 * 32 + 2, i + 1, i - 1, i + 32, i - 32]
    assert len(kn.gain_lookup_ties(10, 15)) > 0 and len(kn.gain_lookup_ties(32, 16)) > 0
    for fw, fh in [(32, 32), (20, 12), (16, 16), (12, 12), (32, 4), (4, 64), (1, 16), (50, 40), (64, 64)]:
        assert kn.gain_lookup_ties(fw, fh) == [], (fw, fh)
    # on a tie the lookup takes the slot that starts at the boundary
    assert not np.array_equal(kn.gain_neighbours(10, 15), kn.gain_neighbours(10, 15, lower_on_tie=True))


@pytest.mark.parametrize("row", KLT_CONFIG_ROWS, ids=[r.id for r in KLT_CONFIG_ROWS])
def test_oracle_tracker_matches_restatement(orc, row):
    cfg, f1, P0, P1, X0 = _two_frames(orc, row)
    ref = _restate(row, cfg, P0, P1, X0)
    agree, both, dpos, dgain = _diff(f1, ref)
    print(f"{row.id}: agree {agree:.4f}, tracked by both {both}, max |dpos| {dpos:.2e} px, "
          f"max |dgain| {dgain:.2e}")
    assert agree >= MIN_AGREE and both >= 12, (agree, both)
    assert dpos < POS_TOL_PX and dgain < GAIN_TOL, (dpos, dgain)
    if row.gain and row.fw != row.fh:
        # the table of a square grid (the 8-neighbourhood) is visibly wrong on this grid
        fw, fh = row.fw, row.fh
        sy, sx = np.divmod(np.arange(fw * fh), fw)
        square = np.stack([np.clip(sy + oy, 0, fh - 1) * fw + np.clip(sx + ox, 0, fw - 1)
                           for ox, oy in [(1, 1), (-1, -1), (1, 1), (-1, -1), (1, 0), (-1, 0), (0, 1), (0, -1)]], 1)
        _, _, dpos2, dgain2 = _diff(f1, _restate(row, cfg, P0, P1, X0, nbr=square))
        assert dpos2 > POS_TOL_PX or dgain2 > GAIN_TOL, (dpos2, dgain2)
    if kn.gain_lookup_ties(row.fw, row.fh) and row.gain:
        # and so is the other tie convention (DESIGN.md section 2)
        alt = kn.gain_neighbours(row.fw, row.fh, lower_on_tie=True)
        _, _, dpos3, dgain3 = _diff(f1, _restate(row, cfg, P0, P1, X0, nbr=alt))
        assert dpos3 > POS_TOL_PX or dgain3 > GAIN_TOL, (dpos3, dgain3)
