"""Independent numpy restatement of SURVEY.md Appendix A.1 / A.2 / A.6 (pyramid with derivatives,
[1 3 3 1] reduction, Shi-Tomasi cornerness, separable non-max suppression), written from the shader
formulas in float64 with np.pad(mode="edge") for CLAMP_TO_EDGE, against the C++ oracle.  A second
implementation in another language that agrees with the oracle to fp32 rounding is the strongest
pin available for the front end: the reference ships no golden vectors (parity unpinned).  The
restatement itself is tests/klt_numpy.py; tests/test_oracle_klt_config.py runs it across the
tracker configurations."""
import numpy as np
import pytest

from helpers import live_cfg, seq
from klt_numpy import cornerness, level0, nonmax_survivors, reduce1331, track_2x2, track_gain


@pytest.mark.parametrize("W,H,L", [(328, 250, 4), (97, 61, 3)])
def test_pyramid_matches_numpy_restatement(orc, W, H, L):
    s = seq(H, W, 13, n=1)
    k = orc.OracleKlt(live_cfg(), W, H, L, 4, 4)
    k.detect(s.frames[0])
    P = level0(s.frames[0])
    for l in range(L):
        got = k.pyramid(1, l).astype(np.float64)
        assert got.shape == P.shape
        assert np.abs(got - P).max() < 2e-4, f"level {l}: {np.abs(got - P).max()}"
        P = reduce1331(P)


def test_cornerness_and_nonmax_match_numpy_restatement(orc):
    W, H = 328, 250
    s = seq(H, W, 17, n=1)
    cfg = live_cfg(min_corner=1500.0)
    k = orc.OracleKlt(cfg, W, H, 3, 64, 64)   # 4096 slots: every candidate gets a slot
    feats, n = k.detect(s.frames[0])
    P0 = k.pyramid(1, 0).astype(np.float64)   # the oracle's own level 0 (pinned above)
    ref = cornerness(P0, 1500.0, 10.0, W, H)
    got = k.cornerness().astype(np.float64)
    # fp32 sums of ~49 products of magnitude up to 1e4: compare relative to the local scale
    scale = np.maximum(1.0, np.abs(ref) + 1500.0)
    assert (np.abs(got - ref) / scale).max() < 2e-5
    assert ((got > 0) == (ref > 0)).mean() > 0.9995      # threshold flips only at the margin of rounding
    surv = nonmax_survivors(got, cfg.minDistance)       # non-max on the oracle's own map: exact
    assert k.num_candidates() == int(surv.sum()) == n
    ys, xs = np.nonzero(surv)
    want = {(int(x), int(y)) for x, y in zip(xs, ys)}
    live = feats["status"] >= 0
    have = {(int(np.floor(px * W)), int(np.floor(py * H))) for px, py in feats["pos"][live]}
    assert have == want
    # strongest first
    cs = np.array([got[int(np.floor(py * H)), int(np.floor(px * W))] for px, py in feats["pos"][live]])
    assert np.all(np.diff(cs) <= 0)


def _two_frames(orc, gain, W=192, H=144, L=4, fw=8, fh=8):
    s = seq(H, W, 29, n=2)
    cfg = live_cfg(gain=gain, min_corner=800.0)
    cfg.nLevels = L
    k = orc.OracleKlt(cfg, W, H, L, fw, fh)
    f0, n0 = k.first(s.frames[0])
    f1, _ = k.track(s.frames[1])
    P0 = {l: k.pyramid(0, l).astype(np.float64) for l in range(L)}
    P1 = {l: k.pyramid(1, l).astype(np.float64) for l in range(L)}
    X0 = np.where((f0["status"] >= 0)[:, None], f0["pos"].astype(np.float64), -1.0)
    return cfg, f1, P0, P1, X0, n0


def _compare(f1, ref, W, H):
    o_ok, r_ok = f1["status"] == 0, ref[:, 0] >= 0
    assert (o_ok == r_ok).mean() >= 0.95, (o_ok.sum(), r_ok.sum())
    both = o_ok & r_ok
    assert both.sum() >= 20
    d = np.abs(f1["pos"][both].astype(np.float64) - ref[both, :2]) * [W, H]
    assert d.max() < 5e-3, d.max()
    return both


def test_2x2_tracker_matches_numpy_restatement(orc):
    W, H, L = 192, 144, 4
    cfg, f1, P0, P1, X0, n0 = _two_frames(orc, False, W, H, L)
    ref = track_2x2(P0, P1, X0, W, H, levels=[3, 1], n_iter=5, hw=3, conv=cfg.convergenceThreshold,
                    ssd_thr=cfg.SSD_Threshold, margin=cfg.trackBorderMargin)
    _compare(f1, ref, W, H)


def test_gain_tracker_matches_numpy_restatement(orc):
    W, H, L, fw, fh = 192, 144, 4, 8, 8
    cfg, f1, P0, P1, X0, n0 = _two_frames(orc, True, W, H, L, fw, fh)
    ref = track_gain(P0, P1, X0, W, H, fw, fh, levels=[3, 1], n_iter=cfg.nIterations, hw=3,
                     conv=cfg.convergenceThreshold, ssd_thr=cfg.SSD_Threshold, margin=cfg.trackBorderMargin)
    both = _compare(f1, ref, W, H)
    assert np.abs(f1["gain"][both] - ref[both, 2]).max() < 2e-3
