"""Shared helpers of the parity tests."""
import collections
import os
import subprocess
import tempfile

import numpy as np

from coslam_b200 import synth
from coslam_b200.ctypes_defs import COSL_KLT_COMPAT_ITER5, KltConfig


def ba_same_decisions(want, got, prob):
    """Two BA solves of `prob` (each (info, downloaded problem)) took the same decisions: info[5..10]
    (iterations, stop, nfev, njev, nlss, total trials) and [13] (outliers) equal; the solutions equal up to
    the order of the device's atomic sums; fixed parameters untouched; the second reports its device time."""
    (iw, pw), (ig, pg) = want, got
    assert np.array_equal(iw[5:11], ig[5:11]), (iw[:14], ig[:14])
    assert iw[13] == ig[13]
    assert np.array_equal(pw.outlier, pg.outlier)
    assert abs(iw[12] - ig[12]) <= 1e-9 * iw[12] + 1e-12
    assert np.abs(pw.R - pg.R).max() < 1e-9 and np.abs(pw.t - pg.t).max() < 1e-9
    if prob.n:
        assert np.abs(pw.X - pg.X).max() < 1e-8
    assert np.array_equal(pg.R[:prob.m_con], prob.R[:prob.m_con])
    assert np.array_equal(pg.t[:prob.m_con], prob.t[:prob.m_con])
    assert np.array_equal(pg.X[:prob.n_con], prob.X[:prob.n_con])
    assert ig[11] > 0


def live_cfg(gain=True, min_corner=3000.0):
    c = KltConfig.coslam_live(with_gain=gain)
    c.minCornerness = min_corner
    return c


KltRow = collections.namedtuple("KltRow", "id gain window n_levels level_skip n_iter iter5 fw fh")

# Tracker configurations beyond the live CoSLAM settings, one per code path of the trackers: window
# half-width 1, 2, 3, 4, 7 and 15, level lists with and without level 0 (levelSkip 0 = nLevels - 1),
# 1, 2, 5, 7, 8 and 12 iterations, ITER5 on and off, and slot grids whose gain-tracker wait sets
# overflow (32x4, 4x64, 1x16: the per-pass kernels run) or whose neighbour lookups land exactly on
# slot boundaries (10x15).  The ref_defaults rows are KLT_SequenceTrackerConfig()'s own defaults.
KLT_CONFIG_ROWS = [
    KltRow("ref_defaults", False, 5, 3, 2, 12, True, 32, 32),
    KltRow("ref_defaults_gain", True, 5, 3, 2, 12, False, 32, 32),
    KltRow("iter_exact", False, 5, 3, 2, 7, False, 32, 32),
    KltRow("hw1_every_level", True, 3, 4, 1, 12, False, 20, 12),
    KltRow("hw4_gain", True, 9, 5, 2, 12, False, 32, 32),
    KltRow("hw4_2x2", False, 9, 5, 2, 12, False, 32, 32),
    KltRow("hw7", True, 15, 4, 3, 8, False, 16, 16),
    KltRow("hw15_gain", True, 31, 3, 2, 5, False, 12, 12),
    KltRow("hw15_2x2", False, 31, 3, 2, 5, False, 12, 12),
    KltRow("one_iter", True, 6, 6, 2, 1, False, 32, 32),
    KltRow("two_iter", True, 6, 6, 2, 2, False, 32, 32),
    KltRow("top_only", True, 6, 4, 5, 12, False, 32, 32),
    KltRow("default_skip", True, 6, 5, 0, 12, False, 32, 32),
    KltRow("single_level_gain", True, 5, 1, 2, 12, False, 32, 32),
    KltRow("single_level_2x2", False, 5, 1, 2, 12, False, 32, 32),
    KltRow("wait_set_32x4", True, 6, 6, 2, 12, False, 32, 4),
    KltRow("wait_set_4x64", True, 6, 6, 2, 12, False, 4, 64),
    KltRow("wait_set_1x16", True, 6, 6, 2, 12, False, 1, 16),
    KltRow("texel_tie_10x15", True, 6, 6, 2, 12, False, 10, 15),
]


def row_cfg(row, min_corner):
    """The KltConfig of a KLT_CONFIG_ROWS row: the reference defaults' thresholds for ref_defaults*,
    the live CoSLAM thresholds otherwise."""
    c = KltConfig.reference_defaults() if row.id.startswith("ref_defaults") else KltConfig.coslam_live()
    c.trackWithGain = int(row.gain)
    c.windowWidth = row.window
    c.nLevels = row.n_levels
    c.levelSkip = row.level_skip
    c.nIterations = row.n_iter
    c.compat = COSL_KLT_COMPAT_ITER5 if row.iter5 else 0
    c.minCornerness = min_corner
    return c


def seq(h, w, seed, n=4, **kw):
    return synth.ImageSequence(h, w, seed, n_frames=n, **kw)


def compare_features(fa, fb, W, H, pos_tol_px=2e-3, gain_tol=1e-3, max_flip_frac=0.002):
    """Compare two cosl_klt_feature tables (oracle vs CUDA).  Returns dict of statistics and raises
    on violation.  Status flips are allowed for a small fraction of slots (threshold decisions on
    fp32 sums that are reduced in a different order on the GPU).  The defaults allow 2e-3 px on the
    position and at most max(1, 0.2 %) of the slots for a threshold decision."""
    assert len(fa) == len(fb)
    sa, sb = fa["status"], fb["status"]
    flips = sa != sb
    n = len(fa)
    both = (~flips) & (sa >= 0)
    d = np.abs(fa["pos"][both] - fb["pos"][both]) * np.array([W, H], np.float32)
    dmax = float(d.max()) if d.size else 0.0
    tr = (~flips) & (sa == 0)
    gmax = float(np.abs(fa["gain"][tr] - fb["gain"][tr]).max()) if tr.any() else 0.0
    stats = dict(n=n, flips=int(flips.sum()), pos_max_px=dmax, gain_max=gmax)
    assert flips.sum() <= max(1, int(max_flip_frac * n)), stats
    assert dmax <= pos_tol_px, stats
    assert gmax <= gain_tol, stats
    return stats


def pose_inputs():
    """The 40 seeded intraCamEstimate cases: (K, R0, t0, Ms, ms, tau, prev_errs)."""
    rng = np.random.default_rng(2024)
    for k in range(40):
        n = int(rng.integers(6, 193))
        K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n_pts=n, seed=300 + k,
                                                       outlier_frac=float(rng.uniform(0, 0.25)),
                                                       rot_deg=float(rng.uniform(0.1, 3.0)),
                                                       trans=float(rng.uniform(0.01, 0.2)))
        pe = np.abs(rng.normal(0, 4, n)) if k % 3 == 0 else None
        tau = float(rng.choice([6.0, 10.0, 20.0]))
        yield K, R0, t0, Ms, ms, tau, pe


def so3_inputs():
    rng = np.random.default_rng(5)
    return [np.ascontiguousarray(w) for w in list(rng.normal(0, 1, (20, 3))) + [np.zeros(3), np.array([1e-8, 0, 0])]]


def posegraph_inputs():
    """The 12 seeded chains: (fixed, R, t, id1, id2, eR_list, et_list)."""
    for seed in range(12):
        g = synth.make_pose_chains([10 + 7 * seed], key_every=3 + seed % 6, seed=100 + seed, lead_free=seed % 3,
                                   shift=0.02 * (1 + seed % 4))
        yield g["fixed"], g["R"], g["t"], g["id1"], g["id2"], g["eR_list"], g["et_list"]


def run_facade_caller(exe, frames, W, H, gain, feed_every):
    """Runs oracle/_ref/gpuklt_ref_caller (the reference's GPUKLT facade on the shim) on the frames.
    Returns {"F": rows (frame, slot, track length, x, y), "N": rows (frame, count), "X": rows (frame,
    externally fed points that found a slot)} as float64 arrays."""
    with tempfile.TemporaryDirectory() as d:
        raw = os.path.join(d, "frames.raw")
        with open(raw, "wb") as f:
            f.write(np.stack(frames).astype(np.uint8).tobytes())
        out = subprocess.run([exe, raw, str(W), str(H), str(len(frames)), str(int(gain)), str(feed_every)],
                             capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    rows = {"F": [], "N": [], "X": []}
    for line in out.stdout.splitlines():
        p = line.split()
        if p and p[0] in rows:
            rows[p[0]].append([float(v) for v in p[1:]])
    return {k: np.asarray(v, np.float64).reshape(-1, 5 if k == "F" else 2) for k, v in rows.items()}
