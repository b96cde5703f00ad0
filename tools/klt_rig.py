"""CoSLAM's multi-camera tracker cadence on c3, through one camera group and through 4 single-camera
trackers.  Prints one JSON line (card name and power limit included).

CoSLAM::initMapMultiCam seeds every camera's tracker with the existing map points (GPUKLT::first with
present points), featureTracking runs next() on every camera each frame, and NewMapPtsNCC::output feeds
new inter-camera points to the cameras of ONE CoSLAM camera group at most every 4th frame, each feed
followed by an advanceFrame (app/SL_CoSLAM.cpp:1368-1371).  Here: first with 100 present points per
camera, 40 frames of next through pinned host buffers, and on every 4th frame a feed of 100 points to
cameras {0, 1} + an advance of those two.  The group arm uses cosl_klt_group_first_present / _next /
_feed / _advance_cams; the singles arm is what a caller without those calls runs.  Round 0 of each arm
is a warm-up; the arms alternate.

  python tools/klt_rig.py [--frames 40] [--feed-every 4] [--feed 100] [--rounds 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--feed-every", type=int, default=4)
    ap.add_argument("--feed", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch
    from coslam_b200 import api, synth
    torch.cuda.set_device(a.device)
    n_frames, feed_every, n_fa = a.frames, a.feed_every, a.frames // a.feed_every
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    cfg = bench.klt_cfg()
    seqs = bench.make_sequences(0)
    fidx = seqs[0].frame_index
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    rng = np.random.default_rng(synth.BASE_SEED + 500)

    def pts(n):
        return np.stack([rng.uniform(0.02, 0.98, n), rng.uniform(0.02, 0.98, n), np.zeros(n)], 1).astype(np.float32)

    present = [pts(100) for _ in range(KC)]
    feeds = [[pts(a.feed), pts(a.feed)] for _ in range(n_fa)]
    grp = api.KltGroup(cfg, KC, W, H, L, FW, FH, device=a.device)
    stream = torch.cuda.ExternalStream(grp.stream(), device=a.device)
    grp_args = [grp.host_ptrs(row) for row in host]
    singles = [api.KltTracker(cfg, W, H, L, FW, FH, device=a.device) for _ in range(KC)]
    nb = C.c_int(0)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def group_round():
        grp.first([host[0][c] for c in range(KC)], present=present)
        t_fa, ex_ms, i = 0.0, 0.0, 1
        t0 = time.perf_counter()
        for f in range(n_frames):
            grp.next_raw(grp_args[fidx(i)])
            i += 1
            if f % feed_every == feed_every - 1:
                t = time.perf_counter()
                grp.feed(feeds[f // feed_every] + [None] * (KC - 2))
                ev0.record(stream)
                grp.advance([0, 1])
                ev1.record(stream)
                grp.sync()
                t_fa += time.perf_counter() - t
                ex_ms += ev0.elapsed_time(ev1)
        return time.perf_counter() - t0, t_fa, ex_ms, grp.feats.copy()

    def singles_round():
        for c in range(KC):
            singles[c].detect(host[0][c], present[c])
            singles[c].advance()
        t_fa, i = 0.0, 1
        t0 = time.perf_counter()
        for f in range(n_frames):
            row = host[fidx(i)]
            for c in range(KC):
                api._ck(api.LIB.cosl_klt_redetect(singles[c].h, row[c].ctypes.data, W, C.byref(singles[c].feats),
                                                  C.byref(nb)))
                api._ck(api.LIB.cosl_klt_advance(singles[c].h))
            i += 1
            if f % feed_every == feed_every - 1:
                t = time.perf_counter()
                for c in (0, 1):
                    singles[c].feed(feeds[f // feed_every][c])
                    singles[c].advance()
                    api._ck(api.LIB.cosl_klt_group_sync(singles[c].h))
                t_fa += time.perf_counter() - t
        return time.perf_counter() - t0, t_fa, 0.0, np.stack([s._out() for s in singles])

    res = {"group": [], "singles": []}
    same = True
    for r in range(a.rounds + 1):
        g = group_round()
        s = singles_round()
        same = same and g[3].tobytes() == s[3].tobytes()
        if r:
            res["group"].append(g[:3])
            res["singles"].append(s[:3])
    grp.close()
    for s in singles:
        s.close()

    def summary(rows, exchange):
        tot = [1e3 * t / n_frames for t, _, _ in rows]
        out = {"ms_per_frame_set": float(np.mean(tot)), "ms_per_frame_set_range": [min(tot), max(tot)],
               "feed_advance_ms_per_call": float(np.mean([1e3 * fa / n_fa for _, fa, _ in rows]))}
        if exchange:
            out["exchange_device_ms_per_call"] = float(np.mean([ex / n_fa for _, _, ex in rows]))
        return out

    gs, ss = summary(res["group"], True), summary(res["singles"], False)
    print(json.dumps({
        "metric": "ms_per_frame_set", "value": gs["ms_per_frame_set"], "unit": "ms", "higher_is_better": False,
        "group": gs, "singles": ss, "singles_over_group": ss["ms_per_frame_set"] / gs["ms_per_frame_set"],
        "bit_identical_to_singles": bool(same),
        "config": {"workload": f"c3 rig cadence: first with 100 present points/cam, {n_frames} x next through "
                               f"pinned host buffers, every {feed_every}th frame feed {a.feed} points to cameras "
                               "{0, 1} + advance those two; one camera group vs 4 single-camera trackers",
                   "rounds": a.rounds, "feed_frames": n_fa,
                   "singles": "per frame cosl_klt_redetect + cosl_klt_advance for each camera (one synchronise "
                              "each), called directly through ctypes",
                   "feed_advance": "host wall time of feed + advance + stream synchronise",
                   "exchange": "CUDA events around cosl_klt_group_advance_cams (pyramid slice exchange + "
                               "feature copy of 2 cameras)"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
