"""A c3-like rig whose cameras differ in size (2 x 1280x720 + 2 x 640x480, 50 x 40 = 2000 slots, live
settings), tracked three ways: one mixed camera group (cosl_klt_group_create_sizes), one group per
size, and four single-camera trackers.  Each round runs first, then --frames frames of next through
pinned host buffers; round 0 of each arm is a warm-up and the arms alternate.  The three arms must
produce identical feature tables.  Prints one JSON line (card name and power limit included).

  python tools/klt_mixed_rig.py [--frames 60] [--rounds 3]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (tracker settings, card identity)

SIZES = [(1280, 720), (1280, 720), (640, 480), (640, 480)]
FW, FH, L, N_SEQ = 50, 40, 6, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch
    from coslam_b200 import api, synth
    torch.cuda.set_device(a.device)
    KC = len(SIZES)
    cfg = bench.klt_cfg()
    seqs = [synth.ImageSequence(h, w, synth.BASE_SEED + 700 + c, n_frames=N_SEQ) for c, (w, h) in enumerate(SIZES)]
    # frames 0, 1, ..., N-1, N-2, ..., 1, 0, 1, ...: the motion stays smooth over any number of frames
    cyc = list(range(N_SEQ)) + list(range(N_SEQ - 2, 0, -1))
    fidx = lambda i: cyc[i % len(cyc)]  # noqa: E731
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)] for k in range(N_SEQ)]

    mixed = api.KltGroup(cfg, KC, [w for w, _ in SIZES], [h for _, h in SIZES], L, FW, FH, device=a.device)
    mixed_args = [mixed.host_ptrs(row) for row in host]
    by_size = [(api.KltGroup(cfg, 2, w, h, L, FW, FH, device=a.device), cams)
               for (w, h), cams in (((1280, 720), [0, 1]), ((640, 480), [2, 3]))]
    by_size_args = [[g.host_ptrs([row[c] for c in cams]) for row in host] for g, cams in by_size]
    singles = [api.KltTracker(cfg, w, h, L, FW, FH, device=a.device) for w, h in SIZES]
    nb = C.c_int(0)

    def mixed_round():
        mixed.first(host[0])
        t0 = time.perf_counter()
        for i in range(1, a.frames + 1):
            mixed.next_raw(mixed_args[fidx(i)])
        return time.perf_counter() - t0, mixed.feats.copy()

    def by_size_round():
        for g, cams in by_size:
            g.first([host[0][c] for c in cams])
        t0 = time.perf_counter()
        for i in range(1, a.frames + 1):
            for k, (g, _) in enumerate(by_size):
                g.next_raw(by_size_args[k][fidx(i)])
        t = time.perf_counter() - t0
        out = np.zeros_like(mixed.feats)
        for g, cams in by_size:
            out[cams] = g.feats
        return t, out

    def singles_round():
        for c in range(KC):
            singles[c].first(host[0][c])
        t0 = time.perf_counter()
        for i in range(1, a.frames + 1):
            row = host[fidx(i)]
            for c in range(KC):
                api._ck(api.LIB.cosl_klt_redetect(singles[c].h, row[c].ctypes.data, SIZES[c][0],
                                                  C.byref(singles[c].feats), C.byref(nb)))
                api._ck(api.LIB.cosl_klt_advance(singles[c].h))
        return time.perf_counter() - t0, np.stack([s._out() for s in singles])

    arms = {"mixed_group": mixed_round, "group_per_size": by_size_round, "singles": singles_round}
    res = {k: [] for k in arms}
    same = True
    for r in range(a.rounds + 1):
        outs = {}
        for k, fn in arms.items():
            t, outs[k] = fn()
            if r:
                res[k].append(1e3 * t / a.frames)
        same = same and all(outs[k].tobytes() == outs["mixed_group"].tobytes() for k in arms)
    mixed.close()
    for g, _ in by_size:
        g.close()
    for s in singles:
        s.close()

    summ = {k: {"ms_per_frame_set": float(np.mean(v)), "ms_per_frame_set_range": [min(v), max(v)]}
            for k, v in res.items()}
    print(json.dumps({
        "metric": "ms_per_frame_set", "value": summ["mixed_group"]["ms_per_frame_set"], "unit": "ms",
        "higher_is_better": False, **summ,
        "group_per_size_over_mixed": summ["group_per_size"]["ms_per_frame_set"] / summ["mixed_group"]["ms_per_frame_set"],
        "singles_over_mixed": summ["singles"]["ms_per_frame_set"] / summ["mixed_group"]["ms_per_frame_set"],
        "identical_tables": bool(same),
        "config": {"workload": f"2 x 1280x720 + 2 x 640x480, {FW}x{FH} slots, {L} levels, live settings; first, then "
                               f"{a.frames} x next through pinned host buffers",
                   "rounds": a.rounds,
                   "group_per_size": "two 2-camera groups, cosl_klt_group_next on each (one synchronise each)",
                   "singles": "per frame cosl_klt_redetect + cosl_klt_advance for each camera (one synchronise "
                              "each), called directly through ctypes"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
