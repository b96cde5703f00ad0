"""CoSLAM's multi-camera tracker cadence on c3 with the next frame set prefetched while the host maps.
Prints one JSON line (card name and power limit included).

The cadence of tools/klt_rig.py: first with 100 present points per camera, then 40 frames of next
through pinned host buffers, and after every 4th frame a feed of 100 points to cameras {0, 1} + an
advance of those two (CoSLAM::genNewMapPoints -> NewMapPtsNCC::output, app/SL_CoSLAM.cpp:1368-1371).
Three arms, one camera group each, alternated over the rounds (round 0 is a warm-up):

  sync      cosl_klt_group_next, then feed + advance_cams: every frame waits for the host's mapping
  prefetch  cosl_klt_group_prefetch(n+1) right after frame n's tables are back, then the mapping,
            then cosl_klt_group_run_prefetched: frame n+1's upload and pyramid run under the mapping
  submit    submit_prefetched(n), prefetch(n+1), collect(n), mapping, submit_prefetched(n+1)

--map-us stands in for the rest of CoSLAM's per-frame host work: a busy wait of that many
microseconds after each frame's tables are on the host, before the feed.  Every arm's tables and
counts of every frame are hashed; the arms must agree bit for bit.

  python tools/klt_prefetch_rig.py [--frames 40] [--feed-every 4] [--feed 100] [--rounds 3] [--map-us 0]"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)

ARMS = ("sync", "prefetch", "submit")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--feed-every", type=int, default=4)
    ap.add_argument("--feed", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--map-us", type=float, default=0.0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch
    from coslam_b200 import api, synth
    torch.cuda.set_device(a.device)
    n_frames, feed_every = a.frames, a.feed_every
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
    feeds = [[pts(a.feed), pts(a.feed)] + [None] * (KC - 2) for _ in range(n_frames // feed_every)]
    groups = {arm: api.KltGroup(cfg, KC, W, H, L, FW, FH, device=a.device) for arm in ARMS}
    args = [groups["sync"].host_ptrs(row) for row in host]  # pointer arrays, shared by the arms
    LIB, ck = api.LIB, api._ck

    def mapping(g, f, digest):
        digest.update(g.feats.tobytes())
        digest.update(g.counts.tobytes())
        t = time.perf_counter() + 1e-6 * a.map_us
        while time.perf_counter() < t:
            pass
        if f % feed_every == feed_every - 1:
            ids, fed = g.feed(feeds[f // feed_every])
            digest.update(b"".join(i.tobytes() for i in ids[:2]) + fed.tobytes())
            g.advance([0, 1])

    def run(arm):
        g = groups[arm]
        g.first(host[0], present=present)
        digest = hashlib.sha256()
        dest, cnt = g._dest, g.counts.ctypes.data
        ptrs = [args[fidx(i)] for i in range(1, n_frames + 1)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "sync":
            for f in range(n_frames):
                ck(LIB.cosl_klt_group_next(g.h, ptrs[f][0], ptrs[f][1], dest, cnt))
                mapping(g, f, digest)
        elif arm == "prefetch":
            ck(LIB.cosl_klt_group_prefetch(g.h, None, ptrs[0][0], ptrs[0][1]))
            for f in range(n_frames):
                ck(LIB.cosl_klt_group_run_prefetched(g.h, dest, cnt))
                if f + 1 < n_frames:
                    ck(LIB.cosl_klt_group_prefetch(g.h, None, ptrs[f + 1][0], ptrs[f + 1][1]))
                mapping(g, f, digest)
        else:
            ck(LIB.cosl_klt_group_prefetch(g.h, None, ptrs[0][0], ptrs[0][1]))
            ck(LIB.cosl_klt_group_submit_prefetched(g.h))
            for f in range(n_frames):
                if f + 1 < n_frames:
                    ck(LIB.cosl_klt_group_prefetch(g.h, None, ptrs[f + 1][0], ptrs[f + 1][1]))
                ck(LIB.cosl_klt_group_collect(g.h, dest, cnt))
                mapping(g, f, digest)
                if f + 1 < n_frames:
                    ck(LIB.cosl_klt_group_submit_prefetched(g.h))
        dt = time.perf_counter() - t0
        return dt, digest.hexdigest()

    times = {arm: [] for arm in ARMS}
    digests = set()
    for r in range(a.rounds + 1):
        for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
            dt, dg = run(arm)
            digests.add(dg)
            if r:
                times[arm].append(1e3 * dt / n_frames)
    for g in groups.values():
        g.close()

    def summary(v):
        return {"ms_per_frame_set": float(np.mean(v)), "ms_per_frame_set_range": [min(v), max(v)]}

    res = {arm: summary(times[arm]) for arm in ARMS}
    print(json.dumps({
        "metric": "ms_per_frame_set", "value": res["prefetch"]["ms_per_frame_set"], "unit": "ms",
        "higher_is_better": False, **res,
        "sync_over_prefetch": res["sync"]["ms_per_frame_set"] / res["prefetch"]["ms_per_frame_set"],
        "sync_over_submit": res["sync"]["ms_per_frame_set"] / res["submit"]["ms_per_frame_set"],
        "bit_identical_across_arms": len(digests) == 1,
        "config": {"workload": f"c3 rig cadence: first with 100 present points/cam, {n_frames} x next through "
                               f"pinned host buffers, every {feed_every}th frame feed {a.feed} points to cameras "
                               "{0, 1} + advance those two",
                   "map_us": a.map_us, "rounds": a.rounds,
                   "timing": "host wall time of the whole frame loop (ends with the last frame's tables on "
                             "the host), per frame set"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
