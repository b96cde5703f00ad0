"""What the pose graph costs the SLAM thread: the blocking calls against the pose-graph solver handle
(cosl_posegraph_solver).  Prints one JSON line (card name and power limit included).

Leg 1, post-BA shape.  KLT frame sets of c3 (4 x 1280x720, live settings) go through
cosl_klt_group_submit_prefetched / _prefetch / _collect; after every 10th frame set's tables are back there is
one chain spread (synth.make_pose_chains, key frame every 20; shapes 4 x 150 and 8 x 4 000 nodes, each in a loop
of its own), then frame n+1 is prefetched and submitted.  Arms, one frame loop each, alternated round by round
(round 0 is a warm-up):
  sync      cosl_posegraph_spread_chains
  handle    cosl_posegraph_solver_submit_chains, at once cosl_posegraph_solver_collect
  overlap   submit_chains, then frame n+1's prefetch, then collect
Reported per shape and arm (medians over the spreads of the timed rounds):
  blocked_us        host time blocked in the spread calls (sync; submit + collect)
  submit_us / collect_us   of which submit, collect
  device_ms         the handle's CUDA-event time of the copies and the kernel
  frame_ms          host wall time of a frame set that carries a spread: KLT collect, spread, prefetch, submit
  frame_ms_plain    the same for the frame sets without one
Every arm's spread results and KLT tables are hashed; the arms must agree bit for bit.

Leg 2, merge graphs.  synth.make_merge_graph(100, C, n_constraints=2, n_scale_ids=1, noise=0.01) for C = 4, 8, 13;
the blocking cosl_posegraph_solve and submit + collect on one handle alternate, medians of --merge-reps each after
a warm-up: sync_ms (the whole call), submit_ms (host time of submit), collect_ms (time blocked in collect),
device_ms, and whether the results are bit-identical.

  python tools/posegraph_solver_rig.py [--frames 200] [--rounds 3] [--merge-reps 20]"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)

ARMS = ("sync", "handle", "overlap")
SHAPES = {"4x150": [150] * 4, "8x4000": [4000] * 8}
EVERY = 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--merge-reps", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth

    if not torch.cuda.is_available():
        raise SystemExit("posegraph_solver_rig: needs a CUDA device")
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    seqs = bench.make_sequences(0)
    fidx = seqs[0].frame_index
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    grp = api.KltGroup(bench.klt_cfg(), KC, W, H, L, FW, FH, device=a.device)
    ptrs = [grp.host_ptrs(row) for row in host]
    solver = api.PoseGraphSolver(a.device)
    LIB, ck = api.LIB, api._ck
    dms = C.c_double(0)

    def leg1(shape):
        # pre-marshalled C-ABI arguments: the timed calls are the library's alone
        g = synth.make_pose_chains(SHAPES[shape], key_every=20, seed=77, shift=0.05)
        args, N, _keep = api._chain_args(g["chain_off"], g["fixed"], g["R"], g["t"], g["eR"], g["et"])
        nR, nt = np.empty((N, 3, 3)), np.empty((N, 3))

        def run(arm):
            dest, cnt = grp._dest, grp.counts.ctypes.data
            frame_ptrs = [ptrs[fidx(i)] for i in range(a.frames + 1)]
            grp.first(host[0])
            klt_digest, pg_digest = hashlib.sha256(), hashlib.sha256()
            rec = {k: [] for k in ("blocked_us", "submit_us", "collect_us", "device_ms", "frame_ms", "frame_ms_plain")}
            ck(LIB.cosl_klt_group_prefetch(grp.h, None, frame_ptrs[1][0], frame_ptrs[1][1]))
            ck(LIB.cosl_klt_group_submit_prefetched(grp.h))
            torch.cuda.synchronize()
            for f in range(1, a.frames + 1):
                t0 = time.perf_counter()
                ck(LIB.cosl_klt_group_collect(grp.h, dest, cnt))
                more = f < a.frames
                spread = f % EVERY == 0
                prefetched = False
                if spread and arm == "sync":
                    t1 = time.perf_counter()
                    ck(LIB.cosl_posegraph_spread_chains(*args, nR.ctypes.data, nt.ctypes.data, a.device))
                    rec["blocked_us"].append(1e6 * (time.perf_counter() - t1))
                elif spread:
                    t1 = time.perf_counter()
                    ck(LIB.cosl_posegraph_solver_submit_chains(solver.h, *args))
                    t2 = time.perf_counter()
                    if arm == "overlap" and more:
                        ck(LIB.cosl_klt_group_prefetch(grp.h, None, frame_ptrs[f + 1][0], frame_ptrs[f + 1][1]))
                        prefetched = True
                    t3 = time.perf_counter()
                    ck(LIB.cosl_posegraph_solver_collect(solver.h, nR.ctypes.data, nt.ctypes.data, None,
                                                         C.byref(dms)))
                    t4 = time.perf_counter()
                    rec["submit_us"].append(1e6 * (t2 - t1))
                    rec["collect_us"].append(1e6 * (t4 - t3))
                    rec["blocked_us"].append(1e6 * ((t2 - t1) + (t4 - t3)))
                    rec["device_ms"].append(dms.value)
                if more and not prefetched:
                    ck(LIB.cosl_klt_group_prefetch(grp.h, None, frame_ptrs[f + 1][0], frame_ptrs[f + 1][1]))
                if more:
                    ck(LIB.cosl_klt_group_submit_prefetched(grp.h))
                rec["frame_ms" if spread else "frame_ms_plain"].append(1e3 * (time.perf_counter() - t0))
                klt_digest.update(grp.feats.tobytes() + grp.counts.tobytes())
                if spread:
                    pg_digest.update(nR.tobytes() + nt.tobytes())
            return rec, klt_digest.hexdigest(), pg_digest.hexdigest()

        recs = {arm: [] for arm in ARMS}
        klt_digests, pg_digests = set(), set()
        for r in range(a.rounds + 1):
            for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
                rec, kd, pd = run(arm)
                klt_digests.add(kd)
                pg_digests.add(pd)
                if r:
                    recs[arm].append(rec)

        def med(arm, key):
            v = [x for rr in recs[arm] for x in rr[key]]
            return round(float(np.median(v)), 4) if v else None

        keys = ("blocked_us", "submit_us", "collect_us", "device_ms", "frame_ms", "frame_ms_plain")
        return {"nodes": N, **{arm: {k: med(arm, k) for k in keys} for arm in ARMS},
                "spread_bit_identical_across_arms": len(pg_digests) == 1,
                "klt_bit_identical_across_arms": len(klt_digests) == 1}

    def leg2(cams):
        g = synth.make_merge_graph(100, cams, seed=100 * cams, n_constraints=2, n_scale_ids=1, noise=0.01)
        args, n, _keep = api._graph_args(g["fixed"], g["R"], g["t"], g["id1"], g["id2"], g["eR"], g["et"],
                                         g["scale_col"], g["n_scale"])
        ns = int(g["n_scale"])
        out = {k: (np.empty((n, 3, 3)), np.empty((n, 3)), np.empty(max(1, ns))) for k in ("sync", "handle")}
        rec = {k: [] for k in ("sync_ms", "submit_ms", "collect_ms", "device_ms")}
        same = True
        for rep in range(a.merge_reps + 2):
            nR, nt, s = out["sync"]
            t0 = time.perf_counter()
            ck(LIB.cosl_posegraph_solve(*args, nR.ctypes.data, nt.ctypes.data, s.ctypes.data, a.device))
            t1 = time.perf_counter()
            hR, ht, hs = out["handle"]
            ck(LIB.cosl_posegraph_solver_submit(solver.h, *args))
            t2 = time.perf_counter()
            ck(LIB.cosl_posegraph_solver_collect(solver.h, hR.ctypes.data, ht.ctypes.data, hs.ctypes.data,
                                                 C.byref(dms)))
            t3 = time.perf_counter()
            same &= all(np.array_equal(x.view(np.uint64), y.view(np.uint64))
                        for x, y in zip((nR, nt, s[:ns]), (hR, ht, hs[:ns])))
            if rep >= 2:
                rec["sync_ms"].append(1e3 * (t1 - t0))
                rec["submit_ms"].append(1e3 * (t2 - t1))
                rec["collect_ms"].append(1e3 * (t3 - t2))
                rec["device_ms"].append(dms.value)
        return {"nodes": n, "edges": int(len(g["id1"])), **{k: round(float(np.median(v)), 4) for k, v in rec.items()},
                "bit_identical": bool(same)}

    spreads = {shape: leg1(shape) for shape in SHAPES}
    merges = {f"C={cams}": leg2(cams) for cams in (4, 8, 13)}
    solver.close()
    grp.close()
    print(json.dumps({
        "tool": "posegraph_solver_rig", "card": bench.gpu_identity(a.device),
        "leg1": {"workload": (f"c3 KLT frame sets (4 x {W}x{H}, {FW * FH} slots) through submit_prefetched / "
                              f"prefetch / collect; every {EVERY}th frame set one chain spread (key frame every 20)"),
                 "frames_per_arm": a.frames, "timed_rounds": a.rounds, **spreads},
        "leg2": {"workload": "make_merge_graph(100 key frames, C cameras, 2 constraint edges, one scale)",
                 "reps": a.merge_reps, **merges}}))


if __name__ == "__main__":
    main()
