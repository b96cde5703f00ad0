"""What the per-frame pose update costs the tracking thread: the blocking batch call against the pose solver
handle (cosl_pose_solver).  KLT frame sets of c3 (4 x 1280x720, live settings) go through
cosl_klt_group_submit_prefetched / _prefetch / _collect; after frame n's tables are back, the poses of frame n
are solved (4 cameras x 192 points of synth.make_pose_case, eight input sets in turn, default options, fresh
for every solve), then frame n+1 is prefetched and submitted.  Prints one JSON line (card name and power
limit included).

Arms, one frame loop each, alternated round by round (round 0 is a warm-up):
  none      no pose solve: the KLT frame set alone
  batch     cosl_pose_intracam_batch
  handle    cosl_pose_solver_submit, at once cosl_pose_solver_collect
  overlap   cosl_pose_solver_submit, then frame n+1's prefetch, then cosl_pose_solver_collect

Reported per arm (medians over the frames of the timed rounds):
  pose_host_us    host time blocked in the pose calls (batch; submit + collect)
  submit_us / collect_us   of which submit, collect
  device_ms       the handle's CUDA-event time of the copies and the kernel
  prefetch_us     host time of frame n+1's prefetch call (with a pose in flight in the overlap arm)
  frame_ms        host wall time per frame set: KLT collect, pose, prefetch, submit
Every arm's KLT tables and pose results (R, t, every option field, ok) are hashed per frame; the arms must agree
bit for bit.

  python tools/pose_solver_rig.py [--frames 200] [--rounds 3]"""
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

ARMS = ("none", "batch", "handle", "overlap")
N_SETS, N_PTS = 8, 192


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import PoseOpt

    if not torch.cuda.is_available():
        raise SystemExit("pose_solver_rig: needs a CUDA device")
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    seqs = bench.make_sequences(0)
    fidx = seqs[0].frame_index
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    grp = api.KltGroup(bench.klt_cfg(), KC, W, H, L, FW, FH, device=a.device)
    ptrs = [grp.host_ptrs(row) for row in host]
    solver = api.PoseSolver(a.device, KC, KC * N_PTS)
    LIB, ck = api.LIB, api._ck

    # pre-marshalled C-ABI arguments of the pose input sets: the timed calls are the library's alone
    sets = []
    for k in range(N_SETS):
        cases = [synth.make_pose_case(N_PTS, W, H, seed=300 + KC * k + c) for c in range(KC)]
        args, _, keep = api._pose_batch_args([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                                             [c[3] for c in cases], [c[4] for c in cases], 10.0, None, None)
        sets.append((args, keep))
    tmpl = (PoseOpt * KC)(*[PoseOpt.defaults() for _ in range(KC)])
    R, t, ok = np.empty((KC, 9)), np.empty((KC, 3)), np.zeros(KC, np.int32)
    dms = C.c_double(0)

    def run(arm):
        g = grp
        dest, cnt = g._dest, g.counts.ctypes.data
        frame_ptrs = [ptrs[fidx(i)] for i in range(a.frames + 1)]
        g.first(host[0])
        klt_digest, pose_digest = hashlib.sha256(), hashlib.sha256()
        rec = {k: [] for k in ("pose_host_us", "submit_us", "collect_us", "device_ms", "prefetch_us", "frame_ms")}
        ck(LIB.cosl_klt_group_prefetch(g.h, None, frame_ptrs[1][0], frame_ptrs[1][1]))
        ck(LIB.cosl_klt_group_submit_prefetched(g.h))
        torch.cuda.synchronize()
        for f in range(1, a.frames + 1):
            args = sets[f % N_SETS][0]
            opts = (PoseOpt * KC)()
            C.memmove(opts, tmpl, C.sizeof(tmpl))
            t0 = time.perf_counter()
            ck(LIB.cosl_klt_group_collect(g.h, dest, cnt))
            more = f < a.frames
            pf = 0.0
            if arm == "batch":
                t1 = time.perf_counter()
                ck(LIB.cosl_pose_intracam_batch(*args, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                a.device))
                rec["pose_host_us"].append(1e6 * (time.perf_counter() - t1))
            elif arm in ("handle", "overlap"):
                t1 = time.perf_counter()
                ck(LIB.cosl_pose_solver_submit(solver.h, *args, opts))
                t2 = time.perf_counter()
                if arm == "overlap" and more:
                    ck(LIB.cosl_klt_group_prefetch(g.h, None, frame_ptrs[f + 1][0], frame_ptrs[f + 1][1]))
                    pf = time.perf_counter() - t2
                t3 = time.perf_counter()
                ck(LIB.cosl_pose_solver_collect(solver.h, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                C.byref(dms)))
                t4 = time.perf_counter()
                rec["submit_us"].append(1e6 * (t2 - t1))
                rec["collect_us"].append(1e6 * (t4 - t3))
                rec["pose_host_us"].append(1e6 * ((t2 - t1) + (t4 - t3)))
                rec["device_ms"].append(dms.value)
            if more and arm != "overlap":
                t5 = time.perf_counter()
                ck(LIB.cosl_klt_group_prefetch(g.h, None, frame_ptrs[f + 1][0], frame_ptrs[f + 1][1]))
                pf = time.perf_counter() - t5
            if more:
                ck(LIB.cosl_klt_group_submit_prefetched(g.h))
                rec["prefetch_us"].append(1e6 * pf)
            rec["frame_ms"].append(1e3 * (time.perf_counter() - t0))
            klt_digest.update(g.feats.tobytes() + g.counts.tobytes())
            if arm != "none":
                pose_digest.update(R.tobytes() + t.tobytes() + ok.tobytes() + bytes(opts))
        return rec, klt_digest.hexdigest(), pose_digest.hexdigest()

    recs = {arm: [] for arm in ARMS}
    klt_digests, pose_digests = set(), set()
    for r in range(a.rounds + 1):
        for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
            rec, kd, pd = run(arm)
            klt_digests.add(kd)
            if arm != "none":
                pose_digests.add(pd)
            if r:
                recs[arm].append(rec)
    solver.close()
    grp.close()

    def med(arm, key):
        v = [x for rr in recs[arm] for x in rr[key]]
        return round(float(np.median(v)), 4) if v else None

    keys = ("pose_host_us", "submit_us", "collect_us", "device_ms", "prefetch_us", "frame_ms")
    print(json.dumps({
        "tool": "pose_solver_rig", "card": bench.gpu_identity(a.device),
        "workload": (f"c3 KLT frame sets (4 x {W}x{H}, {FW * FH} slots) through submit_prefetched / prefetch / "
                     f"collect; per frame one pose solve of {KC} cameras x {N_PTS} points"),
        "frames_per_arm": a.frames, "timed_rounds": a.rounds,
        **{arm: {k: med(arm, k) for k in keys} for arm in ARMS},
        "pose_bit_identical_across_arms": len(pose_digests) == 1,
        "klt_bit_identical_across_arms": len(klt_digests) == 1}))


if __name__ == "__main__":
    main()
