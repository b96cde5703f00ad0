"""The KLT detector link between two trackers on bench.py's c3 workload (4 x 1280x720, 2 000 slots per camera,
live settings, frames resident in HBM).  Prints one JSON line (card name and power limit included).

Frame n+1's tracker reads the feature set frame n's klt_select_refill writes, so every frame set runs the chain
tracker(n) -> klt_nm_verify(n) -> klt_select_refill(n) -> tracker(n+1).  The rig reports:

  selection   per camera over --count-frames synchronous next() calls: the raw candidate count nCand (counter
              [3]), the features the refill placed nSel (slots with status 1) and the live tracks before it
              nPresent (status 0), as median / min / max
  profile     device time per frame set of the klt_detect and klt_select profile classes (CUDA events around
              the prefilter + verify and around the select / refill), over --frames next_dev calls
  link_us     from a torch.profiler trace of --trace-frames next_dev calls: per frame set, the durations of
              verify and select and the gaps tracker end -> verify start -> (verify end) -> select start ->
              select end -> next tracker start, as medians (a negative gap: the kernel started before the one
              ahead of it ended, as a programmatic dependent launch may)
  device_ms   device time per frame set, profiler and profile classes off, over --frames next_dev calls

  python tools/klt_detector_link_rig.py OUT_DIR [--frames 200] [--trace-frames 40] [--count-frames 40]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)
from coslam_b200 import api  # noqa: E402


def kernels(trace, name):
    return sorted((e["ts"], e["ts"] + e["dur"]) for e in trace["traceEvents"]
                  if e.get("cat") == "kernel" and name in e.get("name", ""))


def link(track, verify, select):
    """Medians in us over the frame sets of the trace; the k-th launch of each kernel is frame k's."""
    n = min(len(track) - 1, len(verify), len(select))
    rows = []
    for k in range(n):
        rows.append({"tracker_end_to_verify_start": verify[k][0] - track[k][1],
                     "verify_dur": verify[k][1] - verify[k][0],
                     "verify_end_to_select_start": select[k][0] - verify[k][1],
                     "select_dur": select[k][1] - select[k][0],
                     "select_end_to_next_tracker_start": track[k + 1][0] - select[k][1],
                     "tracker_end_to_next_tracker_start": track[k + 1][0] - track[k][1]})
    if not rows:
        return {}
    out = {"frames": len(rows), **{k: round(float(np.median([r[k] for r in rows])), 2) for k in rows[0]}}
    # the part of the link the detector kernels and their two launch gaps hold
    out["verify_start_gap_plus_select"] = round(float(np.median(
        [r["tracker_end_to_verify_start"] + r["verify_end_to_select_start"] + r["select_dur"] for r in rows])), 2)
    return out


def stats(v):
    return {"median": float(np.median(v)), "min": int(np.min(v)), "max": int(np.max(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--trace-frames", type=int, default=40)
    ap.add_argument("--count-frames", type=int, default=40)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    C, W, H = bench.KLT_C, bench.KLT_W, bench.KLT_H
    seqs = bench.make_sequences(0)
    cfg, tracker = bench.klt_cfg(), "klt_gain_fused"
    grp = api.KltGroup(cfg, C, W, H, bench.KLT_L, bench.KLT_FW, bench.KLT_FH)
    stream = torch.cuda.ExternalStream(grp.stream())
    host = [[seqs[c].frames[k] for c in range(C)] for k in range(bench.KLT_FRAMES)]
    dev = [[torch.from_numpy(f).cuda() for f in row] for row in host]
    ptrs = [[t.data_ptr() for t in row] for row in dev]
    torch.cuda.synchronize()
    grp.first(host[0])
    fidx = seqs[0].frame_index
    i = 1

    def run(n):
        nonlocal i
        for _ in range(n):
            grp.next_dev(ptrs[fidx(i)], W)
            i += 1

    run(20)  # warm-up: the track counts settle within a few frames
    grp.sync()
    # selection counts: synchronous next() reads every camera's counters and table back
    n_cand, n_sel, n_pres = [[] for _ in range(C)], [[] for _ in range(C)], [[] for _ in range(C)]
    for _ in range(args.count_frames):
        feats, _ = grp.next(host[fidx(i)])
        i += 1
        for c in range(C):
            n_cand[c].append(api.LIB.cosl_klt_debug_num_candidates(grp.h, c))
            n_sel[c].append(int((feats[c]["status"] == 1).sum()))
            n_pres[c].append(int((feats[c]["status"] == 0).sum()))
    # device time, profiler and profile classes off
    run(10)
    grp.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run(args.frames)
    e1.record(stream)
    grp.sync()
    dev_ms = e0.elapsed_time(e1) / args.frames
    # profile classes (their CUDA events sit between the kernels, so this is a run of its own)
    grp.profile_enable(True)
    run(args.frames)
    grp.sync()
    prof = grp.profile()
    grp.profile_enable(False)
    classes = {k: {"us_per_frame_set": 1e3 * v[0] / max(1, v[1]), "calls": v[1]} for k, v in prof.items()
               if k in ("klt_detect", "klt_select")}
    # trace
    run(10)
    grp.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as p:
        run(args.trace_frames)
        grp.sync()
    path = os.path.join(args.out, "klt_detector_link.json")
    p.export_chrome_trace(path)
    trace = json.load(open(path))
    lk = link(kernels(trace, tracker), kernels(trace, "klt_nm_verify"), kernels(trace, "klt_select_refill"))
    grp.close()
    print(json.dumps({
        "metric": "klt_detector_link_us", "value": lk.get("verify_start_gap_plus_select"), "unit": "us",
        "higher_is_better": False,
        "selection": {"per_camera": [{"nCand": stats(n_cand[c]), "nSel": stats(n_sel[c]),
                                      "nPresent": stats(n_pres[c])} for c in range(C)],
                      "frames": args.count_frames, "slots_per_camera": bench.KLT_FW * bench.KLT_FH},
        "profile": classes,
        "link_us": lk,
        "device_ms_per_frame_set": dev_ms,
        "config": {"workload": f"c3: {C} cameras {W}x{H}, {bench.KLT_FW}x{bench.KLT_FH} slots, next_dev",
                   "frames": args.frames, "trace_frames": args.trace_frames},
        "trace": path,
        "gpu": bench.gpu_identity(torch.cuda.current_device())}))


if __name__ == "__main__":
    main()
