"""torch.profiler trace of back-to-back KLT frames (bench.py's c3 workload, frames resident in HBM).

  python tools/klt_overlap_trace.py OUT_DIR [--frames 20] [--no-gain]

Writes OUT_DIR/klt_next_dev.json (Chrome trace) and prints, per frame pair, whether frame n+1's
klt_front overlaps frame n's klt_nm_verify / klt_select_refill, the device time per frame, the host
time to enqueue one cosl_klt_group_next_dev call (measured without the profiler) and the split of
the pyramid chain into kernels and the gaps between them (chain_split), and how far each front pass
runs ahead of the tracker before it (lookahead).  The host must
enqueue a frame faster than the device runs it, or the queue drains and the overlap is lost."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from coslam_b200 import api  # noqa: E402


def kernels(trace, name):
    return sorted((e["ts"], e["ts"] + e["dur"]) for e in trace["traceEvents"]
                  if e.get("cat") == "kernel" and name in e.get("name", ""))


def chain_split(front, pyr, track):
    """Median per frame, in us, of the pyramid chain klt_front -> klt_pyr_down_tma x (L - 2) -> tracker
    on the device timeline: the gap from the front pass's end to the first level's start, each
    level's duration and the gap before the next, the tail (front pass end to last level end) and
    the gap from the tail's end to the tracker's start.  A programmatic dependent launch starts
    before the kernel ahead of it ends, so its gap can be negative and its duration includes the
    wait."""
    rows = []
    for k, (f0, f1) in enumerate(front):
        nxt = front[k + 1][0] if k + 1 < len(front) else float("inf")
        lv = [p for p in pyr if f0 <= p[0] < nxt]
        tr = [t for t in track if t[0] >= f1]
        if not lv or not tr:
            continue
        r = {"front_to_level2_gap": lv[0][0] - f1, "tail": lv[-1][1] - f1,
             "tail_to_tracker_gap": tr[0][0] - lv[-1][1]}
        for i, (a, b) in enumerate(lv):
            r[f"level{i + 2}_dur"] = b - a
            if i + 1 < len(lv):
                r[f"level{i + 2}_to_{i + 3}_gap"] = lv[i + 1][0] - b
        rows.append(r)
    if not rows:
        return {}
    keys = [k for k in rows[0] if all(k in r for r in rows)]
    return {"frames": len(rows), **{k: round(float(np.median([r[k] for r in rows])), 2) for k in keys}}


def lookahead(front, pyr, track, verify, select, n_levels):
    """Per frame pair (n, n+1), from the k-th launch of each kernel being frame k's: whether front(n+1)
    starts before tracker(n) does, the detector span (klt_nm_verify start -> klt_select_refill end)
    of frame n and front(n+1)'s duration, the time from tail(n+1)'s end to tracker(n)'s end (> 0: the
    tail is done before the next tracker can start) and from tracker(n)'s end to tracker(n+1)'s start.
    Medians in us, and the count of frame pairs where front(n+1) runs ahead.  With fewer than 3
    levels there is no tail kernel and the front pass's end stands for the tail's."""
    per = n_levels - 2
    tails = [pyr[i + per - 1] for i in range(0, len(pyr) - per + 1, per)] if per > 0 else front
    n = min(len(front), len(track), len(verify), len(select), len(tails))
    rows, ahead = [], 0
    for k in range(n - 1):
        ahead += front[k + 1][0] < track[k][0]
        rows.append({"detector_span": select[k][1] - verify[k][0], "front_dur": front[k + 1][1] - front[k + 1][0],
                     "tail_end_to_tracker_end": track[k][1] - tails[k + 1][1],
                     "tracker_end_to_next_tracker_start": track[k + 1][0] - track[k][1]})
    if not rows:
        return {}
    return {"front_ahead_of_tracker": f"{ahead} of {len(rows)} frame pairs",
            **{k: round(float(np.median([r[k] for r in rows])), 2) for k in rows[0]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--no-gain", action="store_true", help="the 2x2 tracker (bench.py's klt_2x2 line)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    C, W, H = bench.KLT_C, bench.KLT_W, bench.KLT_H
    seqs = bench.make_sequences(0)
    if args.no_gain:
        from coslam_b200.ctypes_defs import KltConfig
        cfg, tracker = KltConfig.coslam_live(with_gain=False), "klt_track_2x2"
    else:
        cfg, tracker = bench.klt_cfg(), "klt_gain_fused"
    grp = api.KltGroup(cfg, C, W, H, bench.KLT_L, bench.KLT_FW, bench.KLT_FH)
    stream = torch.cuda.ExternalStream(grp.stream())
    dev = [[torch.from_numpy(seqs[c].frames[k]).cuda() for c in range(C)] for k in range(bench.KLT_FRAMES)]
    ptrs = [[t.data_ptr() for t in row] for row in dev]
    torch.cuda.synchronize()
    grp.first([seqs[c].frames[0] for c in range(C)])
    fidx = seqs[0].frame_index
    i = 1

    def run(n, host_times=None):
        nonlocal i
        for _ in range(n):
            t0 = time.perf_counter()
            grp.next_dev(ptrs[fidx(i)], W)
            if host_times is not None:
                host_times.append(time.perf_counter() - t0)
            i += 1

    run(10)
    grp.sync()
    # device time per frame, profiler off
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run(200)
    e1.record(stream)
    grp.sync()
    dev_ms = e0.elapsed_time(e1) / 200
    # host enqueue time, in bursts of 8 calls from an idle queue: in a long run the host gets ahead of
    # the device until the launch queue is full, and from then on each call waits for a frame to finish
    host = []
    for _ in range(25):
        run(8, host)
        grp.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        run(args.frames)
        grp.sync()
    path = os.path.join(args.out, "klt_next_dev.json")
    prof.export_chrome_trace(path)
    trace = json.load(open(path))
    front, verify, select = (kernels(trace, k) for k in ("klt_front", "klt_nm_verify", "klt_select_refill"))
    n = min(len(front), len(verify), len(select))
    overl = 0
    for k in range(n - 1):
        f0, f1 = front[k + 1]
        ov = any(f0 < b and a < f1 for a, b in (verify[k], select[k]))
        overl += ov
    print(json.dumps({
        "gpu": bench.gpu_identity(torch.cuda.current_device()),
        "frames_traced": n,
        "front_overlaps_previous_detector": f"{overl} of {n - 1} frame pairs",
        "device_ms_per_frame": dev_ms,
        "host_enqueue_ms_per_call": {"median": 1e3 * float(np.median(host)), "p90": 1e3 * float(np.percentile(host, 90))},
        "pyramid_chain_us": chain_split(front, kernels(trace, "klt_pyr_down_tma"), kernels(trace, tracker)),
        "lookahead_us": lookahead(front, kernels(trace, "klt_pyr_down_tma"), kernels(trace, tracker), verify, select,
                                  bench.KLT_L),
        "trace": path}))
    grp.close()


if __name__ == "__main__":
    main()
