"""Cost of the KLT position covariances (cosl_klt_set_covariance) on the c3 rig.  Prints one JSON line (card name
and power limit included).

Two camera groups of bench.py's c3 geometry and tracker settings, one unarmed and one armed (noise_var 0: the
residual variance estimated per slot), fed the same frames.  Two paths, arms alternated over the rounds (round 0
is a warm-up):

  next_dev  --frames back-to-back cosl_klt_group_next_dev on frames resident in HBM, device-timed with CUDA
            events on the group's stream (bench.py's headline path); the armed group's covariances stay on the
            device, as its feature table does
  pipeline  cosl_klt_group_submit(n + 1) before cosl_klt_group_collect(n) from pinned host frames, host wall
            time of the loop; the armed group also reads back and hands out every frame's covariances
            (download_covariance after each collect)

Both groups' tables and counts of every pipelined frame are hashed; the arms must agree bit for bit.

  python tools/klt_cov_rig.py [--frames 200] [--rounds 5]"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)

ARMS = ("unarmed", "armed")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch
    from coslam_b200 import api
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    cfg = bench.klt_cfg()
    seqs = bench.make_sequences(0)
    fidx = seqs[0].frame_index
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory() for c in range(KC)] for k in range(bench.KLT_FRAMES)]
    dev = [[h.cuda() for h in row] for row in host]
    hnp = [[h.numpy() for h in row] for row in host]
    groups = {arm: api.KltGroup(cfg, KC, W, H, L, FW, FH, device=a.device) for arm in ARMS}
    groups["armed"].set_covariance(0.0)
    ptrs = [groups["unarmed"].host_ptrs(row) for row in hnp]
    n = a.frames

    def run_dev(g):
        g.first(hnp[0])
        for i in range(1, 4):  # warm-up
            g.next_dev([t.data_ptr() for t in dev[fidx(i)]], W)
        g.sync()
        stream = torch.cuda.ExternalStream(g.stream(), device=a.device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(4, 4 + n):
            g.next_dev([t.data_ptr() for t in dev[fidx(i)]], W)
        e1.record(stream)
        g.sync()
        return e0.elapsed_time(e1) / n

    def run_pipe(g, armed):
        g.first(hnp[0])
        digest = hashlib.sha256()
        g.sync()
        t0 = time.perf_counter()
        g.submit_raw(ptrs[fidx(1)])
        for i in range(2, n + 2):
            if i <= n:
                g.submit_raw(ptrs[fidx(i)])
            feats, counts = g.collect()
            if armed:
                g.download_covariance()
            digest.update(feats.tobytes())
            digest.update(counts.tobytes())
        dt = time.perf_counter() - t0
        return 1e3 * dt / n, digest.hexdigest()

    t_dev = {arm: [] for arm in ARMS}
    t_pipe = {arm: [] for arm in ARMS}
    digests = set()
    for r in range(a.rounds + 1):
        for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
            g = groups[arm]
            ms = run_dev(g)
            mp, dg = run_pipe(g, arm == "armed")
            digests.add(dg)
            if r:
                t_dev[arm].append(ms)
                t_pipe[arm].append(mp)
    cov = groups["armed"].download_covariance()
    for g in groups.values():
        g.close()
    live = np.isfinite(cov[..., 0])

    def summary(v):
        return {"ms_per_frame_set": float(np.median(v)), "range": [float(min(v)), float(max(v))]}

    dev_s = {arm: summary(t_dev[arm]) for arm in ARMS}
    pipe_s = {arm: summary(t_pipe[arm]) for arm in ARMS}
    cost = 1e3 * (dev_s["armed"]["ms_per_frame_set"] - dev_s["unarmed"]["ms_per_frame_set"])
    print(json.dumps({
        "metric": "armed_cost_us_per_frame_set", "value": cost, "unit": "us", "higher_is_better": False,
        "next_dev": dev_s, "pipeline": pipe_s,
        "pipeline_armed_cost_us": 1e3 * (pipe_s["armed"]["ms_per_frame_set"] - pipe_s["unarmed"]["ms_per_frame_set"]),
        "bit_identical_tables": len(digests) == 1,
        "covariances_per_frame_set": int(live.sum()),
        "median_xx_yy_px2": [float(np.median(cov[..., 0][live])), float(np.median(cov[..., 2][live]))],
        "config": {"workload": f"c3: {KC} cameras {W}x{H}, {FW}x{FH} slots, {n} frames per arm and round",
                   "rounds": a.rounds,
                   "timing": "next_dev: CUDA events on the group's stream; pipeline: host wall time of submit / "
                             "collect with two frames in flight; medians over the rounds"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
