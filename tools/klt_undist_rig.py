"""Cost of the KLT undistortion stage (cosl_klt_set_undistortion) on the c3 rig.  Prints one JSON line (card name
and power limit included).

Three camera groups of bench.py's c3 geometry and tracker settings fed the same frames: unarmed, undistortion
armed, and undistortion plus position covariances armed (noise_var 0).  Each camera gets its own lens (a mild
and a strong barrel, a pincushion with tangential terms, and one with skew).  Two paths, arms alternated over
the rounds (round 0 is a warm-up):

  next_dev  --frames back-to-back cosl_klt_group_next_dev on frames resident in HBM, device-timed with CUDA
            events on the group's stream (bench.py's headline path); the armed groups' results stay on the
            device, as the feature table does
  pipeline  cosl_klt_group_submit(n + 1) before cosl_klt_group_collect(n) from pinned host frames, host wall
            time of the loop; the armed groups also read back and hand out every frame's undistorted positions
            (and covariances) with download_undistorted after each collect

Every group's tables and counts of every pipelined frame are hashed; the arms must agree bit for bit.

  python tools/klt_undist_rig.py [--frames 200] [--rounds 5]"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)
import undist_dense as U  # noqa: E402  (the lenses)

ARMS = ("unarmed", "undist", "undist_cov")


def lenses(n, W, H):
    names = list(U.CALIBS)
    Ks, kcs = [], []
    for c in range(n):
        K0, kc, W0, H0 = U.CALIBS[names[c % len(names)]]
        Ks.append(np.diag([W / W0, H / H0, 1.0]) @ K0)
        kcs.append(kc)
    return np.array(Ks), np.array(kcs)


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
    Ks, kcs = lenses(KC, W, H)
    groups["undist"].set_undistortion(Ks, kcs)
    groups["undist_cov"].set_undistortion(Ks, kcs)
    groups["undist_cov"].set_covariance(0.0)
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
                g.download_undistorted()
            digest.update(feats.tobytes())
            digest.update(counts.tobytes())
        dt = time.perf_counter() - t0
        return 1e3 * dt / n, digest.hexdigest()

    t_dev = {arm: [] for arm in ARMS}
    t_pipe = {arm: [] for arm in ARMS}
    digests = set()
    for r in range(a.rounds + 1):
        order = ARMS[r % 3:] + ARMS[:r % 3]
        for arm in (order if r % 2 == 0 else order[::-1]):
            g = groups[arm]
            ms = run_dev(g)
            mp, dg = run_pipe(g, arm != "unarmed")
            digests.add(dg)
            if r:
                t_dev[arm].append(ms)
                t_pipe[arm].append(mp)
    pos, ucov = groups["undist_cov"].download_undistorted()
    for g in groups.values():
        g.close()
    live = np.isfinite(pos[..., 0])

    def summary(v):
        return {"ms_per_frame_set": float(np.median(v)), "range": [float(min(v)), float(max(v))]}

    dev_s = {arm: summary(t_dev[arm]) for arm in ARMS}
    pipe_s = {arm: summary(t_pipe[arm]) for arm in ARMS}

    def cost(s, arm):
        return 1e3 * (s[arm]["ms_per_frame_set"] - s["unarmed"]["ms_per_frame_set"])

    print(json.dumps({
        "metric": "undist_cost_us_per_frame_set", "value": cost(dev_s, "undist"), "unit": "us",
        "higher_is_better": False,
        "next_dev": dev_s, "pipeline": pipe_s,
        "next_dev_cost_us": {arm: cost(dev_s, arm) for arm in ARMS[1:]},
        "pipeline_cost_us": {arm: cost(pipe_s, arm) for arm in ARMS[1:]},
        "bit_identical_tables": len(digests) == 1,
        "positions_per_frame_set": int(live.sum()),
        "covariances_per_frame_set": int(np.isfinite(ucov[..., 0]).sum()),
        "config": {"workload": f"c3: {KC} cameras {W}x{H}, {FW}x{FH} slots, {n} frames per arm and round",
                   "rounds": a.rounds,
                   "timing": "next_dev: CUDA events on the group's stream; pipeline: host wall time of submit / "
                             "collect (+ download_undistorted) with two frames in flight; medians over the rounds"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
