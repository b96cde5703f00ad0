"""What measurement covariances (cosl_pose_solver_submit_cov) cost the per-frame pose solve: one unarmed handle solves
the same inputs with cosl_pose_solver_submit and with cosl_pose_solver_submit_cov in alternation (which goes first
alternates too), at 4 x 192 (bench.py's pose workload) and 13 x 192 points (synth.make_pose_case, default options,
tau = 10; covariances with standard deviations of 0.15 to 1.5 px along random axes, seeded).  Reported per shape
(medians over --reps solves of each after a warm-up):
  device_ms    collect's CUDA-event time: the copies (with the whitening factors for submit_cov) and the solve
  extra_ms     submit_cov minus submit device_ms
  rounds       re-weighting rounds (nIterRW) and LM iterations of the last round (nIterLM), summed over cameras:
               the two solves take different paths, so part of extra_ms is iterations rather than arithmetic
  submit_us    host time of the submit call (the covariance checks and factors run there)
Prints one JSON line with the card's name and power limit.

  python tools/pose_obscov_rig.py [--reps 200]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bench  # noqa: E402  (card identity)
import pose_obscov_dense as od  # noqa: E402  (the covariances the tests draw)

SHAPES = ((4, 192), (13, 192))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import PoseOpt

    if not torch.cuda.is_available():
        raise SystemExit("pose_obscov_rig: needs a CUDA device")
    LIB, ck = api.LIB, api._ck
    res = {"tool": "pose_obscov_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for Cn, N in SHAPES:
        cases = [synth.make_pose_case(N, 1280, 720, seed=100 + c) for c in range(Cn)]
        args, _, keep = api._pose_batch_args([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                                             [c[3] for c in cases], [c[4] for c in cases], 10.0, None, None)
        rng = np.random.default_rng(Cn)
        covx = [np.ascontiguousarray(od.random_covx(N, rng)[0].reshape(N, 4)) for _ in range(Cn)]
        cp = (C.c_void_p * Cn)(*[c.ctypes.data for c in covx])
        s = api.PoseSolver(a.device, Cn, Cn * N)
        R, t, ok = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32)
        dms = C.c_double(0)
        rec = {k: [] for k in ("submit", "submit_cov", "submit_us", "submit_cov_us")}
        iters = {}
        for r in range(a.reps + 5):
            for k in (("submit", "submit_cov") if r % 2 == 0 else ("submit_cov", "submit")):
                opts = (PoseOpt * Cn)(*[PoseOpt.defaults() for _ in range(Cn)])
                t0 = time.perf_counter()
                if k == "submit":
                    ck(LIB.cosl_pose_solver_submit(s.h, *args, opts))
                else:
                    ck(LIB.cosl_pose_solver_submit_cov(s.h, *args[:7], cp, *args[7:], opts))
                dt = time.perf_counter() - t0
                ck(LIB.cosl_pose_solver_collect(s.h, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                C.byref(dms)))
                iters[k] = {"nIterRW": sum(o.nIterRW for o in opts), "nIterLM": sum(o.nIterLM for o in opts)}
                if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                    rec[k].append(dms.value)
                    rec[k + "_us"].append(1e6 * dt)
        s.close()
        med = {k: float(np.median(v)) for k, v in rec.items()}
        res["shapes"][f"{Cn}x{N}"] = {
            "device_ms": {"submit": med["submit"], "submit_cov": med["submit_cov"]},
            "spread_ms": {k: [float(min(rec[k])), float(max(rec[k]))] for k in ("submit", "submit_cov")},
            "extra_ms": med["submit_cov"] - med["submit"], "rounds": iters,
            "submit_us": {"submit": med["submit_us"], "submit_cov": med["submit_cov_us"]}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
