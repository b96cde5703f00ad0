"""What Gaussian pose priors (cosl_pose_solver_submit_prior) cost the per-frame pose solve: two unarmed handles, one
solving with a prior on every camera and one without, alternated (which goes first alternates too), at 4 x 192
(bench.py's pose workload) and 13 x 192 points (synth.make_pose_case, default options, tau = 10).  The priors are
seeded and consistent with the true pose, as a frame-to-frame prior is: covariances with standard deviations of 0.01
down to 0.001 rad or units, and the true pose a draw from each.  Reported per shape (medians over --reps solves of
each after a warm-up):
  device_ms    collect's CUDA-event time: the copies (with the prior records for the prior submit) and the solve
  extra_ms     prior minus plain device_ms
  rounds       re-weighting rounds (nIterRW) and LM iterations of the last round (nIterLM), summed over cameras:
               the two solves take different paths, so part of extra_ms is iterations rather than arithmetic
  submit_us    host time of the submit call (the prior checks and factors run there)
Prints one JSON line with the card's name and power limit.

  python tools/pose_prior_rig.py [--reps 200]"""
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
import pose_prior_dense as ppd  # noqa: E402  (the priors the tests draw)

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
        raise SystemExit("pose_prior_rig: needs a CUDA device")
    LIB, ck = api.LIB, api._ck
    res = {"tool": "pose_prior_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for Cn, N in SHAPES:
        cases = [synth.make_pose_case(N, 1280, 720, seed=100 + c) for c in range(Cn)]
        args, _, keep = api._pose_batch_args([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                                             [c[3] for c in cases], [c[4] for c in cases], 10.0, None, None)
        rng = np.random.default_rng(Cn)
        recs = [api._pose_prior(*ppd.drawn_prior(c[5], c[6], rng, max_deg=5.0, cond=1e2, scale=1e-4)) for c in cases]
        pp = (C.c_void_p * Cn)(*[r.ctypes.data for r in recs])
        hs = {"plain": api.PoseSolver(a.device, Cn, Cn * N), "prior": api.PoseSolver(a.device, Cn, Cn * N)}
        R, t, ok = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32)
        dms = C.c_double(0)
        rec = {k: [] for k in ("plain", "prior", "plain_us", "prior_us")}
        iters = {}
        for r in range(a.reps + 5):
            for k in (("plain", "prior") if r % 2 == 0 else ("prior", "plain")):
                s = hs[k]
                opts = (PoseOpt * Cn)(*[PoseOpt.defaults() for _ in range(Cn)])
                t0 = time.perf_counter()
                if k == "plain":
                    ck(LIB.cosl_pose_solver_submit(s.h, *args, opts))
                else:
                    ck(LIB.cosl_pose_solver_submit_prior(s.h, *args[:7], None, pp, *args[7:], opts))
                dt = time.perf_counter() - t0
                ck(LIB.cosl_pose_solver_collect(s.h, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                C.byref(dms)))
                iters[k] = {"nIterRW": sum(o.nIterRW for o in opts), "nIterLM": sum(o.nIterLM for o in opts)}
                if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                    rec[k].append(dms.value)
                    rec[k + "_us"].append(1e6 * dt)
        for s in hs.values():
            s.close()
        med = {k: float(np.median(v)) for k, v in rec.items()}
        res["shapes"][f"{Cn}x{N}"] = {
            "device_ms": {"plain": med["plain"], "prior": med["prior"]},
            "spread_ms": {k: [float(min(rec[k])), float(max(rec[k]))] for k in ("plain", "prior")},
            "extra_ms": med["prior"] - med["plain"], "rounds": iters,
            "submit_us": {"plain": med["plain_us"], "prior": med["prior_us"]}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
