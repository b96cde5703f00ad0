"""What the map-point update (cosl_pose_solver_submit_mappts) costs the per-frame pose solve: two armed handles, one
running submit_prior (no prior, no covariances) and one submit_mappts with the same solve plus map points, alternated
(which goes first alternates too), at 4 x 192 solve points + 4 x 2000 map points and 13 x 192 + 13 x 1000
(synth.make_pose_case, default options, tau = 10; map points seen by the true pose, prior means 1 to 10 cm off, 1 px
observations, gate 5.991).  Reported per shape (medians over --reps submits of each after a warm-up):
  device_ms    collect's CUDA-event time: copies, solve, covariance stage and, for mappts, the update and its copy
  extra_ms     mappts minus plain device_ms
  submit_us    host time of the submit call (the map-point checks and staging run there)
  updated      points with status 0 in the last mappts submit
Prints one JSON line with the card's name and power limit.

  python tools/pose_mappts_rig.py [--reps 200]"""
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
import pose_dense as pd  # noqa: E402
import pose_mappts_dense as md  # noqa: E402  (the map points the tests draw)

SHAPES = ((4, 192, 2000), (13, 192, 1000))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import PoseOpt

    if not torch.cuda.is_available():
        raise SystemExit("pose_mappts_rig: needs a CUDA device")
    LIB, ck = api.LIB, api._ck
    res = {"tool": "pose_mappts_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for Cn, N, NM in SHAPES:
        cases = [synth.make_pose_case(N, 1280, 720, seed=100 + c) for c in range(Cn)]
        args, _, keep = api._pose_batch_args([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                                             [c[3] for c in cases], [c[4] for c in cases], 10.0, None, None)
        rng = np.random.default_rng(Cn)
        mp = []
        for K, _, _, _, _, Rt, tt in cases:
            Xt = md.view_points(K, Rt, tt, rng, NM, 1280, 720, 3.0, 20.0)
            P0 = np.array([md.random_spd(rng, 3, 1e-4, 1e-2) for _ in range(NM)])
            X0 = Xt + np.array([rng.multivariate_normal(np.zeros(3), p) for p in P0])
            u, v = pd.project(K, Rt, tt, Xt)
            m = np.column_stack([u, v]) + rng.normal(0.0, 1.0, (NM, 2))
            mp.append((np.ascontiguousarray(X0), np.ascontiguousarray(P0.reshape(NM, 9)), np.ascontiguousarray(m)))
        nmap = np.full(Cn, NM, np.int32)
        ptrs = [(C.c_void_p * Cn)(*[e[k].ctypes.data for e in mp]) for k in range(3)]
        hs = {"plain": api.PoseSolver(a.device, Cn, Cn * N), "mappts": api.PoseSolver(a.device, Cn, Cn * N)}
        for s in hs.values():
            s.set_covariance(1.0)
        hs["mappts"].reserve_mappts(Cn * NM)
        R, t, ok = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32)
        status = np.empty(Cn * NM, np.int32)
        dms = C.c_double(0)
        rec = {k: [] for k in ("plain", "mappts", "plain_us", "mappts_us")}
        for r in range(a.reps + 5):
            for k in (("plain", "mappts") if r % 2 == 0 else ("mappts", "plain")):
                s = hs[k]
                opts = (PoseOpt * Cn)(*[PoseOpt.defaults() for _ in range(Cn)])
                t0 = time.perf_counter()
                if k == "plain":
                    ck(LIB.cosl_pose_solver_submit_prior(s.h, *args[:7], None, None, *args[7:], opts))
                else:
                    ck(LIB.cosl_pose_solver_submit_mappts(s.h, *args[:7], None, None, *args[7:], opts,
                                                          nmap.ctypes.data, *ptrs, None, md.GATE_95))
                dt = time.perf_counter() - t0
                ck(LIB.cosl_pose_solver_collect(s.h, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                C.byref(dms)))
                if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                    rec[k].append(dms.value)
                    rec[k + "_us"].append(1e6 * dt)
        ck(LIB.cosl_pose_solver_download_mappts(hs["mappts"].h, None, None, None, status.ctypes.data))
        for s in hs.values():
            s.close()
        med = {k: float(np.median(v)) for k, v in rec.items()}
        res["shapes"][f"{Cn}x{N}+{Cn}x{NM}"] = {
            "device_ms": {"plain": med["plain"], "mappts": med["mappts"]},
            "spread_ms": {k: [float(min(rec[k])), float(max(rec[k]))] for k in ("plain", "mappts")},
            "extra_ms": med["mappts"] - med["plain"],
            "submit_us": {"plain": med["plain_us"], "mappts": med["mappts_us"]},
            "updated": int((status == 0).sum())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
