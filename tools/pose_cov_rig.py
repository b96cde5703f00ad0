"""What the pose solver's covariance stage (cosl_pose_solver_set_covariance) costs: two handles, one armed and one
not, solve the same inputs in alternation (which goes first alternates too), at 4 x 192 (bench.py's pose workload)
and 13 x 192 points (synth.make_pose_case, default options, tau = 10).  Reported per shape (medians over --reps
solves per handle after a warm-up):
  device_ms    collect's CUDA-event time: copies, the solve kernel and, armed, the stage and its read-back
  stage_ms     armed minus unarmed device_ms
  download_us  host time of cosl_pose_solver_download_covariance (cov, err and out)
The armed and unarmed poses must agree bit for bit.  Prints one JSON line with the card's name and power limit.

  python tools/pose_cov_rig.py [--reps 200]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (card identity)

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
        raise SystemExit("pose_cov_rig: needs a CUDA device")
    LIB, ck = api.LIB, api._ck
    res = {"tool": "pose_cov_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for Cn, N in SHAPES:
        cases = [synth.make_pose_case(N, 1280, 720, seed=100 + c) for c in range(Cn)]
        args, _, keep = api._pose_batch_args([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                                             [c[3] for c in cases], [c[4] for c in cases], 10.0, None, None)
        hs = {"unarmed": api.PoseSolver(a.device, Cn, Cn * N), "armed": api.PoseSolver(a.device, Cn, Cn * N)}
        hs["armed"].set_covariance(0.25)
        R, t, ok = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32)
        cov, err, out = np.empty((Cn, 36)), np.empty(Cn * N), np.empty((Cn, 4))
        dms = C.c_double(0)
        rec = {"unarmed": [], "armed": [], "download_us": []}
        poses = {k: set() for k in hs}
        for r in range(a.reps + 5):
            for k in (("unarmed", "armed") if r % 2 == 0 else ("armed", "unarmed")):
                s = hs[k]
                opts = (PoseOpt * Cn)(*[PoseOpt.defaults() for _ in range(Cn)])
                ck(LIB.cosl_pose_solver_submit(s.h, *args, opts))
                ck(LIB.cosl_pose_solver_collect(s.h, R.ctypes.data, t.ctypes.data, opts, ok.ctypes.data,
                                                C.byref(dms)))
                poses[k].add(R.tobytes() + t.tobytes() + ok.tobytes() + bytes(opts))
                if k == "armed":
                    t0 = time.perf_counter()
                    ck(LIB.cosl_pose_solver_download_covariance(s.h, cov.ctypes.data, err.ctypes.data,
                                                                out.ctypes.data))
                    dt = time.perf_counter() - t0
                if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                    rec[k].append(dms.value)
                    if k == "armed":
                        rec["download_us"].append(1e6 * dt)
        for s in hs.values():
            s.close()
        med = {k: float(np.median(v)) for k, v in rec.items()}
        res["shapes"][f"{Cn}x{N}"] = {
            "device_ms": {"unarmed": med["unarmed"], "armed": med["armed"]},
            "spread_ms": {k: [float(min(rec[k])), float(max(rec[k]))] for k in ("unarmed", "armed")},
            "stage_ms": med["armed"] - med["unarmed"], "download_us": med["download_us"],
            "valid_cameras": int(out[:, 3].sum()),
            "poses_bit_identical": len(poses["armed"]) == 1 and poses["armed"] == poses["unarmed"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
