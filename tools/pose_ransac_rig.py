"""What PnP RANSAC (cosl_pose_solver_set_ransac) costs the per-frame pose solve: two handles on the same inputs, one
armed for every camera and one unarmed, alternated (which goes first alternates too), at 4 x 192 (64 and 256
hypotheses), 13 x 1000 (256) and 12 x 600 (2000, the multi-camera initialisation).  Cameras from
tests/pnp_dense.scene: 40 % gross outliers, R0 30 degrees off, 2 px threshold, tau = 10.  Reported per setting
(medians over --reps submits of each after a warm-up):
  armed_ms, unarmed_ms   collect's CUDA-event time: copies, RANSAC (armed) and the solve
  replaced               cameras whose start RANSAC replaced in the last armed submit
  cv2_ms                 a host reference, not the reference project's code: cv2.solvePnPRansac(SOLVEPNP_EPNP) with
                         the same iteration count (its adaptive stop at confidence 1 - 1e-12 may end it sooner) and
                         threshold over the same cameras, one thread, median of 3
Prints one JSON line with the card's name and power limit.

  python tools/pose_ransac_rig.py [--reps 50]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bench  # noqa: E402  (card identity)
import pnp_dense as pn  # noqa: E402  (the cameras the tests draw)

SETTINGS = ((4, 192, 64), (4, 192, 256), (13, 1000, 256), (12, 600, 2000))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    from coslam_b200 import api

    res = {"tool": "pose_ransac_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "settings": {}}
    for C, n, nh in SETTINGS:
        rng = np.random.default_rng(C * 7 + n)
        cams = [pn.scene(rng, n, 0.4, 30.0) for _ in range(C)]
        args = [[c[k] for c in cams] for k in range(5)]
        armed = api.PoseSolver(a.device, C, C * n)
        plain = api.PoseSolver(a.device, C, C * n)
        armed.set_ransac(np.ones(C, bool), nh, 2.0, 6, 1)
        t = {"armed": [], "unarmed": []}
        for r in range(a.reps + 3):
            order = [("armed", armed), ("unarmed", plain)]
            for name, s in order if r % 2 == 0 else order[::-1]:
                s.submit(*args, 10.0)
                ms = s.collect()[4]
                if r >= 3:
                    t[name].append(ms)
        st = armed.download_ransac()
        cv = []
        try:
            import cv2

            cv2.setNumThreads(1)
            for _ in range(3):
                t0 = time.perf_counter()
                for K, _, _, M, m, _, _, _ in cams:
                    cv2.solvePnPRansac(M, m, K, None, iterationsCount=nh, reprojectionError=2.0, confidence=1 - 1e-12,
                                       flags=cv2.SOLVEPNP_EPNP)
                cv.append((time.perf_counter() - t0) * 1e3)
        except ImportError:
            pass
        res["settings"][f"{C}x{n}_h{nh}"] = {
            "armed_ms": float(np.median(t["armed"])), "unarmed_ms": float(np.median(t["unarmed"])),
            "replaced": int((st["status"] == 0).sum()), "cv2_ms": float(np.median(cv)) if cv else None}
        armed.close()
        plain.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
