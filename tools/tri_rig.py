"""What the triangulation handle (cosl_tri_solver) costs: device time per submit and host time of the submit call at
two shapes, 13 camera entries x 1 000 points x 3 views (newMapPoints for a full rig) and the post-BA refresh of a c3
window (80 camera entries = 20 key frames x 4 cameras, 18 600 points of 2 to 8 views), with a pose covariance on every
other entry and a 2x2 covariance on every view (the draws of tests/test_gpu_tri.py).  Two handles per shape take turns
(which goes first alternates), so both see the same conditions.  Reported per shape (medians over --reps submits
after a warm-up):
  device_ms    collect's CUDA-event time: the copy in, tri_kernel and the copy back
  submit_us    host time of the submit call (the checks and the staging run there)
  good         points with status 0
There is no host baseline: the reference's triangulation is not in this tree.  Prints one JSON line with the card's
name and power limit.

  python tools/tri_rig.py [--reps 200]"""
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
import test_gpu_tri as gt  # noqa: E402  (the points the tests draw)

SHAPES = {"13x1000x3": (39, 1000, 3, 3), "c3_refresh_18600x2-8": (80, 18600, 2, 8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api

    if not torch.cuda.is_available():
        raise SystemExit("tri_rig: needs a CUDA device")
    LIB, ck, ptr = api.LIB, api._ck, api._ptr
    res = {"tool": "tri_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for name, (nc, n, lo, hi) in SHAPES.items():
        rng = np.random.default_rng(nc)
        K, R, t, cc = gt._table(rng, nc)
        off, cam, m, covm = gt._points(rng, K, R, t, n, lo, hi)
        K, R, t, m = (np.ascontiguousarray(x, np.float64) for x in (K, R, t, m))
        covm = np.ascontiguousarray(covm, np.float64).reshape(-1, 4)
        cc = [None if P is None else np.ascontiguousarray(P) for P in cc]
        cp = (C.c_void_p * nc)(*[None if P is None else P.ctypes.data for P in cc])
        hs = [api.TriSolver(a.device, nc, n, int(off[-1])) for _ in range(2)]
        status = np.empty(n, np.int32)
        dms = C.c_double(0)
        dev, us = [], []
        for r in range(a.reps + 5):
            for s in (hs if r % 2 == 0 else hs[::-1]):
                t0 = time.perf_counter()
                ck(LIB.cosl_tri_solver_submit(s.h, nc, ptr(K), ptr(R), ptr(t), cp, n, ptr(off), ptr(cam), ptr(m),
                                              ptr(covm), 1.0, 6.0))
                dt = time.perf_counter() - t0
                ck(LIB.cosl_tri_solver_collect(s.h, None, None, None, status.ctypes.data, C.byref(dms)))
                if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                    dev.append(dms.value)
                    us.append(1e6 * dt)
        for s in hs:
            s.close()
        res["shapes"][name] = {"cams": nc, "points": n, "views": int(off[-1]),
                               "device_ms": float(np.median(dev)),
                               "spread_ms": [float(min(dev)), float(max(dev))],
                               "submit_us": float(np.median(us)),
                               "good": int((status == 0).sum())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
