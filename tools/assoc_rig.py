"""What the registration handle (cosl_assoc_solver) costs: device time per submit and host time of the submit call at
two shapes, the c3 shape (4 camera entries x 2 000 features, 20 000 map points searching 1 to 4 of them) and a
13-camera rig (13 x 1 024 features, 6 000 points), with a pose covariance on every other entry, a 2x2 covariance on
every feature, 10 % of the features owned and 0 to 3 track observations each (the draws of tests/test_gpu_assoc.py).
Two handles per shape take turns (which goes first alternates), so both see the same conditions.  Reported per shape
(medians over --reps submits after a warm-up):
  device_ms    collect's CUDA-event time: the copy in, the binning, search and claim kernels and the copy back
  submit_us    host time of the submit call (the checks and the staging run there)
  registered   query pairs with status 0
and the same with gate = +inf (the *_ungated keys), where every cell is scanned: the cost of a brute-force scan over
every feature of each searched entry, with the same kernels.
There is no host baseline: the reference's getProjectionCovMat is not in this tree.  Prints one JSON line with the
card's name and power limit.

  python tools/assoc_rig.py [--reps 200]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import assoc_dense as ad  # noqa: E402  (the scenes the tests draw)
import bench  # noqa: E402  (card identity)

SHAPES = {"c3_4x2000_20000": (4, 2000, 20000), "rig_13x1024_6000": (13, 1024, 6000)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api

    if not torch.cuda.is_available():
        raise SystemExit("assoc_rig: needs a CUDA device")
    LIB, ck, ptr = api.LIB, api._ck, api._ptr
    res = {"tool": "assoc_rig", "card": bench.gpu_identity(a.device), "reps": a.reps, "shapes": {}}
    for name, (nc, nf, n) in SHAPES.items():
        kw = ad.scene(np.random.default_rng(nc), nc, nf, n, 1, 4)
        K, R, t, mf, X = (np.ascontiguousarray(kw[k], np.float64) for k in ("K", "R", "t", "mf", "X"))
        P = np.ascontiguousarray(kw["P"], np.float64).reshape(-1, 9)
        covf = np.ascontiguousarray(kw["covf"], np.float64).reshape(-1, 4)
        trkM = np.ascontiguousarray(kw["trk_m"], np.float64)
        wh, fo, own, to, tc, qo, qc = (np.ascontiguousarray(kw[k], np.int32) for k in
                                       ("wh", "feat_off", "owned", "trk_off", "trk_cam", "q_off", "q_cam"))
        cc = [None if Pc is None else np.ascontiguousarray(Pc) for Pc in kw["cam_cov"]]
        cp = (C.c_void_p * nc)(*[None if Pc is None else Pc.ctypes.data for Pc in cc])
        nq = int(qo[-1])
        hs = [api.AssocSolver(a.device, nc, n, nq, int(fo[-1]), int(to[-1])) for _ in range(2)]
        status = np.empty(nq, np.int32)
        dms = C.c_double(0)
        row = {"cams": nc, "features": int(fo[-1]), "points": n, "queries": nq}
        for gname, gate in (("", ad.GATE_99), ("_ungated", float("inf"))):
            dev, us = [], []
            for r in range(a.reps + 5):
                for s in (hs if r % 2 == 0 else hs[::-1]):
                    t0 = time.perf_counter()
                    ck(LIB.cosl_assoc_solver_submit(s.h, nc, ptr(K), ptr(R), ptr(t), cp, ptr(wh), ptr(fo), ptr(mf),
                                                    ptr(covf), ptr(own), ptr(to), ptr(tc), ptr(trkM), n, ptr(X),
                                                    ptr(P), ptr(qo), ptr(qc), 1.0, gate, 20.0))
                    dt = time.perf_counter() - t0
                    ck(LIB.cosl_assoc_solver_collect(s.h, status.ctypes.data, None, None, None, C.byref(dms)))
                    if r >= 5:  # warm-up: module load, first-touch of the pinned buffers
                        dev.append(dms.value)
                        us.append(1e6 * dt)
            row.update({"device_ms" + gname: float(np.median(dev)),
                        "spread_ms" + gname: [float(min(dev)), float(max(dev))],
                        "submit_us" + gname: float(np.median(us)),
                        "registered" + gname: int((status == 0).sum())})
        for s in hs:
            s.close()
        res["shapes"][name] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
