"""Time of cosl_posegraph_solve (the camera-group merge's pose graph on the GPU) against the CPU oracle.
Prints one JSON line (card name and power limit included).

Workloads: key-frame graphs of a merge as MergeCameraGroup::_constructGraphForKeyFrms builds them --
100 key frames x 4, 8 and 13 cameras, 2 constraint edges sharing one unknown scale, noisy measurements
-- and a chain of 2000 nodes with one loop closure and one uncertain edge.  Per workload: wall time of a
call (it ends in a stream synchronise) after warm-up, the host part of it (validation, numbering,
planning, lists) as the library reports it, and the oracle's time for the same graph (envelope Cholesky
on one core, oracle/posegraph_oracle.cpp).

  python tools/posegraph_general_bench.py [--reps 20] [--warmup 3] [--device 0]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (card identity)
from coslam_b200 import api, synth  # noqa: E402
from oracle import orc_pg_general as orc  # noqa: E402

KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et")


def _args(g):
    return [g[k] for k in KEYS] + [g["scale_col"], g["n_scale"]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-reps", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    work = [(f"merge_100x{c}", synth.make_merge_graph(100, c, seed=c, n_constraints=2, noise=0.01))
            for c in (4, 8, 13)]
    work.append(("loop_2000", synth.make_pose_graph(2000, seed=1, loops=1, n_scale=1, uncertain=1, noise=0.01)))
    res = {}
    for name, g in work:
        args = _args(g)
        for _ in range(a.warmup):
            api.posegraph_solve(*args, device=a.device)
        wall, host = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            out = api.posegraph_solve(*args, device=a.device)
            wall.append(1e3 * (time.perf_counter() - t0))
            host.append(api.posegraph_last_host_ms())
        ot = []
        for _ in range(a.oracle_reps):
            t0 = time.perf_counter()
            ref = orc.posegraph_solve(*args)
            ot.append(1e3 * (time.perf_counter() - t0))
        err = max(float(np.abs(x - y).max()) for x, y in zip(out[:2], ref[:2]))
        res[name] = {"nodes": int(len(g["fixed"])), "edges": int(len(g["id1"])), "scales": int(g["n_scale"]),
                     "ms_per_call": float(np.median(wall)), "ms_per_call_min": float(np.min(wall)),
                     "host_ms": float(np.median(host)), "oracle_ms": float(np.median(ot)),
                     "max_abs_diff_vs_oracle": err}
    print(json.dumps({
        "metric": "ms_per_call_merge_100x13", "value": res["merge_100x13"]["ms_per_call"], "unit": "ms",
        "higher_is_better": False, "workloads": res,
        "config": {"reps": a.reps, "warmup": a.warmup, "oracle_reps": a.oracle_reps,
                   "timing": "host wall time of api.posegraph_solve (H2D, 2 x (assemble + tile solve), finish, "
                             "D2H, stream synchronise), median over reps; host_ms = cosl_posegraph_last_host_ms"},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
