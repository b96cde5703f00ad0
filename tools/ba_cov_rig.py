"""What the BA covariance stage (cosl_ba_solver_set_covariance) costs on the device, on the c4 global BA and the c3 /
c2 local BA of tools/ba_setup_timing.py:
  - the stage's device time (download_covariance's out[4], globaltimer) against one LM trial of the same solve
    (info[11] / info[10] of run: the robust loop's time over its trials);
  - the submitted c3 BA (collect's info[11]: device time from submit to the end of the graph) armed and unarmed,
    on two handles, alternated;
  - the smallest relative pivot L_ii^2 / S_ii each scene reaches (the singularity threshold is 1e-12);
  - the card's name and power limit, read in the same run.
Usage: python tools/ba_cov_rig.py [--reps N] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from coslam_b200 import api, synth  # noqa: E402
from coslam_b200.ctypes_defs import BaOptions  # noqa: E402

CASES = {"c4": lambda: synth.make_ba_scene(bench.BA_CAMS, bench.BA_KF, bench.BA_PTS, bench.KLT_W, bench.KLT_H,
                                           seed=synth.BASE_SEED + 4, m_con=bench.BA_CAMS, n_con=0)[0],
         "c3": lambda: synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=synth.BASE_SEED + 3, m_con=8, n_con=2)[0],
         "c2": lambda: synth.make_ba_scene(2, 5, 5000, 640, 480, seed=synth.BASE_SEED + 2, m_con=4, n_con=2)[0]}


def options(name):
    o = BaOptions.defaults()
    if name == "c4":
        o.outer_iters, o.inner_iters = 1, 10
    return o


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def stage_vs_trial(name, reps):
    prob = CASES[name]()
    s = api.BaSolver(prob.copy(), options(name))
    s.set_covariance(1.0)
    plan = s.plan_info()
    s.run()  # warm-up: module load, pools, the stage's buffers
    stage, trial, piv = [], [], []
    for _ in range(reps):
        s.reset(prob.copy())
        info = s.run()
        _, _, out = s.download_covariance()
        stage.append(out["device_ms"])
        trial.append(1e3 * info[11] / max(1, info[10]))
        piv.append(out["min_pivot"])
    s.close()
    st, tr = float(np.median(stage)), float(np.median(trial))
    return {"scene": name, "free_cameras": prob.m - prob.m_con, "points": prob.n, "observations": prob.nobs,
            "blocks": plan["blocks"], "tiles": plan["tiles"], "stage_ms": st, "stage_ms_min": float(min(stage)),
            "lm_trial_ms": tr, "stage_over_trial": st / tr, "min_relative_pivot": float(min(piv))}


def submitted_c3(reps):
    prob = CASES["c3"]()
    opt = options("c3")
    hs = {"unarmed": api.BaSolver(prob.copy(), opt), "armed": api.BaSolver(prob.copy(), opt)}
    hs["armed"].set_covariance(1.0)
    ms = {k: [] for k in hs}
    for k, s in hs.items():  # graphs built, memory warm
        s.submit()
        s.collect()
    for _ in range(reps):
        for k, s in hs.items():
            s.reset(prob.copy())
            s.submit()
            ms[k].append(1e3 * s.collect()[11])
    for s in hs.values():
        s.close()
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"submitted_c3_ms": med, "armed_minus_unarmed_ms": med["armed"] - med["unarmed"],
            "spread_ms": {k: [float(min(v)), float(max(v))] for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "stage": [stage_vs_trial(n, a.reps) for n in ("c2", "c3", "c4")],
           "submit": submitted_c3(a.reps)}
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
