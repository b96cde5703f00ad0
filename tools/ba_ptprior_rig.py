"""What point priors (cosl_ba_solver_set_pt_prior) cost the BA on the device, on the c2 / c3 local BA and the c4 global
BA of tools/ba_cov_rig.py: device time per LM trial of run_fixed(10), with a prior on every free point against none,
from the solver's section timers (CUDA events around every stage of the host loop: linearisation, Schur contraction,
solve, back substitution, cost).  Two handles on the same problem, alternated; the card's name and power limit are
read in the same run.
Usage: python tools/ba_ptprior_rig.py [--reps N] [--trials T] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from coslam_b200 import api  # noqa: E402
from tools.ba_cov_rig import CASES, card, options  # noqa: E402
from tools.ba_prior_rig import timed  # noqa: E402


def priors(prob, rng):
    """a prior on every free point: the point, moved 1 cm, with 3 cm standard deviations"""
    pts = np.arange(prob.n_con, prob.n)
    X = prob.X[pts] + 0.01 * rng.normal(size=(len(pts), 3))
    cov = np.tile(9e-4 * np.eye(3), (len(pts), 1, 1))
    return pts, X, cov


def scene(name, reps, trials):
    prob = CASES[name]()
    hs = {"unarmed": api.BaSolver(prob.copy(), options(name)), "armed": api.BaSolver(prob.copy(), options(name))}
    hs["armed"].set_pt_prior(*priors(prob, np.random.default_rng(1)))
    for s in hs.values():  # warm-up: module load, pools
        timed(s, prob, trials)
    per = {k: [] for k in hs}
    sec = {k: [] for k in hs}
    for _ in range(reps):
        for k, s in hs.items():
            t, n = timed(s, prob, trials)
            per[k].append(sum(t.values()) / n)
            sec[k].append({q: v / n for q, v in t.items()})
    for s in hs.values():
        s.close()
    med = {k: float(np.median(v)) for k, v in per.items()}
    secs = {k: {q: float(np.median([d[q] for d in v])) for q in v[0]} for k, v in sec.items()}
    return {"scene": name, "observations": prob.nobs, "free_points": prob.n - prob.n_con, "priors": prob.n - prob.n_con,
            "free_cameras": prob.m - prob.m_con, "trials": trials, "device_ms_per_trial": med,
            "spread_ms": {k: [float(min(v)), float(max(v))] for k, v in per.items()},
            "armed_over_unarmed": med["armed"] / med["unarmed"], "sections_ms_per_trial": secs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--trials", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "scenes": [scene(n, a.reps, a.trials) for n in ("c2", "c3", "c4")]}
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
