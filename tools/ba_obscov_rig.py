"""What measurement covariances (cosl_ba_solver_set_obs_cov) cost the BA on the device, on the c4 global BA and the
c3 / c2 local BA of tools/ba_cov_rig.py: device time per LM trial of run_fixed, armed (a random anisotropic 2x2
covariance per observation) against unarmed, from the solver's section timers (CUDA events around every stage of
the host loop: linearisation, Schur contraction, solve, back substitution, cost).  Two handles on the same problem,
alternated; the card's name and power limit are read in the same run.
Usage: python tools/ba_obscov_rig.py [--reps N] [--trials T] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from coslam_b200 import api  # noqa: E402
from tools.ba_cov_rig import CASES, card, options  # noqa: E402


def covx(n, rng):
    th = rng.uniform(0, np.pi, n)
    s = rng.uniform(0.3, 1.5, (n, 2))
    R = np.stack([np.stack([np.cos(th), -np.sin(th)], -1), np.stack([np.sin(th), np.cos(th)], -1)], -2)
    S = R * s[:, None, :]
    return S @ S.transpose(0, 2, 1)


def timed(s, prob, trials):
    s.reset(prob.copy())
    s.profile_enable(True)
    info = s.run_fixed(trials)
    t = s.timers()
    s.profile_enable(False)
    return {k: v[0] for k, v in t.items()}, int(info[10])


def scene(name, reps, trials):
    prob = CASES[name]()
    hs = {"unarmed": api.BaSolver(prob.copy(), options(name)), "armed": api.BaSolver(prob.copy(), options(name))}
    hs["armed"].set_obs_cov(covx(prob.nobs, np.random.default_rng(1)))
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
    return {"scene": name, "observations": prob.nobs, "free_cameras": prob.m - prob.m_con, "points": prob.n,
            "trials": trials, "device_ms_per_trial": med, "spread_ms": {k: [float(min(v)), float(max(v))]
                                                                         for k, v in per.items()},
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
