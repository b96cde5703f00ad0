"""What a new bundle-adjustment problem costs the SLAM thread: a fresh solver handle per BA against one handle
that loads each problem (cosl_ba_solver_load).  CoSLAM never solves the same shape twice, so every BA is a
new problem either way.  KLT frames of c3 (4 x 1280x720, live settings) go through
cosl_klt_group_submit / _collect, frame n+1 submitted before frame n is collected.

  local     every --ba-every-th frame a c3 local BA (20 poses, the oldest two key frames fixed, default
            robust options), each request a different window (seed), submitted when none is in flight and
            picked up by cosl_ba_solver_query once per frame
  intercam  every frame an inter-camera pose BA (4 free cameras, 800 fixed and up to ~60 free points, a
            new point count every frame), submitted after the frame's KLT submit and collected in the same frame

Arms, alternated round by round:
  create    cosl_ba_solver_create + submit ... collect + download + destroy per BA
  load      one handle: cosl_ba_solver_load + submit ... collect + download per BA

Reported per arm (median over the rounds after the warm-up round 0):
  request_ms      host wall time of the request (create + submit, or load + submit)
  setup_ms        of which create, or load
  submit_ms       of which submit (the first submit of a fresh handle captures and instantiates its graph;
                  after a load the graph is updated or instantiated again)
  finish_ms       host wall time of collect + download (+ destroy)
  frame_ms_ba     ms per KLT frame set (its submit + collect + the BA calls made in that frame) with a BA
                  in flight
Every BA result is compared with the one the other arm gave for the same problem (decisions and outliers
equal, parameters within 1e-9 / 1e-8).

  python tools/ba_load_rig.py [--frames 200] [--ba-every 10] [--rounds 4]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--ba-every", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import BaOptions

    if not torch.cuda.is_available():
        raise SystemExit("ba_load_rig: needs a CUDA device")
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    seqs = bench.make_sequences(0)
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    grp = api.KltGroup(bench.klt_cfg(), KC, W, H, L, FW, FH, device=a.device)
    rng = np.random.default_rng(5)
    local = [synth.make_ba_scene(4, 5, 20000, W, H, seed=synth.BASE_SEED + 3 + 100 * k, m_con=8, n_con=2)[0]
             for k in range(4)]
    inter = [synth.make_ba_scene(4, 1, int(rng.integers(940, 990)), 640, 480, seed=900 + k, m_con=0, n_con=800,
                                 window=0, p_vis=1.0)[0] for k in range(16)]
    opt_local = BaOptions.defaults()
    opt_local.device = a.device
    opt_inter = BaOptions.defaults()
    opt_inter.device = a.device
    opt_inter.outer_iters, opt_inter.inner_iters = 1, 10
    opt_inter.opts[2] = 1e-6  # ends the round before the accept decisions reach the noise floor

    def run_arm(kind, mode):
        probs, opt = (local, opt_local) if mode == "local" else (inter, opt_inter)
        every = a.ba_every if mode == "local" else 1
        keep = api.BaSolver(probs[0].copy(), opt) if kind == "load" else None
        rec = {k: [] for k in ("request_ms", "setup_ms", "submit_ms", "finish_ms", "frame_ms_ba", "frame_ms_idle")}
        results = {}
        st = {"busy": False, "k": 0}
        grp.first(host[0])
        grp.submit(host[1 % len(host)])

        def request():
            k = st["k"] % len(probs)
            st["k"] += 1
            p = probs[k].copy()
            t0 = time.perf_counter()
            if kind == "create":
                s = api.BaSolver(p, opt)
            else:
                s = keep
                s.load(p)
            t1 = time.perf_counter()
            s.submit()
            t2 = time.perf_counter()
            rec["setup_ms"].append(1e3 * (t1 - t0))
            rec["submit_ms"].append(1e3 * (t2 - t1))
            rec["request_ms"].append(1e3 * (t2 - t0))
            st.update(busy=True, s=s, prob=k)

        def finish():
            s = st["s"]
            t0 = time.perf_counter()
            info = s.collect()
            res = s.download().copy()
            if kind == "create":
                s.close()
            rec["finish_ms"].append(1e3 * (time.perf_counter() - t0))
            results.setdefault(st["prob"], (info.copy(), res))
            st["busy"] = False

        for f in range(1, a.frames + 1):
            t0 = time.perf_counter()
            if f % every == 0 and not st["busy"]:
                request()
            in_flight = st["busy"]
            if f < a.frames:
                grp.submit(host[(f + 1) % len(host)])
            grp.collect()
            if st["busy"] and (mode == "intercam" or st["s"].done()):
                finish()
            (rec["frame_ms_ba"] if in_flight else rec["frame_ms_idle"]).append(1e3 * (time.perf_counter() - t0))
        if st["busy"]:
            finish()
        if keep is not None:
            keep.close()
        return rec, results

    out = {"tool": "ba_load_rig", "card": bench.gpu_identity(a.device), "frames_per_arm": a.frames,
           "timed_rounds": a.rounds - 1}
    for mode in ("local", "intercam"):
        rounds = {"create": [], "load": []}
        res = {"create": {}, "load": {}}
        for r in range(a.rounds):
            for kind in (("create", "load") if r % 2 == 0 else ("load", "create")):
                rec, results = run_arm(kind, mode)
                rounds[kind].append(rec)
                for k, v in results.items():
                    res[kind].setdefault(k, v)
        same = []
        for k in res["create"]:
            if k in res["load"]:
                (iw, pw), (ig, pg) = res["create"][k], res["load"][k]
                same.append(bool(np.array_equal(iw[5:11], ig[5:11]) and iw[13] == ig[13]
                                 and np.array_equal(pw.outlier, pg.outlier)
                                 and np.abs(pw.R - pg.R).max() < 1e-9 and np.abs(pw.t - pg.t).max() < 1e-9
                                 and np.abs(pw.X - pg.X).max() < 1e-8))

        def med(kind, key):
            v = [x for rr in rounds[kind][1:] for x in rr[key]]
            return round(float(np.median(v)), 4) if v else None

        keys = ("request_ms", "setup_ms", "submit_ms", "finish_ms", "frame_ms_ba", "frame_ms_idle")
        p0 = (local if mode == "local" else inter)[0]
        out[mode] = {"workload": (f"{p0.m} poses ({p0.m_con} fixed), ~{p0.n} points ({p0.n_con} fixed), "
                                  f"~{p0.nobs} obs; a BA every {a.ba_every if mode == 'local' else 1} frame(s)"),
                     "ba_per_arm": {k: sum(len(rr["request_ms"]) for rr in rounds[k][1:]) for k in rounds},
                     "results_equal_across_arms": f"{sum(same)}/{len(same)}",
                     "create": {k: med("create", k) for k in keys},
                     "load": {k: med("load", k) for k in keys}}
    print(json.dumps(out))
    grp.close()


if __name__ == "__main__":
    main()
