"""Local BA beside KLT tracking on c3 (4 x 1280x720, live settings; local BA of 20 poses / 20 k points,
the oldest two key frames fixed, default robust options: 5 rounds x <= 10 iterations), the reference's threading shape against the
submitted BA.  KLT frames go through cosl_klt_group_submit / _collect (frame n+1 submitted before frame n
is collected); every --ba-every-th frame starts a local BA (reset to the same problem) when none is in
flight, and the SLAM thread checks once per frame whether it has finished:

  thread   cosl_ba_solver_run + download on a second host thread (requestForBA / _bundleAdjustmentThread
           of the reference); "finished" is the thread having exited
  submit   cosl_ba_solver_submit on the SLAM thread; cosl_ba_solver_query once per frame, then collect +
           download

Reported per arm (median over the rounds after the warm-up round 0; the arms alternate in a round):
  klt_ms_ba / klt_ms_idle   ms per KLT frame set (submit + collect) with / without a BA in flight
  ba_latency_ms             wall time from the BA request to the frame that picks up its result
  ba_cpu_s                  host CPU seconds per BA: thread time of the BA thread (thread arm), or of
                            the SLAM thread inside submit / query / collect / download (submit arm)
  proc_cpu_s_per_frame      process CPU seconds per frame over the whole arm (every thread)
  us_per_trial              info[11] / info[10]: the device loop's time per LM trial (the thread arm's
                            info[11] is the host's wall time of its loop, which keeps the device busy)
Every BA result is compared with the first one (decisions and outliers equal, parameters within 1e-9).

  python tools/ba_async_rig.py [--frames 400] [--ba-every 10] [--rounds 4]"""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--ba-every", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import BaOptions

    if not torch.cuda.is_available():
        raise SystemExit("ba_async_rig: needs a CUDA device")
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    seqs = bench.make_sequences(0)
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    grp = api.KltGroup(bench.klt_cfg(), KC, W, H, L, FW, FH, device=a.device)
    prob, _ = synth.make_ba_scene(4, 5, 20000, W, H, seed=synth.BASE_SEED + 3, m_con=8, n_con=2)
    opt = BaOptions.defaults()
    opt.device = a.device
    solver = api.BaSolver(prob.copy(), opt)

    def arm(kind):
        grp.first(host[0])
        klt_ba, klt_idle, lat, cpu, trial_us, results = [], [], [], [], [], []
        state = {"busy": False}
        p0 = time.process_time()
        grp.submit(host[1 % len(host)])
        for f in range(1, a.frames + 1):
            t0 = time.perf_counter()
            if f % a.ba_every == 0 and not state["busy"]:
                solver.reset(prob.copy())
                state.update(busy=True, t_req=t0, cpu=0.0)
                if kind == "thread":
                    def work():
                        c0 = time.thread_time()
                        state["info"] = solver.run()
                        state["result"] = solver.download().copy()
                        state["cpu"] = time.thread_time() - c0
                    state["th"] = threading.Thread(target=work)
                    state["th"].start()
                else:
                    c0 = time.thread_time()
                    solver.submit()
                    state["cpu"] += time.thread_time() - c0
            in_flight = state["busy"]
            if f < a.frames:
                grp.submit(host[(f + 1) % len(host)])
            grp.collect()
            if state["busy"]:  # bBusyBAing
                if kind == "thread":
                    finished = not state["th"].is_alive()
                    if finished:
                        state["th"].join()
                else:
                    c0 = time.thread_time()
                    finished = solver.done()
                    if finished:
                        state["info"] = solver.collect()
                        state["result"] = solver.download().copy()
                    state["cpu"] += time.thread_time() - c0
                if finished:
                    state["busy"] = False
                    lat.append(1e3 * (time.perf_counter() - state["t_req"]))
                    cpu.append(state["cpu"])
                    trial_us.append(1e6 * state["info"][11] / max(1.0, state["info"][10]))
                    results.append((state["info"].copy(), state["result"]))
            (klt_ba if in_flight else klt_idle).append(1e3 * (time.perf_counter() - t0))
        if state["busy"]:  # not picked up inside the window: finish it, do not count it
            if kind == "thread":
                state["th"].join()
            else:
                solver.collect()
        return {"klt_ms_ba": klt_ba, "klt_ms_idle": klt_idle, "ba_latency_ms": lat, "ba_cpu_s": cpu,
                "us_per_trial": trial_us, "proc_cpu_s_per_frame": [(time.process_time() - p0) / a.frames],
                "results": results}

    rounds = {"thread": [], "submit": []}
    for r in range(a.rounds):
        for kind in (("thread", "submit") if r % 2 == 0 else ("submit", "thread")):
            rounds[kind].append(arm(kind))
    # the two arms compute the same BA: every result against the first one
    allres = [(k, res) for k in rounds for rr in rounds[k] for res in rr["results"]]
    ref_info, ref_p = allres[0][1]
    same = {k: [] for k in rounds}
    for kind, (info, p) in allres:
        same[kind].append(bool(np.array_equal(info[5:11], ref_info[5:11]) and info[13] == ref_info[13]
                               and np.array_equal(p.outlier, ref_p.outlier)
                               and np.abs(p.R - ref_p.R).max() < 1e-9 and np.abs(p.X - ref_p.X).max() < 1e-8))

    def med(kind, key):
        v = [x for rr in rounds[kind][1:] for x in rr[key]]
        return round(float(np.median(v)), 4) if v else None

    keys = ("klt_ms_ba", "klt_ms_idle", "ba_latency_ms", "ba_cpu_s", "proc_cpu_s_per_frame", "us_per_trial")
    out = {
        "tool": "ba_async_rig",
        "card": bench.gpu_identity(a.device),
        "workload": f"c3: KLT 4 x {W}x{H} submit/collect frames, local BA (20 poses, 20k points, "
                    f"{opt.outer_iters} robust rounds x <= {opt.inner_iters} LM iterations) requested every "
                    f"{a.ba_every}th frame when none is in flight; {a.frames} frames per arm, {a.rounds - 1} timed rounds",
        "ba_per_arm": {k: sum(len(rr["results"]) for rr in rounds[k][1:]) for k in rounds},
        "lm_trials_per_ba": int(ref_info[10]),
        "results_equal_first": {k: f"{sum(v)}/{len(v)}" for k, v in same.items()},
        "thread": {k: med("thread", k) for k in keys},
        "submit": {k: med("submit", k) for k in keys},
    }
    print(json.dumps(out))
    solver.close()
    grp.close()


if __name__ == "__main__":
    main()
