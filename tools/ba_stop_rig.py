"""Stopping a stale local BA for a new key frame, on c3 (4 x 1280x720 KLT frames, live settings; local BA windows
of 20 poses / 20 k points, the oldest two key frames fixed, default robust options: 5 rounds x <= 10 iterations).
KLT frames go through cosl_klt_group_submit / _collect (frame n+1 submitted before frame n is collected); every
--ba-every-th frame requests a local BA of the next window (one of --windows problems, loaded with
cosl_ba_solver_load), and the SLAM thread checks once per frame whether the BA in flight has finished:

  refuse   the reference's policy (requestForBA while busy): a request that finds a BA in flight is dropped
  stop     the stale BA is stopped (cosl_ba_solver_stop), collected and discarded, and the new window is loaded
           and submitted

Reported per arm (median over the rounds after the warm-up round 0; the arms alternate in a round):
  requests / served / refused / stopped   BA requests made, BAs that ran to their end and were picked up,
                                          requests dropped, BAs stopped
  stop_to_done_ms          host clock from stop() until query reports the request done (stop arm)
  stopped_device_ms        info[11] of a stopped request: its device time from submit to the end of its loop
  stopped_trials           LM trials a stopped request had run
  klt_ms_ba / klt_ms_idle  ms per KLT frame set (submit + collect) with / without a BA in flight; the frame
                           that stops a BA includes the stop, the wait and the new load + submit

  python tools/ba_stop_rig.py [--frames 400] [--ba-every 10] [--rounds 4] [--windows 4]"""
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
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--ba-every", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()

    import torch

    from coslam_b200 import api, synth
    from coslam_b200.ctypes_defs import BaOptions

    if not torch.cuda.is_available():
        raise SystemExit("ba_stop_rig: needs a CUDA device")
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    seqs = bench.make_sequences(0)
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    grp = api.KltGroup(bench.klt_cfg(), KC, W, H, L, FW, FH, device=a.device)
    windows = [synth.make_ba_scene(4, 5, 20000, W, H, seed=synth.BASE_SEED + 3 + w, m_con=8, n_con=2)[0]
               for w in range(a.windows)]
    opt = BaOptions.defaults()
    opt.device = a.device
    solver = api.BaSolver(windows[0].copy(), opt)
    for w in windows:  # every window's graph shape once
        solver.load(w.copy())
        solver.submit()
        solver.collect()

    def arm(kind):
        grp.first(host[0])
        st = {"busy": False, "next": 0}
        out = {k: [] for k in ("klt_ms_ba", "klt_ms_idle", "stop_to_done_ms", "stopped_device_ms",
                               "stopped_trials")}
        cnt = {"requests": 0, "served": 0, "refused": 0, "stopped": 0}

        def start():
            solver.load(windows[st["next"] % len(windows)].copy())
            st["next"] += 1
            solver.submit()
            st["busy"] = True

        grp.submit(host[1 % len(host)])
        for f in range(1, a.frames + 1):
            t0 = time.perf_counter()
            in_flight = st["busy"]
            if f % a.ba_every == 0:
                cnt["requests"] += 1
                if not st["busy"]:
                    start()
                elif kind == "refuse":
                    cnt["refused"] += 1
                else:
                    ts = time.perf_counter()
                    solver.stop()
                    while not solver.done():
                        pass
                    out["stop_to_done_ms"].append(1e3 * (time.perf_counter() - ts))
                    info = solver.collect()
                    if info[6] == 8:
                        cnt["stopped"] += 1
                        out["stopped_device_ms"].append(1e3 * info[11])
                        out["stopped_trials"].append(info[10])
                    else:  # it had ended on its own: picked up as served
                        cnt["served"] += 1
                        solver.download()
                    start()
            if f < a.frames:
                grp.submit(host[(f + 1) % len(host)])
            grp.collect()
            if st["busy"] and solver.done():
                solver.collect()
                solver.download()
                cnt["served"] += 1
                st["busy"] = False
            (out["klt_ms_ba"] if in_flight or st["busy"] else out["klt_ms_idle"]).append(
                1e3 * (time.perf_counter() - t0))
        if st["busy"]:  # not picked up inside the window: finish it, do not count it
            solver.collect()
        out.update({k: [v] for k, v in cnt.items()})
        return out

    rounds = {"refuse": [], "stop": []}
    for r in range(a.rounds):
        for kind in (("refuse", "stop") if r % 2 == 0 else ("stop", "refuse")):
            rounds[kind].append(arm(kind))

    def med(kind, key):
        v = [x for rr in rounds[kind][1:] for x in rr[key]]
        return round(float(np.median(v)), 4) if v else None

    def mx(kind, key):
        v = [x for rr in rounds[kind][1:] for x in rr[key]]
        return round(float(np.max(v)), 4) if v else None

    keys = ("requests", "served", "refused", "stopped", "klt_ms_ba", "klt_ms_idle")
    res = {k: {key: med(k, key) for key in keys} for k in rounds}
    for key in ("stop_to_done_ms", "stopped_device_ms", "stopped_trials"):
        res["stop"][key] = med("stop", key)
        res["stop"][key + "_max"] = mx("stop", key)
    print(json.dumps({
        "tool": "ba_stop_rig",
        "card": bench.gpu_identity(a.device),
        "workload": f"c3: KLT 4 x {W}x{H} submit/collect frames, a local BA (20 poses, 20k points, {opt.outer_iters} "
                    f"robust rounds x <= {opt.inner_iters} LM iterations, {a.windows} windows in turn) requested every "
                    f"{a.ba_every}th frame; {a.frames} frames per arm, {a.rounds - 1} timed rounds; per-arm counts "
                    "are medians per round",
        **res,
    }))
    solver.close()
    grp.close()


if __name__ == "__main__":
    main()
