"""Per-camera frame ops (cosl_klt_group_step, _submit_step) on c3: 4 x 1280x720, 2000 slots, live settings.
Prints one JSON line (card name and power limit included).

  all_next   all-NEXT steps against cosl_klt_group_next of the same build, and (--parent-lib) of
             another build of the library: ms per frame set, tables compared bit for bit
  cadence    first, then cycles of 4 x TRACK + 1 x NEXT on every camera: one group through
             group_step against 4 single trackers (track / redetect + advance) and against
             all-NEXT group_next frames
  skip_rig   camera 3 skipped on every other step (the others re-detect): group_step against
             4 single trackers that get the same frames, and against all-NEXT
  pipelined  the cadence and the skip rig through cosl_klt_group_submit_step / _collect (step n+1
             submitted before step n is collected), against their group_step arms; and all-NEXT
             frames through cosl_klt_group_submit / _collect, the pipelined form of group_next
  exchange   device time (CUDA events) of exchanging one camera's pyramid slices
             (cosl_klt_group_advance_cams of camera 3), which a step skipping one camera of four pays

Frames come from pinned host buffers; every synchronous arm synchronises once per frame set, every
pipelined arm collects (reads back and waits for) every frame set.  Round 0 of each arm is a
warm-up; the arms alternate within a round.

  python tools/klt_step_rig.py [--frames 40] [--rounds 3] [--parent-lib PATH]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402  (c3 geometry, sequences, tracker settings, card identity)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--parent-lib", default=None, help="another build's libcoslam_b200.so for all_next")
    a = ap.parse_args()
    import torch
    from coslam_b200 import api
    from coslam_b200.ctypes_defs import COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK, FEAT_DTYPE
    torch.cuda.set_device(a.device)
    KC, W, H, FW, FH, L = bench.KLT_C, bench.KLT_W, bench.KLT_H, bench.KLT_FW, bench.KLT_FH, bench.KLT_L
    F = FW * FH
    cfg = bench.klt_cfg()
    seqs = bench.make_sequences(0)
    fidx = seqs[0].frame_index
    host = [[torch.from_numpy(seqs[c].frames[k]).pin_memory().numpy() for c in range(KC)]
            for k in range(bench.KLT_FRAMES)]
    n_frames = a.frames
    nb = C.c_int(0)
    ops_next = np.full(KC, COSL_KLT_OP_NEXT, np.uint8)
    ops_track = np.full(KC, COSL_KLT_OP_TRACK, np.uint8)
    ops_skip3 = ops_next.copy()
    ops_skip3[3] = COSL_KLT_OP_SKIP
    cadence = [ops_track if f % 5 < 4 else ops_next for f in range(n_frames)]
    skip_rig = [ops_skip3 if f % 2 == 0 else ops_next for f in range(n_frames)]

    grp = api.KltGroup(cfg, KC, W, H, L, FW, FH, device=a.device)
    args = [grp.host_ptrs(row) for row in host]
    singles = [api.KltTracker(cfg, W, H, L, FW, FH, device=a.device) for _ in range(KC)]
    dest = grp._dest
    counts = grp.counts.ctypes.data

    def step(ops, k):
        ptrs, pitch = args[fidx(k)]
        api._ck(api.LIB.cosl_klt_group_step(grp.h, ops.ctypes.data, ptrs, pitch, dest, counts))

    def group_sched(sched):
        grp.first(host[0])
        t0 = time.perf_counter()
        for f, ops in enumerate(sched):
            step(ops, f + 1)
        return time.perf_counter() - t0, grp.feats.copy()

    def submit_step(ops, k):
        ptrs, pitch = args[fidx(k)]
        api._ck(api.LIB.cosl_klt_group_submit_step(grp.h, ops.ctypes.data, ptrs, pitch))

    def submit_next(_ops, k):
        ptrs, pitch = args[fidx(k)]
        api._ck(api.LIB.cosl_klt_group_submit(grp.h, ptrs, pitch))

    def collect():
        api._ck(api.LIB.cosl_klt_group_collect(grp.h, dest, counts))

    def group_pipelined(sched, submit):
        """frame set f + 1 submitted before f is collected; every frame set collected"""
        grp.first(host[0])
        t0 = time.perf_counter()
        submit(sched[0], 1)
        for f in range(1, len(sched)):
            submit(sched[f], f + 1)
            collect()
        collect()
        return time.perf_counter() - t0, grp.feats.copy()

    def group_next():
        grp.first(host[0])
        t0 = time.perf_counter()
        for f in range(n_frames):
            grp.next_raw(args[fidx(f + 1)])
        return time.perf_counter() - t0, grp.feats.copy()

    def singles_sched(sched):
        for c in range(KC):
            singles[c].detect(host[0][c])
            singles[c].advance()
        t0 = time.perf_counter()
        for f, ops in enumerate(sched):
            row = host[fidx(f + 1)]
            for c in range(KC):
                if ops[c] == COSL_KLT_OP_SKIP:
                    continue
                call = api.LIB.cosl_klt_track if ops[c] == COSL_KLT_OP_TRACK else api.LIB.cosl_klt_redetect
                api._ck(call(singles[c].h, row[c].ctypes.data, W, C.byref(singles[c].feats), C.byref(nb)))
                api._ck(api.LIB.cosl_klt_advance(singles[c].h))
        return time.perf_counter() - t0, np.stack([s._out() for s in singles])

    parent = None
    if a.parent_lib:
        P = C.CDLL(os.path.abspath(a.parent_lib))
        vp = C.c_void_p
        P.cosl_klt_group_create.argtypes = [C.POINTER(type(cfg))] + [C.c_int] * 9 + [C.POINTER(vp)]
        P.cosl_klt_group_first.argtypes = [vp, vp, C.c_size_t, vp, vp]
        P.cosl_klt_group_next.argtypes = [vp, vp, C.c_size_t, vp, vp]
        P.cosl_klt_destroy.argtypes = [vp]
        ph = vp()
        assert P.cosl_klt_group_create(C.byref(cfg), KC, W, H, L, FW, FH, 0, 0, a.device, C.byref(ph)) == 0
        pfeats = np.zeros((KC, F), FEAT_DTYPE)
        pcounts = np.zeros(KC, np.int32)
        pdest = (C.c_void_p * KC)(*[pfeats[c].ctypes.data for c in range(KC)])
        parent = (P, ph, pfeats, pcounts, pdest)

    def parent_next():
        P, ph, pfeats, pcounts, pdest = parent
        p0, pitch0 = args[fidx(0)]
        assert P.cosl_klt_group_first(ph, p0, pitch0, pdest, pcounts.ctypes.data) == 0
        t0 = time.perf_counter()
        for f in range(n_frames):
            ptrs, pitch = args[fidx(f + 1)]
            assert P.cosl_klt_group_next(ph, ptrs, pitch, pdest, pcounts.ctypes.data) == 0
        return time.perf_counter() - t0, pfeats.copy()

    arms = {
        "all_next_step": lambda: group_sched([ops_next] * n_frames),
        "all_next_group_next": group_next,
        "cadence_step": lambda: group_sched(cadence),
        "cadence_singles": lambda: singles_sched(cadence),
        "skip_rig_step": lambda: group_sched(skip_rig),
        "skip_rig_singles": lambda: singles_sched(skip_rig),
        "cadence_submit_step": lambda: group_pipelined(cadence, submit_step),
        "skip_rig_submit_step": lambda: group_pipelined(skip_rig, submit_step),
        "all_next_submit": lambda: group_pipelined([ops_next] * n_frames, submit_next),
    }
    if parent:
        arms["all_next_parent_group_next"] = parent_next
    times = {k: [] for k in arms}
    same = {"all_next_step_vs_group_next": True, "cadence_step_vs_singles": True,
            "skip_rig_step_vs_singles": True, "cadence_submit_step_vs_step": True,
            "skip_rig_submit_step_vs_step": True, "all_next_submit_vs_group_next": True}
    if parent:
        same["all_next_group_next_vs_parent"] = True
    stream = torch.cuda.ExternalStream(grp.stream(), device=a.device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def exchange_ms(n=20):
        ms = []
        for _ in range(n):
            ev0.record(stream)
            grp.advance([3])
            ev1.record(stream)
            grp.sync()
            ms.append(ev0.elapsed_time(ev1))
        return float(np.median(ms))

    exch = []
    for r in range(a.rounds + 1):
        out = {}
        for k, fn in arms.items():
            dt, out[k] = fn()
            if r:
                times[k].append(1e3 * dt / n_frames)
        same["all_next_step_vs_group_next"] &= out["all_next_step"].tobytes() == out["all_next_group_next"].tobytes()
        same["cadence_step_vs_singles"] &= out["cadence_step"].tobytes() == out["cadence_singles"].tobytes()
        same["skip_rig_step_vs_singles"] &= out["skip_rig_step"].tobytes() == out["skip_rig_singles"].tobytes()
        same["cadence_submit_step_vs_step"] &= out["cadence_submit_step"].tobytes() == out["cadence_step"].tobytes()
        same["skip_rig_submit_step_vs_step"] &= (out["skip_rig_submit_step"].tobytes()
                                                 == out["skip_rig_step"].tobytes())
        same["all_next_submit_vs_group_next"] &= (out["all_next_submit"].tobytes()
                                                  == out["all_next_group_next"].tobytes())
        if r:
            exch.append(exchange_ms())
        if parent:
            same["all_next_group_next_vs_parent"] &= (out["all_next_group_next"].tobytes()
                                                      == out["all_next_parent_group_next"].tobytes())
    grp.close()
    for s in singles:
        s.close()
    if parent:
        parent[0].cosl_klt_destroy(parent[1])
    ms = {k: {"ms_per_frame_set": float(np.mean(v)), "range": [min(v), max(v)]} for k, v in times.items()}
    m = {k: v["ms_per_frame_set"] for k, v in ms.items()}
    print(json.dumps({
        "metric": "cadence_ms_per_frame_set", "value": m["cadence_step"], "unit": "ms", "higher_is_better": False,
        "arms": ms,
        "ratios": {"all_next_step_over_group_next": m["all_next_step"] / m["all_next_group_next"],
                   "cadence_singles_over_step": m["cadence_singles"] / m["cadence_step"],
                   "cadence_step_over_all_next": m["cadence_step"] / m["all_next_group_next"],
                   "skip_rig_singles_over_step": m["skip_rig_singles"] / m["skip_rig_step"],
                   "skip_rig_step_over_all_next": m["skip_rig_step"] / m["all_next_group_next"],
                   "cadence_submit_step_over_step": m["cadence_submit_step"] / m["cadence_step"],
                   "skip_rig_submit_step_over_step": m["skip_rig_submit_step"] / m["skip_rig_step"],
                   "cadence_submit_step_over_all_next_submit": m["cadence_submit_step"] / m["all_next_submit"],
                   **({"group_next_over_parent": m["all_next_group_next"] / m["all_next_parent_group_next"]}
                      if parent else {})},
        "exchange_one_camera_device_ms": {"ms": float(np.mean(exch)), "range": [min(exch), max(exch)]},
        "bit_identical": same,
        "config": {"workload": f"c3 ({KC} x {W}x{H}, {F} slots, live settings), first + {n_frames} frame sets "
                               "through pinned host buffers, one synchronise (synchronous arms) or one "
                               "collect (pipelined arms) per frame set",
                   "cadence": "4 x TRACK + 1 x NEXT on every camera",
                   "skip_rig": "camera 3 skipped on every other step, the others NEXT",
                   "rounds": a.rounds, "parent_lib": bool(parent)},
        "gpu": bench.gpu_identity(a.device)}))


if __name__ == "__main__":
    main()
