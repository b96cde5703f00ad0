"""The pose solver handle (cosl_pose_solver): the batch call's results bit for bit, the reference vectors,
submit that does not wait for the device, the state rules, and handles that do not block each other."""
import os
import threading
import time

import numpy as np
import pytest

from coslam_b200 import synth
from coslam_b200.ctypes_defs import PoseOpt

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pose_ref.npz")
OPT_FIELDS = [f for f, _ in PoseOpt._fields_]


def _batch_case(seeds_npts, prev_mask=None, seed=0):
    """(Ks, R0s, t0s, Ms, ms, prev) of synth pose cases; prev_mask[c] False gives camera c no prevErrs."""
    cases = [synth.make_pose_case(n_pts=n, seed=s) for s, n in seeds_npts]
    rng = np.random.default_rng(seed)
    prev = [np.abs(rng.normal(0, 4, len(c[3]))) for c in cases]
    if prev_mask is not None:
        prev = [p if keep else None for p, keep in zip(prev, prev_mask)]
    return ([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases],
            [c[4] for c in cases], prev)


def _empty_camera(case, c):
    """case with camera c given no points"""
    Ks, R0s, t0s, Ms, ms, prev = case
    Ms, ms, prev = list(Ms), list(ms), list(prev)
    Ms[c], ms[c] = np.empty((0, 3)), np.empty((0, 2))
    prev[c] = None if prev[c] is None else np.empty(0)
    return Ks, R0s, t0s, Ms, ms, prev


CASES = {
    # the cases of test_gpu_pose_ba.py::test_pose_prev_errs_and_batch
    "c4_prev": _batch_case([(10 + i, n) for i, n in enumerate((192, 150, 33, 192))], [True, True, False, True]),
    "c1": _batch_case([(40, 192)]),
    "c1_no_prev": _batch_case([(41, 120)], [False]),
    "c13": _batch_case([(50 + c, 60 + 11 * c) for c in range(13)], seed=1),
    "empty_camera": _empty_camera(_batch_case([(70 + c, 100) for c in range(4)], seed=2), 1),
    "mixed_prev": _batch_case([(80 + c, 90) for c in range(6)], [True, False, False, True, False, True], seed=3),
}


def _batch(api, case, tau=10.0):
    Ks, R0s, t0s, Ms, ms, prev = case
    return api.pose_intracam_batch(Ks, R0s, t0s, Ms, ms, tau, prev)


def _submit(s, case, tau=10.0):
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, tau, prev)


def _assert_same_bits(a, b):
    ok_a, R_a, t_a, op_a = a[:4]
    ok_b, R_b, t_b, op_b = b[:4]
    assert np.array_equal(ok_a, ok_b)
    assert np.array_equal(R_a.view(np.uint64), R_b.view(np.uint64))
    assert np.array_equal(t_a.view(np.uint64), t_b.view(np.uint64))
    assert len(op_a) == len(op_b)
    for c in range(len(op_a)):
        for f in OPT_FIELDS:
            x, y = getattr(op_a[c], f), getattr(op_b[c], f)
            assert np.array(x).tobytes() == np.array(y).tobytes(), (c, f, x, y)


@pytest.mark.parametrize("name", sorted(CASES))
def test_same_bits_as_the_batch_call(api, name):
    case = CASES[name]
    ref = _batch(api, case)
    s = api.PoseSolver(0, len(case[3]), sum(len(a) for a in case[3]))
    _submit(s, case)
    got = s.collect()
    _assert_same_bits(got, ref)
    assert got[4] > 0.0
    # the handle solves the next request as the first
    _submit(s, case)
    _assert_same_bits(s.collect(), ref)
    s.close()


def test_matches_the_oracle(api, orc):
    Ks, R0s, t0s, Ms, ms, prev = CASES["mixed_prev"]
    s = api.PoseSolver(0, 13, 4000)
    _submit(s, CASES["mixed_prev"])
    ok, R, t, opts, _ = s.collect()
    for c in range(len(Ms)):
        ok_o, R_o, t_o, op_o = orc.pose_intracam(Ks[c], R0s[c], t0s[c], Ms[c], ms[c], 10.0, prev[c])
        assert ok_o == ok[c] and opts[c].nIterRW == op_o.nIterRW
        assert np.abs(R_o - R[c]).max() < 1e-8 and np.abs(t_o - t[c]).max() < 1e-8
    s.close()


def _golden():
    d = np.load(G)
    for c in range(int(d["ncases"])):
        pe = d[f"c{c}_prev"]
        yield dict(K=d[f"c{c}_K"], R0=d[f"c{c}_R0"], t0=d[f"c{c}_t0"], Ms=d[f"c{c}_Ms"], ms=d[f"c{c}_ms"],
                   tau=float(d[f"c{c}_tau"]), prev=None if len(pe) == 0 else pe, ok=bool(d[f"c{c}_ok"]),
                   R=d[f"c{c}_R"], t=d[f"c{c}_t"], nIterRW=int(d[f"c{c}_opt"][7]))


def test_reference_vectors(api):
    """The golden cases of test_pose_ref.py::test_cuda_batch_matches_reference_vectors as one batch, and every
    golden case alone with its own tau: the batch call's bits, within 1e-8 of the compiled reference."""
    gs = list(_golden())
    s = api.PoseSolver(0, 4, 1000)
    cs = gs[:4]
    case = ([g["K"] for g in cs], [g["R0"] for g in cs], [g["t0"] for g in cs], [g["Ms"] for g in cs],
            [g["ms"] for g in cs], [g["prev"] for g in cs])
    _submit(s, case)
    got = s.collect()
    _assert_same_bits(got, _batch(api, case))
    ok, R, t = got[:3]
    n = 0
    for i, g in enumerate(cs):
        if g["tau"] != 10.0:
            continue
        assert ok[i] == g["ok"]
        assert np.abs(R[i] - g["R"]).max() < 1e-8 and np.abs(t[i] - g["t"]).max() < 1e-8
        n += 1
    assert n >= 1
    for g in gs:
        one = ([g["K"]], [g["R0"]], [g["t0"]], [g["Ms"]], [g["ms"]], [g["prev"]])
        _submit(s, one, g["tau"])
        got = s.collect()
        _assert_same_bits(got, _batch(api, one, g["tau"]))
        ok, R, t, opts, _ = got
        assert ok[0] == g["ok"] and opts[0].nIterRW == g["nIterRW"]
        assert np.abs(R[0] - g["R"]).max() < 1e-8 and np.abs(t[0] - g["t"]).max() < 1e-8
    s.close()


def _sleep_on(stream_ptr):
    """Queue a busy kernel of 1e9 SM cycles (0.5 s or more on an H100, whose SM clock is at most 1.98 GHz) on
    the handle's stream."""
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(stream_ptr)):
        torch.cuda._sleep(1_000_000_000)


def test_submit_does_not_wait_and_copies_its_inputs(api):
    case = CASES["c4_prev"]
    ref = _batch(api, case)
    Ks, R0s, t0s, Ms, ms, prev = [[np.array(a, np.float64) if a is not None else None for a in x] for x in case]
    s = api.PoseSolver(0, 4, 1000)
    assert s.stream()
    _sleep_on(s.stream())
    t0 = time.perf_counter()
    s.submit(Ks, R0s, t0s, Ms, ms, 10.0, prev)
    t_submit = time.perf_counter() - t0
    assert not s.done()
    for arrs in (Ks, R0s, t0s, Ms, ms, prev):  # the caller reuses its arrays
        for a in arrs:
            if a is not None:
                a.fill(np.nan)
    got = s.collect()
    t_all = time.perf_counter() - t0
    assert t_submit < 0.1 < t_all, (t_submit, t_all)
    _assert_same_bits(got, ref)
    assert 0.0 < got[4] < 100.0  # the copies and the kernel, not the sleep queued ahead of them
    s.close()


def test_state_rules(api):
    case = CASES["c4_prev"]
    ref = _batch(api, case)
    s = api.PoseSolver(0, 4, 600)
    with pytest.raises(api.CoslError, match="error -6"):
        s.done()
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    _submit(s, case)
    with pytest.raises(api.CoslError, match="error -6"):
        _submit(s, case)
    _assert_same_bits(s.collect(), ref)
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    # over capacity: too many cameras, too many points, then a request that fits
    with pytest.raises(api.CoslError, match="error -1"):
        _submit(s, CASES["mixed_prev"])
    with pytest.raises(api.CoslError, match="error -1"):
        _submit(s, _batch_case([(90, 300), (91, 301)]))
    # the checks of the batch call: options that differ between cameras, a bad camera
    Ks, R0s, t0s, Ms, ms, prev = case
    opts = (PoseOpt * 4)(*[PoseOpt.defaults() for _ in range(4)])
    opts[2].maxIterLM = 50
    with pytest.raises(api.CoslError, match="error -1"):
        s.submit(Ks, R0s, t0s, Ms, ms, 10.0, prev, opts)
    L = api.LIB
    args, _opts, keep = api._pose_batch_args(Ks, R0s, t0s, Ms, ms, 10.0, prev, None)
    bad = np.array([192, -1, 33, 192], np.int32)
    assert L.cosl_pose_solver_submit(s.h, args[0], args[1], args[2], args[3], bad.ctypes.data, *args[5:],
                                     _opts) == -1
    assert b"bad camera 1" in L.cosl_last_error()
    _submit(s, case)
    _assert_same_bits(s.collect(), ref)
    # destroy waits for a solve in flight
    t0 = time.perf_counter()
    _sleep_on(s.stream())
    _submit(s, case)
    assert L.cosl_pose_solver_destroy(s.h) == 0
    assert time.perf_counter() - t0 > 0.25
    s.h = None


def _solve_many(api, device, case, n, out, key):
    s = api.PoseSolver(device, len(case[3]), sum(len(a) for a in case[3]))
    res = []
    for _ in range(n):
        _submit(s, case)
        res.append(s.collect())
    s.close()
    out[key] = res


def _run_threads(api, jobs):
    out, threads = {}, []
    for key, (device, case) in jobs.items():
        threads.append(threading.Thread(target=_solve_many, args=(api, device, case, 50, out, key)))
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return out


def test_two_handles_on_two_threads(api):
    jobs = {"a": (0, CASES["c4_prev"]), "b": (0, CASES["mixed_prev"])}
    refs = {k: _batch(api, case) for k, (_, case) in jobs.items()}
    out = _run_threads(api, jobs)
    for k in jobs:
        assert len(out[k]) == 50
        for r in out[k]:
            _assert_same_bits(r, refs[k])


def test_one_handle_per_device(api):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    jobs = {d: (d, CASES["c4_prev"]) for d in (0, 1)}
    refs = {d: api.pose_intracam_batch(*CASES["c4_prev"][:5], 10.0, CASES["c4_prev"][5], device=d) for d in (0, 1)}
    out = _run_threads(api, jobs)
    for d in jobs:
        assert len(out[d]) == 50
        for r in out[d]:
            _assert_same_bits(r, refs[d])
