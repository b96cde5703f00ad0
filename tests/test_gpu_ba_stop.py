"""Stopping a bundle adjustment early (cosl_ba_solver_stop) and reading its progress without waiting
(cosl_ba_solver_progress).  A stopped loop ends its round with reason 8 at the next decision point, starts no
further round and still runs the outlier pass; with one robust round a BA stopped after k iterations leaves
what a fresh solve with inner_iters = k leaves.  A stop made with nothing running stops nothing."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

import ba_dense
from coslam_b200 import synth
from helpers import ba_same_decisions
from test_gpu_ba_async import SCENES, _opt, _sleep_on, _submitted, _torch_cuda

COSL_E_INVALID = -1
STOPPED = 8
gpu = pytest.mark.gpu


def _c3():
    """a c3 local BA window: 4 cameras x 5 key frames, 20 k points (about 0.12 ms per LM trial on the device)"""
    return synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=3, m_con=8, n_con=2)[0]


def _same_solution(want, got, prob):
    """ba_same_decisions for a stopped solve against a fresh one: the same counted iterations, cost, outliers
    and parameters (up to the order of the atomic sums); nfev / nlss and the stop reason may differ."""
    (iw, pw), (ig, pg) = want, got
    assert iw[5] == ig[5] and iw[13] == ig[13], (iw[:14], ig[:14])
    assert np.array_equal(pw.outlier, pg.outlier)
    assert abs(iw[12] - ig[12]) <= 1e-9 * iw[12] + 1e-12
    assert np.abs(pw.R - pg.R).max() < 1e-9 and np.abs(pw.t - pg.t).max() < 1e-9
    assert np.abs(pw.X - pg.X).max() < 1e-8
    assert np.array_equal(pg.R[:prob.m_con], prob.R[:prob.m_con])
    assert np.array_equal(pg.X[:prob.n_con], prob.X[:prob.n_con])


def _outliers_match_dense(state, opt):
    """the outlier flags of `state` are those of the float64 residuals at its parameters (|e| >= max_err),
    away from the threshold by more than the rounding of the device's residuals"""
    r = np.sqrt((ba_dense.residuals(state) ** 2).sum(1))
    want = r >= opt.max_err if opt.max_err > 0 else np.zeros(len(r), bool)
    clear = np.abs(r - opt.max_err) > 1e-9 * max(opt.max_err, 1.0)
    assert clear.mean() > 0.99
    assert np.array_equal(state.outlier.astype(bool)[clear], want[clear])


def _poll(s, until, timeout=30.0):
    """progress() records while the request runs, up to the first that satisfies `until`"""
    seen = []
    deadline = time.perf_counter() + timeout
    while time.perf_counter() < deadline:
        p = s.progress()
        seen.append(p)
        if until(p) or not p["running"]:
            break
    return seen


def _check_monotone(records):
    """counters of one robust round never decrease, its accepted cost never increases"""
    started = [p for p in records if p["round"] > 0]
    for a, b in zip(started, started[1:]):
        assert b["round"] >= a["round"] and b["iteration"] >= a["iteration"] and b["trials"] >= a["trials"], (a, b)
        assert b["cost"] <= a["cost"] and b["init_cost"] == a["init_cost"], (a, b)
        assert b["stop_requested"] >= a["stop_requested"], (a, b)


def _final_equals_info(p, info, rounds):
    assert not p["running"]
    assert p["round"] == rounds
    assert p["iteration"] == info[5] and p["trials"] == info[10]
    assert p["cost"] == info[12] == info[1]


def _warm(api, prob, opt):
    """a handle whose graph is built, reset to the start of `prob`"""
    s = api.BaSolver(prob.copy(), opt)
    s.submit()
    s.collect()
    s.reset(prob.copy())
    return s


@gpu
def test_stop_with_nothing_running_stops_nothing(api):
    make, opt = SCENES["c2_robust"]
    prob = make()
    want = _submitted(api, prob, opt)
    s = api.BaSolver(prob.copy(), opt)
    s.stop()  # before any request
    assert not s.progress()["running"] and not s.progress()["stop_requested"]
    s.submit()
    info = s.collect()
    assert info[6] != STOPPED
    ba_same_decisions(want, (info, s.download()), prob)
    s.stop()  # after the request has been collected: the next one runs to its end
    s.reset(prob.copy())
    s.submit()
    info = s.collect()
    ba_same_decisions(want, (info, s.download()), prob)
    s.reset(prob.copy())
    info = s.run()
    ba_same_decisions(want, (info, s.download()), prob)
    s.close()


@gpu
def test_stop_before_the_device_starts(api):
    torch = _torch_cuda()
    make, opt = SCENES["c2_robust"]
    prob = make()
    s = _warm(api, prob, opt)
    _sleep_on(torch, s, int(1.5e9))
    s.submit()
    s.stop()
    p = s.progress()
    assert p["running"] and p["stop_requested"] and p["round"] == 0
    info = s.collect()
    assert info[6] == STOPPED and info[5] == 0 and info[1] == info[0], info[:14]
    got = s.download()
    fresh = api.BaSolver(prob.copy(), opt)
    start = fresh.download()
    fresh.close()
    assert np.array_equal(got.R, start.R) and np.array_equal(got.t, prob.t) and np.array_equal(got.X, prob.X)
    assert info[13] == got.outlier.sum()
    _outliers_match_dense(got, opt)
    _final_equals_info(s.progress(), info, 1)
    s.close()


def _replay_matches(api, prob, info, got):
    k = int(info[5])
    want = _submitted(api, prob, _opt(1, k))
    _same_solution(want, got, prob)


@gpu
def test_stop_mid_run_submitted(api):
    prob, opt = _c3(), _opt(1, 10)
    s = _warm(api, prob, opt)
    s.submit()
    seen = _poll(s, lambda p: p["iteration"] >= 2)
    s.stop()
    info = s.collect()
    final = s.progress()
    got = (info, s.download())
    s.close()
    _check_monotone(seen + [final])
    _final_equals_info(final, info, 1)
    if info[6] != STOPPED:
        print(f"the BA had ended with reason {int(info[6])} before the stop reached it")
        return
    _replay_matches(api, prob, info, got)


@gpu
def test_stop_a_synchronous_run_from_another_thread(api):
    prob, opt = _c3(), _opt(1, 10)
    s = api.BaSolver(prob.copy(), opt)
    seen, finished = [], threading.Event()

    def helper():
        deadline = time.perf_counter() + 30.0
        while not finished.is_set() and time.perf_counter() < deadline:
            p = s.progress()
            if p["running"]:
                seen.append(p)
                if p["iteration"] >= 2:
                    s.stop()
                    return

    th = threading.Thread(target=helper)
    th.start()
    info = s.run()  # ctypes releases the GIL for the call
    finished.set()
    th.join()
    final = s.progress()
    got = (info, s.download())
    s.close()
    assert seen, "the helper thread never saw the run"
    _check_monotone(seen + [final])
    _final_equals_info(final, info, 1)
    if info[6] != STOPPED:
        print(f"the BA had ended with reason {int(info[6])} before the stop reached it")
        return
    _replay_matches(api, prob, info, got)


@gpu
def test_stop_during_a_multi_round_robust_ba(api):
    prob, opt = _c3(), _opt(5, 10)
    s = _warm(api, prob, opt)
    s.submit()
    seen = _poll(s, lambda p: p["round"] >= 2 and p["iteration"] >= 1)
    at = seen[-1]
    s.stop()
    info = s.collect()
    final = s.progress()
    got = s.download()
    s.close()
    _final_equals_info(final, info, final["round"])
    if info[6] != STOPPED:
        print(f"the BA had ended with reason {int(info[6])} before the stop reached it")
        return
    assert at["round"] >= 2 and final["round"] == at["round"], (at, final)
    assert info[12] <= at["init_cost"]
    assert np.isfinite(got.R).all() and np.isfinite(got.t).all() and np.isfinite(got.X).all()
    assert info[13] == got.outlier.sum()
    _outliers_match_dense(got, opt)


@gpu
def test_handle_after_a_stop(api):
    prob, opt = _c3(), _opt(2, 10)
    s = _warm(api, prob, opt)
    s.submit()
    _poll(s, lambda p: p["iteration"] >= 1)
    s.stop()
    s.collect()
    make, _ = SCENES["c2_robust"]
    other = make()
    want = _submitted(api, other, opt)
    s.load(other.copy())
    s.submit()
    got = (s.collect(), s.download())
    s.close()
    ba_same_decisions(want, got, other)


@gpu
@pytest.mark.skipif(not (_torch_cuda() and _torch_cuda().cuda.device_count() >= 2), reason="needs two GPUs")
def test_multi_rank_solver_refuses_stop(api):
    L = api.LIB
    uid = (C.c_uint8 * 128)()
    assert L.cosl_nccl_unique_id(uid) == 0
    prob = synth.make_ba_scene(2, 3, 400, 320, 240, seed=6, m_con=2, n_con=2)[0]
    rc = [None, None]

    def rank(r):
        comm = C.c_void_p()
        assert L.cosl_ba_comm_create(uid, r, 2, r, C.byref(comm)) == 0
        opt = _opt()
        opt.device = r
        p = prob.copy()
        h = C.c_void_p()
        assert L.cosl_ba_solver_create(C.byref(p.struct()), C.byref(opt), comm, C.byref(h)) == 0
        rc[r] = L.cosl_ba_solver_stop(h)
        L.cosl_ba_solver_destroy(h)
        L.cosl_ba_comm_destroy(comm)

    th = [threading.Thread(target=rank, args=(r,)) for r in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert rc == [COSL_E_INVALID, COSL_E_INVALID]
