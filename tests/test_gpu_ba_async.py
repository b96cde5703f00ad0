"""Non-blocking bundle adjustment (cosl_ba_solver_submit / _query / _collect): the device-controlled
robust loop takes the decisions of cosl_ba_solver_run -- same iterations, stop reason, evaluation
counters, trials and outliers, and the oracle's solution -- returns to the caller before the device has
run it, keeps the state rules of the solver handle, and runs beside a KLT camera group without changing
its tables.  The last four tests need no GPU."""
import ctypes as C
import os
import re
import threading
import time

import numpy as np
import pytest

from coslam_b200 import synth
from coslam_b200.ctypes_defs import BaOptions
from helpers import ba_same_decisions, live_cfg, seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA, COSL_E_STATE = -1, -2, -6
gpu = pytest.mark.gpu


def _torch_cuda():
    try:
        import torch
        return torch if torch.cuda.is_available() else None
    except Exception:
        return None


def _opt(outer=2, inner=10, max_err=6.0, **opts):
    o = BaOptions.defaults()
    o.outer_iters, o.inner_iters, o.max_err = outer, inner, max_err
    for k, v in opts.items():
        o.opts[int(k[1:])] = v
    return o


SCENES = {
    # c2: 2 cams x 5 key frames, oldest 2 key frames fixed
    "c2_robust": (lambda: synth.make_ba_scene(2, 5, 5000, 640, 480, seed=7, m_con=4, n_con=2)[0], _opt()),
    "c2_plain": (lambda: synth.make_ba_scene(2, 5, 5000, 640, 480, seed=7, m_con=4, n_con=2)[0], _opt(max_err=0.0)),
    # InterCamPoseEstimator pattern: every camera free, most points fixed.  With eps2 = 1e-12 its 40
    # iterations per round run on at the noise floor, where a cost decrease is about 1e-16 of the cost and
    # its sign depends on the order of the device's atomic sums, so the accept decisions there are not
    # reproducible; eps2 = 1e-6 ends each round while every decision is far from a tie
    "intercam": (lambda: synth.make_ba_scene(4, 1, 400, 640, 480, seed=9, m_con=0, n_con=340, window=0,
                                             p_vis=1.0)[0], _opt(3, 40, o2=1e-6)),
    # 12 key frames, one fixed point, two robust rounds
    "kf12": (lambda: synth.make_ba_scene(4, 12, 2500, 1280, 720, seed=33, m_con=4, n_con=1)[0], _opt(2, 6)),
}


def _run(api, prob, opt):
    s = api.BaSolver(prob.copy(), opt)
    info = s.run()
    p = s.download()
    s.close()
    return info, p


def _submitted(api, prob, opt):
    s = api.BaSolver(prob.copy(), opt)
    s.submit()
    info = s.collect()
    p = s.download()
    s.close()
    return info, p


def _oracle_close(orc, prob, opt, got):
    """the tolerances of test_gpu_pose_ba._ba_compare"""
    ig, pg = got
    po = prob.copy()
    io = orc.ba_solve(po, opt)
    assert abs(ig[1] - io[1]) <= 1e-6 * io[1] + 1e-9, (ig[:10], io[:10])
    assert np.abs(pg.R - po.R).max() < 1e-6 and np.abs(pg.t - po.t).max() < 1e-6
    assert np.abs(pg.X - po.X).max() < 1e-5


@gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_submit_matches_run_and_oracle(api, orc, name):
    make, opt = SCENES[name]
    prob = make()
    want = _run(api, prob, opt)
    got = _submitted(api, prob, opt)
    ba_same_decisions(want, got, prob)
    _oracle_close(orc, prob, opt, got)


def _weightless_point(prob):
    """a free point seen only by fixed cameras, every observation far beyond max_err: its weights are 0,
    so V = 0 and with tau = 0 (mu = 0) its damped inverse is NaN, which makes the first trial's cost
    non-finite (the point has no free camera, so the reduced system stays finite)"""
    p = prob.copy()
    i = p.n_con
    o0, o1 = int(p.ptr[i]), int(p.ptr[i + 1])
    assert 0 < o1 - o0 <= p.m_con
    p.cam[o0:o1] = np.arange(o1 - o0, dtype=np.int32)
    p.xy[o0:o1] += 500.0
    return p


def _edge_cases():
    c2 = lambda: synth.make_ba_scene(2, 5, 3000, 640, 480, seed=7, m_con=4, n_con=2)[0]  # noqa: E731
    return {
        # no free camera: the ns == 0 launch sequence
        "no_free_camera": (lambda: synth.make_ba_scene(2, 3, 400, 320, 240, seed=6, m_con=6, n_con=2)[0], _opt()),
        # reduced system of <= 2 blocks (ba_tile_two) / larger than a CTA (blocked solve)
        "two_blocks": (c2, _opt()),
        "blocked": (lambda: synth.make_ba_scene(4, 12, 3000, 640, 480, seed=5, m_con=4, n_con=0,
                                                outlier_frac=0.0)[0], _opt(1, 6, max_err=0.0)),
        "eps1_at_first_iteration": (c2, _opt(o1=1e30)),
        "eps2": (c2, _opt(o2=1e-2)),
        "eps3": (c2, _opt(1, 10, max_err=0.0, o3=1e30)),
        "one_inner_iteration": (c2, _opt(3, 1)),
        "non_finite_trial_cost": (lambda: _weightless_point(synth.make_ba_scene(2, 5, 3000, 640, 480, seed=7,
                                                                                m_con=4, n_con=2)[0]),
                                  _opt(1, 10, o0=0.0)),
    }


@gpu
@pytest.mark.parametrize("name", list(_edge_cases()))
def test_edge_shapes_and_stop_reasons(api, name):
    make, opt = _edge_cases()[name]
    prob = make()
    want = _run(api, prob, opt)
    got = _submitted(api, prob, opt)
    ba_same_decisions(want, got, prob)
    s = api.BaSolver(prob.copy(), opt)
    plan, ns = s.plan_info(), s.stats()["ns"]
    s.close()
    stop = int(got[0][6])
    if name == "no_free_camera":
        assert ns == 0
    if name == "two_blocks":
        assert plan["small_solve"] == 1
    if name == "blocked":
        assert plan["small_solve"] == 0 and plan["blocks"] > 2
    if name == "eps1_at_first_iteration":
        assert stop == 1 and got[0][5] == 0 and got[0][9] == 0
    if name == "eps2":
        assert stop == 2
    if name == "eps3":
        assert stop == 3 and got[0][5] == 1
    if name == "one_inner_iteration":
        assert got[0][5] == 1
    if name == "non_finite_trial_cost":
        assert stop == 7 and got[0][9] >= 1


@gpu
def test_submit_returns_before_the_device_runs_it(api):
    torch = _torch_cuda()
    make, opt = SCENES["c2_robust"]
    prob = make()
    want = _run(api, prob, opt)
    s = api.BaSolver(prob.copy(), opt)
    s.submit()  # the first submit builds the graph; time a later one
    s.collect()
    s.reset(prob.copy())
    ext = torch.cuda.ExternalStream(s.stream())
    with torch.cuda.stream(ext):
        t0 = time.perf_counter()
        torch.cuda._sleep(int(1.5e9))  # about a second at H100 clocks
    s.submit()
    dt = time.perf_counter() - t0
    assert dt < 0.25, dt
    assert not s.done()
    info = s.collect()
    ba_same_decisions(want, (info, s.download()), prob)
    s.close()


@gpu
def test_reuse_and_mixing_with_run(api):
    make, opt = SCENES["kf12"]
    prob = make()
    want = _run(api, prob, opt)
    s = api.BaSolver(prob.copy(), opt)
    for what in ("submit", "submit", "run", "submit", "run", "run", "submit"):
        s.reset(prob.copy())
        if what == "run":
            info = s.run()
        else:
            s.submit()
            deadline = time.perf_counter() + 30.0
            while not s.done() and time.perf_counter() < deadline:
                time.sleep(1e-4)
            info = s.collect()
        ba_same_decisions(want, (info, s.download()), prob)
    s.close()


def _sleep_on(torch, s, cycles=int(3e8)):
    with torch.cuda.stream(torch.cuda.ExternalStream(s.stream())):
        torch.cuda._sleep(cycles)


@gpu
def test_state_errors(api):
    torch = _torch_cuda()
    L = api.LIB
    make, opt = SCENES["c2_robust"]
    prob = make()
    s = api.BaSolver(prob.copy(), opt)
    info = np.zeros(16)
    done = C.c_int(-1)
    assert L.cosl_ba_solver_query(s.h, C.byref(done)) == COSL_E_STATE
    assert L.cosl_ba_solver_collect(s.h, info.ctypes.data) == COSL_E_STATE
    _sleep_on(torch, s)
    assert L.cosl_ba_solver_submit(s.h) == 0
    st = prob.struct()
    assert L.cosl_ba_solver_run(s.h, info.ctypes.data) == COSL_E_STATE
    assert L.cosl_ba_solver_run_fixed(s.h, 3, info.ctypes.data) == COSL_E_STATE
    assert L.cosl_ba_solver_reset(s.h, C.byref(st)) == COSL_E_STATE
    assert L.cosl_ba_solver_download(s.h, C.byref(st)) == COSL_E_STATE
    assert L.cosl_ba_solver_submit(s.h) == COSL_E_STATE
    assert L.cosl_ba_solver_query(s.h, None) == COSL_E_INVALID
    assert L.cosl_ba_solver_query(s.h, C.byref(done)) == 0 and done.value == 0
    assert L.cosl_ba_solver_collect(s.h, info.ctypes.data) == 0
    assert info[10] > 0
    assert L.cosl_ba_solver_collect(s.h, info.ctypes.data) == COSL_E_STATE
    assert L.cosl_ba_solver_query(s.h, C.byref(done)) == COSL_E_STATE
    assert L.cosl_ba_solver_download(s.h, C.byref(st)) == 0
    # destroy with a submit in flight waits for it
    _sleep_on(torch, s)
    assert L.cosl_ba_solver_reset(s.h, C.byref(prob.struct())) == 0
    assert L.cosl_ba_solver_submit(s.h) == 0
    s.close()
    torch.cuda.synchronize()


@gpu
@pytest.mark.skipif(not (_torch_cuda() and _torch_cuda().cuda.device_count() >= 2), reason="needs two GPUs")
def test_multi_rank_solver_refuses_submit(api):
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
        rc[r] = L.cosl_ba_solver_submit(h)
        L.cosl_ba_solver_destroy(h)
        L.cosl_ba_comm_destroy(comm)

    th = [threading.Thread(target=rank, args=(r,)) for r in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert rc == [COSL_E_INVALID, COSL_E_INVALID]


@gpu
def test_concurrent_with_klt_tracking(api, orc):
    """a c3 local BA submitted while a c3 KLT group runs submitted frames on its own stream: the KLT
    tables are those of the same frames without the BA, the BA's result that of run"""
    W, H, NF = 1280, 720, 8
    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 700 + c, n=NF) for c in range(4)]
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731

    def klt_run(ba=None):
        g = api.KltGroup(cfg, 4, W, H, 6, 32, 32)
        g.first(frames(0))
        out = []
        for k in range(1, NF):
            g.submit(frames(k))
            if k == 2 and ba is not None:
                ba.submit()
            if k > 1:
                f, n = g.collect()
                out.append((f.copy(), n.copy()))
        f, n = g.collect()
        out.append((f.copy(), n.copy()))
        g.close()
        return out

    prob = synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=3, m_con=8, n_con=2)[0]
    opt = _opt(2, 10)
    want_ba = _run(api, prob, opt)
    want = klt_run()
    s = api.BaSolver(prob.copy(), opt)
    got = klt_run(s)
    info = s.collect()
    got_ba = (info, s.download())
    s.close()
    assert len(want) == len(got)
    for k, ((fw, nw), (fg, ng)) in enumerate(zip(want, got)):
        assert np.array_equal(nw, ng), k
        assert fw.tobytes() == fg.tobytes(), k
    ba_same_decisions(want_ba, got_ba, prob)
    _oracle_close(orc, prob, opt, got_ba)


# ---------------------------------------------------------------- no GPU needed
def test_header_declares_the_calls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    for name, args in (("submit", ["cosl_ba_solver* s"]), ("query", ["cosl_ba_solver* s", "int* done"]),
                       ("collect", ["cosl_ba_solver* s", "double info[COSL_BA_INFOSZ]"])):
        decl = re.search(r"\bint\s+cosl_ba_solver_%s\s*\(([^)]*)\)\s*;" % name, src)
        assert decl, name
        assert [a.strip() for a in decl.group(1).split(",")] == args


def test_library_exports_the_calls_and_the_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    for name in ("submit", "query", "collect"):
        assert hasattr(lib, "cosl_ba_solver_" + name)
        assert callable(getattr(api.BaSolver, {"query": "done"}.get(name, name), None))
    assert api.LIB.cosl_ba_solver_query.argtypes == [C.c_void_p, C.POINTER(C.c_int)]


def test_null_handle_is_invalid(api):
    info = np.zeros(16)
    done = C.c_int(0)
    assert api.LIB.cosl_ba_solver_submit(None) == COSL_E_INVALID
    assert api.LIB.cosl_ba_solver_query(None, C.byref(done)) == COSL_E_INVALID
    assert api.LIB.cosl_ba_solver_collect(None, info.ctypes.data) == COSL_E_INVALID


@pytest.mark.skipif(_torch_cuda() is not None, reason="checks the no-GPU failure mode")
def test_no_solver_without_a_gpu(api):
    """Without a device there is no solver to submit to: creation reports COSL_E_CUDA and leaves the
    handle NULL, which submit refuses (no CPU fallback)."""
    prob = synth.make_ba_scene(2, 3, 200, 320, 240, seed=6, m_con=2, n_con=2)[0]
    h = C.c_void_p()
    assert api.LIB.cosl_ba_solver_create(C.byref(prob.struct()), C.byref(_opt()), None, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    assert api.LIB.cosl_ba_solver_submit(h) == COSL_E_INVALID
