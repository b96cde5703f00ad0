"""Loading new problems into a live BA solver (cosl_ba_solver_load): after each load of a differently shaped
problem into one handle, run and submit / collect take the decisions of a fresh cosl_ba_solver_create + run
on that problem, with its solution, statistics and solve plan; load returns before the device has set the
problem up, owns copies of its input, refuses malformed problems without losing the loaded one, and keeps
the state rules of the handle.  The tests at the end need no GPU."""
import ctypes as C
import os
import re
import threading
import time

import numpy as np
import pytest

from coslam_b200 import synth
from coslam_b200.ctypes_defs import BaOptions
from coslam_b200.problem import BAProblem
from helpers import ba_same_decisions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA, COSL_E_STATE = -1, -2, -6
gpu = pytest.mark.gpu


def _torch_cuda():
    try:
        import torch
        return torch if torch.cuda.is_available() else None
    except Exception:
        return None


# eps2 = 1e-6 ends each round while every accept decision is far from a tie (the inter-camera pattern runs on
# at the noise floor with eps2 = 1e-12, where the decisions depend on the order of the device's atomic sums)
def _opt():
    o = BaOptions.defaults()
    o.outer_iters, o.inner_iters, o.max_err = 2, 10, 6.0
    o.opts[2] = 1e-6
    return o


def _no_points(prob):
    z = np.zeros(0)
    return BAProblem(prob.K, prob.R, prob.t, z.reshape(0, 3), np.zeros(1, np.int64), np.zeros(0, np.int32),
                     z.reshape(0, 2), prob.m_con, 0)


def _c2():
    return synth.make_ba_scene(2, 5, 5000, 640, 480, seed=synth.BASE_SEED + 2, m_con=4, n_con=2)[0]


def _c3():
    return synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=synth.BASE_SEED + 3, m_con=8, n_con=2)[0]


# growing and shrinking, in this order
SEQUENCE = [
    ("c2_local", _c2),
    ("c3_local", _c3),
    ("intercam", lambda: synth.make_ba_scene(4, 1, 985, 640, 480, seed=9, m_con=0, n_con=800, window=0,
                                             p_vis=1.0)[0]),  # 58 free points
    ("no_free_camera", lambda: synth.make_ba_scene(2, 3, 400, 320, 240, seed=6, m_con=6, n_con=2)[0]),
    ("one_free_camera", lambda: synth.make_ba_scene(1, 3, 400, 320, 240, seed=8, m_con=2, n_con=2)[0]),
    ("free_10", lambda: synth.make_ba_scene(2, 6, 3000, 640, 480, seed=11, m_con=2, n_con=1)[0]),
    ("free_11", lambda: synth.make_ba_scene(1, 12, 3000, 640, 480, seed=12, m_con=1, n_con=1)[0]),
    ("free_20", lambda: synth.make_ba_scene(4, 6, 3000, 640, 480, seed=13, m_con=4, n_con=1)[0]),
    ("free_28", lambda: synth.make_ba_scene(4, 8, 3000, 640, 480, seed=14, m_con=4, n_con=1)[0]),
    ("no_points", lambda: _no_points(_c2())),
    ("c4_slice_40kf", lambda: synth.make_ba_scene(4, 40, 10000, 1280, 720, seed=synth.BASE_SEED + 4, m_con=4,
                                                  n_con=0)[0]),
]


def _fresh(api, prob, opt):
    s = api.BaSolver(prob.copy(), opt)
    info = s.run()
    p = s.download()
    st, plan = s.stats(), s.plan_info()
    s.close()
    return (info, p), st, plan


def _oracle_close(orc, prob, opt, got):
    """the tolerances of test_gpu_pose_ba._ba_compare"""
    ig, pg = got
    po = prob.copy()
    io = orc.ba_solve(po, opt)
    assert abs(ig[1] - io[1]) <= 1e-6 * io[1] + 1e-9, (ig[:10], io[:10])
    assert np.abs(pg.R - po.R).max() < 1e-6 and np.abs(pg.t - po.t).max() < 1e-6
    if prob.n:
        assert np.abs(pg.X - po.X).max() < 1e-5


@gpu
def test_one_handle_loads_every_shape_like_a_fresh_one(api, orc):
    opt = _opt()
    s = api.BaSolver(synth.make_ba_scene(2, 3, 400, 320, 240, seed=6, m_con=2, n_con=2)[0], opt)
    for name, make in SEQUENCE:
        prob = make()
        want, st, plan = _fresh(api, prob, opt)
        s.load(prob.copy())
        assert s.stats() == st, name
        assert s.plan_info() == plan, name
        got_run = (s.run(), s.download(prob.copy()))
        s.load(prob.copy())
        s.submit()
        got_sub = (s.collect(), s.download(prob.copy()))
        for got in (got_run, got_sub):
            ba_same_decisions(want, got, prob)
        assert got_sub[0][11] > 0, name
        if prob.n:
            _oracle_close(orc, prob, opt, got_sub)
        if name in ("free_10", "free_11", "free_20"):
            assert plan["small_solve"] == 1, name
        if name == "free_28":
            assert plan["small_solve"] == 0 and plan["blocks"] > 2
        if name == "no_free_camera":
            assert st["ns"] == 0
    s.close()


def _sleep_on(torch, s, cycles):
    with torch.cuda.stream(torch.cuda.ExternalStream(s.stream())):
        torch.cuda._sleep(cycles)


@gpu
def test_load_and_submit_return_before_the_device_runs_them(api):
    torch = _torch_cuda()
    opt = _opt()
    c2, c3 = _c2(), _c3()
    want2, want3 = _fresh(api, c2, opt)[0], _fresh(api, c3, opt)[0]
    s = api.BaSolver(c3.copy(), opt)
    s.submit()  # the first submit builds the graph
    s.collect()
    for prob, want in ((c2, want2), (c3, want3)):
        ext = torch.cuda.ExternalStream(s.stream())
        with torch.cuda.stream(ext):
            t0 = time.perf_counter()
            torch.cuda._sleep(int(1.5e9))  # about a second at H100 clocks
        s.load(prob.copy())
        s.submit()
        dt = time.perf_counter() - t0
        assert dt < 0.25, dt
        assert not s.done()
        info = s.collect()
        ba_same_decisions(want, (info, s.download(prob.copy())), prob)
    s.close()


@gpu
def test_load_copies_its_input(api):
    torch = _torch_cuda()
    opt = _opt()
    c2, c3 = _c2(), _c3()
    want = _fresh(api, c3, opt)[0]
    s = api.BaSolver(c2.copy(), opt)
    mine = _c3()  # BAProblem.copy() shares the index arrays
    _sleep_on(torch, s, int(3e8))  # the device has not consumed anything when the arrays change
    s.load(mine)
    for a in (mine.ptr, mine.cam):
        a[:] = 0
    for a in (mine.xy, mine.X, mine.R, mine.t):
        a[:] = np.nan
    s.submit()
    got = (s.collect(), s.download(c3.copy()))
    ba_same_decisions(want, got, c3)
    s.close()


def _malformed(prob):
    out = {}
    p = prob.copy()
    p.ptr[1], p.ptr[2] = p.ptr[2], p.ptr[1]  # not monotone
    out["ptr"] = p
    p = prob.copy()
    p.cam[5] = p.m  # camera index out of range
    out["camera_index"] = p
    p = prob.copy()
    i = int(np.argmax(np.diff(p.ptr) >= 2))
    p.cam[p.ptr[i] + 1] = p.cam[p.ptr[i]]  # the same (point, camera) pair twice
    out["repeated_pair"] = p
    p = prob.copy()
    p.m_con = p.m + 1
    out["m_con"] = p
    return out


@gpu
def test_malformed_problem_keeps_the_loaded_one(api):
    L = api.LIB
    opt = _opt()
    c2, c3 = _c2(), _c3()
    want = _fresh(api, c3, opt)[0]
    s = api.BaSolver(c2.copy(), opt)
    s.load(c3.copy())
    for name, bad in _malformed(c3).items():
        assert L.cosl_ba_solver_load(s.h, C.byref(bad.struct())) == COSL_E_INVALID, name
        assert L.cosl_ba_solver_load(s.h, None) == COSL_E_INVALID
        ba_same_decisions(want, (s.run(), s.download(c3.copy())), c3)
        s.reset(c3.copy())
    s.close()


@gpu
def test_load_while_a_submit_is_in_flight(api):
    torch = _torch_cuda()
    L = api.LIB
    opt = _opt()
    c2, c3 = _c2(), _c3()
    want = _fresh(api, c2, opt)[0]
    s = api.BaSolver(c2.copy(), opt)
    _sleep_on(torch, s, int(3e8))
    s.submit()
    assert L.cosl_ba_solver_load(s.h, C.byref(c3.struct())) == COSL_E_STATE
    info = s.collect()
    ba_same_decisions(want, (info, s.download(c2.copy())), c2)
    s.close()


@gpu
@pytest.mark.skipif(not (_torch_cuda() and _torch_cuda().cuda.device_count() >= 2), reason="needs two GPUs")
def test_multi_rank_solver_refuses_load(api):
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
        rc[r] = L.cosl_ba_solver_load(h, C.byref(p.struct()))
        L.cosl_ba_solver_destroy(h)
        L.cosl_ba_comm_destroy(comm)

    th = [threading.Thread(target=rank, args=(r,)) for r in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert rc == [COSL_E_INVALID, COSL_E_INVALID]


# ---------------------------------------------------------------- no GPU needed
def test_header_declares_load():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+cosl_ba_solver_load\s*\(([^)]*)\)\s*;", src)
    assert decl
    assert [a.strip() for a in decl.group(1).split(",")] == ["cosl_ba_solver* s", "const cosl_ba_problem* prob"]


def test_library_exports_load_and_the_binding_declares_it(api):
    from coslam_b200.ctypes_defs import BaProblem
    assert hasattr(C.CDLL(api.LIB_PATH), "cosl_ba_solver_load")
    assert callable(getattr(api.BaSolver, "load", None))
    assert api.LIB.cosl_ba_solver_load.argtypes == [C.c_void_p, C.POINTER(BaProblem)]


def test_null_handle_is_invalid(api):
    prob = synth.make_ba_scene(2, 3, 200, 320, 240, seed=6, m_con=2, n_con=2)[0]
    assert api.LIB.cosl_ba_solver_load(None, C.byref(prob.struct())) == COSL_E_INVALID


def test_pair_entry_count_beyond_32_bit_offsets_is_refused(api):
    """one free point seen by 66 000 free cameras: 66 000 * 66 001 / 2 > 2^31 - 1 pair entries, refused on the
    host before anything is allocated for them (with or without a device)"""
    m = 66000
    K = np.tile(np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]]), (m, 1, 1))
    R = np.tile(np.eye(3), (m, 1, 1))
    t = np.zeros((m, 3))
    t[:, 2] = 5.0
    prob = BAProblem(K, R, t, np.zeros((1, 3)), np.array([0, m], np.int64), np.arange(m, dtype=np.int32),
                     np.full((m, 2), 300.0), 0, 0)
    h = C.c_void_p()
    o = BaOptions.defaults()
    assert api.LIB.cosl_ba_solver_create(C.byref(prob.struct()), C.byref(o), None, C.byref(h)) == COSL_E_INVALID
    assert not h.value
    assert b"32-bit" in api.LIB.cosl_last_error()
