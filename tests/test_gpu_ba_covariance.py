"""The BA solver's covariance stage (cosl_ba_solver_set_covariance / _download_covariance) on the GPU: parity with
the float64 references of tests/ba_cov_dense.py, the selected inversion on its own (cosl_ba_debug_tile_selinv),
run / submit / chart independence, that arming leaves the BA alone, the error codes, and what the numbers mean
(the spread of BA solutions under pixel noise of known variance)."""
import ctypes as C

import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd
from coslam_b200 import synth
from coslam_b200.problem import BAProblem
from helpers import ba_same_decisions
from test_gpu_ba_async import _opt, _sleep_on, _torch_cuda

gpu = pytest.mark.gpu
COSL_E_NUMERIC, COSL_E_STATE = -4, -6
VAR = 2.5


def _raw_download(api, s):
    """download_covariance through the C-ABI into buffers filled with 7: (rc, camCov, ptCov, out)"""
    cam = np.full((s.prob.m, 6, 6), 7.0)
    pt = np.full((s.prob.n, 3, 3), 7.0)
    out = (C.c_double * 8)(*([7.0] * 8))
    rc = api.LIB.cosl_ba_solver_download_covariance(s.h, cam.ctypes.data_as(C.c_void_p),
                                                    pt.ctypes.data_as(C.c_void_p), out)
    return rc, cam, pt, list(out)


def _armed_run(api, prob, opt, var=VAR):
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(var)
    info = s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    return info, state, cam, pt, inf


def _close(got, want, tol):
    for g, w in zip(got, want):
        err, same = cd.block_errors(g, w)
        assert same
        assert err.size == 0 or err.max() <= tol, (float(err.max()), tol)
        print(f"max block error {float(err.max()) if err.size else 0.0:.3g} (bound {tol:.3g})")


def _no_steps(outer=1):
    """options whose LM stops at its first gradient test: the parameters stay where they are"""
    return _opt(outer, 10, max_err=6.0, o1=1e300)


# ---------------------------------------------------------------- parity
@gpu
@pytest.mark.parametrize("name", sorted(cd.cov_rows()))
def test_parity_with_the_dense_reference(api, name):
    prob, opt = cd.make(name)
    info, state, cam, pt, inf = _armed_run(api, prob, opt)
    wcam, wpt, winf, H = cd.cov_full(state, opt.max_err, VAR)
    tol = cd.far_tolerance(state, H, 1e-8)
    _close((cam, pt), (wcam, wpt), tol)
    assert inf["pixel_var"] == VAR
    assert inf["dof"] == winf["dof"] and inf["unconstrained"] == winf["unconstrained"]
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= max(1e-9, tol) * winf["sigma2_hat"]
    assert inf["device_ms"] > 0 and 1e-12 <= inf["min_pivot"] <= 1.0
    if name == "unobserved_points":
        assert inf["unconstrained"] >= 3 and np.isnan(pt).any()
    if name == "tukey_mixed":
        assert (cd.weights(state, opt.max_err)[1] == 0).sum() > 0


@gpu
def test_two_block_c2_scene_against_the_schur_form(api):
    prob = synth.make_ba_scene(2, 8, 5000, 640, 480, seed=7, m_con=4, n_con=2)[0]
    opt = _opt(2, 10)
    s = api.BaSolver(prob.copy(), opt)
    plan = s.plan_info()
    assert plan["blocks"] == 2 and plan["small_solve"] == 1
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    wcam, wpt, winf = cd.cov_schur(state, opt.max_err, VAR)
    _close((cam, pt), (wcam, wpt), 1e-8)
    assert inf["dof"] == winf["dof"]


@gpu
def test_banded_scene_of_many_blocks_against_the_schur_form(api):
    prob = cd.banded()
    opt = _opt(1, 10)
    s = api.BaSolver(prob.copy(), opt)
    plan = s.plan_info()
    assert prob.m - prob.m_con >= 40 and plan["blocks"] > 2 and plan["nd_depth"] >= 1, plan
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    wcam, wpt, winf = cd.cov_schur(state, opt.max_err, VAR)
    _close((cam, pt), (wcam, wpt), 1e-8)
    assert inf["dof"] == winf["dof"]


# ---------------------------------------------------------------- the selected inversion on its own
def _spd(mf, pat, param, rng):
    adj = np.eye(mf, dtype=np.uint8)
    for a in range(mf):
        for b in range(a + 1, mf):
            on = pat == "dense" or (pat == "band" and b - a <= param) or (
                pat == "random" and (rng.random() < param or b - a <= 2)) or (
                pat == "split" and b - a <= param and (a < mf // 2) == (b < mf // 2))
            adj[a, b] = adj[b, a] = on
    ns = 6 * mf
    S = rng.uniform(-1, 1, (ns, ns)) * np.kron(adj, np.ones((6, 6)))
    S = (S + S.T) / 2
    S[np.diag_indices(ns)] = np.abs(S).sum(1) + 1.0
    return S, adj


@gpu
@pytest.mark.parametrize("args", [(1, "dense", 0), (7, "band", 2), (12, "dense", 0), (40, "dense", 0),
                                  (29, "dense", 0), (100, "random", 0.05), (200, "band", 20, 2),
                                  (396, "band", 35, 3),
                                  # block-diagonal (no operation in any step) and two connected components
                                  (12, "band", 0), (20, "band", 0), (25, "band", 0), (30, "band", 0),
                                  (61, "band", 0), (100, "band", 0), (100, "band", 0, 2), (40, "split", 3),
                                  (41, "split", 2, 1)])
def test_debug_selinv_matches_the_inverse(api, args):
    mf, pat, param = args[:3]
    depth = args[3] if len(args) > 3 else -1
    S, adj = _spd(mf, pat, param, np.random.default_rng(mf))
    Z, fail, info = api.ba_debug_tile_selinv(S, adj, depth)
    assert fail == 0
    Sinv = np.linalg.inv(S)
    B = lambda M, a, c: M[6 * a:6 * a + 6, 6 * c:6 * c + 6]  # noqa: E731
    dn = np.array([np.linalg.norm(B(Sinv, a, a)) for a in range(mf)])
    worst = 0.0
    for a in range(mf):
        for c in range(a + 1):
            z = B(Z, a, c)
            if adj[a, c]:
                assert z.any()
            if z.any():
                worst = max(worst, np.linalg.norm(z - B(Sinv, a, c)) / np.sqrt(dn[a] * dn[c]))
    assert worst < 1e-10, (info, worst)
    assert not np.triu(Z, 6).any()
    if pat == "band" and param == 0:  # block-diagonal: no tile off the diagonal, one task per block
        assert info["tiles"] == info["blocks"] and info["selinv_tasks"] == info["blocks"], info
    print(f"{args}: {info}, worst block error {worst:.2g}")


@gpu
@pytest.mark.parametrize("mf", [7, 40])
def test_debug_selinv_flags_a_singular_system(api, mf):
    S, adj = _spd(mf, "band", 2, np.random.default_rng(5))
    S[6 * (mf // 2):6 * (mf // 2) + 6, :] = 0.0
    S[:, 6 * (mf // 2):6 * (mf // 2) + 6] = 0.0
    _, fail, _ = api.ba_debug_tile_selinv(S, adj)
    assert fail == 1


# ---------------------------------------------------------------- run, submit, chart
@gpu
@pytest.mark.parametrize("scene", ["c3", "banded"])
def test_run_and_submit_agree(api, scene):
    """At the same parameters (the LM stops at its first gradient test) run and submit give the same covariances.
    The stage's fp64 atomic sums (linearisation, Schur contraction, pair pass) add in another order on every call
    and H^-1 amplifies that by its condition: 3e-9 was measured at c3, so the bound is the parity bound."""
    prob = (synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=3, m_con=8, n_con=2)[0] if scene == "c3"
            else cd.banded())
    opt = _no_steps()
    a = api.BaSolver(prob.copy(), opt)
    a.set_covariance(VAR)
    ia = a.run()
    ca, pa, fa = a.download_covariance()
    b = api.BaSolver(prob.copy(), opt)
    b.set_covariance(VAR)
    b.submit()
    ib = b.collect()
    cb, pb, fb = b.download_covariance()
    assert ia[5] == ib[5] == 0 and ia[6] == ib[6] == 1  # the parameters did not move
    assert np.array_equal(a.download().X, b.download().X)
    a.close()
    b.close()
    _close((cb, pb), (ca, pa), 1e-8)
    assert fa["dof"] == fb["dof"] and abs(fa["sigma2_hat"] - fb["sigma2_hat"]) <= 1e-12 * fa["sigma2_hat"]


@gpu
def test_stopped_ba_covariance_is_that_of_its_parameters(api):
    prob = bd.rotated_start()
    opt = _opt(1, 10, max_err=0.0)
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(VAR)
    s.submit()
    while True:  # stop once the loop has moved the parameters (v != 0), or let it end
        p = s.progress()
        if p["iteration"] >= 2 or not p["running"]:
            break
    s.stop()
    info = s.collect()
    got = s.download()
    cam, pt, _ = s.download_covariance()
    s.close()
    # a fresh handle at those parameters: its rotation chart starts there (v = 0) instead of at prob.R
    fresh = api.BaSolver(BAProblem(got.K.copy(), got.R, got.t, got.X, got.ptr.copy(), got.cam.copy(), got.xy.copy(),
                                   got.m_con, got.n_con), _opt(1, 10, max_err=0.0, o1=1e300))
    fresh.set_covariance(VAR)
    fresh.run()
    cam2, pt2, _ = fresh.download_covariance()
    fresh.close()
    _close((cam2, pt2), (cam, pt), 1e-9)
    print(f"stopped with reason {int(info[6])} after {int(info[5])} iterations")


# ---------------------------------------------------------------- arming leaves the BA alone
@gpu
def test_arming_does_not_change_the_ba(api):
    # eps2 = 1e-6: the second run starts at the optimum, where eps2 = 1e-12 would leave the accept decisions to
    # the order of the device's atomic sums (see test_gpu_ba_async's intercam scene), armed or not
    prob, opt = synth.make_ba_scene(2, 5, 5000, 640, 480, seed=7, m_con=4, n_con=2)[0], _opt(2, 10, o2=1e-6)
    plain = api.BaSolver(prob.copy(), opt)
    armed = api.BaSolver(prob.copy(), opt)
    armed.set_covariance(VAR)
    for _ in range(2):  # run -> covariance -> run
        want = (plain.run(), bd.fresh(plain.download()))
        got = (armed.run(), bd.fresh(armed.download()))
        ba_same_decisions(want, got, prob)
        assert armed.download_covariance()[2]["dof"] > 0
    plain.close()
    armed.close()


@gpu
def test_submit_armed_unarmed_armed(api):
    prob = synth.make_ba_scene(2, 5, 5000, 640, 480, seed=7, m_con=4, n_con=2)[0]
    opt = _opt()
    ref = api.BaSolver(prob.copy(), opt)
    ref.submit()
    want = (ref.collect(), bd.fresh(ref.download()))
    ref.close()
    s = api.BaSolver(prob.copy(), opt)
    first = None
    for arm in (VAR, 0.0, VAR):
        s.reset(prob.copy())
        s.set_covariance(arm)
        s.submit()
        got = (s.collect(), bd.fresh(s.download()))
        ba_same_decisions(want, got, prob)
        if arm:
            cam, pt, _ = s.download_covariance()
            if first is None:
                first = (cam, pt)
            else:
                _close((cam, pt), first, 1e-9)
        else:
            assert _raw_download(api, s)[0] == COSL_E_STATE
    s.close()


# ---------------------------------------------------------------- errors
@gpu
def test_state_errors(api):
    torch = _torch_cuda()
    prob = synth.make_ba_scene(2, 5, 3000, 640, 480, seed=7, m_con=4, n_con=2)[0]
    s = api.BaSolver(prob.copy(), _opt())
    assert _raw_download(api, s)[0] == COSL_E_STATE  # nothing armed yet
    s.set_covariance(VAR)
    assert _raw_download(api, s)[0] == COSL_E_STATE  # armed, but no BA since
    s.run()
    assert _raw_download(api, s)[0] == 0
    s.load(prob.copy())
    assert _raw_download(api, s)[0] == COSL_E_STATE  # a load since
    s.run()
    s.reset(prob.copy())
    assert _raw_download(api, s)[0] == COSL_E_STATE  # a reset since
    _sleep_on(torch, s, int(5e8))
    s.submit()
    assert _raw_download(api, s)[0] == COSL_E_STATE  # in flight
    assert api.LIB.cosl_ba_solver_set_covariance(s.h, 1.0) == COSL_E_STATE
    s.collect()
    assert _raw_download(api, s)[0] == 0
    assert api.LIB.cosl_ba_solver_set_covariance(s.h, -1.0) == -1
    s.close()


@gpu
@pytest.mark.parametrize("case", ["gauge_free", "long_tracks"])
def test_singular_systems(api, case):
    """No fixed camera or point (a 7-dimensional gauge), or a free camera with one observation: the BA collects with
    COSL_OK, the covariance is refused with COSL_E_NUMERIC and nothing is written."""
    if case == "gauge_free":
        b = bd.rig_intrinsics()
        prob, opt = BAProblem(b.K.copy(), b.R, b.t, b.X, b.ptr.copy(), b.cam.copy(), b.xy.copy(), 0, 0), _opt(1, 5)
    else:
        prob, opt = bd.make("long_tracks")
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(VAR)
    s.submit()
    info = s.collect()
    assert info[1] <= info[0]
    rc, cam, pt, out = _raw_download(api, s)
    assert rc == COSL_E_NUMERIC
    assert (cam == 7.0).all() and (pt == 7.0).all() and out == [7.0] * 8
    assert "singular" in api.LIB.cosl_last_error().decode()
    s.close()


# ---------------------------------------------------------------- meaning
@gpu
def test_covariance_predicts_the_spread_of_solutions(api):
    """Mean NEES of ~200 BA solutions under fresh pixel noise of variance sigma^2 is the dimension (6 per camera,
    3 per point) within 15 %."""
    truth = cd.small_nonrobust()
    sigma = 0.5
    opt = _opt(1, 30, max_err=0.0)
    rng = np.random.default_rng(99)
    s = api.BaSolver(truth.copy(), opt)
    s.set_covariance(sigma ** 2)
    Rt = truth.R.reshape(-1, 3, 3)
    nc, np_ = [], []
    for _ in range(200):
        p = truth.copy()
        p.xy = truth.xy + rng.normal(0, sigma, truth.xy.shape)
        s.load(p)
        s.run()
        got = s.download()
        cam, pt, _ = s.download_covariance()
        for j in range(truth.m_con, truth.m):
            dR = got.R.reshape(-1, 3, 3)[j] @ Rt[j].T
            w = 0.5 * np.array([dR[2, 1] - dR[1, 2], dR[0, 2] - dR[2, 0], dR[1, 0] - dR[0, 1]])
            e = np.concatenate([w, got.t[j] - truth.t[j]])
            nc.append(e @ np.linalg.solve(cam[j], e))
        d = got.X - truth.X
        np_.extend(np.einsum("ni,ni->n", d, np.linalg.solve(pt, d[:, :, None])[:, :, 0]))
    s.close()
    mc, mp = float(np.mean(nc)), float(np.mean(np_))
    print(f"mean NEES: cameras {mc:.3f} (6), points {mp:.3f} (3)")
    assert abs(mc - 6) <= 0.15 * 6 and abs(mp - 3) <= 0.15 * 3
