"""Measurement covariances on the GPU (cosl_ba_solver_set_obs_cov, cosl_sba_motstr_levmar_x_cov; DESIGN.md 4.7), on
the edge rows of tests/ba_dense.py: per-camera intrinsics, long tracks, unobserved points, Tukey mixed, unsorted
observations.

  1. Sigma = I: run, run_fixed and submit take the unarmed handle's decisions and return its outlier flags, costs and
     parameters.  (The device's fp64 atomic sums add in another order on every call, so two unarmed handles agree to
     the last bits only up to that order; L = I itself is exact.)
  2. Sigma = 4 I: run_fixed returns the unarmed parameters and a quarter of its costs.
  3. Anisotropic, heteroscedastic Sigma: one LM trial against the dense whitened step (ba_obscov_dense.check_wtrial,
     the bounds of test_ba_dense_ref), and after run a whitened gradient at 1e-8 of its initial norm.
  4. The covariance stage with Sigma set against pixel_var (J^T W Lambda J)^-1.
  5. Monte Carlo: noise drawn from each observation's own Sigma; the mean NEES is the dimension, and the weighted
     solutions scatter less than unweighted ones of the same data.
  6. cosl_sba_motstr_levmar_x_cov: NULL is cosl_sba_motstr_levmar_x, covx agrees with the handle.
  7. State: COSL_E_STATE during a submit; load clears the covariances, reset keeps them."""
import ctypes as C

import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
from helpers import ba_same_decisions
from test_gpu_ba_async import _opt, _sleep_on, _torch_cuda
from test_gpu_ba_covariance import _close

pytestmark = pytest.mark.gpu
COSL_E_STATE = -6
ROWS = ["rig_intrinsics", "long_tracks", "unobserved_points", "tukey_mixed", "unsorted_observations"]
VAR = 2.5


def _covx(prob, seed=5):
    return od.random_covx(prob.nobs, np.random.default_rng(seed))[0]


def _solve(api, prob, opt, how, covx=None, trials=3):
    s = api.BaSolver(prob.copy(), opt)
    if covx is not None:
        s.set_obs_cov(covx)
    if how == "run":
        info = s.run()
    elif how == "run_fixed":
        info = s.run_fixed(trials)
    else:
        s.submit()
        info = s.collect()
    out = (info, bd.fresh(s.download()))
    s.close()
    return out


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


# ---------------------------------------------------------------- 1, 2: isotropic covariances
@pytest.mark.parametrize("how", ["run", "run_fixed", "submit"])
@pytest.mark.parametrize("name", ROWS)
def test_identity_is_the_unarmed_handle(api, name, how):
    prob, opt = bd.make(name)
    # eps2 = 1e-6: at the optimum eps2 = 1e-12 leaves the accept decisions to the order of the device's atomic sums,
    # armed or not (see test_gpu_ba_covariance.test_arming_does_not_change_the_ba)
    opt.opts[2] = 1e-6
    want = _solve(api, prob, opt, how)
    got = _solve(api, prob, opt, how, np.tile(np.eye(2), (prob.nobs, 1, 1)))
    ba_same_decisions(want, got, prob)
    (iw, pw), (ig, pg) = want, got
    assert np.array_equal(pw.outlier, pg.outlier)
    assert abs(ig[0] - iw[0]) <= 1e-12 * iw[0] and abs(ig[1] - iw[1]) <= 1e-9 * iw[1], (ig[:2], iw[:2])
    print(f"{name} {how}: |dR| {np.abs(pw.R - pg.R).max():.2e} |dX| {np.abs(pw.X - pg.X).max():.2e}")


@pytest.mark.parametrize("name", ROWS)
def test_scaled_identity_quarters_the_cost(api, name):
    prob, opt = bd.make(name)
    (iw, pw) = _solve(api, prob, opt, "run_fixed")
    (ig, pg) = _solve(api, prob, opt, "run_fixed", np.tile(4.0 * np.eye(2), (prob.nobs, 1, 1)))
    assert np.array_equal(iw[5:11], ig[5:11])
    for k in (0, 1, 12):
        assert abs(4.0 * ig[k] - iw[k]) <= 1e-12 * iw[k], (k, ig[k], iw[k])
    errs = {a: _rel(getattr(pg, a), getattr(pw, a)) for a in ("R", "t", "X")}
    print(name, errs)
    assert max(errs.values()) <= 1e-12, errs


# ---------------------------------------------------------------- 3: anisotropic covariances
@pytest.mark.parametrize("name", ROWS)
def test_one_trial_is_the_dense_whitened_step(api, name):
    prob, opt = bd.make(name)
    covx = _covx(prob)
    info, after = _solve(api, prob, opt, "run_fixed", covx, trials=1)
    r = od.check_wtrial(prob, covx, info, after, opt)
    print(name, " ".join(f"{k} {v:.2e}" for k, v in r.items()))


@pytest.mark.parametrize("name", ROWS)
def test_run_zeroes_the_whitened_gradient(api, name):
    """Non-robust (the Tukey weights of the last round were frozen at its start), so the gradient at the returned
    parameters is the one the LM loop drove to zero."""
    prob, _ = bd.make(name)
    covx = _covx(prob)
    opt = _opt(1, 60, max_err=0.0)
    info, got = _solve(api, prob, opt, "run", covx)
    g0 = od.normal_equations(prob, 0.0, covx)[1]
    g1 = od.normal_equations(got, 0.0, covx)[1]
    ratio = float(np.linalg.norm(g1) / np.linalg.norm(g0))
    print(f"{name}: {int(info[5])} iterations, stop {int(info[6])}, |g| / |g0| = {ratio:.2e}")
    assert ratio <= 1e-8
    assert abs(info[1] - od.whitened_cost(got, np.ones(got.nobs), od.factors(covx))) <= 1e-9 * info[1]


# ---------------------------------------------------------------- 4: covariance stage
@pytest.mark.parametrize("name", ["rig_intrinsics", "long_tracks_seen", "unobserved_points", "tukey_mixed",
                                  "unsorted_observations"])
def test_covariance_stage_is_the_dense_inverse(api, name):
    prob, opt = cd.make(name)
    covx = _covx(prob)
    s = api.BaSolver(prob.copy(), opt)
    s.set_obs_cov(covx)
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    assert cd.decision_margin(state, opt.max_err) >= 1e-6
    wcam, wpt, winf, H = od.cov_full(state, opt.max_err, VAR, covx)
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-8))
    assert inf["dof"] == winf["dof"] and inf["unconstrained"] == winf["unconstrained"]
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= 1e-9 * winf["sigma2_hat"]


# ---------------------------------------------------------------- 5: meaning
def _errors(truth, got, cam, pt):
    """per free camera (w, dt) and per point dX of a solution, and their NEES under (cam, pt)"""
    Rt = truth.R.reshape(-1, 3, 3)
    ec = []
    for j in range(truth.m_con, truth.m):
        dR = got.R.reshape(-1, 3, 3)[j] @ Rt[j].T
        w = 0.5 * np.array([dR[2, 1] - dR[1, 2], dR[0, 2] - dR[2, 0], dR[1, 0] - dR[0, 1]])
        ec.append(np.concatenate([w, got.t[j] - truth.t[j]]))
    ec = np.array(ec)
    d = got.X - truth.X
    nees_c = np.einsum("ja,ja->j", ec, np.linalg.solve(cam[truth.m_con:], ec[:, :, None])[:, :, 0])
    nees_p = np.einsum("ni,ni->n", d, np.linalg.solve(pt, d[:, :, None])[:, :, 0])
    return ec, d, nees_c, nees_p


def test_monte_carlo_nees_and_scatter(api):
    truth = cd.small_nonrobust()
    rng = np.random.default_rng(77)
    covx, S = od.random_covx(truth.nobs, rng)
    opt = _opt(1, 30, max_err=0.0)
    wtd = api.BaSolver(truth.copy(), opt)
    plain = api.BaSolver(truth.copy(), opt)
    wtd.set_covariance(1.0)  # covariances in px^2
    nc, np_, sw, su = [], [], np.zeros(2), np.zeros(2)
    for _ in range(200):
        p = truth.copy()
        p.xy = truth.xy + od.draw_noise(S, rng)
        wtd.load(p)
        wtd.set_obs_cov(covx)  # load clears them
        wtd.run()
        got = wtd.download()
        cam, pt, _ = wtd.download_covariance()
        ec, d, a, b = _errors(truth, got, cam, pt)
        nc.extend(a)
        np_.extend(b)
        sw += [(ec * ec).sum(), (d * d).sum()]
        plain.load(p.copy())
        plain.run()
        ecu, du, _, _ = _errors(truth, plain.download(), cam, pt)
        su += [(ecu * ecu).sum(), (du * du).sum()]
    wtd.close()
    plain.close()
    mc, mp = float(np.mean(nc)), float(np.mean(np_))
    print(f"mean NEES: cameras {mc:.3f} (6), points {mp:.3f} (3); mean square error weighted / unweighted: "
          f"cameras {sw[0] / su[0]:.3f}, points {sw[1] / su[1]:.3f}")
    assert abs(mc - 6) <= 0.15 * 6 and abs(mp - 3) <= 0.15 * 3
    assert sw[0] < su[0] and sw[1] < su[1]


# ---------------------------------------------------------------- 6: the sba entry point
def _sba_args(name):
    """(problem, p, rot0, vmask, the problem sorted by camera within each point, its permutation): sba's
    measurements are point-major by ascending camera, the order of vmask"""
    prob, _ = bd.make(name)
    dq = np.random.default_rng(21).normal(size=(prob.m, 3)) * 0.02
    p, rot0, vmask = bd.pack_sba(prob, dq)
    srt, perm = bd.sorted_permutation(prob)
    return prob, p, rot0, vmask, srt, perm


@pytest.mark.parametrize("name", ["rig_intrinsics", "unsorted_observations"])
def test_sba_null_covx_is_the_plain_call(api, name):
    prob, p0, rot0, vmask, srt, _ = _sba_args(name)
    opts = np.array([1e-7, 1e-12, 1e-12, 0.0, 1e-16])
    pa, pb = p0.copy(), p0.copy()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    ia = np.zeros(10)
    ra = api.LIB.cosl_sba_motstr_levmar_x(prob.n, prob.n_con, prob.m, prob.m_con, vp(vmask), vp(pa), 11, 3,
                                          vp(srt.xy), 2, vp(rot0), 6, 0, vp(opts), vp(ia), 0)
    rb, ib = api.sba_motstr_levmar_x(pb, rot0, vmask, srt.xy, 6, opts, prob.n_con, prob.m_con)
    assert ra == rb == 6
    assert np.array_equal(ia[5:10], ib[5:10]) and abs(ia[0] - ib[0]) <= 1e-12 * ia[0]
    assert abs(ia[1] - ib[1]) <= 1e-9 * ia[1] and np.abs(pa - pb).max() < 1e-9


@pytest.mark.parametrize("name", ["rig_intrinsics", "unsorted_observations"])
def test_sba_covx_agrees_with_the_handle(api, name):
    prob, p0, rot0, vmask, srt, perm = _sba_args(name)
    opts = np.array([1e-7, 1e-12, 1e-12, 0.0, 1e-16])
    covx = _covx(prob)[perm]
    up = bd.unpack_sba(p0, rot0, vmask, srt.xy.copy(), prob.m_con, prob.n_con)
    p = p0.copy()
    it, info = api.sba_motstr_levmar_x(p, rot0, vmask, srt.xy, 6, opts, prob.n_con, prob.m_con, covx=covx)
    opt = _opt(1, 6, max_err=0.0)
    opt.opts[:] = opts
    ih, ph = _solve(api, up, opt, "run", covx)
    assert it == int(ih[5]) and np.array_equal(info[5:10], ih[5:10]), (info, ih[:10])
    assert abs(info[0] - ih[0]) <= 1e-12 * ih[0] and abs(info[1] - ih[1]) <= 1e-9 * ih[1]
    got = bd.unpack_sba(p, rot0, vmask, srt.xy, prob.m_con, prob.n_con)
    assert np.abs(got.R - ph.R).max() < 1e-9 and np.abs(got.t - ph.t).max() < 1e-9
    assert np.abs(got.X - ph.X).max() < 1e-8
    # and the covariances made a difference
    plain = p0.copy()
    api.sba_motstr_levmar_x(plain, rot0, vmask, srt.xy, 6, opts, prob.n_con, prob.m_con)
    assert np.abs(plain - p).max() > 1e-6


# ---------------------------------------------------------------- 7: state rules
def test_state_rules(api):
    torch = _torch_cuda()
    prob, opt = bd.make("rig_intrinsics")
    opt.opts[2] = 1e-6  # as in test_identity_is_the_unarmed_handle
    covx = _covx(prob)
    s = api.BaSolver(prob.copy(), opt)
    _sleep_on(torch, s, int(5e8))
    s.submit()
    c = np.ascontiguousarray(covx, np.float64)
    assert api.LIB.cosl_ba_solver_set_obs_cov(s.h, c.ctypes.data_as(C.c_void_p)) == COSL_E_STATE
    assert api.LIB.cosl_ba_solver_set_obs_cov(s.h, None) == COSL_E_STATE
    s.collect()
    # an invalid set keeps what the handle had (here: nothing)
    bad = c.copy()
    bad[3] = [[1.0, 2.0], [2.0, 1.0]]
    assert api.LIB.cosl_ba_solver_set_obs_cov(s.h, bad.ctypes.data_as(C.c_void_p)) == -1
    assert "observation 3 " in api.LIB.cosl_last_error().decode()
    unarmed = _solve(api, prob, opt, "run")
    armed = _solve(api, prob, opt, "run", covx)
    s.reset(prob.copy())
    ba_same_decisions(unarmed, (s.run(), bd.fresh(s.download())), prob)
    # reset keeps them (run and submit)
    s.set_obs_cov(covx)
    for how in ("run", "submit"):
        s.reset(prob.copy())
        if how == "run":
            info = s.run()
        else:
            s.submit()
            info = s.collect()
        ba_same_decisions(armed, (info, bd.fresh(s.download())), prob)
    # an invalid set after a valid one keeps the valid one
    assert api.LIB.cosl_ba_solver_set_obs_cov(s.h, bad.ctypes.data_as(C.c_void_p)) == -1
    s.reset(prob.copy())
    ba_same_decisions(armed, (s.run(), bd.fresh(s.download())), prob)
    # load clears them (run and submit), and NULL clears them
    for how in ("run", "submit"):
        s.load(prob.copy())
        if how == "run":
            info = s.run()
        else:
            s.submit()
            info = s.collect()
        ba_same_decisions(unarmed, (info, bd.fresh(s.download())), prob)
    s.set_obs_cov(covx)
    s.set_obs_cov(None)
    s.reset(prob.copy())
    ba_same_decisions(unarmed, (s.run(), bd.fresh(s.download())), prob)
    s.close()
