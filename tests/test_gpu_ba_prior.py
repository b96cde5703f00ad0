"""Camera priors on the GPU (cosl_ba_solver_set_cam_prior; DESIGN.md 4.8), on the edge rows of tests/ba_dense.py and
tests/ba_cov_dense.py and on `banded`, whose reduced system the plan splits into many blocks (the persistent tile
solve rather than ba_tile_two):
  1. one LM trial with priors on a subset of the free cameras against the dense prior-augmented step, with and
     without measurement covariances;
  2. run (non-robust) drives the full gradient, observations plus priors, to 1e-8 of its start; info[1] is the
     restated cost;
  3. the covariance stage against pixel_var (H + sum J^T P^-1 J)^-1, sigma2_hat, dof and the prior count;
  4. edges: a gauge fixed by priors alone, a prior camera no observation sees, P = 1e12 I, set and cleared;
  5. run and submit take the same decisions; a stop during a submit still collects with reason 8, and progress()'s
     cost includes the priors;
  6. Monte Carlo: means drawn from N(truth, P), noise from covx; the mean NEES is the dimension;
  7. state and validation."""
import ctypes as C

import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
import ba_prior_dense as pd
from coslam_b200.problem import BAProblem
from helpers import ba_same_decisions
from test_gpu_ba_async import _opt, _sleep_on, _torch_cuda
from test_gpu_ba_covariance import COSL_E_NUMERIC, _close, _raw_download

pytestmark = pytest.mark.gpu
COSL_E_INVALID, COSL_E_STATE = -1, -6
STOPPED = 8
ROWS = ["rig_intrinsics", "long_tracks", "unobserved_points", "tukey_mixed", "unsorted_observations", "banded"]
COV_ROWS = ["rig_intrinsics", "long_tracks_seen", "unobserved_points", "tukey_mixed", "unsorted_observations",
            "banded"]
VAR = 2.5


def _make(name):
    if name == "banded":
        return cd.banded(), bd.options()
    return bd.make(name)


def _make_cov(name):
    if name == "banded":
        return cd.banded(), bd.options()
    return cd.make(name)


def _priors(prob, seed, every=2, deg=3.0, scale=1.0):
    """priors on every `every`-th free camera, means deg degrees and 5 cm away from prob's cameras"""
    rng = np.random.default_rng(seed)
    cams = np.arange(prob.m_con, prob.m)[::every]
    R, t = pd.offset_means(prob, cams, rng, deg=deg)
    return pd.Priors(cams, R, t, pd.random_cov(len(cams), rng) * scale)


def _arm(s, pr):
    s.set_cam_prior(pr.cams, pr.R, pr.t, pr.cov)


def _solve(api, prob, opt, how, pr=None, covx=None, trials=3):
    s = api.BaSolver(prob.copy(), opt)
    if covx is not None:
        s.set_obs_cov(covx)
    if pr is not None:
        _arm(s, pr)
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


# ---------------------------------------------------------------- 1, 2: the LM loop
@pytest.mark.parametrize("weighted", [False, True], ids=["plain", "covx"])
@pytest.mark.parametrize("name", ROWS)
def test_one_trial_is_the_dense_prior_step(api, name, weighted):
    prob, opt = _make(name)
    covx = od.random_covx(prob.nobs, np.random.default_rng(5))[0] if weighted else None
    pr = _priors(prob, 7)
    info, after = _solve(api, prob, opt, "run_fixed", pr, covx, trials=1)
    r = pd.check_ptrial(prob, covx, pr, info, after, opt)
    print(name, " ".join(f"{k} {v:.2e}" for k, v in r.items()))


@pytest.mark.parametrize("name", ROWS)
def test_run_zeroes_the_full_gradient(api, name):
    prob, _ = _make(name)
    pr = _priors(prob, 8)
    opt = _opt(1, 60, max_err=0.0)
    info, got = _solve(api, prob, opt, "run", pr)
    g0 = pd.normal_equations(prob, 0.0, None, pr)[1]
    g1 = pd.normal_equations(got, 0.0, None, pr)[1]
    ratio = float(np.linalg.norm(g1) / np.linalg.norm(g0))
    print(f"{name}: {int(info[5])} iterations, stop {int(info[6])}, |g| / |g0| = {ratio:.2e}")
    assert ratio <= 1e-8
    assert abs(info[1] - pd.total_cost(got, None, pr)) <= 1e-9 * info[1]
    assert abs(info[0] - pd.total_cost(prob, None, pr)) <= 1e-9 * info[0]


# ---------------------------------------------------------------- 3: covariance stage
@pytest.mark.parametrize("name", COV_ROWS)
def test_covariance_stage_is_the_dense_inverse(api, name):
    prob, opt = _make_cov(name)
    pr = _priors(prob, 9)
    s = api.BaSolver(prob.copy(), opt)
    _arm(s, pr)
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    assert cd.decision_margin(state, opt.max_err) >= 1e-6
    wcam, wpt, winf, H = pd.cov_full(state, opt.max_err, VAR, None, pr)
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-8))
    assert inf["dof"] == winf["dof"] and inf["unconstrained"] == winf["unconstrained"]
    assert inf["priors"] == len(pr)
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= 1e-9 * winf["sigma2_hat"]


# ---------------------------------------------------------------- 4: edges
def _gauge_free():
    p = cd.small_nonrobust()
    rng = np.random.default_rng(40)
    xy = p.xy + rng.normal(0, 0.3, p.xy.shape)
    return BAProblem(p.K.copy(), p.R, p.t, p.X, p.ptr.copy(), p.cam.copy(), xy, 0, 0)


def test_priors_fix_the_gauge(api):
    prob = _gauge_free()
    opt = _opt(1, 30, max_err=0.0)
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(1.0)
    s.run()
    assert _raw_download(api, s)[0] == COSL_E_NUMERIC
    rng = np.random.default_rng(41)
    cams = np.array([0, 4])  # 1.2 m apart
    cov = pd.random_cov(2, rng)
    R, t = pd.draw_means(prob, cams, cov, rng)
    pr = pd.Priors(cams, R, t, cov)
    s.reset(prob.copy())
    _arm(s, pr)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    wcam, wpt, winf, H = pd.cov_full(state, 0.0, 1.0, None, pr)
    assert not winf["singular"]
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-7))
    assert inf["dof"] == winf["dof"] and inf["priors"] == 2


def _with_blind_camera(base):
    """base with one more free camera, appended, that no observation sees"""
    m = base.m
    R = np.concatenate([base.R.reshape(-1, 3, 3), (pd.so3_exp([0.02, -0.01, 0.03]) @ base.R.reshape(-1, 3, 3)[-1])[None]])
    t = np.concatenate([base.t, (base.t[-1] + [0.3, 0.01, -0.02])[None]])
    Kr = base.K.reshape(m, -1)
    K = np.concatenate([Kr, Kr[-1:]]).reshape((m + 1,) + base.K.shape[1:])
    return BAProblem(K, R, t, base.X.copy(), base.ptr.copy(), base.cam.copy(), base.xy.copy(), base.m_con,
                     base.n_con)


def test_unobserved_prior_camera_goes_to_its_mean(api):
    prob = _with_blind_camera(cd.make("rig_intrinsics")[0])
    j = prob.m - 1
    rng = np.random.default_rng(42)
    cov = pd.random_cov(1, rng)
    R, t = pd.offset_means(prob, [j], rng, deg=2.0)
    pr = pd.Priors([j], R, t, cov)
    s = api.BaSolver(prob.copy(), _opt(1, 60, max_err=0.0))
    _arm(s, pr)
    s.set_covariance(VAR)
    s.run()
    got = s.download()
    cam, _, inf = s.download_covariance()
    s.close()
    print("R", np.abs(got.R.reshape(-1, 3, 3)[j] - R[0]).max(), "t", np.abs(got.t[j] - t[0]).max())
    assert np.abs(got.R.reshape(-1, 3, 3)[j] - R[0]).max() <= 1e-10
    assert np.abs(got.t[j] - t[0]).max() <= 1e-10
    want = VAR * cov[0]
    assert np.abs(cam[j] - want).max() <= 1e-8 * np.abs(want).max()
    assert inf["priors"] == 1


@pytest.mark.parametrize("how", ["run", "run_fixed", "submit"])
@pytest.mark.parametrize("name", ["rig_intrinsics", "tukey_mixed", "banded"])
def test_a_loose_prior_is_the_unarmed_handle(api, name, how):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6  # as test_gpu_ba_obscov: eps2 = 1e-12 leaves the accept decisions to the atomic sums' order
    cams = np.arange(prob.m_con, prob.m)
    R, t = pd.offset_means(prob, cams, np.random.default_rng(43), deg=1.0)
    pr = pd.Priors(cams, R, t, np.tile(1e12 * np.eye(6), (len(cams), 1, 1)))
    ba_same_decisions(_solve(api, prob, opt, how), _solve(api, prob, opt, how, pr), prob)


@pytest.mark.parametrize("name", ["rig_intrinsics", "banded"])
def test_cleared_or_loaded_over_is_never_set(api, name):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6
    unarmed = _solve(api, prob, opt, "run")
    s = api.BaSolver(prob.copy(), opt)
    for clear in ("none", "empty", "load"):
        _arm(s, _priors(prob, 10))
        if clear == "none":
            s.set_cam_prior(None)
            s.reset(prob.copy())
        elif clear == "empty":
            s.set_cam_prior([], [], [], [])
            s.reset(prob.copy())
        else:
            s.load(prob.copy())
        for how in ("run", "submit"):
            s.reset(prob.copy())
            if how == "run":
                info = s.run()
            else:
                s.submit()
                info = s.collect()
            ba_same_decisions(unarmed, (info, bd.fresh(s.download())), prob)
    s.close()


# ---------------------------------------------------------------- 5: entry points
@pytest.mark.parametrize("name", ROWS)
def test_run_and_submit_agree(api, name):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6
    pr = _priors(prob, 11)
    ba_same_decisions(_solve(api, prob, opt, "run", pr), _solve(api, prob, opt, "submit", pr), prob)
    a = _solve(api, prob, opt, "run_fixed", pr, trials=4)
    b = _solve(api, prob, opt, "run_fixed", pr, trials=4)
    ba_same_decisions(a, b, prob)


def test_stop_during_a_prior_armed_submit(api):
    torch = _torch_cuda()
    prob, opt = _make("rig_intrinsics")
    pr = _priors(prob, 12)
    s = api.BaSolver(prob.copy(), opt)
    _arm(s, pr)
    _sleep_on(torch, s, int(5e8))
    s.submit()
    s.stop()
    info = s.collect()
    assert int(info[6]) == STOPPED
    p = s.progress()
    want = pd.total_cost(prob, None, pr, opt.max_err)
    assert abs(p["cost"] - want) <= 1e-9 * want and abs(info[0] - want) <= 1e-9 * want
    assert pd.prior_cost(prob, pr) > 1e-3 * want  # the priors are a visible part of it
    # a full armed submit: its progress reports the final cost, priors included
    s.reset(prob.copy())
    s.submit()
    info = s.collect()
    p = s.progress()
    got = s.download()
    s.close()
    assert p["cost"] == info[12] and int(info[6]) != STOPPED
    assert info[12] >= pd.prior_cost(got, pr) > 0


# ---------------------------------------------------------------- 6: Monte Carlo
def test_monte_carlo_nees(api):
    truth = cd.small_nonrobust()
    rng = np.random.default_rng(78)
    covx, S = od.random_covx(truth.nobs, rng)
    cams = np.arange(truth.m_con, truth.m)
    cov = pd.random_cov(len(cams), rng)
    s = api.BaSolver(truth.copy(), _opt(1, 30, max_err=0.0))
    s.set_covariance(1.0)
    nc, np_ = [], []
    for _ in range(200):
        p = bd.fresh(truth)
        p.xy = truth.xy + od.draw_noise(S, rng)
        R, t = pd.draw_means(truth, cams, cov, rng)
        s.load(p)
        s.set_obs_cov(covx)
        s.set_cam_prior(cams, R, t, cov)
        s.run()
        got = s.download()
        cam, pt, inf = s.download_covariance()
        assert inf["priors"] == len(cams)
        Rt, Rg = truth.R.reshape(-1, 3, 3), got.R.reshape(-1, 3, 3)
        for j in cams:
            ec = np.concatenate([pd.so3_log(Rg[j] @ Rt[j].T), got.t[j] - truth.t[j]])
            nc.append(float(ec @ np.linalg.solve(cam[j], ec)))
        d = got.X - truth.X
        np_.extend(np.einsum("ni,ni->n", d, np.linalg.solve(pt, d[:, :, None])[:, :, 0]))
    s.close()
    mc, mp = float(np.mean(nc)), float(np.mean(np_))
    print(f"mean NEES: cameras {mc:.3f} (6), points {mp:.3f} (3)")
    # chi^2 bands: 200 x 4 camera samples and 200 x 60 point samples (correlated within a run), +-15 %
    assert abs(mc - 6) <= 0.15 * 6 and abs(mp - 3) <= 0.15 * 3


# ---------------------------------------------------------------- 7: state and validation
def _raw_set(api, s, cams, R, t, cov, n=None):
    vp = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)  # noqa: E731
    cams = None if cams is None else np.ascontiguousarray(cams, np.int32)
    R = None if R is None else np.ascontiguousarray(R, np.float64)
    t = None if t is None else np.ascontiguousarray(t, np.float64)
    cov = None if cov is None else np.ascontiguousarray(cov, np.float64)
    k = len(cams) if n is None else n
    rc = api.LIB.cosl_ba_solver_set_cam_prior(s.h, k, vp(cams), vp(R), vp(t), vp(cov))
    return rc, api.LIB.cosl_last_error().decode()


def _bad_cases(prob, pr):
    """name -> (cams, R, t, cov) with prior 1 (and prior 2, which must not be named) broken"""
    def edit(f):
        c, R, t, P = pr.cams.copy(), pr.R.copy(), pr.t.copy(), pr.cov.copy()
        for k in (1, 2):
            f(k, c, R, t, P)
        return c, R, t, P

    def at(k, c, R, t, P, j):
        c[k] = j

    out = {
        "fixed_camera": edit(lambda k, c, R, t, P: at(k, c, R, t, P, prob.m_con - 1)),
        "past_the_end": edit(lambda k, c, R, t, P: at(k, c, R, t, P, prob.m)),
        "repeated": edit(lambda k, c, R, t, P: at(k, c, R, t, P, c[0])),
        "not_orthonormal": edit(lambda k, c, R, t, P: R.__setitem__(k, R[k] * (1 + 1e-8))),
        "reflection": edit(lambda k, c, R, t, P: R.__setitem__(k, -R[k])),
        "nan_t": edit(lambda k, c, R, t, P: t.__setitem__((k, 1), np.nan)),
        "inf_cov": edit(lambda k, c, R, t, P: P.__setitem__((k, 2, 2), np.inf)),
        "asymmetric": edit(lambda k, c, R, t, P: P.__setitem__((k, 0, 4), P[k, 0, 4] + 1e-9 * P[k].max())),
        "indefinite": edit(lambda k, c, R, t, P: P.__setitem__(k, P[k] - 2 * np.eye(6) * np.linalg.eigvalsh(P[k])[0])),
    }
    return out


def test_state_and_validation(api):
    torch = _torch_cuda()
    prob, opt = _make("rig_intrinsics")
    opt.opts[2] = 1e-6
    pr = _priors(prob, 13, every=1)
    assert len(pr) >= 3
    s = api.BaSolver(prob.copy(), opt)
    _sleep_on(torch, s, int(5e8))
    s.submit()
    assert _raw_set(api, s, pr.cams, pr.R, pr.t, pr.cov)[0] == COSL_E_STATE
    assert _raw_set(api, s, None, None, None, None, n=0)[0] == COSL_E_STATE
    s.collect()
    unarmed = _solve(api, prob, opt, "run")
    armed = _solve(api, prob, opt, "run", pr)
    other = _priors(prob, 14, every=1)
    armed_other = _solve(api, prob, opt, "run", other)
    # every invalid set names prior 1 and keeps what the handle had: first nothing, then `pr`
    for keep, want in ((None, unarmed), (pr, armed)):
        if keep is not None:
            _arm(s, keep)
        for name, (c, R, t, P) in _bad_cases(prob, other).items():
            rc, msg = _raw_set(api, s, c, R, t, P)
            assert rc == COSL_E_INVALID and "prior 1 " in msg, (name, rc, msg)
        rc, msg = _raw_set(api, s, other.cams, other.R, other.t, other.cov, n=-1)
        assert rc == COSL_E_INVALID
        s.reset(prob.copy())
        ba_same_decisions(want, (s.run(), bd.fresh(s.download())), prob)
    # reset keeps them (run and submit); a valid set replaces them
    for how in ("run", "submit"):
        s.reset(prob.copy())
        if how == "run":
            info = s.run()
        else:
            s.submit()
            info = s.collect()
        ba_same_decisions(armed, (info, bd.fresh(s.download())), prob)
    _arm(s, other)
    s.reset(prob.copy())
    ba_same_decisions(armed_other, (s.run(), bd.fresh(s.download())), prob)
    # load clears them
    s.load(prob.copy())
    ba_same_decisions(unarmed, (s.run(), bd.fresh(s.download())), prob)
    with pytest.raises(ValueError):
        s.set_cam_prior(pr.cams, pr.R[:-1], pr.t, pr.cov)
    s.close()
