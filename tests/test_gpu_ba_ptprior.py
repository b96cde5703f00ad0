"""Point priors on the GPU (cosl_ba_solver_set_pt_prior; DESIGN.md 4.9), on the edge rows of tests/ba_dense.py and
tests/ba_cov_dense.py and on `banded`, whose reduced system the plan splits into many blocks:
  1. one LM trial with priors on a subset of the free points against the dense prior-augmented step, without and
     with measurement covariances and with camera priors set as well; the path without free cameras;
  2. run (non-robust) drives the full gradient, observations plus priors, to 1e-8 of its start;
  3. the covariance stage against pixel_var H^-1, with prior points of zero and one weighted observation, sigma2_hat,
     dof, out[3] and out[7];
  4. edges: an unobserved prior point goes to its mean with ptCov = pixel_var P, a gauge fixed by three prior points,
     P = 1e12 I against the unarmed handle, set / clear / load / reset;
  5. run and submit take the same decisions, also after the priors changed between two submits; a stop during a
     prior-armed submit;
  6. Monte Carlo: means drawn from N(truth, P); the mean point NEES is 3;
  7. state and validation."""
import ctypes as C

import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd
import ba_obscov_dense as od
import ba_prior_dense as pd
import ba_ptprior_dense as ppd
from coslam_b200.problem import BAProblem
from helpers import ba_same_decisions
from test_ba_ptprior_dense_ref import _with_sparse_points, gauge_free, gauge_points
from test_gpu_ba_async import _opt, _sleep_on, _torch_cuda
from test_gpu_ba_covariance import COSL_E_NUMERIC, _close, _raw_download

pytestmark = pytest.mark.gpu
COSL_E_INVALID, COSL_E_STATE = -1, -6
STOPPED = 8
ROWS = ["rig_intrinsics", "long_tracks", "unobserved_points", "tukey_mixed", "unsorted_observations", "banded"]
COV_ROWS = ["rig_intrinsics", "long_tracks_seen", "unobserved_points", "tukey_mixed", "unsorted_observations",
            "banded", "sparse_points"]
VAR = 2.5


def _make(name):
    if name == "banded":
        return cd.banded(), bd.options()
    return bd.make(name)


def _make_cov(name):
    if name == "banded":
        return cd.banded(), bd.options()
    if name == "sparse_points":  # two more free points, one unobserved and one seen once
        prob, opt = cd.make("rig_intrinsics")
        return _with_sparse_points(prob, np.random.default_rng(50)), opt
    return cd.make(name)


def _pts(prob, seed, every=3, dist=0.05, scale=1.0, extra=()):
    """priors on every `every`-th free point (and on `extra`), means `dist` away from prob's points"""
    rng = np.random.default_rng(seed)
    extra = np.asarray(extra, np.int64)
    pts = np.union1d(np.arange(prob.n_con, prob.n)[::every], extra[extra >= prob.n_con])
    return ppd.PtPriors(pts, ppd.offset_pt_means(prob, pts, rng, dist), ppd.random_pt_cov(len(pts), rng) * scale)


def _cams(prob, seed):
    rng = np.random.default_rng(seed)
    cams = np.arange(prob.m_con, prob.m)[::2]
    R, t = pd.offset_means(prob, cams, rng, deg=3.0)
    return pd.Priors(cams, R, t, pd.random_cov(len(cams), rng))


def _arm(s, pp, pr=None):
    s.set_pt_prior(pp.pts, pp.X, pp.cov)
    if pr is not None:
        s.set_cam_prior(pr.cams, pr.R, pr.t, pr.cov)


def _solve(api, prob, opt, how, pp=None, pr=None, covx=None, trials=3):
    s = api.BaSolver(prob.copy(), opt)
    if covx is not None:
        s.set_obs_cov(covx)
    if pp is not None:
        _arm(s, pp, pr)
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


def _no_free_cameras(prob):
    return BAProblem(prob.K.copy(), prob.R.copy(), prob.t.copy(), prob.X.copy(), prob.ptr.copy(), prob.cam.copy(),
                     prob.xy.copy(), prob.m, prob.n_con)


# ---------------------------------------------------------------- 1, 2: the LM loop
@pytest.mark.parametrize("kind", ["plain", "covx", "cams"])
@pytest.mark.parametrize("name", ROWS)
def test_one_trial_is_the_dense_point_prior_step(api, name, kind):
    prob, opt = _make(name)
    covx = od.random_covx(prob.nobs, np.random.default_rng(5))[0] if kind != "plain" else None
    pr = _cams(prob, 6) if kind == "cams" else None
    pp = _pts(prob, 7, extra=bd.unobserved_indices(prob)[:3])
    info, after = _solve(api, prob, opt, "run_fixed", pp, pr, covx, trials=1)
    r = ppd.check_pptrial(prob, covx, pr, pp, info, after, opt)
    print(name, kind, " ".join(f"{k} {v:.2e}" for k, v in r.items()))


@pytest.mark.parametrize("name", ["rig_intrinsics", "unobserved_points", "banded"])
def test_trial_without_free_cameras(api, name):
    prob = _no_free_cameras(_make(name)[0])
    opt = _make(name)[1]
    pp = _pts(prob, 17, every=2, extra=bd.unobserved_indices(prob)[:3])
    info, after = _solve(api, prob, opt, "run_fixed", pp, trials=1)
    ppd.check_pptrial(prob, None, None, pp, info, after, opt)
    info, got = _solve(api, prob, _opt(1, 40, max_err=0.0), "run", pp)
    g0 = ppd.normal_equations(prob, 0.0, None, None, pp)[1]
    g1 = ppd.normal_equations(got, 0.0, None, None, pp)[1]
    assert np.linalg.norm(g1) <= 1e-8 * np.linalg.norm(g0)


@pytest.mark.parametrize("name", ROWS)
def test_run_zeroes_the_full_gradient(api, name):
    prob, _ = _make(name)
    pp = _pts(prob, 8, extra=bd.unobserved_indices(prob)[:3])
    pr = _cams(prob, 9)
    opt = _opt(1, 60, max_err=0.0)
    info, got = _solve(api, prob, opt, "run", pp, pr)
    g0 = ppd.normal_equations(prob, 0.0, None, pr, pp)[1]
    g1 = ppd.normal_equations(got, 0.0, None, pr, pp)[1]
    ratio = float(np.linalg.norm(g1) / np.linalg.norm(g0))
    print(f"{name}: {int(info[5])} iterations, stop {int(info[6])}, |g| / |g0| = {ratio:.2e}")
    assert ratio <= 1e-8
    assert abs(info[1] - ppd.total_cost(got, None, pr, pp)) <= 1e-9 * info[1]
    assert abs(info[0] - ppd.total_cost(prob, None, pr, pp)) <= 1e-9 * info[0]


# ---------------------------------------------------------------- 3: covariance stage
def _sparse_points(prob, max_err):
    """free points with zero and with one weighted observation"""
    e = bd.residuals(prob)
    w = bd.tukey_weights(np.sqrt((e * e).sum(1)), max_err)
    cnt = np.bincount(bd.point_of(prob)[w > 0], minlength=prob.n)
    free = np.arange(prob.n) >= prob.n_con
    return np.flatnonzero(free & (cnt == 0)), np.flatnonzero(free & (cnt == 1))


@pytest.mark.parametrize("name", COV_ROWS)
def test_covariance_stage_is_the_dense_inverse(api, name):
    prob, opt = _make_cov(name)
    z, one = _sparse_points(prob, opt.max_err)
    pp = _pts(prob, 10, every=4, extra=np.concatenate([z[:4], one[:4]]))
    s = api.BaSolver(prob.copy(), opt)
    _arm(s, pp)
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    assert cd.decision_margin(state, opt.max_err) >= 1e-6
    wcam, wpt, winf, H = ppd.cov_full(state, opt.max_err, VAR, None, None, pp)
    z1, one1 = _sparse_points(state, opt.max_err)
    print(name, "prior points with 0 / 1 weighted observations:", len(np.intersect1d(z1, pp.pts)),
          len(np.intersect1d(one1, pp.pts)), "unconstrained", winf["unconstrained"])
    assert np.isfinite(pt[pp.pts]).all()
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-8))
    assert inf["dof"] == winf["dof"] and inf["unconstrained"] == winf["unconstrained"]
    assert inf["pt_priors"] == len(pp) and inf["priors"] == 0
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= 1e-9 * winf["sigma2_hat"]


def test_covariance_with_both_kinds_of_priors(api):
    prob, opt = _make_cov("rig_intrinsics")
    pp, pr = _pts(prob, 11), _cams(prob, 12)
    s = api.BaSolver(prob.copy(), opt)
    _arm(s, pp, pr)
    s.set_covariance(VAR)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    wcam, wpt, winf, H = ppd.cov_full(state, opt.max_err, VAR, None, pr, pp)
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-8))
    assert inf["dof"] == winf["dof"] and inf["priors"] == len(pr) and inf["pt_priors"] == len(pp)
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= 1e-9 * winf["sigma2_hat"]


# ---------------------------------------------------------------- 4: edges
def test_unobserved_prior_point_goes_to_its_mean(api):
    prob, _ = cd.make("unobserved_points")
    u = bd.unobserved_indices(prob)
    i = int(u[u >= prob.n_con][0])
    rng = np.random.default_rng(42)
    cov = ppd.random_pt_cov(1, rng)
    pp = ppd.PtPriors([i], ppd.offset_pt_means(prob, [i], rng, 0.2), cov)
    s = api.BaSolver(prob.copy(), _opt(1, 60, max_err=0.0))
    _arm(s, pp)
    s.set_covariance(VAR)
    s.run()
    got = s.download()
    _, pt, inf = s.download_covariance()
    s.close()
    assert np.abs(got.X[i] - pp.X[0]).max() <= 1e-10
    want = VAR * cov[0]
    assert np.abs(pt[i] - want).max() <= 1e-8 * np.abs(want).max()
    assert inf["pt_priors"] == 1


def test_point_priors_fix_the_gauge(api):
    prob = gauge_free()
    opt = _opt(1, 30, max_err=0.0)
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(1.0)
    s.run()
    assert _raw_download(api, s)[0] == COSL_E_NUMERIC
    pts = gauge_points(prob, 3)
    cov = ppd.random_pt_cov(3, np.random.default_rng(41))
    pp = ppd.PtPriors(pts, ppd.draw_pt_means(prob, pts, cov, np.random.default_rng(43)), cov)
    s.reset(prob.copy())
    _arm(s, pp)
    s.run()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    s.close()
    wcam, wpt, winf, H = ppd.cov_full(state, 0.0, 1.0, None, None, pp)
    assert not winf["singular"]
    _close((cam, pt), (wcam, wpt), cd.far_tolerance(state, H, 1e-7))
    assert inf["dof"] == winf["dof"] and inf["pt_priors"] == 3


@pytest.mark.parametrize("how", ["run", "run_fixed", "submit"])
@pytest.mark.parametrize("name", ["rig_intrinsics", "tukey_mixed", "banded"])
def test_a_loose_prior_is_the_unarmed_handle(api, name, how):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6  # as test_gpu_ba_obscov: eps2 = 1e-12 leaves the accept decisions to the atomic sums' order
    pts = np.arange(prob.n_con, prob.n)
    pp = ppd.PtPriors(pts, ppd.offset_pt_means(prob, pts, np.random.default_rng(44)),
                      np.tile(1e12 * np.eye(3), (len(pts), 1, 1)))
    # an unobserved point with a loose prior is damped towards its mean instead of staying put: leave those out
    keep = ~np.isin(pts, bd.unobserved_indices(prob))
    ba_same_decisions(_solve(api, prob, opt, how), _solve(api, prob, opt, how, pp.subset(keep)), prob)


@pytest.mark.parametrize("name", ["rig_intrinsics", "banded"])
def test_cleared_or_loaded_over_is_never_set(api, name):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6
    unarmed = _solve(api, prob, opt, "run")
    s = api.BaSolver(prob.copy(), opt)
    for clear in ("none", "empty", "load"):
        _arm(s, _pts(prob, 13))
        if clear == "none":
            s.set_pt_prior(None)
        elif clear == "empty":
            s.set_pt_prior([], [], [])
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


def test_clearing_one_kind_keeps_the_other(api):
    prob, opt = _make("rig_intrinsics")
    opt.opts[2] = 1e-6
    pp, pr = _pts(prob, 14), _cams(prob, 15)
    only_pts, both = _solve(api, prob, opt, "run", pp), _solve(api, prob, opt, "run", pp, pr)
    s = api.BaSolver(prob.copy(), opt)
    s.set_cam_prior(pr.cams, pr.R, pr.t, pr.cov)
    only_cams = (s.run(), bd.fresh(s.download()))
    s.reset(prob.copy())
    _arm(s, pp, pr)
    s.set_cam_prior(None)
    ba_same_decisions(only_pts, (s.run(), bd.fresh(s.download())), prob)
    s.reset(prob.copy())
    s.set_cam_prior(pr.cams, pr.R, pr.t, pr.cov)
    ba_same_decisions(both, (s.run(), bd.fresh(s.download())), prob)
    s.reset(prob.copy())
    s.set_pt_prior(None)
    ba_same_decisions(only_cams, (s.run(), bd.fresh(s.download())), prob)
    s.close()


# ---------------------------------------------------------------- 5: entry points
@pytest.mark.parametrize("name", ROWS)
def test_run_and_submit_agree(api, name):
    prob, opt = _make(name)
    opt.opts[2] = 1e-6
    pp = _pts(prob, 16)
    ba_same_decisions(_solve(api, prob, opt, "run", pp), _solve(api, prob, opt, "submit", pp), prob)
    a = _solve(api, prob, opt, "run_fixed", pp, trials=4)
    b = _solve(api, prob, opt, "run_fixed", pp, trials=4)
    ba_same_decisions(a, b, prob)


def test_submit_after_the_priors_changed(api):
    prob, opt = _make("rig_intrinsics")
    opt.opts[2] = 1e-6
    p1, p2 = _pts(prob, 18), _pts(prob, 19, every=2)
    s = api.BaSolver(prob.copy(), opt)
    results = []
    for pp in (None, p1, p2, p2.subset(np.arange(len(p2)) % 2 == 0), None):
        s.reset(prob.copy())
        if pp is None:
            s.set_pt_prior(None)
        else:
            _arm(s, pp)
        s.submit()
        info = s.collect()
        results.append((pp, (info, bd.fresh(s.download()))))
    s.close()
    for pp, got in results:
        ba_same_decisions(_solve(api, prob, opt, "run", pp), got, prob)


def test_stop_during_a_prior_armed_submit(api):
    torch = _torch_cuda()
    prob, opt = _make("rig_intrinsics")
    pp = _pts(prob, 20)
    s = api.BaSolver(prob.copy(), opt)
    _arm(s, pp)
    _sleep_on(torch, s, int(5e8))
    s.submit()
    s.stop()
    info = s.collect()
    assert int(info[6]) == STOPPED
    p = s.progress()
    want = ppd.total_cost(prob, None, None, pp, opt.max_err)
    assert abs(p["cost"] - want) <= 1e-9 * want and abs(info[0] - want) <= 1e-9 * want
    assert ppd.pt_prior_cost(prob, pp) > 1e-3 * want  # the priors are a visible part of it
    s.reset(prob.copy())
    s.submit()
    info = s.collect()
    p = s.progress()
    got = s.download()
    s.close()
    assert p["cost"] == info[12] and int(info[6]) != STOPPED
    assert info[12] >= ppd.pt_prior_cost(got, pp) > 0


# ---------------------------------------------------------------- 6: Monte Carlo
def test_monte_carlo_nees(api):
    truth = cd.small_nonrobust()
    rng = np.random.default_rng(79)
    covx, S = od.random_covx(truth.nobs, rng)
    pts = np.arange(truth.n_con, truth.n)[::2]
    cov = ppd.random_pt_cov(len(pts), rng, sig=(0.002, 0.02))
    s = api.BaSolver(truth.copy(), _opt(1, 30, max_err=0.0))
    s.set_covariance(1.0)
    nees, nees_prior = [], []
    for _ in range(200):
        p = bd.fresh(truth)
        p.xy = truth.xy + od.draw_noise(S, rng)
        s.load(p)
        s.set_obs_cov(covx)
        s.set_pt_prior(pts, ppd.draw_pt_means(truth, pts, cov, rng), cov)
        s.run()
        got = s.download()
        _, pt, inf = s.download_covariance()
        assert inf["pt_priors"] == len(pts)
        d = got.X - truth.X
        q = np.einsum("ni,ni->n", d, np.linalg.solve(pt, d[:, :, None])[:, :, 0])
        nees.extend(q[truth.n_con:])
        nees_prior.extend(q[pts])
    s.close()
    m, mp = float(np.mean(nees)), float(np.mean(nees_prior))
    print(f"mean point NEES {m:.3f} (3), prior points {mp:.3f} (3)")
    assert abs(m - 3) <= 0.15 * 3 and abs(mp - 3) <= 0.15 * 3


# ---------------------------------------------------------------- 7: state and validation
def _raw_set(api, s, pts, X, cov, n=None):
    vp = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)  # noqa: E731
    pts = None if pts is None else np.ascontiguousarray(pts, np.int32)
    X = None if X is None else np.ascontiguousarray(X, np.float64)
    cov = None if cov is None else np.ascontiguousarray(cov, np.float64)
    k = len(pts) if n is None else n
    rc = api.LIB.cosl_ba_solver_set_pt_prior(s.h, k, vp(pts), vp(X), vp(cov))
    return rc, api.LIB.cosl_last_error().decode()


def _bad_cases(prob, pp):
    """name -> (pts, X, cov) with prior 1 (and prior 2, which must not be named) broken"""
    def edit(f):
        c, X, P = pp.pts.copy(), pp.X.copy(), pp.cov.copy()
        for k in (1, 2):
            f(k, c, X, P)
        return c, X, P

    def at(k, c, j):
        c[k] = j

    return {
        "fixed_point": edit(lambda k, c, X, P: at(k, c, prob.n_con - 1)),
        "negative": edit(lambda k, c, X, P: at(k, c, -1)),
        "past_the_end": edit(lambda k, c, X, P: at(k, c, prob.n)),
        "repeated": edit(lambda k, c, X, P: at(k, c, c[0])),
        "nan_X": edit(lambda k, c, X, P: X.__setitem__((k, 1), np.nan)),
        "inf_cov": edit(lambda k, c, X, P: P.__setitem__((k, 2, 2), np.inf)),
        "asymmetric": edit(lambda k, c, X, P: P.__setitem__((k, 0, 2), P[k, 0, 2] + 1e-9 * P[k].max())),
        "indefinite": edit(lambda k, c, X, P: P.__setitem__(k, P[k] - 2 * np.eye(3) * np.linalg.eigvalsh(P[k])[0])),
        "zero": edit(lambda k, c, X, P: P.__setitem__(k, 0.0)),
    }


def test_state_and_validation(api):
    torch = _torch_cuda()
    prob, opt = _make("rig_intrinsics")
    assert prob.n_con >= 1
    opt.opts[2] = 1e-6
    pp = _pts(prob, 21, every=5)
    assert len(pp) >= 3
    s = api.BaSolver(prob.copy(), opt)
    _sleep_on(torch, s, int(5e8))
    s.submit()
    assert _raw_set(api, s, pp.pts, pp.X, pp.cov)[0] == COSL_E_STATE
    assert _raw_set(api, s, None, None, None, n=0)[0] == COSL_E_STATE
    s.collect()
    unarmed = _solve(api, prob, opt, "run")
    armed = _solve(api, prob, opt, "run", pp)
    other = _pts(prob, 22, every=4)
    armed_other = _solve(api, prob, opt, "run", other)
    # every invalid set names prior 1 and keeps what the handle had: first nothing, then `pp`
    for keep, want in ((None, unarmed), (pp, armed)):
        if keep is not None:
            _arm(s, keep)
        for name, (c, X, P) in _bad_cases(prob, other).items():
            rc, msg = _raw_set(api, s, c, X, P)
            assert rc == COSL_E_INVALID and "prior 1 " in msg, (name, rc, msg)
        rc, msg = _raw_set(api, s, other.pts, other.X, other.cov, n=-1)
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
        s.set_pt_prior(pp.pts, pp.X[:-1], pp.cov)
    s.close()
