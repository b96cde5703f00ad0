"""The BA solver's covariance stage at its edge shapes (the scenes of tests/ba_cov_dense.py's EDGE_ROWS): no free
camera (no reduced system, min_pivot = +inf), every point fixed (no pair pass), free cameras that see only fixed
points, single-observation and weight-dropped points on free cameras, one camera pair whose Schur items split,
camera groups that share no point (uncoupled blocks of the selected inversion, a block-diagonal S), fixed points as
the only gauge, and 50 000 points (more than one pass of ba_cov_begin's clear).  Each regular scene runs through
run and through submit / collect against the float64 reference at the downloaded parameters; the scenes with a
camera that sees nothing are refused; one armed handle takes problems of other shapes in turn."""
import numpy as np
import pytest

import ba_cov_dense as cd
from test_gpu_ba_async import _opt
from test_gpu_ba_covariance import COSL_E_NUMERIC, VAR, _close, _no_steps, _raw_download

pytestmark = pytest.mark.gpu


def _solve(api, prob, opt, how):
    """(state, camCov, ptCov, info, plan, stats) of one armed BA on a fresh handle by run or by submit / collect."""
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(VAR)
    if how == "run":
        s.run()
    else:
        s.submit()
        s.collect()
    state = s.download()
    cam, pt, inf = s.download_covariance()
    plan, stats = s.plan_info(), s.stats()
    s.close()
    return state, cam, pt, inf, plan, stats


def _against_reference(state, cam, pt, inf, max_err, what):
    """parity with the reference at state; returns the bound used"""
    margin = cd.decision_margin(state, max_err) if max_err > 0 else 1.0
    assert margin >= 1e-6, (what, "a Tukey decision at the rounding floor", margin)
    wcam, wpt, winf, H = cd.reference(state, max_err, VAR)
    tol = cd.far_tolerance(state, H, 1e-8) if H is not None else 1e-8
    print(f"{what}: ", end="")
    _close((cam, pt), (wcam, wpt), tol)
    assert inf["pixel_var"] == VAR
    assert inf["dof"] == winf["dof"] and inf["unconstrained"] == winf["unconstrained"], (inf, winf)
    assert abs(inf["sigma2_hat"] - winf["sigma2_hat"]) <= max(1e-9, tol) * winf["sigma2_hat"]
    if state.m == state.m_con:
        assert inf["min_pivot"] == np.inf  # no free camera, no pivot
    else:
        assert 1e-12 <= inf["min_pivot"] <= 1.0
    return tol


@pytest.mark.parametrize("how", ["run", "submit"])
@pytest.mark.parametrize("name", sorted(cd.EDGE_ROWS))
def test_parity_with_the_dense_reference(api, name, how):
    prob, opt = cd.make_edge(name)
    state, cam, pt, inf, plan, stats = _solve(api, prob, opt, how)
    _against_reference(state, cam, pt, inf, opt.max_err, f"{name} ({how})")
    mf = prob.m - prob.m_con
    assert stats["ns"] == 6 * mf
    if name == "structure_only":
        assert not cam.any()
    if name == "motion_only":
        assert not pt.any() and stats["pair_entries"] == 0
    if name in ("single_observation_points_fixed", "weight_dropped_points"):
        assert np.isnan(pt[-10:]).all()
    if name == "one_long_pair_fixed":
        # buckets (0,0), (0,1), (1,1) of 532 entries each, cut into items of <= 128 entries
        assert stats["pair_entries"] == 3 * 532 and stats["pair_items"] == 3 * 5
    if name.startswith("groups_"):
        k, g = map(int, name.split("_")[1].split("x"))
        if g in (6, 10):  # the groups fall on the planner's cuts: uncoupled blocks, no tile off the diagonal
            assert plan["blocks"] == k and plan["tiles"] == k, plan
        else:  # 25 free cameras: three blocks of unequal rows (54 / 48 / 48)
            assert plan["blocks"] == 3, plan
    if name == "points_fix_gauge":
        assert prob.m_con == 0 and (np.linalg.eigvalsh(cam) > 0).all()


@pytest.mark.parametrize("name", sorted(cd.SINGULAR_EDGE_ROWS))
def test_blind_camera_is_refused(api, name):
    """A free camera without observations (first, middle or last block of three): the BA collects with COSL_OK, the
    covariance is refused with COSL_E_NUMERIC and nothing is written; the min-pivot reduction sees the singular
    block wherever it is."""
    prob, opt = cd.make_edge(name)
    s = api.BaSolver(prob.copy(), opt)
    assert s.plan_info()["blocks"] == 3
    s.set_covariance(VAR)
    s.submit()
    s.collect()
    rc, cam, pt, out = _raw_download(api, s)
    assert rc == COSL_E_NUMERIC
    assert (cam == 7.0).all() and (pt == 7.0).all() and out == [7.0] * 8
    assert "singular" in api.LIB.cosl_last_error().decode()
    s.close()


def test_many_points_twice_on_one_handle(api):
    """50 000 points, no LM step: two stages on one handle agree with each other and the reference; a T that the
    second stage did not clear completely would double some point blocks."""
    prob, _ = cd.make_edge("many_points")
    opt = _no_steps()
    s = api.BaSolver(prob.copy(), opt)
    s.set_covariance(VAR)
    got = []
    for _ in range(2):
        info = s.run()
        assert info[5] == 0  # the parameters did not move
        got.append(s.download_covariance())
    state = s.download()
    s.close()
    print("second against first: ", end="")
    _close(got[1][:2], got[0][:2], 1e-9)
    for cam, pt, inf in got:
        _against_reference(state, cam, pt, inf, opt.max_err, "many_points")


# one handle, problems of other shapes in turn: multi-block, no free camera, an uncoupled pair, a singular one,
# every point fixed, the first again.  max_err 30 keeps motion_only's cameras observed at the start.
RELOADS = ["groups_3x10", "structure_only", "groups_2x6", "groups_3x10_blind1", "motion_only", "groups_3x10"]


@pytest.mark.parametrize("how", ["run", "submit"])
def test_reloads_on_one_armed_handle(api, how):
    opt = _opt(1, 10, max_err=30.0, o1=1e300)  # no LM step: a fresh handle sees the same parameters
    probs = [cd.make_edge(name)[0] for name in RELOADS]
    s = api.BaSolver(probs[0].copy(), opt)
    s.set_covariance(VAR)
    for name, prob in zip(RELOADS, probs):
        s.load(prob.copy())
        if how == "run":
            s.run()
        else:
            s.submit()
            s.collect()
        if name in cd.SINGULAR_EDGE_ROWS:
            assert _raw_download(api, s)[0] == COSL_E_NUMERIC, name
            continue
        cam, pt, inf = s.download_covariance()
        state = s.download()
        fstate, fcam, fpt, finf, _, _ = _solve(api, prob, opt, how)
        assert np.array_equal(state.X, fstate.X) and np.array_equal(state.t, fstate.t)
        H = cd.reference(state, opt.max_err, VAR)[3]
        print(f"{name} reloaded against a fresh handle: ", end="")
        _close((cam, pt), (fcam, fpt), cd.far_tolerance(state, H, 1e-9))
        assert inf["dof"] == finf["dof"] and inf["unconstrained"] == finf["unconstrained"]
        assert inf["min_pivot"] == finf["min_pivot"] or abs(inf["min_pivot"] - finf["min_pivot"]) <= 1e-9 * finf[
            "min_pivot"]
        _against_reference(state, cam, pt, inf, opt.max_err, f"{name} reloaded ({how})")
    s.close()
