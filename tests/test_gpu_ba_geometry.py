"""The bundle adjustment on scenes beyond a one-camera rig (tests/ba_dense.py): per-camera intrinsics with
fx != fy and skew, depths from 0.3 to 800 m, a world 1e4 m from the origin, starts several degrees off, point
runs that cross warp and block boundaries, points nobody observes, Tukey weights at the cut-off and points
whose observations are not sorted by camera.  On every row:
  - one trial of BaSolver.run_fixed(1) passes the dense float64 checks (backward error, forward error,
    costs before and after), which print their measured values beside their bounds;
  - four trials agree with the CPU oracle;
  - the robust solve (2 rounds of 10 iterations; 1 round without robust weights) takes the same decisions
    through run and through submit / collect, and lands where the oracle's does.
cosl_sba_motstr_levmar_x is checked with each camera's own (fx, cx, cy, ar, s) and a nonzero initial local
rotation on fixed and free cameras."""
import ctypes as C

import numpy as np
import pytest

import ba_dense as D
from helpers import ba_same_decisions

pytestmark = pytest.mark.gpu

ROWS = list(D.ROWS)


def robust_options(max_err):
    # eps4 = 1e-9 ends a round on a relative cost reduction far above the noise of the device's atomic sums,
    # so that run and submit take every decision away from a tie.  Without robust weights a second round
    # would restart at the converged point of the same problem, where every decision is such a tie: one round
    opt = D.options(max_err)
    opt.outer_iters, opt.inner_iters = (2 if max_err > 0 else 1), 10
    opt.opts[4] = 1e-9
    return opt


def displacement_close(got, want, start, rel):
    """|got - want| <= rel |want - start| + the rounding of the stored values, per array (t, X) and for R."""
    for a in ("t", "X"):
        g, w, s = getattr(got, a), getattr(want, a), getattr(start, a)
        tol = rel * np.abs(w - s).max() + 4 * D.EPS * np.abs(w).max()
        assert np.abs(g - w).max() <= tol, (a, np.abs(g - w).max(), tol)
    tolR = rel * np.abs(want.R - start.R).max() + 8 * D.EPS
    assert np.abs(got.R - want.R).max() <= tolR, ("R", np.abs(got.R - want.R).max(), tolR)


def fixed_untouched(got, prob):
    assert np.array_equal(got.R[:prob.m_con], prob.R[:prob.m_con])
    assert np.array_equal(got.t[:prob.m_con], prob.t[:prob.m_con])
    assert np.array_equal(got.X[:prob.n_con], prob.X[:prob.n_con])
    u = D.unobserved_indices(prob)
    assert np.array_equal(got.X[u], prob.X[u])


@pytest.mark.parametrize("name", ROWS)
def test_one_trial_passes_the_dense_checks(api, name):
    prob, opt = D.make(name)
    s = api.BaSolver(D.fresh(prob), opt)
    info = s.run_fixed(1)
    after = s.download()
    s.close()
    r = D.check_trial(prob, info, after, opt)
    fixed_untouched(after, prob)
    print(name, " ".join(f"{k} {v:.2e}" for k, v in r.items()))


@pytest.mark.parametrize("name", ROWS)
def test_four_trials_match_the_oracle(api, orc, name):
    prob, opt = D.make(name)
    pg, po = D.fresh(prob), D.fresh(prob)
    s = api.BaSolver(pg, opt)
    ig = s.run_fixed(4)
    s.download()
    s.close()
    io = orc.ba_run_fixed(po, opt, 4)
    assert ig[9] == io[9] == 4
    # 1e-9 relative, or the float64 cancellation bound of the scene where it is larger (far_offset)
    tol = max(1e-9, D.Trial(prob, opt).cost_tol(po))
    assert abs(ig[0] - io[0]) <= tol * io[0] and abs(ig[1] - io[1]) <= tol * io[1], (ig[:2], io[:2], tol)
    displacement_close(pg, po, prob, 1e-6)
    fixed_untouched(pg, prob)
    print(name, f"cost {abs(ig[1] - io[1]) / io[1]:.2e} (bound {tol:.1e})")


@pytest.mark.parametrize("name", ROWS)
def test_robust_solve_submit_matches_run_and_oracle(api, orc, name):
    prob, opt = D.make(name)
    opt = robust_options(opt.max_err)
    runs = []
    for submitted in (False, True):
        s = api.BaSolver(D.fresh(prob), opt)
        if submitted:
            s.submit()
            info = s.collect()
        else:
            info = s.run()
        runs.append((info, s.download()))
        s.close()
    ba_same_decisions(runs[0], runs[1], prob)
    ig, pg = runs[1]
    fixed_untouched(pg, prob)
    po = D.fresh(prob)
    io = orc.ba_solve(po, opt)
    assert np.array_equal(ig[5:11], io[5:11]), (ig[:11], io[:11])
    tol = max(1e-9, D.Trial(prob, opt).cost_tol(po))
    assert abs(ig[12] - io[12]) <= tol * io[12], (ig[12], io[12], tol)
    displacement_close(pg, po, prob, 1e-6)
    assert np.array_equal(pg.outlier, po.outlier)


def test_unsorted_observations_equal_the_sorted_permutation(api):
    """Observations of a point in any camera order give the answer of the sorted list (the Schur pair lists
    compare camera indices, not positions), up to the order of the atomic sums."""
    prob, opt = D.make("unsorted_observations")
    srt, perm = D.sorted_permutation(prob)
    out = []
    for p in (prob, srt):
        s = api.BaSolver(D.fresh(p), robust_options(opt.max_err))
        info = s.run()
        out.append((info, s.download()))
        s.close()
    (ia, pa), (ib, pb) = out
    assert np.array_equal(ia[5:11], ib[5:11])
    assert abs(ia[12] - ib[12]) <= 1e-9 * ib[12]
    assert np.abs(pa.R - pb.R).max() < 1e-9 and np.abs(pa.t - pb.t).max() < 1e-9 and np.abs(pa.X - pb.X).max() < 1e-8
    assert np.array_equal(pa.outlier[perm], pb.outlier)
    # the one-call entry point accepts it too (and keeps it: the solvers above loaded the same lists)
    q = D.fresh(prob)
    info = api.ba_solve(q, opt)
    assert info[1] < info[0] and np.array_equal(q.cam, prob.cam) and np.array_equal(q.xy, prob.xy)


def test_unobserved_points_change_nothing(api):
    """The same scene without its unobserved points: the same trials and costs; the unobserved points come
    back bit for bit."""
    prob, opt = D.make("unobserved_points")
    u = D.unobserved_indices(prob)
    keep = np.setdiff1d(np.arange(prob.n), u)
    k = np.diff(prob.ptr)[keep]
    without = D.BAProblem(prob.K.copy(), prob.R, prob.t, prob.X[keep], np.concatenate([[0], np.cumsum(k)]),
                          prob.cam.copy(), prob.xy.copy(), prob.m_con, prob.n_con - 1)
    res = []
    for p in (prob, without):
        s = api.BaSolver(D.fresh(p), robust_options(opt.max_err))
        res.append((s.run(), s.download()))
        s.close()
    (ia, pa), (ib, pb) = res
    assert np.array_equal(ia[5:11], ib[5:11])
    assert abs(ia[0] - ib[0]) <= 1e-12 * ib[0] and abs(ia[12] - ib[12]) <= 1e-9 * ib[12]
    assert np.array_equal(pa.X[u], prob.X[u])
    assert np.abs(pa.X[keep] - pb.X).max() < 1e-8 and np.abs(pa.t - pb.t).max() < 1e-9


# ---------------------------------------------------------------- cosl_sba_motstr_levmar_x
def _sba(fn, prob, p, rot0, vmask, itmax, opts, *dev):
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    info = np.zeros(10)
    rc = fn(prob.n, prob.n_con, prob.m, prob.m_con, vp(vmask), vp(p), 11, 3, vp(prob.xy), 2, vp(rot0), itmax, 0,
            vp(opts), vp(info), *dev)
    return rc, info


def test_sba_wrapper_with_per_camera_intrinsics_and_initial_rotations(api, orc):
    prob, _ = D.make("rig_intrinsics")
    rng = np.random.default_rng(21)
    dq = rng.normal(size=(prob.m, 3)) * 0.04  # every camera, fixed ones included, starts with a local rotation
    p0, rot0, vmask = D.pack_sba(prob, dq)
    c0 = p0[:11 * prob.m].reshape(prob.m, 11)
    assert np.any(c0[:, 3] != 1.0) and np.any(c0[:, 4] != 0.0)
    opts = np.array([1e-7, 1e-12, 1e-12, 0.0, 1e-16])
    itmax = 4
    pg = p0.copy()
    rg, ig = _sba(api.LIB.cosl_sba_motstr_levmar_x, prob, pg, rot0, vmask, itmax, opts, 0)
    po = p0.copy()
    ro, io = _sba(orc.lib().orc_sba_motstr_levmar_x, prob, po, rot0, vmask, itmax, opts)
    assert rg == ro == itmax, (rg, ro)
    # the same problem unpacked in numpy, through cosl_ba_solve
    up = D.unpack_sba(p0, rot0, vmask, prob.xy, prob.m_con, prob.n_con)
    opt = D.options(0.0)
    opt.outer_iters, opt.inner_iters = 1, itmax
    opt.opts[:] = opts
    iu = api.ba_solve(up, opt)
    assert np.array_equal(ig[5:10], iu[5:10]) and np.array_equal(ig[5:10], io[5:10]), (ig, iu, io)
    assert abs(ig[0] - iu[0]) <= 1e-12 * iu[0] and abs(ig[1] - iu[1]) <= 1e-9 * iu[1], (ig[:2], iu[:2])
    assert abs(ig[1] - io[1]) <= 1e-9 * io[1], (ig[:2], io[:2])
    want, _, _ = D.pack_sba(up, np.zeros((prob.m, 3)))
    cg, cw = pg[:11 * prob.m].reshape(prob.m, 11), want[:11 * prob.m].reshape(prob.m, 11)
    # the wrapper hands back each free camera's rotation relative to rot0: vec(q(R) (x) conj(rot0))
    qR = D.R_to_quat(up.R)
    rel = D.quat_mul(qR, rot0 * [1, -1, -1, -1])
    rel[rel[:, 0] < 0] *= -1
    free = slice(prob.m_con, prob.m)
    assert np.abs(cg[free, 5:8] - rel[free, 1:]).max() < 1e-9
    assert np.abs(cg[free, 8:] - cw[free, 8:]).max() < 1e-9
    assert np.abs(pg[11 * prob.m:] - want[11 * prob.m:]).max() < 1e-8
    assert np.abs(pg - po).max() < 1e-6
    # fixed cameras keep their (intrinsics and) initial local rotation, fixed points stay put
    assert np.array_equal(pg[:11 * prob.m_con], p0[:11 * prob.m_con])
    assert np.array_equal(cg[:, :5], c0[:, :5])
    nf = 11 * prob.m + 3 * prob.n_con
    assert np.array_equal(pg[11 * prob.m:nf], p0[11 * prob.m:nf])
    assert ig[1] < ig[0]
