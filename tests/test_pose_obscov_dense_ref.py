"""The whitened pose references of tests/pose_obscov_dense.py without a GPU, before any GPU test trusts them: the
factors against the covariances they whiten, identity covariances reproduce pose_dense and pose_cov_dense, Sigma = 4I
quarters the cost exactly, and the whitened solve lands on the minimiser that scipy.optimize.least_squares finds for
the same whitened residuals."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import pose_cov_dense as cd
import pose_dense as pd
import pose_obscov_dense as od
from coslam_b200 import synth

TAU = 10.0


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _case(seed, n=192, **kw):
    K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n_pts=n, seed=seed, **kw)
    return K, R0, t0, Ms, ms


def test_factors_whiten_their_covariances():
    rng = np.random.default_rng(3)
    cov, _ = od.random_covx(500, rng)
    Lf = od.factors(cov)
    L = np.zeros((500, 2, 2))
    L[:, 0, 0], L[:, 0, 1], L[:, 1, 1] = Lf[:, 0], Lf[:, 1], Lf[:, 2]
    assert (Lf[:, 0] > 0).all() and (Lf[:, 2] > 0).all()
    cond = np.linalg.cond(cov)
    assert cond.max() > 50 and cond.max() <= 100 * (1 + 1e-9)
    err = np.abs(np.einsum("nba,nbc,ncd->nad", L, L, cov) - np.eye(2)).max()
    assert err <= 1e-13 * cond.max(), err
    one = od.factors(od.identity(3))
    assert np.array_equal(_bits(one), _bits(np.tile([1.0, -0.0, 1.0], (3, 1))))
    assert np.array_equal(_bits(od.factors(4 * od.identity(3))), _bits(np.tile([0.5, -0.0, 0.5], (3, 1))))


@pytest.mark.parametrize("seed,prev,opt", [(3, False, pd.DEFAULT_OPT), (17, True, pd.DEFAULT_OPT),
                                           (29, True, (100, 1) + pd.DEFAULT_OPT[2:])])
def test_identity_covariances_are_pose_dense(seed, prev, opt):
    K, R0, t0, Ms, ms = _case(seed)
    pe = np.abs(np.random.default_rng(seed).normal(0, 4, len(Ms))) if prev else None
    ok, R, t, f = pd.estimate(K, R0, t0, Ms, ms, TAU, pe, opt)
    for covx in (None, od.identity(len(Ms)), od.identity(len(Ms)).reshape(-1, 2, 2)):
        ok_w, R_w, t_w, f_w = od.estimate(K, R0, t0, Ms, ms, TAU, pe, opt, covx)
        assert ok_w == ok and np.array_equal(_bits(R_w), _bits(R)) and np.array_equal(_bits(t_w), _bits(t))
        assert {k: np.float64(v).tobytes() for k, v in f_w.items()} == {k: np.float64(v).tobytes() for k, v in f.items()}
    st, st_w = cd.cov_stage(K, R, t, Ms, ms, TAU, 1.0), od.cov_stage(K, R, t, Ms, ms, TAU, 1.0, od.identity(len(Ms)))
    assert np.array_equal(_bits(st_w["H"]), _bits(st["H"])) and np.array_equal(_bits(st_w["e"]), _bits(st["e"]))
    assert st_w["dof"] == st["dof"] and st_w["sigma2_hat"] == pytest.approx(st["sigma2_hat"], rel=1e-14)


def test_four_identity_quarters_the_cost():
    K, R0, t0, Ms, ms = _case(5)
    n = len(Ms)
    W = pd.prev_weights(n, TAU, None)
    L1, L4 = od.factors(od.identity(n)), od.factors(4 * od.identity(n))
    assert od.cost(K, R0, t0, W, Ms, ms, L4) == od.cost(K, R0, t0, W, Ms, ms, L1) / 4
    # err0 is the cost at the start of the last re-weighting round: one round starts both at R0, t0
    opt = (100, 1) + pd.DEFAULT_OPT[2:]
    _, _, _, f1 = od.estimate(K, R0, t0, Ms, ms, TAU, None, opt)
    _, _, _, f4 = od.estimate(K, R0, t0, Ms, ms, TAU, None, opt, 4 * od.identity(n))
    assert f4["err0"] == f1["err0"] / 4


@pytest.mark.parametrize("seed", [7, 23, 41])
def test_whitened_solve_reaches_the_least_squares_minimum(seed):
    """prevErrs None and maxIterRW = 1: every weight is 1, so the solve minimises sum |L (m - project)|^2; scipy's
    trust-region solver on the same residuals in the same chart finds the same pose."""
    rng = np.random.default_rng(seed)
    K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(192, seed=seed, noise_px=0.0, outlier_frac=0.0)
    cov, S = od.random_covx(len(Ms), rng)
    ms = ms + od.draw_noise(S, rng)
    opt = (100, 1) + pd.DEFAULT_OPT[2:]
    ok, R, t, f = od.estimate(K, R0, t0, Ms, ms, TAU, None, opt, cov)
    Lf = od.factors(cov)

    def res(x):
        u, v = pd.project(K, R0 @ pd.exp_map(x[:3]), t0 + x[3:], Ms)
        return np.concatenate(od.whiten(Lf, ms[:, 0] - u, ms[:, 1] - v))

    sol = least_squares(res, np.zeros(6), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    R_ls, t_ls = R0 @ pd.exp_map(sol.x[:3]), t0 + sol.x[3:]
    assert ok and f["nIterRW"] == 1
    # the solve stops once |delta|^2 < epsParamChangeLM or the cost moves by less than epsErrorChangeLM: its pose is
    # the minimiser's to about 1e-7 and its cost the minimum's to far below one part in 1e9
    assert np.abs(R - R_ls).max() < 1e-6 and np.abs(t - t_ls).max() < 1e-6, (np.abs(R - R_ls).max(),
                                                                              np.abs(t - t_ls).max())
    assert od.cost(K, R, t, np.ones(len(Ms)), Ms, ms, Lf) == pytest.approx(2 * sol.cost, rel=1e-9)
