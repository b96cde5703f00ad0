"""The covariance references of tests/ba_cov_dense.py against each other, without a GPU, so that the reference is
pinned before it judges the device: the full-H inverse with the solver-chart Jacobian (x4 chart factor), the
same with the Jacobian taken straight through exp([w]x), and the Schur form."""
import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd

VAR = 2.5


@pytest.mark.parametrize("name", sorted(cd.cov_rows()))
def test_references_agree_on_the_dense_scenes(name):
    prob, opt = cd.make(name)
    cam, pt, info, H = cd.cov_full(prob, opt.max_err, VAR)
    cam_x, pt_x, info_x, _ = cd.cov_full(prob, opt.max_err, VAR, jac=cd.expmap_jacobian)
    cam_s, pt_s, info_s = cd.cov_schur(prob, opt.max_err, VAR)
    tol = cd.far_tolerance(prob, H, 1e-9)
    for a, b in ((cam_x, cam), (cam_s, cam), (pt_x, pt), (pt_s, pt)):
        err, same = cd.block_errors(a, b)
        assert same
        assert err.max() <= tol, (name, float(err.max()), tol)
    assert info == info_s
    assert info_x["dof"] == info["dof"] and info_x["unconstrained"] == info["unconstrained"]
    # fixed blocks are zero, free blocks symmetric positive definite
    assert not cam[:prob.m_con].any() and not pt[:prob.n_con].any()
    free = cam[prob.m_con:]
    assert np.allclose(free, free.transpose(0, 2, 1), rtol=0, atol=max(1e-12, tol) * np.abs(free).max())
    if name != "far_offset":  # there float64 cannot resolve H (far_tolerance is near 1)
        assert (np.linalg.eigvalsh(free) > 0).all()


def test_long_tracks_is_singular():
    """Its last camera has one observation: H has no inverse (what the device reports as COSL_E_NUMERIC)."""
    prob, opt = bd.make("long_tracks")
    _, w, _ = cd.weights(prob, opt.max_err)
    assert ((prob.cam == prob.m - 1) & (w > 0)).sum() == 1
    H = cd.cov_full(cd.long_tracks_seen(), opt.max_err, VAR)[3]
    assert np.linalg.cond(H) < 1e12


def test_unobserved_and_tukey_rows_leave_points_out():
    prob, opt = bd.make("unobserved_points")
    _, pt, info, _ = cd.cov_full(prob, opt.max_err, VAR)
    gone = bd.unobserved_indices(prob)
    free_gone = gone[gone >= prob.n_con]
    assert info["unconstrained"] == len(free_gone) > 0
    assert np.isnan(pt[free_gone]).all()
    assert not pt[gone[gone < prob.n_con]].any()
    prob, opt = bd.make("tukey_mixed")
    _, w, _ = cd.weights(prob, opt.max_err)
    assert (w == 0).sum() > prob.nobs // 5  # the outliers drop out of H


def test_banded_scene_is_dissected():
    prob = cd.banded()
    cam, pt, info, _ = cd.cov_full(prob, 0.0, 1.0)
    cam_s, pt_s, _ = cd.cov_schur(prob, 0.0, 1.0)
    assert prob.m - prob.m_con >= 40
    for a, b in ((cam_s, cam), (pt_s, pt)):
        err, same = cd.block_errors(a, b)
        assert same and err.max() < 1e-8
