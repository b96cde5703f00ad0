"""The covariance references of tests/ba_cov_dense.py against each other, without a GPU, so that the reference is
pinned before it judges the device: the full-H inverse with the solver-chart Jacobian (x4 chart factor), the
same with the Jacobian taken straight through exp([w]x), and the Schur form."""
import numpy as np
import pytest

import ba_cov_dense as cd
import ba_dense as bd

VAR = 2.5


SMALL_EDGE_ROWS = sorted(set(cd.EDGE_ROWS) - set(cd.LARGE))


@pytest.mark.parametrize("name", sorted(cd.cov_rows()) + SMALL_EDGE_ROWS)
def test_references_agree_on_the_dense_scenes(name):
    prob, opt = cd.make(name) if name in cd.cov_rows() else cd.make_edge(name)
    cam, pt, info, H = cd.cov_full(prob, opt.max_err, VAR)
    cam_x, pt_x, info_x, _ = cd.cov_full(prob, opt.max_err, VAR, jac=cd.expmap_jacobian)
    cam_s, pt_s, info_s = cd.cov_schur(prob, opt.max_err, VAR)
    tol = cd.far_tolerance(prob, H, 1e-9)
    for a, b in ((cam_x, cam), (cam_s, cam), (pt_x, pt), (pt_s, pt)):
        err, same = cd.block_errors(a, b)
        assert same
        assert err.max(initial=0) <= tol, (name, float(err.max(initial=0)), tol)
    assert info == info_s
    assert info_x["dof"] == info["dof"] and info_x["unconstrained"] == info["unconstrained"]
    # fixed blocks are zero, free blocks symmetric positive definite
    assert not cam[:prob.m_con].any() and not pt[:prob.n_con].any()
    free = cam[prob.m_con:]
    assert np.allclose(free, free.transpose(0, 2, 1), rtol=0, atol=max(1e-12, tol) * np.abs(free).max(initial=0))
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


@pytest.mark.parametrize("name", sorted(cd.EDGE_ROWS) + sorted(cd.SINGULAR_EDGE_ROWS))
def test_edge_scenes_are_tie_free_and_on_their_path(name):
    """Every Tukey decision of an edge scene is at least 1e-6 relative away from max_err, and each scene has the
    structure that sends the device down the path it is there for."""
    prob, opt = cd.make_edge(name)
    assert cd.decision_margin(prob, opt.max_err) >= 1e-6
    _, w, unc = cd.weights(prob, opt.max_err)
    mf = prob.m - prob.m_con
    if name == "structure_only":
        assert mf == 0 and prob.n_con < prob.n
    if name == "motion_only":
        assert prob.n_con == prob.n and mf > 0
    if name in ("single_observation_points_fixed", "weight_dropped_points"):
        lone = np.nonzero(np.diff(prob.ptr) <= 2)[0][-10:]
        assert unc[lone].all() and prob.m_con >= 2
        if name == "weight_dropped_points":  # one observation of each beyond 3 max_err, the other kept
            e = np.sqrt((cd.residuals(prob) ** 2).sum(1))
            assert (e[prob.ptr[lone]] >= 3 * opt.max_err).all() and (cd.tukey_weights(e[prob.ptr[lone] + 1],
                                                                                    opt.max_err) > 0).all()
    if name == "one_long_pair_fixed":
        assert mf == 2 and prob.n == 532 and prob.n_con == 0
    if name == "points_fix_gauge":
        assert prob.m_con == 0 and prob.n_con >= 3
        X = prob.X[:prob.n_con]
        assert np.linalg.matrix_rank(X[1:] - X[0], tol=1e-3) >= 2  # not collinear
    if name == "many_points":
        assert 6 * prob.n > 1024 * 256  # more than one pass of ba_cov_begin's grid-stride clear


@pytest.mark.parametrize("name", sorted(cd.SINGULAR_EDGE_ROWS))
def test_group_with_a_blind_camera_is_singular(name):
    """A free camera that sees nothing: H fails Cholesky or has a relative pivot below the device's 1e-12."""
    prob, opt = cd.make_edge(name)
    assert (prob.cam != 1 + 10 * int(name[-1]) + 5).all()
    with pytest.raises(np.linalg.LinAlgError):  # H has six zero rows
        cd.cov_full(prob, opt.max_err, VAR)
    regular = cd.make_edge("groups_3x10")[0]
    assert cd.min_relative_pivot(cd.cov_full(regular, opt.max_err, VAR)[3]) > 1e-6


def test_single_observation_points_would_leak_into_U():
    """The scene can catch the bug it is there for: with the A^T A of the points left out of H added back into
    their free cameras' U, the camera blocks move by more than 1e-3."""
    prob, opt = cd.make_edge("single_observation_points_fixed")
    cam, _, _, H = cd.cov_full(prob, opt.max_err, VAR)
    e, w, unc = cd.weights(prob, opt.max_err)
    raw = cd.tukey_weights(np.sqrt((e * e).sum(1)), opt.max_err)
    pt_of = cd.point_of(prob)
    leak = np.nonzero(unc[pt_of] & (raw > 0) & (prob.cam >= prob.m_con))[0]
    assert len(leak) >= 5
    A = cd.omega_jacobian(prob)[:, :, :6] * np.sqrt(raw)[:, None, None]
    H2 = H.copy()
    for o in leak:
        c = 6 * (prob.cam[o] - prob.m_con) + np.arange(6)
        H2[np.ix_(c, c)] += A[o].T @ A[o]
    C2 = VAR * np.linalg.inv(H2)
    moved = [np.linalg.norm(C2[6 * j:6 * j + 6, 6 * j:6 * j + 6] - cam[prob.m_con + j]) / np.linalg.norm(cam[prob.m_con + j])
             for j in range(prob.m - prob.m_con)]
    assert max(moved) > 1e-3, moved


def test_structure_and_motion_only_blocks():
    """No free camera: every camera block is zero and a point's block is var V^-1.  Every point fixed: every point
    block is zero."""
    prob, opt = cd.make_edge("structure_only")
    cam, pt, info = cd.cov_schur(prob, opt.max_err, VAR)
    assert not cam.any() and info["dof"] > 0
    e, w, unc = cd.weights(prob, opt.max_err)
    B = cd.omega_jacobian(prob)[:, :, 6:] * np.sqrt(w)[:, None, None]
    V = np.zeros((prob.n, 3, 3))
    np.add.at(V, cd.point_of(prob), np.einsum("nia,nib->nab", B, B))
    live = (np.arange(prob.n) >= prob.n_con) & ~unc
    assert np.allclose(pt[live], VAR * np.linalg.inv(V[live]), rtol=1e-12, atol=0)
    prob, opt = cd.make_edge("motion_only")
    cam, pt, info = cd.cov_schur(prob, opt.max_err, VAR)
    assert not pt.any() and (np.linalg.eigvalsh(cam[prob.m_con:]) > 0).all()


def test_schur_reference_on_many_points():
    """cov_schur (pinned to cov_full on every smaller scene) at 50 000 points: SPD blocks, the NaN pattern of the
    points left out, dof."""
    prob, opt = cd.make_edge("many_points")
    cam, pt, info = cd.cov_schur(prob, opt.max_err, VAR)
    _, w, unc = cd.weights(prob, opt.max_err)
    assert (np.linalg.eigvalsh(cam[prob.m_con:]) > 0).all() and not cam[:prob.m_con].any()
    assert np.isnan(pt[unc]).all() and (np.linalg.eigvalsh(pt[~unc]) > 0).all()
    assert info["unconstrained"] == unc.sum() > 0
    assert info["dof"] == 2 * int((w > 0).sum()) - 6 * (prob.m - prob.m_con) - 3 * int((~unc).sum())


def test_banded_scene_is_dissected():
    prob = cd.banded()
    cam, pt, info, _ = cd.cov_full(prob, 0.0, 1.0)
    cam_s, pt_s, _ = cd.cov_schur(prob, 0.0, 1.0)
    assert prob.m - prob.m_con >= 40
    for a, b in ((cam_s, cam), (pt_s, pt)):
        err, same = cd.block_errors(a, b)
        assert same and err.max() < 1e-8
