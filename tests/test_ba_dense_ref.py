"""The dense float64 reference of one BA trial (tests/ba_dense.py), on the CPU, before any GPU test trusts it:
on every scene row one trial of the CPU oracle (oracle/ba_oracle.cpp, analytic Jacobian, Schur complement,
Cholesky) equals the dense step under check_trial's float64 bounds; the complex-step Jacobian blocks equal
the oracle's analytic A and B; the scene rows have the shapes they are named for; and the helpers that pack
cosl_sba_motstr_levmar_x's parameter block round-trip."""
import numpy as np
import pytest

import ba_dense as D
from coslam_b200.problem import BAProblem

ROWS = list(D.ROWS)


@pytest.mark.parametrize("name", ROWS)
def test_oracle_trial_equals_the_dense_step(orc, name):
    prob, opt = D.make(name)
    after = D.fresh(prob)
    info = orc.ba_run_fixed(after, opt, 1)
    r = D.check_trial(prob, info, after, opt)
    print(name, " ".join(f"{k} {v:.2e}" for k, v in r.items()))


@pytest.mark.parametrize("name", ROWS)
def test_complex_step_blocks_equal_the_oracle_jacobian(orc, name):
    """d xhat / d(v, t) and d xhat / dX of every observation, to 1e-12 relative plus the scene's cancellation
    bound rho (far_offset: the analytic blocks are formed from a cancelling R X + t)."""
    prob, _ = D.make(name)
    Jl = D.local_jacobian(prob)
    rho, _ = D.cancellation(prob)
    pt = D.point_of(prob)
    q0 = D.R_to_quat(prob.R)
    worst = 0.0
    for o in range(prob.nobs):
        j = prob.cam[o]
        xy, A, B = orc.ba_project(prob.K[j], q0[j], np.zeros(3), prob.t[j], prob.X[pt[o]])
        got = np.concatenate([A, B], 1)
        err = np.abs(got - Jl[o]).max() / np.abs(Jl[o]).max()
        assert err <= 1e-12 + 4 * rho[o], (o, err, rho[o])
        worst = max(worst, err)
    print(name, f"worst block error {worst:.2e}")


def test_K_is_read_whole():
    """The reference uses every entry of K: fx, fy, skew and the principal point move the projection."""
    prob, _ = D.make("rig_intrinsics")
    x0 = D.project(prob)[0]
    for k in (0, 1, 2, 4, 5):
        p = D.fresh(prob)
        p.K[:, k] += 1.0
        assert np.abs(D.project(p)[0] - x0).max() > 1e-3, k
    assert not np.shares_memory(p.K, prob.K)


def test_rows_have_their_shapes():
    prob, _ = D.make("rig_intrinsics")
    K = prob.K.reshape(-1, 3, 3)
    assert sorted(set(K[:, 0, 0])) == [350.0, 800.0, 1400.0]
    assert np.allclose(sorted(set(np.round(K[:, 1, 1] / K[:, 0, 0], 6))), [0.92, 1.0, 1.07])
    assert sorted(set(K[:, 0, 1])) == [-4.0, 0.0, 3.5]
    for j, (W, H) in enumerate(D.RIG_SIZES):
        assert K[j, 0, 2] != W / 2 and K[j, 1, 2] != H / 2
    assert prob.m == 12 and prob.m_con == 3
    _, P = D.project(D.make("wide_and_deep")[0])
    assert P[:, 2].min() < 0.35 and P[:, 2].max() > 600 and np.abs(P[:, 0] / P[:, 2]).max() > 1.8
    deep = D.make("wide_and_deep")[0]
    far = np.nonzero(deep.X[:, 2] > 600)[0]
    assert len(far)
    C = -np.einsum("jba,jb->ja", deep.R.reshape(-1, 3, 3), deep.t)  # camera centres
    base = np.linalg.norm(C[:, None] - C[None], axis=2).max()
    assert (np.degrees(base / deep.X[far, 2]) < 0.05).sum() >= 3  # parallax over the whole baseline
    assert np.abs(D.make("far_offset")[0].X).min(0).max() > 2e3
    rs = D.make("rotated_start")[0]
    ri = D.rig_intrinsics(seed=13, dR=0.0)
    q = D.R_to_quat(rs.R.reshape(-1, 3, 3)[3:] @ ri.R.reshape(-1, 3, 3)[3:].transpose(0, 2, 1))
    ang = np.degrees(2 * np.arcsin(np.linalg.norm(q[:, 1:], axis=1)))
    assert ang.min() > 2.9 and ang.max() < 8.1 and np.linalg.norm(q[:, 1:], axis=1).max() > 0.06


def test_long_track_runs_straddle_warps_and_blocks():
    """The runs of the 33-, 64- and 100-camera points cross warp (32) and 256-thread block boundaries of the
    point-major kernels, and the last camera's single observation opens a 128-thread block of the
    camera-major kernel."""
    prob, _ = D.make("long_tracks")
    k = np.diff(prob.ptr)
    assert sorted(k)[-3:] == sorted(D.LONG) and k.max() > 32
    starts, pos = D.long_track_layout(prob)
    assert starts[0] % 256 == 250 and starts[2] % 256 == 250 and starts[1] % 32 == 30
    for s, L in zip(starts, D.LONG):
        assert (s + L - 1) // 32 > s // 32  # crosses a warp
    assert (starts[0] + D.LONG[0] - 1) // 256 > starts[0] // 256
    assert (starts[2] + D.LONG[2] - 1) // 256 > starts[2] // 256
    assert len(pos) == 1 and pos[0] % 128 == 0 and pos[0] > 0
    assert np.all(prob.ptr[np.nonzero(k == D.LONG[2])[0][0]] >= 256)


def test_unobserved_and_unsorted_rows(orc):
    """Unobserved points: first fixed, first free, middle, last; they leave the oracle's cost and every other
    parameter alone and come back unchanged.  Unsorted observations: the oracle's answer is that of the
    sorted permutation."""
    prob, opt = D.make("unobserved_points")
    u = D.unobserved_indices(prob)
    assert u[0] == 0 and u[1] == prob.n_con and u[-1] == prob.n - 1 and len(u) == 4
    keep = np.setdiff1d(np.arange(prob.n), u)
    k = np.diff(prob.ptr)[keep]
    without = BAProblem(prob.K.copy(), prob.R, prob.t, prob.X[keep], np.concatenate([[0], np.cumsum(k)]),
                        prob.cam.copy(), prob.xy.copy(), prob.m_con, prob.n_con - 1)
    a, b = D.fresh(prob), D.fresh(without)
    ia, ib = orc.ba_run_fixed(a, opt, 4), orc.ba_run_fixed(b, opt, 4)
    assert ia[1] == ib[1] and np.array_equal(a.X[keep], b.X) and np.array_equal(a.R, b.R)
    assert np.array_equal(a.X[u], prob.X[u])

    prob, opt = D.make("unsorted_observations")
    srt, perm = D.sorted_permutation(prob)
    assert not np.array_equal(perm, np.arange(prob.nobs))
    a, b = D.fresh(prob), D.fresh(srt)
    ia, ib = orc.ba_run_fixed(a, opt, 4), orc.ba_run_fixed(b, opt, 4)
    assert abs(ia[1] - ib[1]) <= 1e-12 * ib[1]
    assert np.abs(a.X - b.X).max() < 1e-10 and np.abs(a.t - b.t).max() < 1e-10


def test_tukey_row_has_residuals_at_the_cut_off():
    prob, _ = D.make("tukey_mixed")
    e = np.sqrt((D.residuals(prob) ** 2).sum(1))
    near = np.abs(e / D.MAX_ERR - 1)
    assert ((near < 2e-9) & (e < D.MAX_ERR)).sum() >= 8 and ((near < 2e-9) & (e > D.MAX_ERR)).sum() >= 8
    assert 0.2 < (e >= D.MAX_ERR).mean() < 0.35


def test_sba_packing_round_trips():
    """pack_sba -> unpack_sba gives the problem back: K (ar fx to one rounding), R, t, X, observations."""
    prob, _ = D.make("rig_intrinsics")
    rng = np.random.default_rng(3)
    dq = rng.normal(size=(prob.m, 3)) * 0.05
    p, rot0, vmask = D.pack_sba(prob, dq)
    c = p[:11 * prob.m].reshape(prob.m, 11)
    assert np.array_equal(c[:, 5:8], dq) and np.any(c[:, 3] != 1.0) and np.any(c[:, 4] != 0.0)
    assert np.allclose(np.linalg.norm(rot0, axis=1), 1.0, rtol=0, atol=1e-15)
    back = D.unpack_sba(p, rot0, vmask, prob.xy, prob.m_con, prob.n_con)
    assert np.array_equal(back.K[:, [0, 1, 2, 5, 8]], prob.K[:, [0, 1, 2, 5, 8]])
    assert np.abs(back.K[:, 4] - prob.K[:, 4]).max() <= 2 * D.EPS * prob.K[:, 4].max()
    assert np.abs(back.R - prob.R).max() < 1e-15 * 8
    assert np.array_equal(back.t, prob.t) and np.array_equal(back.X, prob.X)
    assert np.array_equal(back.ptr, prob.ptr) and np.array_equal(back.cam, prob.cam)
