"""Bundle-adjustment problems at the edges of the device path, each built directly as a BAProblem:
motion only, structure only (no free camera: the ns == 0 update path), free cameras that see nothing
or only fixed points, points that only fixed cameras see, single-observation points, two camera
groups without a shared point (two uncoupled blocks of the one-CTA solve), and one camera pair whose
shared points fill several Schur work items.

Every scene is checked twice:
  - one LM trial of BaSolver.run_fixed(1) against a dense numpy step: (J^T W J + mu I) delta = J^T W e
    with mu = tau max diag(J^T W J), J by complex-step differentiation of the KRTS projection with
    the local-quaternion rotation update (exact to roundoff, also along the nearly free ray direction
    of a single-observation point);
  - four fixed trials against the CPU oracle: the same cost to 1e-9 relative."""
import ctypes as C

import numpy as np
import pytest

from coslam_b200.ctypes_defs import BaOptions
from coslam_b200.problem import BAProblem

pytestmark = pytest.mark.gpu

K0 = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
MAX_ERR = 6.0


def quat_to_R(w, x, y, z):
    """Rotation matrices of (possibly complex) unit quaternions, batched over the leading axis."""
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def state(base, p):
    """(R [m,3,3], t [m,3], X [n,3]) for parameters p = [free cameras (v, t) ..., free points X ...] on
    top of `base`; v is the vector part of the rotation update dq (R = R(dq) R0, w = sqrt(1 - |v|^2)).
    p may be complex (complex-step derivatives)."""
    mf, nf = base.m - base.m_con, base.n - base.n_con
    R = base.R.reshape(-1, 3, 3).astype(p.dtype)
    t = base.t.astype(p.dtype)
    X = base.X.astype(p.dtype)
    if mf:
        cams = p[:6 * mf].reshape(mf, 6)
        v = cams[:, :3]
        dR = quat_to_R(np.sqrt(1.0 - (v * v).sum(1)), v[:, 0], v[:, 1], v[:, 2])
        R[base.m_con:] = dR @ R[base.m_con:]
        t[base.m_con:] = cams[:, 3:]
    X[base.n_con:] = p[6 * mf:].reshape(nf, 3)
    return R, t, X


def residuals(base, p):
    """x - xhat [nobs, 2] at parameters p"""
    R, t, X = state(base, p)
    pt = np.repeat(np.arange(base.n), np.diff(base.ptr))
    Pc = np.einsum("nij,nj->ni", R[base.cam], X[pt]) + t[base.cam]
    u = np.einsum("nij,nj->ni", base.K.reshape(-1, 3, 3)[base.cam], Pc)
    return base.xy - u[:, :2] / u[:, 2:3]


def pack(base):
    mf = base.m - base.m_con
    cams = np.zeros((mf, 6))
    cams[:, 3:] = base.t[base.m_con:]
    return np.concatenate([cams.ravel(), base.X[base.n_con:].ravel()])


def tukey_sqrt_weights(base, max_err):
    """sqrt of the robust weights frozen at the start of a round, per residual component"""
    if max_err <= 0:
        return np.ones(2 * base.nobs)
    r = residuals(base, pack(base))
    en = np.sqrt((r * r).sum(1)) / max_err
    return np.sqrt(np.where(en < 1.0, (1 - en * en) ** 2, 0.0)).repeat(2)


def dense_step(base, opt):
    """The first LM trial in dense form: (state after the step, its weighted cost, the start cost)."""
    sw = tukey_sqrt_weights(base, opt.max_err)
    eps = lambda p: residuals(base, p).ravel() * sw
    p0 = pack(base)
    e0 = eps(p0)
    h = 1e-20
    J = np.empty((e0.size, p0.size))  # d xhat / d p = -d eps / d p
    for k in range(p0.size):
        d = p0.astype(np.complex128)
        d[k] += 1j * h
        J[:, k] = -eps(d).imag / h
    JtJ = J.T @ J
    mu = opt.opts[0] * JtJ.diagonal().max()
    delta = np.linalg.solve(JtJ + mu * np.eye(p0.size), J.T @ e0)
    return state(base, p0 + delta), float((eps(p0 + delta) ** 2).sum()), float((e0 ** 2).sum())


# ---------------------------------------------------------------- scenes
def scene(vis, m, m_con, n_con, seed):
    """Cameras 0.25 apart along x (camera 0: R = I, t = 0), points 4-7 in front of them, observations =
    projections + 0.3 px noise; free cameras and points start slightly off.  vis[i] = cameras that see
    point i."""
    rng = np.random.default_rng(seed)
    n = len(vis)
    R = np.empty((m, 3, 3))
    t = np.empty((m, 3))
    for j in range(m):
        v = np.zeros(3) if j == 0 else rng.normal(size=3) * 0.03
        R[j] = quat_to_R(np.sqrt(1 - v @ v), *v)
        t[j] = -R[j] @ np.array([0.25 * j, 0.1 * (j % 2), 0.0])
    X = np.column_stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.0, 1.0, n), rng.uniform(4.0, 7.0, n)])
    X[0] = [0.0, 0.0, 5.0]  # straight ahead of camera 0
    cam = np.concatenate([np.asarray(sorted(v), np.int32) for v in vis])
    ptr = np.concatenate([[0], np.cumsum([len(v) for v in vis])]).astype(np.int64)
    truth = BAProblem(np.tile(K0.ravel(), (m, 1)), R, t, X, ptr, cam, np.zeros((len(cam), 2)), m_con, n_con)
    truth.xy[:] = truth.xy - residuals(truth, pack(truth)) + rng.normal(0, 0.3, (len(cam), 2))
    prob = truth.copy()
    for j in range(m_con, m):
        v = rng.normal(size=3) * 0.002
        prob.R[j] = (quat_to_R(np.sqrt(1 - v @ v), *v) @ R[j]).ravel()
        prob.t[j] += rng.normal(0, 0.01, 3)
    prob.X[n_con:] += rng.normal(0, 0.02, (n - n_con, 3))
    return prob


def random_vis(rng, n, cams, kmin=2, kmax=4):
    cams = np.asarray(cams)
    return [list(rng.choice(cams, size=int(rng.integers(kmin, min(kmax, len(cams)) + 1)), replace=False))
            for _ in range(n)]


def make(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "motion_only":  # n_con == n
        return scene(random_vis(rng, 60, range(6), 3, 5), 6, 1, 60, 1)
    if name == "structure_only":  # m_con == m: no reduced system
        return scene(random_vis(rng, 60, range(5)), 5, 5, 5, 2)
    if name == "free_camera_sees_nothing":
        return scene(random_vis(rng, 60, range(5)), 6, 1, 3, 3)
    if name == "free_camera_sees_only_fixed_points":
        vis = [v + [5] if 5 not in v else v for v in random_vis(rng, 15, range(6))]
        return scene(vis + random_vis(rng, 45, range(5)), 6, 1, 15, 4)
    if name == "points_seen_only_by_fixed_cameras":
        return scene(random_vis(rng, 50, range(6)) + [[0, 1]] * 10, 6, 2, 0, 5)
    if name == "single_observation_points":
        return scene(random_vis(rng, 50, range(6)) + [[1 + k % 5] for k in range(10)], 6, 1, 0, 6)
    if name.startswith("two_groups_"):  # camera 0 fixed, free groups 1..g and g+1..2g share no point
        g = int(name.rsplit("_", 1)[1])
        va = [v + [0] if k % 3 == 0 else v for k, v in enumerate(random_vis(rng, 6 * g, range(1, g + 1), 2, 5))]
        vb = [v + [0] if k % 3 == 0 else v for k, v in enumerate(random_vis(rng, 6 * g, range(g + 1, 2 * g + 1), 2, 5))]
        return scene(va + vb, 2 * g + 1, 1, 0, 7)
    if name == "one_long_pair":  # 532 = 4 x 128 + 20 shared free points of the two free cameras
        return scene([[0, 1, 2]] * 532, 3, 1, 0, 8)
    raise KeyError(name)


SCENES = ["motion_only", "structure_only", "free_camera_sees_nothing", "free_camera_sees_only_fixed_points",
          "points_seen_only_by_fixed_cameras", "single_observation_points", "two_groups_6", "two_groups_10",
          "one_long_pair"]


def options():
    opt = BaOptions.defaults()
    opt.max_err = MAX_ERR
    return opt


def check_step(api, prob, opt):
    (R, t, X), cost_want, cost0 = dense_step(prob, opt)
    assert cost_want < cost0  # the first trial is a descent step
    s = api.BaSolver(prob.copy(), opt)
    info = s.run_fixed(1)
    got = s.download()
    s.close()
    assert int(info[9]) == 1
    assert abs(info[0] - cost0) <= 1e-9 * cost0
    assert abs(info[1] - cost_want) <= 1e-6 * cost_want, (info[1], cost_want)
    assert np.abs(got.X - X).max() < 1e-6
    assert np.abs(got.t - t).max() < 1e-6
    assert np.abs(got.R - R.reshape(-1, 9)).max() < 1e-7


def check_oracle(api, orc, prob, opt, trials=4):
    pg, po = prob.copy(), prob.copy()
    s = api.BaSolver(pg, opt)
    ig = s.run_fixed(trials)
    s.download()
    plan, stats = s.plan_info(), s.stats()
    s.close()
    io = orc.ba_run_fixed(po, opt, trials)
    assert ig[9] == io[9] == trials
    assert abs(ig[1] - io[1]) <= 1e-9 * io[1], (ig[1], io[1])
    assert np.abs(pg.X - po.X).max() < 1e-6 and np.abs(pg.t - po.t).max() < 1e-6
    # fixed cameras and points are left alone
    assert np.array_equal(pg.R[:prob.m_con], prob.R[:prob.m_con]) and np.array_equal(pg.X[:prob.n_con], prob.X[:prob.n_con])
    return plan, stats, pg, po


@pytest.mark.parametrize("name", SCENES)
def test_one_trial_equals_dense_step(api, name):
    check_step(api, make(name), options())


@pytest.mark.parametrize("name", SCENES)
def test_four_trials_match_the_oracle(api, orc, name):
    prob = make(name)
    plan, stats, _, _ = check_oracle(api, orc, prob, options())
    mf = prob.m - prob.m_con
    assert stats["ns"] == 6 * mf
    if name.startswith("two_groups_"):
        # the groups fall on split_blocks' cut: two blocks without a coupling tile, one CTA
        assert plan["blocks"] == 2 and plan["small_solve"] == 1 and plan["tiles"] == 2
    if name == "one_long_pair":
        # buckets (0,0), (0,1), (1,1) of 532 entries each, cut into items of <= 128 entries
        assert stats["pair_entries"] == 3 * 532 and stats["pair_items"] == 3 * 5


def test_observation_exactly_at_max_err_has_weight_zero(api, orc):
    """Camera 0 (fixed, R = I, t = 0) sees the fixed point 0 at (0, 0, 5) exactly max_err = 6 px off, at
    every iteration: its Tukey weight is 0 on the device as in the dense step and the oracle (the costs
    would differ by 36 otherwise), and both flag it an outlier."""
    rng = np.random.default_rng(9)
    vis = [[0, 1, 2, 3]] + random_vis(rng, 59, range(6))
    prob = scene(vis, 6, 1, 1, 9)
    prob.xy[0] = [326.0, 240.0]  # observation 0 = (point 0, camera 0)
    r = residuals(prob, pack(prob))
    assert np.sqrt((r[0] ** 2).sum()) == MAX_ERR and tukey_sqrt_weights(prob, MAX_ERR)[0] == 0.0
    check_step(api, prob, options())
    check_oracle(api, orc, prob, options())
    opt = options()
    opt.outer_iters, opt.inner_iters = 2, 3
    pg, po = prob.copy(), prob.copy()
    ig = api.ba_solve(pg, opt)
    io = orc.ba_solve(po, opt)
    assert pg.outlier[0] == po.outlier[0] == 1
    assert np.array_equal(pg.outlier, po.outlier) and ig[13] == io[13]


def duplicate_problem():
    """Point 3 observed twice by free camera 2."""
    rng = np.random.default_rng(12)
    vis = random_vis(rng, 40, range(5))
    vis[3] = [1, 2, 2]
    return scene(vis, 5, 1, 0, 12)


def test_duplicate_observation_is_refused(api, orc):
    """The Schur contraction keeps one entry per camera pair of a point; a repeated (point, camera)
    pair would lose half of W_b V^-1 W_a^T and count W_a V^-1 e twice, so it is refused on both sides."""
    prob = duplicate_problem()
    with pytest.raises(api.CoslError, match="twice"):
        api.BaSolver(prob, options())
    with pytest.raises(api.CoslError, match="twice"):
        api.ba_solve(prob.copy(), options())
    s = prob.struct()
    info = np.zeros(16)
    assert orc.lib().orc_ba_run_fixed(C.byref(s), C.byref(options()), 1, info.ctypes.data_as(C.c_void_p)) == -1
