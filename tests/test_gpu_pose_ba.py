"""CUDA pose / bundle-adjustment paths vs the CPU oracle, through the C-ABI (needs a GPU)."""
import numpy as np
import pytest

from coslam_b200 import synth
from coslam_b200.ctypes_defs import BaOptions, PoseOpt

pytestmark = pytest.mark.gpu

REL_RMS_TOL = 1e-4  # north_star: within 1e-4 relative reprojection RMS of the reference path


@pytest.mark.parametrize("seed,n", [(1, 192), (2, 64), (3, 7)])
def test_pose_parity(api, orc, seed, n):
    K, R0, t0, Ms, ms, Rt, tt = synth.make_pose_case(n_pts=n, seed=seed)
    ok_o, R_o, t_o, op_o = orc.pose_intracam(K, R0, t0, Ms, ms, 10.0)
    ok_g, R_g, t_g, op_g = api.pose_intracam(K, R0, t0, Ms, ms, 10.0)
    assert ok_o == ok_g
    assert np.abs(R_o - R_g).max() < 1e-8 and np.abs(t_o - t_g).max() < 1e-8
    assert op_o.nIterRW == op_g.nIterRW
    assert abs(op_o.err - op_g.err) <= 1e-6 * max(1.0, abs(op_o.err))


def test_pose_prev_errs_and_batch(api, orc):
    cases = [synth.make_pose_case(n_pts=n, seed=10 + i) for i, n in enumerate((192, 150, 33, 192))]
    rng = np.random.default_rng(0)
    prev = [np.abs(rng.normal(0, 4, len(c[3]))) for c in cases]
    prev[2] = None
    ok, R, t, opts = api.pose_intracam_batch([c[0] for c in cases], [c[1] for c in cases],
                                             [c[2] for c in cases], [c[3] for c in cases],
                                             [c[4] for c in cases], 10.0, prev)
    for i, c in enumerate(cases):
        ok_o, R_o, t_o, op_o = orc.pose_intracam(c[0], c[1], c[2], c[3], c[4], 10.0, prev[i])
        assert ok_o == ok[i]
        assert np.abs(R_o - R[i]).max() < 1e-8 and np.abs(t_o - t[i]).max() < 1e-8


def _ba_compare(api, orc, prob, opt, tol=REL_RMS_TOL):
    pg, po = prob.copy(), prob.copy()
    info_g = api.ba_solve(pg, opt)
    info_o = orc.ba_solve(po, opt)
    rms_g, rms_o = pg.rms(), po.rms()
    assert abs(rms_g - rms_o) <= tol * rms_o, (rms_g, rms_o)
    assert abs(info_g[1] - info_o[1]) <= 1e-6 * info_o[1] + 1e-9, (info_g[:10], info_o[:10])
    assert np.abs(pg.R - po.R).max() < 1e-6 and np.abs(pg.t - po.t).max() < 1e-6
    assert np.abs(pg.X - po.X).max() < 1e-5
    return pg, po, info_g, info_o


@pytest.mark.parametrize("robust", [True, False])
def test_ba_local_parity_c2(api, orc, robust):
    """BASELINE c2: 2 cams x 5 key frames, 5 k points, oldest 2 key frames fixed, 2 fixed points."""
    prob, truth = synth.make_ba_scene(2, 5, 5000, 640, 480, seed=7, m_con=4, n_con=2)
    opt = BaOptions.defaults()
    opt.outer_iters, opt.inner_iters = 2, 10
    if not robust:
        opt.max_err = 0.0
    pg, po, ig, io = _ba_compare(api, orc, prob, opt)
    assert ig[10] == io[10]  # same number of LM trials
    # fixed cameras / points untouched
    assert np.array_equal(pg.R[:4], prob.R[:4]) and np.array_equal(pg.X[:2], prob.X[:2])
    if robust:
        assert np.array_equal(pg.outlier, po.outlier)
        assert pg.rms(~truth["is_outlier"]) < 0.8


def test_ba_intercam_pattern(api, orc):
    """InterCamPoseEstimator pattern (app/SL_InterCamPoseEstimator.cpp:95): all cameras free,
    first nPtsCon points fixed."""
    prob, truth = synth.make_ba_scene(4, 1, 400, 640, 480, seed=9, m_con=0, n_con=340, window=0,
                                      p_vis=1.0)
    opt = BaOptions.defaults()
    opt.max_err, opt.outer_iters, opt.inner_iters = 6.0, 3, 40
    _ba_compare(api, orc, prob, opt)


def test_ba_large_reduced_system(api, orc):
    """Reduced system larger than one CTA's shared memory -> blocked Cholesky path."""
    prob, truth = synth.make_ba_scene(4, 12, 3000, 640, 480, seed=5, m_con=4, n_con=0,
                                      outlier_frac=0.0)
    assert 6 * (prob.m - prob.m_con) > 200
    opt = BaOptions.defaults()
    opt.max_err, opt.outer_iters, opt.inner_iters = 0.0, 1, 6
    _ba_compare(api, orc, prob, opt)


def test_ba_c3_properties(api):
    """BASELINE c3 local BA at full size: cost decreases monotonically over accepted steps,
    constrained parameters stay put, inlier RMS reaches the noise floor."""
    prob, truth = synth.make_ba_scene(4, 5, 20000, 1280, 720, seed=3, m_con=8, n_con=2)
    opt = BaOptions.defaults()
    opt.outer_iters, opt.inner_iters = 2, 10
    p = prob.copy()
    info = api.ba_solve(p, opt)
    assert info[1] < info[0]
    assert np.array_equal(p.R[:8], prob.R[:8]) and np.array_equal(p.t[:8], prob.t[:8])
    assert np.array_equal(p.X[:2], prob.X[:2])
    # observations that start beyond the Tukey cut-off keep weight 0 (a point whose observations all
    # do never moves) -- judge the fit on what the solver itself kept
    kept = ~p.outlier.astype(bool)
    assert p.rms(kept) < 0.8
    assert (p.outlier.astype(bool) & truth["is_outlier"]).sum() > 0.95 * truth["is_outlier"].sum()
    # info[13] is counted on the device by the solver handle as well (not only patched by cosl_ba_solve)
    s = api.BaSolver(prob.copy(), opt)
    info_s = s.run()
    ps = s.download()
    assert info_s[13] == ps.outlier.sum() > 0
    s.close()


def test_sba_signature_wrapper(api, orc):
    """cosl_sba_motstr_levmar_x with BundleRTS packing (app/SL_CoSLAMBA.cpp:337-356)."""
    import ctypes as C
    prob, truth = synth.make_ba_scene(2, 4, 300, 640, 480, seed=4, m_con=2, n_con=1,
                                      outlier_frac=0.0)
    m, n = prob.m, prob.n

    def pack():
        p = np.zeros(m * 11 + n * 3)
        rot0 = np.zeros((m, 4))
        for j in range(m):
            K = prob.K[j]
            p[11 * j:11 * j + 5] = [K[0], K[2], K[5], K[4] / K[0], K[1]]
            p[11 * j + 8:11 * j + 11] = prob.t[j]
            rot0[j] = orc.mat2quat(prob.R[j].reshape(3, 3))
        p[m * 11:] = prob.X.ravel()
        return p, rot0

    vmask = np.zeros((n, m), np.int8)
    pt = np.repeat(np.arange(n), np.diff(prob.ptr))
    vmask[pt, prob.cam] = 1
    opts = np.array([1e-7, 1e-12, 1e-12, 0, 1e-16])
    pg, rot0 = pack()
    po, _ = pack()
    ig, io = np.zeros(10), np.zeros(10)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rg = api.LIB.cosl_sba_motstr_levmar_x(n, 1, m, 2, vp(vmask), vp(pg), 11, 3, vp(prob.xy), 2,
                                          vp(rot0), 20, 0, vp(opts), vp(ig), 0)
    ro = orc.lib().orc_sba_motstr_levmar_x(n, 1, m, 2, vp(vmask), vp(po), 11, 3, vp(prob.xy), 2,
                                           vp(rot0), 20, 0, vp(opts), vp(io))
    # iteration counts may differ slightly at the eps2 = 1e-12 stop test (fp64 sums are reduced in a
    # different -- and, through the atomics of the contraction, run-dependent -- order on the GPU);
    # the converged result must agree
    assert rg >= 0 and abs(rg - ro) <= 2
    assert abs(ig[1] - io[1]) <= 1e-6 * io[1]
    assert np.abs(pg - po).max() < 1e-6
    assert ig[1] < ig[0]


def test_ba_dense_covisibility_blocked_path(api, orc):
    """All cameras see all points -> full envelope: the skyline factorisation degenerates to the
    plain dense blocked Cholesky (reduced system 174 x 174 > one CTA's shared memory)."""
    prob, truth = synth.make_ba_scene(30, 1, 600, 640, 480, seed=15, m_con=1, n_con=0, window=0,
                                      p_vis=0.9, outlier_frac=0.0)
    assert 6 * (prob.m - prob.m_con) == 174
    opt = BaOptions.defaults()
    opt.max_err, opt.outer_iters, opt.inner_iters = 0.0, 1, 8
    _ba_compare(api, orc, prob, opt)


def test_ba_c4_slice_parity(api, orc):
    """A 40-key-frame slice of the c4 scene (banded co-visibility, reduced system 936 x 936):
    fixed number of LM trials -> identical cost trajectory as the oracle."""
    prob, truth = synth.make_ba_scene(4, 40, 6000, 1280, 720, seed=16, m_con=4, n_con=0)
    opt = BaOptions.defaults()
    pg, po = prob.copy(), prob.copy()
    s = api.BaSolver(pg, opt)
    ig = s.run_fixed(4)
    s.download()
    io = orc.ba_run_fixed(po, opt, 4)
    assert ig[9] == io[9] == 4
    assert abs(ig[1] - io[1]) <= 1e-9 * io[1], (ig[1], io[1])
    assert abs(pg.rms() - po.rms()) <= REL_RMS_TOL * po.rms()
    assert np.abs(pg.X - po.X).max() < 1e-6


def test_ba_robust_two_rounds_fixed_point_parity(api, orc):
    """12 key frames, one fixed point, two robust rounds: same solution as the oracle."""
    prob, truth = synth.make_ba_scene(4, 12, 2500, 1280, 720, seed=33, m_con=4, n_con=1)
    opt = BaOptions.defaults()
    opt.outer_iters, opt.inner_iters = 2, 6
    _ba_compare(api, orc, prob, opt)


def test_ba_time_ordered_points_two_solvers_agree(api, orc):
    """Points sorted by home key frame (map-creation order, ADVICE r1): same solution as the oracle
    -- the single-GPU counterpart of the sharded test in tools/mgpu_ba_check.py."""
    prob, truth = synth.make_ba_scene(4, 20, 3000, 1280, 720, seed=34, m_con=4, n_con=0, sort_by_home=True)
    opt = BaOptions.defaults()
    opt.outer_iters, opt.inner_iters = 2, 6
    _ba_compare(api, orc, prob, opt)
