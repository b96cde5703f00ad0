"""PnP RANSAC on the pose solver handle (cosl_pose_solver_set_ransac, DESIGN.md 5.7): parity with the float64
restatement of tests/pnp_dense.py at the initialisation shapes, bit-identity where RANSAC keeps R0 and when disarmed,
recovery from a poor start through the real handle, every status, the refusals and the state rules."""
import numpy as np
import pytest

import pnp_dense as pn
from pnp_dense import MC_ANGLE_DEG, MC_CENTRE_REL

pytestmark = pytest.mark.gpu

TAU = 10.0
THR = 2.0
REL = 1e-9


def _cams(seed, counts, out_frac=0.4, rot_deg=30.0):
    rng = np.random.default_rng(seed)
    return [pn.scene(rng, n, out_frac, rot_deg) for n in counts]


def _submit(s, cams, **kw):
    s.submit([c[0] for c in cams], [c[1] for c in cams], [c[2] for c in cams], [c[3] for c in cams],
             [c[4] for c in cams], TAU, **kw)
    return s.collect()


def _bits(*arrs):
    return [np.ascontiguousarray(a).view(np.uint8).tobytes() for a in arrs]


def _collected(res):
    ok, R, t, opts, _ = res
    return _bits(ok, R, t) + [bytes(opts)]


@pytest.mark.parametrize("C,n", [(4, 192), (13, 1000), (12, 600)])
def test_parity_with_restatement(api, C, n):
    nh, seed, min_inl = 2000, 0x5EED0000 + C, 6
    counts = [n - 37 * (c % 3) for c in range(C)]
    cams = _cams(C * 1000 + n, counts)
    use = np.ones(C, bool)
    use[C - 1] = False  # one camera not selected
    s = api.PoseSolver(0, C, sum(counts))
    s.set_ransac(use, nh, THR, min_inl, seed)
    _submit(s, cams)
    got = s.download_ransac()
    hy = s.download_ransac_hyps()
    assert hy["idx"].shape == (C, nh, 5)
    for c, (K, R0, t0, M, m, _, _, _) in enumerate(cams):
        ref = pn.ransac_camera(K, R0, t0, M, m, c, use[c], nh, THR, min_inl, seed)
        assert got["status"][c] == ref["status"], c
        assert got["h"][c] == ref["h"], c
        if not use[c]:
            continue
        assert np.array_equal(hy["idx"][c], ref["idx"]), c
        ok = hy["inliers"][c] >= 0
        assert np.array_equal(ok, ref["ok"]), c
        # inlier counts identical except for points within 1e-9 of the threshold (at the restatement's pose)
        dif = np.nonzero(hy["inliers"][c] != ref["cnt"])[0]
        for h in dif:
            u, v, _ = pn.project(K, ref["hR"][h][None], ref["ht"][h][None], M[None])
            e = np.hypot(m[:, 0] - u[0], m[:, 1] - v[0])
            assert abs(int(hy["inliers"][c][h]) - int(ref["cnt"][h])) <= int((np.abs(e - THR) < 1e-9).sum()), (c, h)
        assert len(dif) <= 2, (c, dif)
        scale = max(1.0, np.abs(ref["t"]).max())
        assert np.abs(got["R"][c] - ref["R"]).max() <= REL
        assert np.abs(got["t"][c] - ref["t"]).max() <= REL * scale
        assert got["inliers"][c] == ref["inliers"]
        assert np.array_equal(got["inl"][c], ref["flags"])
    assert (got["status"][:C - 1] == pn.REPLACED).all()
    s.close()


def _within(R, t, Rt, tt, M):
    depth = np.mean((M @ Rt.T + tt)[:, 2])
    ang, dc = pn.pose_error(R, t, Rt, tt)
    return ang < MC_ANGLE_DEG and dc < MC_CENTRE_REL * depth


def test_recovery_in_one_submit(api):
    """R0 120 degrees off and a camera centre one mean depth away, 10 % gross outliers: the armed submit returns the
    true pose within the Monte-Carlo bounds for every camera, the unarmed one for at most one of them (the float64
    restatement's count)."""
    C = 6
    rng = np.random.default_rng(79)
    cams = [pn.scene(rng, 300, 0.1, 120.0, shift=1.0) for _ in range(C)]
    s = api.PoseSolver(0, C, 300 * C)
    ok0, R0s, t0s, _, _ = _submit(s, cams)
    s.set_ransac(np.ones(C, bool), 500, THR, 6, 3)
    ok1, R1, t1, _, _ = _submit(s, cams)
    st = s.download_ransac()
    assert (st["status"] == pn.REPLACED).all()
    unarmed = 0
    for c, (_, _, _, M, _, Rt, tt, _) in enumerate(cams):
        assert ok1[c] and _within(R1[c], t1[c], Rt, tt, M), c
        unarmed += bool(ok0[c]) and _within(R0s[c], t0s[c], Rt, tt, M)
    assert unarmed <= 1
    s.close()


def test_recovery_through_the_handle(api):
    """R0 30 degrees off, 40 % gross outliers.  RANSAC's start is within the Monte-Carlo bounds for every camera and
    the solve runs unchanged from it.  Without prevErrs that solve is led by the outliers from any start, so the
    second submit of the recipe (prevErrs from the start's inlier flags, pnp_dense.prev_errs) returns the true pose
    within the bounds, where the unarmed submit does not."""
    C = 6
    cams = _cams(77, [300] * C, out_frac=0.4, rot_deg=30.0)
    s = api.PoseSolver(0, C, 300 * C)
    ok0, R0s, t0s, _, _ = _submit(s, cams)
    s.set_ransac(np.ones(C, bool), 500, THR, 6, 3)
    ok1, R1, t1, _, _ = _submit(s, cams)
    st = s.download_ransac()
    unarmed = 0
    for c, (_, _, _, M, _, Rt, tt, _) in enumerate(cams):
        assert st["status"][c] == pn.REPLACED and _within(st["R"][c], st["t"][c], Rt, tt, M), c
        unarmed += bool(ok0[c]) and _within(R0s[c], t0s[c], Rt, tt, M)
    assert unarmed <= 1  # 1 of these 6 (the float64 restatement's count)
    # the solve ran unchanged from that start: an unarmed handle started there computes the same bits
    u = api.PoseSolver(0, C, 300 * C)
    started = [(c[0], st["R"][i], st["t"][i]) + c[3:] for i, c in enumerate(cams)]
    assert _bits(ok1, R1, t1) == _bits(*_submit(u, started)[:3])
    u.close()
    # the recipe's second submit, still armed: R0 wins now (status 4) and the prevErrs keep the solve there
    prev = [pn.prev_errs(f) for f in st["inl"]]
    ok2, R2, t2, _, _ = _submit(s, started, prev_list=prev)
    assert (s.download_ransac()["status"] == pn.KEPT).all()
    for c, (_, _, _, M, _, Rt, tt, _) in enumerate(cams):
        assert ok2[c] and _within(R2[c], t2[c], Rt, tt, M), c
    # the same with priors and map points: the RANSAC stage does not read them, and the solve starts from its pose
    s.set_covariance(1.0)
    s.reserve_mappts(64)
    rng = np.random.default_rng(5)
    prior = [(Rt, tt, np.diag([1e-2] * 3 + [1.0] * 3)) for (_, _, _, _, _, Rt, tt, _) in cams]
    mp = []
    for (K, _, _, _, _, Rt, tt, _) in cams:
        X = pn.scene(rng, 8, 0.0, 0.0)[3]
        uu, vv, _ = pn.project(K, Rt[None], tt[None], X[None])
        mp.append((X, np.array([np.eye(3) * 1e-3] * 8), np.stack([uu[0], vv[0]], 1)))
    ok3, R3, t3, _, _ = _submit(s, cams, prior=prior, mappts=mp, gate=5.99)
    st3 = s.download_ransac()
    assert _bits(st["R"], st["t"], st["status"], st["sse"]) == _bits(st3["R"], st3["t"], st3["status"], st3["sse"])
    ok4, R4, t4, _, _ = _submit(s, started, prior=prior, mappts=mp, gate=5.99, prev_list=prev)
    for c, (_, _, _, M, _, Rt, tt, _) in enumerate(cams):
        assert ok4[c] and _within(R4[c], t4[c], Rt, tt, M), c
    s.set_ransac(None, 0, 0)
    ok5, R5, t5, _, _ = _submit(s, started, prior=prior, mappts=mp, gate=5.99)
    assert _bits(ok3, R3, t3) == _bits(ok5, R5, t5)
    s.close()


def test_hypotheses_download_is_bounded(api):
    """The diagnostics always describe the last submit: a later, smaller set_ransac does not change their shape, a
    buffer smaller than the submit's hypothesis count is refused before anything is written, and a larger one takes
    the hypotheses at its own stride."""
    import ctypes as C_

    C, n = 2, 120
    cams = _cams(31, [n] * C)
    s = api.PoseSolver(0, C, C * n)
    s.set_ransac(np.ones(C, bool), 300, THR, 6, 7)
    _submit(s, cams)
    full = s.download_ransac_hyps()
    s.set_ransac(np.ones(C, bool), 64, THR, 6, 7)  # no reallocation: the buffers still hold the 300
    again = s.download_ransac_hyps()
    assert again["idx"].shape == (C, 300, 5) and all(np.array_equal(full[k], again[k]) for k in full)
    small = np.full((C, 64, 5), -7, np.int32)
    nh = C_.c_int(0)
    assert api.LIB.cosl_pose_solver_download_ransac_hyps(s.h, 64, C_.byref(nh), small.ctypes.data, None, None,
                                                         None) == -1
    assert nh.value == 300 and (small == -7).all()
    big = np.full((C, 400), -7, np.int32)
    assert api.LIB.cosl_pose_solver_download_ransac_hyps(s.h, 400, None, None, None, big.ctypes.data, None) == 0
    assert np.array_equal(big[:, :300], full["inliers"]) and (big[:, 300:] == -7).all()
    s.set_ransac(np.ones(C, bool), 500, THR, 6, 7)  # reallocates: the last submit's hypotheses are gone
    with pytest.raises(api.CoslError, match="error -6"):
        s.download_ransac_hyps()
    s.close()


def _kept_cams(seed, C, n):
    """Cameras whose R0 is the true pose with noise-free inliers and 40 % outliers: R0 wins"""
    rng = np.random.default_rng(seed)
    cams = []
    for _ in range(C):
        K, _, _, M, m, Rt, tt, out = pn.scene(rng, n, 0.4, 0.0, noise=0.0)
        cams.append((K, Rt, tt, M, m, Rt, tt, out))
    return cams


def test_bit_identity_when_r0_is_kept(api):
    C, n = 4, 192
    cams = _kept_cams(11, C, n)
    a = api.PoseSolver(0, C, C * n)
    b = api.PoseSolver(0, C, C * n)
    for s in (a, b):
        s.set_covariance(1.0)
        s.reserve_mappts(16)
    a.set_ransac(np.ones(C, bool), 256, THR, 6, 9)
    mp = [(c[3][:4], np.array([np.eye(3) * 1e-3] * 4), c[4][:4]) for c in cams]
    ra = _submit(a, cams, mappts=mp, gate=5.99)
    st = a.download_ransac()
    assert (st["status"] == pn.KEPT).all() and (st["h"] == -1).all()
    rb = _submit(b, cams, mappts=mp, gate=5.99)
    assert _collected(ra) == _collected(rb)
    assert _bits(*a.download_covariance()[::2]) == _bits(*b.download_covariance()[::2])
    ma, mb = a.download_mappts(), b.download_mappts()
    assert all(_bits(ma[k]) == _bits(mb[k]) for k in ma)
    a.close()
    b.close()


def test_disarmed_is_never_armed_and_armed_repeats(api):
    C, n = 3, 250
    cams = _cams(21, [n] * C)
    a = api.PoseSolver(0, C, C * n)
    b = api.PoseSolver(0, C, C * n)
    a.set_ransac(np.ones(C, bool), 300, THR, 6, 1)
    r1 = _submit(a, cams)
    d1 = a.download_ransac()
    r2 = _submit(a, cams)
    d2 = a.download_ransac()
    assert _collected(r1) == _collected(r2)
    assert _bits(d1["R"], d1["t"], d1["sse"], *d1["inl"]) == _bits(d2["R"], d2["t"], d2["sse"], *d2["inl"])
    a.set_ransac(None, 0, 0)
    assert _collected(_submit(a, cams)) == _collected(_submit(b, cams))
    with pytest.raises(api.CoslError, match="error -6: .*did not run RANSAC"):
        a.download_ransac()
    a.close()
    b.close()


def _status_cams(seed):
    rng = np.random.default_rng(seed)
    good = pn.scene(rng, 200, 0.3, 30.0)
    few = pn.scene(rng, 4, 0.0, 30.0)
    K, R0, t0, M, m, Rt, tt, out = pn.scene(rng, 120, 0.0, 30.0)
    line = np.linspace(0, 1, 120)[:, None] * np.array([1.0, 0.5, 0.2]) + M[0]  # collinear scene
    u, v, _ = pn.project(K, Rt[None], tt[None], line[None])
    col = (K, R0, t0, line, np.stack([u[0], v[0]], 1), Rt, tt, out)
    junk = pn.scene(rng, 120, 1.0, 30.0)  # all outliers
    unsel = pn.scene(rng, 50, 0.3, 30.0)
    return [good, few, col, junk, unsel]


def test_every_status(api):
    cams = _status_cams(3)
    use = np.array([1, 1, 1, 1, 0], bool)
    nh, min_inl, seed = 400, 40, 4
    s = api.PoseSolver(0, len(cams), sum(len(c[3]) for c in cams))
    s.set_ransac(use, nh, THR, min_inl, seed)
    _submit(s, cams)
    got = s.download_ransac()
    want = [pn.ransac_camera(c[0], c[1], c[2], c[3], c[4], i, use[i], nh, THR, min_inl, seed)["status"]
            for i, c in enumerate(cams)]
    assert list(got["status"]) == want
    assert set(want) == {pn.REPLACED, pn.TOO_FEW, pn.KEPT, pn.FEW_INLIERS, pn.NOT_SELECTED}, want
    # a camera with fewer than 5 points and an unselected one keep R0 and report its score
    for c in (1, 4):
        assert got["h"][c] == -1 and np.array_equal(got["R"][c], cams[c][1])
    s.close()


def test_refusals_and_state(api):
    C, n = 2, 100
    cams = _cams(8, [n] * C)
    s = api.PoseSolver(0, C, C * n)
    s.set_ransac(np.ones(C, bool), 64, THR, 6, 2)
    _submit(s, cams)
    ref = s.download_ransac()
    for bad in [dict(n_hyp=0), dict(n_hyp=(1 << 20) + 1), dict(err_thres=0.0), dict(err_thres=np.nan),
                dict(err_thres=np.inf), dict(min_inliers=4)]:
        kw = dict(n_hyp=64, err_thres=THR, min_inliers=6, seed=2)
        kw.update(bad)
        with pytest.raises(api.CoslError, match="error -1: cosl_pose_solver_set_ransac"):
            s.set_ransac(np.ones(C, bool), **kw)
    with pytest.raises(api.CoslError, match="error -1: .*cameras"):
        s.set_ransac(np.ones(C + 1, bool), 64, THR, 6, 2)
    _submit(s, cams)  # the old setting still holds
    again = s.download_ransac()
    assert _bits(ref["R"], ref["t"], ref["sse"]) == _bits(again["R"], again["t"], again["sse"])
    with pytest.raises(api.CoslError, match="error -1: .*armed for 2"):
        _submit(s, cams[:1])
    _submit(s, cams)
    # in flight
    s.submit([c[0] for c in cams], [c[1] for c in cams], [c[2] for c in cams], [c[3] for c in cams],
             [c[4] for c in cams], TAU)
    with pytest.raises(api.CoslError, match="error -6"):
        s.set_ransac(np.ones(C, bool), 64, THR, 6, 2)
    with pytest.raises(api.CoslError, match="error -6"):
        s.download_ransac()
    s.collect()
    # nullable outputs
    assert api.LIB.cosl_pose_solver_download_ransac(s.h, None, None, None, None) == 0
    assert api.LIB.cosl_pose_solver_download_ransac_hyps(s.h, 0, None, None, None, None, None) == 0
    s.close()
