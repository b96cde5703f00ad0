"""The registration restatement of tests/assoc_dense.py without a GPU, before any GPU test trusts it: S matches central
differences of H_X and H_c and the spread of projections drawn from P_X and P_c, P_X = P_c = 0 leaves the plain
Mahalanobis distance under Sigma_f, the ungated search is the reference's searchMahaNearestFeatPt, the adjugate form
is the |L^-1 nu|^2 of a Cholesky factor, every status is reached in its order, ties go to the lower feature index,
claims do not depend on the order of points and queries, and a Monte-Carlo chain whose statistics fix the bounds of the
GPU test."""
import math

import numpy as np
import pytest

import assoc_dense as ad
import pose_dense as pd
import pose_mappts_dense as md
import tri_dense as td

# the Monte-Carlo bounds tests/test_gpu_assoc.py uses, fixed from test_monte_carlo_chain below
MC_D2 = (1.6, 2.3)
MC_PRECISION = (0.98, 1.0)
MC_RECALL = (0.95, 1.0)
MC_TRIALS = 30


def _camera(seed):
    rng = np.random.default_rng(seed)
    R, t = td.rig(rng, 2)
    X = td.scene_points(rng, 8)
    return rng, R, t, X


def test_S_matches_central_differences():
    rng, R, t, X = _camera(1)
    h = 1e-6
    for Ri, ti in zip(R, t):
        for Xj in X[:4]:
            PX, Pc = md.random_spd(rng, 3, 1e-4, 1e-2), md.random_spd(rng, 6, 1e-8, 1e-6)
            proj = lambda Rr, tt, XX: md.jacobians(td.K_TRI, Rr, tt, XX)[0]  # noqa: E731
            HX, Hc = np.empty((2, 3)), np.empty((2, 6))
            for k in range(3):
                d = np.zeros(3)
                d[k] = h
                HX[:, k] = (proj(Ri, ti, Xj + d) - proj(Ri, ti, Xj - d)) / (2 * h)
            for k in range(6):
                d = np.zeros(6)
                d[k] = h
                Hc[:, k] = (proj(Ri @ pd.exp_map(d[:3]), ti + d[3:], Xj) -
                            proj(Ri @ pd.exp_map(-d[:3]), ti - d[3:], Xj)) / (2 * h)
            want = HX @ PX @ HX.T + Hc @ Pc @ Hc.T
            _, _, S = ad.predict(td.K_TRI, Ri, ti, Pc, Xj, PX)
            assert np.linalg.norm(S - want) <= 1e-6 * np.linalg.norm(want)
            _, _, S0 = ad.predict(td.K_TRI, Ri, ti, None, Xj, PX)
            assert np.linalg.norm(S0 - HX @ PX @ HX.T) <= 1e-6 * np.linalg.norm(want)


def test_S_matches_the_spread_of_projections():
    """Projections of X drawn from P_X through poses drawn from P_c (the chart R exp([w]x), t + dt) spread as S, to the
    sampling error of 40 000 draws and the linearisation at these small covariances."""
    rng, R, t, X = _camera(2)
    n = 40000
    for Ri, ti, Xj in zip(R, t, X[:2]):
        PX, Pc = md.random_spd(rng, 3, 1e-5, 1e-3), md.random_spd(rng, 6, 1e-8, 1e-6)
        _, m, S = ad.predict(td.K_TRI, Ri, ti, Pc, Xj, PX)
        dX = rng.multivariate_normal(np.zeros(3), PX, n)
        dp = rng.multivariate_normal(np.zeros(6), Pc, n)
        ms = np.array([md.jacobians(td.K_TRI, Ri @ pd.exp_map(d[:3]), ti + d[3:], Xj + x)[0] for x, d in zip(dX, dp)])
        C = np.cov(ms.T)
        assert np.abs(ms.mean(0) - m).max() <= 0.05 * math.sqrt(S.trace())
        assert np.linalg.norm(C - S) <= 0.04 * np.linalg.norm(S), (C, S)


def test_quad_is_the_cholesky_form():
    rng = np.random.default_rng(3)
    A = np.array([md.random_spd(rng, 2, 1e-2, 1e3) for _ in range(500)])
    nu = rng.normal(0.0, 10.0, (500, 2))
    L = np.linalg.cholesky(A)
    z = np.linalg.solve(L, nu[..., None])[..., 0]
    want = (z * z).sum(1)
    assert (np.abs(ad.quad(A, nu) - want) <= 1e-10 * want).all()  # condition numbers up to 1e5
    assert np.isnan(ad.quad(np.array([[[1.0, 2.0], [2.0, 1.0]]]), np.ones((1, 2)))).all()


def _one_entry(rng, n_feats, n_pts, covf=True):
    kw = ad.scene(rng, 1, n_feats, n_pts, 1, 1, half=covf, owned_share=0.0, trk_hi=0)
    return kw


def test_zero_covariances_give_the_plain_mahalanobis_distance():
    rng = np.random.default_rng(4)
    kw = _one_entry(rng, 300, 50)
    kw["P"] = np.zeros_like(kw["P"])
    kw["cam_cov"] = [np.zeros((6, 6))]
    r = ad.associate(**kw, gate=math.inf)
    Sf = kw["covf"]
    for q in np.flatnonzero(np.isin(r["status"], (0, 6))):
        m = r["pred"][q, :2]
        assert np.array_equal(r["pred"][q, 2:], np.zeros(3))
        nu = kw["mf"] - m
        d = np.einsum("fi,fi->f", nu, np.linalg.solve(Sf, nu[..., None])[..., 0])
        assert r["feat"][q] == np.argmin(d)
        assert r["d2"][q, 0] == pytest.approx(d.min(), rel=1e-12)
        assert r["d2"][q, 1] == pytest.approx(np.partition(d, 1)[1], rel=1e-12)


@pytest.mark.parametrize("seed", [5, 6])
def test_ungated_search_is_the_references(seed):
    """With gate = +inf and Sigma_f = pixel_var I, f* is searchMahaNearestFeatPt's feature for var = S + pixel_var I
    (its 1 / maxDist scaling does not move the argmin), for every pair that reaches the search."""
    rng = np.random.default_rng(seed)
    kw = _one_entry(rng, 200, 60, covf=False)
    kw["covf"] = None
    pv = 0.7
    r = ad.associate(**kw, pixel_var=pv, gate=math.inf)
    searched = np.isin(r["status"], (0, 4, 5, 6))
    assert searched.sum() >= 40
    for q in np.flatnonzero(searched):
        p = r["pred"][q]
        var = np.array([[p[2], p[3]], [p[3], p[4]]]) + pv * np.eye(2)
        assert r["feat"][q] == ad.search_maha_nearest(p[:2], var, 3.0 * pv, kw["mf"])


def _pix(u, v, z=4.0):
    """The point at depth z that projects to (u, v) in status_scene's camera (exact in binary for these values)"""
    return np.array([(u - 320.0) * z / 512.0, (v - 240.0) * z / 512.0, z])


def status_scene():
    """One entry, K = [512 0 320; 0 512 240; 0 0 1], R = I, t = 0, 640 x 480, and purpose-built points and features;
    (keyword arguments, the expected status and feature of every pair, names).  P_X is 1e-6 I (S about 0.016 px^2) and
    Sigma_f = I, so at gate 9.21 a feature 1 px away is inside and one 20 px away is not."""
    K = np.array([[[512.0, 0.0, 320.0], [0.0, 512.0, 240.0], [0.0, 0.0, 1.0]]])
    pts, feats, want = [], [], []

    def add(name, X, fs, status, pick=0):
        """fs: (u, v, owned, track) per feature; pick: which of them the pair should report"""
        base = len(feats)
        feats.extend(fs)
        pts.append(X)
        want.append((name, status, base + pick if status not in (1, 2, 3, 7) else -1))

    add("registered", _pix(100.0, 100.0), [(101.0, 100.0, 0, None)], 0)
    add("registered on the image's corner", _pix(0.0, 0.0), [(0.5, 0.5, 0, None)], 0)
    add("registered on a cell boundary", _pix(64.0, 96.0), [(64.0, 96.0, 0, None), (63.5, 95.5, 0, None)], 0)
    add("behind", np.array([0.1, 0.1, -4.0]), [], 1)
    add("behind beats outside", np.array([-50.0, 0.0, -4.0]), [], 1)
    add("outside at u = W", _pix(640.0, 200.0), [(639.5, 200.0, 0, None)], 2)
    add("outside at v < 0", _pix(300.0, -0.5), [(300.0, 0.2, 0, None)], 2)
    add("no feature in the gate", _pix(400.0, 300.0), [(420.0, 300.0, 0, None)], 3)
    add("owned", _pix(200.0, 400.0), [(200.5, 400.0, 1, None)], 4)
    add("owned beats the track", _pix(250.0, 400.0), [(250.5, 400.0, 1, (10.0, 10.0))], 4)
    add("track disagrees", _pix(300.0, 400.0), [(300.5, 400.0, 0, (300.0 + 40.0, 400.0))], 5)
    add("track agrees", _pix(350.0, 400.0), [(350.5, 400.0, 0, (350.0, 400.2))], 0)
    add("claim kept", _pix(500.0, 100.0), [(500.5, 100.0, 0, None)], 0)
    feats_before = len(feats)
    pts.append(_pix(500.0, 101.5))  # farther from the same feature: loses it
    want.append(("claim lost", 6, feats_before - 1))
    add("depth 0 is non-finite", np.array([1.0, 0.0, 0.0]), [], 7)
    mf = np.array([[f[0], f[1]] for f in feats])
    owned = np.array([f[2] for f in feats], np.int32)
    tl = np.array([0 if f[3] is None else 1 for f in feats])
    trk_m = np.array([f[3] for f in feats if f[3] is not None])
    n = len(pts)
    kw = dict(K=K, R=np.eye(3)[None], t=np.zeros((1, 3)), cam_cov=None, wh=np.array([[640, 480]], np.int32),
              feat_off=np.array([0, len(mf)], np.int32), mf=mf, X=np.array(pts), P=np.array([1e-6 * np.eye(3)] * n),
              q_off=np.arange(n + 1, dtype=np.int32), q_cam=np.zeros(n, np.int32), covf=None, owned=owned,
              trk_off=np.concatenate([[0], np.cumsum(tl)]).astype(np.int32), trk_cam=np.zeros(len(trk_m), np.int32),
              trk_m=trk_m)
    return kw, np.array([w[1] for w in want]), np.array([w[2] for w in want]), [w[0] for w in want]


def test_every_status_and_its_order():
    kw, status, feat, names = status_scene()
    r = ad.associate(**kw, pixel_var=1.0, gate=ad.GATE_99, track_gate=ad.GATE_99)
    for i, name in enumerate(names):
        assert (r["status"][i], r["feat"][i]) == (status[i], feat[i]), name
    assert np.isnan(r["pred"][status == 1]).all() and np.isnan(r["pred"][status == 7]).all()
    assert np.isfinite(r["pred"][np.isin(status, (0, 2, 3, 4, 5, 6))]).all()
    assert np.isnan(r["d2"][np.isin(status, (1, 2, 7))]).all()
    assert np.isinf(r["d2"][status == 3]).all()
    assert set(status.tolist()) == set(range(8))
    # track_gate = +inf turns the track check off
    off = ad.associate(**kw, pixel_var=1.0, gate=ad.GATE_99)
    assert off["status"][names.index("track disagrees")] == 0


def test_ties_go_to_the_lower_feature_index():
    kw, _, _, _ = status_scene()
    kw.update(mf=np.array([[101.0, 100.0], [99.0, 100.0], [100.0, 101.0], [101.0, 100.0]]), owned=None, trk_off=None,
              trk_cam=None, trk_m=None, feat_off=np.array([0, 4], np.int32), X=_pix(100.0, 100.0)[None],
              P=np.array([1e-6 * np.eye(3)]), q_off=np.array([0, 1], np.int32), q_cam=np.zeros(1, np.int32))
    r = ad.associate(**kw)
    assert r["status"][0] == 0 and r["feat"][0] == 0 and r["d2"][0, 0] == r["d2"][0, 1]


def permuted(kw, rng):
    """kw with its points and each point's queries in a random order; (kw', the pair of kw at each pair of kw')"""
    n = len(kw["X"])
    perm = rng.permutation(n)
    qo = kw["q_off"]
    src, counts = [], []
    for j in perm:
        q = np.arange(qo[j], qo[j + 1])
        src.extend(rng.permutation(q))
        counts.append(len(q))
    src = np.array(src, np.int64)
    out = dict(kw, X=kw["X"][perm], P=kw["P"][perm], q_cam=kw["q_cam"][src],
               q_off=np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
    return out, src


def test_claims_do_not_depend_on_the_order_of_points_and_queries():
    rng = np.random.default_rng(7)
    kw = ad.scene(rng, 3, 150, 400, 1, 3, sigma_x=(1e-3, 4e-2))
    a = ad.associate(**kw, track_gate=20.0)
    assert (a["status"] == 6).sum() >= 10  # the draw has claims to resolve
    kw2, src = permuted(kw, rng)
    b = ad.associate(**kw2, track_gate=20.0)
    for k in ("status", "feat", "d2", "pred"):
        assert np.array_equal(a[k][src], b[k], equal_nan=True), k


def test_monte_carlo_chain():
    """Points triangulated by tri_dense from two key frames, then registered in a later frame whose features are drawn
    from each true point's projection with Sigma_f noise (30 % missing, half as many uniform clutter features, 10 %
    owned, tracks of the two key-frame observations): the true matches' mean d2 sits near 2 (2 dof, cut at the gate),
    and precision and recall at gate 9.21 are high."""
    rng = np.random.default_rng(8800)
    res = []
    for _ in range(MC_TRIALS):
        kw, truth, owned = ad.mc_trial(rng)
        res.append((ad.associate(**kw, gate=ad.GATE_99, track_gate=ad.GATE_99), truth, owned))
    d2, prec, rec = ad.mc_stats(res)
    print(f"chain: mean d2 of true matches {d2:.3f}, precision {prec:.4f}, recall {rec:.4f}")
    assert MC_D2[0] <= d2 <= MC_D2[1]
    assert MC_PRECISION[0] <= prec <= MC_PRECISION[1]
    assert MC_RECALL[0] <= rec <= MC_RECALL[1]
