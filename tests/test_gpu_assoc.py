"""The registration handle (cosl_assoc_solver, DESIGN.md 5.6): parity with the float64 restatement of
tests/assoc_dense.py (identical status and feat, d2 and pred within 1e-9 relative) at the c3 shape, at a 13-camera rig,
ungated, on image borders and cell boundaries, with an entry without features and with long tracks; every status;
identical bits across submits and after permuting points and queries; refusals and the state rules; a Monte-Carlo run
within the bounds the CPU run of tests/test_assoc_dense_ref.py fixed; and the chain from the triangulation and pose
handles through registration into the pose solver's map-point update."""
import math

import numpy as np
import pytest

import assoc_dense as ad
import pose_mappts_dense as md
import tri_dense as td
from test_assoc_dense_ref import (MC_D2, MC_PRECISION, MC_RECALL, MC_TRIALS, _pix, permuted, status_scene)
from test_pose_mappts_dense_ref import MC_NEES as UPDATE_NEES
from test_pose_mappts_dense_ref import MC_REJECT as UPDATE_REJECT

pytestmark = pytest.mark.gpu

REL = 1e-9


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _solver(api, kw):
    return api.AssocSolver(0, len(kw["K"]), len(kw["X"]), max(1, int(kw["q_off"][-1])), max(1, len(kw["mf"])),
                           0 if kw.get("trk_off") is None else int(kw["trk_off"][-1]))


def _run(s, kw, **sc):
    s.submit(**kw, **sc)
    return s.collect()


def _close(a, b):
    """equal NaN and inf patterns, finite values within REL relative"""
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
    f = np.isfinite(b)
    assert (np.abs(a[f] - b[f]) <= REL * np.abs(b[f]) + 1e-12).all(), np.abs(a[f] - b[f]).max()


def _check_parity(got, ref):
    bad = np.flatnonzero((got["status"] != ref["status"]) | (got["feat"] != ref["feat"]))
    assert len(bad) == 0, (bad[:10], got["status"][bad[:10]], ref["status"][bad[:10]])
    _close(got["d2"], ref["d2"])
    _close(got["pred"], ref["pred"])


SHAPES = {
    # the c3 shape: 4 cameras x 2 000 features, 20 000 map points searching 1 to 4 of them
    "c3_4x2000_20000": dict(seed=1, entries=4, feats=2000, pts=20000),
    # a full rig: 13 cameras x 1 024 features
    "rig_13x1024_6000": dict(seed=2, entries=13, feats=1024, pts=6000),
    # no gate: the plain nearest feature of every pair, every cell scanned
    "ungated_4x500_1500": dict(seed=3, entries=4, feats=500, pts=1500, gate=math.inf),
    # an entry of an earlier frame without features, and tracks of up to 40 observations
    "empty_long_tracks_5x400_2000": dict(seed=4, entries=5, feats=400, pts=2000, empty=1, trk=40),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_the_restatement(api, shape):
    sh = SHAPES[shape]
    rng = np.random.default_rng(sh["seed"])
    kw = ad.scene(rng, sh["entries"], sh["feats"], sh["pts"], 1, 4, n_empty=sh.get("empty", 0),
                  trk_hi=sh.get("trk", 3))
    sc = dict(pixel_var=0.8, gate=sh.get("gate", ad.GATE_99), track_gate=20.0)
    s = _solver(api, kw)
    got = _run(s, kw, **sc)
    s.close()
    assert got["device_ms"] > 0
    ref = ad.associate(**kw, **sc)
    _check_parity(got, ref)
    counts = np.bincount(got["status"], minlength=8).tolist()
    print(f"{shape}: statuses {counts}, {got['device_ms']:.3f} ms")
    assert counts[0] > 0 and counts[3 if sh.get("gate", 1) < math.inf else 0] > 0


def test_borders_and_cell_boundaries(api):
    """Points projecting exactly onto cell boundaries and the image's edges (u, v multiples of 32 from 0 to W and H),
    features exactly on cell boundaries and just off them, at a gate whose box ends near a boundary."""
    kw, _, _, _ = status_scene()
    us, vs = np.arange(0.0, 641.0, 32.0), np.arange(0.0, 481.0, 32.0)
    X = np.array([_pix(u, v) for u in us for v in vs])
    rng = np.random.default_rng(12)
    base = np.array([[u, v] for u in us for v in vs])
    mf = np.concatenate([base, base + [1e-9, 0.0], base - [0.0, 1e-9], base + rng.normal(0.0, 2.0, base.shape)])
    n = len(X)
    kw.update(mf=mf, owned=None, trk_off=None, trk_cam=None, trk_m=None, feat_off=np.array([0, len(mf)], np.int32),
              X=X, P=np.array([md.random_spd(rng, 3, 1e-6, 1e-4) for _ in range(n)]),
              q_off=np.arange(n + 1, dtype=np.int32), q_cam=np.zeros(n, np.int32))
    s = _solver(api, kw)
    for gate in (0.5, 4.0, ad.GATE_99, math.inf):
        got = _run(s, kw, gate=gate)
        ref = ad.associate(**kw, gate=gate)
        _check_parity(got, ref)
        assert (got["status"] == 2).sum() == len(vs) + len(us) - 1  # u = W or v = H
    s.close()


def test_every_status(api):
    kw, status, feat, names = status_scene()
    s = _solver(api, kw)
    sc = dict(pixel_var=1.0, gate=ad.GATE_99, track_gate=ad.GATE_99)
    got = _run(s, kw, **sc)
    for i, name in enumerate(names):
        assert (got["status"][i], got["feat"][i]) == (status[i], feat[i]), name
    _check_parity(got, ad.associate(**kw, **sc))
    off = _run(s, kw, pixel_var=1.0, gate=ad.GATE_99)  # track_gate = +inf: no track check
    assert off["status"][names.index("track disagrees")] == 0
    # ties go to the lower feature index
    kw.update(mf=np.array([[101.0, 100.0], [99.0, 100.0], [101.0, 100.0]]), owned=None, trk_off=None, trk_cam=None,
              trk_m=None, feat_off=np.array([0, 3], np.int32), X=_pix(100.0, 100.0)[None],
              P=np.array([1e-6 * np.eye(3)]), q_off=np.array([0, 1], np.int32), q_cam=np.zeros(1, np.int32))
    got = _run(s, kw)
    assert got["status"][0] == 0 and got["feat"][0] == 0 and got["d2"][0, 0] == got["d2"][0, 1]
    s.close()


def test_identical_bits_across_submits_and_orders(api):
    rng = np.random.default_rng(21)
    kw = ad.scene(rng, 4, 800, 5000, 1, 4, sigma_x=(1e-3, 4e-2))
    sc = dict(track_gate=20.0)
    s = _solver(api, kw)
    a = _run(s, kw, **sc)
    b = _run(s, kw, **sc)
    for k in ("status", "feat", "d2", "pred"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    assert (a["status"] == 6).sum() >= 50
    kw2, src = permuted(kw, rng)
    c = _run(s, kw2, **sc)
    s.close()
    for k in ("status", "feat", "d2", "pred"):
        assert np.array_equal(_bits(a[k][src]), _bits(c[k])), k


def _bad(kind, kw):
    """One bad submit: (keyword arguments, message)"""
    kw = {k: (v.copy() if isinstance(v, np.ndarray) else list(v) if isinstance(v, list) else v) for k, v in kw.items()}
    sc = dict(pixel_var=1.0, gate=ad.GATE_99, track_gate=20.0)
    fo, qo = kw["feat_off"], kw["q_off"]
    if kind == "K":
        kw["K"][2, 0, 2] = np.nan
        msg = "K, R or t of camera 2 is not finite"
    elif kind == "rotation":
        kw["R"][1] *= 1.0 + 1e-6
        msg = "R of camera 1's prior is not a rotation"
    elif kind == "indefinite":
        w, V = np.linalg.eigh(kw["cam_cov"][0])
        w[0] = -w[0]
        kw["cam_cov"][0] = (V * w) @ V.T
        msg = "P of camera 0's prior is not positive definite"
    elif kind == "wh":
        kw["wh"][2] = [5000, 480]
        msg = "image size 5000 x 480 of camera 2 is not in \\[1, 4096\\]"
    elif kind == "featOff":
        kw["feat_off"][2] = fo[1] - 1
        msg = "camera 1 has -1 features"
    elif kind == "mf":
        kw["mf"][fo[1] + 3, 1] = np.inf
        msg = f"feature {fo[1] + 3}: m is not finite"
    elif kind == "covf":
        kw["covf"][7] = [[1.0, 0.5], [0.4, 1.0]]
        msg = "feature 7: covf is not"
    elif kind == "owned":
        kw["owned"][9] = 2
        msg = "feature 9: owned 2 is not 0 or 1"
    elif kind == "track camera":
        f = int(np.flatnonzero(np.diff(kw["trk_off"]) > 0)[4])
        kw["trk_cam"][kw["trk_off"][f]] = len(kw["K"])
        msg = f"track observation {kw['trk_off'][f]} of feature {f}: camera {len(kw['K'])} is not in"
    elif kind == "track m":
        f = int(np.flatnonzero(np.diff(kw["trk_off"]) > 0)[4])
        kw["trk_m"][kw["trk_off"][f], 0] = np.nan
        msg = f"track observation {kw['trk_off'][f]} of feature {f}: m is not finite"
    elif kind == "X":
        kw["X"][5, 2] = np.nan
        msg = "point 5: X is not finite"
    elif kind == "P":
        kw["P"][5][0, 1] += 1e-3
        msg = "point 5: P is not finite, symmetric and positive definite"
    elif kind == "query camera":
        kw["q_cam"][qo[6]] = len(kw["K"])
        msg = f"query {qo[6]} of point 6: camera {len(kw['K'])} is not in"
    elif kind == "twice":
        j = int(np.flatnonzero(np.diff(qo) >= 2)[0])
        kw["q_cam"][qo[j] + 1] = kw["q_cam"][qo[j]]
        msg = f"query {qo[j] + 1} of point {j}: camera {kw['q_cam'][qo[j]]} is queried twice"
    elif kind == "monotone":
        kw["q_off"][6] = qo[5] - 1
        msg = "point 5 has -1 queries, not 0 to 32"
    elif kind == "pixel_var":
        sc["pixel_var"] = math.inf
        msg = "pixel_var inf is not a finite value > 0"
    elif kind == "gate":
        sc["gate"] = 0.0
        msg = "gate 0 is not > 0"
    elif kind == "track_gate":
        sc["track_gate"] = math.nan
        msg = "track_gate nan is not > 0"
    return kw, sc, msg


BAD = ("K", "rotation", "indefinite", "wh", "featOff", "mf", "covf", "owned", "track camera", "track m", "X", "P",
       "query camera", "twice", "monotone", "pixel_var", "gate", "track_gate")


def test_refusals_and_state_rules(api):
    rng = np.random.default_rng(31)
    kw = ad.scene(rng, 3, 100, 40, 1, 2)
    sc = dict(pixel_var=1.0, gate=ad.GATE_99, track_gate=20.0)
    s = api.AssocSolver(0, 3, 40, int(kw["q_off"][-1]), 300, int(kw["trk_off"][-1]))
    first = _run(s, kw, **sc)
    for kind in BAD:
        bad, bsc, msg = _bad(kind, kw)
        with pytest.raises(api.CoslError, match=rf"error -1: cosl_assoc_solver_submit: {msg}"):
            s.submit(**bad, **bsc)
        again = _run(s, kw, **sc)  # the handle stays usable
        for k in ("status", "feat", "d2", "pred"):
            assert np.array_equal(_bits(again[k]), _bits(first[k])), (kind, k)
    # counts above the reserved sizes
    big = dict(kw, K=np.concatenate([kw["K"], kw["K"][:1]]), R=np.concatenate([kw["R"], kw["R"][:1]]),
               t=np.concatenate([kw["t"], kw["t"][:1]]), wh=np.concatenate([kw["wh"], kw["wh"][:1]]),
               cam_cov=kw["cam_cov"] + [None], feat_off=np.append(kw["feat_off"], kw["feat_off"][-1]))
    with pytest.raises(api.CoslError, match="error -1: .*4 cameras exceed the handle's 3"):
        s.submit(**big, **sc)
    more = dict(kw, feat_off=np.array([0, 0, 0, 301], np.int32), mf=np.zeros((301, 2)), covf=None, owned=None,
                trk_off=None, trk_cam=None, trk_m=None)
    with pytest.raises(api.CoslError, match="error -1: .*301 features exceed the handle's 300"):
        s.submit(**more, **sc)
    with pytest.raises(api.CoslError, match="error -1: .*41 points exceed the handle's 40"):
        s.submit(**dict(kw, X=np.concatenate([kw["X"], kw["X"][:1]]), P=np.concatenate([kw["P"], kw["P"][:1]]),
                        q_off=np.append(kw["q_off"], kw["q_off"][-1])), **sc)
    assert kw["q_off"][-1] < 120
    with pytest.raises(api.CoslError, match=rf"error -1: .*queries exceed the handle's {kw['q_off'][-1]}"):
        s.submit(**dict(kw, q_off=np.arange(41, dtype=np.int32) * 3, q_cam=np.tile([0, 1, 2], 40)), **sc)
    with pytest.raises(api.CoslError, match="error -1: .*point 0 has 33 queries, not 0 to 32"):
        s.submit(**dict(kw, q_off=np.concatenate([[0], np.full(40, 33)]).astype(np.int32),
                        q_cam=np.arange(33) % 3), **sc)
    # one request in flight: a second submit refused, the first unharmed
    s.submit(**kw, **sc)
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(**kw, **sc)
    while not s.done():
        pass
    got = s.collect()
    assert np.array_equal(_bits(got["d2"]), _bits(first["d2"]))
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    with pytest.raises(api.CoslError, match="error -6"):
        s.done()
    # nullable outputs
    s.submit(**kw, **sc)
    status = np.empty(len(first["status"]), np.int32)
    assert api.LIB.cosl_assoc_solver_collect(s.h, status.ctypes.data, None, None, None, None) == 0
    assert np.array_equal(status, first["status"])
    assert s.stream() is not None
    s.close()


def test_monte_carlo(api):
    """test_assoc_dense_ref.test_monte_carlo_chain's trials on the device, drawn from another seed"""
    rng = np.random.default_rng(8801)
    res = []
    for _ in range(MC_TRIALS):
        kw, truth, owned = ad.mc_trial(rng)
        s = _solver(api, kw)
        res.append((_run(s, kw, gate=ad.GATE_99, track_gate=ad.GATE_99), truth, owned))
        s.close()
    d2, prec, rec = ad.mc_stats(res)
    print(f"device chain: mean d2 of true matches {d2:.3f}, precision {prec:.4f}, recall {rec:.4f}")
    assert MC_D2[0] <= d2 <= MC_D2[1]
    assert MC_PRECISION[0] <= prec <= MC_PRECISION[1]
    assert MC_RECALL[0] <= rec <= MC_RECALL[1]


def test_chain_through_the_handles(api):
    """Two key frames solved by the pose solver with its covariance stage and their points triangulated by TriSolver;
    a later frame solved the same way, its features the points' observations (30 % missing) plus clutter; the points
    registered there with the later pose's covariance and tracks of the key-frame observations; then the registered
    points gated and updated by PoseSolver.submit(mappts=...) on that frame, whose mean NEES and rejection rate stay
    within the bounds of the map-point update's own Monte-Carlo run."""
    rng = np.random.default_rng(9200)
    ps = api.PoseSolver(0, 2, 60)
    ps.set_covariance(1.0)
    ps.reserve_mappts(20)
    ts = api.TriSolver(0, 2, 20, 40)
    asv = api.AssocSolver(0, 3, 20, 20, 40, 80)
    res, updates = [], []
    for _ in range(60):
        Xt, fr = td.chain_trial(rng, n_frames=3)
        keys, cur = fr[:2], fr[2]
        ps.submit([md.K_MC] * 2, [f["R0"] for f in keys], [f["t0"] for f in keys], [f["Ms"] for f in keys],
                  [f["ms"] for f in keys], md.TAU_MC)
        ok, R, t, _, _ = ps.collect()
        cov, _, _ = ps.download_covariance()
        assert ok.all()
        off, cam = td.chain_views(len(Xt))
        m = np.stack([keys[0]["m"], keys[1]["m"]], 1).reshape(-1, 2)
        Sm = np.stack([keys[0]["Sm"], keys[1]["Sm"]], 1).reshape(-1, 2, 2)
        ts.submit([md.K_MC] * 2, R, t, off, cam, m, covm=Sm, cam_cov=list(cov))
        tri = ts.collect()
        good = np.flatnonzero(tri["status"] == 0)
        ps.submit([md.K_MC], [cur["R0"]], [cur["t0"]], [cur["Ms"]], [cur["ms"]], md.TAU_MC)
        ok2, R2, t2, _, _ = ps.collect()
        cov2, _, _ = ps.download_covariance()
        assert ok2.all()
        seen = np.flatnonzero(rng.random(len(Xt)) >= 0.3)
        n_cl = 10
        mf = np.concatenate([cur["m"][seen], rng.uniform([0.0, 0.0], [md.W_MC, md.H_MC], (n_cl, 2))])
        covf = np.concatenate([cur["Sm"][seen], [md.random_spd(rng, 2, 0.25, 2.25) for _ in range(n_cl)]])
        trk_n = np.concatenate([np.full(len(seen), 2), np.zeros(n_cl, int)])
        kw = dict(K=[md.K_MC] * 3, R=np.concatenate([R, R2]), t=np.concatenate([t, t2]),
                  cam_cov=[cov[0], cov[1], cov2[0]], wh=[[md.W_MC, md.H_MC]] * 3,
                  feat_off=[0, 0, 0, len(mf)], mf=mf, covf=covf, owned=None,
                  trk_off=np.concatenate([[0], np.cumsum(trk_n)]), trk_cam=np.tile([0, 1], len(seen)),
                  trk_m=np.stack([keys[0]["m"][seen], keys[1]["m"][seen]], 1).reshape(-1, 2),
                  X=tri["X"][good], P=tri["P"][good], q_off=np.arange(len(good) + 1), q_cam=np.full(len(good), 2))
        got = _run(asv, kw, gate=ad.GATE_99, track_gate=ad.GATE_99)
        truth = np.full(len(Xt), -1)
        truth[seen] = np.arange(len(seen))
        res.append((got, truth[good], np.zeros(len(mf), np.int32)))
        reg = np.flatnonzero(got["status"] == 0)
        if not len(reg):
            continue
        f = got["feat"][reg]
        ps.submit([md.K_MC], [cur["R0"]], [cur["t0"]], [cur["Ms"]], [cur["ms"]], md.TAU_MC,
                  mappts=[(tri["X"][good][reg], tri["P"][good][reg], mf[f], covf[f])], gate=md.GATE_95)
        assert ps.collect()[0].all()
        updates.append((ps.download_mappts(), Xt[good][reg]))
    ps.close()
    ts.close()
    asv.close()
    d2, prec, rec = ad.mc_stats(res, (md.W_MC, md.H_MC))
    ne, rej = [], []
    for up, X in updates:
        s0 = up["status"] == 0
        assert ((up["status"] == 0) | (up["status"] == 1)).all()
        ne.append(md.nees(up["X"][s0], up["P"][s0], X[s0]))
        rej.append(up["status"] == 1)
    nees, r = float(np.mean(np.concatenate(ne))), float(np.mean(np.concatenate(rej)))
    print(f"chain: mean d2 of true matches {d2:.3f}, precision {prec:.4f}, recall {rec:.4f}; "
          f"update mean NEES {nees:.3f}, rejected {r:.4f}")
    assert MC_D2[0] <= d2 <= MC_D2[1]
    assert MC_PRECISION[0] <= prec <= MC_PRECISION[1]
    assert MC_RECALL[0] <= rec <= MC_RECALL[1]
    assert UPDATE_NEES[0] <= nees <= UPDATE_NEES[1]
    assert UPDATE_REJECT[0] <= r <= UPDATE_REJECT[1]
