"""The triangulation handle (cosl_tri_solver, DESIGN.md 5.5): parity with the float64 restatement of tests/tri_dense.py
at the newMapPoints, post-BA refresh and 32-view shapes with mixed camCov / covm presence; every status; points are
independent and submits deterministic; refusals and the state rules; a Monte-Carlo run within the bounds the CPU run of
tests/test_tri_dense_ref.py fixed; and the chain from two key frames' pose solves through triangulation into the pose
solver's map-point update on later frames."""
import math

import numpy as np
import pytest

import pose_mappts_dense as md
import tri_dense as td
from test_pose_mappts_dense_ref import MC_NEES as UPDATE_NEES
from test_pose_mappts_dense_ref import MC_REJECT as UPDATE_REJECT
from test_tri_dense_ref import MC_MAX_ERR, MC_NEES, MC_REJECT, MC_TRIALS, mc_stats, mc_trial, status_cases

pytestmark = pytest.mark.gpu

REL = 1e-9


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _table(rng, n_entries, cov_every=2):
    """A camera table of n_entries entries over the scene, with a pose covariance on every cov_every-th entry."""
    R, t = td.rig(rng, n_entries, spread=1.5)
    K = np.array([td.K_TRI] * n_entries)
    cc = [md.random_spd(rng, 6, 1e-8, 1e-6) if c % cov_every == 0 else None for c in range(n_entries)]
    return K, R, t, cc


def _points(rng, K, R, t, n_pts, lo, hi, covm=True, outliers=0.02):
    """n_pts points with lo to hi views each on distinct entries of the table, observed with noise from a random
    Sigma_m (0.5 to 1.5 px), a share moved 20 px; (off, cam, m, covm or None)."""
    counts = rng.integers(lo, hi + 1, n_pts)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    cam = np.concatenate([rng.choice(len(K), c, replace=False) for c in counts]).astype(np.int32)
    Xt = td.scene_points(rng, n_pts)
    Sm = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in range(off[-1])])
    m = np.empty((off[-1], 2))
    for j in range(n_pts):
        v = slice(off[j], off[j + 1])
        m[v] = td.observe(td.K_TRI, R[cam[v]], t[cam[v]], Xt[j], Sm[v], rng)
    m[rng.random(off[-1]) < outliers] += 20.0
    return off, cam, m, Sm if covm else None


def _run(s, K, R, t, cc, off, cam, m, covm, pixel_var=1.0, max_err=math.inf):
    s.submit(K, R, t, off, cam, m, covm=covm, cam_cov=cc, pixel_var=pixel_var, max_err=max_err)
    return s.collect()


def _check_parity(got, ref, max_err):
    """statuses equal except within REL of a threshold; X, P and stat within REL where the status says they are
    computed, NaN where it says they are not"""
    st, rs = got["status"], ref["status"]
    near = (np.abs(ref["stat"][:, 3] - 1.0) <= REL) | (np.abs(ref["stat"][:, 1] - max_err) <= REL * max_err)
    same = ~near
    assert np.array_equal(st[same], rs[same]), np.flatnonzero(st != rs)[:10]
    fin = same & np.isin(rs, (0, 2, 3))
    dX = np.linalg.norm(got["X"] - ref["X"], axis=1)
    assert (dX[fin] <= REL * np.linalg.norm(ref["X"], axis=1)[fin]).all(), dX[fin].max()
    dP = np.linalg.norm(got["P"] - ref["P"], axis=(1, 2))
    assert (dP[fin] <= REL * np.linalg.norm(ref["P"], axis=(1, 2))[fin]).all(), dP[fin].max()
    assert np.array_equal(_bits(got["P"]), _bits(np.swapaxes(got["P"], 1, 2)))
    dS = np.abs(got["stat"] - ref["stat"])
    assert (dS[fin] <= REL * np.abs(ref["stat"][fin]) + 1e-12).all(), dS[fin].max(axis=0)
    gone = same & np.isin(rs, (1, 4))
    for k in ("X", "P", "stat"):
        assert np.isnan(got[k][gone]).all(), k
    return int(near.sum())


SHAPES = {
    # newMapPoints for a full rig: 13 cameras at the first and the current frame, and one more view
    "new_13x1000x2-3": dict(seed=1, entries=39, pts=1000, lo=2, hi=3, covm=True),
    # the post-BA refresh of a c3 window: 20 key frames of 4 cameras, up to 8 views per point
    "refresh_c3_18600x8": dict(seed=2, entries=80, pts=18600, lo=2, hi=8, covm=False),
    # an outlier in any of 32 views gives e_max >= max_err, so this shape draws fewer
    "500x32": dict(seed=3, entries=40, pts=500, lo=32, hi=32, covm=True, outliers=0.004),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_the_restatement(api, shape):
    sh = SHAPES[shape]
    rng = np.random.default_rng(sh["seed"])
    K, R, t, cc = _table(rng, sh["entries"], cov_every=2 if sh["covm"] else 3)
    off, cam, m, covm = _points(rng, K, R, t, sh["pts"], sh["lo"], sh["hi"], sh["covm"], sh.get("outliers", 0.02))
    max_err = 6.0
    s = api.TriSolver(0, sh["entries"], sh["pts"], off[-1])
    got = _run(s, K, R, t, cc, off, cam, m, covm, 0.8, max_err)
    s.close()
    assert got["device_ms"] > 0
    ref = td.triangulate_all(K, R, t, cc, off, cam, m, covm, 0.8, max_err)
    near = _check_parity(got, ref, max_err)
    counts = np.bincount(got["status"], minlength=5).tolist()
    print(f"{shape}: statuses {counts}, {near} at a threshold, {got['device_ms']:.3f} ms")
    assert counts[0] > 0.8 * sh["pts"]


def test_every_status(api):
    cases = status_cases()
    K = np.array([k for c in cases for k in c[1]])
    R = np.array([r for c in cases for r in c[2]])
    t = np.array([x for c in cases for x in c[3]])
    m = np.concatenate([c[4] for c in cases])
    off = np.arange(len(cases) + 1, dtype=np.int32) * 2
    cam = np.arange(2 * len(cases), dtype=np.int32)
    s = api.TriSolver(0, len(K), len(cases), len(m))
    # one max_err per submit: the cases that need a small one run in a second submit
    for small in (False, True):
        sel = [i for i, c in enumerate(cases) if (c[5] < 1.0) == small]
        v = np.concatenate([np.arange(2 * i, 2 * i + 2) for i in sel])
        max_err = min(cases[i][5] for i in sel)
        got = _run(s, K, R, t, None, np.arange(len(sel) + 1) * 2, cam[v], m[v], None, 1.0, max_err)
        ref = td.triangulate_all(K, R, t, None, np.arange(len(sel) + 1) * 2, cam[v], m[v], None, 1.0, max_err)
        want = [cases[i][6] for i in sel]
        assert got["status"].tolist() == want, [cases[i][0] for i in sel]
        _check_parity(got, ref, max_err)
    s.close()
    assert off[-1] == len(m)


def test_points_are_independent_and_submits_deterministic(api):
    rng = np.random.default_rng(61)
    K, R, t, cc = _table(rng, 39)
    off, cam, m, covm = _points(rng, K, R, t, 2000, 2, 5)
    s = api.TriSolver(0, 39, 2000, off[-1])
    a = _run(s, K, R, t, cc, off, cam, m, covm)
    b = _run(s, K, R, t, cc, off, cam, m, covm)
    for k in ("X", "P", "stat", "status"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    j = 777
    m2 = m.copy()
    m2[off[j]] += [0.7, -0.4]
    c = _run(s, K, R, t, cc, off, cam, m2, covm)
    s.close()
    assert not np.array_equal(_bits(a["X"][j]), _bits(c["X"][j]))
    keep = np.arange(2000) != j
    for k in ("X", "P", "stat", "status"):
        assert np.array_equal(_bits(a[k][keep]), _bits(c[k][keep])), k


def _bad(kind, K, R, t, cc, off, cam, m, covm):
    """One bad submit: (args, message)"""
    K, R, t, off, cam, m, covm = (x.copy() for x in (K, R, t, off, cam, m, covm))
    cc = list(cc)
    pv, me = 1.0, 5.0
    if kind == "K":
        K[3, 0, 2] = np.nan
        msg = "K, R or t of camera 3 is not finite"
    elif kind == "t":
        t[3, 1] = np.inf
        msg = "K, R or t of camera 3 is not finite"
    elif kind == "rotation":
        R[3] *= 1.0 + 1e-6
        msg = "R of camera 3's prior is not a rotation"
    elif kind == "asymmetric":
        cc[2] = cc[2].copy()
        cc[2][0, 4] += 1e-9 * np.abs(np.diag(cc[2])).max()
        msg = "P of camera 2's prior is not symmetric"
    elif kind == "indefinite":
        w, V = np.linalg.eigh(cc[2])
        w[0] = -w[0]
        cc[2] = (V * w) @ V.T
        msg = "P of camera 2's prior is not positive definite"
    elif kind == "m":
        m[off[5] + 1, 0] = np.nan
        msg = f"view {off[5] + 1} of point 5: m is not finite"
    elif kind == "covm":
        covm[off[5]] = [[1.0, 0.5], [0.4, 1.0]]
        msg = f"view {off[5]} of point 5: covm is not"
    elif kind == "camera":
        cam[off[5]] = len(K)
        msg = f"view {off[5]} of point 5: camera {len(K)} is not in"
    elif kind == "twice":
        cam[off[5] + 1] = cam[off[5]]
        msg = f"view {off[5] + 1} of point 5: camera {cam[off[5]]} is used twice"
    elif kind == "one view":
        off[6:] -= off[6] - off[5] - 1
        msg = "point 5 has 1 views"
    elif kind == "monotone":
        off[6] = off[5] - 1
        msg = "point 5 has -1 views"
    elif kind == "first":
        off[0] = 1
        msg = "viewOff\\[0\\] = 1 is not 0"
    elif kind == "pixel_var":
        pv = 0.0
        msg = "pixel_var 0 is not a finite value > 0"
    elif kind == "max_err":
        me = math.nan
        msg = "max_err nan is not > 0"
    return (K, R, t, off, cam, m), dict(covm=covm, cam_cov=cc, pixel_var=pv, max_err=me), msg


BAD = ("K", "t", "rotation", "asymmetric", "indefinite", "m", "covm", "camera", "twice", "one view", "monotone",
       "first", "pixel_var", "max_err")


def test_refusals_and_state_rules(api):
    rng = np.random.default_rng(71)
    K, R, t, cc = _table(rng, 8)
    off, cam, m, covm = _points(rng, K, R, t, 20, 2, 4)
    s = api.TriSolver(0, 8, 20, off[-1] + 40)
    first = _run(s, K, R, t, cc, off, cam, m, covm, 1.0, 5.0)
    for kind in BAD:
        args, kw, msg = _bad(kind, K, R, t, cc, off, cam, m, covm)
        with pytest.raises(api.CoslError, match=rf"error -1: cosl_tri_solver_submit: {msg}"):
            s.submit(*args, **kw)
        again = _run(s, K, R, t, cc, off, cam, m, covm, 1.0, 5.0)  # the handle stays usable
        assert np.array_equal(_bits(again["X"]), _bits(first["X"])), kind
    # counts above the reserved sizes
    with pytest.raises(api.CoslError, match="error -1: .*9 cameras exceed the handle's 8"):
        s.submit(np.concatenate([K, K[:1]]), np.concatenate([R, R[:1]]), np.concatenate([t, t[:1]]), off, cam, m)
    with pytest.raises(api.CoslError, match="error -1: .*21 points exceed the handle's 20"):
        s.submit(K, R, t, np.concatenate([off, [off[-1] + 2]]), np.concatenate([cam, [0, 1]]),
                 np.concatenate([m, m[:2]]))
    many = np.arange(21, dtype=np.int32) * 8
    with pytest.raises(api.CoslError, match=rf"error -1: .*views exceed the handle's {off[-1] + 40}"):
        s.submit(K, R, t, many, np.tile(np.arange(8), 20), np.zeros((160, 2)))
    with pytest.raises(api.CoslError, match="error -1: .*point 0 has 33 views, not 2 to 32"):
        s.submit(K, R, t, [0, 33], np.arange(33) % 8, np.zeros((33, 2)))
    L = api.LIB
    with pytest.raises(api.CoslError, match="error -1: .*null argument"):
        api._ck(L.cosl_tri_solver_submit(s.h, 8, api._ptr(K), api._ptr(R), api._ptr(t), None, 20, api._ptr(off),
                                         None, api._ptr(m), None, 1.0, 5.0))
    # one request in flight: a second submit refused, the first unharmed
    s.submit(K, R, t, off, cam, m, covm=covm, cam_cov=cc, pixel_var=1.0, max_err=5.0)
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(K, R, t, off, cam, m, covm=covm, cam_cov=cc, pixel_var=1.0, max_err=5.0)
    while not s.done():
        pass
    got = s.collect()
    assert np.array_equal(_bits(got["X"]), _bits(first["X"]))
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    with pytest.raises(api.CoslError, match="error -6"):
        s.done()
    # nullable outputs
    s.submit(K, R, t, off, cam, m, covm=covm, cam_cov=cc, pixel_var=1.0, max_err=5.0)
    status = np.empty(20, np.int32)
    assert L.cosl_tri_solver_collect(s.h, None, None, None, status.ctypes.data, None) == 0
    assert np.array_equal(status, first["status"])
    assert s.stream() is not None
    s.close()


def test_monte_carlo(api):
    """test_tri_dense_ref.test_monte_carlo's trials on the device, drawn from another seed"""
    rng = np.random.default_rng(5501)
    s = api.TriSolver(0, 8, 20, 20 * 8)
    for n_views, trials in MC_TRIALS.items():
        res = []
        for _ in range(trials):
            K, R, t, Pc, off, cam, m, covm, Xt = mc_trial(rng, n_views)
            res.append((_run(s, K, R, t, Pc, off, cam, m, covm, 1.0, MC_MAX_ERR), Xt))
        nees, rej = mc_stats(res)
        print(f"{n_views} views: mean NEES {nees:.3f}, rejected {rej:.4f}")
        assert MC_NEES[0] <= nees <= MC_NEES[1]
        assert MC_REJECT[0] <= rej <= MC_REJECT[1]
    s.close()


def test_chain_into_the_map_point_update(api):
    """Two key frames solved by the pose solver with its covariance stage; their points triangulated with those poses
    and covariances; the status-0 points then gated and updated by PoseSolver.submit(mappts=...) on two later frames.
    The update's mean NEES and rejection rate stay within the bounds of the map-point update's own Monte-Carlo run."""
    rng = np.random.default_rng(9100)
    ps = api.PoseSolver(0, 2, 60)
    ps.set_covariance(1.0)
    ps.reserve_mappts(20)
    ts = api.TriSolver(0, 2, 20, 40)
    results, kept = [], 0
    for _ in range(60):
        Xt, fr = td.chain_trial(rng)
        keys = fr[:2]
        ps.submit([md.K_MC] * 2, [f["R0"] for f in keys], [f["t0"] for f in keys], [f["Ms"] for f in keys],
                  [f["ms"] for f in keys], md.TAU_MC)
        ok, R, t, _, _ = ps.collect()
        cov, _, st = ps.download_covariance()
        assert ok.all() and (st[:, 3] == 1.0).all()
        off, cam = td.chain_views(len(Xt))
        m = np.stack([keys[0]["m"], keys[1]["m"]], 1).reshape(-1, 2)
        Sm = np.stack([keys[0]["Sm"], keys[1]["Sm"]], 1).reshape(-1, 2, 2)
        tri = _run(ts, [md.K_MC] * 2, R, t, list(cov), off, cam, m, Sm)
        good = tri["status"] == 0
        kept += int(good.sum())
        for f in fr[2:]:
            ps.submit([md.K_MC], [f["R0"]], [f["t0"]], [f["Ms"]], [f["ms"]], md.TAU_MC,
                      mappts=[(tri["X"][good], tri["P"][good], f["m"][good], f["Sm"][good])], gate=md.GATE_95)
            assert ps.collect()[0].all()
            up = ps.download_mappts()
            results.append((up, Xt[good]))
    ps.close()
    ts.close()
    ne, rej = [], []
    for up, X in results:
        s0 = up["status"] == 0
        assert ((up["status"] == 0) | (up["status"] == 1)).all()
        ne.append(md.nees(up["X"][s0], up["P"][s0], X[s0]))
        rej.append(up["status"] == 1)
    nees, r = float(np.mean(np.concatenate(ne))), float(np.mean(np.concatenate(rej)))
    print(f"chain: {kept} points triangulated, update mean NEES {nees:.3f}, rejected {r:.4f}")
    assert kept >= 0.95 * 60 * 20
    assert UPDATE_NEES[0] <= nees <= UPDATE_NEES[1]
    assert UPDATE_REJECT[0] <= r <= UPDATE_REJECT[1]
