"""The map-point update of the pose solver (cosl_pose_solver_submit_mappts, DESIGN.md 5.4): the solve and its stage are
submit_prior's bit for bit; the update matches the float64 restatement of tests/pose_mappts_dense.py at the device's
own pose and stage covariance; every status is reached; points are independent; bad map points and the state rules
are refused; and a Monte-Carlo run within the bounds the CPU run of tests/test_pose_mappts_dense_ref.py fixed."""
import math

import numpy as np
import pytest

import pose_cov_dense as cd
import pose_dense as pd
import pose_mappts_dense as md
import pose_prior_dense as ppd
from coslam_b200 import synth
from test_gpu_pose_covariance import _bits, _same_solve
from test_gpu_pose_obscov import _covx, _same_stage
from test_pose_mappts_dense_ref import MC_D2, MC_NEES, MC_REJECT, mc_stats

pytestmark = pytest.mark.gpu

TAU = 10.0
VAR = 1.0
GATE = md.GATE_95
REL = 1e-9


def _case(seeds_npts, seed=0):
    """(Ks, R0s, t0s, Ms, ms, prev) of synth pose cases, and their true poses"""
    cs = [synth.make_pose_case(n, 1280, 720, seed=s) for s, n in seeds_npts]
    rng = np.random.default_rng(seed)
    prev = [np.abs(rng.normal(0, 4, n)) if c % 3 != 1 else None for c, (_, n) in enumerate(seeds_npts)]
    case = ([c[0] for c in cs], [c[1] for c in cs], [c[2] for c in cs], [c[3] for c in cs], [c[4] for c in cs], prev)
    return case, [(c[5], c[6]) for c in cs]


def _map_points(case, truth, counts, seed, covm=True, outliers=0.05):
    """Per camera: n map points seen by the true pose at depths 3 to 20, a prior mean drawn from a random P0 (1 to 10
    cm), observations with noise from a random Sigma_m (0.5 to 1.5 px) and a share of outliers moved 30 px; None for
    n = 0.  covm False passes no Sigma_m (pixel_var I)."""
    rng = np.random.default_rng(seed)
    out = []
    for c, n in enumerate(counts):
        if n == 0:
            out.append(None)
            continue
        K, (Rt, tt) = case[0][c], truth[c]
        Xt = md.view_points(K, Rt, tt, rng, n, 1280, 720, 3.0, 20.0)
        P0 = np.array([md.random_spd(rng, 3, 1e-4, 1e-2) for _ in range(n)])
        X0 = Xt + np.array([rng.multivariate_normal(np.zeros(3), p) for p in P0])
        Sm = np.array([md.random_spd(rng, 2, 0.25, 2.25) for _ in range(n)])
        u, v = pd.project(K, Rt, tt, Xt)
        m = np.column_stack([u, v]) + np.array([rng.multivariate_normal(np.zeros(2), s) for s in Sm])
        m[rng.random(n) < outliers] += 30.0
        out.append((X0, P0, m, Sm if covm else None))
    return out


def _solver(case, api, nmap):
    s = api.PoseSolver(0, len(case[3]), max(1, sum(len(a) for a in case[3])))
    s.set_covariance(VAR)
    s.reserve_mappts(nmap)
    return s


def _run(s, case, covx=None, prior=None, mappts=None, gate=GATE):
    Ks, R0s, t0s, Ms, ms, prev = case
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, covx=covx, prior=prior, mappts=mappts, gate=gate)
    res = s.collect(), s.download_covariance()
    return res + ((s.download_mappts(),) if mappts is not None else ())


def _nmap(mappts):
    return sum(0 if e is None else len(e[0]) for e in mappts)


def _check_parity(res, mappts, case, pixel_var=VAR):
    """the device's update against md.update_all at the device's own R_opt, t_opt and stage covariance"""
    (ok, R, t, _, dms), (cov, _, st), got = res
    assert dms > 0
    near, j = 0, 0
    for c, e in enumerate(mappts):
        if e is None:
            continue
        X0, P0, m = e[:3]
        Sm = e[3] if len(e) > 3 else None
        n = len(X0)
        Sm = np.broadcast_to(pixel_var * np.eye(2), (n, 2, 2)) if Sm is None else Sm
        ref = md.update_all(case[0][c], R[c], t[c], cov[c], X0, P0, m, Sm, GATE, st[c, 3] == 1.0)
        sl = slice(j, j + n)
        assert (got["cam"][sl] == c).all()
        at_gate = np.abs(ref["d2_0"] - GATE) <= REL * GATE
        near += int(at_gate.sum())
        same = ~at_gate
        assert np.array_equal(got["status"][sl][same], ref["status"][same]), c
        both = same & (ref["status"] == 0)
        dX = np.linalg.norm(got["X"][sl] - ref["X"], axis=1)
        assert (dX[both] <= REL * np.linalg.norm(ref["X"], axis=1)[both]).all(), (c, dX.max())
        kept = same & (ref["status"] != 0)
        assert np.array_equal(got["X"][sl][kept], ref["X"][kept]), c
        dP = np.linalg.norm(got["P"][sl] - ref["P"], axis=(1, 2))
        assert (dP[same] <= REL * np.linalg.norm(ref["P"], axis=(1, 2))[same]).all(), (c, dP.max())
        assert np.array_equal(_bits(got["P"][sl]), _bits(np.swapaxes(got["P"][sl], 1, 2)))
        for k in ("d2_0", "d2_1"):
            a, b = got[k][sl][same], ref[k][same]
            assert np.array_equal(np.isnan(a), np.isnan(b)), (c, k)
            f = ~np.isnan(b)
            assert (np.abs(a[f] - b[f]) <= REL * np.abs(b[f]) + 1e-12).all(), (c, k)
        e_fin = np.abs(ref["e0"][np.isfinite(ref["e0"])])
        assert cd.residual_error(got["e0"][sl], ref["e0"]) <= 1e-9 * max(1.0, e_fin.max(initial=0.0)), c
        j += n
    assert j == len(got["status"])
    return near


@pytest.mark.parametrize("with_covx,with_prior", [(False, False), (True, False), (False, True), (True, True)])
def test_the_solve_is_submit_priors(api, with_covx, with_prior):
    case, truth = _case([(50 + c, 60 + 11 * c) for c in range(13)], seed=1)
    C = len(case[3])
    covx = _covx(case, 11) if with_covx else None
    rng = np.random.default_rng(12)
    prior = [ppd.drawn_prior(R0, t0, rng) if c % 2 else None for c, (R0, t0) in enumerate(zip(case[1], case[2]))]
    prior = prior if with_prior else None
    mappts = _map_points(case, truth, [40] * C, 13)
    s = _solver(case, api, _nmap(mappts))
    plain = _run(s, case, covx, prior)
    got = _run(s, case, covx, prior, mappts)
    s.close()
    _same_solve(got[0], plain[0])
    _same_stage(got[1], plain[1])


def test_matches_the_restatement_4x192x2000(api):
    case, truth = _case([(100 + c, 192) for c in range(4)])
    mappts = _map_points(case, truth, [2000] * 4, 21)
    s = _solver(case, api, _nmap(mappts))
    res = _run(s, case, mappts=mappts)
    s.close()
    near = _check_parity(res, mappts, case)
    st = res[2]["status"]
    print(f"statuses {np.bincount(st, minlength=4).tolist()}, {near} at the gate")
    assert (st == 0).sum() > 6000 and (st == 1).sum() > 200


def test_matches_the_restatement_13_mixed(api):
    """13 cameras with mixed solve and map-point counts: camera 4 has no map points, camera 7 no solve points but a
    prior (its stage covariance comes from the prior alone), covm on some cameras and pixel_var I on the others, and
    measurement covariances on the solve"""
    case, truth = _case([(50 + c, 60 + 11 * c) for c in range(13)], seed=1)
    C = len(case[3])
    case[3][7], case[4][7] = case[3][7][:0], case[4][7][:0]
    case[5][7] = None if case[5][7] is None else case[5][7][:0]
    rng = np.random.default_rng(31)
    prior = [None] * C
    prior[7] = ppd.drawn_prior(case[1][7], case[2][7], rng, max_deg=2.0, scale=1e-4)
    counts = [37 * c + 5 for c in range(C)]
    counts[4] = 0
    mappts = _map_points(case, truth, counts, 32)
    mappts = [e if e is None or c % 3 else e[:3] for c, e in enumerate(mappts)]
    s = _solver(case, api, _nmap(mappts) + 10)
    res = _run(s, case, _covx(case, 33), prior, mappts)
    s.close()
    assert res[1][2][7, 3] == 1.0
    _check_parity(res, mappts, case)
    assert not (res[2]["cam"] == 4).any() and (res[2]["status"][res[2]["cam"] == 7] == 0).any()


def test_every_status(api):
    """camera 0: a normal camera with a point far from its observation (gated out), one behind the camera and one
    at its centre; camera 1 has 2 solve points and no prior, so its stage covariance is singular (status 3)"""
    case, truth = _case([(140, 120), (141, 120)], seed=6)
    case[3][1], case[4][1], case[5][1] = case[3][1][:2], case[4][1][:2], None
    mappts = _map_points(case, truth, [30, 10], 41, outliers=0.0)
    s = _solver(case, api, 40)
    (_, R, t, _, _), _ = _run(s, case)  # the solve is deterministic: the same pose again below
    X0, P0, m, Sm = mappts[0]
    X0[1] = R[0].T @ (np.array([0.0, 0.0, -5.0]) - t[0])
    X0[2] = md.centre_point(R[0], t[0])
    m[3] += 300.0
    res = _run(s, case, mappts=mappts)
    s.close()
    assert np.array_equal(_bits(res[0][1]), _bits(R))
    got = res[2]
    assert res[1][2][1, 3] == 0.0
    assert (got["status"][got["cam"] == 1] == 3).all() and np.isnan(got["d2_0"][got["cam"] == 1]).all()
    assert got["status"][1] == 2 and got["status"][2] == 2 and got["status"][3] == 1
    assert (got["status"][[0] + list(range(4, 30))] == 0).sum() > 20
    assert np.array_equal(_bits(got["X"][1:3]), _bits(X0[1:3]))
    _check_parity(res, mappts, case)


def test_points_are_independent(api):
    case, truth = _case([(100 + c, 192) for c in range(4)])
    mappts = _map_points(case, truth, [300] * 4, 51)
    s = _solver(case, api, 1200)
    a = _run(s, case, mappts=mappts)[2]
    X0, P0, m, Sm = (x.copy() for x in mappts[1])
    k = 17
    X0[k] += 0.01
    P0[k] *= 2.0
    m[k] -= 0.5
    mp2 = list(mappts)
    mp2[1] = (X0, P0, m, Sm)
    b = _run(s, case, mappts=mp2)[2]
    s.close()
    j = 300 + k
    assert not np.array_equal(_bits(a["X"][j]), _bits(b["X"][j]))
    keep = np.arange(len(a["status"])) != j
    for key in ("X", "P", "d2_0", "d2_1", "e0", "status"):
        assert np.array_equal(np.asarray(a[key])[keep].view(np.uint8), np.asarray(b[key])[keep].view(np.uint8)), key


def _bad(kind, e):
    X0, P0, m, Sm = (x.copy() for x in e)
    if kind == "X":
        X0[5, 1] = np.nan
    elif kind == "m":
        m[5, 0] = np.inf
    elif kind == "asymmetric":
        P0[5, 0, 2] += 1e-9 * np.abs(np.diagonal(P0[5])).max()
    elif kind == "indefinite":
        w, V = np.linalg.eigh(P0[5])
        w[0] = -w[0]
        P0[5] = (V * w) @ V.T
    elif kind == "covm":
        Sm[5] = [[1.0, 0.5], [0.4, 1.0]]
    return X0, P0, m, Sm


BAD = {"X": "X or m is not finite", "m": "X or m is not finite", "asymmetric": "P is not finite, symmetric",
       "indefinite": "P is not finite, symmetric", "covm": "covm is not"}


def test_refusals_and_state_rules(api):
    case, truth = _case([(100 + c, 192) for c in range(4)])
    Ks, R0s, t0s, Ms, ms, prev = case
    mappts = _map_points(case, truth, [50] * 4, 61)
    s = _solver(case, api, 200)
    for kind, msg in BAD.items():
        mp = list(mappts)
        mp[2] = _bad(kind, mappts[2])
        with pytest.raises(api.CoslError, match=rf"error -1: cosl_pose_solver_submit_mappts: map point 5 of camera "
                                                rf"2: {msg}"):
            s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mp, gate=GATE)
        assert _run(s, case, mappts=mappts)[2]["status"].size == 200, kind
    for gate in (0.0, -1.0, math.nan, math.inf):
        with pytest.raises(api.CoslError, match="error -1: .*gate"):
            s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=gate)
    with pytest.raises(api.CoslError, match="error -1: .*201 map points exceed the 200 reserved"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, gate=GATE,
                 mappts=mappts[:3] + [tuple(np.concatenate([x, x[:1]]) for x in mappts[3])])
    first = _run(s, case, mappts=mappts)[2]
    # in flight: submit, reserve and download refused; the solve in flight is unharmed
    s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=GATE)
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=GATE)
    with pytest.raises(api.CoslError, match="error -6"):
        s.reserve_mappts(400)
    with pytest.raises(api.CoslError, match="error -6"):
        s.download_mappts()
    s.collect()
    again = s.download_mappts()
    for key in ("X", "P", "d2_0", "status"):
        assert np.array_equal(np.asarray(again[key]).view(np.uint8), np.asarray(first[key]).view(np.uint8)), key
    out = np.empty(200, np.int32)
    assert api.LIB.cosl_pose_solver_download_mappts(s.h, None, None, None, out.ctypes.data) == 0  # nullable
    assert np.array_equal(out, first["status"])
    # a plain submit: nothing to download
    _run(s, case)
    with pytest.raises(api.CoslError, match="error -6: .*not a submit_mappts"):
        s.download_mappts()
    # unarmed
    s.set_covariance(0.0)
    with pytest.raises(api.CoslError, match="error -6: .*not armed"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=GATE)
    s.set_covariance(VAR)
    # unreserved, after reserve(0), and a reserve that grows the handle
    s.reserve_mappts(0)
    with pytest.raises(api.CoslError, match="error -6: .*no map points reserved"):
        s.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=GATE)
    s.reserve_mappts(1000)
    grown = _run(s, case, mappts=mappts)[2]
    assert np.array_equal(_bits(grown["X"]), _bits(first["X"]))
    s.close()
    fresh = api.PoseSolver(0, 4, 4 * 192)
    fresh.set_covariance(VAR)
    with pytest.raises(api.CoslError, match="error -6: .*no map points reserved"):
        fresh.submit(Ks, R0s, t0s, Ms, ms, TAU, prev, mappts=mappts, gate=GATE)
    with pytest.raises(api.CoslError, match="error -6"):
        fresh.download_mappts()
    fresh.close()


def test_monte_carlo(api):
    """test_pose_mappts_dense_ref.test_monte_carlo's frames on the device: 300 frames of 20 map points, 20 frames per
    submit (one camera each), the pose and its covariance from the device's own solve of 30 points at 1 px"""
    rng = np.random.default_rng(7301)
    s = api.PoseSolver(0, 20, 20 * 30)
    s.set_covariance(1.0)
    s.reserve_mappts(20 * 20)
    frames = []
    for _ in range(15):
        fr = [md.mc_frame(rng) for _ in range(20)]
        s.submit([md.K_MC] * 20, [f["R0"] for f in fr], [f["t0"] for f in fr], [f["Ms"] for f in fr],
                 [f["ms"] for f in fr], md.TAU_MC, mappts=[(f["X0"], f["P0"], f["m"], f["Sm"]) for f in fr],
                 gate=GATE)
        ok, _, _, _, _ = s.collect()
        assert ok.all()
        got = s.download_mappts()
        for c, f in enumerate(fr):
            sel = got["cam"] == c
            frames.append((f, {k: got[k][sel] for k in ("X", "P", "d2_0", "status")}))
    s.close()
    m_nees, m_d2, rej = mc_stats(frames)
    print(f"mean NEES {m_nees:.3f}, mean d2_0 {m_d2:.3f}, rejected {rej:.4f}")
    assert MC_NEES[0] <= m_nees <= MC_NEES[1]
    assert MC_D2[0] <= m_d2 <= MC_D2[1]
    assert MC_REJECT[0] <= rej <= MC_REJECT[1]
