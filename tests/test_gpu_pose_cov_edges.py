"""The pose solver's covariance stage (pose_cov_kernel) at the pose solve's edge rows (tests/pose_edge_cases.py):
1 to 20 000 points on the 128-thread CTA, tau 6 / 10 / 20, prevErrs at the Tukey cut-off, every forwarded option,
and the exits (a point at depth 0, whose residual is inf).  Every row runs as a one-camera submit on an armed
PoseSolver and as part of one multi-camera submit per tau and options, against tests/pose_cov_dense.py at the device's own
R_opt, t_opt."""
import math

import numpy as np
import pytest

import pose_cov_dense as cd
import pose_edge_cases as pc
from coslam_b200.ctypes_defs import PoseOpt
from pose_edge_cases import c_opt, same_bits

pytestmark = pytest.mark.gpu

VAR = 0.25
TIE = 1e-9  # a point whose residual is this close to tau (relative) has a weight decided at the rounding floor


@pytest.fixture(scope="module")
def solved(api):
    """name -> (inputs, one-camera result, multi-camera result); results are (R, t, cov, err, stats)."""
    rows = {r["name"]: pc.case_inputs(r) for r in pc.ROWS}
    s = api.PoseSolver(0, len(rows), sum(len(x[3]) for x in rows.values()))
    s.set_covariance(VAR)
    one, multi = {}, {}
    for name, (K, R0, t0, Ms, ms, tau, prev, opt) in rows.items():
        s.submit([K], [R0], [t0], [Ms], [ms], tau, [prev], opts=(PoseOpt * 1)(c_opt(opt)))
        _, R, t, _, _ = s.collect()
        cov, err, st = s.download_covariance()
        one[name] = (R[0], t[0], cov[0], err[0], st[0])
    for key in sorted({(x[5], x[7]) for x in rows.values()}):  # one submit per (tau, options)
        names = [n for n, x in rows.items() if (x[5], x[7]) == key]
        cols = list(zip(*[rows[n] for n in names]))
        s.submit(*cols[:5], key[0], list(cols[6]), opts=(PoseOpt * len(names))(*[c_opt(key[1])] * len(names)))
        _, R, t, _, _ = s.collect()
        cov, err, st = s.download_covariance()
        for c, n in enumerate(names):
            multi[n] = (R[c], t[c], cov[c], err[c], st[c])
    s.close()
    return {n: (rows[n], one[n], multi[n]) for n in rows}


@pytest.mark.parametrize("r", pc.ROWS, ids=lambda r: r["name"])
def test_matches_the_dense_reference(solved, r):
    (K, R0, t0, Ms, ms, tau, prev, opt), (R, t, cov, err, st), multi = solved[r["name"]]
    for a, b in zip((R, t, cov, err, st), multi):  # the camera's CTA does not depend on its neighbours
        assert same_bits(a, b), r["name"]
    ref = cd.cov_stage(K, R, t, Ms, ms, tau, VAR)
    de = cd.residual_error(err, ref["e"])
    assert len(err) == len(Ms) and de <= 1e-9, (r["name"], de)
    assert st[1] == ref["dof"]
    valid = st[3] == 1.0
    assert np.isnan(cov).all() != valid and valid == ref["valid"], (r["name"], st, ref["min_pivot"])
    if r["name"] in ("live1", "live2"):  # 2 or 4 equations for 6 unknowns
        assert not valid and st[1] < 0
    fin = np.isfinite(ref["e"])
    near = np.abs(ref["e"][fin] - tau) <= TIE * tau
    if near.any():
        print(f"{r['name']}: {int(near.sum())} residual(s) within {TIE:g} of tau; only valid and NaN compared")
        return
    if ref["dof"] > 0:
        assert st[0] == pytest.approx(ref["sigma2_hat"], rel=1e-10)
    else:
        assert math.isnan(st[0])
    if not valid:
        print(f"{r['name']}: singular (min pivot {st[2]:.1e}), e within {de:.1e}")
        return
    assert st[2] == pytest.approx(ref["min_pivot"], rel=1e-6)
    # kappa(H) is about 1e3 on every valid row, so the summation-order noise of H stays far below the bound
    kappa = float(np.linalg.cond(ref["H"]))
    bound = 1e-9
    rel = float(np.linalg.norm(cov - ref["cov"]) / np.linalg.norm(ref["cov"]))
    print(f"{r['name']} (n={len(Ms)}): cov {rel:.2e} (bound {bound:.0e}, kappa {kappa:.1e}), e {de:.1e}")
    assert rel <= bound
    assert same_bits(cov, cov.T)
