"""The per-frame pose kernel (pose_intracam_kernel, coslam_b200/csrc/pose.cu) at its edge shapes
(tests/pose_edge_cases.py): point counts from 1 to 20 000 on the 128-thread CTA, the live tau = 6 with
prevErrs, solvePnPRobust's tau 20 and 6, weights at the Tukey cut-off, every forwarded option and the
failure exits.  Every row runs through pose_intracam and through a one-camera batch call with its options,
against the oracle and, where stored, the reference's own outputs (tests/golden/pose_edges_ref.npz).

Tie-free rows take the same discrete path as the oracle, so counts and lambda must be equal and the costs
and pose agree to summation-order rounding.  On tie rows (a decision at the rounding floor) only ok,
retTypeLM and the pose are compared."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_dense as pd
import pose_edge_cases as pc
from coslam_b200 import synth
from coslam_b200.ctypes_defs import PoseOpt
from pose_edge_cases import OPT_KEYS, c_opt, golden_rows, opt_vector, same_bits

pytestmark = pytest.mark.gpu

INT_KEYS = ("retTypeLM", "npts", "nIterLM", "nIterRW")
ERR_KEYS = ("err0", "err", "errRW")


def fields(o):
    f = {k: float(getattr(o, "lambda_" if k == "lambda" else k)) for k in OPT_KEYS}
    f["npts"] = o.npts
    return f


def err_close(a, b):
    """|a - b| <= 1e-9 |b| + 1e-12; equal infinities and two NaNs count as equal.  err0, err and errRW of a
    later round are costs at, and with Tukey weights taken at, a pose that agrees with the oracle's only to
    its summation-order noise (up to 2e-9 here), so they move by up to 1.8e-10 relative on an H100 (live255).
    The floor covers the 1- and 2-point rows, which end at costs of about 1e-27."""
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    return a == b or abs(a - b) <= 1e-9 * abs(b) + 1e-12


def compare(name, tie, ok, R, t, f, ok_e, R_e, t_e, f_e, what):
    """The checks of one solve against an expected one (f_e may lack npts); returns the worst differences."""
    assert ok == ok_e, (name, what)
    assert f["retTypeLM"] == f_e["retTypeLM"], (name, what, f["retTypeLM"], f_e["retTypeLM"])
    d = {}
    if R_e is not None:
        d["Rt"] = max(np.abs(R - R_e).max(), np.abs(t - t_e).max())
        assert d["Rt"] <= 1e-8, (name, what, d)
    if not tie:
        for k in INT_KEYS:
            if k in f_e:
                assert f[k] == f_e[k], (name, what, k, f[k], f_e[k])
        for k in ("lambda", "lambda0"):
            assert same_bits(f[k], f_e[k]), (name, what, k, f[k], f_e[k])
        for k in ERR_KEYS:
            assert err_close(f[k], f_e[k]), (name, what, k, f[k], f_e[k])
            if np.isfinite(f_e[k]) and f[k] != f_e[k]:
                d["err"] = max(d.get("err", 0.0), abs(f[k] - f_e[k]) / max(abs(f_e[k]), 1e-2))
    return d


def gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt):
    """The row through pose_intracam and through a one-camera batch call; both must agree bit for bit."""
    ok, R, t, o = api.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    opts = (PoseOpt * 1)(c_opt(opt))
    okb, Rb, tb, ob = api.pose_intracam_batch([K], [R0], [t0], [Ms], [ms], tau, [prev], opts=opts)
    assert okb[0] == ok and same_bits(Rb[0], R) and same_bits(tb[0], t)
    assert same_bits(opt_vector(ob[0]), opt_vector(o)) and ob[0].npts == o.npts
    return ok, R, t, fields(o)


@pytest.mark.parametrize("r", pc.ROWS, ids=lambda r: r["name"])
def test_full_solve_matches_oracle(api, orc, r):
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(r)
    ok, R, t, f = gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt)
    ok_o, R_o, t_o, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    f_o = fields(o)
    if r["exit"] == "rw0":  # the oracle hands back the option block it was given
        assert ok and ok_o and f["nIterRW"] == 0 == f_o["nIterRW"]
        assert same_bits(R, R0) and same_bits(t, t0) and same_bits(R_o, R0) and same_bits(t_o, t0)
        return
    d = compare(r["name"], r["tie"], ok, R, t, f, ok_o, R_o, t_o, f_o, "oracle")
    print(f"{r['name']} (n={r['n']}{', tie' if r['tie'] else ''}): worst |GPU - oracle|"
          + "".join(f" {k} {v:.1e}" for k, v in d.items()))


def test_full_solve_matches_reference_golden(api):
    n = 0
    for r, g in golden_rows():
        if "ref_ok" not in g:
            continue
        ok, R, t, f = gpu_solves(api, g["K"], g["R0"], g["t0"], g["Ms"], g["ms"], g["tau"], g["prev"], g["opt"])
        f_g = dict(zip(OPT_KEYS, g["ref_opt"]))
        d = compare(r["name"], r["tie"], ok, R, t, f, bool(g["ref_ok"]), g.get("ref_R"), g.get("ref_t"), f_g,
                    "reference")
        print(f"{r['name']} (n={r['n']}): worst |GPU - reference|" + "".join(f" {k} {v:.1e}" for k, v in d.items()))
        n += 1
    assert n >= 30


def rotation_log(R):
    return Rotation.from_matrix(R).as_rotvec()


def step_of(R0, t0, R, t):
    """delta = (log(R0^T R), t - t0) of the trial pose R0 exp(delta), t0 + delta_t."""
    return np.concatenate([rotation_log(R0.T @ R), t - t0])


STEP_ROWS = [r for r in pc.ROWS if r["exit"] is None and not r["tie"] and r["opt"] == pc.DEFAULT_OPT]


@pytest.mark.parametrize("r", STEP_ROWS, ids=lambda r: r["name"])
def test_one_step(api, orc, r):
    """maxIterLM = maxIterRW = 1: the output is the first trial pose whatever the step's fate."""
    K, R0, t0, Ms, ms, tau, prev, _ = pc.case_inputs(r)
    opt = (1, 1) + pc.DEFAULT_OPT[2:]
    ok, R, t, f = gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt)
    _, R_o, t_o, _ = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    W = pd.prev_weights(len(Ms), tau, prev)
    A, _, _ = pd.one_step(K, R0, t0, Ms, ms, W, opt[5])
    kappa = np.linalg.cond(A, np.inf)
    d_gpu, d_orc = step_of(R0, t0, R, t), step_of(R0, t0, R_o, t_o)
    # the per-point arithmetic is the oracle's, only the summation order differs; 1e-15 covers recovering
    # delta from the rounded trial pose
    e_orc = np.abs(d_gpu - d_orc).max()
    tol = (1e-13 + 1e-16 * kappa) * np.abs(d_orc).max() + 1e-15
    msg = f"{r['name']}: kappa {kappa:.1e}, |d| {np.abs(d_orc).max():.1e}, |d_gpu - d_orc| {e_orc:.1e} (tol {tol:.1e})"
    assert e_orc <= tol, msg
    _, _, d_ex = pd.exact_step(K, R0, t0, Ms, ms, W, opt[5])
    e_ex = np.abs(d_gpu - d_ex).max()
    if kappa <= 1e8:
        rel = e_ex / max(np.abs(d_ex).max(), 1e-300) if e_ex > 1e-15 else 0.0
        msg += f", |d_gpu - d_exact| {e_ex:.1e} ({rel:.1e} rel)"
        assert e_ex <= 1e-4 * np.abs(d_ex).max() + 1e-15, msg
    else:
        msg += f", not compared with the exact step (kappa > 1e8; |d_gpu - d_exact| {e_ex:.1e})"
    c = pd.cost(K, R0, t0, W, Ms, ms)
    assert abs(f["err0"] - c) <= 1e-13 * abs(c), (f["err0"], c)
    print(msg + f", err0 rel {abs(f['err0'] - c) / max(abs(c), 1e-300):.1e}")


def test_depth0_exit(api, orc):
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row("x_depth0"))
    ok, R, t, f = gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt)
    _, _, _, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    assert not ok and same_bits(R, R0) and same_bits(t, t0)
    f_o = fields(o)
    for k in OPT_KEYS + ("npts",):
        assert same_bits(f[k], f_o[k]) or (np.isnan(f[k]) and np.isnan(f_o[k])), (k, f[k], f_o[k])
    assert f["err0"] == np.inf and np.isnan(f["err"]) and f["errRW"] == -1 and f["lambda"] == 1e19
    assert f["retTypeLM"] == -1 and f["nIterLM"] == 21 and f["nIterRW"] == 0


def test_zero_iteration_exits(api, orc):
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row("x_rw0"))
    ok, R, t, f = gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt)
    assert ok and f["nIterRW"] == 0 and same_bits(R, R0) and same_bits(t, t0)
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row("x_lm0"))
    ok, R, t, f = gpu_solves(api, K, R0, t0, Ms, ms, tau, prev, opt)
    assert same_bits(R, R0) and same_bits(t, t0)
    _, _, _, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    assert ok and f["nIterLM"] == 0 == o.nIterLM and f["nIterRW"] == o.nIterRW


def ragged_batch():
    rng = np.random.default_rng(77)
    counts = [0, 1, 5, 129, 2000] + [int(x) for x in rng.integers(2, 2000, 295)]
    cams = []
    for c, n in enumerate(counts):
        K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n, seed=9000 + c, outlier_frac=0.10, rot_deg=0.2,
                                                          trans=0.01)
        prev = pc.reproj_errors(K, R0, t0, Ms, ms) if c % 2 == 0 else None
        cams.append((K, R0, t0, Ms, ms, prev))
    return cams


def test_batch_cameras_are_independent(api):
    cams = ragged_batch()
    args = [list(x) for x in zip(*cams)]
    ok, R, t, opts = api.pose_intracam_batch(*args[:5], 6.0, args[5])
    for c, (K, R0, t0, Ms, ms, prev) in enumerate(cams):
        ok1, R1, t1, o1 = api.pose_intracam(K, R0, t0, Ms, ms, 6.0, prev)
        assert ok1 == ok[c] and same_bits(R1, R[c]) and same_bits(t1, t[c]), c
        assert same_bits(opt_vector(o1), opt_vector(opts[c])) and o1.npts == opts[c].npts == len(Ms), c
    s = api.PoseSolver(0, len(cams), sum(len(c[3]) for c in cams))
    try:
        s.submit(*args[:5], 6.0, args[5])
        ok2, R2, t2, opts2, _ = s.collect()
    finally:
        s.close()
    assert np.array_equal(ok2, ok) and same_bits(R2, R) and same_bits(t2, t)
    for c in range(len(cams)):
        assert same_bits(opt_vector(opts2[c]), opt_vector(opts[c])) and opts2[c].npts == opts[c].npts, c
    print(f"{len(cams)} cameras, {sum(len(c[3]) for c in cams)} points, {int(ok.sum())} ok")
