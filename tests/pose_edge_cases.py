"""The edge-case table of the per-frame pose solve (intraCamEstimate, slam/SL_IntraCamPose.cpp:626-709),
shared by tests/golden/make_pose_edges_golden.py, tests/test_pose_dense_ref.py and
tests/test_gpu_pose_edges.py.  Every row is generated from its seed, so rows too large for the golden
file are rebuilt at test time.

A row is (name, n, seed, tau, prev, opt, tie, exit):
  prev  how prevErrs is built: None (solvePnPRobust: all weights 1), "live" (|reprojection error| at
        R0/t0, as SingleSLAM passes the previous frame's errors) or one of the cut-off variants of "live"
        (see case_inputs).
  opt   (maxIterLM, maxIterRW, epsErrorChangeLM, epsParamChangeLM, epsErrorChangeRW, lambda0).
  tie   True where some decision of the trajectory sits at the rounding floor, so two correct
        implementations that sum in different orders may take different paths.  test_pose_dense_ref.py
        asserts that every row marked False keeps a decision margin of at least 1e-9.
  exit  None, or the failure / undefined-by-reference exit the row reaches: "depth0" (a point at depth
        exactly 0), "rw0" (maxIterRW = 0), "lm0" (maxIterLM = 0).
"""
import os

import numpy as np

import pose_dense
from coslam_b200 import synth
from coslam_b200.ctypes_defs import PoseOpt

DEFAULT_OPT = (100, 5, 1e-7, 1e-6, 1e-6, 1e-3)
GOLDEN_MAX_PTS = 2048  # rows with more points are compared with the oracle only


def _opt(maxIterLM=100, maxIterRW=5, epsErr=1e-7, epsParam=1e-6, epsRW=1e-6, lambda0=1e-3):
    return (maxIterLM, maxIterRW, epsErr, epsParam, epsRW, lambda0)


CASES = (
    # live: tau = 6, prevErrs, 10 % outliers, default options; 1..2 points per thread of the 128-thread CTA
    # and up to 157 (20 000 points)
    # and up to 157 (20 000 points).  Five or six points leave the 6x6 system so ill-conditioned that a
    # different summation order moves R/t by up to 1.2e-8 on some seeds; the seeds of live5 and pnp6_tau20
    # are ones where it moves them by less than 1e-9, so the 1e-8 bound measures the kernel, not the seed.
    *[(f"live{n}", n, 110 if n == 5 else 100 + n, 6.0, "live", DEFAULT_OPT, False, None)
      for n in (1, 2, 5, 6, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 2000, 4099, 20000)],
    # solvePnPRobust: no prevErrs, tau 20 and 6
    # (seed 212 would leave pnp6_tau6 three points of weight > 0: six equations for six unknowns, whose
    # solution moves by 3e-6 between summation orders; seed 211 keeps all six)
    *[(f"pnp{n}_tau{int(tau)}", n, seed, tau, None, DEFAULT_OPT, False, None)
      for n, tau, seed in ((6, 20.0, 233), (6, 6.0, 211), (500, 20.0, 720), (500, 6.0, 706),
                           (2000, 20.0, 2220), (2000, 6.0, 2206))],
    # weights at the Tukey cut-off
    ("w_eq_tau", 129, 301, 6.0, "eq_tau", DEFAULT_OPT, False, None),
    ("w_below_tau", 129, 302, 6.0, "below_tau", DEFAULT_OPT, False, None),
    ("w_negative", 129, 303, 6.0, "negative", DEFAULT_OPT, False, None),
    ("w_zeros", 129, 304, 6.0, "zeros", DEFAULT_OPT, False, None),
    ("w_all_above", 129, 305, 6.0, "all_above", DEFAULT_OPT, False, None),
    # forwarded options
    ("o_lm1_rw1", 129, 401, 6.0, "live", _opt(1, 1), False, None),
    ("o_lm2_rw1", 129, 402, 6.0, "live", _opt(2, 1), False, None),
    ("o_lm100_rw2", 129, 403, 6.0, "live", _opt(100, 2), False, None),
    ("o_lm100_rw20", 129, 404, 6.0, "live", _opt(100, 20), False, None),
    ("o_lm1_rw20", 129, 405, 6.0, "live", _opt(1, 20), False, None),
    ("o_lambda0_0", 129, 406, 6.0, "live", _opt(lambda0=0.0), False, None),
    ("o_lambda0_1e6", 129, 407, 6.0, "live", _opt(lambda0=1e6), False, None),
    ("o_epsParam_1e3", 129, 408, 6.0, "live", _opt(epsParam=1e3), False, None),
    ("o_epsErr_1e3", 129, 409, 6.0, "live", _opt(epsErr=1e3), False, None),
    # exits
    ("x_depth0", 129, 501, 6.0, None, DEFAULT_OPT, False, "depth0"),
    ("x_eps0_seed9", 300, 9, 10.0, None, _opt(100, 20, 0.0, 0.0, 0.0), True, None),
    ("x_eps0_seed12", 300, 12, 10.0, None, _opt(100, 20, 0.0, 0.0, 0.0), True, None),
    ("x_rw0", 33, 502, 6.0, "live", _opt(maxIterRW=0), False, "rw0"),
    ("x_lm0", 33, 503, 6.0, "live", _opt(maxIterLM=0), False, "lm0"),
)
FIELDS = ("name", "n", "seed", "tau", "prev", "opt", "tie", "exit")
ROWS = [dict(zip(FIELDS, c)) for c in CASES]


def row(name):
    return next(r for r in ROWS if r["name"] == name)


def reproj_errors(K, R, t, Ms, ms):
    u, v = pose_dense.project(K, R, t, Ms)
    du, dv = u - ms[:, 0], v - ms[:, 1]
    return np.sqrt(du * du + dv * dv)


def case_inputs(r):
    """(K, R0, t0, Ms, ms, tau, prevErrs or None, opt) of row r."""
    n, seed, tau = r["n"], r["seed"], r["tau"]
    if r["name"].startswith("x_eps0"):
        K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n, seed=seed)
    elif r["prev"] is None:
        K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n, seed=seed, outlier_frac=0.10)
    else:  # a tracked camera: small motion since the pose the errors were measured at
        K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n, seed=seed, outlier_frac=0.10, rot_deg=0.2,
                                                       trans=0.01)
    if r["exit"] == "depth0":
        # world frame = camera frame of R0, so R0 is exactly I and the last point's depth
        # 0*x + 0*y + 1*(-t0[2]) + t0[2] is exactly 0 (its projection is +-inf)
        Ms = Ms @ R0.T
        R0 = np.eye(3)
        Ms[-1] = (0.5, -0.25, -t0[2])
    prev = None
    if r["prev"] is not None:
        prev = reproj_errors(K, R0, t0, Ms, ms)
        k = np.arange(n)
        if r["prev"] == "eq_tau":          # weight exactly 0
            prev[k % 5 == 0] = tau
        elif r["prev"] == "below_tau":     # the largest error below tau: weight ~ 5e-32
            prev[k % 5 == 0] = np.nextafter(tau, 0.0)
        elif r["prev"] == "negative":      # the weight reads |prevErr|
            prev[k % 2 == 0] *= -1.0
        elif r["prev"] == "zeros":         # weight exactly 1
            prev[k % 3 == 0] = 0.0
        elif r["prev"] == "all_above":     # every weight 0 in the first round
            prev = tau + np.abs(prev)
    return K, R0, t0, Ms, ms, tau, prev, r["opt"]


# ---- shared by the CPU and GPU tests
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pose_edges_ref.npz")
OPT_KEYS = ("lambda", "lambda0", "err0", "err", "errRW", "retTypeLM", "nIterLM", "nIterRW")
ATTR = {"lambda": "lambda_"}


def c_opt(opt):
    o = PoseOpt.defaults()
    o.maxIterLM, o.maxIterRW, o.epsErrorChangeLM, o.epsParamChangeLM, o.epsErrorChangeRW, o.lambda0 = opt
    return o


def opt_vector(o):
    return np.array([float(getattr(o, ATTR.get(k, k))) for k in OPT_KEYS])


def golden_rows():
    d = np.load(G)
    for c in d["names"]:
        c = str(c)
        g = dict(K=d[f"{c}_K"], R0=d[f"{c}_R0"], t0=d[f"{c}_t0"], Ms=d[f"{c}_Ms"], ms=d[f"{c}_ms"],
                 tau=float(d[f"{c}_tau"]), prev=d[f"{c}_prev"] if len(d[f"{c}_prev"]) else None,
                 opt=tuple(d[f"{c}_opt_in"]))
        g["opt"] = (int(g["opt"][0]), int(g["opt"][1])) + g["opt"][2:]
        for k in ("ok", "opt", "R", "t"):
            if f"{c}_{k}" in d.files:
                g["ref_" + k] = d[f"{c}_{k}"]
        yield row(c), g


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.uint64), np.asarray(b, np.float64).view(np.uint64))
