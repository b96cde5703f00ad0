"""The whitened pose restatement (tests/pose_obscov_dense.py) against the reference's own covariance-weighted solve,
intraCamCovEstimate, compiled from the unmodified reference file into oracle/_ref/libintracam_cov_ref.so with the
harness's getProjectionCovMat handing back the caller's 2x2 covariance (oracle/ref_stubs_cov/primitives_cov.cpp).
With prevErrs = NULL and maxIterRW = 1 every Tukey weight is 1 and the two are the same algorithm (DESIGN.md 5.2):
the same LM control on J^T Sigma^-1 J and sum e^T Sigma^-1 e, which the reference forms with Sigma^-1 and the
restatement as (L J)^T (L J) and |L e|^2.  Compared as test_gpu_pose_edges.py compares the kernel with the
oracle: ok and retTypeLM equal, R and t within 1e-8; where no decision lies within 1e-7 of its threshold also the
counts and lambda equal bit for bit and the costs within 1e-9 relative."""
import math

import numpy as np
import pytest

import pose_dense as pd
import pose_obscov_dense as od
from coslam_b200 import synth
from oracle import ref_cov

pytestmark = pytest.mark.skipif(not ref_cov.available(), reason="oracle/_ref/libintracam_cov_ref.so is not built")

TAU = 10.0
ONE_ROUND = (100, 1) + pd.DEFAULT_OPT[2:]
# (name, points, outlier fraction, options): frame-sized and small point counts, outliers that no weight removes,
# a large starting lambda that the solve walks down over 5 to 7 accepted steps with the stop left to the cost-change
# test, and a cap on the LM iterations.  Not here: a large lambda with the default epsParamChangeLM, which stops on a
# small step well short of the minimum; err is then the cost of the trial before it, a pose the reference does not
# return, so its difference cannot be bounded from the outputs
ROWS = [
    ("n192", 192, 0.0, ONE_ROUND),
    ("n192_outliers", 192, 0.05, ONE_ROUND),
    ("n8", 8, 0.0, ONE_ROUND),
    ("n30", 30, 0.0, ONE_ROUND),
    ("n1000", 1000, 0.0, ONE_ROUND),
    ("lambda1e8_errstop", 192, 0.0, (100, 1, 1e-4, 1e-12, 1e-6, 1e8)),
    ("lambda1e9_errstop", 192, 0.0, (100, 1, 1e-4, 1e-12, 1e-6, 1e9)),
    ("lambda1e8_lm2", 192, 0.0, (2, 1, 1e-7, 1e-6, 1e-6, 1e8)),
]


def _case(seed, n, outliers):
    K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(n, seed=seed, noise_px=0.0, outlier_frac=outliers, rot_deg=2.0,
                                                   trans=0.1)
    rng = np.random.default_rng(seed)
    covx, S = od.random_covx(n, rng)
    return K, R0, t0, Ms, ms + od.draw_noise(S, rng), covx


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("row", ROWS, ids=lambda r: r[0])
def test_restatement_equals_reference_cov_estimate(row, seed):
    name, n, outliers, opt = row
    K, R0, t0, Ms, ms, covx = _case(1000 * seed + n, n, outliers)
    ok_r, R_r, t_r, o = ref_cov.intracam_cov_estimate(K, R0, t0, Ms, ms, covx, TAU, None, opt)
    ok, R, t, f = od.estimate(K, R0, t0, Ms, ms, TAU, None, opt, covx)
    margin = min((m for _, m in od.margins(K, R0, t0, Ms, ms, TAU, None, opt, covx)), default=math.inf)
    assert ok == ok_r and f["retTypeLM"] == o["retTypeLM"]
    dR, dt = np.abs(R - R_r).max(), np.abs(t - t_r).max()
    print(f"{name} seed {seed}: nIterLM {f['nIterLM']}, smallest margin {margin:.1e}, |dense - reference| R {dR:.1e} "
          f"t {dt:.1e}")
    assert dR <= 1e-8 and dt <= 1e-8
    if margin < 1e-7:
        return
    assert (f["nIterLM"], f["nIterRW"]) == (o["nIterLM"], o["nIterRW"])
    assert f["lambda_"] == o["lambda"] and f["lambda0"] == o["lambda0"]
    assert f["err0"] == o["err0"] or abs(f["err0"] - o["err0"]) <= 1e-9 * abs(o["err0"]) + 1e-12
    # err and errRW are the cost at the returned pose.  The two solves form J^T Sigma^-1 J in different operation
    # orders, so their poses differ by ~1e-10 (not the 1e-12 of two summation orders), and a pose short of the minimum
    # (the LM-iteration cap) has a cost that moves with it: the bound adds twice the restatement's cost difference
    # between the two returned poses
    L, W = od.factors(covx), np.ones(n)
    moved = abs(od.cost(K, R, t, W, Ms, ms, L) - od.cost(K, R_r, t_r, W, Ms, ms, L))
    for k in ("err", "errRW"):
        assert f[k] == o[k] or abs(f[k] - o[k]) <= 1e-9 * abs(o[k]) + 2 * moved + 1e-12, (k, f[k], o[k], moved)


def test_reference_cov_estimate_with_identity_is_intracam_estimate():
    """The harness's primitives: with Sigma = I, intraCamCovEstimate's cost and step are intraCamEstimate's (one
    round, unit weights), so the two reference solves agree to rounding."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref/libintracam_ref.so is not built")
    K, R0, t0, Ms, ms, _, _ = synth.make_pose_case(192, seed=9)
    ok_c, R_c, t_c, o_c = ref_cov.intracam_cov_estimate(K, R0, t0, Ms, ms, od.identity(192), TAU, None, ONE_ROUND)
    ok, R, t, o = ref.intracam_estimate(K, R0, t0, Ms, ms, TAU, None, ONE_ROUND)
    assert ok_c == ok and o_c["nIterLM"] == o["nIterLM"] and o_c["lambda"] == o["lambda"]
    assert np.abs(R_c - R).max() <= 1e-10 and np.abs(t_c - t).max() <= 1e-10
    assert o_c["err"] == pytest.approx(o["err"], rel=1e-12)
