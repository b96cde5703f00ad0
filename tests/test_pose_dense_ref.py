"""The pose edge-case table (tests/pose_edge_cases.py) on the CPU: the oracle against the reference's own
outputs (tests/golden/pose_edges_ref.npz, and the compiled reference live where it is built), and the
vectorized float64 restatement tests/pose_dense.py against the oracle."""
import numpy as np
import pytest

import pose_dense as pd
import pose_edge_cases as pc
from pose_edge_cases import OPT_KEYS, c_opt, golden_rows, opt_vector, same_bits


def test_golden_covers_the_table():
    names = {r["name"] for r, _ in golden_rows()}
    assert names == {r["name"] for r in pc.ROWS if r["n"] <= pc.GOLDEN_MAX_PTS}
    for r, g in golden_rows():  # the stored inputs are the table's
        K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(r)
        assert same_bits(Ms, g["Ms"]) and same_bits(ms, g["ms"]) and same_bits(R0, g["R0"]), r["name"]
        assert (prev is None) == (g["prev"] is None) and (prev is None or same_bits(prev, g["prev"])), r["name"]
        assert opt == g["opt"] and tau == g["tau"], r["name"]


def test_oracle_reproduces_reference_edges_bit_for_bit(orc):
    from oracle import ref
    live = ref.available()
    n = 0
    for r, g in golden_rows():
        if "ref_ok" not in g:
            continue
        a = (g["K"], g["R0"], g["t0"], g["Ms"], g["ms"], g["tau"], g["prev"])
        ok, R, t, o = orc.pose_intracam(*a, opt=c_opt(g["opt"]))
        assert ok == bool(g["ref_ok"]), r["name"]
        assert same_bits(opt_vector(o), g["ref_opt"]), (r["name"], opt_vector(o), g["ref_opt"])
        if "ref_R" in g:
            assert same_bits(R, g["ref_R"]) and same_bits(t, g["ref_t"]), r["name"]
        if live:
            ok_l, R_l, t_l, o_l = ref.intracam_estimate(*a, opt_in=g["opt"])
            assert ok_l == bool(g["ref_ok"]), r["name"]
            assert same_bits([o_l[k] for k in OPT_KEYS], g["ref_opt"]), r["name"]
            if "ref_R" in g:
                assert same_bits(R_l, g["ref_R"]) and same_bits(t_l, g["ref_t"]), r["name"]
        n += 1
    assert n >= 30


DENSE_ROWS = [r for r in pc.ROWS if not r["tie"] and r["exit"] in (None, "lm0")]


@pytest.mark.parametrize("r", DENSE_ROWS, ids=lambda r: r["name"])
def test_dense_restatement_equals_oracle(orc, r):
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(r)
    ok_d, R_d, t_d, f = pd.estimate(K, R0, t0, Ms, ms, tau, prev, opt)
    ok, R, t, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    assert ok_d == ok
    assert (f["retTypeLM"], f["npts"], f["nIterLM"], f["nIterRW"]) == (o.retTypeLM, o.npts, o.nIterLM, o.nIterRW)
    assert f["lambda_"] == o.lambda_ and f["lambda0"] == o.lambda0
    dR, dt = np.abs(R_d - R).max(), np.abs(t_d - t).max()
    print(f"{r['name']}: |dense - oracle| R {dR:.1e} t {dt:.1e}")
    assert dR <= 1e-8 and dt <= 1e-8


@pytest.mark.parametrize("r", [r for r in pc.ROWS if not r["tie"] and r["exit"] != "depth0"],
                         ids=lambda r: r["name"])
def test_tie_free_rows_keep_their_margins(r):
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(r)
    m = pd.margins(K, R0, t0, Ms, ms, tau, prev, opt)
    worst = min(m, key=lambda x: x[1], default=("none", np.inf))
    print(f"{r['name']}: {len(m)} decisions, smallest margin {worst[1]:.1e} at {worst[0]}")
    assert worst[1] >= 1e-9, worst


@pytest.mark.parametrize("name", [r["name"] for r in pc.ROWS if r["tie"]])
def test_tie_rows_are_ties(name):
    """A row marked tie does reach a decision at the rounding floor; otherwise it should be tie-free."""
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row(name))
    assert min(m for _, m in pd.margins(K, R0, t0, Ms, ms, tau, prev, opt)) < 1e-9


def test_exit_rows_take_their_exits(orc):
    """depth 0: lambda passes 1e18 before any step is accepted; maxIterLM = 0: no LM step at all."""
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row("x_depth0"))
    ok, R, t, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
    assert not ok and o.retTypeLM == -1 and o.nIterRW == 0
    assert same_bits(R, R0) and same_bits(t, t0)
    for name in ("x_rw0", "x_lm0"):
        K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row(name))
        ok, R, t, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
        assert ok and same_bits(R, R0) and same_bits(t, t0), name
    # the eps-0 rows leave through lambda > 1e18 after accepted steps; LM running out of iterations
    for name in ("x_eps0_seed9", "x_eps0_seed12"):
        K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row(name))
        ok, R, t, o = orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))
        assert not ok and o.retTypeLM == -1 and o.nIterRW >= 1, name
    K, R0, t0, Ms, ms, tau, prev, opt = pc.case_inputs(pc.row("o_lm1_rw1"))
    assert orc.pose_intracam(K, R0, t0, Ms, ms, tau, prev, opt=c_opt(opt))[3].retTypeLM == 1
