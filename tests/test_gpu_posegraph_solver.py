"""The pose-graph solver handle (cosl_posegraph_solver): the synchronous calls' results bit for bit, chain and
general requests on one handle whose buffers grow and are reused, submit that does not wait and copies its
inputs, the synchronous calls' error codes, the state rules, and handles on threads beside a KLT group."""
import ctypes as C
import os
import re
import threading
import time

import numpy as np
import pytest

from coslam_b200.synth import ImageSequence, make_merge_graph, make_pose_chains, make_pose_graph, scale_columns

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHAIN_KEYS = ("chain_off", "fixed", "R", "t", "eR", "et")
GRAPH_KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et", "scale_col", "n_scale")
E_INVALID, E_NUMERIC, E_STATE = -1, -4, -6


def _golden_chains():
    z = np.load(os.path.join(HERE, "golden", "posegraph_ref.npz"))
    out = []
    for i in range(int(z["n_chain_cases"])):
        n = len(z[f"c{i}_fixed"])
        eR, et = np.zeros((n, 3, 3)), np.zeros((n, 3))
        eR[:n - 1], et[:n - 1] = z[f"c{i}_eR_list"], z[f"c{i}_et_list"]
        out.append(dict(chain_off=np.array([0, n], np.int32), fixed=z[f"c{i}_fixed"], R=z[f"c{i}_R"],
                        t=z[f"c{i}_t"], eR=eR, et=et))
    return out


def _merge_golden():
    z = np.load(os.path.join(HERE, "golden", "posegraph_merge_ref.npz"))
    out = []
    for i in range(int(z["n_cases"])):
        c = {k: z[f"c{i}_{k}"] for k in ("fixed", "R", "t", "id1", "id2", "eR", "et", "scale_id")}
        c["scale_col"], c["n_scale"] = scale_columns(c["scale_id"])
        out.append(c)
    return out


def _chain_cases():
    """Small first, then the 8 x 4 000 case (the buffers grow), then smaller ones (they are reused)."""
    return (_golden_chains()[:1]
            + [make_pose_chains([37], key_every=5, seed=37)]
            + [make_pose_chains([4000] * 8, key_every=20, seed=5, shift=0.05)]
            + _golden_chains()[1:]
            + [make_pose_chains([300, 1, 2, 77, 0, 513], key_every=9, seed=893),
               make_pose_chains([130, 130], key_every=11, lead_free=4, seed=260),
               make_pose_chains([64], key_every=1, seed=64),
               make_pose_chains([4, 150, 150, 150], key_every=10, seed=9)])


def _graph_cases():
    return ([make_merge_graph(100, 4, seed=400, n_constraints=2, n_scale_ids=1, noise=0.01),
             make_merge_graph(30, 13, seed=390, n_constraints=3, n_scale_ids=2, noise=0.01),
             make_pose_graph(300, seed=300, fixed_every=50, loops=4, parallel=3, reverse=3, fixed_pairs=1,
                             n_scale=2, uncertain=4),
             make_pose_graph(90, seed=90, components=2, loops=2, reverse=2, n_scale=2, uncertain=3),
             make_pose_graph(3, seed=3),
             # no free node: answered on the host by the synchronous call
             dict(make_pose_graph(12, seed=12), fixed=np.ones(12, np.uint8))]
            + _merge_golden())


def _same_bits(a, b):
    assert a.shape == b.shape
    assert np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


def _sync_chains(api, g):
    return api.posegraph_spread_chains(*(g[k] for k in CHAIN_KEYS))


def _sync_graph(api, g):
    return api.posegraph_solve(*(g[k] for k in GRAPH_KEYS))


def _check_chain(api, s, g, ref=None):
    ref = ref if ref is not None else _sync_chains(api, g)
    s.submit_chains(*(g[k] for k in CHAIN_KEYS))
    nR, nt, scale, ms = s.collect()
    _same_bits(nR, ref[0])
    _same_bits(nt, ref[1])
    assert scale is None
    assert np.isfinite(ms) and ms > 0.0
    return ms


def _check_graph(api, s, g, ref=None):
    ref = ref if ref is not None else _sync_graph(api, g)
    s.submit(*(g[k] for k in GRAPH_KEYS))
    nR, nt, scale, ms = s.collect()
    for x, y in zip((nR, nt, scale), ref):
        _same_bits(x, y)
    # a graph without free nodes runs nothing on the device
    assert np.isfinite(ms) and (ms > 0.0 if (np.asarray(g["fixed"]) == 0).any() else ms >= 0.0)
    return ms


def test_chain_parity_one_handle(api):
    s = api.PoseGraphSolver(0)
    for g in _chain_cases():
        _check_chain(api, s, g)
    s.close()


def test_general_parity_alternating_with_chains(api):
    s = api.PoseGraphSolver(0)
    chains = _chain_cases()
    for i, g in enumerate(_graph_cases()):
        _check_graph(api, s, g)
        _check_chain(api, s, chains[i % len(chains)])
    s.close()


def test_empty_chain_table_is_in_flight(api):
    s = api.PoseGraphSolver(0)
    for off in ([0], [0, 0, 0]):
        s.submit_chains(off, np.zeros(0, np.uint8), *[np.zeros((0, 3, 3)), np.zeros((0, 3))] * 2)
        with pytest.raises(api.CoslError, match="error -6"):
            s.submit_chains(off, np.zeros(0, np.uint8), *[np.zeros((0, 3, 3)), np.zeros((0, 3))] * 2)
        nR, nt, scale, ms = s.collect()
        assert nR.shape == (0, 3, 3) and nt.shape == (0, 3) and scale is None and ms >= 0.0
    s.close()


def _sleep_on(stream_ptr):
    """Queue a busy kernel of 1e9 SM cycles (0.5 s or more on an H100, whose SM clock is at most 1.98 GHz) on
    the handle's stream."""
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(stream_ptr)):
        torch.cuda._sleep(1_000_000_000)


def _own(g, keys, dtypes):
    return {k: (np.array(g[k], dtypes[k]) if k in dtypes else g[k]) for k in keys}


CHAIN_DT = dict(chain_off=np.int32, fixed=np.uint8, R=np.float64, t=np.float64, eR=np.float64, et=np.float64)
GRAPH_DT = dict(fixed=np.uint8, R=np.float64, t=np.float64, id1=np.int32, id2=np.int32, eR=np.float64,
                et=np.float64, scale_col=np.int32)


def _scribble(arrs):
    for a in arrs.values():
        if isinstance(a, np.ndarray):
            a.fill(np.iinfo(a.dtype).max if a.dtype.kind in "iu" else np.nan)


def test_submit_does_not_wait_and_copies_its_inputs(api):
    s = api.PoseGraphSolver(0)
    gc = _own(make_pose_chains([4000] * 8, key_every=20, seed=5, shift=0.05), CHAIN_KEYS, CHAIN_DT)
    ref = _sync_chains(api, gc)
    _sleep_on(s.stream())
    t0 = time.perf_counter()
    s.submit_chains(*(gc[k] for k in CHAIN_KEYS))
    t_submit = time.perf_counter() - t0
    assert not s.done()
    _scribble(gc)
    nR, nt, _, ms = s.collect()
    assert t_submit < 0.1 < time.perf_counter() - t0, t_submit
    _same_bits(nR, ref[0])
    _same_bits(nt, ref[1])
    assert 0.0 < ms < 100.0  # the copies and the kernel, not the sleep queued ahead of them

    gg = _own(make_merge_graph(30, 13, seed=390, n_constraints=3, n_scale_ids=2, noise=0.01), GRAPH_KEYS, GRAPH_DT)
    ref = _sync_graph(api, gg)
    _sleep_on(s.stream())
    s.submit(*(gg[k] for k in GRAPH_KEYS))
    assert not s.done()
    _scribble(gg)
    got = s.collect()
    for x, y in zip(got[:3], ref):
        _same_bits(x, y)
    s.close()


def _code(fn):
    """(code, message without the function name) of a call; (0, '') when it succeeds"""
    from coslam_b200 import api
    try:
        fn()
        return 0, ""
    except api.CoslError as e:
        m = re.match(r"coslam_b200 error (-?\d+): [a-z_]+: (.*)$", str(e), re.S)
        assert m, str(e)
        return int(m.group(1)), m.group(2)


def _handle_code(s, submit):
    """the error of a request at submit or, failing that, at collect; where it came"""
    code, msg = _code(submit)
    if code:
        return code, msg, "submit"
    code, msg = _code(s.collect)
    return code, msg, "collect"


def _graph_error_cases():
    """the malformed requests of test_gpu_posegraph_general.py::test_error_cases"""
    g = make_pose_graph(10, seed=1, n_scale=1, uncertain=1)
    base = {k: (np.copy(g[k]) if isinstance(g[k], np.ndarray) else g[k]) for k in GRAPH_KEYS}
    cases = []

    def case(name, where, **over):
        c = dict(base)
        c.update(over)
        cases.append((name, where, c))

    id1 = np.copy(g["id1"])
    id1[0] = 10
    case("index", "submit", id1=id1)
    id2 = np.copy(g["id2"])
    id2[1] = g["id1"][1]
    case("self-loop", "submit", id2=id2)
    sc = np.copy(g["scale_col"])
    sc[sc >= 0] = 1
    case("scale column", "submit", scale_col=sc)
    case("column without a row", "submit", n_scale=2)
    case("no fixed node", "submit", fixed=np.zeros_like(g["fixed"]))
    two = make_pose_graph(20, seed=2, components=2)
    fx = np.copy(two["fixed"])
    fx[10] = 0
    cases.append(("component without a fixed node", "submit", dict(two, fixed=fx)))
    et = np.copy(g["et"])
    et[g["scale_col"] >= 0] = 0.0
    case("singular", "collect", et=et)
    R = np.copy(g["R"])
    R[0, 0, 0] = np.nan
    case("non-finite", "collect", R=R)
    return cases, base


def test_errors_match_the_synchronous_calls(api):
    s = api.PoseGraphSolver(0)
    cases, good = _graph_error_cases()
    good_ref = _sync_graph(api, good)
    for name, where, c in cases:
        want = _code(lambda: _sync_graph(api, c))
        assert want[0] in (E_INVALID, E_NUMERIC), (name, want)
        got = _handle_code(s, lambda: s.submit(*(c[k] for k in GRAPH_KEYS)))
        assert got == want + (where,), name
        _check_graph(api, s, good, good_ref)
    # a chain without a fixed node: only the kernel sees it
    bad = make_pose_chains([8, 6], seed=2, fixed_masks=[[1, 0, 0, 0, 1, 0, 0, 0], [0] * 6])
    want = _code(lambda: _sync_chains(api, bad))
    assert want[0] == E_INVALID and "no fixed node" in want[1]
    assert _handle_code(s, lambda: s.submit_chains(*(bad[k] for k in CHAIN_KEYS))) == want + ("collect",)
    # a malformed chain table
    off = np.array([0, 5, 3], np.int32)
    arrs = (np.zeros(3, np.uint8), np.zeros((3, 3, 3)), np.zeros((3, 3)), np.zeros((3, 3, 3)), np.zeros((3, 3)))
    want = _code(lambda: api.posegraph_spread_chains(off, *arrs))
    assert want[0] == E_INVALID and "non-decreasing" in want[1]
    assert _handle_code(s, lambda: s.submit_chains(off, *arrs)) == want + ("submit",)
    ok = make_pose_chains([37, 120, 5], key_every=6, seed=4, shift=0.1)
    _check_chain(api, s, ok)
    _check_graph(api, s, good, good_ref)
    s.close()


def test_state_rules(api):
    L = api.LIB
    g = make_pose_chains([4000] * 2, key_every=20, seed=7)
    gg = make_pose_graph(40, seed=40, fixed_every=9, loops=3, n_scale=1, uncertain=2)
    ref = _sync_chains(api, g)
    s = api.PoseGraphSolver(0)
    with pytest.raises(api.CoslError, match="error -6"):
        s.done()
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    _sleep_on(s.stream())
    s.submit_chains(*(g[k] for k in CHAIN_KEYS))
    # a second request of either kind
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit_chains(*(g[k] for k in CHAIN_KEYS))
    with pytest.raises(api.CoslError, match="error -6"):
        s.submit(*(gg[k] for k in GRAPH_KEYS))
    # query reaches done without collect
    t0, polls = time.perf_counter(), 0
    while not s.done():
        polls += 1
        assert time.perf_counter() - t0 < 30.0, "the request did not finish"
        time.sleep(0.01)
    assert polls > 0
    nR, nt, _, _ = s.collect()
    _same_bits(nR, ref[0])
    _same_bits(nt, ref[1])
    with pytest.raises(api.CoslError, match="error -6"):
        s.collect()
    assert L.cosl_posegraph_solver_query(s.h, C.byref(C.c_int(0))) == E_STATE
    # destroy waits for a request in flight
    _sleep_on(s.stream())
    s.submit(*(gg[k] for k in GRAPH_KEYS))
    t0 = time.perf_counter()
    assert L.cosl_posegraph_solver_destroy(s.h) == 0
    assert time.perf_counter() - t0 > 0.25
    s.h = None


def _solve_many(api, jobs, n, out, key, errors):
    try:
        s = api.PoseGraphSolver(0)
        res = []
        for i in range(n):
            kind, g = jobs[i % len(jobs)]
            if kind == "chains":
                s.submit_chains(*(g[k] for k in CHAIN_KEYS))
            else:
                s.submit(*(g[k] for k in GRAPH_KEYS))
            res.append(s.collect()[:3])
        s.close()
        out[key] = res
    except Exception as e:  # noqa: BLE001  (reported by the main thread)
        errors.append(e)


def test_two_handles_on_two_threads_beside_klt(api):
    from coslam_b200.ctypes_defs import KltConfig
    jobs = {"a": [("chains", make_pose_chains([4000] * 8, key_every=20, seed=5, shift=0.05)),
                  ("graph", make_merge_graph(100, 4, seed=400, n_constraints=2, n_scale_ids=1, noise=0.01))],
            "b": [("graph", make_merge_graph(30, 13, seed=390, n_constraints=3, n_scale_ids=2, noise=0.01)),
                  ("chains", make_pose_chains([4, 150, 150, 150], key_every=10, seed=9))]}
    refs = {k: [(_sync_chains(api, g) + (None,)) if kind == "chains" else _sync_graph(api, g) for kind, g in v]
            for k, v in jobs.items()}
    W, H = 1280, 720
    seqs = [ImageSequence(H, W, 500 + c, n_frames=6) for c in range(4)]
    frames = [[seqs[c].frames[k] for c in range(4)] for k in range(6)]
    grp = api.KltGroup(KltConfig.coslam_live(with_gain=True), 4, W, H, 6, 50, 40)
    grp.first(frames[0])
    out, errors = {}, []
    n = 12
    threads = [threading.Thread(target=_solve_many, args=(api, jobs[k], n, out, k, errors)) for k in jobs]
    for t in threads:
        t.start()
    klt_frames = 0
    while any(t.is_alive() for t in threads) or klt_frames < 4:
        grp.submit(frames[1 + klt_frames % 5])
        grp.collect()
        klt_frames += 1
    for t in threads:
        t.join()
    grp.close()
    assert not errors, errors
    for k in jobs:
        assert len(out[k]) == n
        for i, got in enumerate(out[k]):
            for x, y in zip(got, refs[k][i % len(jobs[k])]):
                if y is None:
                    assert x is None
                else:
                    _same_bits(x, y)
