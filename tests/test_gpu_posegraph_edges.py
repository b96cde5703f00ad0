"""The pose-graph solvers at their edge shapes against the dense float64 least-squares reference
tests/posegraph_dense.py (pinned to the compiled reference's vectors by tests/test_posegraph_dense_ref.py).

Chain kernel (posegraph_chain_kernel, cosl_posegraph_spread_chains): 256 threads, each owns a chunk of
per = ceil(n / 256) nodes.  Lengths 1 .. 4096 (per = 1, 2, 3, 4, 16) with fixed nodes on chunk starts, on
chunk ends, filling whole chunks, only at one end (one run crossing every chunk), at both ends (one run
spanning every chunk), in adjacent pairs across chunk boundaries, alternating, and inside the chain (free
leading and trailing runs), all in one launch per mask family.

General solve (cosl_posegraph_solve and one PoseGraphSolver submit / collect, bit for bit the same):
the tile plan has mf = 2 nF + ceil(nScale / 6) units of 6 rows, blocks of BA_BLK_CAMS = 10 units (ba_plan.h):
mf <= 10 is one block and <= 20 two (the single-CTA ba_tile_two), more the task kernel.  Scale columns
>= 6 live in a second (third) scale unit whose unused rows are padding.  A pure chain of >= 34 free nodes
is band-like with a nested dissection (two-sided elimination from 31).  Metamorphic checks: node and edge
permutations, edge reversals and a unit change must not move the result.

Degenerate projections: M of rank 2, 1 and 0 (the nearest rotation is unique only for rank 2), and M with
det < 0, each in the identity frame (exact zero columns) and in generic frames (singular values that
vanish without being exact zeros).  Where the projection ties, the kernel's R must be a proper rotation
exactly as far from M as the reference's.

Tolerances: 1e-9 absolute on R and t (O(1) values) for general graphs.  Chains: 1000 n eps (times
max(1, |t|) on t): the kernel composes up to n - 1 rigid transforms and the reference eliminates n nodes,
so both drift by O(n eps); at n = 4096 a sequential float64 composition differs from the reference by
1.6e-11 on R, against a tolerance of 9.1e-10."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import posegraph_dense as dense
from coslam_b200.synth import make_pose_chains

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
TOL = 1e-9
GAP = 1e-6  # sv[1] + sv[2] above this: the projection is unique and the matrices are compared
GRAPH_KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et", "scale_col", "n_scale")
CHAIN_KEYS = ("chain_off", "fixed", "R", "t", "eR", "et")


def _same_bits(a, b):
    assert a.shape == b.shape
    assert np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


def _check(nR, nt, ref, fixed, R, t, tol_R, tol_t):
    """nR / nt against the reference; returns the number of free nodes whose projection ties."""
    fx = np.asarray(fixed).astype(bool)
    _same_bits(nR[fx], R[fx])
    _same_bits(nt[fx], t[fx])
    gap = ref["sv"][:, 1] + ref["sv"][:, 2]
    uniq, tie = ~fx & (gap > GAP), ~fx & (gap <= GAP)
    tol_R = np.broadcast_to(tol_R, fx.shape)
    assert np.all(np.abs(nR[uniq] - ref["newR"][uniq]).max(axis=(1, 2)) < tol_R[uniq])
    if tie.any():
        Rt = nR[tie]
        assert np.abs(np.einsum("nji,njk->nik", Rt, Rt) - np.eye(3)).max() < 1e-12
        assert np.all(np.linalg.det(Rt) > 0)
        dist = np.linalg.norm(Rt - ref["M"][tie], axis=(1, 2))
        assert np.abs(dist - dense.min_distance(ref["M"][tie], ref["sv"][tie])).max() < 1e-12
    assert np.all(np.abs(nt - ref["newt"]).max(axis=1) < np.broadcast_to(tol_t, fx.shape))
    return int(tie.sum())


# ---------------------------------------------------------------------------------------------------------
# chain kernel

LENGTHS = (1, 2, 255, 256, 257, 511, 512, 513, 769, 4096)


def _mask(n, kind, rng):
    per = -(-n // 256)
    k = np.arange(n)
    m = {
        "chunk_starts": k % per == 0,
        "chunk_ends": k % per == per - 1,
        "whole_chunks": (k // per) % 3 == 1,
        "first_only": k == 0,
        "last_only": k == n - 1,
        "both_ends": (k == 0) | (k == n - 1),
        "pairs_across_chunks": (k % per == per - 1) & ((k // per) % 5 == 2) | (k % per == 0) & ((k // per) % 5 == 3),
        "adjacent_pairs": k % 41 >= 39,
        "alternating": k % 2 == 1,
        "inner": (k == n // 3) | (k == (2 * n) // 3) | (k == n // 2),
        "random": rng.random(n) < 0.03,
    }[kind].astype(np.uint8)
    if not m.any():  # a chain needs a fixed node
        m[n // 2] = 1
    return m


@pytest.mark.parametrize("kind", ["chunk_starts", "chunk_ends", "whole_chunks", "first_only", "last_only",
                                  "both_ends", "pairs_across_chunks", "adjacent_pairs", "alternating", "inner",
                                  "random"])
def test_chains_at_chunk_boundaries(api, kind):
    rng = np.random.default_rng(len(kind))
    masks = [_mask(n, kind, rng) for n in LENGTHS]
    g = make_pose_chains(list(LENGTHS), seed=len(kind), shift=0.05, fixed_masks=masks)
    nR, nt = api.posegraph_spread_chains(*(g[k] for k in CHAIN_KEYS))
    ref = dense.solve_chains(*(g[k] for k in CHAIN_KEYS))
    n_of = np.repeat(np.asarray(LENGTHS), LENGTHS)
    tol_R = np.maximum(1e-12, 1000 * n_of * EPS)
    _check(nR, nt, ref, g["fixed"], g["R"], g["t"], tol_R, tol_R * np.maximum(1.0, np.abs(g["t"]).max()))


# ---------------------------------------------------------------------------------------------------------
# general solve


def _units(g):
    """mf and the bandwidth of the unit adjacency pg_prepare builds (units 2f, 2f+1 per free node f, unit
    2 nF + c // 6 per scale column c)."""
    fx = g["fixed"].astype(bool)
    free_of = np.cumsum(~fx) - 1
    nF = int((~fx).sum())
    mf = 2 * nF + -(-int(g["n_scale"]) // 6)
    bw = 0
    for i, j, c in zip(g["id1"], g["id2"], g["scale_col"]):
        if not fx[i] and not fx[j]:
            bw = max(bw, 2 * abs(int(free_of[i]) - int(free_of[j])))
        for k in (i, j):
            if c >= 0 and not fx[k]:
                bw = max(bw, abs(2 * nF + c // 6 - (2 * int(free_of[k]) + 1)))
    return mf, bw


def _plan_shape(mf, bw):
    """ba_make_plan's ordering decision (ba_plan.h): band-like, and the nested-dissection depth."""
    sepw = bw + 1
    band = mf >= 4 * sepw and mf > 6 * 10
    depth, best = 0, 1e30
    if band:
        sep_blocks = -(-sepw // 10)
        for d in range(6):
            interior = (mf - (2 ** d - 1) * sepw) / 2 ** d
            if interior < 20:
                break
            path = interior / 10 / 2.0 + d * sep_blocks
            if path < best - 0.75:
                best, depth = path, d
    return band, depth


def _rot(rng, scale):
    return Rotation.from_rotvec(rng.normal(size=3) * scale).as_matrix()


def _graph(n_free, n_fixed, n_scale=0, seed=0, loops=2, lonely=False, isolated=False, noise=0.02):
    """A chain over n_free + n_fixed nodes (fixed ones spread along it, the first included), `loops` loop
    closures, two uncertain edges per scale column (scale 0.5 + 0.25 c); with `lonely` the last column's
    edges both join a fixed node to the same free node; with `isolated` the last free node is joined to
    two fixed nodes only.  Edges are measured from true poses with `noise`; fixed nodes are then moved."""
    rng = np.random.default_rng(seed)
    n = n_free + n_fixed
    chain = n - 1 if isolated else n
    fixed = np.zeros(n, np.uint8)
    fixed[np.round(np.linspace(0, chain - 1, n_fixed)).astype(int)] = 1
    Rt, tt = [_rot(rng, 1.0)], [rng.normal(size=3)]
    for _ in range(n - 1):
        Rt.append(_rot(rng, 0.05) @ Rt[-1])
        tt.append(tt[-1] + rng.normal(size=3) * 0.1)
    Rt, tt = np.array(Rt), np.array(tt)
    id1, id2, eR, et, col = [], [], [], [], []

    def edge(a, b, c=-1):
        R = Rt[b] @ Rt[a].T
        tr = tt[b] - R @ tt[a]
        if c >= 0:
            tr = tr / (0.5 + 0.25 * c)
        id1.append(a)
        id2.append(b)
        eR.append(_rot(rng, noise) @ R)
        et.append(tr + rng.normal(size=3) * noise)
        col.append(c)

    for k in range(chain - 1):
        edge(k, k + 1)
    fx_nodes = np.flatnonzero(fixed)
    if isolated:
        edge(int(fx_nodes[0]), n - 1)
        edge(n - 1, int(fx_nodes[-1]))
    for _ in range(loops):
        a, b = sorted(rng.choice(chain, 2, replace=False))
        if not (fixed[a] and fixed[b]):
            edge(int(a), int(b))
    free = np.flatnonzero(fixed[:chain] == 0)  # the isolated node keeps its two edges only
    for c in range(n_scale):
        if lonely and c == n_scale - 1:
            f = int(free[len(free) // 2])
            edge(int(fx_nodes[0]), f, c)
            edge(f, int(fx_nodes[-1]), c)
            continue
        for _ in range(2):
            a, b = rng.choice(chain, 2, replace=False)
            if fixed[a] and fixed[b]:
                b = int(rng.choice(free))
            edge(int(a), int(b), c)
    R, t = Rt.copy(), tt.copy()
    for k in fx_nodes:
        R[k] = _rot(rng, noise) @ R[k]
        t[k] += rng.normal(size=3) * noise
    return dict(fixed=fixed, R=R, t=t, id1=np.asarray(id1, np.int32), id2=np.asarray(id2, np.int32),
                eR=np.asarray(eR), et=np.asarray(et), scale_col=np.asarray(col, np.int32), n_scale=n_scale)


def _solve_both(api, g):
    """posegraph_solve and one PoseGraphSolver submit / collect: the same bits."""
    nR, nt, s = api.posegraph_solve(*(g[k] for k in GRAPH_KEYS))
    h = api.PoseGraphSolver(0)
    try:
        h.submit(*(g[k] for k in GRAPH_KEYS))
        hR, ht, hs, _ = h.collect()
    finally:
        h.close()
    _same_bits(nR, hR)
    _same_bits(nt, ht)
    _same_bits(s, hs)
    return nR, nt, s


def _check_graph(api, g, tol=TOL):
    nR, nt, s = _solve_both(api, g)
    ref = dense.solve(*(g[k] for k in GRAPH_KEYS))
    ties = _check(nR, nt, ref, g["fixed"], g["R"], g["t"], tol, tol)
    assert np.all(np.abs(s - ref["scale"]) <= tol * np.abs(ref["scale"]))
    return (nR, nt, s), ties


@pytest.mark.parametrize("n_free,n_scale,mf,blocks", [
    (4, 7, 10, 1),     # one block; scale columns 6.. in a second scale unit, 5 padding rows
    (5, 6, 11, 2),     # one full scale unit; two blocks (ba_tile_two)
    (9, 12, 20, 2),    # two full scale units
    (10, 5, 21, 3),    # three blocks: the task kernel; one padding row
    (14, 7, 30, 3),
    (14, 13, 31, 4),   # three scale units, the last with 5 padding rows
])
def test_scale_units_and_tile_plan_boundaries(api, n_free, n_scale, mf, blocks):
    g = _graph(n_free, 3, n_scale, seed=100 * n_free + n_scale, loops=2, lonely=True, isolated=True)
    m, bw = _units(g)
    assert m == mf and not _plan_shape(m, bw)[0] and -(-m // 10) == blocks
    lonely = g["scale_col"] == n_scale - 1
    touched = {int(k) for k in np.r_[g["id1"][lonely], g["id2"][lonely]] if not g["fixed"][k]}
    assert len(touched) == 1
    iso = len(g["fixed"]) - 1
    at_iso = (g["id1"] == iso) | (g["id2"] == iso)
    others = g["id1"][at_iso] + g["id2"][at_iso] - iso
    assert not g["fixed"][iso] and at_iso.sum() == 2 and np.all(g["fixed"][others])
    _check_graph(api, g)


def test_hub_node_with_300_edges(api):
    """One free hub joined to 150 leaves by two edges each (one in each direction), some leaves fixed,
    uncertain edges on two scale columns: every unit links to the hub's, so the plan keeps the natural
    order over ceil(mf / 10) blocks."""
    rng = np.random.default_rng(11)
    nl = 150
    n = nl + 2
    Rt = np.array([_rot(rng, 1.0) for _ in range(n)])
    tt = rng.normal(size=(n, 3))
    fixed = np.zeros(n, np.uint8)
    fixed[0] = 1
    fixed[2::5] = 1
    id1, id2, eR, et, col = [0], [1], [Rt[1] @ Rt[0].T], [tt[1] - Rt[1] @ Rt[0].T @ tt[0]], [-1]
    for q, leaf in enumerate(range(2, n)):
        for a, b in ((1, leaf), (leaf, 1)):
            R = Rt[b] @ Rt[a].T
            c = q % 2 if q < 8 and a == 1 else -1
            tr = (tt[b] - R @ tt[a]) / (1.0 if c < 0 else 0.5 + 0.25 * c)
            id1.append(a)
            id2.append(b)
            eR.append(_rot(rng, 0.02) @ R)
            et.append(tr + rng.normal(size=3) * 0.02)
            col.append(c)
    g = dict(fixed=fixed, R=Rt, t=tt, id1=np.asarray(id1, np.int32), id2=np.asarray(id2, np.int32),
             eR=np.asarray(eR), et=np.asarray(et), scale_col=np.asarray(col, np.int32), n_scale=2)
    assert np.sum((g["id1"] == 1) | (g["id2"] == 1)) == 301
    mf, bw = _units(g)
    assert not _plan_shape(mf, bw)[0] and mf > 200
    _check_graph(api, g)


@pytest.mark.parametrize("n_free,depth", [(31, 0), (33, 0), (34, 1), (37, 1), (100, 2)])
def test_band_like_chain_plans(api, n_free, depth):
    """A pure chain: units 2f and 2f + 2 are neighbours, bandwidth 2.  From mf > 60 the plan is band-like
    (two-sided elimination); from 34 free nodes (mf = 68) it is cut by nested dissection."""
    g = _graph(n_free, 2, seed=n_free, loops=0)
    mf, bw = _units(g)
    assert mf == 2 * n_free and bw == 2 and _plan_shape(mf, bw) == (True, depth)
    _check_graph(api, g)


def _metamorphic_base():
    return _graph(30, 4, n_scale=7, seed=77, loops=4, lonely=True, isolated=True)


def test_relabeling_nodes_and_edges_does_not_move_the_result(api):
    g = _metamorphic_base()
    (R0, t0, s0), _ = _check_graph(api, g)
    rng = np.random.default_rng(5)
    n, ne = len(g["fixed"]), len(g["id1"])
    p, q = rng.permutation(n), rng.permutation(ne)  # node k -> p[k]; edge e of h is edge q[e] of g
    h = dict(g)
    for k in ("fixed", "R", "t"):
        h[k] = np.empty_like(g[k])
        h[k][p] = g[k]
    h["id1"], h["id2"] = p[g["id1"][q]].astype(np.int32), p[g["id2"][q]].astype(np.int32)
    h["eR"], h["et"], h["scale_col"] = g["eR"][q], g["et"][q], g["scale_col"][q]
    (R1, t1, s1), _ = _check_graph(api, h)
    assert np.abs(R1[p] - R0).max() < 1e-10 and np.abs(t1[p] - t0).max() < 1e-10
    assert np.all(np.abs(s1 - s0) <= 1e-10 * np.abs(s0))


def test_reversing_edges_does_not_move_the_result(api):
    g = _metamorphic_base()
    (R0, t0, s0), _ = _check_graph(api, g)
    rev = np.random.default_rng(6).random(len(g["id1"])) < 0.5
    assert rev.sum() > 5 and (rev & (g["scale_col"] >= 0)).any()
    h = dict(g, id1=np.where(rev, g["id2"], g["id1"]).astype(np.int32),
             id2=np.where(rev, g["id1"], g["id2"]).astype(np.int32))
    RT = np.swapaxes(g["eR"], 1, 2)
    h["eR"] = np.where(rev[:, None, None], RT, g["eR"])
    h["et"] = np.where(rev[:, None], -np.einsum("eab,eb->ea", RT, g["et"]), g["et"])
    (R1, t1, s1), _ = _check_graph(api, h)
    assert np.abs(R1 - R0).max() < 1e-10 and np.abs(t1 - t0).max() < 1e-10
    assert np.all(np.abs(s1 - s0) <= 1e-10 * np.abs(s0))


def test_a_unit_change_scales_the_translations_only(api):
    g = _metamorphic_base()
    (R0, t0, s0), _ = _check_graph(api, g)
    h = dict(g, t=g["t"] * 1000.0, et=g["et"] * 1000.0)
    R1, t1, s1 = _solve_both(api, h)
    assert np.abs(R1 - R0).max() < 1e-10
    assert np.abs(t1 - 1000.0 * t0).max() < 1e-10 * 1000.0 * np.abs(t0).max()
    assert np.all(np.abs(s1 - s0) <= 1e-10 * np.abs(s0))


# ---------------------------------------------------------------------------------------------------------
# degenerate projections

RX, RY, RZ = np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])
# (G, R0): the fixed node's rotation is R0 and every edge rotation R_e becomes G R_e G^T, so M = G M_I G^T R0
# with M_I the matrix in the identity frame, and a unique nearest rotation moves the same way.  With G = I
# and a generic R0, M keeps exact zero ROWS but no zero column: the Jacobi SVD then has to recognise a
# vanishing singular value that is not an exact zero.
IDENTITY = (np.eye(3), np.eye(3))
FRAMES = [(np.eye(3), Rotation.from_rotvec([-0.7, 0.9, 0.1]).as_matrix()),
          (np.eye(3), Rotation.from_rotvec([2.0, -0.4, 1.1]).as_matrix()),
          (Rotation.from_rotvec([0.3, 1.2, -0.8]).as_matrix(), Rotation.from_rotvec([-1.5, 0.2, 0.6]).as_matrix()),
          (Rotation.from_rotvec([-2.2, 0.5, 0.4]).as_matrix(), Rotation.from_rotvec([0.1, -0.3, 2.7]).as_matrix())]
FRAME_IDS = ["R0_a", "R0_b", "G_R0_a", "G_R0_b"]


def _parallel_edges(rotations, frame, seed=0):
    """Fixed node 0 (R = R0) and free node 1 joined by one edge 0 -> 1 per rotation (as G R_e G^T):
    M = G mean(rotations) G^T R0."""
    G, R0 = frame
    rng = np.random.default_rng(seed)
    ne = len(rotations)
    return dict(fixed=np.array([1, 0], np.uint8), R=np.stack([R0, np.eye(3)]),
                t=np.array([[0.2, -0.1, 0.3], [1.0, 1.0, 1.0]]), id1=np.zeros(ne, np.int32),
                id2=np.ones(ne, np.int32), eR=np.stack([G @ Re @ G.T for Re in rotations]),
                et=rng.normal(size=(ne, 3)), scale_col=np.full(ne, -1, np.int32), n_scale=0)


RANK_DEFICIENT = [
    ([np.eye(3), np.eye(3), RX, RY], np.diag([0.5, 0.5, 0.0]), 0),  # rank 2: the nearest rotation is G G^T R0
    ([np.eye(3), RX], np.diag([1.0, 0.0, 0.0]), 1),                # rank 1: any rotation about G x
    ([np.eye(3), RX, RY, RZ], np.zeros((3, 3)), 1),                # zero: any rotation
]


def _rank_deficient(api, frame, rotations, M, ties):
    G, R0 = frame
    g = _parallel_edges(rotations, frame)
    ref = dense.solve(*(g[k] for k in GRAPH_KEYS))
    assert np.abs(ref["M"][1] - G @ M @ G.T @ R0).max() < 1e-14
    (nR, _, _), n_ties = _check_graph(api, g)
    assert n_ties == ties
    if ties == 0:
        assert np.abs(nR[1] - R0).max() < 1e-14


@pytest.mark.parametrize("rotations,M,ties", RANK_DEFICIENT)
def test_rank_deficient_projections_give_rotations(api, rotations, M, ties):
    _rank_deficient(api, IDENTITY, rotations, M, ties)


@pytest.mark.parametrize("frame", FRAMES, ids=FRAME_IDS)
@pytest.mark.parametrize("rotations,M,ties", RANK_DEFICIENT, ids=["rank2", "rank1", "zero"])
def test_rank_deficient_projections_in_rotated_frames(api, frame, rotations, M, ties):
    _rank_deficient(api, frame, rotations, M, ties)


def _half_turn(frame):
    """fixed(R0) - free - fixed(G Rx180 G^T R0) with identity edges: M = G diag(1, 0, 0) G^T R0."""
    G, R0 = frame
    return (np.array([1, 0, 1], np.uint8), np.stack([R0, np.eye(3), G @ RX @ G.T @ R0]),
            np.array([[0.0, 0, 0], [0.3, 0.1, 0], [1.0, 0.5, -0.2]]), np.stack([np.eye(3)] * 3),
            np.array([[0.5, 0.2, 0.0], [0.4, 0.1, 0.1], [0.0, 0, 0]]))


def _chain_half_turn(api, frame):
    G, R0 = frame
    fixed, R, t, eR, et = _half_turn(frame)
    nR, nt = api.posegraph_spread_chains(np.array([0, 3], np.int32), fixed, R, t, eR, et)
    ref = dense.solve_chains(np.array([0, 3]), fixed, R, t, eR, et)
    assert np.abs(ref["M"][1] - G @ np.diag([1.0, 0.0, 0.0]) @ G.T @ R0).max() < 1e-14
    assert _check(nR, nt, ref, fixed, R, t, TOL, TOL) == 1


def test_chain_half_turn_interpolation_is_a_rotation(api):
    """The interpolation weight of the free node is 1/2: M = diag(1, 0, 0) has rank 1 and any rotation
    about x is nearest.  The free node must still get a proper rotation."""
    _chain_half_turn(api, IDENTITY)


@pytest.mark.parametrize("frame", FRAMES, ids=FRAME_IDS)
def test_chain_half_turn_in_rotated_frames(api, frame):
    _chain_half_turn(api, frame)


def _general_half_turn(api, frame):
    fixed, R, t, eR, et = _half_turn(frame)
    g = dict(fixed=fixed, R=R, t=t, id1=np.array([0, 1], np.int32), id2=np.array([1, 2], np.int32), eR=eR[:2],
             et=et[:2], scale_col=np.array([-1, -1], np.int32), n_scale=0)
    assert _check_graph(api, g)[1] == 1


def test_half_turn_interpolation_in_the_general_solve(api):
    """The chain of test_chain_half_turn_interpolation_is_a_rotation as a general graph."""
    _general_half_turn(api, IDENTITY)


@pytest.mark.parametrize("frame", FRAMES, ids=FRAME_IDS)
def test_half_turn_in_the_general_solve_in_rotated_frames(api, frame):
    _general_half_turn(api, frame)


def _reflection(api, frame):
    rots = [np.eye(3), Rotation.from_euler("x", 175, degrees=True).as_matrix(),
            Rotation.from_euler("y", 160, degrees=True).as_matrix()]
    M = np.mean(rots, axis=0)
    S = np.linalg.svd(M, compute_uv=False)
    assert abs(np.linalg.det(M) + 0.032) < 1e-3 and np.allclose(S, [0.45, 0.34, 0.21], atol=0.01)
    G, R0 = frame
    g = _parallel_edges(rots, frame, seed=1)
    ref = dense.solve(*(g[k] for k in GRAPH_KEYS))
    assert np.abs(ref["M"][1] - G @ M @ G.T @ R0).max() < 1e-14 and ref["sv"][1, 2] < 0
    assert _check_graph(api, g)[1] == 0


def test_reflection_with_distinct_singular_values(api):
    """Parallel edges {I, Rx(175 deg), Ry(160 deg)}: M has det < 0 and distinct singular values, so the
    nearest rotation flips the smallest singular direction and is unique."""
    _reflection(api, IDENTITY)


@pytest.mark.parametrize("frame", FRAMES, ids=FRAME_IDS)
def test_reflection_in_rotated_frames(api, frame):
    _reflection(api, frame)
