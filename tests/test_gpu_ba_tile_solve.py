"""The BA's reduced-camera-system solve (ba_tile_two / ba_tile_solve of coslam_b200/csrc/ba_tile.cuh)
against dense float64 references, through cosl_ba_debug_tile_solve.

Every system is built the way a Schur complement arises: a sum of rank-3 "point" terms G V^-1 G^T
over camera subsets plus a positive diagonal, so that its 6x6 block pattern is exactly the
co-visibility `adj` handed to the planner.  The checks:
  - scaled residual |Sx - b|_inf / (|S|_inf |x|_inf + |b|_inf) <= RES_TOL;
  - forward error against scipy's Cholesky, |x - x_ref|_inf / |x_ref|_inf <= kappa_1(S) * FWD_TOL;
  - the failure flag is clear, and three solves of the same system give the same bits (the updates of
    a tile are applied in one fixed order, hot successors included).
Both bounds come from the float64 error bound of a Cholesky solve (unit roundoff 1.1e-16 times a
modest growth factor)."""
import numpy as np
import pytest
import scipy.linalg as sla

pytestmark = pytest.mark.gpu

RES_TOL = 1e-14
FWD_TOL = 1e-14


def point_system(mf, subsets, seed, diag=1.0):
    """(S, b, adj): S = sum over subsets of G V^-1 G^T (G: 6|subset| x 3, V: 3x3 SPD) + a positive
    diagonal; adj[a, b] = 1 iff a and b share a subset."""
    rng = np.random.default_rng(seed)
    n = 6 * mf
    S = np.zeros((n, n))
    adj = np.zeros((mf, mf), np.uint8)
    for cams in subsets:
        cams = np.asarray(sorted(set(int(c) for c in cams)), np.int64)
        if len(cams) == 0:
            continue
        idx = (6 * cams[:, None] + np.arange(6)).ravel()
        G = rng.normal(size=(len(idx), 3))
        A = rng.normal(size=(3, 3))
        V = A @ A.T + 0.5 * np.eye(3)
        S[np.ix_(idx, idx)] += G @ np.linalg.solve(V, G.T)
        adj[np.ix_(cams, cams)] = 1
    S[np.diag_indices(n)] += diag * (0.5 + rng.random(n))
    b = rng.normal(size=n)
    return S, b, adj


def chain_subsets(rng, cams, extra, kmax=5):
    """Subsets over `cams` that connect them (consecutive pairs) plus `extra` random ones."""
    cams = list(cams)
    subs = [cams[i:i + 2] for i in range(len(cams) - 1)]
    for _ in range(extra if len(cams) > 1 else 0):
        k = int(rng.integers(2, min(kmax, len(cams)) + 1))
        subs.append(rng.choice(cams, size=k, replace=False))
    return subs


def band_subsets(mf, bw):
    """One point per window of bw + 1 consecutive cameras: co-visibility |a - b| <= bw."""
    return [range(s, s + bw + 1) for s in range(mf - bw)]


def solve(api, S, b, adj, nd_depth=-1, repeats=3):
    """Solve `repeats` times; the solutions must be bit-identical and the failure flag clear."""
    xs = []
    for _ in range(repeats):
        x, fail, info = api.ba_debug_tile_solve(S, b, adj, nd_depth)
        assert fail == 0, info
        xs.append(x)
    for x in xs[1:]:
        assert np.array_equal(x.view(np.uint64), xs[0].view(np.uint64)), "solve is not bit-reproducible"
    return xs[0], info


def check_accuracy(S, b, x):
    Sf = np.tril(S) + np.tril(S, -1).T  # what the solver reads
    nrm = np.abs(Sf).sum(1).max()
    res = np.abs(Sf @ x - b).max() / (nrm * np.abs(x).max() + np.abs(b).max())
    assert res <= RES_TOL, res
    c = sla.cho_factor(Sf, lower=True)
    xr = sla.cho_solve(c, b)
    rcond, info = sla.lapack.dpocon(c[0], nrm, uplo="L")
    assert info == 0 and rcond > 0
    fwd = np.abs(x - xr).max() / np.abs(xr).max()
    assert fwd <= FWD_TOL / rcond, (fwd, 1.0 / rcond)


def split_point(mf):
    """First camera of the second block when ba_plan.h's split_blocks cuts mf cameras in natural order."""
    q = (mf + 9) // 10
    return mf // q + (1 if mf % q else 0)


@pytest.mark.parametrize("coupled", [True, False], ids=["coupled", "uncoupled"])
@pytest.mark.parametrize("mf", list(range(1, 21)))
def test_one_cta_path(api, mf, coupled):
    """Up to 20 cameras = one or two blocks of 6k rows, k = 1..10: ba_tile_two.  Uncoupled: the two
    blocks of split_blocks share no point (the t10 < 0 case; inside one block for mf <= 10)."""
    rng = np.random.default_rng(100 + mf)
    h = split_point(mf) if mf > 10 else (mf + 1) // 2
    if coupled:
        subs = chain_subsets(rng, range(mf), mf)
    else:
        subs = chain_subsets(rng, range(h), h) + chain_subsets(rng, range(h, mf), mf - h)
    S, b, adj = point_system(mf, subs, seed=mf + (0 if coupled else 1000))
    x, info = solve(api, S, b, adj)
    assert info["small_solve"] == 1 and info["grid"] == 1
    assert info["blocks"] == (1 if mf <= 10 else 2)
    if mf > 10:
        assert info["tiles"] == (3 if coupled else 2)  # t10 exists or not
    check_accuracy(S, b, x)


@pytest.mark.parametrize("mf", [21, 29, 31, 59])
def test_unequal_block_splits(api, mf):
    """Blocks of 7 cameras (21: 42 rows, not a multiple of 8), 10 and 9 (29, 59), 8 and 7 (31): the
    persistent kernel with padded identities of several sizes in one system."""
    rng = np.random.default_rng(mf)
    S, b, adj = point_system(mf, chain_subsets(rng, range(mf), 2 * mf), seed=mf)
    x, info = solve(api, S, b, adj)
    assert info["small_solve"] == 0 and info["blocks"] == (mf + 9) // 10 and info["grid"] >= 2
    check_accuracy(S, b, x)


@pytest.mark.parametrize("mf", [40, 61])
def test_dense_covisibility(api, mf):
    rng = np.random.default_rng(mf)
    subs = [range(mf)] + [rng.choice(mf, size=mf // 2, replace=False) for _ in range(8)]
    S, b, adj = point_system(mf, subs, seed=mf)
    assert adj.all()
    x, info = solve(api, S, b, adj)
    nb = (mf + 9) // 10
    assert info["small_solve"] == 0 and info["blocks"] == nb and info["tiles"] == nb * (nb + 1) // 2
    check_accuracy(S, b, x)


@pytest.mark.parametrize("mf,extra", [(50, 40), (100, 60), (150, 150)])
def test_random_sparse_patterns(api, mf, extra):
    """Irregular co-visibility: not band-like, the natural order and fill."""
    rng = np.random.default_rng(7 * mf)
    S, b, adj = point_system(mf, chain_subsets(rng, range(mf), extra), seed=mf)
    x, info = solve(api, S, b, adj)
    assert info["small_solve"] == 0 and info["nd_depth"] == 0
    check_accuracy(S, b, x)


@pytest.mark.parametrize("mf,ncomp,interleave", [(50, 2, False), (45, 3, True), (33, 3, False)])
def test_disconnected_components(api, mf, ncomp, interleave):
    """Two or three components; interleaved ones share every block, contiguous ones are cut mid-block."""
    rng = np.random.default_rng(mf + ncomp)
    cams = np.arange(mf)
    groups = [cams[g::ncomp] for g in range(ncomp)] if interleave else np.array_split(cams, ncomp)
    subs = [s for g in groups for s in chain_subsets(rng, g, len(g))]
    S, b, adj = point_system(mf, subs, seed=mf)
    x, info = solve(api, S, b, adj)
    assert info["small_solve"] == 0
    check_accuracy(S, b, x)


# (61, 14): just above the band-like threshold (mf >= 4 (bw + 1) and mf > 60), too short to dissect;
# (121, 29): band-like with one level of dissection; (796, 35): the c4 band, which the planner can
# dissect three levels deep -- separators with diagonal scratch tiles (the rhs parts of the SUM task)
# and backward lists of lengths that are not multiples of 4 (tests/test_ba_plan.py checks both on
# the plan of the same pattern).
@pytest.mark.parametrize("nd_depth", [0, 1, 2, 3])
@pytest.mark.parametrize("mf,bw", [(61, 14), (121, 29), (796, 35)])
def test_band_forced_dissection_depth(api, mf, bw, nd_depth):
    S, b, adj = point_system(mf, band_subsets(mf, bw), seed=mf + bw)
    x, info = solve(api, S, b, adj, nd_depth)
    assert info["nd_depth"] == nd_depth and info["small_solve"] == 0
    check_accuracy(S, b, x)


def test_band_automatic_depth(api):
    S, b, adj = point_system(796, band_subsets(796, 35), seed=831)
    x, info = solve(api, S, b, adj)
    assert info["nd_depth"] >= 2
    check_accuracy(S, b, x)


def ba_scaling(mf):
    """Rotation rows x 1e3 against translation rows, as the camera blocks of a BA's reduced system."""
    return np.tile(np.array([1e3, 1e3, 1e3, 1.0, 1.0, 1.0]), mf)


@pytest.mark.parametrize("scale", ["ba_rows", 1e-20, 1e20])
@pytest.mark.parametrize("mf", [13, 45])
def test_scaled_systems(api, mf, scale):
    """Pivots far from 1 but inside (1e-30, 1e30) solve with the failure flag clear."""
    rng = np.random.default_rng(mf)
    S, b, adj = point_system(mf, chain_subsets(rng, range(mf), mf), seed=mf)
    if scale == "ba_rows":
        d = ba_scaling(mf)
        S, b = S * d[:, None] * d[None, :], b * d
    else:
        S = S * scale
    x, info = solve(api, S, b, adj)
    assert info["small_solve"] == (1 if mf <= 20 else 0)
    check_accuracy(S, b, x)


@pytest.mark.parametrize("defect", ["indefinite", "zero_block", "nan"])
@pytest.mark.parametrize("mf", [13, 45])
def test_failure_flag(api, mf, defect):
    """A non-SPD system raises the failure flag; the call itself still succeeds."""
    rng = np.random.default_rng(mf)
    S, b, adj = point_system(mf, chain_subsets(rng, range(mf), mf), seed=mf)
    c = mf - 2  # a camera of the last block
    if defect == "indefinite":
        S[6 * c + 1, 6 * c + 1] = -S[6 * c + 1, 6 * c + 1]
    elif defect == "zero_block":
        S[6 * c:6 * c + 6, :] = 0.0
        S[:, 6 * c:6 * c + 6] = 0.0
    else:
        S[6 * c + 4, 6 * (c - 1) + 2] = np.nan  # lower triangle of the (c, c - 1) coupling
    x, fail, info = api.ba_debug_tile_solve(S, b, adj)
    assert fail == 1
    assert info["small_solve"] == (1 if mf <= 20 else 0)
    # a valid system solved right after it clears the flag again
    S2, b2, adj2 = point_system(mf, chain_subsets(rng, range(mf), mf), seed=mf + 1)
    _, fail2, _ = api.ba_debug_tile_solve(S2, b2, adj2)
    assert fail2 == 0
