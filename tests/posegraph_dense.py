"""A plain float64 least-squares reference of GlobalPoseGraph's two solves (computeNewCameraRotations and
computeNewCameraTranslations / ...Translations4, slam/SL_GlobalPoseEstimation.cpp), independent of the
CUDA kernels and of the C++ oracles: no closed form, no normal equations.

Every edge e = (i -> j) with at least one free end gives, per slot, three rows
    x_j - R_e x_i               = 0      rotation slots 0..2: x = column s of R_k
    x_j - R_e x_i               = t_e    translation slot, known scale
    x_j - R_e x_i - s_c t_e     = 0      translation slot, scale column c (an extra unknown)
with the fixed ends moved to the right-hand side; an edge between two fixed nodes gives no row.  The
three rotation slots share one matrix.  Small systems are solved by numpy.linalg.lstsq (SVD) on the dense
matrix, larger ones by scipy's sparse LU on the augmented system [[I, A], [A^T, 0]] [r; x] = [b; 0].
Each free node's rotation M is projected with numpy.linalg.svd as U diag(1, 1, det(U V^T)) V^T.
TEST INFRASTRUCTURE: used by tests/ only."""
import warnings

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

DENSE_MAX = 1000  # unknowns per slot up to which the dense SVD least-squares solve is used


def _lstsq(A, B, method):
    m, n = A.shape
    if method == "dense" or (method == "auto" and n <= DENSE_MAX):
        x, _, rank, _ = np.linalg.lstsq(A.toarray(), B, rcond=None)
        if rank < n:
            raise ValueError(f"rank-deficient system: rank {rank} of {n} unknowns")
        return x
    K = sp.bmat([[sp.identity(m, format="csc"), A], [A.T, None]], format="csc")
    rhs = np.vstack([B, np.zeros((n, B.shape[1]))])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", spla.MatrixRankWarning)  # reported below as a ValueError
        x = spla.spsolve(K, rhs)
    x = np.asarray(x).reshape(m + n, B.shape[1])[m:]
    if not np.isfinite(x).all():
        raise ValueError("rank-deficient system")
    return x


def project(M):
    """Nearest rotation (Frobenius) of each 3x3 of M (..., 3, 3) and the signed singular values
    (s0, s1, det(U V^T) s2) of the projection.  The projection is unique iff sv[..., 1] + sv[..., 2] > 0;
    ||R - M||_F is then, and for every minimiser of a tie, sqrt(||M||_F^2 + 3 - 2 sum(sv))."""
    U, S, Vt = np.linalg.svd(M)
    d = np.sign(np.linalg.det(U @ Vt))
    D = np.ones(M.shape[:-2] + (3,))
    D[..., 2] = d
    sv = S.copy()
    sv[..., 2] *= d
    return (U * D[..., None, :]) @ Vt, sv


def min_distance(M, sv):
    """min over rotations R of ||R - M||_F."""
    return np.sqrt(np.maximum(0.0, np.sum(M * M, axis=(-2, -1)) + 3.0 - 2.0 * sv.sum(axis=-1)))


def solve(fixed, R, t, id1, id2, eR, et, scale_col=None, n_scale=0, method="auto"):
    """The least-squares solution of a general pose graph.  Returns a dict with newR (n,3,3), newt (n,3),
    scale (n_scale,), M (n,3,3): the unprojected rotation of every free node (the input R of a fixed one),
    and sv (n,3): the signed singular values of M's projection ((1, 1, 1) for a fixed node).
    method: "dense" (lstsq), "sparse" (augmented system) or "auto" (dense up to DENSE_MAX unknowns)."""
    fixed = np.asarray(fixed).astype(bool)
    n = fixed.size
    R = np.asarray(R, np.float64).reshape(n, 3, 3)
    t = np.asarray(t, np.float64).reshape(n, 3)
    id1 = np.asarray(id1, np.int64)
    id2 = np.asarray(id2, np.int64)
    eR = np.asarray(eR, np.float64).reshape(-1, 3, 3)
    et = np.asarray(et, np.float64).reshape(-1, 3)
    sc = np.full(id1.size, -1, np.int64) if scale_col is None else np.asarray(scale_col, np.int64)
    n_scale = int(n_scale)
    free = np.flatnonzero(~fixed)
    nF = free.size
    freeOf = np.full(n, -1, np.int64)
    freeOf[free] = np.arange(nF)
    rows = np.flatnonzero(~(fixed[id1] & fixed[id2]))
    i, j, Re, te, c = id1[rows], id2[rows], eR[rows], et[rows], sc[rows]
    m = rows.size
    if nF == 0:  # nothing to solve (and no scale column can have a row)
        return dict(newR=R.copy(), newt=t.copy(), scale=np.zeros(n_scale), M=R.copy(), sv=np.ones((n, 3)))
    # A: +I at (edge, node j), -R_e at (edge, node i), for the free ends
    ri, ci, vi = [], [], []
    q = np.arange(m)
    u = np.arange(3)
    fj = ~fixed[j]
    ri.append((3 * q[fj, None] + u).ravel())
    ci.append((3 * freeOf[j[fj], None] + u).ravel())
    vi.append(np.ones(3 * fj.sum()))
    fi = ~fixed[i]
    ri.append(np.broadcast_to((3 * q[fi, None, None] + u[:, None]), (fi.sum(), 3, 3)).ravel())
    ci.append(np.broadcast_to((3 * freeOf[i[fi], None, None] + u[None, :]), (fi.sum(), 3, 3)).ravel())
    vi.append(-Re[fi].ravel())
    r_all, c_all, v_all = np.concatenate(ri), np.concatenate(ci), np.concatenate(vi)
    A = sp.csc_matrix((v_all, (r_all, c_all)), shape=(3 * m, 3 * nF))
    # rotation slots: b = R_e X_i (fixed i) - X_j (fixed j), one column per slot
    Xi = np.where(fixed[i, None, None], R[i], 0.0)
    Xj = np.where(fixed[j, None, None], R[j], 0.0)
    Brot = (Re @ Xi - Xj).reshape(3 * m, 3)
    # translation slot: b = t_e (known scale) + R_e t_i (fixed i) - t_j (fixed j); scale columns -t_e
    ti = np.where(fixed[i, None], t[i], 0.0)
    tj = np.where(fixed[j, None], t[j], 0.0)
    bt = np.einsum("eab,eb->ea", Re, ti) - tj + np.where(c[:, None] < 0, te, 0.0)
    unc = np.flatnonzero(c >= 0)
    S = sp.csc_matrix(((-te[unc]).ravel(), ((3 * unc[:, None] + u).ravel(), np.repeat(c[unc], 3))),
                      shape=(3 * m, n_scale))
    At = sp.hstack([A, S], format="csc")
    xr = _lstsq(A, Brot, method)
    xt = _lstsq(At, bt.reshape(3 * m, 1), method)[:, 0]
    M = R.copy()
    M[free] = xr.reshape(nF, 3, 3)  # rows: component u of column s, i.e. M[u, s]
    newR, newt = R.copy(), t.copy()
    sv = np.ones((n, 3))
    newR[free], sv[free] = project(M[free])
    newt[free] = xt[:3 * nF].reshape(nF, 3)
    return dict(newR=newR, newt=newt, scale=xt[3 * nF:].copy(), M=M, sv=sv)


def solve_chains(chain_off, fixed, R, t, eR, et, method="auto"):
    """solve() of every chain of a posegraph_spread_chains batch (edge k = node k -> k+1, stored at k).
    Returns the batch's newR, newt, M and sv."""
    out = dict(newR=np.empty_like(R), newt=np.empty_like(t), M=np.empty_like(R), sv=np.empty(t.shape))
    for a, b in zip(chain_off[:-1], chain_off[1:]):
        a, b = int(a), int(b)
        if b == a:
            continue
        ids = np.arange(b - a - 1)
        r = solve(fixed[a:b], R[a:b], t[a:b], ids, ids + 1, eR[a:b - 1], et[a:b - 1], method=method)
        for k in out:
            out[k][a:b] = r[k]
    return out
