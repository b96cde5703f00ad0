// posegraph.cu -- post-BA pose-graph spreading for chain graphs (SURVEY.md 8f-2), sm_90a.
//
// Replaces, for the graphs RobustBundleRTS::constructCameraGraphs builds (one chain per camera, node k
// -> node k+1, key-frame nodes fixed; reference app/SL_CoSLAMRobustBA.cpp:182-232), the two sparse
// least-squares solves of RobustBundleRTS::updateNonKeyCameraPoses (:233-250):
//   GlobalPoseGraph::computeNewCameraRotations     slam/SL_GlobalPoseEstimation.cpp:52-218
//       min sum_k |X_{k+1} - R_k X_k|_F^2 over the free nodes, then nearest rotation (:205-211)
//   GlobalPoseGraph::computeNewCameraTranslations  slam/SL_GlobalPoseEstimation.cpp:220-359
//       min sum_k |t_{k+1} - R_k t_k - t_k,k+1|^2
// R_k is orthogonal, so with P_k = R_{k-1} ... R_a (product of the edge rotations from the fixed node a on
// the left of a run of free nodes) the substitution Y_k = P_k^T X_k turns every residual into
// Y_{k+1} - Y_k: the least-squares solution is the LINEAR INTERPOLATION of Y between the two fixed ends
// (constant when only one end is fixed), and the same substitution spreads the translation residual of a
// run uniformly over its edges.  No linear system is left: the work is one segmented scan of rigid
// transforms (P_k, q_k) per chain plus a 3x3 polar projection per free node.
//
// Data layout (device, fp64): nodes of all chains concatenated in frame order; R row-major 3x3 / node,
// t 3 / node, edge k (node k -> k+1) stored at index k (the slot of a chain's last node is unused).
// Kernel: one CTA per chain, each thread owns a contiguous chunk of nodes; chunk composites are scanned
// across the CTA in shared memory; newR/newt hold (P_k, q_k) between the two passes.
// Algorithmic bytes / node: 216 read (R, t, edge R, edge t, flag) + 96 written.
//
// The second half of the file solves GENERAL graphs with shared unknown scales (cosl_posegraph_solve,
// the camera-group merge): normal equations on the BA's tile Cholesky, see the comment above PgItem.
#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <functional>
#include <map>
#include <new>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tile_solve.h"

namespace coslam {
namespace {

constexpr int PG_THREADS = 256;

struct Rigid {
  double R[9];
  double t[3];
};

__device__ __forceinline__ void rigid_identity(Rigid& a) {
#pragma unroll
  for (int i = 0; i < 9; ++i) a.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  a.t[0] = a.t[1] = a.t[2] = 0.0;
}
// c = b after a :  x -> b.R (a.R x + a.t) + b.t
__device__ __forceinline__ void rigid_compose(const Rigid& a, const Rigid& b, Rigid& c) {
  Rigid o;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
      o.R[3 * i + j] = b.R[3 * i] * a.R[j] + b.R[3 * i + 1] * a.R[3 + j] + b.R[3 * i + 2] * a.R[6 + j];
    o.t[i] = b.R[3 * i] * a.t[0] + b.R[3 * i + 1] * a.t[1] + b.R[3 * i + 2] * a.t[2] + b.t[i];
  }
  c = o;
}
__device__ __forceinline__ void load_edge(const double* eR, const double* et, int k, Rigid& e) {
#pragma unroll
  for (int i = 0; i < 9; ++i) e.R[i] = eR[9 * (size_t)k + i];
#pragma unroll
  for (int i = 0; i < 3; ++i) e.t[i] = et[3 * (size_t)k + i];
}

// nearest rotation (Frobenius) of a 3x3: one-sided Jacobi SVD M = U S V^T, R = U diag(1,1,det) V^T with
// the sign flip on the smallest singular direction.
__device__ void nearest_rotation(const double* M, double* Rout) {
  double A[9], W[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    A[i] = M[i];
    W[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double a = 0, b = 0, c = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        a += A[3 * i + p] * A[3 * i + p];
        b += A[3 * i + q] * A[3 * i + q];
        c += A[3 * i + p] * A[3 * i + q];
      }
      const double rel = fabs(c) / sqrt(a * b + 1e-300);
      off = fmax(off, rel);
      if (rel < 1e-18) continue;
      const double zeta = (b - a) / (2.0 * c);
      const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        double x = A[3 * i + p], y = A[3 * i + q];
        A[3 * i + p] = cs * x - sn * y;
        A[3 * i + q] = sn * x + cs * y;
        x = W[3 * i + p];
        y = W[3 * i + q];
        W[3 * i + p] = cs * x - sn * y;
        W[3 * i + q] = sn * x + cs * y;
      }
    }
    if (off < 1e-17) break;
  }
  double S[3], U[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double s = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
    S[j] = s;
    const double inv = s > 0 ? 1.0 / s : 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) U[3 * i + j] = A[3 * i + j] * inv;
  }
  // A singular value that is zero or at roundoff level next to the largest (M of rank < 3) leaves its column
  // of U zero, or -- when the Jacobi sweeps cannot orthogonalise a vanishing column (its squared norm falls
  // under the 1e-300 floor of `rel`) -- parallel to another one, and Q below would not be orthogonal.  Such
  // a direction does not enter ||R - M|| beyond roundoff, so U is completed to a right-handed orthonormal
  // basis instead: any completion is a nearest rotation, and det(U) = det(W) = 1.  Outputs with every
  // singular value above 16 eps of the largest keep the plain path.
  // (Every index below is a constant after unrolling: U stays in registers.)
  const double sTiny = 16.0 * DBL_EPSILON * fmax(S[0], fmax(S[1], S[2]));
  bool zero[3] = {S[0] <= sTiny, S[1] <= sTiny, S[2] <= sTiny};
  const int nZero = zero[0] + zero[1] + zero[2];
  if (nZero == 3) {
#pragma unroll
    for (int i = 0; i < 9; ++i) U[i] = W[i];
  } else if (nZero > 0) {
    if (nZero == 2) {  // a unit vector orthogonal to the remaining column u, into the first zero column
      double u[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) u[i] = !zero[0] ? U[3 * i] : (!zero[1] ? U[3 * i + 1] : U[3 * i + 2]);
      // the coordinate axis least aligned with u, minus its component along u
      const int m = (fabs(u[0]) <= fabs(u[1]) && fabs(u[0]) <= fabs(u[2])) ? 0 : (fabs(u[1]) <= fabs(u[2]) ? 1 : 2);
      const double um = m == 0 ? u[0] : (m == 1 ? u[1] : u[2]);
      double v[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) v[i] = (i == m ? 1.0 : 0.0) - um * u[i];
      const double inv = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
      const int z = zero[0] ? 0 : 1;
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (j == z) {
#pragma unroll
          for (int i = 0; i < 3; ++i) U[3 * i + j] = v[i] * inv;
          zero[j] = false;  // the cross product below fills the last one
        }
    }
    // the zero column z = (column z+1) x (column z+2): det(U) = +1
#pragma unroll
    for (int z = 0; z < 3; ++z)
      if (zero[z]) {
        const int p = (z + 1) % 3, q = (z + 2) % 3;
        U[z] = U[3 + p] * U[6 + q] - U[6 + p] * U[3 + q];
        U[3 + z] = U[6 + p] * U[q] - U[p] * U[6 + q];
        U[6 + z] = U[p] * U[3 + q] - U[3 + p] * U[q];
      }
  }
  double Q[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Q[3 * i + j] = U[3 * i] * W[3 * j] + U[3 * i + 1] * W[3 * j + 1] + U[3 * i + 2] * W[3 * j + 2];
  const double det = Q[0] * (Q[4] * Q[8] - Q[5] * Q[7]) - Q[1] * (Q[3] * Q[8] - Q[5] * Q[6]) +
                     Q[2] * (Q[3] * Q[7] - Q[4] * Q[6]);
  if (det < 0) {
    int sm = 0;
    if (S[1] < S[sm]) sm = 1;
    if (S[2] < S[sm]) sm = 2;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double u = sm == 0 ? U[3 * i] : (sm == 1 ? U[3 * i + 1] : U[3 * i + 2]);
        const double w = sm == 0 ? W[3 * j] : (sm == 1 ? W[3 * j + 1] : W[3 * j + 2]);
        Q[3 * i + j] -= 2.0 * u * w;
      }
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) Rout[i] = Q[i];
}

// One CTA per chain.  Element k of the scan is the edge (k-1 -> k); a run restarts at the element that
// FOLLOWS a fixed node, so the composite stored for node k maps the coordinates of the nearest fixed node
// on its left (or of the chain's first node) to node k, and a fixed node on the right end of a run
// carries the composite of the whole run.
__global__ void __launch_bounds__(PG_THREADS)
posegraph_chain_kernel(const int* __restrict__ chainOff, const unsigned char* __restrict__ fixed,
                       const double* __restrict__ R, const double* __restrict__ t,
                       const double* __restrict__ eR, const double* __restrict__ et,
                       double* __restrict__ newR, double* __restrict__ newt, int* __restrict__ anchor,
                       int* __restrict__ status) {
  __shared__ Rigid s_agg[PG_THREADS];
  __shared__ int s_head[PG_THREADS];   // chunk contains a run head
  __shared__ int s_lastFix[PG_THREADS];
  __shared__ int s_firstFix[PG_THREADS];
  const int c = blockIdx.x, tid = threadIdx.x;
  const int n0 = chainOff[c], n = chainOff[c + 1] - n0;
  if (n <= 0) return;
  const int per = (n + PG_THREADS - 1) / PG_THREADS;
  const int lo = min(n, tid * per), hi = min(n, lo + per);

  // pass 1: composite of the chunk (from its last run head on), fixed-node positions
  Rigid acc;
  rigid_identity(acc);
  int head = 0, lastFix = -1, firstFix = n;
  for (int k = lo; k < hi; ++k) {
    const int g = n0 + k;
    if (k == 0 || fixed[g - 1]) {
      head = 1;
      rigid_identity(acc);
    }
    if (k > 0) {
      Rigid e;
      load_edge(eR, et, g - 1, e);
      if (!fixed[g - 1]) rigid_compose(acc, e, acc);
      else acc = e;
    }
    if (fixed[g]) {
      lastFix = k;
      if (firstFix == n) firstFix = k;
    }
  }
  s_agg[tid] = acc;
  s_head[tid] = head;
  s_lastFix[tid] = lastFix;
  s_firstFix[tid] = firstFix;
  __syncthreads();
  // segmented inclusive scan over the chunk composites (Hillis-Steele), max / min scans of the fixed ids
  for (int d = 1; d < PG_THREADS; d <<= 1) {
    Rigid mine = s_agg[tid], left;
    int mh = s_head[tid], lh = 0, lf = s_lastFix[tid];
    const bool has = tid >= d;
    if (has) {
      left = s_agg[tid - d];
      lh = s_head[tid - d];
      lf = max(lf, s_lastFix[tid - d]);
    }
    int ff = s_firstFix[tid];
    if (tid + d < PG_THREADS) ff = min(ff, s_firstFix[tid + d]);
    __syncthreads();
    if (has && !mh) {
      rigid_compose(left, mine, mine);
      s_agg[tid] = mine;
      s_head[tid] = lh;
    }
    s_lastFix[tid] = lf;
    s_firstFix[tid] = ff;
    __syncthreads();
  }
  // pass 2: per-node composite and anchors
  Rigid pre;
  if (tid > 0) pre = s_agg[tid - 1];
  else rigid_identity(pre);
  int a = tid > 0 ? s_lastFix[tid - 1] : -1;
  for (int k = lo; k < hi; ++k) {
    const int g = n0 + k;
    if (k == 0) rigid_identity(pre);
    else {
      Rigid e;
      load_edge(eR, et, g - 1, e);
      if (!fixed[g - 1]) rigid_compose(pre, e, pre);
      else pre = e;
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) newR[9 * (size_t)g + i] = pre.R[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) newt[3 * (size_t)g + i] = pre.t[i];
    anchor[2 * (size_t)g] = a;
    if (fixed[g]) a = k;
  }
  // right anchors: walk the chunk backwards
  int b = tid + 1 < PG_THREADS ? s_firstFix[tid + 1] : n;
  for (int k = hi - 1; k >= lo; --k) {
    const int g = n0 + k;
    anchor[2 * (size_t)g + 1] = b;
    if (fixed[g]) b = k;
  }
  __syncthreads();  // (P,q) of the whole chain are in newR/newt (global, same CTA -> visible after the barrier)
  __threadfence_block();

  // pass 3: the closed-form least-squares solution per free node, in place.  A node only reads the
  // composites of ITSELF and of its right anchor (a fixed node, overwritten only by its own thread with
  // its input pose afterwards), so fixed nodes are finalised after a second barrier.
  for (int k = tid; k < n; k += PG_THREADS) {
    const int g = n0 + k;
    if (fixed[g]) continue;
    const int la = anchor[2 * (size_t)g], rb = anchor[2 * (size_t)g + 1];
    if (la < 0 && rb >= n) {
      atomicExch(status, 1 + c);  // no fixed node in this chain: the system is rank deficient
      continue;
    }
    double P[9], q[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) P[i] = newR[9 * (size_t)g + i];
#pragma unroll
    for (int i = 0; i < 3; ++i) q[i] = newt[3 * (size_t)g + i];
    double X[9], tk[3];
    if (rb >= n) {  // only the left end is fixed: exact propagation
      const double* Ra = R + 9 * (size_t)(n0 + la);
      const double* ta = t + 3 * (size_t)(n0 + la);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) X[3 * i + j] = P[3 * i] * Ra[j] + P[3 * i + 1] * Ra[3 + j] + P[3 * i + 2] * Ra[6 + j];
        tk[i] = P[3 * i] * ta[0] + P[3 * i + 1] * ta[1] + P[3 * i + 2] * ta[2] + q[i];
      }
    } else {
      const int gb = n0 + rb;
      double Pb[9], qb[3];
#pragma unroll
      for (int i = 0; i < 9; ++i) Pb[i] = newR[9 * (size_t)gb + i];
#pragma unroll
      for (int i = 0; i < 3; ++i) qb[i] = newt[3 * (size_t)gb + i];
      const double* Rb = R + 9 * (size_t)gb;
      const double* tb = t + 3 * (size_t)gb;
      // Yb = Pb^T Rb, ub = Pb^T (tb - qb)
      double Yb[9], ub[3], d[3] = {tb[0] - qb[0], tb[1] - qb[1], tb[2] - qb[2]};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) Yb[3 * i + j] = Pb[i] * Rb[j] + Pb[3 + i] * Rb[3 + j] + Pb[6 + i] * Rb[6 + j];
        ub[i] = Pb[i] * d[0] + Pb[3 + i] * d[1] + Pb[6 + i] * d[2];
      }
      double Y[9], u[3];
      if (la >= 0) {
        const double* Ra = R + 9 * (size_t)(n0 + la);
        const double* ta = t + 3 * (size_t)(n0 + la);
        const double w = (double)(k - la) / (double)(rb - la);
#pragma unroll
        for (int i = 0; i < 9; ++i) Y[i] = Ra[i] + w * (Yb[i] - Ra[i]);
#pragma unroll
        for (int i = 0; i < 3; ++i) u[i] = ta[i] + w * (ub[i] - ta[i]);
      } else {  // only the right end is fixed
#pragma unroll
        for (int i = 0; i < 9; ++i) Y[i] = Yb[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) u[i] = ub[i];
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) X[3 * i + j] = P[3 * i] * Y[j] + P[3 * i + 1] * Y[3 + j] + P[3 * i + 2] * Y[6 + j];
        tk[i] = P[3 * i] * u[0] + P[3 * i + 1] * u[1] + P[3 * i + 2] * u[2] + q[i];
      }
    }
    double Rn[9];
    nearest_rotation(X, Rn);
    // the right anchor's composite must stay intact until every node of the run has read it: free
    // nodes only overwrite their OWN slot
#pragma unroll
    for (int i = 0; i < 9; ++i) newR[9 * (size_t)g + i] = Rn[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) newt[3 * (size_t)g + i] = tk[i];
  }
  __syncthreads();
  for (int k = tid; k < n; k += PG_THREADS) {
    const int g = n0 + k;
    if (!fixed[g]) continue;
#pragma unroll
    for (int i = 0; i < 9; ++i) newR[9 * (size_t)g + i] = R[9 * (size_t)g + i];
#pragma unroll
    for (int i = 0; i < 3; ++i) newt[3 * (size_t)g + i] = t[3 * (size_t)g + i];
  }
}

// =====================================================================================================
// General pose graphs (cosl_posegraph_solve): the normal equations of the rotation and translation
// least-squares systems of GlobalPoseGraph (slam/SL_GlobalPoseEstimation.cpp:52-218, :361-525) as ONE
// SPD system in the tile layout of ba_plan.h, solved by the BA's tile Cholesky (tile_solve.h).
//
// Every edge e = (i -> j) with a row contributes, per 3-vector unknown ("slot") of its end nodes,
//     x_j - R_e x_i (- s_c t_e for the translation slot of an uncertain edge) = b_e
// where the slots are the three columns of R_k (rotations) and t_k (translations).  All four slots
// share the 3x3 blocks of R_e, so the unknowns of a free node form two planner "cameras" (units) of
// six rows: unit 2f = [col 0 | col 1], unit 2f+1 = [col 2 | t].  Scale column c lives in row c % 6
// of unit 2 nF + c / 6; unused rows of the last scale unit hold a 1 on the diagonal and a zero rhs.
// =====================================================================================================
struct PgItem {  // one 6x6 block of the lower triangle: rows of unit uR, columns of unit uC
  int uR, uC, rOff, cOff;
  int e0, e1;  // edges between two different nodes: range in PgDev::pairEdges
};

struct PgDev {
  const double *R, *t, *eR, *et;
  const unsigned char* fixed;
  const int *id1, *id2, *scaleCol;  // scaleCol: -1 = known scale
  const int *freeNode, *freeOf;     // free index <-> node
  const int *nodeOff, *nodeEdges;   // per free node: its edges (all have rows), by edge index
  const int *colOff, *colEdges;     // per scale column: its edges with rows, by edge index
  const int* pairEdges;
  const int* unitPos;                // unit -> index of its first row in the block-padded vector
  const PgItem* items;
  const int *itemOff, *diagBlk, *order, *blkCam0, *blkRows;
  int nF, nScale;
};

// index of slot s (0..2: column s of R_k, 3: t_k) of free node k in the block-padded vector
__device__ __forceinline__ int pg_pos(const PgDev& d, int k, int s) {
  return d.unitPos[2 * d.freeOf[k] + (s >> 1)] + 3 * (s & 1);
}
__device__ __forceinline__ int pg_scale_pos(const PgDev& d, int c) {
  return d.unitPos[2 * d.nF + c / 6] + c % 6;
}

// residual b_e - (A x0)_e of slot s of edge e (x0 == nullptr: x0 = 0, i.e. the right-hand side b_e)
__device__ void pg_edge_res(const PgDev& d, const double* __restrict__ x0, int e, int s, double v[3]) {
  const int i = d.id1[e], j = d.id2[e];
  const double* Re = d.eR + 9 * (size_t)e;
  const int c = (s == 3 && d.scaleCol) ? d.scaleCol[e] : -1;
  double xi[3] = {0, 0, 0}, xj[3] = {0, 0, 0};
  for (int u = 0; u < 3; ++u) {
    if (s < 3) {
      xi[u] = d.fixed[i] ? d.R[9 * (size_t)i + 3 * u + s] : (x0 ? x0[pg_pos(d, i, s) + u] : 0.0);
      xj[u] = d.fixed[j] ? d.R[9 * (size_t)j + 3 * u + s] : (x0 ? x0[pg_pos(d, j, s) + u] : 0.0);
    } else {
      xi[u] = d.fixed[i] ? d.t[3 * (size_t)i + u] : (x0 ? x0[pg_pos(d, i, 3) + u] : 0.0);
      xj[u] = d.fixed[j] ? d.t[3 * (size_t)j + u] : (x0 ? x0[pg_pos(d, j, 3) + u] : 0.0);
    }
  }
  const double sc = (c >= 0 && x0) ? x0[pg_scale_pos(d, c)] : 0.0;
  for (int u = 0; u < 3; ++u) {
    double r = (s == 3 && c < 0) ? d.et[3 * (size_t)e + u] : 0.0;
    r += Re[3 * u] * xi[0] + Re[3 * u + 1] * xi[1] + Re[3 * u + 2] * xi[2] - xj[u];
    if (c >= 0) r += sc * d.et[3 * (size_t)e + u];
    v[u] = r;
  }
}

// entry (row r of unit uA, column c of unit uB) of the normal matrix
__device__ double pg_entry(const PgDev& d, int uA, int r, int uB, int c, int e0, int e1) {
  const int nodeUnits = 2 * d.nF;
  if (uA >= nodeUnits && uB >= nodeUnits) {  // scale x scale: diagonal
    const int ca = 6 * (uA - nodeUnits) + r, cb = 6 * (uB - nodeUnits) + c;
    if (ca != cb) return 0.0;
    if (ca >= d.nScale) return 1.0;
    double v = 0.0;
    for (int q = d.colOff[ca]; q < d.colOff[ca + 1]; ++q) {
      const double* te = d.et + 3 * (size_t)d.colEdges[q];
      v += te[0] * te[0] + te[1] * te[1] + te[2] * te[2];
    }
    return v;
  }
  if (uA >= nodeUnits || uB >= nodeUnits) {  // translation slot x scale column
    int un = uA, rn = r, us = uB, cs = c;
    if (uA >= nodeUnits) {
      un = uB;
      rn = c;
      us = uA;
      cs = r;
    }
    const int col = 6 * (us - nodeUnits) + cs;
    if (!(un & 1) || rn < 3 || col >= d.nScale) return 0.0;
    const int f = un >> 1, p = d.freeNode[f], u = rn - 3;
    double v = 0.0;
    for (int q = d.nodeOff[f]; q < d.nodeOff[f + 1]; ++q) {
      const int e = d.nodeEdges[q];
      if (d.scaleCol[e] != col) continue;
      const double* te = d.et + 3 * (size_t)e;
      const double* Re = d.eR + 9 * (size_t)e;
      v += (d.id2[e] == p) ? -te[u] : Re[u] * te[0] + Re[3 + u] * te[1] + Re[6 + u] * te[2];
    }
    return v;
  }
  // node x node: the same 3x3 block for every slot, zero between different slots
  if (2 * (uA & 1) + r / 3 != 2 * (uB & 1) + c / 3) return 0.0;
  const int p = d.freeNode[uA >> 1], q2 = d.freeNode[uB >> 1], a = r % 3, b = c % 3;
  double v = 0.0;
  if (p == q2) {
    const int f = uA >> 1;
    for (int q = d.nodeOff[f]; q < d.nodeOff[f + 1]; ++q) {
      const int e = d.nodeEdges[q];
      if (d.id2[e] == p) {
        v += (a == b) ? 1.0 : 0.0;
      } else {  // (R_e^T R_e)(a, b)
        const double* Re = d.eR + 9 * (size_t)e;
        v += Re[a] * Re[b] + Re[3 + a] * Re[3 + b] + Re[6 + a] * Re[6 + b];
      }
    }
  } else {
    for (int q = e0; q < e1; ++q) {
      const int e = d.pairEdges[q];
      const double* Re = d.eR + 9 * (size_t)e;
      v -= (d.id1[e] == p) ? Re[3 * b + a] : Re[3 * a + b];  // p -> q2: -R_e^T; q2 -> p: -R_e
    }
  }
  return v;
}

// right-hand side (A^T (b - A x0)) of row r of unit u
__device__ double pg_rhs(const PgDev& d, const double* __restrict__ x0, int u, int r) {
  const int nodeUnits = 2 * d.nF;
  double v = 0.0, res[3];
  if (u >= nodeUnits) {
    const int col = 6 * (u - nodeUnits) + r;
    if (col >= d.nScale) return 0.0;
    for (int q = d.colOff[col]; q < d.colOff[col + 1]; ++q) {
      const int e = d.colEdges[q];
      pg_edge_res(d, x0, e, 3, res);
      const double* te = d.et + 3 * (size_t)e;
      v -= te[0] * res[0] + te[1] * res[1] + te[2] * res[2];
    }
    return v;
  }
  const int f = u >> 1, p = d.freeNode[f], s = 2 * (u & 1) + r / 3, a = r % 3;
  for (int q = d.nodeOff[f]; q < d.nodeOff[f + 1]; ++q) {
    const int e = d.nodeEdges[q];
    pg_edge_res(d, x0, e, s, res);
    if (d.id2[e] == p) {
      v += res[a];
    } else {
      const double* Re = d.eR + 9 * (size_t)e;
      v -= Re[a] * res[0] + Re[3 + a] * res[1] + Re[6 + a] * res[2];
    }
  }
  return v;
}

// One CTA per tile of the plan (fill included): zero it, then write the blocks that land in it and,
// for a diagonal tile, the block's right-hand side (padding rows 0), as ba_prep_kernel leaves them.
// Every entry is one thread's sum over a CSR list in a fixed order: no atomics, bit-reproducible.
__global__ void __launch_bounds__(256)
pg_assemble(PgDev d, const double* __restrict__ x0, double* __restrict__ tiles, double* __restrict__ rhs) {
  const int tl = blockIdx.x, tid = threadIdx.x;
  double2* tile2 = reinterpret_cast<double2*>(tiles + (size_t)tl * 4096);
#pragma unroll
  for (int u = 0; u < 8; ++u) tile2[tid + 256 * u] = make_double2(0.0, 0.0);
  __syncthreads();
  double* tile = tiles + (size_t)tl * 4096;
  const int i0 = d.itemOff[tl], n = (d.itemOff[tl + 1] - i0) * 36;
  for (int q = tid; q < n; q += 256) {
    const PgItem it = d.items[i0 + q / 36];
    const int r = (q % 36) / 6, c = q % 6;
    if (it.uR == it.uC && r < c) continue;  // diagonal block: lower half
    tile[(it.cOff + c) * 64 + it.rOff + r] = pg_entry(d, it.uR, r, it.uC, c, it.e0, it.e1);
  }
  const int k = d.diagBlk[tl];
  if (k >= 0 && tid < 64) {
    double v = 0.0;
    if (tid < d.blkRows[k]) v = pg_rhs(d, x0, d.order[d.blkCam0[k] + tid / 6], tid % 6);
    rhs[(size_t)k * 64 + tid] = v;
  }
}

// x = x1 + x2 (solve + refinement); per node: nearest rotation of the free nodes, copies of the fixed
// ones (slam/SL_GlobalPoseEstimation.cpp:205-216, :505-513); the scales; out[.. + 1] = 1 on a
// non-finite result.
__global__ void __launch_bounds__(128)
pg_finish(PgDev d, int nNodes, const double* __restrict__ x1, const double* __restrict__ x2,
          double* __restrict__ newR, double* __restrict__ newt, double* __restrict__ scale,
          double* __restrict__ nonFinite) {
  const int k = blockIdx.x * 128 + threadIdx.x;
  bool bad = false;
  if (k < nNodes) {
    if (d.fixed[k]) {
#pragma unroll
      for (int i = 0; i < 9; ++i) newR[9 * (size_t)k + i] = d.R[9 * (size_t)k + i];
#pragma unroll
      for (int i = 0; i < 3; ++i) newt[3 * (size_t)k + i] = d.t[3 * (size_t)k + i];
    } else {
      double M[9], Rn[9];
      for (int a = 0; a < 3; ++a) {
        const int p = pg_pos(d, k, a);
        for (int u = 0; u < 3; ++u) M[3 * u + a] = x1[p + u] + x2[p + u];  // column a of R_k
      }
      for (int i = 0; i < 9; ++i) bad |= !isfinite(M[i]);
      nearest_rotation(M, Rn);
      const int p = pg_pos(d, k, 3);
      for (int i = 0; i < 9; ++i) {
        newR[9 * (size_t)k + i] = Rn[i];
        bad |= !isfinite(Rn[i]);
      }
      for (int u = 0; u < 3; ++u) {
        const double v = x1[p + u] + x2[p + u];
        newt[3 * (size_t)k + u] = v;
        bad |= !isfinite(v);
      }
    }
  }
  if (k < d.nScale) {
    const int p = pg_scale_pos(d, k);
    const double v = x1[p] + x2[p];
    scale[k] = v;
    bad |= !isfinite(v);
  }
  if (bad) *nonFinite = 1.0;
}

thread_local double g_pgHostMs = 0.0;

// Where a prepare step packs a request's inputs: stage(bytes, &buf) points buf at a host buffer of at least
// `bytes` bytes (pageable for the synchronous calls, the handle's pinned buffer for a submit) or returns an
// error code.
using StageFn = std::function<int(size_t, char**)>;

// ---- chain spreading: prepare (checks, layout, packing) and enqueue (copies, kernel), shared by
// cosl_posegraph_spread_chains and cosl_posegraph_solver_submit_chains.
// Slab: inputs [R 9N | t 3N | eR 9N | et 3N | chainOff C+1 | fixed N], outputs [newR 9N | newt 3N | status]
// (read back together), then the anchors [2N].
struct ChainJob {
  int nChains = 0, N = 0;  // N == 0: nothing to solve and nothing to write
  size_t oR = 0, ot = 0, oeR = 0, oet = 0, oOff = 0, oFixed = 0, inBytes = 0, oOut = 0, oAnchor = 0, bytes = 0;
  const int* chainOff = nullptr;  // the caller's arrays
  const uint8_t* fixed = nullptr;
  const double *R = nullptr, *t = nullptr, *eR = nullptr, *et = nullptr;
  const char* staged = nullptr;  // the packed inputs (bytes [0, inBytes) of the slab), or nullptr
};

size_t chain_out_bytes(int N) { return 96 * (size_t)N + 4; }

// outs: the synchronous call's {newR, newt}, checked with the inputs; nullptr for a submit (collect takes
// them).  Without `stage` nothing is packed and the copies read the caller's arrays, which outlive the
// synchronous call: that saves it a host copy of its inputs.
int chain_prepare(const char* fn, int nChains, const int* chainOff, const uint8_t* fixed, const double* R,
                  const double* t, const double* eR, const double* et, const double* const* outs,
                  const StageFn& stage, ChainJob& j) {
  j = ChainJob();
  if (nChains < 0 || !chainOff) return set_error(COSL_E_INVALID, "%s: bad chain table", fn);
  if (nChains == 0) return COSL_OK;
  const int N = chainOff[nChains];
  for (int c = 0; c < nChains; ++c)
    if (chainOff[c + 1] < chainOff[c] || chainOff[0] != 0)
      return set_error(COSL_E_INVALID, "%s: chainOff must start at 0 and be non-decreasing", fn);
  if (N == 0) return COSL_OK;
  if (!fixed || !R || !t || !eR || !et || (outs && (!outs[0] || !outs[1])))
    return set_error(COSL_E_INVALID, "%s: null array", fn);
  SlabLayout L;
  j.oR = L.take(72 * (size_t)N);
  j.ot = L.take(24 * (size_t)N);
  j.oeR = L.take(72 * (size_t)N);
  j.oet = L.take(24 * (size_t)N);
  j.oOff = L.take(4 * (size_t)(nChains + 1));
  j.oFixed = L.take((size_t)N);
  j.inBytes = L.bytes;
  j.oOut = L.take(chain_out_bytes(N));
  j.oAnchor = L.take(8 * (size_t)N);
  j.bytes = L.bytes;
  j.nChains = nChains;
  j.N = N;
  j.chainOff = chainOff;
  j.fixed = fixed;
  j.R = R;
  j.t = t;
  j.eR = eR;
  j.et = et;
  if (stage) {
    char* h = nullptr;
    COSL_TRY(stage(j.inBytes, &h));
    std::memcpy(h + j.oR, R, 72 * (size_t)N);
    std::memcpy(h + j.ot, t, 24 * (size_t)N);
    std::memcpy(h + j.oeR, eR, 72 * (size_t)N);
    std::memcpy(h + j.oet, et, 24 * (size_t)N);
    std::memcpy(h + j.oOff, chainOff, 4 * (size_t)(nChains + 1));
    std::memcpy(h + j.oFixed, fixed, (size_t)N);
    j.staged = h;
  }
  return COSL_OK;
}

// The spread (j.N > 0) on `s` into `slab` (j.bytes): the inputs in one copy from j.staged or section by section
// from the caller's arrays, the kernel, and the outputs in one copy into hostOut (chain_out_bytes, laid out
// as the slab's output region) or into newR, newt and *status.
int chain_enqueue(const char* fn, const ChainJob& j, char* slab, cudaStream_t s, char* hostOut, double* newR,
                  double* newt, int* status) {
  const int N = j.N;
  double *dR = reinterpret_cast<double*>(slab + j.oR), *dt = reinterpret_cast<double*>(slab + j.ot);
  double *deR = reinterpret_cast<double*>(slab + j.oeR), *det = reinterpret_cast<double*>(slab + j.oet);
  int* dOff = reinterpret_cast<int*>(slab + j.oOff);
  unsigned char* dFixed = reinterpret_cast<unsigned char*>(slab + j.oFixed);
  double* dnR = reinterpret_cast<double*>(slab + j.oOut);
  double* dnt = dnR + 9 * (size_t)N;
  int* dStatus = reinterpret_cast<int*>(dnt + 3 * (size_t)N);
  int* dAnchor = reinterpret_cast<int*>(slab + j.oAnchor);
  int rc = COSL_OK;
  auto step = [&](cudaError_t e, const char* what) {
    if (rc == COSL_OK && e != cudaSuccess)
      rc = set_error(COSL_E_CUDA, "%s: %s: %s", fn, what, cudaGetErrorString(e));
  };
  const cudaMemcpyKind h2d = cudaMemcpyHostToDevice, d2h = cudaMemcpyDeviceToHost;
  if (j.staged) {
    step(cudaMemcpyAsync(slab, j.staged, j.inBytes, h2d, s), "H2D");
  } else {
    step(cudaMemcpyAsync(dR, j.R, 72 * (size_t)N, h2d, s), "H2D");
    step(cudaMemcpyAsync(dt, j.t, 24 * (size_t)N, h2d, s), "H2D");
    step(cudaMemcpyAsync(deR, j.eR, 72 * (size_t)N, h2d, s), "H2D");
    step(cudaMemcpyAsync(det, j.et, 24 * (size_t)N, h2d, s), "H2D");
    step(cudaMemcpyAsync(dOff, j.chainOff, 4 * (size_t)(j.nChains + 1), h2d, s), "H2D");
    step(cudaMemcpyAsync(dFixed, j.fixed, (size_t)N, h2d, s), "H2D");
  }
  step(cudaMemsetAsync(dStatus, 0, 4, s), "memset");
  if (rc != COSL_OK) return rc;
  COSL_LAUNCH(posegraph_chain_kernel, j.nChains, PG_THREADS, 0, s, dOff, dFixed, dR, dt, deR, det, dnR, dnt,
              dAnchor, dStatus);
  step(cudaGetLastError(), "launch");
  if (hostOut) {
    step(cudaMemcpyAsync(hostOut, dnR, chain_out_bytes(N), d2h, s), "D2H");
  } else {
    step(cudaMemcpyAsync(newR, dnR, 72 * (size_t)N, d2h, s), "D2H");
    step(cudaMemcpyAsync(newt, dnt, 24 * (size_t)N, d2h, s), "D2H");
    step(cudaMemcpyAsync(status, dStatus, 4, d2h, s), "D2H");
  }
  return rc;
}

// the error the kernel reports through its status word
int chain_status(const char* fn, int status) {
  if (status != 0)
    return set_error(COSL_E_INVALID, "%s: chain %d has no fixed node (rank-deficient system)", fn, status - 1);
  return COSL_OK;
}

// ---- general graphs: prepare (validation, numbering, plan, CSR lists, layout, packing) and enqueue (copies,
// assembly, two tile solves, finish), shared by cosl_posegraph_solve and cosl_posegraph_solver_submit.
struct PgSlab {  // offsets of the slab's sections; [0, in) is the packed input, uploaded in one copy
  size_t R, t, eR, et, fixed, id1, id2, sc, freeNode, freeOf, nodeOff, nodeEdges, colOff, colEdges, pair, unitPos,
      items, itemOff, plan, cnt, in;
  size_t rhs, tiles, rhsS, Linv, y, x, x1, out, bytes;
};

struct PgJob {
  int N = 0, nScale = 0, nF = 0;  // nF == 0: no free node, answered on the host (fixed nodes are copied)
  BaPlan P;
  TileLaunch tile;
  TileImage img;  // layout of the plan's lists, at o.plan
  size_t nCnt = 0, nOut = 0;  // counters of the tile solve; doubles of the output region
  PgSlab o = {};
};

int pg_find(std::vector<int>& parent, int a) {
  while (parent[a] != a) a = parent[a] = parent[parent[a]];
  return a;
}

// outs: the synchronous call's {newR, newt, scale}, checked with the inputs; nullptr for a submit.
int pg_prepare(const char* fn, int nNodes, const uint8_t* fixed, const double* R, const double* t, int nEdges,
               const int* id1, const int* id2, const double* eR, const double* et, const int* scaleCol, int nScale,
               const void* const* outs, const StageFn& stage, PgJob& j) {
  j = PgJob();
  if (nNodes < 0 || nEdges < 0 || nScale < 0) return set_error(COSL_E_INVALID, "%s: negative count", fn);
  if (nNodes > 0 && (!fixed || !R || !t || (outs && (!outs[0] || !outs[1]))))
    return set_error(COSL_E_INVALID, "%s: null node array", fn);
  if (nEdges > 0 && (!id1 || !id2 || !eR || !et)) return set_error(COSL_E_INVALID, "%s: null edge array", fn);
  if (outs && nScale > 0 && !outs[2]) return set_error(COSL_E_INVALID, "%s: null scale array", fn);
  const int N = nNodes, E = nEdges;
  j.N = N;
  j.nScale = nScale;
  // ---- validation: indices, self-loops, rows of the scale columns, components without a fixed node
  std::vector<int> parent(N), colRows(nScale, 0);
  for (int k = 0; k < N; ++k) parent[k] = k;
  for (int e = 0; e < E; ++e) {
    const int i = id1[e], j2 = id2[e], c = scaleCol ? scaleCol[e] : -1;
    if (i < 0 || i >= N || j2 < 0 || j2 >= N)
      return set_error(COSL_E_INVALID, "%s: edge %d joins node %d to node %d (%d nodes)", fn, e, i, j2, N);
    if (i == j2) return set_error(COSL_E_INVALID, "%s: edge %d is a self-loop on node %d", fn, e, i);
    if (c < -1 || c >= nScale)
      return set_error(COSL_E_INVALID, "%s: edge %d has scale column %d (%d columns)", fn, e, c, nScale);
    if (fixed[i] && fixed[j2]) continue;  // no rows (:59, :368)
    if (c >= 0) ++colRows[c];
    const int a = pg_find(parent, i), b = pg_find(parent, j2);
    if (a != b) parent[std::max(a, b)] = std::min(a, b);
  }
  for (int c = 0; c < nScale; ++c)
    if (!colRows[c]) return set_error(COSL_E_INVALID, "%s: scale column %d gets no row", fn, c);
  {
    std::vector<uint8_t> anchored(N, 0);
    for (int k = 0; k < N; ++k)
      if (fixed[k]) anchored[pg_find(parent, k)] = 1;
    for (int k = 0; k < N; ++k)
      if (!fixed[k] && !anchored[pg_find(parent, k)])
        return set_error(COSL_E_INVALID,
                         "%s: node %d lies in a connected component without a fixed node (rank-deficient system)",
                         fn, k);
  }
  // ---- numbering: free nodes, units (two per free node, one per 6 scale columns)
  std::vector<int> freeNode, freeOf(N, -1);
  for (int k = 0; k < N; ++k)
    if (!fixed[k]) {
      freeOf[k] = (int)freeNode.size();
      freeNode.push_back(k);
    }
  const int nF = (int)freeNode.size();
  if (nF == 0) return COSL_OK;  // nothing to solve (and no scale column can have a row)
  j.nF = nF;
  const int nG = (nScale + 5) / 6, mf = 2 * nF + nG;
  // ---- CSR lists in edge order: per free node, per scale column, per node pair
  std::vector<int> nodeOff(nF + 1, 0), colOff(nScale + 1, 0);
  for (int e = 0; e < E; ++e) {
    const int i = id1[e], j2 = id2[e], c = scaleCol ? scaleCol[e] : -1;
    if (fixed[i] && fixed[j2]) continue;
    if (!fixed[i]) ++nodeOff[freeOf[i] + 1];
    if (!fixed[j2]) ++nodeOff[freeOf[j2] + 1];
    if (c >= 0) ++colOff[c + 1];
  }
  for (int f = 0; f < nF; ++f) nodeOff[f + 1] += nodeOff[f];
  for (int c = 0; c < nScale; ++c) colOff[c + 1] += colOff[c];
  std::vector<int> nodeEdges(std::max(1, nodeOff[nF])), colEdges(std::max(1, colOff[nScale]));
  std::map<std::pair<int, int>, std::vector<int>> pairs;  // free-free edges per unordered free pair
  std::vector<std::pair<int, int>> scaleAdj;             // (scale group, free node) with an uncertain edge
  {
    std::vector<int> nf(nodeOff.begin(), nodeOff.end() - 1), cf(colOff.begin(), colOff.end() - 1);
    for (int e = 0; e < E; ++e) {
      const int i = id1[e], j2 = id2[e], c = scaleCol ? scaleCol[e] : -1;
      if (fixed[i] && fixed[j2]) continue;
      if (!fixed[i]) nodeEdges[nf[freeOf[i]]++] = e;
      if (!fixed[j2]) nodeEdges[nf[freeOf[j2]]++] = e;
      if (c >= 0) {
        colEdges[cf[c]++] = e;
        if (!fixed[i]) scaleAdj.push_back({c / 6, freeOf[i]});
        if (!fixed[j2]) scaleAdj.push_back({c / 6, freeOf[j2]});
      }
      if (!fixed[i] && !fixed[j2])
        pairs[{std::min(freeOf[i], freeOf[j2]), std::max(freeOf[i], freeOf[j2])}].push_back(e);
    }
    std::sort(scaleAdj.begin(), scaleAdj.end());
    scaleAdj.erase(std::unique(scaleAdj.begin(), scaleAdj.end()), scaleAdj.end());
  }
  // ---- unit adjacency and the plan
  std::vector<uint8_t> adj((size_t)mf * mf, 0);
  auto link = [&](int a, int b) {
    adj[(size_t)a * mf + b] = 1;
    adj[(size_t)b * mf + a] = 1;
  };
  for (const auto& pr : pairs) {
    link(2 * pr.first.first, 2 * pr.first.second);
    link(2 * pr.first.first + 1, 2 * pr.first.second + 1);
  }
  for (const auto& sa : scaleAdj) link(2 * nF + sa.first, 2 * sa.second + 1);
  j.P = ba_make_plan(mf, adj);
  const BaPlan& P = j.P;
  if (P.nb <= 0) return set_error(COSL_E_NUMERIC, "%s: planning the solve failed", fn);
  j.tile = tile_launch_plan(P);
  j.img = tile_image(P, j.tile);
  // ---- items: every structurally non-zero 6x6 block of the lower triangle, grouped by tile
  std::vector<int> unitPos(mf);
  for (int u = 0; u < mf; ++u) unitPos[u] = P.camBlk[u] * 64 + P.camOff[u];
  std::vector<int> pairEdges;
  std::vector<PgItem> raw;
  auto addItem = [&](int a, int b, int e0, int e1) {
    // the unit later in the elimination order owns the rows
    if (unitPos[a] < unitPos[b]) std::swap(a, b);
    raw.push_back({a, b, P.camOff[a], P.camOff[b], e0, e1});
  };
  for (int u = 0; u < mf; ++u) addItem(u, u, 0, 0);
  for (const auto& pr : pairs) {
    const int e0 = (int)pairEdges.size();
    pairEdges.insert(pairEdges.end(), pr.second.begin(), pr.second.end());
    const int e1 = (int)pairEdges.size();
    addItem(2 * pr.first.first, 2 * pr.first.second, e0, e1);
    addItem(2 * pr.first.first + 1, 2 * pr.first.second + 1, e0, e1);
  }
  for (const auto& sa : scaleAdj) addItem(2 * nF + sa.first, 2 * sa.second + 1, 0, 0);
  if (pairEdges.empty()) pairEdges.push_back(0);
  const int nTiles = P.nTiles, nb = P.nb;
  auto tileOf = [&](const PgItem& it) { return P.tileIdx[(size_t)P.camBlk[it.uR] * nb + P.camBlk[it.uC]]; };
  std::vector<int> itemOff(nTiles + 1, 0);
  for (const PgItem& it : raw) ++itemOff[tileOf(it) + 1];
  for (int q = 0; q < nTiles; ++q) itemOff[q + 1] += itemOff[q];
  std::vector<PgItem> items(raw.size());
  {
    std::vector<int> fill(itemOff.begin(), itemOff.end() - 1);
    for (const PgItem& it : raw) items[fill[tileOf(it)]++] = it;
  }
  std::vector<int> sc(E);
  for (int e = 0; e < E; ++e) sc[e] = scaleCol ? scaleCol[e] : -1;
  // ---- one slab: inputs (uploaded in one copy, counters included as zeros), work, outputs
  const size_t nTilesAll = (size_t)nTiles + P.nScratch;
  j.nCnt = (size_t)P.nCounters + 2 + j.tile.order.size();
  SlabLayout L;
  auto put = [&](size_t bytes) { return L.take(std::max<size_t>(bytes, 8)); };
  PgSlab& o = j.o;
  o.R = put(72 * (size_t)N), o.t = put(24 * (size_t)N), o.eR = put(72 * (size_t)E), o.et = put(24 * (size_t)E);
  o.fixed = put(N), o.id1 = put(4 * (size_t)E), o.id2 = put(4 * (size_t)E), o.sc = put(4 * (size_t)E);
  o.freeNode = put(4 * (size_t)nF), o.freeOf = put(4 * (size_t)N);
  o.nodeOff = put(4 * nodeOff.size()), o.nodeEdges = put(4 * nodeEdges.size());
  o.colOff = put(4 * colOff.size()), o.colEdges = put(4 * colEdges.size());
  o.pair = put(4 * pairEdges.size()), o.unitPos = put(4 * (size_t)mf);
  o.items = put(sizeof(PgItem) * items.size()), o.itemOff = put(4 * itemOff.size());
  o.plan = put(j.img.bytes), o.cnt = put(4 * j.nCnt);
  o.in = L.bytes;
  o.rhs = put(8 * (size_t)nb * 64), o.tiles = put(8 * nTilesAll * 4096);
  o.rhsS = put(8 * (size_t)std::max(1, P.nScratch) * 64), o.Linv = put(8 * (size_t)nb * 4096);
  o.y = put(8 * (size_t)nb * 64), o.x = put(8 * (size_t)nb * 64), o.x1 = put(8 * (size_t)nb * 64);
  // outputs, contiguous: [newR 9N | newt 3N | scale | pivot failure | non-finite]
  j.nOut = 12 * (size_t)N + nScale + 2;
  o.out = put(8 * j.nOut);
  o.bytes = L.bytes;
  char* h = nullptr;
  COSL_TRY(stage(o.in, &h));
  std::memset(h, 0, o.in);
  auto pack = [&](size_t off, const void* src, size_t bytes) {
    if (bytes) std::memcpy(h + off, src, bytes);
  };
  pack(o.R, R, 72 * (size_t)N);
  pack(o.t, t, 24 * (size_t)N);
  pack(o.eR, eR, 72 * (size_t)E);
  pack(o.et, et, 24 * (size_t)E);
  pack(o.fixed, fixed, N);
  pack(o.id1, id1, 4 * (size_t)E);
  pack(o.id2, id2, 4 * (size_t)E);
  pack(o.sc, sc.data(), 4 * (size_t)E);
  pack(o.freeNode, freeNode.data(), 4 * (size_t)nF);
  pack(o.freeOf, freeOf.data(), 4 * (size_t)N);
  pack(o.nodeOff, nodeOff.data(), 4 * nodeOff.size());
  pack(o.nodeEdges, nodeEdges.data(), 4 * nodeEdges.size());
  pack(o.colOff, colOff.data(), 4 * colOff.size());
  pack(o.colEdges, colEdges.data(), 4 * colEdges.size());
  pack(o.pair, pairEdges.data(), 4 * pairEdges.size());
  pack(o.unitPos, unitPos.data(), 4 * (size_t)mf);
  pack(o.items, items.data(), sizeof(PgItem) * items.size());
  pack(o.itemOff, itemOff.data(), 4 * itemOff.size());
  tile_image_write(P, j.tile, j.img, reinterpret_cast<unsigned char*>(h + o.plan));
  return COSL_OK;
}

// The solve (j.nF > 0) on `s` into `slab` (j.o.bytes): the packed inputs in one copy, assembly and tile solve
// twice, pg_finish, and the output region (j.nOut doubles) in one copy into hostOut.
int pg_enqueue(const char* fn, PgJob& j, char* slab, const char* staged, double* hostOut, cudaStream_t s) {
  COSL_TRY(tile_launch_device(j.tile));
  const PgSlab& o = j.o;
  const int N = j.N, nScale = j.nScale, nb = j.P.nb;
  auto at = [&](size_t off) { return slab + off; };
  PgDev d;
  d.R = reinterpret_cast<const double*>(at(o.R));
  d.t = reinterpret_cast<const double*>(at(o.t));
  d.eR = reinterpret_cast<const double*>(at(o.eR));
  d.et = reinterpret_cast<const double*>(at(o.et));
  d.fixed = reinterpret_cast<const unsigned char*>(at(o.fixed));
  d.id1 = reinterpret_cast<const int*>(at(o.id1));
  d.id2 = reinterpret_cast<const int*>(at(o.id2));
  d.scaleCol = reinterpret_cast<const int*>(at(o.sc));
  d.freeNode = reinterpret_cast<const int*>(at(o.freeNode));
  d.freeOf = reinterpret_cast<const int*>(at(o.freeOf));
  d.nodeOff = reinterpret_cast<const int*>(at(o.nodeOff));
  d.nodeEdges = reinterpret_cast<const int*>(at(o.nodeEdges));
  d.colOff = reinterpret_cast<const int*>(at(o.colOff));
  d.colEdges = reinterpret_cast<const int*>(at(o.colEdges));
  d.pairEdges = reinterpret_cast<const int*>(at(o.pair));
  d.unitPos = reinterpret_cast<const int*>(at(o.unitPos));
  d.items = reinterpret_cast<const PgItem*>(at(o.items));
  d.itemOff = reinterpret_cast<const int*>(at(o.itemOff));
  const TileLists tl = tile_lists(j.img, at(o.plan));
  d.diagBlk = tl.diagBlk;
  d.order = tl.order;
  d.blkCam0 = tl.blkCam0;
  d.blkRows = tl.blkRows;
  d.nF = j.nF;
  d.nScale = nScale;
  double* out = reinterpret_cast<double*>(at(o.out));
  BaTileDev b = tile_dev(j.P, j.tile, tl);
  b.rhs = reinterpret_cast<double*>(at(o.rhs));
  b.tiles = reinterpret_cast<double*>(at(o.tiles));
  b.rhsS = reinterpret_cast<double*>(at(o.rhsS));
  b.Linv = reinterpret_cast<double*>(at(o.Linv));
  b.y = reinterpret_cast<double*>(at(o.y));
  b.x = reinterpret_cast<double*>(at(o.x));
  b.cnt = reinterpret_cast<int*>(at(o.cnt));
  b.sc = out + 12 * (size_t)N + nScale;  // the pivot-failure flag
  double* x1 = reinterpret_cast<double*>(at(o.x1));
  int rc = COSL_OK;
  auto cuda_step = [&](cudaError_t e, const char* what) {
    if (rc == COSL_OK && e != cudaSuccess)
      rc = set_error(COSL_E_CUDA, "%s: %s: %s", fn, what, cudaGetErrorString(e));
  };
  cuda_step(cudaMemcpyAsync(slab, staged, o.in, cudaMemcpyHostToDevice, s), "H2D");
  cuda_step(cudaMemsetAsync(b.sc, 0, 16, s), "memset");
  // Normal equations square the condition number (chains of n free nodes: ~n^2), so the solve is
  // followed by one refinement step: assemble again with the residual A^T (b - A x1) as rhs, solve,
  // x = x1 + x2 (the same step as oracle/posegraph_general_oracle.cpp).
  for (int pass = 0; pass < 2 && rc == COSL_OK; ++pass) {
    if (pass == 1) {
      cuda_step(cudaMemcpyAsync(x1, b.x, 8 * (size_t)nb * 64, cudaMemcpyDeviceToDevice, s), "D2D");
      cuda_step(cudaMemsetAsync(b.cnt, 0, 4 * j.nCnt, s), "memset");
    }
    if (rc != COSL_OK) break;
    COSL_LAUNCH(pg_assemble, j.P.nTiles, 256, 0, s, d, pass ? x1 : nullptr, b.tiles, b.rhs);
    cuda_step(cudaGetLastError(), "pg_assemble");
    if (rc == COSL_OK) rc = tile_solve_enqueue(j.tile, b, s);
  }
  if (rc == COSL_OK) {
    const int nThr = std::max(N, nScale);
    COSL_LAUNCH(pg_finish, (unsigned)div_up(nThr, 128), 128, 0, s, d, N, x1, b.x, out, out + 9 * (size_t)N,
                out + 12 * (size_t)N, out + 12 * (size_t)N + nScale + 1);
    cuda_step(cudaGetLastError(), "pg_finish");
  }
  cuda_step(cudaMemcpyAsync(hostOut, out, 8 * j.nOut, cudaMemcpyDeviceToHost, s), "D2H");
  return rc;
}

// The flags pg_finish and the tile solve leave in the output region, then newR, newt and the scales.
int pg_result(const char* fn, int N, int nScale, const double* out, double* newR, double* newt, double* scale) {
  if (out[12 * (size_t)N + nScale] != 0.0)
    return set_error(COSL_E_NUMERIC, "%s: non-positive pivot in the normal equations", fn);
  if (out[12 * (size_t)N + nScale + 1] != 0.0) return set_error(COSL_E_NUMERIC, "%s: non-finite result", fn);
  std::memcpy(newR, out, sizeof(double) * 9 * (size_t)N);
  std::memcpy(newt, out + 9 * (size_t)N, sizeof(double) * 3 * (size_t)N);
  if (nScale) std::memcpy(scale, out + 12 * (size_t)N, sizeof(double) * nScale);
  return COSL_OK;
}

}  // namespace
}  // namespace coslam

using namespace coslam;

extern "C" int cosl_posegraph_spread_chains(int nChains, const int* chainOff, const uint8_t* fixed,
                                            const double* R, const double* t, const double* eR,
                                            const double* et, double* newR, double* newt, int device) {
  const char* fn = "cosl_posegraph_spread_chains";
  const double* outs[2] = {newR, newt};
  ChainJob j;
  COSL_TRY(chain_prepare(fn, nChains, chainOff, fixed, R, t, eR, et, outs, StageFn(), j));
  if (j.N == 0) return COSL_OK;
  COSL_CUDA(cudaSetDevice(device));
  keep_pool(device);
  cudaStream_t s = cudaStreamPerThread;
  char* slab = nullptr;
  COSL_CUDA(cudaMallocAsync(&slab, j.bytes, s));
  int status = 0;
  int rc = chain_enqueue(fn, j, slab, s, nullptr, newR, newt, &status);
  const cudaError_t e = cudaStreamSynchronize(s);
  if (rc == COSL_OK && e != cudaSuccess) rc = set_error(COSL_E_CUDA, "%s: sync: %s", fn, cudaGetErrorString(e));
  cudaFreeAsync(slab, s);
  if (rc != COSL_OK) return rc;
  return chain_status(fn, status);
}

extern "C" double cosl_posegraph_last_host_ms(void) { return g_pgHostMs; }

extern "C" int cosl_posegraph_solve(int nNodes, const uint8_t* fixed, const double* R, const double* t,
                                    int nEdges, const int* id1, const int* id2, const double* eR,
                                    const double* et, const int* scaleCol, int nScale, double* newR,
                                    double* newt, double* scale, int device) {
  const auto tHost0 = std::chrono::steady_clock::now();
  g_pgHostMs = 0.0;
  const char* fn = "cosl_posegraph_solve";
  const void* outs[3] = {newR, newt, scale};
  std::vector<char> host;
  auto stage = [&](size_t bytes, char** buf) {
    host.resize(bytes);
    *buf = host.data();
    return (int)COSL_OK;
  };
  PgJob j;
  COSL_TRY(pg_prepare(fn, nNodes, fixed, R, t, nEdges, id1, id2, eR, et, scaleCol, nScale, outs, stage, j));
  const int N = j.N;
  if (j.nF == 0) {  // fixed nodes are copied
    std::memcpy(newR, R, sizeof(double) * 9 * (size_t)N);
    std::memcpy(newt, t, sizeof(double) * 3 * (size_t)N);
    return COSL_OK;
  }
  g_pgHostMs = 1e3 * std::chrono::duration<double>(std::chrono::steady_clock::now() - tHost0).count();
  // ---- device
  COSL_CUDA(cudaSetDevice(device));
  keep_pool(device);
  cudaStream_t s = cudaStreamPerThread;
  char* slab = nullptr;
  {
    const cudaError_t e = cudaMallocAsync(&slab, j.o.bytes, s);
    if (e == cudaErrorMemoryAllocation) {
      cudaGetLastError();
      return set_error(COSL_E_NOMEM, "%s: device allocation of %zu bytes failed", fn, j.o.bytes);
    }
    if (e != cudaSuccess) return set_error(COSL_E_CUDA, "%s: cudaMallocAsync: %s", fn, cudaGetErrorString(e));
  }
  std::vector<double> hout(j.nOut);
  int rc = pg_enqueue(fn, j, slab, host.data(), hout.data(), s);
  const cudaError_t e = cudaStreamSynchronize(s);
  if (rc == COSL_OK && e != cudaSuccess) rc = set_error(COSL_E_CUDA, "%s: sync: %s", fn, cudaGetErrorString(e));
  cudaFreeAsync(slab, s);
  if (rc != COSL_OK) return rc;
  return pg_result(fn, N, nScale, hout.data(), newR, newt, scale);
}

// A pose-graph solver handle.  One request in flight at a time, of either kind; the device slab and the
// pinned staging buffers serve both kinds and grow when a request does not fit.
struct cosl_posegraph_solver {
  int device = 0;
  RequestStream rq;
  char* slab = nullptr;  // from the device's stream-ordered pool, on rq.stream
  char* h_in = nullptr;  // pinned: the packed inputs
  char* h_out = nullptr; // pinned: the output region of the slab
  size_t slabBytes = 0, inBytes = 0, outBytes = 0;
  bool chains = false;    // the request in flight: a chain spread or a general solve
  int N = 0, nScale = 0;  // its nodes (0: nothing to write) and scale columns
};

namespace {

void free_pg_solver(cosl_posegraph_solver* s) {
  cudaSetDevice(s->device);
  if (s->slab) cudaFreeAsync(s->slab, s->rq.stream);
  s->rq.destroy();
  if (s->h_in) cudaFreeHost(s->h_in);
  if (s->h_out) cudaFreeHost(s->h_out);
  delete s;
}

// Grows a pinned buffer to `need` bytes.  Only called with nothing in flight, so no copy reads the old one.
int grow_pinned(const char* fn, char** buf, size_t* cap, size_t need) {
  if (need <= *cap) return COSL_OK;
  if (*buf) cudaFreeHost(*buf);
  *buf = nullptr;
  *cap = 0;
  const cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(buf), need, cudaHostAllocPortable);
  if (e != cudaSuccess) {
    *buf = nullptr;
    cudaGetLastError();
    return set_error(e == cudaErrorMemoryAllocation ? COSL_E_NOMEM : COSL_E_CUDA,
                     "%s: pinned allocation of %zu bytes failed: %s", fn, need, cudaGetErrorString(e));
  }
  *cap = need;
  return COSL_OK;
}

// Grows the device slab in stream order: the old slab goes back to the pool behind the work already on
// the handle's stream, and the new one comes out of it without a device synchronisation.
int grow_slab(const char* fn, cosl_posegraph_solver* s, size_t need) {
  if (need <= s->slabBytes) return COSL_OK;
  if (s->slab) cudaFreeAsync(s->slab, s->rq.stream);
  s->slab = nullptr;
  s->slabBytes = 0;
  const cudaError_t e = cudaMallocAsync(&s->slab, need, s->rq.stream);
  if (e != cudaSuccess) {
    s->slab = nullptr;
    cudaGetLastError();
    return set_error(e == cudaErrorMemoryAllocation ? COSL_E_NOMEM : COSL_E_CUDA,
                     "%s: device allocation of %zu bytes failed: %s", fn, need, cudaGetErrorString(e));
  }
  s->slabBytes = need;
  return COSL_OK;
}

StageFn stage_pinned(const char* fn, cosl_posegraph_solver* s) {
  return [fn, s](size_t bytes, char** buf) {
    COSL_TRY(grow_pinned(fn, &s->h_in, &s->inBytes, bytes));
    *buf = s->h_in;
    return (int)COSL_OK;
  };
}

}  // namespace

extern "C" {

int cosl_posegraph_solver_create(int device, cosl_posegraph_solver** out) {
  if (!out || device < 0) return set_error(COSL_E_INVALID, "cosl_posegraph_solver_create: bad argument");
  *out = nullptr;
  COSL_TRY(check_device(device));
  cosl_posegraph_solver* s = new (std::nothrow) cosl_posegraph_solver;
  if (!s) return set_error(COSL_E_NOMEM, "cosl_posegraph_solver_create: out of host memory");
  s->device = device;
  auto init = [&]() {
    COSL_CUDA(cudaSetDevice(device));
    keep_pool(device);
    return s->rq.create();
  };
  const int rc = init();
  if (rc != COSL_OK) {
    free_pg_solver(s);
    return rc;
  }
  *out = s;
  return COSL_OK;
}

int cosl_posegraph_solver_destroy(cosl_posegraph_solver* s) {
  if (!s) return set_error(COSL_E_INVALID, "null pose-graph solver handle");
  free_pg_solver(s);
  return COSL_OK;
}

int cosl_posegraph_solver_submit_chains(cosl_posegraph_solver* s, int nChains, const int* chainOff,
                                        const uint8_t* fixed, const double* R, const double* t,
                                        const double* eR, const double* et) {
  const char* fn = "cosl_posegraph_solver_submit_chains";
  if (!s) return set_error(COSL_E_INVALID, "null pose-graph solver handle");
  COSL_TRY(s->rq.idle(fn));
  COSL_CUDA(cudaSetDevice(s->device));
  ChainJob j;
  COSL_TRY(chain_prepare(fn, nChains, chainOff, fixed, R, t, eR, et, nullptr, stage_pinned(fn, s), j));
  if (j.N > 0) {
    COSL_TRY(grow_pinned(fn, &s->h_out, &s->outBytes, chain_out_bytes(j.N)));
    COSL_TRY(grow_slab(fn, s, j.bytes));
  }
  s->chains = true;
  s->N = j.N;
  s->nScale = 0;
  return s->rq.submit(fn, [&]() {
    return j.N > 0 ? chain_enqueue(fn, j, s->slab, s->rq.stream, s->h_out, nullptr, nullptr, nullptr) : (int)COSL_OK;
  });
}

int cosl_posegraph_solver_submit(cosl_posegraph_solver* s, int nNodes, const uint8_t* fixed, const double* R,
                                 const double* t, int nEdges, const int* id1, const int* id2, const double* eR,
                                 const double* et, const int* scaleCol, int nScale) {
  const char* fn = "cosl_posegraph_solver_submit";
  if (!s) return set_error(COSL_E_INVALID, "null pose-graph solver handle");
  COSL_TRY(s->rq.idle(fn));
  COSL_CUDA(cudaSetDevice(s->device));
  PgJob j;
  COSL_TRY(pg_prepare(fn, nNodes, fixed, R, t, nEdges, id1, id2, eR, et, scaleCol, nScale, nullptr,
                      stage_pinned(fn, s), j));
  const int N = j.N;
  COSL_TRY(grow_pinned(fn, &s->h_out, &s->outBytes, 8 * (12 * (size_t)N + nScale + 2)));
  if (j.nF == 0) {  // answered on the host, as the synchronous call does: the fixed nodes are copied
    double* out = reinterpret_cast<double*>(s->h_out);
    std::memcpy(out, R, sizeof(double) * 9 * (size_t)N);
    std::memcpy(out + 9 * (size_t)N, t, sizeof(double) * 3 * (size_t)N);
    out[12 * (size_t)N] = out[12 * (size_t)N + 1] = 0.0;  // no failure flags (nScale is 0)
  } else {
    COSL_TRY(grow_slab(fn, s, j.o.bytes));
  }
  s->chains = false;
  s->N = N;
  s->nScale = nScale;
  return s->rq.submit(fn, [&]() {
    return j.nF > 0 ? pg_enqueue(fn, j, s->slab, s->h_in, reinterpret_cast<double*>(s->h_out), s->rq.stream)
                    : (int)COSL_OK;
  });
}

int cosl_posegraph_solver_query(cosl_posegraph_solver* s, int* done) {
  if (!s || !done) return set_error(COSL_E_INVALID, "cosl_posegraph_solver_query: null argument");
  COSL_TRY(s->rq.pending("cosl_posegraph_solver_query"));
  COSL_CUDA(cudaSetDevice(s->device));
  return s->rq.query(done);
}

int cosl_posegraph_solver_collect(cosl_posegraph_solver* s, double* newR, double* newt, double* scale,
                                  double* device_ms) {
  const char* fn = "cosl_posegraph_solver_collect";
  if (!s) return set_error(COSL_E_INVALID, "null pose-graph solver handle");
  COSL_TRY(s->rq.pending(fn));
  if ((s->N > 0 && (!newR || !newt)) || (s->nScale > 0 && !scale))
    return set_error(COSL_E_INVALID, "%s: null output array", fn);
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.wait(device_ms));
  const int N = s->N;
  if (!s->chains) return pg_result(fn, N, s->nScale, reinterpret_cast<const double*>(s->h_out), newR, newt, scale);
  if (N == 0) return COSL_OK;
  const double* out = reinterpret_cast<const double*>(s->h_out);
  int status = 0;
  std::memcpy(&status, out + 12 * (size_t)N, sizeof(int));
  COSL_TRY(chain_status(fn, status));
  std::memcpy(newR, out, sizeof(double) * 9 * (size_t)N);
  std::memcpy(newt, out + 9 * (size_t)N, sizeof(double) * 3 * (size_t)N);
  return COSL_OK;
}

void* cosl_posegraph_solver_stream(cosl_posegraph_solver* s) { return s ? (void*)s->rq.stream : nullptr; }

}  // extern "C"
