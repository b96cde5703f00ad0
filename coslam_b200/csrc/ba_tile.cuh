// ba_tile.cuh -- device side of the reduced-camera-system solve (fp64, sm_90a).
//
// Replaces the dense LAPACK solve inside sba_motstr_levmar_x (reference call
// app/SL_CoSLAMBA.cpp:360-363; BA-4 step v and 8f-1 of SURVEY.md).  Planning (ordering, blocking,
// symbolic fill, task DAG) is done once per solver on the host, see ba_plan.h.
//
// Storage in HBM:  S = [ rhs (nb*64, block padded) | tiles ]: tile t = 64x64 doubles, column-major
// (element (r, c) at c*64 + r), only the structurally non-zero lower tiles of the permuted system
// exist; the tiles the Schur contraction can write come first, so [rhs | those tiles] is one
// contiguous buffer for the multi-GPU all-reduce.  Linv[k] (64x64, column-major), y and x are block
// padded like rhs.
//
// ba_tile_solve: ONE persistent launch for factorisation + both substitutions.  Every CTA takes the
// next task of the critical-path-first list with an atomic ticket, waits (one polling thread,
// ld.acquire.gpu) until the per-tile counters say its operands are final, executes it on tiles
// staged in shared memory, publishes the result (fence + red.release on the counter).  All tile
// reads bypass L1 (ld.global.cg): tiles are rewritten by other SMs during the launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ba_plan.h"
#include "tile_solve.h"  // BaTileDev

namespace coslam {

constexpr int BA_LDS = 68;                                   // smem leading dimension of a staged tile
constexpr int BA_TILE_SMEM_DOUBLES = 3 * BA_TB * BA_LDS + 8 * BA_TB + 8 * BA_TB + 2 * BA_TB + 96;
constexpr int BA_TILE_SMEM = BA_TILE_SMEM_DOUBLES * (int)sizeof(double);
constexpr int BA_NTHREADS = 256;

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ba_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void red_release_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// global column-major 64x64 tile -> shared [col][row] with leading dimension LD; all 8 loads of a
// thread are in flight before the first shared store (one L2 round trip per tile)
template <int LD>
__device__ __forceinline__ void tile_load(const double* __restrict__ g, double* __restrict__ s, int tid) {
  double2 v[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const double2*>(g) + tid + BA_NTHREADS * u);
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int e = 2 * (tid + BA_NTHREADS * u);
    const int c = e >> 6, r = e & 63;
    *reinterpret_cast<double2*>(s + c * LD + r) = v[u];
  }
}

// two tiles at once (16 loads in flight)
template <int LD>
__device__ __forceinline__ void tile_load2(const double* __restrict__ g0, double* __restrict__ s0,
                                           const double* __restrict__ g1, double* __restrict__ s1, int tid) {
  double2 v0[8], v1[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    v0[u] = __ldcg(reinterpret_cast<const double2*>(g0) + tid + BA_NTHREADS * u);
    v1[u] = __ldcg(reinterpret_cast<const double2*>(g1) + tid + BA_NTHREADS * u);
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int e = 2 * (tid + BA_NTHREADS * u);
    const int c = e >> 6, r = e & 63;
    *reinterpret_cast<double2*>(s0 + c * LD + r) = v0[u];
    *reinterpret_cast<double2*>(s1 + c * LD + r) = v1[u];
  }
}

// ---------------------------------------------------------------------------------------------
// acc(r, c) = sum_{p < kk} sA[p][r] * sB[p][c]   (both operands staged [p][row], ld = BA_LDS)
// Tensor-core version: fp64 DMMA m8n8k4.  Warp w owns rows 16*(w&3).. (2 fragments) and columns
// 32*(w>>2).. (4 fragments); lane l holds A(row l/4, k l%4), B(k l%4, col l/4) and
// C(row l/4, cols 2*(l%4), 2*(l%4)+1) of each 8x8 fragment.  BA_LDS = 68 makes the fragment loads
// conflict free (half-warp: 4*(l%4) + l/4 covers 16 distinct bank pairs).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

struct TileAcc {
  double c[2][4][2];
};

__device__ __forceinline__ void tile_gemm_dmma(const double* __restrict__ sA, const double* __restrict__ sB,
                                               int kk, int tid, TileAcc& acc) {
  const int lane = tid & 31, w = tid >> 5;
  const int mB = (w & 3) * 16 + (lane >> 2), nB = (w >> 2) * 32 + (lane >> 2), kl = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) acc.c[mi][ni][0] = acc.c[mi][ni][1] = 0.0;
  for (int p0 = 0; p0 < kk; p0 += 4) {
    const double* pa = sA + (p0 + kl) * BA_LDS + mB;
    const double* pb = sB + (p0 + kl) * BA_LDS + nB;
    const double a0 = pa[0], a1 = pa[8];
    const double b0 = pb[0], b1 = pb[8], b2 = pb[16], b3 = pb[24];
    dmma884(acc.c[0][0][0], acc.c[0][0][1], a0, b0);
    dmma884(acc.c[0][1][0], acc.c[0][1][1], a0, b1);
    dmma884(acc.c[0][2][0], acc.c[0][2][1], a0, b2);
    dmma884(acc.c[0][3][0], acc.c[0][3][1], a0, b3);
    dmma884(acc.c[1][0][0], acc.c[1][0][1], a1, b0);
    dmma884(acc.c[1][1][0], acc.c[1][1][1], a1, b1);
    dmma884(acc.c[1][2][0], acc.c[1][2][1], a1, b2);
    dmma884(acc.c[1][3][0], acc.c[1][3][1], a1, b3);
  }
}

// fragment element -> (row, col) inside the 64x64 tile
__device__ __forceinline__ void tile_acc_rc(int tid, int mi, int ni, int e, int& r, int& c) {
  const int lane = tid & 31, w = tid >> 5;
  r = (w & 3) * 16 + 8 * mi + (lane >> 2);
  c = (w >> 2) * 32 + 8 * ni + 2 * (lane & 3) + e;
}

// x = L^-T v for 64 threads (warps 0-1; named barrier 2): blocks last to first, right-looking --
// after x_b = M_b^T v_b every remaining v_p gets its update from block row b at once.
__device__ __forceinline__ void tile_bwd3(const double* __restrict__ sL, const double* __restrict__ sM,
                                          double* __restrict__ sv, double* __restrict__ sx, int nbk, int t) {
  double v = sv[t];
  for (int b = nbk - 1; b >= 0; --b) {
    const bool mine = (t >> 3) == b;
    if (mine) sv[t] = v;
    asm volatile("bar.sync 2, 64;" ::: "memory");
    if (mine) {
      const int q = t & 7;
      double x0 = 0, x1 = 0;
#pragma unroll
      for (int qq = 0; qq < 8; qq += 2) {
        x0 = __fma_rn(sM[b * 64 + qq * 8 + q], sv[8 * b + qq], x0);  // M lower: zero for qq < q
        x1 = __fma_rn(sM[b * 64 + (qq + 1) * 8 + q], sv[8 * b + qq + 1], x1);
      }
      sx[t] = x0 + x1;
    }
    asm volatile("bar.sync 2, 64;" ::: "memory");
    if (t < 8 * b) {
      double s0 = 0, s1 = 0;
#pragma unroll
      for (int q = 0; q < 8; q += 2) {
        s0 = __fma_rn(sL[t * BA_LDS + 8 * b + q], sx[8 * b + q], s0);
        s1 = __fma_rn(sL[t * BA_LDS + 8 * b + q + 1], sx[8 * b + q + 1], s1);
      }
      v -= s0 + s1;
    }
  }
}

// =============================================================================================
// Version 2 of the diagonal-block path: no explicit 64x64 inverse.
//   POTRF2 : factor with 8-column panels and LOOK-AHEAD: warps 0-1 ("panel warps", thread = row)
//            own the pivot chain -- they factor the 8x8 diagonal block redundantly in registers,
//            solve their row of the panel, and apply the rank-8 update to the NEXT panel's columns
//            themselves (kept in registers) -- while warps 2-7 apply it to the rest of the trailing
//            triangle and to the right-hand side, off the chain.  One CTA barrier + one 64-thread
//            named barrier per panel.  Outputs: L (lower, in place), the inverses M_b of the eight
//            8x8 diagonal blocks of L, and y = L^-1 b.
//   TRSM2  : X L^T = A by blocked substitution over the 8 column blocks; every warp owns 8 rows and
//            needs no CTA barrier: T_b = A_b - X_{<b} L_{b,<b}^T and X_b = T_b M_b^T are DMMA m8n8k4
//            products (2b + 2 per block).
//   BWD2   : x = L^-T v by the same blocking, one warp.
// =============================================================================================
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// sT: tile staged column-major with ld BA_LDS (element (r, c) at c*BA_LDS + r), lower part valid,
// identity on the padding.  sBv: right-hand side (64); sYv: y out (64); sM: [8][8][8] M_b[q][q']
// out; sD: 80 doubles scratch.
// The panel warps are alone on their schedulers, so their time is their instruction count: every
// row -- the panel's own rows included -- runs the same row solve (for a panel row it yields the row
// of the Cholesky factor), and the 8x8 inverses are left to the update warps.
__device__ __forceinline__ double ba_rsqrt_pivot(double d) {
  // pivots of a damped Gauss-Newton system lie far inside the float range (checked by the caller)
  double y = (double)rsqrtf((float)d);
  const double h = 0.5 * d;
  y = __fma_rn(y, __fma_rn(-h * y, y, 0.5), y);
  y = __fma_rn(y, __fma_rn(-h * y, y, 0.5), y);
  return y;
}

__device__ __forceinline__ void tile_potrf2(double* __restrict__ sT, double* __restrict__ sBv,
                                            double* __restrict__ sYv, double* __restrict__ sM,
                                            double* __restrict__ sD, int tid, int* s_fail, int nbp = 8) {
  // nbp = number of 8-column panels that hold real rows ((rows + 7) / 8): the padding of a partial block is
  // the identity and needs no work (its L columns stay as staged, its y and M_b are never read)
  const bool isP = tid < 64;
  const int r = tid;
  double a[8], x[8];
  double br = isP ? sBv[r] : 0.0;  // this row's right-hand side, updated along with the look-ahead
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    a[q] = isP ? sT[q * BA_LDS + r] : 0.0;
    x[q] = 0.0;
  }
#pragma unroll 1
  for (int pb = 0; pb < nbp; ++pb) {
    const int c0 = 8 * pb;
    if (isP) {
      if (r >= c0 && r < c0 + 8) {
#pragma unroll
        for (int q = 0; q < 8; ++q) sD[(r - c0) * 8 + q] = a[q];
        sD[64 + r - c0] = br;
      }
      named_bar_sync(1, 64);
      double D[8][8], inv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) D[i][j] = sD[i * 8 + j];
      bool bad = false;
#pragma unroll
      for (int p = 0; p < 8; ++p) {
        double dd = D[p][p];
        if (!(dd > 1e-30 && dd < 1e30)) {  // also catches NaN
          bad = true;
          dd = 1.0;
        }
        const double rs = ba_rsqrt_pivot(dd);
        inv[p] = rs;
#pragma unroll
        for (int i = p + 1; i < 8; ++i) D[i][p] *= rs;
#pragma unroll
        for (int j = p + 1; j < 8; ++j)
#pragma unroll
          for (int i = j; i < 8; ++i) D[i][j] = __fma_rn(-D[i][p], D[j][p], D[i][j]);
      }
      if (r == 0) {  // y of this panel and the reciprocal diagonal, for the other warps
        double yv[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          double s = sD[64 + q];
#pragma unroll
          for (int p = 0; p < q; ++p) s = __fma_rn(-D[q][p], yv[p], s);
          yv[q] = s * inv[q];
          sYv[c0 + q] = yv[q];
          sD[72 + 8 * (pb & 1) + q] = inv[q];  // double buffered: read by the update warps of this panel
        }
        if (bad) *s_fail = 1;
      }
      if (r >= c0) {
        // row solve x L_D^T = a.  For a row of the panel itself (r = c0 + cc) the entries q <= cc are
        // exactly row cc of the Cholesky factor; the ones right of the diagonal are zeroed.
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          double s = a[q];
#pragma unroll
          for (int p = 0; p < q; ++p) s = __fma_rn(-x[p], D[q][p], s);
          x[q] = (c0 + q <= r) ? s * inv[q] : 0.0;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) sT[(c0 + q) * BA_LDS + r] = x[q];
      }
    }
    __syncthreads();  // X and y of this panel are visible; the update warps finished the previous panel
    if (isP) {
      if (pb + 1 < nbp && r >= c0 + 8) {  // look-ahead: next panel's columns of this row, kept in registers
#pragma unroll
        for (int qn = 0; qn < 8; ++qn) a[qn] = sT[(c0 + 8 + qn) * BA_LDS + r];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const double2* xr = reinterpret_cast<const double2*>(sT + (c0 + q) * BA_LDS + c0 + 8);
#pragma unroll
          for (int h2 = 0; h2 < 4; ++h2) {
            const double2 xx = xr[h2];  // X(c0+8+2h2, q), X(c0+9+2h2, q)
            a[2 * h2] = __fma_rn(-x[q], xx.x, a[2 * h2]);
            a[2 * h2 + 1] = __fma_rn(-x[q], xx.y, a[2 * h2 + 1]);
          }
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) br = __fma_rn(-x[q], sYv[c0 + q], br);  // b_r -= X(r, :) y_panel
      }
    } else {
      const int u = tid - 64;  // 0 .. 191
      if (u >= 184) {
        // inverse of the panel's 8x8 factor block, column cc per thread: M e_cc by forward substitution
        const int cc = u - 184;
        double m[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          double s = (q == cc) ? 1.0 : 0.0;
#pragma unroll
          for (int p = 0; p < q; ++p) s = __fma_rn(-sT[(c0 + p) * BA_LDS + c0 + q], m[p], s);
          m[q] = s * sD[72 + 8 * (pb & 1) + q];
          sM[pb * 64 + q * 8 + cc] = m[q];
        }
      }
      // trailing lower triangle right of the NEXT panel (rows / columns >= c0 + 16), in 8x8 blocks on the
      // fp64 tensor cores: C(R0.., C0..) -= X(R0.., c0..c0+7) X(C0.., c0..c0+7)^T = two DMMA.8x8x4 per block.
      // (The scalar version -- a chain of 8 dependent DMULs/DFMAs per element, ~24 elements per thread one
      // after the other -- made the UPDATE warps, not the pivot chain, the slow side of a panel.)
      // Diagonal blocks are computed in full: their upper halves are never read as factor entries.
      {
        const int uw = (tid >> 5) - 2;              // update warp 0..5
        const int lane = tid & 31, g = lane >> 2, kq = lane & 3;
        const int t0 = pb + 2;                      // first 8-row block of the trailing part
        const int nt = nbp - t0;                    // blocks per side (padding blocks need no update)
        const int ntile = nt * (nt + 1) / 2;
        const double* xk0 = sT + (c0 + kq) * BA_LDS;       // X(., c0 + kq)
        const double* xk1 = sT + (c0 + 4 + kq) * BA_LDS;   // X(., c0 + 4 + kq)
        for (int t = uw; t < ntile; t += 6) {
          // t -> (bi >= bj) in the lower triangle of an nt x nt block grid, row by row
          int bi = 0, rem = t;
          while (rem > bi) {
            rem -= bi + 1;
            ++bi;
          }
          const int R0 = 8 * (t0 + bi), C0 = 8 * (t0 + rem);
          double* cp = sT + (C0 + 2 * kq) * BA_LDS + R0 + g;
          double c0v = cp[0], c1v = cp[BA_LDS];
          const double a0 = -xk0[R0 + g], a1 = -xk1[R0 + g];
          const double b0 = xk0[C0 + g], b1 = xk1[C0 + g];
          dmma884(c0v, c1v, a0, b0);
          dmma884(c0v, c1v, a1, b1);
          cp[0] = c0v;
          cp[BA_LDS] = c1v;
        }
      }
    }
  }
  __syncthreads();  // the last panel's inverse block (written by the update warps)
}

// X L^T = A in place in sA (rows = this warp's 8 rows; ld BA_LDS); sL: L staged like sA; sM: M_b.
// nbk = number of 8-column blocks to process.
__device__ __forceinline__ void tile_trsm2(double* __restrict__ sA, const double* __restrict__ sL,
                                           const double* __restrict__ sM, int nbk, int tid) {
  const int lane = tid & 31, w = tid >> 5;
  const int rb = 8 * w, lr = lane >> 2, lk = lane & 3;
  for (int b = 0; b < nbk; ++b) {
    double c0 = 0.0, c1 = 0.0;
    for (int p0 = 0; p0 < 8 * b; p0 += 4) {
      const double av = sA[(p0 + lk) * BA_LDS + rb + lr];         // X(row, p)
      const double bv = sL[(p0 + lk) * BA_LDS + 8 * b + lr];      // L(8b + n, p)
      dmma884(c0, c1, av, bv);
    }
    // T = A_b - acc, written over A_b (C layout: row lr, columns 2 lk, 2 lk + 1)
    double* t0 = sA + (8 * b + 2 * lk) * BA_LDS + rb + lr;
    t0[0] -= c0;
    t0[BA_LDS] -= c1;
    __syncwarp();
    const double a0 = sA[(8 * b + lk) * BA_LDS + rb + lr], a1 = sA[(8 * b + 4 + lk) * BA_LDS + rb + lr];
    const double m0 = sM[b * 64 + lr * 8 + lk], m1 = sM[b * 64 + lr * 8 + 4 + lk];  // B(k, n) = M(n, k)
    double x0 = 0.0, x1 = 0.0;
    dmma884(x0, x1, a0, m0);
    dmma884(x0, x1, a1, m1);
    __syncwarp();
    t0[0] = x0;
    t0[BA_LDS] = x1;
    __syncwarp();
  }
}


// UPDATE task body: C -= A B^T (first update of a scratch tile overwrites), diagonal tiles also
// b_i -= A y_k.  staged: the operands (and y in sY) are already in shared memory.
__device__ __forceinline__ void ba_upd_body(const BaTileDev& d, const BaTask& t, int ti, double* sA, double* sB,
                                            double* sY, int bk, int tid, bool staged) {
  double* gC = d.tiles + (size_t)t.tC * BA_TILE;
  const bool over = (t.flags & 2) != 0;
  double cold[2][4][2];
  if (!over) {  // C prefetch (independent of the operand staging: one round trip for everything)
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          int r, c;
          tile_acc_rc(tid, mi, ni, e, r, c);
          cold[mi][ni][e] = __ldcg(gC + c * BA_TB + r);
        }
  }
  if (!staged) {
    tile_load<BA_LDS>(d.tiles + (size_t)t.tB * BA_TILE, sB, tid);  // B = L_jk and C: awaited up front
    if ((t.flags & 1) && tid < 64) sY[tid] = __ldcg(d.y + (size_t)t.k * BA_TB + tid);
    if (tid == 0 && t.w1i >= 0)
      while (ld_acquire(d.cnt + t.w1i) < t.w1v) {}  // A = L_ik (deferred wait)
    __syncthreads();
    tile_load<BA_LDS>(d.tiles + (size_t)t.tA * BA_TILE, sA, tid);
    __syncthreads();
  }
  if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 4] = ba_globaltimer();
  TileAcc acc;
  tile_gemm_dmma(sA, sB, (bk + 3) & ~3, tid, acc);
  if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 5] = ba_globaltimer();
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int r, c;
        tile_acc_rc(tid, mi, ni, e, r, c);
        gC[c * BA_TB + r] = (over ? 0.0 : cold[mi][ni][e]) - acc.c[mi][ni][e];
      }
  if ((t.flags & 1) && tid < 64) {
    // b_i -= L_ik y_k (sequenced with the updates of the diagonal tile)
    double sum = 0;
    for (int p = 0; p < bk; ++p) sum = __fma_rn(sA[p * BA_LDS + tid], sY[p], sum);
    double* b = (t.l0 >= 0) ? d.rhsS + (size_t)t.l0 * BA_TB + tid : d.rhs + (size_t)t.i * BA_TB + tid;
    *b = (over ? 0.0 : __ldcg(b)) - sum;
  }
}

// ---------------------------------------------------------------------------------------------
// The persistent dataflow kernel.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BA_NTHREADS, 1) ba_tile_solve(BaTileDev d) {
  extern __shared__ double smem[];
  double* sA = smem;                       // [64][68]
  double* sB = sA + BA_TB * BA_LDS;        // [64][68]
  double* sC = sB + BA_TB * BA_LDS;        // [64][68]
  double* sX = sC + BA_TB * BA_LDS;        // [8][64] x vectors of a BWD chunk
  double* sM = sX + 8 * BA_TB;             // [8][8][8] inverses of the diagonal 8x8 blocks
  double* sV = sM + 8 * BA_TB;             // [64]
  double* sY = sV + BA_TB;                 // [64]
  double* sD = sY + BA_TB;                 // [80] panel scratch of tile_potrf2
  __shared__ int s_task, s_fail, s_flag;
  __shared__ BaTask s_ht, s_hu;  // hot successors of the POTRF in flight
  const int tid = threadIdx.x;
  int* const claim = d.cnt + d.nCounters + 2;  // [nTasks]: 1 = somebody executes / executed the task
  const bool special = (int)blockIdx.x < d.nSpecial;
  int* const ticket = d.cnt + d.nCounters + (special ? 0 : 1);
  const int tBase = special ? 0 : d.nA, tCount = special ? d.nA : d.nTasks - d.nA;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      s_task = atomicAdd(ticket, 1);
      s_fail = 0;
    }
    __syncthreads();
    if (s_task >= tCount) break;
    const int ti = tBase + s_task;
    const BaTask t = d.tasks[ti];
    if (tid < 32) {
      if (tid == 0 && d.trace) {
        unsigned int smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        d.trace[8 * (size_t)ti] = smid;
        d.trace[8 * (size_t)ti + 1] = ba_globaltimer();
      }
      // the lanes of warp 0 poll different counters concurrently
      // TRSM defers the wait for its own tile (w0) and UPD the wait for its A operand (w1) until the other
      // operands are on their way into shared memory: on the dependency chains those are the late ones
      if (tid == 0 && t.w0i >= 0 && t.type != BA_T_TRSM)
        while (ld_acquire(d.cnt + t.w0i) < t.w0v) {}
      if (tid == 1 && t.w1i >= 0 && t.type != BA_T_UPD)
        while (ld_acquire(d.cnt + t.w1i) < t.w1v) {}
      if (tid == 2 && t.w2i >= 0)
        while (ld_acquire(d.cnt + t.w2i) < t.w2v) {}
      // (BWD polls the x_i it needs chunk by chunk, see below)
      if (t.type == BA_T_SUM)
        for (int e = t.l0 + tid; e < t.l1; e += 32)
          while (ld_acquire(d.cnt + d.sum[e].tile) < d.sum[e].count) {}
      __syncwarp();
      if (tid == 0 && d.trace) d.trace[8 * (size_t)ti + 2] = ba_globaltimer();
    }
    __syncthreads();
    const int bk = d.blkRows[t.k];
    if (t.type == BA_T_TRSM || t.type == BA_T_UPD) {
      // the CTA that factored the pivot block may already have run this task (hot successors)
      if (tid == 0) s_flag = (atomicCAS(claim + ti, 0, 1) == 0) ? 1 : 0;
      __syncthreads();
      if (!s_flag) continue;
    }
    if (t.type == BA_T_POTRF) {
      if (tid == 255 && t.l0 >= 0) s_ht = d.tasks[t.l0];
      if (tid == 254 && t.l1 >= 0) s_hu = d.tasks[t.l1];
      // stage the lower part (ld BA_LDS), identity on the padding; b into sV
      {
        const double* g = d.tiles + (size_t)t.tC * BA_TILE;
        double2 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const double2*>(g) + tid + BA_NTHREADS * u);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = 2 * (tid + BA_NTHREADS * u);
          const int c = e >> 6, r = e & 63;
          double2 w = v[u];
          if (r >= bk || c >= bk) w.x = (r == c) ? 1.0 : 0.0;
          if (r + 1 >= bk || c >= bk) w.y = (r + 1 == c) ? 1.0 : 0.0;
          *reinterpret_cast<double2*>(sA + c * BA_LDS + r) = w;
        }
        if (tid < 64) sV[tid] = (tid < bk) ? __ldcg(d.rhs + (size_t)t.k * BA_TB + tid) : 0.0;
      }
      __syncthreads();
      if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 4] = ba_globaltimer();
      tile_potrf2(sA, sV, sY, sM, sD, tid, &s_fail, (bk + 7) >> 3);
      if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 5] = ba_globaltimer();
      {
        double* g = d.tiles + (size_t)t.tC * BA_TILE;  // L in place (lower), zeros above
        for (int e = tid; e < BA_TILE; e += BA_NTHREADS) {
          const int c = e >> 6, r = e & 63;
          g[e] = (r >= c) ? sA[c * BA_LDS + r] : 0.0;
        }
        double* gm = d.Linv + (size_t)t.k * BA_TILE;  // the eight 8x8 inverses
        gm[tid] = sM[tid];
        gm[tid + BA_NTHREADS] = sM[tid + BA_NTHREADS];
        if (tid < 64) d.y[(size_t)t.k * BA_TB + tid] = sY[tid];
        if (tid == 0 && s_fail) d.sc[d.scFail] = 1.0;
      }
      // ---- hot successors: the next pivot of the chain needs TRSM(j, k) and UPD(j, j, k) with
      // j = first block of struct(k).  If their other operands are ready, this CTA runs them now
      // with L_kk, the M_b and y_k still in shared memory: two hand-overs, two tile loads and
      // two publish/acquire round trips less per step of the critical path.  Claimed BEFORE the
      // factor is published so that no waiting CTA wins the race; conditions are monotone.
      if (tid == 0) {
        int hot = 0;
        // (descriptors were fetched into shared memory while the factorisation ran)
        const bool rT = t.l0 >= 0 && ld_acquire(d.cnt + s_ht.w0i) >= s_ht.w0v;
        const bool rU = t.l1 >= 0 && ld_acquire(d.cnt + s_hu.w0i) >= s_hu.w0v;
        if (rT && atomicCAS(claim + t.l0, 0, 1) == 0) hot = 1;
        if (hot && rU && atomicCAS(claim + t.l1, 0, 1) == 0) hot = 3;
        s_flag = hot;
      }
      __threadfence();
      __syncthreads();
      const int hot = s_flag;
      if (tid == 0) {
        red_release_add(d.cnt + t.done, 1);
        if (d.trace) d.trace[8 * (size_t)ti + 3] = ba_globaltimer();
      }
      if (hot & 1) {
        const BaTask ht = s_ht;
        double* gX = d.tiles + (size_t)ht.tC * BA_TILE;
        if (d.trace && tid == 0) {
          unsigned int smid;
          asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
          d.trace[8 * (size_t)t.l0] = smid;
          d.trace[8 * (size_t)t.l0 + 1] = d.trace[8 * (size_t)t.l0 + 2] = ba_globaltimer();
        }
        tile_load<BA_LDS>(gX, sB, tid);
        __syncthreads();
        tile_trsm2(sB, sA, sM, (bk + 7) >> 3, tid);  // L_kk is still staged in sA
        __syncthreads();
        if (hot & 2) {
          // the diagonal update first: it is what the next pivot waits for; L_jk is published after
          const BaTask hu = s_hu;
          if (d.trace && tid == 0) {
            unsigned int smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            d.trace[8 * (size_t)t.l1] = smid;
            d.trace[8 * (size_t)t.l1 + 1] = d.trace[8 * (size_t)t.l1 + 2] = ba_globaltimer();
          }
          ba_upd_body(d, hu, t.l1, sB, sB, sY, bk, tid, true);  // X = L_jk staged in sB, y_k in sY
          __threadfence();
          __syncthreads();
          if (tid == 0) {
            red_release_add(d.cnt + hu.done, 1);
            if (d.trace) d.trace[8 * (size_t)t.l1 + 3] = ba_globaltimer();
          }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = 2 * (tid + BA_NTHREADS * u);
          reinterpret_cast<double2*>(gX)[tid + BA_NTHREADS * u] =
              *reinterpret_cast<const double2*>(sB + (e >> 6) * BA_LDS + (e & 63));
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
          red_release_add(d.cnt + ht.done, 1);
          if (d.trace) d.trace[8 * (size_t)t.l0 + 3] = ba_globaltimer();
        }
      }
      continue;
    } else if (t.type == BA_T_TRSM) {
      // L_ik = A_ik L_kk^-T by blocked substitution (tile_trsm2); every warp owns 8 rows
      double* gC = d.tiles + (size_t)t.tC * BA_TILE;
      const double* gm = d.Linv + (size_t)t.tA * BA_TILE;
      tile_load<BA_LDS>(d.tiles + (size_t)t.w1i * BA_TILE, sB, tid);  // L_kk: awaited up front
      sM[tid] = __ldcg(gm + tid);
      sM[tid + BA_NTHREADS] = __ldcg(gm + tid + BA_NTHREADS);
      if (tid == 0 && t.w0i >= 0)
        while (ld_acquire(d.cnt + t.w0i) < t.w0v) {}  // A_ik has received all its updates
      __syncthreads();
      tile_load<BA_LDS>(gC, sA, tid);
      __syncthreads();
      if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 4] = ba_globaltimer();
      tile_trsm2(sA, sB, sM, (bk + 7) >> 3, tid);
      __syncthreads();
      if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 5] = ba_globaltimer();
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = 2 * (tid + BA_NTHREADS * u);
        reinterpret_cast<double2*>(gC)[tid + BA_NTHREADS * u] =
            *reinterpret_cast<const double2*>(sA + (e >> 6) * BA_LDS + (e & 63));
      }
    } else if (t.type == BA_T_UPD) {
      ba_upd_body(d, t, ti, sA, sB, sY, bk, tid, false);
    } else if (t.type == BA_T_SUM) {
      // C += sum of the scratch tiles (fixed order); diagonal tiles also collect their rhs parts
      double2* gC = reinterpret_cast<double2*>(d.tiles + (size_t)t.tC * BA_TILE);
      double2 acc[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = __ldcg(gC + tid + BA_NTHREADS * u);
      double rb = 0;
      const bool dg = (t.flags & 1) && tid < 64;
      if (dg) rb = __ldcg(d.rhs + (size_t)t.i * BA_TB + tid);
      for (int e = t.l0; e < t.l1; ++e) {
        const int st = d.sum[e].tile;
        const double2* gS = reinterpret_cast<const double2*>(d.tiles + (size_t)st * BA_TILE);
        double2 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldcg(gS + tid + BA_NTHREADS * u);
        if (dg) rb += __ldcg(d.rhsS + (size_t)(st - d.nTiles) * BA_TB + tid);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          acc[u].x += v[u].x;
          acc[u].y += v[u].y;
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) gC[tid + BA_NTHREADS * u] = acc[u];
      if (dg) d.rhs[(size_t)t.i * BA_TB + tid] = rb;
    } else {  // BA_T_BWD: x_k = L_kk^-T (y_k - sum_i L_ik^T x_i)
      if (tid < 64) sV[tid] = __ldcg(d.y + (size_t)t.k * BA_TB + tid);
      {  // L_kk and its diagonal inverses, needed last: in flight under the entry loop
        const double* gm = d.Linv + (size_t)t.k * BA_TILE;
        tile_load<BA_LDS>(d.tiles + (size_t)t.tC * BA_TILE, sA, tid);
        sM[tid] = __ldcg(gm + tid);
        sM[tid + BA_NTHREADS] = __ldcg(gm + tid + BA_NTHREADS);
      }
      // warp w owns columns 8w .. 8w+7, lane l rows 2l, 2l+1: every load instruction of a warp reads
      // one whole 512-byte column (coalesced); partial sums stay in registers over ALL entries and
      // are reduced across the lanes once.  The loads of four tiles are in flight together.
      const int lane = tid & 31, wq = tid >> 5;
      double p[8];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) p[jj] = 0.0;
      // Entries are ordered oldest solution first (ba_plan.h).  Per chunk of 4: the tile loads are issued, THEN
      // the chunk's x_i are awaited -- only the last chunk contains the x of the predecessor on the backward
      // chain, and its tiles are already in flight while that predecessor finishes.
      for (int e0 = t.l0; e0 < t.l1; e0 += 4) {
        const int ne = min(4, t.l1 - e0);
        // L_ik must be final before it is read: TRSM(i, k) is not an ancestor of BWD(k) except through x_i,
        // which is awaited only after the loads are issued
        __syncthreads();  // (also: sX of the previous chunk is consumed)
        if (tid < ne)
          while (ld_acquire(d.cnt + d.bwd[e0 + tid].tile) < d.bwd[e0 + tid].fin) {}
        __syncthreads();
        double2 v[4][8];
#pragma unroll
        for (int w4 = 0; w4 < 4; ++w4) {
          const int e = min(w4, ne - 1);
          const double2* col = reinterpret_cast<const double2*>(
              d.tiles + (size_t)d.bwd[e0 + e].tile * BA_TILE + (8 * wq) * BA_TB) + lane;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) v[w4][jj] = __ldcg(col + jj * (BA_TB / 2));
        }
        if (tid < ne)
          while (ld_acquire(d.cnt + d.xdoneBase + d.bwd[e0 + tid].blk) < 1) {}
        __syncthreads();
        if (tid < ne * BA_TB) sX[tid] = __ldcg(d.x + (size_t)d.bwd[e0 + (tid >> 6)].blk * BA_TB + (tid & 63));
        __syncthreads();
#pragma unroll
        for (int w4 = 0; w4 < 4; ++w4) {
          if (w4 < ne) {
            const double2 xv = *reinterpret_cast<const double2*>(sX + w4 * BA_TB + 2 * lane);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) p[jj] = __fma_rn(v[w4][jj].x, xv.x, __fma_rn(v[w4][jj].y, xv.y, p[jj]));
          }
        }
      }
      // transpose-reduce: 8 values x 32 lanes -> lane group (l >> 2) holds column 8w + (l >> 2)
      {
        const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
        double a4[4], a2[2];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const double send = b4 ? p[jj] : p[jj + 4];
          const double keep = b4 ? p[jj + 4] : p[jj];
          a4[jj] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const double send = b3 ? a4[jj] : a4[jj + 2];
          const double keep = b3 ? a4[jj + 2] : a4[jj];
          a2[jj] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
        const double send = b2 ? a2[0] : a2[1];
        double part = (b2 ? a2[1] : a2[0]) + __shfl_xor_sync(0xffffffffu, send, 4);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        __syncthreads();
        // the lane group with bits (b4, b3, b2) holds column 4 b4 + 2 b3 + b2 of this warp
        if ((lane & 3) == 0) sV[8 * wq + (b4 ? 4 : 0) + (b3 ? 2 : 0) + (b2 ? 1 : 0)] -= part;
      }
      __syncthreads();
      if (d.trace && tid == 0) d.trace[8 * (size_t)ti + 4] = ba_globaltimer();
      if (tid < 64) {
        sY[tid] = 0.0;
        tile_bwd3(sA, sM, sV, sY, (bk + 7) >> 3, tid);
      }
      __syncthreads();
      if (tid < 64) d.x[(size_t)t.k * BA_TB + tid] = (tid < bk) ? sY[tid] : 0.0;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      red_release_add(d.cnt + t.done, 1);
      if (d.trace) d.trace[8 * (size_t)ti + 3] = ba_globaltimer();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Reduced systems of ONE or TWO blocks (<= 20 free cameras: the per-key-frame local BA, c2 / c3): the
// whole solve in ONE CTA with the tiles resident in shared memory -- POTRF(0), TRSM(1,0), UPD(1,1,0),
// POTRF(1), BWD(1), BWD(0) with the same tile primitives as the dataflow kernel, but without tickets,
// polling, publishing and the global round trip of every tile between two tasks.
// t00 / t10 / t11: tile indices of the lower block triangle (t10 < 0: structurally zero; t11 < 0: one block).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tile_stage_diag(const double* __restrict__ g, double* __restrict__ sT, int bk, int tid) {
  double2 v[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const double2*>(g) + tid + BA_NTHREADS * u);
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int e = 2 * (tid + BA_NTHREADS * u);
    const int c = e >> 6, r = e & 63;
    double2 w = v[u];
    if (r >= bk || c >= bk) w.x = (r == c) ? 1.0 : 0.0;
    if (r + 1 >= bk || c >= bk) w.y = (r + 1 == c) ? 1.0 : 0.0;
    *reinterpret_cast<double2*>(sT + c * BA_LDS + r) = w;
  }
}

__global__ void __launch_bounds__(BA_NTHREADS, 1) ba_tile_two(BaTileDev d, int t00, int t10, int t11) {
  extern __shared__ double smem[];
  double* sA = smem;                       // block (0,0) -> L00
  double* sB = sA + BA_TB * BA_LDS;        // block (1,0) -> L10
  double* sC = sB + BA_TB * BA_LDS;        // block (1,1) -> L11
  double* sX = sC + BA_TB * BA_LDS;        // x0 [0..63], x1 [64..127]
  double* sM = sX + 8 * BA_TB;
  double* sV = sM + 8 * BA_TB;
  double* sY = sV + BA_TB;
  double* sD = sY + BA_TB;
  __shared__ double sM0[8 * BA_TB], sY0[BA_TB], sR1[BA_TB];
  __shared__ int s_fail;
  const int tid = threadIdx.x;
  const int bk0 = d.blkRows[0];
  const bool two = t11 >= 0;
  const int bk1 = two ? d.blkRows[1] : 0;
  if (tid == 0) s_fail = 0;
  tile_stage_diag(d.tiles + (size_t)t00 * BA_TILE, sA, bk0, tid);
  if (tid < 64) sV[tid] = (tid < bk0) ? __ldcg(d.rhs + tid) : 0.0;
  if (two) {
    tile_stage_diag(d.tiles + (size_t)t11 * BA_TILE, sC, bk1, tid);
    if (t10 >= 0) tile_load<BA_LDS>(d.tiles + (size_t)t10 * BA_TILE, sB, tid);
    if (tid < 64) sR1[tid] = (tid < bk1) ? __ldcg(d.rhs + BA_TB + tid) : 0.0;
  }
  __syncthreads();
  tile_potrf2(sA, sV, sY, sM, sD, tid, &s_fail, (bk0 + 7) >> 3);  // L00 (sA), y0 (sY), M_b of block 0 (sM)
  if (two) {
    if (t10 >= 0) {
      tile_trsm2(sB, sA, sM, (bk0 + 7) >> 3, tid);  // L10 = A10 L00^-T
      __syncthreads();
      TileAcc acc;
      tile_gemm_dmma(sB, sB, (bk0 + 3) & ~3, tid, acc);  // L10 L10^T
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            int r, c;
            tile_acc_rc(tid, mi, ni, e, r, c);
            sC[c * BA_LDS + r] -= acc.c[mi][ni][e];
          }
      if (tid < 64) {  // b1 -= L10 y0
        double sum = 0;
        for (int p = 0; p < bk0; ++p) sum = __fma_rn(sB[p * BA_LDS + tid], sY[p], sum);
        sR1[tid] -= sum;
      }
    }
    // keep y0 and the diagonal inverses of block 0 for its backward step
    sM0[tid] = sM[tid];
    sM0[tid + BA_NTHREADS] = sM[tid + BA_NTHREADS];
    if (tid < 64) sY0[tid] = sY[tid];
    __syncthreads();
    tile_potrf2(sC, sR1, sY, sM, sD, tid, &s_fail, (bk1 + 7) >> 3);  // L11 (sC), y1 (sY), M_b of block 1 (sM)
    if (tid < 64) {
      sV[tid] = sY[tid];
      sX[BA_TB + tid] = 0.0;
      tile_bwd3(sC, sM, sV, sX + BA_TB, (bk1 + 7) >> 3, tid);  // x1 = L11^-T y1
    }
    __syncthreads();
    if (tid < 64) {  // v0 = y0 - L10^T x1
      double sum = 0;
      if (t10 >= 0)
        for (int r = 0; r < bk1; ++r) sum = __fma_rn(sB[tid * BA_LDS + r], sX[BA_TB + r], sum);
      sV[tid] = sY0[tid] - sum;
      sX[tid] = 0.0;
      tile_bwd3(sA, sM0, sV, sX, (bk0 + 7) >> 3, tid);  // x0 = L00^-T v0
    }
    __syncthreads();
    if (tid < 64) {
      d.x[tid] = (tid < bk0) ? sX[tid] : 0.0;
      d.x[BA_TB + tid] = (tid < bk1) ? sX[BA_TB + tid] : 0.0;
    }
  } else {
    if (tid < 64) {
      sV[tid] = sY[tid];
      sX[tid] = 0.0;
      tile_bwd3(sA, sM, sV, sX, (bk0 + 7) >> 3, tid);
    }
    __syncthreads();
    if (tid < 64) d.x[tid] = (tid < bk0) ? sX[tid] : 0.0;
  }
  if (tid == 0 && s_fail) d.sc[d.scFail] = 1.0;
}

// =============================================================================================
// Selected inversion Z = S^-1 on the factor's tile pattern (the covariance stage of the BA, DESIGN.md 4.6;
// task plan: ba_make_selinv_plan in ba_plan.h).  Z has the factor's tile layout; its padding rows and columns
// are zero and its diagonal tiles are stored in full (both triangles).
// =============================================================================================

// acc(r, c) += sum_{p < kk} opA(r, p) opB(p, c) with the DMMA fragments of tile_gemm_dmma.  Both tiles are
// staged column-major (element (r, c) at c * BA_LDS + r); TA: opA = A^T (else A), TB: opB = B (else B^T).
template <bool TA, bool TB>
__device__ __forceinline__ void tile_gemm_acc(const double* __restrict__ sA, const double* __restrict__ sB,
                                              int kk, int tid, TileAcc& acc) {
  const int lane = tid & 31, w = tid >> 5;
  const int mB = (w & 3) * 16 + (lane >> 2), nB = (w >> 2) * 32 + (lane >> 2), kl = lane & 3;
  for (int p0 = 0; p0 < kk; p0 += 4) {
    const int p = p0 + kl;
    double a[2], b[4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) a[mi] = TA ? sA[(mB + 8 * mi) * BA_LDS + p] : sA[p * BA_LDS + mB + 8 * mi];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) b[ni] = TB ? sB[(nB + 8 * ni) * BA_LDS + p] : sB[p * BA_LDS + nB + 8 * ni];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) dmma884(acc.c[mi][ni][0], acc.c[mi][ni][1], a[mi], b[ni]);
  }
}

__device__ __forceinline__ void tile_acc_zero(TileAcc& acc) {
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) acc.c[mi][ni][0] = acc.c[mi][ni][1] = 0.0;
}

// s(r, c) = scale * acc(r, c) inside rows x cols, 0 outside (shared, column-major)
__device__ __forceinline__ void tile_acc_store(const TileAcc& acc, double* __restrict__ s, double scale, int rows,
                                               int cols, int tid) {
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int r, c;
        tile_acc_rc(tid, mi, ni, e, r, c);
        s[c * BA_LDS + r] = (r < rows && c < cols) ? scale * acc.c[mi][ni][e] : 0.0;
      }
}

// shared tile -> global tile; sym: the symmetric part (diagonal tiles of Z)
__device__ __forceinline__ void tile_store(const double* __restrict__ s, double* __restrict__ g, bool sym, int tid) {
  for (int e = tid; e < BA_TILE; e += BA_NTHREADS) {
    const int c = e >> 6, r = e & 63;
    g[e] = sym ? 0.5 * (s[c * BA_LDS + r] + s[r * BA_LDS + c]) : s[c * BA_LDS + r];
  }
}

// X = L_kk^-T in sX (zero outside bk x bk) from L_kk staged in sL (identity padding) and its 8x8 diagonal
// inverses sM: X L^T = I by tile_trsm2.  Ends with a CTA barrier.
__device__ __forceinline__ void tile_inv_t(const double* __restrict__ sL, const double* __restrict__ sM,
                                          double* __restrict__ sX, int bk, int tid) {
  for (int e = tid; e < BA_TILE; e += BA_NTHREADS) {
    const int c = e >> 6, r = e & 63;
    sX[c * BA_LDS + r] = (r == c) ? 1.0 : 0.0;
  }
  __syncthreads();
  tile_trsm2(sX, sL, sM, (bk + 7) >> 3, tid);
  __syncthreads();
  for (int e = tid; e < BA_TILE; e += BA_NTHREADS) {
    const int c = e >> 6, r = e & 63;
    if (r >= bk || c >= bk) sX[c * BA_LDS + r] = 0.0;
  }
  __syncthreads();
}

// min over the rows of a block of L_ii^2 / S_ii (0 where S_ii is not positive or the pivot not finite)
__device__ __forceinline__ double rel_pivot(double l, double s) {
  const double q = l * l / s;
  return (s > 0.0 && q >= 0.0 && q < 1e300) ? q : 0.0;
}

struct BaSelDev {
  const double* L;        // factor tiles (lower; diagonal tiles: identity padding)
  const double* Linv;     // [nb][512]: the 8x8 diagonal inverses of every L_kk (ba_tile_solve's POTRF)
  double* sdiag;          // [nb][64]: diagonal of S before the factorisation (ba_cov_sdiag)
  double* Z;              // Z tiles, the factor's layout
  double* X;              // [nb][4096]: X_k = L_kk^-T
  double* piv;            // [nb]: minimum relative pivot of block k
  const BaSelTask* tasks;
  const BaSelOp* ops;
  const int* blkRows;
  const int* diagTile;    // [nb]: tile index of (k, k)
  int* cnt;               // [nb]: finished off-diagonal tasks of step q
};

constexpr int BA_SELX_SMEM = (2 * BA_TB * BA_LDS + 8 * BA_TB) * (int)sizeof(double);
constexpr int BA_SELS_SMEM = 2 * BA_TB * BA_LDS * (int)sizeof(double);

// One CTA per block: X_k = L_kk^-T and the block's minimum relative pivot.
__global__ void __launch_bounds__(BA_NTHREADS, 1) ba_selinv_xinv(BaSelDev d) {
  extern __shared__ double smem[];
  double* sL = smem;
  double* sX = sL + BA_TB * BA_LDS;
  double* sM = sX + BA_TB * BA_LDS;
  __shared__ double s_red[BA_TB];
  const int tid = threadIdx.x, k = blockIdx.x, bk = d.blkRows[k];
  tile_stage_diag(d.L + (size_t)d.diagTile[k] * BA_TILE, sL, bk, tid);
  sM[tid] = __ldcg(d.Linv + (size_t)k * BA_TILE + tid);
  sM[tid + BA_NTHREADS] = __ldcg(d.Linv + (size_t)k * BA_TILE + tid + BA_NTHREADS);
  __syncthreads();
  if (tid < BA_TB) s_red[tid] = tid < bk ? rel_pivot(sL[tid * BA_LDS + tid], d.sdiag[(size_t)k * BA_TB + tid]) : 1e300;
  tile_inv_t(sL, sM, sX, bk, tid);
  double* g = d.X + (size_t)k * BA_TILE;
  for (int e = tid; e < BA_TILE; e += BA_NTHREADS) g[e] = sX[(e >> 6) * BA_LDS + (e & 63)];
  if (tid == 0) {
    double m = 1e300;
    for (int r = 0; r < bk; ++r) m = fmin(m, s_red[r]);
    d.piv[k] = m;
  }
}

// Z_kk of the diagonal task t (the Z_jk of its step are final): X_k (X_k^T - sum_j L_jk^T Z_jk)
__device__ __forceinline__ void selinv_diag(const BaSelDev& d, const BaSelTask& t, double* sA, double* sB, int tid) {
  const int bk = d.blkRows[t.k];
  TileAcc acc;
  tile_acc_zero(acc);
  for (int o = t.opBegin; o < t.opEnd; ++o) {
    const BaSelOp op = d.ops[o];
    __syncthreads();
    tile_load<BA_LDS>(d.L + (size_t)op.tL * BA_TILE, sA, tid);
    tile_load<BA_LDS>(d.Z + (size_t)op.tZ * BA_TILE, sB, tid);
    __syncthreads();
    tile_gemm_acc<true, true>(sA, sB, (d.blkRows[op.j] + 3) & ~3, tid, acc);  // P += L_jk^T Z_jk
  }
  __syncthreads();
  tile_load<BA_LDS>(d.X + (size_t)t.k * BA_TILE, sB, tid);
  __syncthreads();
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int r, c;
        tile_acc_rc(tid, mi, ni, e, r, c);
        sA[c * BA_LDS + r] = sB[r * BA_LDS + c] - acc.c[mi][ni][e];  // Q = X^T - P
      }
  __syncthreads();
  tile_acc_zero(acc);
  tile_gemm_acc<false, true>(sB, sA, (bk + 3) & ~3, tid, acc);  // X Q
  __syncthreads();
  tile_acc_store(acc, sA, 1.0, bk, bk, tid);
  __syncthreads();
  tile_store(sA, d.Z + (size_t)t.tOut * BA_TILE, true, tid);
}

// One step of the recurrence (pivot k): CTA b < nOff computes Z_ik of task t0 + b; the CTA that finishes
// last computes Z_kk (task t0 + nOff).  nOff == 0: one CTA, Z_kk = X_k X_k^T.
__global__ void __launch_bounds__(BA_NTHREADS, 1) ba_selinv_step(BaSelDev d, int q, int t0, int nOff) {
  extern __shared__ double smem[];
  double* sA = smem;
  double* sB = sA + BA_TB * BA_LDS;
  __shared__ int s_last;
  const int tid = threadIdx.x;
  if (nOff > 0) {
    const BaSelTask t = d.tasks[t0 + blockIdx.x];
    const int bi = d.blkRows[t.i], bk = d.blkRows[t.k];
    TileAcc acc;
    tile_acc_zero(acc);
    for (int o = t.opBegin; o < t.opEnd; ++o) {
      const BaSelOp op = d.ops[o];
      __syncthreads();
      tile_load<BA_LDS>(d.Z + (size_t)op.tZ * BA_TILE, sA, tid);
      tile_load<BA_LDS>(d.L + (size_t)op.tL * BA_TILE, sB, tid);
      __syncthreads();
      const int kk = (d.blkRows[op.j] + 3) & ~3;
      if (op.zT)
        tile_gemm_acc<true, true>(sA, sB, kk, tid, acc);  // G += Z_ji^T L_jk
      else
        tile_gemm_acc<false, true>(sA, sB, kk, tid, acc);  // G += Z_ij L_jk
    }
    __syncthreads();
    tile_acc_store(acc, sA, 1.0, bi, bk, tid);
    tile_load<BA_LDS>(d.X + (size_t)t.k * BA_TILE, sB, tid);
    __syncthreads();
    tile_acc_zero(acc);
    tile_gemm_acc<false, false>(sA, sB, (bk + 3) & ~3, tid, acc);  // G X_k^T = G L_kk^-1
    __syncthreads();
    tile_acc_store(acc, sA, -1.0, bi, bk, tid);
    __syncthreads();
    tile_store(sA, d.Z + (size_t)t.tOut * BA_TILE, false, tid);
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(d.cnt + q, 1) == nOff - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
  }
  selinv_diag(d, d.tasks[t0 + nOff], sA, sB, tid);
}

// Systems of one or two blocks (every local BA): factorisation and selected inversion in ONE CTA with the
// tiles resident in shared memory.  ba_tile_two keeps its factor in shared memory and never stores it, so
// this kernel factors S again with the same primitives (tile_potrf2, tile_trsm2) before inverting.
// Tiles t00 / t10 / t11 as ba_tile_two; S is read from tiles, Z written with the same indices.
constexpr int BA_SEL2_SMEM = (5 * BA_TB * BA_LDS + 16 * BA_TB + 2 * BA_TB + 96 + 2 * BA_TB) * (int)sizeof(double);

__global__ void __launch_bounds__(BA_NTHREADS, 1)
ba_selinv_two(const double* __restrict__ tiles, const int* __restrict__ blkRows, int t00, int t10, int t11,
              double* __restrict__ Z, double* __restrict__ piv, double* __restrict__ failFlag) {
  extern __shared__ double smem[];
  double* sA = smem;                   // S00 -> L00
  double* sB = sA + BA_TB * BA_LDS;    // S10 -> L10 -> (Z11 L10)
  double* sC = sB + BA_TB * BA_LDS;    // S11 -> L11 -> Z11 -> Q
  double* sX0 = sC + BA_TB * BA_LDS;   // L00^-T
  double* sX1 = sX0 + BA_TB * BA_LDS;  // L11^-T -> G -> Z10
  double* sM0 = sX1 + BA_TB * BA_LDS;
  double* sM1 = sM0 + 8 * BA_TB;
  double* sV = sM1 + 8 * BA_TB;        // zero right-hand side
  double* sY = sV + BA_TB;
  double* sD = sY + BA_TB;
  double* sdg = sD + 96;               // diagonal of S00 | S11
  __shared__ int s_fail;
  const int tid = threadIdx.x;
  const int bk0 = blkRows[0];
  const bool two = t11 >= 0;
  const int bk1 = two ? blkRows[1] : 0;
  if (tid == 0) s_fail = 0;
  tile_stage_diag(tiles + (size_t)t00 * BA_TILE, sA, bk0, tid);
  if (two) {
    tile_stage_diag(tiles + (size_t)t11 * BA_TILE, sC, bk1, tid);
    if (t10 >= 0) tile_load<BA_LDS>(tiles + (size_t)t10 * BA_TILE, sB, tid);
  }
  if (tid < BA_TB) sV[tid] = 0.0;
  __syncthreads();
  if (tid < BA_TB) {
    sdg[tid] = sA[tid * BA_LDS + tid];
    sdg[BA_TB + tid] = two ? sC[tid * BA_LDS + tid] : 1.0;
  }
  __syncthreads();
  tile_potrf2(sA, sV, sY, sM0, sD, tid, &s_fail, (bk0 + 7) >> 3);
  if (two) {
    if (t10 >= 0) {
      tile_trsm2(sB, sA, sM0, (bk0 + 7) >> 3, tid);  // L10 = S10 L00^-T
      __syncthreads();
      TileAcc acc;
      tile_gemm_dmma(sB, sB, (bk0 + 3) & ~3, tid, acc);
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            int r, c;
            tile_acc_rc(tid, mi, ni, e, r, c);
            sC[c * BA_LDS + r] -= acc.c[mi][ni][e];
          }
    }
    __syncthreads();
    tile_potrf2(sC, sV, sY, sM1, sD, tid, &s_fail, (bk1 + 7) >> 3);
  }
  if (tid == 0) {
    double m0 = 1e300, m1 = 1e300;
    for (int r = 0; r < bk0; ++r) m0 = fmin(m0, rel_pivot(sA[r * BA_LDS + r], sdg[r]));
    for (int r = 0; r < bk1; ++r) m1 = fmin(m1, rel_pivot(sC[r * BA_LDS + r], sdg[BA_TB + r]));
    piv[0] = m0;
    if (two) piv[1] = m1;
    if (s_fail) *failFlag = 1.0;
  }
  tile_inv_t(sA, sM0, sX0, bk0, tid);
  TileAcc acc;
  if (!two) {
    tile_acc_zero(acc);
    tile_gemm_acc<false, false>(sX0, sX0, (bk0 + 3) & ~3, tid, acc);  // X0 X0^T
    tile_acc_store(acc, sA, 1.0, bk0, bk0, tid);
    __syncthreads();
    tile_store(sA, Z + (size_t)t00 * BA_TILE, true, tid);
    return;
  }
  tile_inv_t(sC, sM1, sX1, bk1, tid);
  tile_acc_zero(acc);
  tile_gemm_acc<false, false>(sX1, sX1, (bk1 + 3) & ~3, tid, acc);  // Z11 = X1 X1^T
  __syncthreads();
  tile_acc_store(acc, sC, 1.0, bk1, bk1, tid);
  __syncthreads();
  tile_store(sC, Z + (size_t)t11 * BA_TILE, true, tid);
  tile_acc_zero(acc);
  if (t10 >= 0) {
    tile_gemm_acc<false, true>(sC, sB, (bk1 + 3) & ~3, tid, acc);  // G = Z11 L10
    __syncthreads();
    tile_acc_store(acc, sX1, 1.0, bk1, bk0, tid);
    __syncthreads();
    tile_acc_zero(acc);
    tile_gemm_acc<false, false>(sX1, sX0, (bk0 + 3) & ~3, tid, acc);  // G X0^T
    __syncthreads();
    tile_acc_store(acc, sX1, -1.0, bk1, bk0, tid);                      // Z10
    __syncthreads();
    tile_store(sX1, Z + (size_t)t10 * BA_TILE, false, tid);
    tile_acc_zero(acc);
    tile_gemm_acc<true, true>(sB, sX1, (bk1 + 3) & ~3, tid, acc);      // P = L10^T Z10
  }
  __syncthreads();
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int r, c;
        tile_acc_rc(tid, mi, ni, e, r, c);
        sC[c * BA_LDS + r] = sX0[r * BA_LDS + c] - acc.c[mi][ni][e];  // Q = X0^T - P
      }
  __syncthreads();
  tile_acc_zero(acc);
  tile_gemm_acc<false, true>(sX0, sC, (bk0 + 3) & ~3, tid, acc);  // Z00 = X0 Q
  __syncthreads();
  tile_acc_store(acc, sA, 1.0, bk0, bk0, tid);
  __syncthreads();
  tile_store(sA, Z + (size_t)t00 * BA_TILE, true, tid);
}

}  // namespace coslam
