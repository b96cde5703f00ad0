// ba_kernels.cuh -- device code of the Schur-complement Levenberg-Marquardt bundle adjustment
// (sm_90a, fp64).  Algorithm: sba_motstr_levmar_x of Lourakis & Argyros with the KRTS camera
// parameterisation of app/SL_CoSLAMBA.cpp:290-378 (SURVEY.md Appendix B).
//
// Data layout in HBM (per solver / per rank):
//   cameras (replicated): camK[m][5] (K0,K1,K2,K4,K5), camR0[m][9] (rotation of q0), pa[m][6] (v,t)
//   points  (this rank's shard): pb[n][3]
//   observations, point-major CSR: cam[N], pt[N], xy[N][2], wgt[N]; with measurement covariances set
//   (cosl_ba_solver_set_obs_cov), obsL[N][3]: the whitening factor L of each observation (DESIGN.md 4.7)
//   camera-major permutation of the free-camera observations: cobs[Nc], ccam[Nc]
//   W[N][18]   W_ij = A_ij^T B_ij (6x3 row-major) of the current linearisation
//   V[n][6], eb[n][3], U[m][21] (packed upper), ea[m][6]
//   pair work list for the Schur contraction: items {rowCam, colCam, begin, end} over entry pairs
//   (obsA, obsB) sorted by camera pair
//   S: block-sparse 64x64 tiles of the permuted reduced camera system + block-padded rhs, see
//   ba_tile.cuh / ba_plan.h
//
// One-observation-per-thread kernels evaluate residuals and the 2x6 / 2x3 Jacobian blocks; per-point
// (resp. per-camera) sums are collapsed with segmented warp shuffles and only segment heads touch
// memory with atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ba_lm.cuh"

namespace coslam {

struct BaDev {
  int m, n, mcon, ncon, mf, ns;
  long long N, Nc;
  const double* camK;
  const double* camR0;
  const int* cam;
  const int* pt;
  const double* xy;
  double* wgt;
  const double* obsL;  // [N][3] (l00, l01, l11) with L^T L = Sigma^-1; read by the OBSCOV instantiations only
  const long long* ptr;
  const int* cobs;
  const int* ccam;
  double* W;
  double* V;
  double* eb;
  double* U;
  double* ea;
  double* tiles;      // reduced camera system, tile t at tiles + 4096 t (column-major 64x64)
  double* rhs;        // block padded: block k at rhs + 64 k
  const int* solIdx;  // per free camera: index of its first row in rhs / x
  double* sc;         // scalars, see BaScalar
};

__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  // valid for non-negative doubles: the bit pattern is monotone
  atomicMax(reinterpret_cast<unsigned long long*>(addr),
            static_cast<unsigned long long>(__double_as_longlong(v)));
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// x = pi(K (R(dq(v)) R0 X + t)); optionally A = dx/d(v,t) (2x6), B = dx/dX (2x3).
// Same formulas as oracle/ba_oracle.cpp:orc_ba_project.
template <bool WANT_A, bool WANT_B>
__device__ __forceinline__ void ba_project(const double* __restrict__ Kc,
                                           const double* __restrict__ R0,
                                           const double* __restrict__ p6, const double X[3],
                                           double xy[2], double A[12], double B[6]) {
  const double v[3] = {p6[0], p6[1], p6[2]};
  const double Y[3] = {R0[0] * X[0] + R0[1] * X[1] + R0[2] * X[2],
                       R0[3] * X[0] + R0[4] * X[1] + R0[5] * X[2],
                       R0[6] * X[0] + R0[7] * X[1] + R0[8] * X[2]};
  const double w = sqrt(1.0 - (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
  double vxY[3], vxvxY[3];
  cross3(v, Y, vxY);
  cross3(v, vxY, vxvxY);
  const double P[3] = {Y[0] + 2 * w * vxY[0] + 2 * vxvxY[0] + p6[3],
                       Y[1] + 2 * w * vxY[1] + 2 * vxvxY[1] + p6[4],
                       Y[2] + 2 * w * vxY[2] + 2 * vxvxY[2] + p6[5]};
  const double iz = 1.0 / P[2];
  const double un = Kc[0] * P[0] + Kc[1] * P[1];
  xy[0] = un * iz + Kc[2];
  xy[1] = Kc[3] * P[1] * iz + Kc[4];
  if (!WANT_A && !WANT_B) return;
  const double Jp[6] = {Kc[0] * iz, Kc[1] * iz, -un * iz * iz, 0.0, Kc[3] * iz,
                        -Kc[3] * P[1] * iz * iz};
  if (WANT_A) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double e[3] = {0, 0, 0};
      e[k] = 1.0;
      double exY[3], exvxY[3], vxexY[3];
      cross3(e, Y, exY);
      cross3(e, vxY, exvxY);
      cross3(v, exY, vxexY);
      const double dw = -v[k] / w;
      double dP[3];
#pragma unroll
      for (int c = 0; c < 3; ++c)
        dP[c] = 2 * dw * vxY[c] + 2 * w * exY[c] + 2 * exvxY[c] + 2 * vxexY[c];
      A[k] = Jp[0] * dP[0] + Jp[1] * dP[1] + Jp[2] * dP[2];
      A[6 + k] = Jp[3] * dP[0] + Jp[4] * dP[1] + Jp[5] * dP[2];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      A[3 + k] = Jp[k];
      A[9 + k] = Jp[3 + k];
    }
  }
  if (WANT_B) {
    // R(dq) from the unit quaternion (w, v), then Rf = R(dq) R0
    const double x = v[0], y = v[1], z = v[2];
    const double Rd[9] = {w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y),
                          2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
                          2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z};
    double Rf[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        Rf[3 * i + j] = Rd[3 * i] * R0[j] + Rd[3 * i + 1] * R0[3 + j] + Rd[3 * i + 2] * R0[6 + j];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      B[k] = Jp[0] * Rf[k] + Jp[1] * Rf[3 + k] + Jp[2] * Rf[6 + k];
      B[3 + k] = Jp[3] * Rf[k] + Jp[4] * Rf[3 + k] + Jp[5] * Rf[6 + k];
    }
  }
}

// Segmented warp reduction by key for contiguous segments: after the call the FIRST lane of every
// run of equal keys holds the run's sum.
template <int NV>
__device__ __forceinline__ void seg_reduce(double* v, int key, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int ko = __shfl_down_sync(0xffffffffu, key, o);
    const bool take = (lane + o < 32) && (ko == key);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const double t = __shfl_down_sync(0xffffffffu, v[k], o);
      if (take) v[k] += t;
    }
  }
}

__device__ __forceinline__ double block_sum_1(double v, double* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_red[wid] = v;
  __syncthreads();
  double t = 0;
  if (wid == 0) {
    t = (lane < (int)(blockDim.x >> 5)) ? s_red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;  // valid in warp 0
}

__device__ __forceinline__ double tukey_w(double e, double s) {
  if (e >= s) return 0;
  e /= s;
  e = 1 - e * e;
  return e * e;
}

// Measurement covariances (DESIGN.md 4.7).  The kernels that form residuals and Jacobians take a template flag
// OBSCOV: with it they multiply the residual (and the Jacobian rows) of observation o by its upper-triangular L,
// L^T L = Sigma_o^-1, so that |L e|^2 = e^T Sigma^-1 e.  Without it they are the unweighted kernels, unchanged.
template <int NC>
__device__ __forceinline__ void ba_whiten(const double* __restrict__ L, double* r0, double* r1) {
  const double l00 = L[0], l01 = L[1], l11 = L[2];
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const double a = r0[k], b = r1[k];
    r0[k] = l00 * a + l01 * b;
    r1[k] = l11 * b;
  }
}

// In place, one observation per thread: (s00, s01, s11) of Sigma -> (l00, l01, l11) of the upper-triangular L with
// L^T L = Sigma^-1.  Sigma^-1 = [s11 -s01; -s01 s00] / det, so l00 = sqrt(s11 / det), l01 = -s01 / sqrt(s11 det),
// l11 = 1 / sqrt(s11): Sigma = I gives L = I and Sigma = s^2 I gives L = I / s exactly.  The host checked that
// every Sigma is positive definite.
__global__ void __launch_bounds__(256) ba_obscov_factor(double* __restrict__ L, long long N) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  double* q = L + 3 * (size_t)o;
  const double a = q[0], b = q[1], c = q[2];
  const double det = a * c - b * b;
  q[0] = sqrt(c / det);
  q[1] = -b / sqrt(c * det);
  q[2] = 1.0 / sqrt(c);
}

// Gaussian camera priors (cosl_ba_solver_set_cam_prior, DESIGN.md 4.8).  Prior k on free camera cam[k] is
// rec[k] = [L (21: the upper-triangular 6x6 factor with L^T L = P^-1, packed by rows) | R_p (9, row-major) | t_p (3)].
// Its residual is r = [Log(R R_p^T); t - t_p] with R = R(q(v)) R0 and t of pa, so it follows a reset that re-anchors
// R0.  The kernels that take a template flag PRIOR add |L r|^2 to the cost and (L J)^T (L J), -(L J)^T L r to U_j and
// ea_j in CTAs beyond their observation range.  The priors are a kernel argument of their own rather than BaDev
// fields, so the instantiations without PRIOR keep their parameter layout and code.
// Point priors (cosl_ba_solver_set_pt_prior, DESIGN.md 4.9) follow the camera ones in the same argument: prior k on
// free point pt[k] is prec[k] = [L (6: the upper-triangular 3x3 factor with L^T L = P^-1, packed by rows) | mu (3)],
// its residual r = X - mu.  The PRIOR instantiations of the residual and trial-cost kernels run one thread per prior
// of either kind, cameras first; ba_linearize_points<PRIOR> adds L^T L and L^T L (mu - X) to V_i and eb_i, and
// ba_cov_mask<PRIOR> keeps every point with a prior in H (has[i] != 0).
struct BaPriorDev {
  const double* rec;  // [n][BA_PRIOR_REC]
  const int* cam;     // [n], distinct free cameras
  int n;
  int np;                    // number of point priors
  const double* prec;        // [np][BA_PTPRIOR_REC]
  const int* pt;             // [np], distinct free points
  const unsigned char* has;  // [n points]: 1 for a point with a prior
};
constexpr int BA_PRIOR_REC = 33;
constexpr int BA_PTPRIOR_REC = 9;

// Whitened prior residual rw = L r of prior k at pa and, with WANT_J, Jw = L dr/d(v, t) (6x6 row-major).
// Log(M) by atan2 with the axis from the skew part below 120 degrees and from the symmetric part above (exact to
// roundoff up to pi); dr_w / dv = Jl^-1(r_w) J_q with the left-Jacobian inverse of SO(3),
// Jl^-1(w) = I - [w]x / 2 + (1 - (th / 2) cot(th / 2)) / th^2 [w]x^2, and J_q = 2 (w_q I + [v]x + v v^T / w_q) the
// chart factor of ba_cov_cams.
template <bool WANT_J>
__device__ __forceinline__ void ba_prior_eval(const BaDev& d, const BaPriorDev& pr, int k,
                                              const double* __restrict__ pa, double rw[6], double Jw[36]) {
  const int j = pr.cam[k];
  const double* __restrict__ q = pr.rec + BA_PRIOR_REC * (size_t)k;
  const double* __restrict__ R0 = d.camR0 + 9 * (size_t)j;
  const double* __restrict__ p6 = pa + 6 * (size_t)j;
  const double x = p6[0], y = p6[1], z = p6[2];
  const double wq = sqrt(1.0 - (x * x + y * y + z * z));
  const double Rd[9] = {wq * wq + x * x - y * y - z * z, 2 * (x * y - wq * z), 2 * (x * z + wq * y),
                        2 * (x * y + wq * z), wq * wq - x * x + y * y - z * z, 2 * (y * z - wq * x),
                        2 * (x * z - wq * y), 2 * (y * z + wq * x), wq * wq - x * x - y * y + z * z};
  double R[9], M[9];  // R = R(q(v)) R0, M = R R_p^T
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) R[3 * a + b] = Rd[3 * a] * R0[b] + Rd[3 * a + 1] * R0[3 + b] + Rd[3 * a + 2] * R0[6 + b];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      M[3 * a + b] = R[3 * a] * q[21 + 3 * b] + R[3 * a + 1] * q[22 + 3 * b] + R[3 * a + 2] * q[23 + 3 * b];
  const double s[3] = {0.5 * (M[7] - M[5]), 0.5 * (M[2] - M[6]), 0.5 * (M[3] - M[1])};
  const double sn = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
  const double cs = 0.5 * (M[0] + M[4] + M[8] - 1.0);
  const double th = atan2(sn, cs);
  double r[6];
  if (cs > -0.5) {
    const double f = th < 1e-4 ? 1.0 + th * th / 6.0 : th / sn;
#pragma unroll
    for (int a = 0; a < 3; ++a) r[a] = f * s[a];
  } else {  // (M + M^T) / 2 - cos th I = (1 - cos th) a a^T: the column of the largest diagonal entry
    const double S0 = M[0] - cs, S1 = M[4] - cs, S2 = M[8] - cs;
    const double s01 = 0.5 * (M[1] + M[3]), s02 = 0.5 * (M[2] + M[6]), s12 = 0.5 * (M[5] + M[7]);
    const int c = (S0 >= S1 && S0 >= S2) ? 0 : (S1 >= S2 ? 1 : 2);
    const double col[3] = {c == 0 ? S0 : (c == 1 ? s01 : s02), c == 0 ? s01 : (c == 1 ? S1 : s12),
                           c == 0 ? s02 : (c == 1 ? s12 : S2)};
    const double f = th / sqrt((1.0 - cs) * (c == 0 ? S0 : (c == 1 ? S1 : S2)));
    const double sg = (col[0] * s[0] + col[1] * s[1] + col[2] * s[2]) < 0.0 ? -f : f;
#pragma unroll
    for (int a = 0; a < 3; ++a) r[a] = sg * col[a];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) r[3 + a] = p6[3 + a] - q[30 + a];
  // rw = L r, L packed by rows: row a holds L[a][a .. 5] from offset 6a - a(a-1)/2
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const int off = 6 * a - a * (a - 1) / 2;
    double t = 0.0;
#pragma unroll
    for (int b = a; b < 6; ++b) t += q[off + b - a] * r[b];
    rw[a] = t;
  }
  if (!WANT_J) return;
  // cot(th / 2) = sin th / (1 - cos th) = sn / (|(sn, cs)| - cs): no trigonometric call, exact up to pi
  const double c2 = th < 1e-2 ? 1.0 / 12.0 + th * th * (1.0 / 720.0 + th * th / 30240.0)
                              : (1.0 - 0.5 * th * sn / (sqrt(sn * sn + cs * cs) - cs)) / (th * th);
  const double wx[9] = {0.0, -r[2], r[1], r[2], 0.0, -r[0], -r[1], r[0], 0.0};
  double Ji[9], Jq[9], Jo[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const double w2 = wx[3 * a] * wx[b] + wx[3 * a + 1] * wx[3 + b] + wx[3 * a + 2] * wx[6 + b];
      Ji[3 * a + b] = (a == b ? 1.0 : 0.0) - 0.5 * wx[3 * a + b] + c2 * w2;
    }
  const double v[3] = {x, y, z}, vx[9] = {0.0, -z, y, z, 0.0, -x, -y, x, 0.0};
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) Jq[3 * a + b] = 2.0 * ((a == b ? wq : 0.0) + vx[3 * a + b] + v[a] * v[b] / wq);
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) Jo[3 * a + b] = Ji[3 * a] * Jq[b] + Ji[3 * a + 1] * Jq[3 + b] + Ji[3 * a + 2] * Jq[6 + b];
  // Jw = L diag(Jo, I)
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const int off = 6 * a - a * (a - 1) / 2;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      double t = 0.0;
#pragma unroll
      for (int c = a; c < 3; ++c) t += q[off + c - a] * Jo[3 * c + b];
      Jw[6 * a + b] = t;
    }
#pragma unroll
    for (int b = 3; b < 6; ++b) Jw[6 * a + b] = b >= a ? q[off + b - a] : 0.0;
  }
}

// |L r|^2 of camera prior k at pa
__device__ __forceinline__ double ba_prior_cost(const BaDev& d, const BaPriorDev& pr, int k,
                                                const double* __restrict__ pa) {
  double rw[6];
  ba_prior_eval<false>(d, pr, k, pa, rw, nullptr);
  return rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2] + rw[3] * rw[3] + rw[4] * rw[4] + rw[5] * rw[5];
}

// Whitened residual rw = L (X - mu) of point prior k
__device__ __forceinline__ void ba_ptprior_eval(const BaPriorDev& pr, int k, const double X[3], double rw[3]) {
  const double* __restrict__ q = pr.prec + BA_PTPRIOR_REC * (size_t)k;
  const double r0 = X[0] - q[6], r1 = X[1] - q[7], r2 = X[2] - q[8];
  rw[0] = q[0] * r0 + q[1] * r1 + q[2] * r2;
  rw[1] = q[3] * r1 + q[4] * r2;
  rw[2] = q[5] * r2;
}

// |L (X - mu)|^2 of point prior k
__device__ __forceinline__ double ba_ptprior_cost(const BaPriorDev& pr, int k, const double X[3]) {
  double rw[3];
  ba_ptprior_eval(pr, k, X, rw);
  return rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2];
}

// The priors' cost of thread k of the CTAs beyond the observations (cameras [0, n), then points [n, n + np)) at
// (pa, pb)
__device__ __forceinline__ double ba_priors_cost(const BaDev& d, const BaPriorDev& pr, long long k,
                                                 const double* __restrict__ pa, const double* __restrict__ pb) {
  if (k < pr.n) return ba_prior_cost(d, pr, (int)k, pa);
  k -= pr.n;
  if (k >= pr.np) return 0.0;
  const int i = pr.pt[k];
  const double X[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
  return ba_ptprior_cost(pr, (int)k, X);
}

// ------------------------------------------------------------------------------------------
// cost / weights / outliers: one observation per thread
// mode 0: sc[SC_COST] += w |e|^2 ; mode 1: wgt = tukey(|e|, maxErr) ; mode 2: outlier = |e|>=maxErr,
// sc[SC_COST] += number of outliers.  OBSCOV: mode 0 sums w |L e|^2; modes 1 and 2 stay on the pixel distance |e|
// (they are launched without it).  PRIOR (mode 0 only): the CTAs beyond the observations add the priors' |L r|^2,
// one camera or point prior per thread.
// ------------------------------------------------------------------------------------------
template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(256)
ba_residual_kernel(BaDev d, const double* __restrict__ pa, const double* __restrict__ pb, int mode,
                   double maxErr, unsigned char* __restrict__ outlier, BaPriorDev pr) {
  __shared__ double s_red[8];
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double c = 0;
  if (o < d.N) {
    const int j = d.cam[o], i = d.pt[o];
    const double X[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
    double h[2];
    ba_project<false, false>(d.camK + 5 * j, d.camR0 + 9 * j, pa + 6 * j, X, h, nullptr, nullptr);
    double dx = d.xy[2 * o] - h[0], dy = d.xy[2 * o + 1] - h[1];
    if (OBSCOV && mode == 0) ba_whiten<1>(d.obsL + 3 * (size_t)o, &dx, &dy);
    const double e2 = dx * dx + dy * dy;
    if (mode == 0) {
      c = d.wgt[o] * e2;
    } else if (mode == 1) {
      d.wgt[o] = tukey_w(sqrt(e2), maxErr);
    } else {
      const int isOut = (sqrt(e2) >= maxErr) ? 1 : 0;
      outlier[o] = (unsigned char)isOut;
      c = (double)isOut;
    }
  }
  if (PRIOR) {
    const long long nb0 = (d.N + blockDim.x - 1) / blockDim.x;
    if ((long long)blockIdx.x >= nb0)
      c = ba_priors_cost(d, pr, ((long long)blockIdx.x - nb0) * blockDim.x + threadIdx.x, pa, pb);
  }
  if (mode == 2) {  // number of outliers -> sc[SC_COST] (info[13] of the solver entry points)
    const double t = block_sum_1(c, s_red);
    if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[SC_COST], t);
  }
  if (mode == 0) {
    const double t = block_sum_1(c, s_red);
    if (threadIdx.x == 0) {
      if (isfinite(t))
        atomicAdd(&d.sc[SC_COST], t);
      else
        d.sc[SC_NONFINITE] = 1.0;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Linearisation, point-major: per observation e, A (2x6), B (2x3) (whitened by L with OBSCOV, scaled by
// sqrt(w)); stores W_ij = A^T B; collapses V_i = sum B^T B and eb_i = sum B^T e per point with segmented shuffles.
// PRIOR: the CTAs beyond the observations add one point prior per thread, V_i += L^T L and eb_i += L^T L (mu - X)
// (eb sums B^T (x - h), and the prior's "x - h" is -r); a prior point that no observation sees gets its V_i here.
// ------------------------------------------------------------------------------------------
template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(256, 2)
ba_linearize_points(BaDev d, const double* __restrict__ pa, const double* __restrict__ pb, BaPriorDev pr) {
  if (blockIdx.x == 0 && threadIdx.x < 2) d.sc[SC_GINF + threadIdx.x] = 0.0;  // |g|_inf, max diag: set by ba_stats_kernel
  if (PRIOR) {
    const long long nb0 = (d.N + blockDim.x - 1) / blockDim.x;
    if ((long long)blockIdx.x >= nb0) {
      const long long k = ((long long)blockIdx.x - nb0) * blockDim.x + threadIdx.x;
      if (k >= pr.np) return;
      const int i = pr.pt[k];
      const double* __restrict__ q = pr.prec + BA_PTPRIOR_REC * (size_t)k;
      const double X[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
      double rw[3];
      ba_ptprior_eval(pr, (int)k, X, rw);
      const double l00 = q[0], l01 = q[1], l02 = q[2], l11 = q[3], l12 = q[4], l22 = q[5];
      const double H[6] = {l00 * l00, l00 * l01, l00 * l02, l01 * l01 + l11 * l11, l01 * l02 + l11 * l12,
                           l02 * l02 + l12 * l12 + l22 * l22};
      const double g[3] = {l00 * rw[0], l01 * rw[0] + l11 * rw[1], l02 * rw[0] + l12 * rw[1] + l22 * rw[2]};
#pragma unroll
      for (int c = 0; c < 6; ++c) atomicAdd(&d.V[6 * (size_t)i + c], H[c]);
#pragma unroll
      for (int c = 0; c < 3; ++c) atomicAdd(&d.eb[3 * (size_t)i + c], -g[c]);
      return;
    }
  }
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  double acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0;
  int key = -1 - lane;  // inactive lanes never merge
  if (o < d.N) {
    const int j = d.cam[o], i = d.pt[o];
    key = i;
    const double X[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
    double h[2], A[12], B[6];
    ba_project<true, true>(d.camK + 5 * j, d.camR0 + 9 * j, pa + 6 * j, X, h, A, B);
    double r0 = d.xy[2 * o] - h[0], r1 = d.xy[2 * o + 1] - h[1];
    if (OBSCOV) {
      const double* L = d.obsL + 3 * (size_t)o;
      ba_whiten<1>(L, &r0, &r1);
      ba_whiten<3>(L, B, B + 3);
      ba_whiten<6>(L, A, A + 6);
    }
    const double sw = sqrt(d.wgt[o]);
    const double e0 = r0 * sw, e1 = r1 * sw;
#pragma unroll
    for (int k = 0; k < 6; ++k) B[k] *= sw;
    if (i >= d.ncon) {
      acc[0] = B[0] * B[0] + B[3] * B[3];
      acc[1] = B[0] * B[1] + B[3] * B[4];
      acc[2] = B[0] * B[2] + B[3] * B[5];
      acc[3] = B[1] * B[1] + B[4] * B[4];
      acc[4] = B[1] * B[2] + B[4] * B[5];
      acc[5] = B[2] * B[2] + B[5] * B[5];
      acc[6] = B[0] * e0 + B[3] * e1;
      acc[7] = B[1] * e0 + B[4] * e1;
      acc[8] = B[2] * e0 + B[5] * e1;
      if (j >= d.mcon) {
#pragma unroll
        for (int k = 0; k < 12; ++k) A[k] *= sw;
        double* Wp = d.W + 18 * (size_t)o;
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int c = 0; c < 3; ++c) Wp[3 * r + c] = A[r] * B[c] + A[6 + r] * B[3 + c];
      }
    }
  }
  seg_reduce<9>(acc, key, lane);
  const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0) || (kprev != key);
  if (head && key >= d.ncon) {
#pragma unroll
    for (int k = 0; k < 6; ++k) atomicAdd(&d.V[6 * (size_t)key + k], acc[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) atomicAdd(&d.eb[3 * (size_t)key + k], acc[6 + k]);
  }
}

// Linearisation, camera-major over the free-camera observations: U_j = sum A^T A (packed upper,
// 21) and ea_j = sum A^T e (6), collapsed per camera with segmented shuffles.  OBSCOV: A and e whitened by L.
// PRIOR: the CTAs beyond the observations add one prior per thread, U_j += Jw^T Jw and ea_j -= Jw^T rw (ea sums
// A^T (x - h), and the prior's "x - h" is -r); a prior camera that no observation sees gets its U_j here.
template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(128)
ba_linearize_cams(BaDev d, const double* __restrict__ pa, const double* __restrict__ pb, BaPriorDev pr) {
  if (PRIOR) {
    const long long nb0 = (d.Nc + blockDim.x - 1) / blockDim.x;
    if ((long long)blockIdx.x >= nb0) {
      const long long k = ((long long)blockIdx.x - nb0) * blockDim.x + threadIdx.x;
      if (k >= pr.n) return;
      double rw[6], Jw[36];
      ba_prior_eval<true>(d, pr, (int)k, pa, rw, Jw);
      const int j = pr.cam[k];
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) {
          double u = 0.0;
#pragma unroll
          for (int r = 0; r < 6; ++r) u += Jw[6 * r + a] * Jw[6 * r + b];
          atomicAdd(&d.U[21 * (size_t)j + t++], u);
        }
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        double g = 0.0;
#pragma unroll
        for (int r = 0; r < 6; ++r) g += Jw[6 * r + a] * rw[r];
        atomicAdd(&d.ea[6 * (size_t)j + a], -g);
      }
      return;
    }
  }
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0;
  int key = -1 - lane;
  if (q < d.Nc) {
    const int o = d.cobs[q], j = d.ccam[q], i = d.pt[o];
    key = j;
    const double X[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
    double h[2], A[12];
    ba_project<true, false>(d.camK + 5 * j, d.camR0 + 9 * j, pa + 6 * j, X, h, A, nullptr);
    double r0 = d.xy[2 * (size_t)o] - h[0], r1 = d.xy[2 * (size_t)o + 1] - h[1];
    if (OBSCOV) {
      const double* L = d.obsL + 3 * (size_t)o;
      ba_whiten<1>(L, &r0, &r1);
      ba_whiten<6>(L, A, A + 6);
    }
    const double sw = sqrt(d.wgt[o]);
    const double e0 = r0 * sw, e1 = r1 * sw;
#pragma unroll
    for (int k = 0; k < 12; ++k) A[k] *= sw;
    int t = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c) acc[t++] = A[r] * A[c] + A[6 + r] * A[6 + c];
#pragma unroll
    for (int r = 0; r < 6; ++r) acc[21 + r] = A[r] * e0 + A[6 + r] * e1;
  }
  seg_reduce<27>(acc, key, lane);
  const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0) || (kprev != key);
  if (head && key >= 0) {
#pragma unroll
    for (int k = 0; k < 21; ++k) atomicAdd(&d.U[21 * (size_t)key + k], acc[k]);
#pragma unroll
    for (int k = 0; k < 6; ++k) atomicAdd(&d.ea[6 * (size_t)key + k], acc[21 + k]);
  }
}

// |g|_inf and max diag over (U, ea) of the free cameras [global after all-reduce] and (V, eb) of
// this rank's free points.
__global__ void __launch_bounds__(256) ba_stats_kernel(BaDev d) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double g = 0, dg = 0;
  if (t < d.n) {
    if (t >= d.ncon) {
      const double* V = d.V + 6 * t;
      const double* e = d.eb + 3 * t;
      g = fmax(fabs(e[0]), fmax(fabs(e[1]), fabs(e[2])));
      dg = fmax(V[0], fmax(V[3], V[5]));
    }
  } else if (t < (long long)d.n + d.m) {
    const int j = (int)(t - d.n);
    if (j >= d.mcon) {
      const double* U = d.U + 21 * (size_t)j;
      const double* e = d.ea + 6 * (size_t)j;
      // packed upper: diagonal entries at offsets 0, 6, 11, 15, 18, 20
      dg = fmax(fmax(U[0], U[6]), fmax(fmax(U[11], U[15]), fmax(U[18], U[20])));
#pragma unroll
      for (int k = 0; k < 6; ++k) g = fmax(g, fabs(e[k]));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    g = fmax(g, __shfl_xor_sync(0xffffffffu, g, o));
    dg = fmax(dg, __shfl_xor_sync(0xffffffffu, dg, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (g > 0) atomic_max_nonneg(&d.sc[SC_GINF], g);
    if (dg > 0) atomic_max_nonneg(&d.sc[SC_MAXDIAG], dg);
  }
}

// S <- 0 with the damped camera blocks U*_j on the diagonal tiles, rhs <- ea.  One CTA per tile
// (blockIdx.x < nTiles) zeroes it and, if it is the diagonal tile of block k (diagBlk[t] = k), writes
// the lower part of U_j + mu I for the cameras order[blkCam0[k] .. blkCam0[k+1]) of that block and
// their slice of rhs.  addU: this rank contributes U/ea/mu (rank 0 only in the multi-GPU case, where
// U/ea are already all-reduced).  Padding rows of a block stay zero (the factorisation treats them
// as identity).
__device__ __forceinline__ void ba_tile_init_body(const BaDev& d, double mu, int addU, const int* __restrict__ diagBlk,
                                                  const int* __restrict__ blkCam0, const int* __restrict__ order) {
  const int t = blockIdx.x;
  double2* tile = reinterpret_cast<double2*>(d.tiles + (size_t)t * 4096);
  const double2 z = make_double2(0.0, 0.0);
#pragma unroll
  for (int u = 0; u < 8; ++u) tile[threadIdx.x + 256 * u] = z;
  const int k = diagBlk[t];
  if (k < 0) return;
  if (threadIdx.x < 64) d.rhs[(size_t)k * 64 + threadIdx.x] = 0.0;
  __syncthreads();
  if (!addU) return;
  const int p0 = blkCam0[k], ncam = blkCam0[k + 1] - p0;
  for (int e = threadIdx.x; e < ncam * 27; e += 256) {
    const int c = e / 27, q = e - 27 * c;
    const int cam = order[p0 + c] + d.mcon;
    const int off = 6 * c;
    if (q < 21) {
      // packed upper index q -> (a <= b); stored at row off+b, column off+a of the lower tile
      int a = 0, rem = q;
      while (rem >= 6 - a) {
        rem -= 6 - a;
        ++a;
      }
      const int b = a + rem;
      double v = d.U[21 * (size_t)cam + q];
      if (a == b) v += mu;
      d.tiles[(size_t)t * 4096 + (off + a) * 64 + off + b] = v;
    } else {
      d.rhs[(size_t)k * 64 + off + (q - 21)] = d.ea[6 * (size_t)cam + (q - 21)];
    }
  }
}

// ------------------------------------------------------------------------------------------
// Schur contraction over camera pairs.  Work item = a run of (obsA, obsB) entries that belong to
// one camera pair (j <= k): block(j,k) -= sum_i W_ij V*_i^-1 W_ik^T (and, for j == k,
// rhs_j -= sum_i W_ij V*_i^-1 eb_i).  One warp per item (ba_schur_pairs_st below); the items of a
// pair add into its block with atomics.
// ------------------------------------------------------------------------------------------
struct BaPairItem {
  int rowCam, colCam;  // free-camera indices (0-based in the reduced system)
  int begin, end;      // entry range
  // destination of the 6x6 block acc(r, c) (r: row camera's parameter, c: column camera's):
  // tiles[dst + (cOff + (trans ? c : r)) * 64 + rOff + (trans ? r : c)] -- the block lands in the
  // LOWER triangle of the permuted system whichever of the two cameras comes first in the ordering
  int dst, rOff, cOff, trans;
  int rhsIdx, pad0, pad1, pad2;  // rhs index of the row camera (diagonal items only)
};

__device__ __forceinline__ void inv3sym_mu(const double* __restrict__ V, double mu, double I[6]) {
  const double a = V[0] + mu, b = V[1], c = V[2], d = V[3] + mu, e = V[4], f = V[5] + mu;
  const double A = d * f - e * e, B = c * e - b * f, C = b * e - c * d;
  const double r = 1.0 / (a * A + b * B + c * C);
  I[0] = A * r;
  I[1] = B * r;
  I[2] = C * r;
  I[3] = (a * f - c * c) * r;
  I[4] = (b * c - a * e) * r;
  I[5] = (a * d - b * b) * r;
}

// One launch in front of every Schur contraction ("prep"): blocks [0, nTiles) initialise the tiles
// (ba_tile_init_body), the following blocks compute the damped inverses V*_i^-1 (one point per thread) and --
// when a linearisation preceded this trial (doStats) -- the gradient / diagonal statistics |g|_inf and
// max diag(U, V) that the host needs for the eps1 test (it reads them with the trial's scalars).  Block 0
// also clears the scalars of the trial and the grid clears the task counters of the solve.  ctl (the submitted
// loop): mu and doStats come from the control block.
__global__ void __launch_bounds__(256)
ba_prep_kernel(BaDev d, const BaCtl* __restrict__ ctl, double mu, int addU, const int* __restrict__ diagBlk,
               const int* __restrict__ blkCam0, const int* __restrict__ order, int* __restrict__ cnt, int nCnt,
               int nTiles, double* __restrict__ Vinv, int doStats, double* __restrict__ zeroBuf,
               long long zeroCount) {
  if (ctl) {
    mu = ctl->mu;
    doStats = ctl->statsPending;
  }
  for (int q = blockIdx.x * 256 + threadIdx.x; q < nCnt; q += gridDim.x * 256) cnt[q] = 0;
  // accumulator of the point back-substitution (ba_back_cams_points)
  for (long long q = (long long)blockIdx.x * 256 + threadIdx.x; q < zeroCount; q += (long long)gridDim.x * 256)
    zeroBuf[q] = 0.0;
  if (blockIdx.x == 0 && threadIdx.x < 6) {
    const int slot[6] = {SC_DP_L2, SC_DL, SC_P_L2, SC_FAIL, SC_COST, SC_NONFINITE};
    d.sc[slot[threadIdx.x]] = 0.0;
  }
  if ((int)blockIdx.x < nTiles) {
    ba_tile_init_body(d, mu, addU, diagBlk, blkCam0, order);
    return;
  }
  const long long t = (long long)(blockIdx.x - nTiles) * 256 + threadIdx.x;
  double g = 0, dg = 0;
  if (t < d.n) {
    double I[6] = {0, 0, 0, 0, 0, 0};
    if (t >= d.ncon) {
      const double* V = d.V + 6 * t;
      inv3sym_mu(V, mu, I);
      if (doStats) {
        const double* e = d.eb + 3 * t;
        g = fmax(fabs(e[0]), fmax(fabs(e[1]), fabs(e[2])));
        dg = fmax(V[0], fmax(V[3], V[5]));
      }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) Vinv[6 * t + k] = I[k];
  } else if (doStats && t < (long long)d.n + d.m) {
    const int j = (int)(t - d.n);
    if (j >= d.mcon) {
      const double* U = d.U + 21 * (size_t)j;
      const double* e = d.ea + 6 * (size_t)j;
      dg = fmax(fmax(U[0], U[6]), fmax(fmax(U[11], U[15]), fmax(U[18], U[20])));
#pragma unroll
      for (int k = 0; k < 6; ++k) g = fmax(g, fabs(e[k]));
    }
  }
  if (doStats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      g = fmax(g, __shfl_xor_sync(0xffffffffu, g, o));
      dg = fmax(dg, __shfl_xor_sync(0xffffffffu, dg, o));
    }
    if ((threadIdx.x & 31) == 0) {
      if (g > 0) atomic_max_nonneg(&d.sc[SC_GINF], g);
      if (dg > 0) atomic_max_nonneg(&d.sc[SC_MAXDIAG], dg);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Pair-list contraction.  The damped inverses V*^-1 are computed once per trial (ba_prep_kernel) and an
// entry carries its point index ({obsA, obsB, point, -}), so the rows of an entry are one dependent load
// below its descriptor.  Gathering those rows with scalar 8-byte loads by the lanes that consume them
// touches ~16 different 128-byte lines per load instruction, and L1TEX wavefronts bound such a kernel;
// the rows are therefore staged.  A warp works on 32 entries at a time:
//   1. STAGE: the 21 16-byte segments of every entry -- W_a (9), W_b (9), V*^-1 (3) -- are copied with
//      cp.async in SEGMENT-major order (consecutive lanes copy consecutive segments of the same row, so
//      one instruction touches ~8 lines instead of 32: ~5 wavefronts per entry), into a row of 42
//      doubles per entry (336 B = 21 x 16 B, an odd multiple of 16 B: conflict-free 16-byte reads);
//   2. CONTRACT: lane j owns entry j, reads its row with 21 LDS.128 and accumulates the whole 6x6 block
//      (+ the 6 right-hand-side terms of diagonal items) in registers: 162 DFMA per entry;
//   3. the next batch is in flight (second buffer) while the current one is contracted;
//   4. at the end of the item the 32 partial blocks are summed through the (now free) staging buffer:
//      lane k adds up element k of all lanes -- 36 + 6 elements, one atomic each.
// ------------------------------------------------------------------------------------------
constexpr int BA_ST_WARPS = 4;
constexpr int BA_ST_ROW = 42;                                   // doubles per staged entry
constexpr int BA_ST_BUF = 32 * BA_ST_ROW;                       // doubles per batch buffer (10752 B)
constexpr int BA_ST_SMEM = BA_ST_WARPS * 2 * BA_ST_BUF * 8;     // 86016 B per CTA (dynamic)

__device__ __forceinline__ void ba_cp_async16(double* smemDst, const double* gsrc) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smemDst);
  // .cg: L2 only.  Allocating in L1 (.ca; the four warps of a CTA work on partner cameras of the same row
  // camera) was tried: no measurable difference at c4.
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gsrc) : "memory");
}

// copy the rows of the batch whose entry descriptors the lanes hold (lane j: entry j; ne valid entries)
__device__ __forceinline__ void ba_st_stage(const BaDev& d, const double* __restrict__ Vinv, int4 ob, int ne,
                                            int lane, double* buf) {
#pragma unroll
  for (int t = 0; t < 9; ++t) {  // W_a and W_b: 32 rows x 9 segments each
    const int sidx = t * 32 + lane, j = sidx / 9, part = sidx - 9 * j;
    const int oa = __shfl_sync(0xffffffffu, ob.x, j), obb = __shfl_sync(0xffffffffu, ob.y, j);
    if (j < ne) {
      ba_cp_async16(buf + j * BA_ST_ROW + 2 * part, d.W + 18 * (size_t)oa + 2 * part);
      ba_cp_async16(buf + j * BA_ST_ROW + 18 + 2 * part, d.W + 18 * (size_t)obb + 2 * part);
    }
  }
#pragma unroll
  for (int t = 0; t < 3; ++t) {  // V*^-1: 32 rows x 3 segments
    const int sidx = t * 32 + lane, j = sidx / 3, part = sidx - 3 * j;
    const int pi = __shfl_sync(0xffffffffu, ob.z, j);
    if (j < ne) ba_cp_async16(buf + j * BA_ST_ROW + 36 + 2 * part, Vinv + 6 * (size_t)pi + 2 * part);
  }
  asm volatile("cp.async.commit_group;\n" ::: "memory");
}

__global__ void __launch_bounds__(32 * BA_ST_WARPS, 2)
ba_schur_pairs_st(BaDev d, const BaPairItem* __restrict__ items, int nItems, const int4* __restrict__ entries,
                  const double* __restrict__ Vinv) {
  extern __shared__ __align__(16) double s_st[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * BA_ST_WARPS + w;
  if (item >= nItems) return;
  const BaPairItem it = items[item];
  const bool diag = (it.rowCam == it.colCam);
  double* buf0 = s_st + (size_t)w * 2 * BA_ST_BUF;
  double acc[36], racc[6];
#pragma unroll
  for (int k = 0; k < 36; ++k) acc[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) racc[k] = 0.0;
  const int nb = (it.end - it.begin + 31) >> 5;
  const int4 zero4 = make_int4(0, 0, 0, 0);
  int4 cur = (it.begin + lane < it.end) ? __ldg(&entries[it.begin + lane]) : zero4;
  int4 nxt = (it.begin + 32 + lane < it.end) ? __ldg(&entries[it.begin + 32 + lane]) : zero4;
  ba_st_stage(d, Vinv, cur, min(32, it.end - it.begin), lane, buf0);
  for (int b = 0; b < nb; ++b) {
    const int e0 = it.begin + 32 * b;
    const int4 mine = cur;  // descriptor of this lane's entry in batch b (point index for e_b)
    cur = nxt;
    if (b + 1 < nb) {
      nxt = (e0 + 64 + lane < it.end) ? __ldg(&entries[e0 + 64 + lane]) : zero4;
      ba_st_stage(d, Vinv, cur, min(32, it.end - (e0 + 32)), lane, buf0 + ((b + 1) & 1) * BA_ST_BUF);
      asm volatile("cp.async.wait_group 1;\n" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    }
    __syncwarp();
    if (e0 + lane < it.end) {
      const double* row = buf0 + (b & 1) * BA_ST_BUF + lane * BA_ST_ROW;
      double wa[18], wb[18], Iv[6];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = *reinterpret_cast<const double2*>(row + 2 * k);
        wa[2 * k] = v.x;
        wa[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = *reinterpret_cast<const double2*>(row + 18 + 2 * k);
        wb[2 * k] = v.x;
        wb[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double2 v = *reinterpret_cast<const double2*>(row + 36 + 2 * k);
        Iv[2 * k] = v.x;
        Iv[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const double b0 = wb[3 * c], b1 = wb[3 * c + 1], b2 = wb[3 * c + 2];
        const double t0 = Iv[0] * b0 + Iv[1] * b1 + Iv[2] * b2;
        const double t1 = Iv[1] * b0 + Iv[3] * b1 + Iv[4] * b2;
        const double t2 = Iv[2] * b0 + Iv[4] * b1 + Iv[5] * b2;
#pragma unroll
        for (int r = 0; r < 6; ++r) acc[6 * r + c] += wa[3 * r] * t0 + wa[3 * r + 1] * t1 + wa[3 * r + 2] * t2;
      }
      if (diag) {
        const double* eb = d.eb + 3 * (size_t)mine.z;
        const double e0v = eb[0], e1v = eb[1], e2v = eb[2];
        const double t0 = Iv[0] * e0v + Iv[1] * e1v + Iv[2] * e2v;
        const double t1 = Iv[1] * e0v + Iv[3] * e1v + Iv[4] * e2v;
        const double t2 = Iv[2] * e0v + Iv[4] * e1v + Iv[5] * e2v;
#pragma unroll
        for (int r = 0; r < 6; ++r) racc[r] += wa[3 * r] * t0 + wa[3 * r + 1] * t1 + wa[3 * r + 2] * t2;
      }
    }
    __syncwarp();  // the buffer of batch b is free again (restaged at iteration b + 1)
  }
  // ---- sum over the 32 lanes through shared memory: red[k * 33 + lane]
  double* red = buf0;  // 42 x 33 doubles = 11088 B <= 2 buffers
#pragma unroll
  for (int k = 0; k < 36; ++k) red[k * 33 + lane] = acc[k];
  if (diag) {
#pragma unroll
    for (int k = 0; k < 6; ++k) red[(36 + k) * 33 + lane] = racc[k];
  }
  __syncwarp();
  double* T = d.tiles + it.dst;
  for (int k = lane; k < (diag ? 42 : 36); k += 32) {
    double sum = 0.0;
#pragma unroll 8
    for (int l = 0; l < 32; ++l) sum += red[k * 33 + l];
    if (k < 36) {
      const int r = k / 6, c = k - 6 * r;
      // only the lower part (row >= col of the tile, i.e. c >= r) of diagonal blocks is kept
      if (!diag || c >= r) {
        const int col = it.cOff + (it.trans ? c : r), row = it.rOff + (it.trans ? r : c);
        atomicAdd(&T[col * 64 + row], -sum);
      }
    } else {
      atomicAdd(&d.rhs[it.rhsIdx + (k - 36)], -sum);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Pair work lists built on the device (solver set-up).  For every free observation a = (camera ja,
// point i) of the camera-major list and every observation b of the same point with camera jb > ja,
// or jb == ja and b >= a: one entry in bucket (ja, jb).  The bucket offsets come from the host's
// count (cosl_ba_solver_load); FILL places {a, b, i} at offset + running index.  (A host version
// wrote 81 MB of entries at c4 and uploaded them, which dominated solver creation.)  The order
// inside a bucket depends on the atomics; the contraction sums the same terms in a different order.
// ------------------------------------------------------------------------------------------
template <bool FILL>
__global__ void __launch_bounds__(256)
ba_pairs_build(BaDev d, unsigned* __restrict__ cnt, const unsigned* __restrict__ off,
               int4* __restrict__ entries) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= d.Nc) return;
  const int a = d.cobs[q], i = d.pt[a];
  if (i < d.ncon) return;
  const int ja = d.cam[a] - d.mcon;
  const long long o0 = d.ptr[i], o1 = d.ptr[i + 1];
  for (long long b = o0; b < o1; ++b) {
    const int jb = d.cam[b] - d.mcon;
    if (jb > ja || (jb == ja && b >= a)) {
      const size_t bucket = (size_t)ja * d.mf + jb;
      const unsigned k = atomicAdd(&cnt[bucket], 1u);
      if (FILL) entries[off[bucket] + k] = make_int4(a, (int)b, i, 0);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Observation index lists built on the device (cosl_ba_solver_load).  ba_index_points expands the
// point-major CSR into pt[o].  ba_index_cams builds the camera-major list of the free-camera
// observations (cobs, ccam) as a STABLE counting sort, so that every camera's observations stay in
// ascending o, the order in which ba_linearize_cams sums them: one warp per chunk of `chunk`
// consecutive observations.  Pass PLACE = false counts each free camera's observations of the chunk
// into hist[chunk][mf] (zeroed before); ba_index_cam_base turns every column into the offsets of the
// chunk in cobs (the camera's start + the counts of the earlier chunks); PLACE = true puts each
// observation at its chunk offset + its rank among the camera's earlier observations of the chunk.
// A warp owns its row of hist, so the running counts need no atomics.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ba_index_points(const long long* __restrict__ ptr, int n, int* __restrict__ pt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (long long o = ptr[i]; o < ptr[i + 1]; ++o) pt[o] = i;
}

template <bool PLACE>
__global__ void __launch_bounds__(256)
ba_index_cams(const int* __restrict__ cam, long long N, int mcon, int mf, int chunk, unsigned* __restrict__ hist,
              int* __restrict__ cobs, int* __restrict__ ccam) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long o0 = w * chunk;
  if (o0 >= N) return;  // warp-uniform
  const long long o1 = min(N, o0 + chunk);
  unsigned* row = hist + w * mf;
  for (long long b = o0; b < o1; b += 32) {
    const long long o = b + lane;
    const int j = o < o1 ? cam[o] - mcon : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, j);
    if (PLACE && j >= 0) {
      const unsigned q = row[j] + __popc(peers & ((1u << lane) - 1u));
      cobs[q] = (int)o;
      ccam[q] = j + mcon;
    }
    __syncwarp();
    if (j >= 0 && lane == 31 - __clz(peers)) row[j] += __popc(peers);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(256)
ba_index_cam_base(unsigned* __restrict__ hist, int nChunks, int mf, const unsigned* __restrict__ camStart) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= mf) return;
  unsigned run = camStart[j];
  for (int c = 0; c < nChunks; ++c) {
    const unsigned v = hist[(size_t)c * mf + j];
    hist[(size_t)c * mf + j] = run;
    run += v;
  }
}

// ------------------------------------------------------------------------------------------
// Back substitution, step 1, point-major, one observation per thread: t_i = sum_j W_ij^T da_j,
// collapsed per point with segmented shuffles; run heads add into acc3[n][3] (zeroed before).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ba_back_subst(BaDev d, const double* __restrict__ dpa, double* __restrict__ acc3) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  double acc[3] = {0, 0, 0};
  int key = -1 - lane;
  if (o < d.N) {
    const int j = d.cam[o], i = d.pt[o];
    key = i;
    if (i >= d.ncon && j >= d.mcon) {
      const double* Wp = d.W + 18 * (size_t)o;
      const double* da = dpa + 6 * (size_t)j;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double s = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r) s += Wp[3 * r + c] * da[r];
        acc[c] = s;
      }
    }
  }
  seg_reduce<3>(acc, key, lane);
  const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0) || (kprev != key);
  if (head && key >= d.ncon) {
#pragma unroll
    for (int c = 0; c < 3; ++c) atomicAdd(&acc3[3 * (size_t)key + c], acc[c]);
  }
}

// Back substitution, step 2, one point per thread: nb holds t_i on entry; db_i = V*_i^-1 (eb_i - t_i),
// nb <- pb + db, plus the point-side parts of |dp|^2, dL, |p|^2.
// ctl (the submitted loop): mu comes from the control block.
__global__ void __launch_bounds__(256)
ba_back_finish(BaDev d, const BaCtl* __restrict__ ctl, const double* __restrict__ pb, double* __restrict__ nb,
               double* __restrict__ dpb, double mu) {
  if (ctl) mu = ctl->mu;
  __shared__ double s_red[8];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double dp2 = 0, dl = 0, p2 = 0;
  if (i < d.n) {
    double x[3] = {pb[3 * i], pb[3 * i + 1], pb[3 * i + 2]};
    double db[3] = {0, 0, 0};
    if (i >= d.ncon) {
      double Iv[6];
      inv3sym_mu(d.V + 6 * i, mu, Iv);
      const double* eb = d.eb + 3 * i;
      const double t0 = eb[0] - nb[3 * i], t1 = eb[1] - nb[3 * i + 1], t2 = eb[2] - nb[3 * i + 2];
      db[0] = Iv[0] * t0 + Iv[1] * t1 + Iv[2] * t2;
      db[1] = Iv[1] * t0 + Iv[3] * t1 + Iv[4] * t2;
      db[2] = Iv[2] * t0 + Iv[4] * t1 + Iv[5] * t2;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dp2 += db[c] * db[c];
        dl += db[c] * (mu * db[c] + eb[c]);
        p2 += x[c] * x[c];
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      dpb[3 * i + c] = db[c];
      nb[3 * i + c] = x[c] + db[c];
    }
  }
  double t = block_sum_1(dp2, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[SC_DP_L2], t);
  t = block_sum_1(dl, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[SC_DL], t);
  t = block_sum_1(p2, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[SC_P_L2], t);
}

// Trial camera parameters na = pa + dpa and the camera-side parts of |dp|^2, dL, |p|^2.
// addSums: only one rank contributes the (replicated) camera-side sums.  ctl: mu from the control block.
__global__ void __launch_bounds__(256)
ba_cam_update(BaDev d, const BaCtl* __restrict__ ctl, const double* __restrict__ pa, const double* __restrict__ sol,
              double* __restrict__ dpa, double* __restrict__ na, double mu, int addSums, double* __restrict__ zeroBuf,
              long long zeroCount) {
  if (ctl) mu = ctl->mu;
  __shared__ double s_red[8];
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  for (long long q = t; q < zeroCount; q += (long long)gridDim.x * blockDim.x) zeroBuf[q] = 0.0;
  double dp2 = 0, dl = 0, p2 = 0;
  if (t < 6 * d.m) {
    const int j = t / 6, r = t - 6 * j;
    double dlt = 0;
    if (j >= d.mcon) {
      dlt = sol[d.solIdx[j - d.mcon] + r];
      dp2 = dlt * dlt;
      dl = dlt * (mu * dlt + d.ea[t]);
      p2 = pa[t] * pa[t];
    }
    dpa[t] = dlt;
    na[t] = pa[t] + dlt;
  }
  double s = block_sum_1(dp2, s_red);
  if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_DP_L2], s);
  s = block_sum_1(dl, s_red);
  if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_DL], s);
  s = block_sum_1(p2, s_red);
  if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_P_L2], s);
}

// ------------------------------------------------------------------------------------------
// Back substitution in two launches (instead of cam update | memset | point accumulate | point finish | cost):
//  ba_back_cams_points: blocks [0, nCamBlocks) form the trial camera parameters na = pa + da and the camera-side
//    parts of |dp|^2, dL, |p|^2 (ba_cam_update); the other blocks accumulate t_i = sum_j W_ij^T da_j per point
//    (one observation per thread, segmented shuffles, heads add into acc3, which the prep kernel zeroed),
//    reading da straight from the solution vector;
//  ba_finish_cost: one observation per thread: db_i = V*_i^-1 (e_b,i - t_i) recomputed from the point's
//    accumulator (read-only here; the FIRST observation of a point stores nb_i = pb_i + db_i and adds the
//    point-side sums), then the weighted squared residual at (na, nb_i) -> cost (whitened with OBSCOV).  Extra
//    threads finish the points that have no observation; with PRIOR, the CTAs after those add the priors' |L r|^2,
//    a camera prior's at na, a point prior's at its trial point recomputed from the accumulator as above (nb is
//    written by other threads of the launch).
// Both take mu from ctl, the control block of the submitted loop, when it is set.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ba_back_cams_points(BaDev d, const BaCtl* __restrict__ ctl, const double* __restrict__ pa,
                    const double* __restrict__ sol, double* __restrict__ dpa, double* __restrict__ na, double mu,
                    int addSums, int nCamBlocks, double* __restrict__ acc3) {
  __shared__ double s_red[8];
  if ((int)blockIdx.x < nCamBlocks) {
    if (ctl) mu = ctl->mu;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    double dp2 = 0, dl = 0, p2 = 0;
    if (t < 6 * d.m) {
      const int j = t / 6, r = t - 6 * j;
      double dlt = 0;
      if (j >= d.mcon) {
        dlt = sol[d.solIdx[j - d.mcon] + r];
        dp2 = dlt * dlt;
        dl = dlt * (mu * dlt + d.ea[t]);
        p2 = pa[t] * pa[t];
      }
      dpa[t] = dlt;
      na[t] = pa[t] + dlt;
    }
    double s = block_sum_1(dp2, s_red);
    if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_DP_L2], s);
    s = block_sum_1(dl, s_red);
    if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_DL], s);
    s = block_sum_1(p2, s_red);
    if (threadIdx.x == 0 && addSums && s != 0) atomicAdd(&d.sc[SC_P_L2], s);
    return;
  }
  const long long o = (long long)(blockIdx.x - nCamBlocks) * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  double acc[3] = {0, 0, 0};
  int key = -1 - lane;
  if (o < d.N) {
    const int j = d.cam[o], i = d.pt[o];
    key = i;
    if (i >= d.ncon && j >= d.mcon) {
      const double* Wp = d.W + 18 * (size_t)o;
      const double* da = sol + d.solIdx[j - d.mcon];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double s = 0;
#pragma unroll
        for (int r = 0; r < 6; ++r) s += Wp[3 * r + c] * da[r];
        acc[c] = s;
      }
    }
  }
  seg_reduce<3>(acc, key, lane);
  const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0) || (kprev != key);
  if (head && key >= d.ncon) {
#pragma unroll
    for (int c = 0; c < 3; ++c) atomicAdd(&acc3[3 * (size_t)key + c], acc[c]);
  }
}

template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(256)
ba_finish_cost(BaDev d, const BaCtl* __restrict__ ctl, const double* __restrict__ na, const double* __restrict__ pb,
               double* __restrict__ nb, const double* __restrict__ acc3, const double* __restrict__ Vinv, double mu,
               BaPriorDev pr) {
  if (ctl) mu = ctl->mu;
  __shared__ double s_red[8];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double dp2 = 0, dl = 0, p2 = 0, c = 0;
  long long o = -1;
  int i = -1;
  bool store = false;
  if (t < d.N) {
    o = t;
    i = d.pt[o];
    store = (d.ptr[i] == o);
  } else if (t < d.N + d.n) {
    i = (int)(t - d.N);
    store = (d.ptr[i + 1] == d.ptr[i]);  // a point nobody observes is finished here
    if (!store) i = -1;
  }
  if (i >= 0) {
    double x[3] = {pb[3 * (size_t)i], pb[3 * (size_t)i + 1], pb[3 * (size_t)i + 2]};
    double db[3] = {0, 0, 0};
    if (i >= d.ncon) {
      const double* Iv = Vinv + 6 * (size_t)i;
      const double* eb = d.eb + 3 * (size_t)i;
      const double t0 = eb[0] - acc3[3 * (size_t)i], t1 = eb[1] - acc3[3 * (size_t)i + 1],
                   t2 = eb[2] - acc3[3 * (size_t)i + 2];
      db[0] = Iv[0] * t0 + Iv[1] * t1 + Iv[2] * t2;
      db[1] = Iv[1] * t0 + Iv[3] * t1 + Iv[4] * t2;
      db[2] = Iv[2] * t0 + Iv[4] * t1 + Iv[5] * t2;
      if (store) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          dp2 += db[k] * db[k];
          dl += db[k] * (mu * db[k] + eb[k]);
          p2 += x[k] * x[k];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) x[k] += db[k];
    if (store) {
#pragma unroll
      for (int k = 0; k < 3; ++k) nb[3 * (size_t)i + k] = x[k];
    }
    if (o >= 0) {
      const int j = d.cam[o];
      double h[2];
      ba_project<false, false>(d.camK + 5 * j, d.camR0 + 9 * j, na + 6 * j, x, h, nullptr, nullptr);
      double dx = d.xy[2 * o] - h[0], dy = d.xy[2 * o + 1] - h[1];
      if (OBSCOV) ba_whiten<1>(d.obsL + 3 * (size_t)o, &dx, &dy);
      c = d.wgt[o] * (dx * dx + dy * dy);
    }
  }
  if (PRIOR) {
    const long long nb0 = (d.N + d.n + blockDim.x - 1) / blockDim.x;
    if ((long long)blockIdx.x >= nb0) {
      const long long k = ((long long)blockIdx.x - nb0) * blockDim.x + threadIdx.x;
      if (k < pr.n) {
        c = ba_prior_cost(d, pr, (int)k, na);
      } else if (k < pr.n + (long long)pr.np) {
        const int kp = (int)(k - pr.n), ip = pr.pt[kp];
        const double* Iv = Vinv + 6 * (size_t)ip;
        const double* eb = d.eb + 3 * (size_t)ip;
        const double t0 = eb[0] - acc3[3 * (size_t)ip], t1 = eb[1] - acc3[3 * (size_t)ip + 1],
                     t2 = eb[2] - acc3[3 * (size_t)ip + 2];
        const double X[3] = {pb[3 * (size_t)ip] + (Iv[0] * t0 + Iv[1] * t1 + Iv[2] * t2),
                             pb[3 * (size_t)ip + 1] + (Iv[1] * t0 + Iv[3] * t1 + Iv[4] * t2),
                             pb[3 * (size_t)ip + 2] + (Iv[2] * t0 + Iv[4] * t1 + Iv[5] * t2)};
        c = ba_ptprior_cost(pr, kp, X);
      }
    }
  }
  double s = block_sum_1(c, s_red);
  if (threadIdx.x == 0) {
    if (isfinite(s)) {
      if (s != 0) atomicAdd(&d.sc[SC_COST], s);
    } else {
      d.sc[SC_NONFINITE] = 1.0;
    }
  }
  s = block_sum_1(dp2, s_red);
  if (threadIdx.x == 0 && s != 0) atomicAdd(&d.sc[SC_DP_L2], s);
  s = block_sum_1(dl, s_red);
  if (threadIdx.x == 0 && s != 0) atomicAdd(&d.sc[SC_DL], s);
  s = block_sum_1(p2, s_red);
  if (threadIdx.x == 0 && s != 0) atomicAdd(&d.sc[SC_P_L2], s);
}

// ------------------------------------------------------------------------------------------
// Covariance stage (cosl_ba_solver_set_covariance, DESIGN.md 4.6).  It re-linearises with the kernels above
// through a BaDev of its own (weights, scalars), so nothing the LM loop keeps between calls changes.  Its
// scalars: [0, SC_NTOT) those of that BaDev, then the slots below.
// ------------------------------------------------------------------------------------------
enum BaCovScalar {
  COV_T0 = SC_NTOT,   // globaltimer at the start of the stage (bits of a uint64)
  COV_NOBS = 17,      // observations with w > 0 that enter H
  COV_NPTS = 18,      // free points with a covariance
  COV_NUNC = 19,      // free points with fewer than two observations of non-zero weight
  COV_SING = 20,      // 1: the reduced system is singular in the gauge
  COV_OUT = 24,       // [8]: the out vector of cosl_ba_solver_download_covariance
  COV_NTOT = 32
};
constexpr double BA_COV_MIN_PIVOT = 1e-12;  // smallest relative pivot L_ii^2 / S_ii of a regular system

__global__ void __launch_bounds__(256)
ba_cov_begin(double* __restrict__ sc, double* __restrict__ T, long long nT, int* __restrict__ cnt, int nCnt) {
  const long long q0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, st = (long long)gridDim.x * blockDim.x;
  for (long long q = q0; q < nT; q += st) T[q] = 0.0;
  for (long long q = q0; q < nCnt; q += st) cnt[q] = 0;
  if (q0 < COV_NTOT - COV_T0) sc[COV_T0 + q0] = 0.0;
  __syncthreads();
  if (q0 == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    *reinterpret_cast<unsigned long long*>(sc + COV_T0) = t;
  }
}

// One thread per point: free points with fewer than two observations of non-zero weight are left out of H
// (their weights are zeroed, unc[i] = 1); counts of the observations and points that enter H.  PRIOR (point
// priors set): a point with a prior always enters H, its V_i holds P^-1.
template <bool PRIOR>
__global__ void __launch_bounds__(256) ba_cov_mask(BaDev d, unsigned char* __restrict__ unc, BaPriorDev pr) {
  __shared__ double s_red[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double nobs = 0, npts = 0, nunc = 0;
  if (i < d.n) {
    int k = 0;
    for (long long o = d.ptr[i]; o < d.ptr[i + 1]; ++o) k += d.wgt[o] > 0.0 ? 1 : 0;
    const bool u = i >= d.ncon && k < 2 && !(PRIOR && pr.has[i]);
    unc[i] = u ? 1 : 0;
    if (u) {
      for (long long o = d.ptr[i]; o < d.ptr[i + 1]; ++o) d.wgt[o] = 0.0;
      nunc = 1;
    } else {
      nobs = k;
      npts = i >= d.ncon ? 1 : 0;
    }
  }
  double t = block_sum_1(nobs, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[COV_NOBS], t);
  t = block_sum_1(npts, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[COV_NPTS], t);
  t = block_sum_1(nunc, s_red);
  if (threadIdx.x == 0 && t != 0) atomicAdd(&d.sc[COV_NUNC], t);
}

// V^-1 of a point left out of H is 0, not the inverse of its zero V (the Schur contraction reads it)
__global__ void __launch_bounds__(256)
ba_cov_vfix(const unsigned char* __restrict__ unc, double* __restrict__ Vinv, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && unc[i])
    for (int k = 0; k < 6; ++k) Vinv[6 * (size_t)i + k] = 0.0;
}

// diagonal of S before the factorisation overwrites it (relative pivots); one CTA of 64 per block
__global__ void ba_cov_sdiag(const double* __restrict__ tiles, const int* __restrict__ diagTile,
                             double* __restrict__ sdiag) {
  const int k = blockIdx.x, r = threadIdx.x;
  sdiag[(size_t)k * 64 + r] = tiles[(size_t)diagTile[k] * 4096 + (size_t)r * 65];
}

// Camera blocks: Z_jj in the solver's chart (v, t), R = R(q(v)) R0, turned into (w, t) with
// R' = exp([w]x) R: w = J dv, J = 2 (w_q I + [v]x + v v^T / w_q), w_q = sqrt(1 - |v|^2).  camCov[j] =
// var * T Z_jj T^T with T = diag(J, I), row-major 6x6; zeros for the fixed cameras.
__global__ void __launch_bounds__(128)
ba_cov_cams(BaDev d, const double* __restrict__ pa, const double* __restrict__ Z, const int* __restrict__ diagTile,
            double var, double* __restrict__ camCov) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d.m) return;
  double* out = camCov + 36 * (size_t)j;
  if (j < d.mcon) {
    for (int k = 0; k < 36; ++k) out[k] = 0.0;
    return;
  }
  const int si = d.solIdx[j - d.mcon], off = si & 63;
  const double* Zt = Z + (size_t)diagTile[si >> 6] * 4096;
  const double v0 = pa[6 * (size_t)j], v1 = pa[6 * (size_t)j + 1], v2 = pa[6 * (size_t)j + 2];
  const double wq = sqrt(1.0 - (v0 * v0 + v1 * v1 + v2 * v2));
  const double v[3] = {v0, v1, v2};
  const double vx[9] = {0.0, -v2, v1, v2, 0.0, -v0, -v1, v0, 0.0};
  double Tm[36];
  for (int k = 0; k < 36; ++k) Tm[k] = 0.0;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Tm[6 * r + c] = 2.0 * ((r == c ? wq : 0.0) + vx[3 * r + c] + v[r] * v[c] / wq);
    Tm[6 * (r + 3) + r + 3] = 1.0;
  }
  double M[36];  // T Z
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double s = 0;
      for (int p = 0; p < 6; ++p) s += Tm[6 * r + p] * Zt[(size_t)(off + c) * 64 + off + p];
      M[6 * r + c] = s;
    }
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double s = 0;
      for (int p = 0; p < 6; ++p) s += M[6 * r + p] * Tm[6 * c + p];
      out[6 * r + c] = var * s;
    }
}

// One pass over the Schur pair entries, one warp per work item: T_i += W_a^T Z_ab W_b (+ its transpose when
// a != b), Z_ab read through the item's destination in the tile layout (ba_schur_pairs_st writes S there).
// T: [n][6] packed symmetric (00, 01, 02, 11, 12, 22), zeroed by ba_cov_begin.
__global__ void __launch_bounds__(128)
ba_cov_pairs(BaDev d, const BaPairItem* __restrict__ items, int nItems, const int4* __restrict__ entries,
             const double* __restrict__ Z, double* __restrict__ T) {
  __shared__ double s_z[4][36];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * 4 + w;
  if (item >= nItems) return;
  const BaPairItem it = items[item];
  for (int k = lane; k < 36; k += 32) {
    const int r = k / 6, c = k - 6 * r;
    s_z[w][k] = Z[(size_t)it.dst + (size_t)(it.cOff + (it.trans ? c : r)) * 64 + it.rOff + (it.trans ? r : c)];
  }
  __syncwarp();
  const double* Zb = s_z[w];
  for (int e = it.begin + lane; e < it.end; e += 32) {
    const int4 en = entries[e];
    const double* Wa = d.W + 18 * (size_t)en.x;
    const double* Wb = d.W + 18 * (size_t)en.y;
    double M[18];  // Z_ab W_b (6x3)
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 3; ++c) {
        double s = 0;
        for (int q = 0; q < 6; ++q) s += Zb[6 * r + q] * Wb[3 * q + c];
        M[3 * r + c] = s;
      }
    double X[9];  // W_a^T M
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double s = 0;
        for (int q = 0; q < 6; ++q) s += Wa[3 * q + r] * M[3 * q + c];
        X[3 * r + c] = s;
      }
    const double f = (en.x != en.y) ? 1.0 : 0.5;  // X + X^T, or the symmetric part of a diagonal term
    double* Ti = T + 6 * (size_t)en.z;
    atomicAdd(Ti + 0, 2.0 * f * X[0]);
    atomicAdd(Ti + 1, f * (X[1] + X[3]));
    atomicAdd(Ti + 2, f * (X[2] + X[6]));
    atomicAdd(Ti + 3, 2.0 * f * X[4]);
    atomicAdd(Ti + 4, f * (X[5] + X[7]));
    atomicAdd(Ti + 5, 2.0 * f * X[8]);
  }
}

// Point blocks: ptCov[i] = var (V_i^-1 + V_i^-1 T_i V_i^-1) (row-major 3x3); zeros for the fixed points, NaN for
// the points left out of H.
__global__ void __launch_bounds__(256)
ba_cov_points(int n, int ncon, const double* __restrict__ Vinv, const double* __restrict__ T,
              const unsigned char* __restrict__ unc, double var, double* __restrict__ ptCov) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double* out = ptCov + 9 * (size_t)i;
  if (i < ncon || unc[i]) {
    const double f = i < ncon ? 0.0 : __longlong_as_double(0x7ff8000000000000LL);
    for (int k = 0; k < 9; ++k) out[k] = f;
    return;
  }
  const int sym[9] = {0, 1, 2, 1, 3, 4, 2, 4, 5};
  double Iv[9], Tm[9], A[9];
  for (int k = 0; k < 9; ++k) {
    Iv[k] = Vinv[6 * (size_t)i + sym[k]];
    Tm[k] = T[6 * (size_t)i + sym[k]];
  }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) A[3 * r + c] = Iv[3 * r] * Tm[c] + Iv[3 * r + 1] * Tm[3 + c] + Iv[3 * r + 2] * Tm[6 + c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      out[3 * r + c] = var * (Iv[3 * r + c] + A[3 * r] * Iv[c] + A[3 * r + 1] * Iv[3 + c] + A[3 * r + 2] * Iv[6 + c]);
}

// The stage's scalars: sigma^2-hat, dof, the minimum relative pivot over the nb blocks, singularity, time, the
// numbers of camera and point priors (each counts as six, resp. three, measurements in dof; their |L r|^2 is in
// sc[SC_COST])
__global__ void ba_cov_end(double* __restrict__ sc, const double* __restrict__ piv, int nb, int mf, double var,
                           int nPrior, int nPtPrior) {
  if (threadIdx.x != 0) return;
  double mp = __longlong_as_double(0x7ff0000000000000LL);  // +inf: no free camera, no pivot
  for (int k = 0; k < nb; ++k) mp = fmin(mp, piv[k]);
  const double dof = 2.0 * sc[COV_NOBS] - 6.0 * mf - 3.0 * sc[COV_NPTS] + 6.0 * nPrior + 3.0 * nPtPrior;
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  const unsigned long long t0 = *reinterpret_cast<const unsigned long long*>(sc + COV_T0);
  sc[COV_SING] = (sc[SC_FAIL] != 0.0 || !(mp >= BA_COV_MIN_PIVOT)) ? 1.0 : 0.0;
  double* out = sc + COV_OUT;
  out[0] = var;
  out[1] = dof > 0 ? sc[SC_COST] / dof : __longlong_as_double(0x7ff8000000000000LL);
  out[2] = dof;
  out[3] = sc[COV_NUNC];
  out[4] = 1e-6 * (double)(t - t0);
  out[5] = mp;
  out[6] = nPrior;
  out[7] = nPtPrior;
}

}  // namespace coslam
