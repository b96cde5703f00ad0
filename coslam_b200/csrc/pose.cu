// pose.cu -- per-frame 6-DoF pose refinement (Tukey-IRLS around Levenberg-Marquardt) on the GPU.
// Replaces intraCamEstimate / intraCamWeightedLMProc / intraCamWeightedLMStep
// (slam/SL_IntraCamPose.cpp:626-709 / 475-549 / 259-303).  One 128-thread CTA per camera runs ALL
// IRLS rounds and LM iterations inside one kernel launch (no host round trips): points are spread
// over the threads, the 6x6 normal equations are reduced with warp shuffles + shared memory, and
// every thread redundantly solves the 6x6 system so that control flow stays uniform.
//
// The Jacobian is the reference's forward difference (eps = 1e-8, :43-117) evaluated with non-fused
// fp64 operations (this file is compiled with -fmad=false) so that the differences see the same
// roundings as the oracle.
//
// An armed pose solver handle (cosl_pose_solver_set_covariance) follows the solve with pose_cov_kernel, the
// covariance of each refined pose with the analytic Jacobian (an extension, not reference parity).
// cosl_pose_solver_submit_prior anchors cameras with Gaussian pose priors (also an extension): the PRIOR
// instantiations of both kernels add each prior's whitened residual to the costs, the LM step and the stage's H.
// A triangulation handle (cosl_tri_solver, also an extension) runs tri_kernel, which shares the map-point update's
// projection, Jacobians and 3x3 Cholesky.
// A registration handle (cosl_assoc_solver, also an extension) bins each entry's features into a uniform grid and
// runs one search thread per (map point, camera entry) pair on the same projection and Jacobians.
// Each handle stages a submit's inputs in one pinned buffer of 256-byte-aligned SlabLayout sections, placed by one
// layout function per handle (pose_layout, tri_layout, assoc_layout) whose offsets index the host buffer and its
// device copy alike and, at the handle's maxima, size both.
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <mutex>
#include <new>

#include <math_constants.h>

#include "common.cuh"

using namespace coslam;

namespace {

constexpr int POSE_THREADS = 128;

struct PoseCam {
  double K[9], R0[9], t0[3];
  int npts;
  int hasPrev;
  long long off;  // offset of this camera's points in the packed arrays
};

struct PoseOut {
  double R[9], t[3];
  double lambda0, lambda, err0, err, errRW;
  int retTypeLM, npts, nIterLM, nIterRW, ok;
};

struct PoseCfg {
  int maxIterLM, maxIterRW;
  double epsErr, epsParam, epsRW, lambda0, tau;
};

__device__ __forceinline__ void so3_exp(const double w[3], double R[9]) {
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (th == 0) {
    R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    return;
  }
  const double a0 = w[0] / th, a1 = w[1] / th, a2 = w[2] / th;
  double s, c;
  sincos(th, &s, &c);
  const double c1 = 1 - c;
  const double a00 = a0 * a0, a01 = a0 * a1, a02 = a0 * a2, a11 = a1 * a1, a12 = a1 * a2,
               a22 = a2 * a2;
  R[0] = -c1 * a11 - c1 * a22 + 1;
  R[1] = c1 * a01 - s * a2;
  R[2] = s * a1 + c1 * a02;
  R[3] = s * a2 + c1 * a01;
  R[4] = -c1 * a00 - c1 * a22 + 1;
  R[5] = c1 * a12 - s * a0;
  R[6] = c1 * a02 - s * a1;
  R[7] = s * a0 + c1 * a12;
  R[8] = -c1 * a00 - c1 * a11 + 1;
}

__device__ __forceinline__ void project(const double K[9], const double R[9], const double t[3],
                                        const double M[3], double m[2]) {
  const double c0 = R[0] * M[0] + R[1] * M[1] + R[2] * M[2] + t[0];
  const double c1 = R[3] * M[0] + R[4] * M[1] + R[5] * M[2] + t[1];
  const double c2 = R[6] * M[0] + R[7] * M[1] + R[8] * M[2] + t[2];
  const double u = K[0] * c0 + K[1] * c1 + K[2] * c2;
  const double v = K[3] * c0 + K[4] * c1 + K[5] * c2;
  const double w = K[6] * c0 + K[7] * c1 + K[8] * c2;
  m[0] = u / w;
  m[1] = v / w;
}

__device__ __forceinline__ void mat33(const double A[9], const double B[9], double C[9]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

__device__ __forceinline__ double tukey(double e, double tau) {
  if (e >= tau) return 0;
  e /= tau;
  e = 1 - e * e;
  return e * e;
}

// block-wide sum of NV doubles; result broadcast to every thread (bitwise identical everywhere)
template <int NV>
__device__ __forceinline__ void block_sum(double* v, double* s_red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double x = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) s_red[wid * NV + k] = x;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double x = s_red[k];
#pragma unroll
    for (int w = 1; w < POSE_THREADS / 32; ++w) x += s_red[w * NV + k];
    v[k] = x;
  }
  __syncthreads();
}

// inverse by Gauss-Jordan elimination with partial pivoting (same algorithm as the oracle)
__device__ bool inv6(const double A[36], double Ainv[36]) {
  double a[6][12];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      a[i][j] = A[6 * i + j];
      a[i][6 + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < 6; ++c) {
    int p = c;
    double best = fabs(a[c][c]);
    for (int r = c + 1; r < 6; ++r)
      if (fabs(a[r][c]) > best) {
        best = fabs(a[r][c]);
        p = r;
      }
    if (best == 0.0) return false;
    if (p != c)
      for (int j = 0; j < 12; ++j) {
        const double tmp = a[c][j];
        a[c][j] = a[p][j];
        a[p][j] = tmp;
      }
    const double d = 1.0 / a[c][c];
    for (int j = 0; j < 12; ++j) a[c][j] *= d;
    for (int r = 0; r < 6; ++r) {
      if (r == c) continue;
      const double f = a[r][c];
      for (int j = 0; j < 12; ++j) a[r][j] -= f * a[c][j];
    }
  }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) Ainv[6 * i + j] = a[i][6 + j];
  return true;
}

// r <- L r with the upper-triangular whitening factor L = {l00, l01, l11} of a point's measurement covariance
// (cosl_pose_solver_submit_cov).  With L = {1, -0, 1} and no fused multiply-add this is the identity, bit for bit.
__device__ __forceinline__ void whiten(const double* L, double& r0, double& r1) {
  r0 = L[0] * r0 + L[1] * r1;
  r1 = L[2] * r1;
}

// Gaussian pose priors (cosl_pose_solver_submit_prior, DESIGN.md 5.3).  Camera c has a prior when has[c] != 0; its
// record is rec[c] = [L (21: the upper-triangular 6x6 factor with L^T L = P^-1, packed by rows) | R_p (9, row-major) |
// t_p (3)], staged by the host.  Every instantiation of both pose kernels takes the records as its last parameter;
// only the PRIOR ones read them.
struct PosePriorDev {
  const double* rec;  // [C][POSE_PRIOR_REC]
  const int* has;     // [C]
};
constexpr int POSE_PRIOR_REC = 33;

// This CTA's prior record, or nullptr for a camera without a prior (uniform over the CTA)
__device__ __forceinline__ const double* prior_record(const PosePriorDev& pr) {
  return pr.has[blockIdx.x] ? pr.rec + POSE_PRIOR_REC * (size_t)blockIdx.x : nullptr;
}

// Whitened prior residual rw = L r at (R, t), r = [Log(R_p^T R); t - t_p], and with WANT_J, Jw = L dr/d(dw, dt)
// (6x6 row-major) for the solver's update R' = R exp([dw]x), t' = t + dt.  Log(M) by atan2 with the axis from the
// skew part below 120 degrees and from the symmetric part above (exact to roundoff up to pi).  dr_w / ddw =
// Jr^-1(r_w), the inverse right Jacobian of SO(3), Jr^-1(w) = I + [w]x / 2 + (1 - (th / 2) cot(th / 2)) / th^2 [w]x^2,
// and dr_t / ddt = I.  q is the record, read from global memory where it is used.
template <bool WANT_J>
__device__ __forceinline__ void prior_eval(const double* __restrict__ q, const double R[9], const double t[3],
                                           double rw[6], double Jw[36]) {
  double M[9];  // R_p^T R
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) M[3 * a + b] = q[21 + a] * R[b] + q[24 + a] * R[3 + b] + q[27 + a] * R[6 + b];
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
  for (int a = 0; a < 3; ++a) r[3 + a] = t[a] - q[30 + a];
  // rw = L r, L packed by rows: row a holds L[a][a .. 5] from offset 6a - a(a-1)/2
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const int off = 6 * a - a * (a - 1) / 2;
    double v = 0.0;
#pragma unroll
    for (int b = a; b < 6; ++b) v += q[off + b - a] * r[b];
    rw[a] = v;
  }
  if (!WANT_J) return;
  // cot(th / 2) = sin th / (1 - cos th) = sn / (|(sn, cs)| - cs): no trigonometric call, exact up to pi
  const double c2 = th < 1e-2 ? 1.0 / 12.0 + th * th * (1.0 / 720.0 + th * th / 30240.0)
                              : (1.0 - 0.5 * th * sn / (sqrt(sn * sn + cs * cs) - cs)) / (th * th);
  const double wx[9] = {0.0, -r[2], r[1], r[2], 0.0, -r[0], -r[1], r[0], 0.0};
  double Ji[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const double w2 = wx[3 * a] * wx[b] + wx[3 * a + 1] * wx[3 + b] + wx[3 * a + 2] * wx[6 + b];
      Ji[3 * a + b] = (a == b ? 1.0 : 0.0) + 0.5 * wx[3 * a + b] + c2 * w2;
    }
  // Jw = L diag(Ji, I)
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const int off = 6 * a - a * (a - 1) / 2;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      double v = 0.0;
#pragma unroll
      for (int c = a; c < 3; ++c) v += q[off + c - a] * Ji[3 * c + b];
      Jw[6 * a + b] = v;
    }
#pragma unroll
    for (int b = 3; b < 6; ++b) Jw[6 * a + b] = b >= a ? q[off + b - a] : 0.0;
  }
}

// |L r|^2 of the prior record q at (R, t)
__device__ __forceinline__ double prior_cost(const double* __restrict__ q, const double R[9], const double t[3]) {
  double rw[6];
  prior_eval<false>(q, R, t, rw, nullptr);
  return rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2] + rw[3] * rw[3] + rw[4] * rw[4] + rw[5] * rw[5];
}

// acc (21 upper-triangle entries of a 6x6 system, then its 6 right-hand-side entries) += the prior's rows at (R, t):
// (L J)^T (L J) and -(L J)^T L r
__device__ __forceinline__ void prior_normal(const double* __restrict__ q, const double R[9], const double t[3],
                                             double acc[27]) {
  double rw[6], Jw[36];
  prior_eval<true>(q, R, t, rw, Jw);
  int k = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int b = a; b < 6; ++b) {
      double v = 0.0;
#pragma unroll
      for (int c = 0; c < 6; ++c) v += Jw[6 * c + a] * Jw[6 * c + b];
      acc[k++] += v;
    }
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    double v = 0.0;
#pragma unroll
    for (int c = 0; c < 6; ++c) v += Jw[6 * c + a] * rw[c];
    acc[21 + a] -= v;
  }
}

// intraCamWeightedCost (:439-456); OBSCOV whitens each residual by Ls (3 per point) before the weight; PRIOR adds
// |L r|^2 of the prior record Pq when the camera has one (Pq != nullptr, uniform over the CTA)
template <bool OBSCOV, bool PRIOR>
__device__ double weighted_cost(const double K[9], const double R[9], const double t[3], int n,
                                const double* Ws, const double* Ms, const double* ms, const double* Ls,
                                double* s_red, const double* Pq) {
  double err[1] = {0};
  for (int i = threadIdx.x; i < n; i += POSE_THREADS) {
    double rm[2];
    project(K, R, t, Ms + 3 * i, rm);
    double dx = ms[2 * i] - rm[0], dy = ms[2 * i + 1] - rm[1];
    if (OBSCOV) whiten(Ls + 3 * i, dx, dy);
    err[0] += (dx * dx + dy * dy) * Ws[i];
  }
  block_sum<1>(err, s_red);
  if (PRIOR && Pq) err[0] += prior_cost(Pq, R, t);
  return err[0];
}

// intraCamWeightedLMStep (:259-303); OBSCOV whitens the residual and both Jacobian rows by Ls before the weight;
// PRIOR adds the rows of the prior record Pq (when not nullptr, uniform over the CTA) before lambda, unweighted
template <bool OBSCOV, bool PRIOR>
__device__ void weighted_step(const double K[9], const double R[9], const double t[3], int n,
                              const double* Ws, const double* Ms, const double* ms, const double* Ls,
                              double param[6], double lambda, const double dRk[3][9],
                              double* s_red, const double* Pq) {
  const double eps = 1e-8;
  double acc[27];  // 21 upper-triangle entries of J^T J + 6 of J^T r
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0;
  for (int i = threadIdx.x; i < n; i += POSE_THREADS) {
    const double* M = Ms + 3 * i;
    double rm0[2], rm[2], J[12];
    project(K, R, t, M, rm0);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double R1[9];
      mat33(R, dRk[k], R1);
      project(K, R1, t, M, rm);
      J[k] = (rm[0] - rm0[0]) / eps;
      J[6 + k] = (rm[1] - rm0[1]) / eps;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double t1[3] = {t[0], t[1], t[2]};
      t1[k] = t[k] + eps;
      project(K, R, t1, M, rm);
      J[3 + k] = (rm[0] - rm0[0]) / eps;
      J[9 + k] = (rm[1] - rm0[1]) / eps;
    }
    if (OBSCOV) {
#pragma unroll
      for (int k = 0; k < 6; ++k) whiten(Ls + 3 * i, J[k], J[6 + k]);
    }
    const double w = Ws[i];
#pragma unroll
    for (int k = 0; k < 12; ++k) J[k] = w * J[k];
    double r0 = -rm0[0] + ms[2 * i], r1 = -rm0[1] + ms[2 * i + 1];
    if (OBSCOV) whiten(Ls + 3 * i, r0, r1);
    r0 = r0 * w;
    r1 = r1 * w;
    int q = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int b = a; b < 6; ++b) acc[q++] += J[a] * J[b] + J[6 + a] * J[6 + b];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += J[a] * r0 + J[6 + a] * r1;
  }
  block_sum<27>(acc, s_red);
  if (PRIOR && Pq) prior_normal(Pq, R, t, acc);
  double sA[36], inv[36];
  int q = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) {
      sA[6 * a + b] = acc[q];
      sA[6 * b + a] = acc[q];
      ++q;
    }
  for (int a = 0; a < 6; ++a) sA[7 * a] += lambda;
  if (!inv6(sA, inv)) {
    for (int a = 0; a < 6; ++a) param[a] = 0;
    return;
  }
  for (int a = 0; a < 6; ++a) {
    double s = 0;
    for (int b = 0; b < 6; ++b) s += inv[6 * a + b] * acc[21 + b];
    param[a] = s;
  }
}

// OBSCOV: every residual and Jacobian row is whitened by the factors LAll (3 per point, packed as the points;
// cosl_pose_solver_submit_cov).  The false instantiation never reads LAll and is the unweighted solve.
// PRIOR (cosl_pose_solver_submit_prior): a camera with a prior in `prior` adds its |L r|^2 to every cost and its rows
// to every LM step, a camera without one computes what the launch without PRIOR computes.  The false instantiation
// never reads `prior`.
template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(POSE_THREADS)
pose_intracam_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll,
                     const double* __restrict__ msAll, const double* __restrict__ prevAll,
                     double* __restrict__ WsAll, PoseCfg cfg, PoseOut* __restrict__ outs,
                     const double* __restrict__ LAll, PosePriorDev prior) {
  __shared__ double s_red[(POSE_THREADS / 32) * 27];
  const double* Pq = PRIOR ? prior_record(prior) : nullptr;
  const PoseCam cam = cams[blockIdx.x];
  const int n = cam.npts;
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
  const double* Ls = OBSCOV ? LAll + 3 * cam.off : nullptr;
  double* Ws = WsAll + cam.off;
  const double tau = cfg.tau;
  double K[9], R[9], t[3], R_opt[9], t_opt[3], R_tmp[9], t_tmp[3], Rlm[9], tlm[3];
  for (int k = 0; k < 9; ++k) {
    K[k] = cam.K[k];
    R[k] = cam.R0[k];
    R_opt[k] = cam.R0[k];
  }
  for (int k = 0; k < 3; ++k) {
    t[k] = cam.t0[k];
    t_opt[k] = cam.t0[k];
  }
  // rotation perturbations exp(eps e_k) of the numeric Jacobian (:56-84)
  double dRk[3][9];
  for (int k = 0; k < 3; ++k) {
    double w[3] = {0, 0, 0};
    w[k] = 1e-8;
    so3_exp(w, dRk[k]);
  }
  for (int i = threadIdx.x; i < n; i += POSE_THREADS)
    Ws[i] = cam.hasPrev ? tukey(fabs(prevAll[cam.off + i]), tau) : 1.0;
  __syncthreads();

  double lambda0 = cfg.lambda0, lambda = cfg.lambda0, err0 = 0, errLM = 0, errRW = -1;
  int retType = 1, nIterLM = 0, k = 0;
  bool ret = true;
  for (; k < cfg.maxIterRW; ++k) {
    // ---- intraCamWeightedLMProc (:475-549) from (R, t) ----
    double param[6];
    lambda = lambda0;
    err0 = weighted_cost<OBSCOV, PRIOR>(K, R, t, n, Ws, Ms, ms, Ls, s_red, Pq);
    errLM = err0;
    for (int q = 0; q < 9; ++q) {
      Rlm[q] = R[q];
      R_tmp[q] = R[q];
    }
    for (int q = 0; q < 3; ++q) {
      tlm[q] = t[q];
      t_tmp[q] = t[q];
    }
    retType = 1;
    int i = 0;
    double err = err0;
    for (; i < cfg.maxIterLM; ++i) {
      weighted_step<OBSCOV, PRIOR>(K, Rlm, tlm, n, Ws, Ms, ms, Ls, param, lambda, dRk, s_red, Pq);
      {  // intraCamUpdatePose (:367-380)
        double dR[9];
        so3_exp(param, dR);
        mat33(Rlm, dR, R_opt);
        t_opt[0] = tlm[0] + param[3];
        t_opt[1] = tlm[1] + param[4];
        t_opt[2] = tlm[2] + param[5];
      }
      double p2 = 0;
      for (int q = 0; q < 6; ++q) p2 += param[q] * param[q];
      if (p2 < cfg.epsParam) {
        for (int q = 0; q < 9; ++q) Rlm[q] = R_opt[q];
        for (int q = 0; q < 3; ++q) tlm[q] = t_opt[q];
        retType = 0;
        break;
      }
      err = weighted_cost<OBSCOV, PRIOR>(K, R_opt, t_opt, n, Ws, Ms, ms, Ls, s_red, Pq);
      if (fabs(err - errLM) < cfg.epsErr) {
        retType = 0;
        break;
      }
      if (err <= errLM) {
        for (int q = 0; q < 9; ++q) {
          Rlm[q] = R_opt[q];
          R_tmp[q] = R_opt[q];
        }
        for (int q = 0; q < 3; ++q) {
          tlm[q] = t_opt[q];
          t_tmp[q] = t_opt[q];
        }
        errLM = err;
        lambda /= 10;
      } else {
        lambda *= 10;
        if (lambda > 1e+18) {
          retType = -1;
          break;
        }
      }
    }
    if (retType == -1) {
      for (int q = 0; q < 9; ++q) R_opt[q] = R_tmp[q];
      for (int q = 0; q < 3; ++q) t_opt[q] = t_tmp[q];
    }
    errLM = err;
    nIterLM = i;
    if (retType < 0) {
      ret = false;
      break;
    }
    // ---- IRLS bookkeeping (:664-702) ----
    lambda0 = lambda;
    if (errRW < 0)
      errRW = errLM;
    else {
      if (fabs(errLM - errRW) < cfg.epsRW) {
        ret = true;
        break;
      }
      errRW = errLM;
    }
    for (int q = 0; q < 9; ++q) R[q] = R_opt[q];
    for (int q = 0; q < 3; ++q) t[q] = t_opt[q];
    for (int p = threadIdx.x; p < n; p += POSE_THREADS) {
      double rm[2];
      project(K, R, t, Ms + 3 * p, rm);
      const double dx = rm[0] - ms[2 * p], dy = rm[1] - ms[2 * p + 1];
      Ws[p] = tukey(sqrt(dx * dx + dy * dy), tau);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    PoseOut o;
    for (int q = 0; q < 9; ++q) o.R[q] = R_opt[q];
    for (int q = 0; q < 3; ++q) o.t[q] = t_opt[q];
    o.lambda0 = lambda0;
    o.lambda = lambda;
    o.err0 = err0;
    o.err = errLM;
    o.errRW = errRW;
    o.retTypeLM = retType;
    o.npts = n;
    o.nIterLM = nIterLM;
    o.nIterRW = k;
    o.ok = ret ? 1 : 0;
    outs[blockIdx.x] = o;
  }
}

// Per-camera layout of the covariance stage's results: cov[36] | sigma2_hat, dof, min relative pivot, valid.
constexpr int POSE_COV_STRIDE = 40;

// Covariance of the refined pose (an extension: the reference reports none).  One CTA per camera, at the
// (R_opt, t_opt) that pose_intracam_kernel wrote into outs, in the solver's own chart R' = R exp([w]x),
// t' = t + dt, order (w, dt):
//   e_i = |project(K, R_opt, t_opt, M_i) - m_i|, w_i = tukey(e_i, tau), H = sum_i w_i J_i^T J_i with the
//   analytic 2x6 Jacobian J_i of project, cov = pixel_var H^-1 by Cholesky.
// res[c] gets cov | {sigma2_hat = sum w e^2 / dof (NaN for dof <= 0), dof = 2 #(w > 0) - 6, the smallest
// relative pivot L_kk^2 / H_kk (0 when the factorisation breaks down), valid}; a break-down or a relative pivot
// below 1e-12 gives a NaN covariance and valid = 0.  errAll gets e_i of every point, in the packed order.
// OBSCOV (cosl_pose_solver_submit_cov) whitens by the factors L_i of LAll: H = sum_i w_i (L_i J_i)^T (L_i J_i) and
// sigma2_hat = sum w |L_i (project - m_i)|^2 / dof; e_i and w_i stay on the pixel distance.
// PRIOR (cosl_pose_solver_submit_prior): a camera with a prior in `prior` adds (L J_p)^T (L J_p) to H and |L r|^2 to
// sigma2_hat's numerator at (R_opt, t_opt), and 6 to dof.
// Every instantiation takes both LAll and `prior`; the false ones never read them.  LAll is not __restrict__: that
// turns its loads into constant-cache loads and changes the OBSCOV instantiation's code.
template <bool OBSCOV, bool PRIOR>
__global__ void __launch_bounds__(POSE_THREADS)
pose_cov_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll,
                const double* __restrict__ msAll, const PoseOut* __restrict__ outs, double tau, double pixel_var,
                double* __restrict__ res, double* __restrict__ errAll, const double* LAll, PosePriorDev prior) {
  __shared__ double s_red[(POSE_THREADS / 32) * 23];
  const PoseCam& cam = cams[blockIdx.x];
  const int n = cam.npts;
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
  double K[9], R[9], t[3];
  for (int k = 0; k < 9; ++k) {
    K[k] = cam.K[k];
    R[k] = outs[blockIdx.x].R[k];
  }
  for (int k = 0; k < 3; ++k) t[k] = outs[blockIdx.x].t[k];
  double acc[23];  // 21 upper-triangle entries of H, sum w e^2, #(w > 0)
#pragma unroll
  for (int k = 0; k < 23; ++k) acc[k] = 0;
  for (int i = threadIdx.x; i < n; i += POSE_THREADS) {
    const double* M = Ms + 3 * i;
    double rm[2];
    project(K, R, t, M, rm);
    const double dx = rm[0] - ms[2 * i], dy = rm[1] - ms[2 * i + 1];
    const double e = sqrt(dx * dx + dy * dy);
    errAll[cam.off + i] = e;
    const double w = tukey(e, tau);
    if (w > 0) {
      // x = K c, c = R M + t; m = x_{0,1} / x_2.  dm/dc rows a, b; dc/dt = I; dc/dw_k = R (e_k x M), so
      // dm_0/dw = M x (R^T a) and dm_1/dw = M x (R^T b)
      const double c0 = R[0] * M[0] + R[1] * M[1] + R[2] * M[2] + t[0];
      const double c1 = R[3] * M[0] + R[4] * M[1] + R[5] * M[2] + t[1];
      const double c2 = R[6] * M[0] + R[7] * M[1] + R[8] * M[2] + t[2];
      const double z = K[6] * c0 + K[7] * c1 + K[8] * c2;
      double J[12];  // rows u, v; columns w0 w1 w2 t0 t1 t2
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        J[3 + k] = (K[k] - rm[0] * K[6 + k]) / z;
        J[9 + k] = (K[3 + k] - rm[1] * K[6 + k]) / z;
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const double* a = J + 6 * r + 3;
        const double q0 = R[0] * a[0] + R[3] * a[1] + R[6] * a[2];
        const double q1 = R[1] * a[0] + R[4] * a[1] + R[7] * a[2];
        const double q2 = R[2] * a[0] + R[5] * a[1] + R[8] * a[2];
        J[6 * r + 0] = M[1] * q2 - M[2] * q1;
        J[6 * r + 1] = M[2] * q0 - M[0] * q2;
        J[6 * r + 2] = M[0] * q1 - M[1] * q0;
      }
      double ew = 0;  // |L (project - m)|, which is e bit for bit when L = I
      if (OBSCOV) {
        const double* L = LAll + 3 * (cam.off + i);
        double r0 = dx, r1 = dy;
        whiten(L, r0, r1);
        ew = sqrt(r0 * r0 + r1 * r1);
#pragma unroll
        for (int k = 0; k < 6; ++k) whiten(L, J[k], J[6 + k]);
      }
      int q = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int b = a; b < 6; ++b) acc[q++] += w * (J[a] * J[b] + J[6 + a] * J[6 + b]);
      }
      acc[21] += w * (OBSCOV ? ew * ew : e * e);
      acc[22] += 1;
    }
  }
  block_sum<23>(acc, s_red);
  if (threadIdx.x != 0) return;
  if constexpr (PRIOR) {  // discarded without PRIOR, so the other instantiations keep their code
    const double* Pq = prior_record(prior);
    if (Pq) {
      double hb[27];  // the prior's 21 entries of H; its 6 right-hand-side entries are not needed here
#pragma unroll
      for (int k = 0; k < 27; ++k) hb[k] = 0;
      prior_normal(Pq, R, t, hb);
#pragma unroll
      for (int k = 0; k < 21; ++k) acc[k] += hb[k];
      acc[21] += prior_cost(Pq, R, t);
      acc[22] += 3;  // six measurements: dof = 2 #(w > 0) - 6 + 6
    }
  }
  // Cholesky H = L L^T in packed lower storage, L(i, j) at i (i + 1) / 2 + j
  double L[21];
  double minPiv = INFINITY;
  bool valid = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const int jj = j * (j + 1) / 2;
    const double h = acc[6 * j - j * (j - 1) / 2];  // H(j, j) in the upper-triangle order of acc
    double d = h;
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[jj + k] * L[jj + k];
    if (!(d > 0)) {
      valid = false;
      minPiv = 0;
      d = 1;  // keeps the remaining arithmetic finite; the covariance is discarded
    } else {
      minPiv = fmin(minPiv, d / h);
    }
    const double ljj = sqrt(d);
    L[jj + j] = ljj;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      const int ii = i * (i + 1) / 2;
      double s = acc[6 * j - j * (j - 1) / 2 + (i - j)];  // H(j, i), i > j
#pragma unroll
      for (int k = 0; k < j; ++k) s -= L[ii + k] * L[jj + k];
      L[ii + j] = s / ljj;
    }
  }
  if (minPiv < 1e-12) valid = false;
  // X = L^-1 (lower triangular, packed as L), then cov = pixel_var X^T X
  double X[21];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    X[j * (j + 1) / 2 + j] = 1.0 / L[j * (j + 1) / 2 + j];
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      const int ii = i * (i + 1) / 2;
      double s = 0;
#pragma unroll
      for (int k = j; k < i; ++k) s += L[ii + k] * X[k * (k + 1) / 2 + j];
      X[ii + j] = -s / L[ii + i];
    }
  }
  double* r = res + POSE_COV_STRIDE * blockIdx.x;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j) {
      double s = 0;
#pragma unroll
      for (int k = j; k < 6; ++k) s += X[k * (k + 1) / 2 + i] * X[k * (k + 1) / 2 + j];
      const double v = valid ? pixel_var * s : NAN;
      r[6 * i + j] = v;
      r[6 * j + i] = v;
    }
  const double dof = 2 * acc[22] - 6;
  r[36] = dof > 0 ? acc[21] / dof : NAN;
  r[37] = dof;
  r[38] = minPiv;
  r[39] = valid ? 1.0 : 0.0;
}

// Map-point update of cosl_pose_solver_submit_mappts (DESIGN.md 5.4, an extension).  Per point, staged as
// MAPPT_IN doubles: X0[3] | P0 (6: xx xy xz yy yz zz) | m[2] | Sigma_m (3: xx xy yy); results as MAPPT_OUT doubles:
// X[3] | P (6, as P0) | d2_0, d2_1, e0 | status.
constexpr int MAPPT_THREADS = 64;
constexpr int MAPPT_IN = 14;
constexpr int MAPPT_OUT = 13;
constexpr int MAPPT_MAX_ITER = 8;

// c = R X + t, m = x_{0,1} / x_2 of x = K c (x_2 into *x2), and the rows of dm/dX = (a; b) R, a and b the rows of
// dm/dc (5.1), as ha = R^T a and hb = R^T b.  Returns c_2, the depth.
__device__ __forceinline__ double mappt_project(const double* K, const double* R, const double* t, const double X[3],
                                                double m[2], double a[3], double b[3], double ha[3], double hb[3],
                                                double* x2) {
  const double c0 = R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0];
  const double c1 = R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1];
  const double c2 = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
  const double u = K[0] * c0 + K[1] * c1 + K[2] * c2;
  const double v = K[3] * c0 + K[4] * c1 + K[5] * c2;
  const double w = K[6] * c0 + K[7] * c1 + K[8] * c2;
  m[0] = u / w;
  m[1] = v / w;
  *x2 = w;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    a[k] = (K[k] - m[0] * K[6 + k]) / w;
    b[k] = (K[3 + k] - m[1] * K[6 + k]) / w;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ha[k] = R[k] * a[0] + R[3 + k] * a[1] + R[6 + k] * a[2];
    hb[k] = R[k] * b[0] + R[3 + k] * b[1] + R[6 + k] * b[2];
  }
  return c2;
}

// Cholesky A = L L^T of a symmetric 3x3 packed as (00 01 02 11 12 22); L lower packed as (00 10 11 20 21 22).
// False on a pivot that is not positive and finite.
__device__ __forceinline__ bool mappt_chol3(const double A[6], double L[6]) {
  const double d0 = A[0];
  if (!(d0 > 0) || !isfinite(d0)) return false;
  L[0] = sqrt(d0);
  L[1] = A[1] / L[0];
  L[3] = A[2] / L[0];
  const double d1 = A[3] - L[1] * L[1];
  if (!(d1 > 0) || !isfinite(d1)) return false;
  L[2] = sqrt(d1);
  L[4] = (A[4] - L[3] * L[1]) / L[2];
  const double d2 = A[5] - L[3] * L[3] - L[4] * L[4];
  if (!(d2 > 0) || !isfinite(d2)) return false;
  L[5] = sqrt(d2);
  return true;
}

// A^-1 = L^-T L^-1 (packed as A) from the factor of mappt_chol3
__device__ __forceinline__ void mappt_chol3_inv(const double L[6], double Ai[6]) {
  const double i00 = 1.0 / L[0], i11 = 1.0 / L[2], i22 = 1.0 / L[5];
  const double i10 = -L[1] * i00 * i11;
  const double i21 = -L[4] * i11 * i22;
  const double i20 = -(L[3] * i00 + L[4] * i10) * i22;
  Ai[0] = i00 * i00 + i10 * i10 + i20 * i20;
  Ai[1] = i10 * i11 + i20 * i21;
  Ai[2] = i20 * i22;
  Ai[3] = i11 * i11 + i21 * i21;
  Ai[4] = i21 * i22;
  Ai[5] = i22 * i22;
}

// r^T S^-1 r of a symmetric 2x2 S = (s00 s01 s11); false unless S is positive definite
__device__ __forceinline__ bool mappt_quad2(const double S[3], const double r[2], double* q) {
  const double det = S[0] * S[2] - S[1] * S[1];
  if (!(S[0] > 0) || !(det > 0)) return false;
  *q = (S[2] * r[0] * r[0] - 2.0 * S[1] * r[0] * r[1] + S[0] * r[1] * r[1]) / det;
  return true;
}

// f(X + s) - f(X) of the update's objective f(X) = (X - X0)^T P0^-1 (X - X0) + (m - pi(X))^T Rf^-1 (m - pi(X)), from
// differences: s^T P0^-1 (2 (X - X0) + s) - dpi^T Rf^-1 (2 nu - dpi), nu = m - pi(X), pm = pi(X) and
// dpi = pi(X + s) - pi(X) = (dx_{0,1} - pm dx_2) / (x_2 + dx_2) with dx = K R s.  Near the minimum the two objectives
// agree to their roundoff (m - pi cancels about 1e-13 px), and their difference would decide a step by noise.
__device__ __forceinline__ double mappt_descent(const double* K, const double* R, const double L0[6], const double Rf[3],
                                               const double X0[3], const double X[3], double w, const double pm[2],
                                               const double nu[2], const double s[3]) {
  const double dc0 = R[0] * s[0] + R[1] * s[1] + R[2] * s[2];
  const double dc1 = R[3] * s[0] + R[4] * s[1] + R[5] * s[2];
  const double dc2 = R[6] * s[0] + R[7] * s[1] + R[8] * s[2];
  const double dx0 = K[0] * dc0 + K[1] * dc1 + K[2] * dc2;
  const double dx1 = K[3] * dc0 + K[4] * dc1 + K[5] * dc2;
  const double dx2 = K[6] * dc0 + K[7] * dc1 + K[8] * dc2;
  const double wn = w + dx2;
  const double dp0 = (dx0 - pm[0] * dx2) / wn, dp1 = (dx1 - pm[1] * dx2) / wn;
  const double q0 = 2.0 * nu[0] - dp0, q1 = 2.0 * nu[1] - dp1;
  const double det = Rf[0] * Rf[2] - Rf[1] * Rf[1];
  const double meas = (Rf[2] * dp0 * q0 - Rf[1] * (dp0 * q1 + dp1 * q0) + Rf[0] * dp1 * q1) / det;
  // s^T P0^-1 (2 d + s) = (L0^-1 s) . (L0^-1 (2 d + s)), d = X - X0
  const double u0 = s[0] / L0[0];
  const double u1 = (s[1] - L0[1] * u0) / L0[2];
  const double u2 = (s[2] - L0[3] * u0 - L0[4] * u1) / L0[5];
  const double e0 = 2.0 * (X[0] - X0[0]) + s[0], e1 = 2.0 * (X[1] - X0[1]) + s[1], e2 = 2.0 * (X[2] - X0[2]) + s[2];
  const double v0 = e0 / L0[0];
  const double v1 = (e1 - L0[1] * v0) / L0[2];
  const double v2 = (e2 - L0[3] * v0 - L0[4] * v1) / L0[5];
  return u0 * v0 + u1 * v1 + u2 * v2 - meas;
}

// S = H P H^T + Rf for H = (ha; hb) (2x3) and P packed as mappt_chol3's A; U = P H^T (3x2, row-major)
__device__ __forceinline__ void mappt_innov(const double ha[3], const double hb[3], const double P[6],
                                            const double Rf[3], double U[6], double S[3]) {
  const double F[9] = {P[0], P[1], P[2], P[1], P[3], P[4], P[2], P[4], P[5]};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    U[2 * i] = F[3 * i] * ha[0] + F[3 * i + 1] * ha[1] + F[3 * i + 2] * ha[2];
    U[2 * i + 1] = F[3 * i] * hb[0] + F[3 * i + 1] * hb[1] + F[3 * i + 2] * hb[2];
  }
  S[0] = ha[0] * U[0] + ha[1] * U[2] + ha[2] * U[4] + Rf[0];
  S[1] = ha[0] * U[1] + ha[1] * U[3] + ha[2] * U[5] + Rf[1];
  S[2] = hb[0] * U[1] + hb[1] * U[3] + hb[2] * U[5] + Rf[2];
}

// One thread per map point; each CTA serves the points [first, end) of one camera, blk[blockIdx.x] = (camera,
// first, end, -), staged by the host.  The camera's K, its refined (R, t) from outs and its stage covariance P_c
// from res (pose_cov_kernel's, in the chart R' = R exp([w]x), t' = t + dt) go to shared memory.  Per point:
//   R_eff = Sigma_m + H_c(X0) P_c H_c(X0)^T, H_c the analytic 2x6 Jacobian of 5.1, H_X = (a; b) R;
//   gate: nu0 = m - pi(X0), S0 = H_X P0 H_X^T + R_eff, d2_0 = nu0^T S0^-1 nu0, update when d2_0 < gate;
//   update: at most MAPPT_MAX_ITER Gauss-Newton steps in Kalman form on (X - X0)^T P0^-1 (X - X0) +
//   (m - pi(X))^T R_eff^-1 (m - pi(X)), X' = X0 + P0 H^T (H P0 H^T + R_eff)^-1 (m - pi(X) + H (X - X0)) at X, taken
//   only when it lowers that objective (mappt_descent < 0) and keeps the depth > 0, stopped once
//   |X' - X| <= 1e-12 max(1, |X'|);
//   P+ = (P0^-1 + H^T R_eff^-1 H)^-1 at X+ by Cholesky; d2_1 = nu1^T (H P+ H^T + R_eff)^-1 nu1 at X+.
// status 0 updated, 1 gated out, 2 not updatable (depth <= 0, a non-finite value, S0 not positive definite), 3 the
// camera's pose covariance is invalid; with status != 0, X0 and P0 come back as given and d2_1 (and d2_0 for 2 and
// 3) is NaN.  e0 = |nu0| is reported as computed whatever the status.
__global__ void __launch_bounds__(MAPPT_THREADS)
pose_mappt_kernel(const int4* __restrict__ blk, const double* __restrict__ in, const PoseCam* __restrict__ cams,
                  const PoseOut* __restrict__ outs, const double* __restrict__ res, double gate,
                  double* __restrict__ out) {
  __shared__ double s_K[9], s_R[9], s_t[3], s_P[36];
  __shared__ int s_valid;
  const int4 b = blk[blockIdx.x];
  const int c = b.x;
  if (threadIdx.x < 9) {
    s_K[threadIdx.x] = cams[c].K[threadIdx.x];
    s_R[threadIdx.x] = outs[c].R[threadIdx.x];
  }
  if (threadIdx.x < 3) s_t[threadIdx.x] = outs[c].t[threadIdx.x];
  if (threadIdx.x < 36) s_P[threadIdx.x] = res[POSE_COV_STRIDE * c + threadIdx.x];
  if (threadIdx.x == 0) s_valid = res[POSE_COV_STRIDE * c + 39] == 1.0;
  __syncthreads();
  const int j = b.y + threadIdx.x;
  if (j >= b.z) return;
  const double* q = in + (size_t)MAPPT_IN * j;
  double* o = out + (size_t)MAPPT_OUT * j;
  const double X0[3] = {q[0], q[1], q[2]};
  double P0[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) P0[k] = q[3 + k];
  const double mo[2] = {q[9], q[10]};
  double pm[2], a[3], bb[3], ha[3], hb[3], w;
  const double z0 = mappt_project(s_K, s_R, s_t, X0, pm, a, bb, ha, hb, &w);
  double nu[2] = {mo[0] - pm[0], mo[1] - pm[1]};
  const double e0 = sqrt(nu[0] * nu[0] + nu[1] * nu[1]);
  int status = 2;
  double d0 = NAN, d1 = NAN, X[3] = {X0[0], X0[1], X0[2]}, P[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) P[k] = P0[k];
  if (!s_valid) {
    status = 3;
  } else if (z0 > 0 && isfinite(pm[0]) && isfinite(pm[1])) {
    // R_eff = Sigma_m + H_c P_c H_c^T; H_c rows (X0 x ha, a) and (X0 x hb, b)
    double Hc[12];
    Hc[0] = X0[1] * ha[2] - X0[2] * ha[1];
    Hc[1] = X0[2] * ha[0] - X0[0] * ha[2];
    Hc[2] = X0[0] * ha[1] - X0[1] * ha[0];
    Hc[6] = X0[1] * hb[2] - X0[2] * hb[1];
    Hc[7] = X0[2] * hb[0] - X0[0] * hb[2];
    Hc[8] = X0[0] * hb[1] - X0[1] * hb[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      Hc[3 + k] = a[k];
      Hc[9 + k] = bb[k];
    }
    double Rf[3] = {q[11], q[12], q[13]};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      double t0 = 0, t1 = 0;
#pragma unroll
      for (int l = 0; l < 6; ++l) {
        t0 += Hc[l] * s_P[6 * l + k];
        t1 += Hc[6 + l] * s_P[6 * l + k];
      }
      Rf[0] += t0 * Hc[k];
      Rf[1] += t0 * Hc[6 + k];
      Rf[2] += t1 * Hc[6 + k];
    }
    double U[6], S[3], L0[6], f0;  // f0: R_eff must be positive definite too
    mappt_innov(ha, hb, P0, Rf, U, S);
    if (mappt_quad2(S, nu, &d0) && isfinite(d0) && mappt_quad2(Rf, nu, &f0) && mappt_chol3(P0, L0)) {
      status = d0 < gate ? 0 : 1;
    } else {
      d0 = NAN;
    }
    if (status == 0) {
      for (int it = 0; it < MAPPT_MAX_ITER; ++it) {
        // Gauss-Newton step from X (U, S, nu, ha, hb at X)
        const double y0 = nu[0] + ha[0] * (X[0] - X0[0]) + ha[1] * (X[1] - X0[1]) + ha[2] * (X[2] - X0[2]);
        const double y1 = nu[1] + hb[0] * (X[0] - X0[0]) + hb[1] * (X[1] - X0[1]) + hb[2] * (X[2] - X0[2]);
        const double det = S[0] * S[2] - S[1] * S[1];
        const double g0 = (S[2] * y0 - S[1] * y1) / det, g1 = (S[0] * y1 - S[1] * y0) / det;
        double Xn[3], pn[2], an[3], bn[3], han[3], hbn[3], wn;
#pragma unroll
        for (int k = 0; k < 3; ++k) Xn[k] = X0[k] + (U[2 * k] * g0 + U[2 * k + 1] * g1);
        const double zn = mappt_project(s_K, s_R, s_t, Xn, pn, an, bn, han, hbn, &wn);
        if (!(zn > 0)) break;
        const double nun[2] = {mo[0] - pn[0], mo[1] - pn[1]};
        const double st[3] = {Xn[0] - X[0], Xn[1] - X[1], Xn[2] - X[2]};
        if (!(mappt_descent(s_K, s_R, L0, Rf, X0, X, w, pm, nu, st) < 0)) break;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          X[k] = Xn[k];
          ha[k] = han[k];
          hb[k] = hbn[k];
        }
        nu[0] = nun[0];
        nu[1] = nun[1];
        pm[0] = pn[0];
        pm[1] = pn[1];
        w = wn;
        const double xn = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
        if (sqrt(st[0] * st[0] + st[1] * st[1] + st[2] * st[2]) <= 1e-12 * fmax(1.0, xn)) break;
        mappt_innov(ha, hb, P0, Rf, U, S);
      }
      // P+ = (P0^-1 + H^T R_eff^-1 H)^-1 at X+
      double Pi[6], Lp[6];
      mappt_chol3_inv(L0, Pi);
      const double det = Rf[0] * Rf[2] - Rf[1] * Rf[1];
      const double w00 = Rf[2] / det, w01 = -Rf[1] / det, w11 = Rf[0] / det;
      int k = 0;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = r; s < 3; ++s) {
          Pi[k] += ha[r] * (w00 * ha[s] + w01 * hb[s]) + hb[r] * (w01 * ha[s] + w11 * hb[s]);
          ++k;
        }
      double Pp[6], Sp[3];
      bool good = mappt_chol3(Pi, Lp);
      if (good) {
        mappt_chol3_inv(Lp, Pp);
        mappt_innov(ha, hb, Pp, Rf, U, Sp);
        good = mappt_quad2(Sp, nu, &d1) && isfinite(d1) && isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
#pragma unroll
        for (int r = 0; r < 6; ++r) good = good && isfinite(Pp[r]);
      }
      if (good) {
#pragma unroll
        for (int r = 0; r < 6; ++r) P[r] = Pp[r];
      } else {
        status = 2;
        d0 = d1 = NAN;
#pragma unroll
        for (int r = 0; r < 3; ++r) X[r] = X0[r];
      }
    }
  }
  if (status != 0) d1 = NAN;
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = X[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) o[3 + k] = P[k];
  o[9] = d0;
  o[10] = d1;
  o[11] = e0;
  o[12] = status;
}

// Multi-view triangulation of cosl_tri_solver_submit (DESIGN.md 5.5, an extension).  The camera table is staged as
// TriCam records; per view, TRI_VIEW doubles m[2] | Sigma_m (xx xy yy); per point, TRI_OUT doubles come back:
// X[3] | P (6: xx xy xz yy yz zz) | f, e_max, parallax, rho | status.  The per-view scratch holds TRI_SCRATCH doubles:
// R_v^-1 (xx xy yy) | the unit ray from X+ to the camera centre.
constexpr int TRI_THREADS = 64;
constexpr int TRI_MAX_VIEWS = 32;
constexpr int TRI_MAX_ITER = 10;
constexpr int TRI_HALVINGS = 4;
constexpr int TRI_VIEW = 5;
constexpr int TRI_OUT = 14;
constexpr int TRI_SCRATCH = 6;

struct TriCam {
  double K[9], Ki[9], R[9], t[3];  // Ki = K^-1, computed by the host
  double P[36];                    // the pose covariance, read only when hasP
  int hasP, pad;
};

// K, R and t of a camera record through the read-only path
__device__ __forceinline__ void tri_cam(const TriCam* __restrict__ c, double K[9], double R[9], double t[3]) {
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    K[k] = __ldg(c->K + k);
    R[k] = __ldg(c->R + k);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = __ldg(c->t + k);
}

// The camera centre -R^T t
__device__ __forceinline__ void tri_centre(const double R[9], const double t[3], double C[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) C[k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);
}

// Rf += H_c P_c H_c^T: a camera's pose covariance P_c (6x6 row-major, chart R' = R exp([w]x), t' = t + dt) as noise of
// the projection of X.  H_c is the analytic 2x6 Jacobian of 5.1 with rows (X x ha, a) and (X x hb, b), a, b, ha, hb as
// mappt_project returns them at X: pose_mappt_kernel's R_eff arithmetic, which keeps its own inline copy (as a call it
// compiles to a different register allocation).
__device__ __forceinline__ void tri_pose_noise(const double X[3], const double a[3], const double b[3],
                                               const double ha[3], const double hb[3], const double* Pc,
                                               double Rf[3]) {
  double Hc[12];
  Hc[0] = X[1] * ha[2] - X[2] * ha[1];
  Hc[1] = X[2] * ha[0] - X[0] * ha[2];
  Hc[2] = X[0] * ha[1] - X[1] * ha[0];
  Hc[6] = X[1] * hb[2] - X[2] * hb[1];
  Hc[7] = X[2] * hb[0] - X[0] * hb[2];
  Hc[8] = X[0] * hb[1] - X[1] * hb[0];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    Hc[3 + k] = a[k];
    Hc[9 + k] = b[k];
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double t0 = 0, t1 = 0;
#pragma unroll
    for (int l = 0; l < 6; ++l) {
      t0 += Hc[l] * Pc[6 * l + k];
      t1 += Hc[6 + l] * Pc[6 * l + k];
    }
    Rf[0] += t0 * Hc[k];
    Rf[1] += t0 * Hc[6 + k];
    Rf[2] += t1 * Hc[6 + k];
  }
}

// mappt_chol3 of A with a smallest relative pivot L_kk^2 / A_kk of at least 1e-12: the positive-definiteness test of
// every 3x3 this stage factors (A of the rays, N of the Gauss-Newton steps and of the covariance).  A point running
// off to infinity leaves N singular to roundoff, where a plain Cholesky may still pass.
__device__ __forceinline__ bool tri_chol3(const double A[6], double L[6]) {
  return mappt_chol3(A, L) && fmin(fmin(L[0] * L[0] / A[0], L[2] * L[2] / A[3]), L[5] * L[5] / A[5]) >= 1e-12;
}

// One thread per point, over its views [off[j], off[j + 1]) (camera vcam[v], observation views[v]):
//   1. X_lin = A^-1 b, A = sum (I - d d^T), b = sum (I - d d^T) C, d = normalize(R^T K^-1 [m; 1]), C = -R^T t, by
//      Cholesky; a smallest relative pivot L_kk^2 / A_kk below 1e-12 (parallel rays) gives status 4;
//   2. R_v = Sigma_m + H_c P_c H_c^T at X_lin (Sigma_m alone without P_c); R_v^-1 goes to the scratch; a non-positive
//      definite R_v gives status 4;
//   3. from X_lin in front of every camera, at most TRI_MAX_ITER Gauss-Newton steps s = N^-1 sum H_X^T R_v^-1 nu_v,
//      N = sum H_X^T R_v^-1 H_X, each taken when it lowers f = sum nu^T R_v^-1 nu (the change formed from differences,
//      as mappt_descent) and keeps every depth > 0, else halved at most TRI_HALVINGS times, and stopped at
//      |s| <= 1e-12 max(1, |X|) or when N is not positive definite (tri_chol3);
//   4. P = N^-1 at X+ by Cholesky, status 4 when N is not positive definite (tri_chol3);
//   5. f, e_max = max |nu_v|, the largest angle between two rays X+ -> C_v, rho = sqrt(trace P) / |X+ - C_last|;
//   6. status 4 degenerate (also any non-finite output), 1 a depth <= 0 at X_lin or X+, 2 rho > 1, 3 e_max >= max_err,
//      else 0; with status 1 or 4 X, P and the statistics are NaN.
// The view loops stay rolled: a point has up to TRI_MAX_VIEWS views.  __maxnreg__ instead of __launch_bounds__
// (TRI_THREADS-thread CTAs either way): under the launch bounds ptxas stopped at 128 registers and spilled.
__global__ void __maxnreg__(168)
tri_kernel(const TriCam* __restrict__ cams, const double* __restrict__ views, const int* __restrict__ off,
           const int* __restrict__ vcam, int nPts, double max_err, double* __restrict__ scratch,
           double* __restrict__ out) {
  const int j = blockIdx.x * TRI_THREADS + threadIdx.x;
  if (j >= nPts) return;
  const int o = off[j], n = off[j + 1] - o;
  const double* q = views + (size_t)TRI_VIEW * o;
  const int* vc = vcam + o;
  double* W = scratch + (size_t)TRI_SCRATCH * o;
  double* r = out + (size_t)TRI_OUT * j;
  double K[9], R[9], t[3];
  // 1. the point closest to every ray
  double A[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
#pragma unroll 1
  for (int v = 0; v < n; ++v) {
    const TriCam* c = cams + vc[v];
    tri_cam(c, K, R, t);
    const double m0 = q[TRI_VIEW * v], m1 = q[TRI_VIEW * v + 1];
    double x[3], d[3], C[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
      x[k] = __ldg(c->Ki + 3 * k) * m0 + __ldg(c->Ki + 3 * k + 1) * m1 + __ldg(c->Ki + 3 * k + 2);
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = R[k] * x[0] + R[3 + k] * x[1] + R[6 + k] * x[2];
    const double dn = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] /= dn;
    tri_centre(R, t, C);
    const double dc = d[0] * C[0] + d[1] * C[1] + d[2] * C[2];
    A[0] += 1.0 - d[0] * d[0];
    A[1] -= d[0] * d[1];
    A[2] -= d[0] * d[2];
    A[3] += 1.0 - d[1] * d[1];
    A[4] -= d[1] * d[2];
    A[5] += 1.0 - d[2] * d[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) b[k] += C[k] - d[k] * dc;
  }
  double L[6], Ai[6], X[3];
  bool good = tri_chol3(A, L);
  if (good) {
    mappt_chol3_inv(L, Ai);
    X[0] = Ai[0] * b[0] + Ai[1] * b[1] + Ai[2] * b[2];
    X[1] = Ai[1] * b[0] + Ai[3] * b[1] + Ai[4] * b[2];
    X[2] = Ai[2] * b[0] + Ai[4] * b[1] + Ai[5] * b[2];
    good = isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
  }
  // 2. the noise of each view, fixed at X_lin
  bool behind = false;
#pragma unroll 1
  for (int v = 0; good && v < n; ++v) {
    const TriCam* c = cams + vc[v];
    tri_cam(c, K, R, t);
    double pm[2], a[3], bb[3], ha[3], hb[3], w;
    behind |= !(mappt_project(K, R, t, X, pm, a, bb, ha, hb, &w) > 0);
    double Rf[3] = {q[TRI_VIEW * v + 2], q[TRI_VIEW * v + 3], q[TRI_VIEW * v + 4]};
    if (__ldg(&c->hasP)) tri_pose_noise(X, a, bb, ha, hb, c->P, Rf);
    const double det = Rf[0] * Rf[2] - Rf[1] * Rf[1];
    good = Rf[0] > 0 && det > 0 && isfinite(det) && isfinite(Rf[1]);
    W[TRI_SCRATCH * v] = Rf[2] / det;
    W[TRI_SCRATCH * v + 1] = -Rf[1] / det;
    W[TRI_SCRATCH * v + 2] = Rf[0] / det;
  }
  if (!good) {
#pragma unroll
    for (int k = 0; k < 13; ++k) r[k] = NAN;
    r[13] = 4;
    return;
  }
  // 3. Gauss-Newton from X_lin
#pragma unroll 1
  for (int it = 0; !behind && it < TRI_MAX_ITER; ++it) {
    double N[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
#pragma unroll 1
    for (int v = 0; v < n; ++v) {
      tri_cam(cams + vc[v], K, R, t);
      double pm[2], a[3], bb[3], ha[3], hb[3], w;
      mappt_project(K, R, t, X, pm, a, bb, ha, hb, &w);
      const double nu0 = q[TRI_VIEW * v] - pm[0], nu1 = q[TRI_VIEW * v + 1] - pm[1];
      const double w00 = W[TRI_SCRATCH * v], w01 = W[TRI_SCRATCH * v + 1], w11 = W[TRI_SCRATCH * v + 2];
      double wa[3], wb[3];  // rows of R_v^-1 H_X
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        wa[k] = w00 * ha[k] + w01 * hb[k];
        wb[k] = w01 * ha[k] + w11 * hb[k];
      }
      int k = 0;
#pragma unroll
      for (int a0 = 0; a0 < 3; ++a0) {
#pragma unroll
        for (int a1 = a0; a1 < 3; ++a1) N[k++] += ha[a0] * wa[a1] + hb[a0] * wb[a1];
        g[a0] += wa[a0] * nu0 + wb[a0] * nu1;
      }
    }
    double Ln[6], Ni[6], s[3];
    if (!tri_chol3(N, Ln)) break;
    mappt_chol3_inv(Ln, Ni);
    s[0] = Ni[0] * g[0] + Ni[1] * g[1] + Ni[2] * g[2];
    s[1] = Ni[1] * g[0] + Ni[3] * g[1] + Ni[4] * g[2];
    s[2] = Ni[2] * g[0] + Ni[4] * g[1] + Ni[5] * g[2];
    bool taken = false;
    double Xn[3];
#pragma unroll 1
    for (int h = 0; !taken && h <= TRI_HALVINGS; ++h) {
      if (h) {
#pragma unroll
        for (int k = 0; k < 3; ++k) s[k] *= 0.5;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) Xn[k] = X[k] + s[k];
      // f(X + s) - f(X) = -sum dpi^T R_v^-1 (2 nu - dpi), dpi = (dx_{0,1} - pi dx_2) / (x_2 + dx_2), dx = K R s
      bool front = true;
      double meas = 0;
#pragma unroll 1
      for (int v = 0; front && v < n; ++v) {
        tri_cam(cams + vc[v], K, R, t);
        double c[3], x[3], dc[3], dx[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          c[k] = R[3 * k] * X[0] + R[3 * k + 1] * X[1] + R[3 * k + 2] * X[2] + t[k];
          dc[k] = R[3 * k] * s[0] + R[3 * k + 1] * s[1] + R[3 * k + 2] * s[2];
        }
        front = R[6] * Xn[0] + R[7] * Xn[1] + R[8] * Xn[2] + t[2] > 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          x[k] = K[3 * k] * c[0] + K[3 * k + 1] * c[1] + K[3 * k + 2] * c[2];
          dx[k] = K[3 * k] * dc[0] + K[3 * k + 1] * dc[1] + K[3 * k + 2] * dc[2];
        }
        const double p0 = x[0] / x[2], p1 = x[1] / x[2];
        const double wn = x[2] + dx[2];
        const double dp0 = (dx[0] - p0 * dx[2]) / wn, dp1 = (dx[1] - p1 * dx[2]) / wn;
        const double q0 = 2.0 * (q[TRI_VIEW * v] - p0) - dp0, q1 = 2.0 * (q[TRI_VIEW * v + 1] - p1) - dp1;
        meas += W[TRI_SCRATCH * v] * dp0 * q0 + W[TRI_SCRATCH * v + 1] * (dp0 * q1 + dp1 * q0) +
                W[TRI_SCRATCH * v + 2] * dp1 * q1;
      }
      taken = front && -meas < 0;
    }
    if (!taken) break;
#pragma unroll
    for (int k = 0; k < 3; ++k) X[k] = Xn[k];
    const double xn = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
    if (sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]) <= 1e-12 * fmax(1.0, xn)) break;
  }
  // 4.-5. covariance and statistics at X+
  double N[6] = {0, 0, 0, 0, 0, 0}, f = 0, emax = 0, dlast = 0;
#pragma unroll 1
  for (int v = 0; v < n; ++v) {
    tri_cam(cams + vc[v], K, R, t);
    double pm[2], a[3], bb[3], ha[3], hb[3], w, C[3];
    behind |= !(mappt_project(K, R, t, X, pm, a, bb, ha, hb, &w) > 0);
    const double nu0 = q[TRI_VIEW * v] - pm[0], nu1 = q[TRI_VIEW * v + 1] - pm[1];
    const double w00 = W[TRI_SCRATCH * v], w01 = W[TRI_SCRATCH * v + 1], w11 = W[TRI_SCRATCH * v + 2];
    f += w00 * nu0 * nu0 + 2.0 * w01 * nu0 * nu1 + w11 * nu1 * nu1;
    const double e = sqrt(nu0 * nu0 + nu1 * nu1);
    emax = e > emax ? e : emax;
    double wa[3], wb[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      wa[k] = w00 * ha[k] + w01 * hb[k];
      wb[k] = w01 * ha[k] + w11 * hb[k];
    }
    int k = 0;
#pragma unroll
    for (int a0 = 0; a0 < 3; ++a0)
#pragma unroll
      for (int a1 = a0; a1 < 3; ++a1) N[k++] += ha[a0] * wa[a1] + hb[a0] * wb[a1];
    tri_centre(R, t, C);
    const double u0 = C[0] - X[0], u1 = C[1] - X[1], u2 = C[2] - X[2];
    const double un = sqrt(u0 * u0 + u1 * u1 + u2 * u2);
    W[TRI_SCRATCH * v + 3] = u0 / un;
    W[TRI_SCRATCH * v + 4] = u1 / un;
    W[TRI_SCRATCH * v + 5] = u2 / un;
    dlast = un;
  }
  double Ln[6], P[6];
  good = tri_chol3(N, Ln);
  if (good) mappt_chol3_inv(Ln, P);
  double par = 0;  // atan2(|u x w|, u . w) is accurate at small angles, where acos is not
#pragma unroll 1
  for (int v = 1; v < n; ++v) {
    const double u0 = W[TRI_SCRATCH * v + 3], u1 = W[TRI_SCRATCH * v + 4], u2 = W[TRI_SCRATCH * v + 5];
#pragma unroll 1
    for (int i = 0; i < v; ++i) {
      const double w0 = W[TRI_SCRATCH * i + 3], w1 = W[TRI_SCRATCH * i + 4], w2 = W[TRI_SCRATCH * i + 5];
      const double x0 = u1 * w2 - u2 * w1, x1 = u2 * w0 - u0 * w2, x2 = u0 * w1 - u1 * w0;
      const double ang = atan2(sqrt(x0 * x0 + x1 * x1 + x2 * x2), u0 * w0 + u1 * w1 + u2 * w2);
      par = ang > par ? ang : par;
    }
  }
  int status = 4;
  if (good) {
    const double rho = sqrt(P[0] + P[3] + P[5]) / dlast;
    const double st[4] = {f, emax, par, rho};
#pragma unroll
    for (int k = 0; k < 3; ++k) good = good && isfinite(X[k]);
#pragma unroll
    for (int k = 0; k < 6; ++k) good = good && isfinite(P[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k) good = good && isfinite(st[k]);
    status = !good ? 4 : behind ? 1 : rho > 1.0 ? 2 : emax >= max_err ? 3 : 0;
    if (status != 1 && status != 4) {
#pragma unroll
      for (int k = 0; k < 3; ++k) r[k] = X[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) r[3 + k] = P[k];
#pragma unroll
      for (int k = 0; k < 4; ++k) r[9 + k] = st[k];
    }
  }
  if (status == 1 || status == 4) {
#pragma unroll
    for (int k = 0; k < 13; ++k) r[k] = NAN;
  }
  r[13] = status;
}

// Map-point registration of cosl_assoc_solver_submit (DESIGN.md 5.6, an extension).  The camera table is staged as
// AssocCam records; per point ASSOC_PT doubles X[3] | P_X (6: xx xy xz yy yz zz); per feature ASSOC_FEAT doubles
// m_f[2] | Sigma_f (xx xy yy) and its cell (an int, cell0 of its entry + cy nx + cx, cx = clamp(floor(x / ASSOC_CELL),
// 0, nx - 1), likewise cy); per track observation 2 doubles m_k.  Per query pair, ASSOC_OUT doubles come back:
// status | feat | d2, d2_2 | pred (m_hat[2], S xx xy yy).
constexpr int ASSOC_THREADS = 64;
constexpr int ASSOC_BIN_THREADS = 256;
constexpr int ASSOC_SCAN_THREADS = 1024;
constexpr int ASSOC_CELL = 32;          // px, the side of a grid cell
constexpr int ASSOC_MAX_SIDE = 4096;    // px, the largest image width or height an entry may have
constexpr int ASSOC_MAX_CELLS = (ASSOC_MAX_SIDE / ASSOC_CELL) * (ASSOC_MAX_SIDE / ASSOC_CELL);  // per entry
constexpr int ASSOC_MAX_QUERIES = 32;   // per point
constexpr int ASSOC_PT = 9;
constexpr int ASSOC_FEAT = 5;
constexpr int ASSOC_OUT = 9;

struct AssocCam {
  double K[9], R[9], t[3];
  double P[36];    // the pose covariance, read only when hasP
  double lam;      // the largest lambda_max(Sigma_f) over the entry's features, from the host
  double W, H;     // image size, px
  int hasP, nx, ny, cell0;  // the entry's grid: nx x ny cells from cell0 on
};

// d2 = |L^-1 nu|^2 with L L^T = A (a symmetric 2x2, xx xy yy): never negative; NaN unless A is positive definite
__device__ __forceinline__ double assoc_d2(const double A[3], double nu0, double nu1) {
  const double l00 = sqrt(A[0]);
  const double l10 = A[1] / l00;
  const double l11 = sqrt(A[2] - l10 * l10);
  const double z0 = nu0 / l00;
  const double z1 = (nu1 - l10 * z0) / l11;
  return z0 * z0 + z1 * z1;
}

// The projection m_hat of X in entry c and S = H_X P_X H_X^T (+ H_c P_c H_c^T with the entry's P_c) + add I; returns
// the depth.
__device__ __forceinline__ double assoc_predict(const AssocCam* __restrict__ c, const double X[3], const double PX[6],
                                                double add, double m[2], double S[3]) {
  double K[9], R[9], t[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    K[k] = __ldg(c->K + k);
    R[k] = __ldg(c->R + k);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = __ldg(c->t + k);
  double a[3], b[3], ha[3], hb[3], w, U[6];
  const double z = mappt_project(K, R, t, X, m, a, b, ha, hb, &w);
  double Rf[3] = {add, 0.0, add};
  if (__ldg(&c->hasP)) tri_pose_noise(X, a, b, ha, hb, c->P, Rf);
  mappt_innov(ha, hb, PX, Rf, U, S);
  return z;
}

// Count the features of every cell; cell[f] was staged by the host.
__global__ void __launch_bounds__(ASSOC_BIN_THREADS)
assoc_count_kernel(const int* __restrict__ cell, int nFeats, int* __restrict__ count) {
  const int f = blockIdx.x * ASSOC_BIN_THREADS + threadIdx.x;
  if (f < nFeats) atomicAdd(count + cell[f], 1);
}

// One CTA per entry: start[cell0 + i] = featOff[e] + the exclusive scan of the entry's cell counts, and the counts
// zeroed for the scatter's cursors.  The last entry also writes start[cells] = featOff[nCams], so that every cell's
// features are [start[i], start[i + 1]).
__global__ void __launch_bounds__(ASSOC_SCAN_THREADS)
assoc_scan_kernel(const AssocCam* __restrict__ cams, const int* __restrict__ featOff, int nCams,
                  int* __restrict__ count, int* __restrict__ start) {
  __shared__ int s_warp[ASSOC_SCAN_THREADS / 32];
  const int e = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = cams[e].cell0, n = cams[e].nx * cams[e].ny;
  int carry = featOff[e];
  for (int base = 0; base < n; base += ASSOC_SCAN_THREADS) {
    const int i = base + threadIdx.x;
    const int v = i < n ? count[c0 + i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    if (i < n) {
      start[c0 + i] = carry + x - v + (warp ? s_warp[warp - 1] : 0);
      count[c0 + i] = 0;
    }
    carry += s_warp[ASSOC_SCAN_THREADS / 32 - 1];
    __syncthreads();
  }
  if (e == nCams - 1 && threadIdx.x == 0) start[c0 + n] = featOff[nCams];
}

// Scatter every feature index into its cell's range of sorted; the order inside a cell is whatever the atomics give.
__global__ void __launch_bounds__(ASSOC_BIN_THREADS)
assoc_scatter_kernel(const int* __restrict__ cell, int nFeats, const int* __restrict__ start, int* __restrict__ cursor,
                     int* __restrict__ sorted) {
  const int f = blockIdx.x * ASSOC_BIN_THREADS + threadIdx.x;
  if (f < nFeats) {
    const int c = cell[f];
    sorted[start[c] + atomicAdd(cursor + c, 1)] = f;
  }
}

// One thread per query pair q (point qPt[q], entry qCam[q]):
//   1. x = R X + t, m_hat = pi(X), S = H_X P_X H_X^T + H_c P_c H_c^T (the second term with the entry's P_c only);
//      status 7 unless depth, m_hat and S are finite, 1 depth <= 0, 2 m_hat outside [0, W) x [0, H);
//   2. over the features of the cells the box |dx| <= sqrt(gate (S + lam I)_xx), |dy| <= sqrt(gate (S + lam I)_yy)
//      covers (widened by 1e-6 relative; lam >= lambda_max(Sigma_f) of every feature of the entry, so the box holds
//      every gate ellipse): d2_f = |L^-1 (m_f - m_hat)|^2, L L^T = S + Sigma_f; f* the least (d2, f) with d2 < gate,
//      d2_2 the second least d2 (+inf without one); status 3 without f*;
//   3. status 4 when f* is owned;
//   4. with a finite track_gate, status 5 when an earlier observation k of f* (entry trkCam[k], m_k) has depth <= 0
//      or not d2_k < track_gate, d2_k = |L^-1 (m_k - pi_k(X))|^2, L L^T = H_X P_X H_X^T + H_c P_c H_c^T + pixel_var I;
//   5. a pair still at status 0 enters the claims: pass one of the claim resolution, key[f*] = min bits of d2.
// The record gets status (0 for a claimant, resolved by assoc_claim_kernel and assoc_final_kernel), feat (-1 for 1, 2,
// 3 and 7), d2 and d2_2 (NaN for 1, 2 and 7; +inf for 3) and pred (NaN for 1 and 7).
__global__ void __launch_bounds__(ASSOC_THREADS)
assoc_search_kernel(const AssocCam* __restrict__ cams, const double* __restrict__ pts,
                    const double* __restrict__ feats, const int* __restrict__ owned,
                    const int* __restrict__ trkOff, const int* __restrict__ trkCam, const double* __restrict__ trkM,
                    const int* __restrict__ qPt, const int* __restrict__ qCam, int nQ,
                    const int* __restrict__ start, const int* __restrict__ sorted, double pixel_var, double gate,
                    double track_gate, unsigned long long* __restrict__ key, double* __restrict__ out) {
  const int q = blockIdx.x * ASSOC_THREADS + threadIdx.x;
  if (q >= nQ) return;
  double* r = out + (size_t)ASSOC_OUT * q;
  const double* pj = pts + (size_t)ASSOC_PT * qPt[q];
  const double X[3] = {pj[0], pj[1], pj[2]};
  const double PX[6] = {pj[3], pj[4], pj[5], pj[6], pj[7], pj[8]};
  const AssocCam* c = cams + qCam[q];
  double m[2], S[3];
  const double z = assoc_predict(c, X, PX, 0.0, m, S);
  int status = !(isfinite(z) && isfinite(m[0]) && isfinite(m[1]) && isfinite(S[0]) && isfinite(S[1]) &&
                 isfinite(S[2])) ? 7
               : !(z > 0) ? 1
               : !(m[0] >= 0 && m[0] < __ldg(&c->W) && m[1] >= 0 && m[1] < __ldg(&c->H)) ? 2 : 0;
  double best = INFINITY, second = INFINITY;
  int fs = -1;
  if (status == 0) {
    const double lam = __ldg(&c->lam);
    const int nx = __ldg(&c->nx), ny = __ldg(&c->ny), c0 = __ldg(&c->cell0);
    const double hx = sqrt(gate * (S[0] + lam)) * (1.0 + 1e-6), hy = sqrt(gate * (S[2] + lam)) * (1.0 + 1e-6);
    const double inv = 1.0 / ASSOC_CELL;
    const int x0 = (int)fmax(0.0, fmin(nx - 1.0, floor((m[0] - hx) * inv)));
    const int x1 = (int)fmax(0.0, fmin(nx - 1.0, floor((m[0] + hx) * inv)));
    const int y0 = (int)fmax(0.0, fmin(ny - 1.0, floor((m[1] - hy) * inv)));
    const int y1 = (int)fmax(0.0, fmin(ny - 1.0, floor((m[1] + hy) * inv)));
#pragma unroll 1
    for (int cy = y0; cy <= y1; ++cy) {
      const int row = c0 + cy * nx;
      const int i1 = start[row + x1 + 1];
#pragma unroll 1
      for (int i = start[row + x0]; i < i1; ++i) {
        const int f = sorted[i];
        const double* ff = feats + (size_t)ASSOC_FEAT * f;
        const double A[3] = {S[0] + ff[2], S[1] + ff[3], S[2] + ff[4]};
        const double d2 = assoc_d2(A, ff[0] - m[0], ff[1] - m[1]);
        if (!(d2 < gate)) continue;
        if (d2 < best || (d2 == best && f < fs)) {
          second = best;
          best = d2;
          fs = f;
        } else if (d2 < second) {
          second = d2;
        }
      }
    }
    if (fs < 0) status = 3;
    else if (owned[fs]) status = 4;
    else if (track_gate < INFINITY) {
#pragma unroll 1
      for (int k = trkOff[fs]; status == 0 && k < trkOff[fs + 1]; ++k) {
        double mk[2], Sk[3];
        const double zk = assoc_predict(cams + trkCam[k], X, PX, pixel_var, mk, Sk);
        const double d2k = assoc_d2(Sk, trkM[2 * (size_t)k] - mk[0], trkM[2 * (size_t)k + 1] - mk[1]);
        if (!(zk > 0) || !(d2k < track_gate)) status = 5;
      }
    }
    if (status == 0) atomicMin(key + fs, (unsigned long long)__double_as_longlong(best));
  }
  r[0] = status;
  r[1] = fs;
  r[2] = status == 1 || status == 2 || status == 7 ? NAN : best;
  r[3] = status == 1 || status == 2 || status == 7 ? NAN : second;
  const bool pred = status != 1 && status != 7;
  r[4] = pred ? m[0] : NAN;
  r[5] = pred ? m[1] : NAN;
  r[6] = pred ? S[0] : NAN;
  r[7] = pred ? S[1] : NAN;
  r[8] = pred ? S[2] : NAN;
}

// Pass two of the claim resolution: among the claimants of f* whose d2 is key[f*], win[f*] = the least point index.
__global__ void __launch_bounds__(ASSOC_BIN_THREADS)
assoc_claim_kernel(const int* __restrict__ qPt, int nQ, const unsigned long long* __restrict__ key,
                   unsigned int* __restrict__ win, const double* __restrict__ out) {
  const int q = blockIdx.x * ASSOC_BIN_THREADS + threadIdx.x;
  if (q >= nQ) return;
  const double* r = out + (size_t)ASSOC_OUT * q;
  if (r[0] != 0) return;
  const int f = (int)r[1];
  if ((unsigned long long)__double_as_longlong(r[2]) == key[f]) atomicMin(win + f, (unsigned int)qPt[q]);
}

// The claimants that lost their feature get status 6.
__global__ void __launch_bounds__(ASSOC_BIN_THREADS)
assoc_final_kernel(const int* __restrict__ qPt, int nQ, const unsigned long long* __restrict__ key,
                   const unsigned int* __restrict__ win, double* __restrict__ out) {
  const int q = blockIdx.x * ASSOC_BIN_THREADS + threadIdx.x;
  if (q >= nQ) return;
  double* r = out + (size_t)ASSOC_OUT * q;
  if (r[0] != 0) return;
  const int f = (int)r[1];
  if ((unsigned long long)__double_as_longlong(r[2]) != key[f] || win[f] != (unsigned int)qPt[q]) r[0] = 6;
}

// PnP RANSAC of an armed pose solver handle (cosl_pose_solver_set_ransac, DESIGN.md 5.7, an extension).  Before the
// solve, ransac_hyp_kernel draws and solves nHyp 5-point EPnP hypotheses per selected camera, ransac_score_kernel
// scores them and the caller's R0, t0 over the camera's points, and ransac_select_kernel picks one per camera and
// rewrites the record's R0, t0 when it replaces them.  tests/pnp_dense.py restates all of it operation for operation.
constexpr int RANSAC_HYP_THREADS = 32;
constexpr int RANSAC_SCORE_THREADS = 128;
constexpr int RANSAC_SEL_THREADS = 128;
constexpr int RANSAC_HYP = 13;   // per hypothesis: R[9] | t[3] | ok
constexpr int RANSAC_RES = 16;   // per camera: R[9] | t[3] | status | inliers | sse | h
constexpr int RANSAC_NDRAW = 256;
constexpr int RANSAC_SWEEPS3 = 12, RANSAC_SWEEPS12 = 16, RANSAC_GN = 5;
constexpr double RANSAC_JACOBI_TOL = 1e-30;
constexpr double RANSAC_PCA_MIN = 1e-12;
// per-thread scratch of ransac_hyp_kernel, in doubles: 12x12 MtM | its eigenvectors | alphas | world points |
// pixels | rho | camera points | K | the best candidate's R, t.  After the 12x12 solve the MtM section holds the
// beta stage (RS_L...).  Little stays in registers across the eigensolver and least-squares calls.
constexpr int RS_A = 0, RS_V = 144, RS_AL = 288, RS_PW = 308, RS_PX = 323, RS_RHO = 333, RS_PC = 339, RS_K = 354,
              RS_BEST = 363, RS_N = 375;
constexpr int RS_L = 0, RS_LSA = 60, RS_LSB = 90, RS_LSX = 96, RS_KA = 101, RS_KS = 110, RS_KV = 119, RS_CC = 128;

// One thread's scratch in shared memory, element i at p[i * RANSAC_HYP_THREADS]: the threads of a warp read
// consecutive doubles, and every index may be computed at run time without local memory.
struct Scr {
  double* p;
  __device__ __forceinline__ double& operator[](int i) const { return p[i * RANSAC_HYP_THREADS]; }
  __device__ __forceinline__ Scr operator+(int o) const { return Scr{p + o * RANSAC_HYP_THREADS}; }
};

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ bool finite_all(const double* x, int n) {
  bool f = true;
  for (int i = 0; i < n; ++i) f &= isfinite(x[i]);
  return f;
}

// Cyclic Jacobi on the symmetric n x n A (row-major): A = V diag(A_kk) V^T afterwards.  Sweeps over (p, q), p < q,
// row by row; each rotation theta = (a_qq - a_pp) / (2 a_pq), t = sign(theta) / (|theta| + sqrt(theta^2 + 1)),
// c = 1 / sqrt(t^2 + 1), s = t c goes to the columns p, q, then the rows p, q, then a_pq = a_qp = 0, and to V's
// columns; a_pq = 0 skips.  A sweep starts only while sum_{p<q} a_pq^2 > RANSAC_JACOBI_TOL sum_p a_pp^2.
__device__ __noinline__ void jacobi_sym(Scr A, Scr V, int n, int sweeps) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) V[n * i + j] = i == j ? 1.0 : 0.0;
  for (int sw = 0; sw < sweeps; ++sw) {
    double off = 0, dia = 0;
    for (int p = 0; p < n; ++p) {
      dia = dia + A[n * p + p] * A[n * p + p];
      for (int q = p + 1; q < n; ++q) off = off + A[n * p + q] * A[n * p + q];
    }
    if (off <= RANSAC_JACOBI_TOL * dia) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[n * p + q];
        if (apq == 0) continue;
        const double theta = (A[n * q + q] - A[n * p + p]) / (2.0 * apq);
        double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
        if (theta < 0) t = -t;
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double xp = A[n * k + p], xq = A[n * k + q];
          A[n * k + p] = c * xp - s * xq;
          A[n * k + q] = s * xp + c * xq;
        }
        for (int k = 0; k < n; ++k) {
          const double xp = A[n * p + k], xq = A[n * q + k];
          A[n * p + k] = c * xp - s * xq;
          A[n * q + k] = s * xp + c * xq;
        }
        A[n * p + q] = 0.0;
        A[n * q + p] = 0.0;
        for (int k = 0; k < n; ++k) {
          const double xp = V[n * k + p], xq = V[n * k + q];
          V[n * k + p] = c * xp - s * xq;
          V[n * k + q] = s * xp + c * xq;
        }
      }
  }
}

// min |A x - b| for A 6 x n (row-major, n <= 5) by Householder QR; A and b are overwritten, x gets n values.
__device__ __noinline__ void lstsq6(Scr A, Scr b, Scr x, int n) {
  for (int k = 0; k < n; ++k) {
    double nrm2 = 0;
    for (int i = k; i < 6; ++i) nrm2 = nrm2 + A[n * i + k] * A[n * i + k];
    const double alpha = A[n * k + k] > 0 ? -sqrt(nrm2) : sqrt(nrm2);
    double v[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) v[i] = i < k ? 0.0 : i == k ? A[n * i + k] - alpha : A[n * i + k];
    double vv = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (i >= k) vv = vv + v[i] * v[i];
    for (int j = k; j < n; ++j) {
      double f = 0;
#pragma unroll
      for (int i = 0; i < 6; ++i)
        if (i >= k) f = f + v[i] * A[n * i + j];
      f = 2.0 * f / vv;
#pragma unroll
      for (int i = 0; i < 6; ++i)
        if (i >= k) A[n * i + j] = A[n * i + j] - f * v[i];
    }
    double f = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (i >= k) f = f + v[i] * b[i];
    f = 2.0 * f / vv;
#pragma unroll
    for (int i = 0; i < 6; ++i)
      if (i >= k) b[i] = b[i] - f * v[i];
  }
  for (int k = n - 1; k >= 0; --k) {
    double a = b[k];
    for (int j = k + 1; j < n; ++j) a = a - A[n * k + j] * x[j];
    x[k] = a / A[n * k + k];
  }
}

// The first n columns of L (6 x 10) over the betas {B11 B12 B13 B14} (n = 4: columns 0, 1, 3, 6) or {B11 B12 B22
// B13 B23} (n = 3 or 5: columns 0 to n - 1) into the least-squares matrix, rho into its right-hand side, and the solve.
__device__ __forceinline__ void betas_lstsq(Scr s, int n) {
  for (int i = 0; i < 6; ++i) {
    for (int j = 0; j < n; ++j) s[RS_LSA + n * i + j] = s[RS_L + 10 * i + (n == 4 ? (j * (j + 1)) / 2 : j)];
    s[RS_LSB + i] = s[RS_RHO + i];
  }
  lstsq6(s + RS_LSA, s + RS_LSB, s + RS_LSX, n);
}

// The pose of the betas b: camera-frame control points sum_k b_k v_k (v_k = column ev[k] of V), the sample's camera
// points, the sign fix and the absolute orientation (pnp_dense.pose_from_betas).  Returns the summed reprojection
// error over the sample in px, +inf when anything is not finite.
__device__ double epnp_pose(Scr s, const int ev[4], const double b[4], double R[9], double t[3]) {
  for (int j = 0; j < 4; ++j)
    for (int k = 0; k < 3; ++k) {
      const int r = 3 * j + k;
      s[RS_CC + r] = b[0] * s[RS_V + 12 * r + ev[0]] + b[1] * s[RS_V + 12 * r + ev[1]] +
                     b[2] * s[RS_V + 12 * r + ev[2]] + b[3] * s[RS_V + 12 * r + ev[3]];
    }
  for (int i = 0; i < 5; ++i)
    for (int k = 0; k < 3; ++k)
      s[RS_PC + 3 * i + k] = s[RS_AL + 4 * i] * s[RS_CC + k] + s[RS_AL + 4 * i + 1] * s[RS_CC + 3 + k] +
                             s[RS_AL + 4 * i + 2] * s[RS_CC + 6 + k] + s[RS_AL + 4 * i + 3] * s[RS_CC + 9 + k];
  if (s[RS_PC + 2] < 0)
    for (int i = 0; i < 15; ++i) s[RS_PC + i] = -s[RS_PC + i];
  double pc0[3], pw0[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double a = s[RS_PC + k], w = s[RS_PW + k];
    for (int i = 1; i < 5; ++i) {
      a = a + s[RS_PC + 3 * i + k];
      w = w + s[RS_PW + 3 * i + k];
    }
    pc0[k] = a / 5.0;
    pw0[k] = w / 5.0;
  }
  double A[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) A[q] = 0.0;
  for (int i = 0; i < 5; ++i) {
    double dc[3], dw[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      dc[k] = s[RS_PC + 3 * i + k] - pc0[k];
      dw[k] = s[RS_PW + 3 * i + k] - pw0[k];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int c = 0; c < 3; ++c) A[3 * a + c] += dc[a] * dw[c];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) s[RS_KS + 3 * a + c] = A[a] * A[c] + A[3 + a] * A[3 + c] + A[6 + a] * A[6 + c];
  jacobi_sym(s + RS_KS, s + RS_KV, 3, RANSAC_SWEEPS3);
  // columns of V by decreasing eigenvalue, ties to the lower index
  const double l0 = s[RS_KS], l1 = s[RS_KS + 4], l2 = s[RS_KS + 8];
  int o[3];
  o[0] = (l0 >= l1 && l0 >= l2) ? 0 : (l1 >= l2 ? 1 : 2);
  {
    const int a = o[0] == 0 ? 1 : 0, c = o[0] == 2 ? 1 : 2;
    const double la = a == 0 ? l0 : l1, lc = c == 1 ? l1 : l2;
    o[1] = la >= lc ? a : c;
    o[2] = la >= lc ? c : a;
  }
  double v1[3], v2[3], v3[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    v1[k] = s[RS_KV + 3 * k + o[0]];
    v2[k] = s[RS_KV + 3 * k + o[1]];
    v3[k] = s[RS_KV + 3 * k + o[2]];
  }
  double u1[3], u2[3], u3[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    u1[i] = A[3 * i] * v1[0] + A[3 * i + 1] * v1[1] + A[3 * i + 2] * v1[2];
    u2[i] = A[3 * i] * v2[0] + A[3 * i + 1] * v2[1] + A[3 * i + 2] * v2[2];
  }
  const double n1 = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) u1[i] = u1[i] / n1;
  const double d12 = u1[0] * u2[0] + u1[1] * u2[1] + u1[2] * u2[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) u2[i] = u2[i] - d12 * u1[i];
  const double n2 = sqrt(u2[0] * u2[0] + u2[1] * u2[1] + u2[2] * u2[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) u2[i] = u2[i] / n2;
  u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
  u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
  u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
  const double detV = v1[0] * (v2[1] * v3[2] - v2[2] * v3[1]) - v2[0] * (v1[1] * v3[2] - v1[2] * v3[1]) +
                      v3[0] * (v1[1] * v2[2] - v1[2] * v2[1]);
  const double sgn = detV < 0 ? -1.0 : 1.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[3 * i + j] = u1[i] * v1[j] + u2[i] * v2[j] + sgn * u3[i] * v3[j];
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = pc0[i] - (R[3 * i] * pw0[0] + R[3 * i + 1] * pw0[1] + R[3 * i + 2] * pw0[2]);
  double K[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) K[q] = s[RS_K + q];
  double err = 0;
  for (int i = 0; i < 5; ++i) {
    const double M[3] = {s[RS_PW + 3 * i], s[RS_PW + 3 * i + 1], s[RS_PW + 3 * i + 2]};
    double m[2];
    project(K, R, t, M, m);
    const double du = s[RS_PX + 2 * i] - m[0], dv = s[RS_PX + 2 * i + 1] - m[1];
    err = err + sqrt(du * du + dv * dv);
  }
  return (isfinite(err) && finite_all(R, 9) && finite_all(t, 3)) ? err : CUDART_INF;
}

// One hypothesis per thread: the sampler, then EPnP on the sample (DESIGN.md 5.7).  hyp[c][h] gets R | t | ok and
// smp[c][h] the 5 indices (-1 without 5 distinct ones); a camera that is not selected or has fewer than 5 points gets
// ok = 0 and indices -1.
__global__ void __launch_bounds__(RANSAC_HYP_THREADS)
ransac_hyp_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll, const double* __restrict__ msAll,
                  const unsigned char* __restrict__ use, int nHyp, unsigned long long seed, double* __restrict__ hyp,
                  int* __restrict__ smp) {
  extern __shared__ double s_scr[];
  const int c = blockIdx.y;
  const int h = blockIdx.x * RANSAC_HYP_THREADS + threadIdx.x;
  if (h >= nHyp) return;
  const Scr s{s_scr + threadIdx.x};
  const PoseCam& cam = cams[c];
  const int n = cam.npts;
  double* out = hyp + RANSAC_HYP * ((size_t)c * nHyp + h);
  int* idx = smp + 5 * ((size_t)c * nHyp + h);
  out[12] = 0.0;
  int i0 = -1, i1 = -1, i2 = -1, i3 = -1, i4 = -1, cnt = 0;
  if (use[c] && n >= 5) {
    const unsigned long long base = seed ^ (((unsigned long long)c << 40) | ((unsigned long long)h << 8));
    for (int j = 0; j < RANSAC_NDRAW && cnt < 5; ++j) {
      const int v = (int)(splitmix64(base ^ (unsigned long long)j) % (unsigned long long)n);
      if (v == i0 || v == i1 || v == i2 || v == i3) continue;
      if (cnt == 0) i0 = v;
      else if (cnt == 1) i1 = v;
      else if (cnt == 2) i2 = v;
      else if (cnt == 3) i3 = v;
      else i4 = v;
      ++cnt;
    }
  }
  if (cnt < 5) i0 = i1 = i2 = i3 = i4 = -1;
  idx[0] = i0;
  idx[1] = i1;
  idx[2] = i2;
  idx[3] = i3;
  idx[4] = i4;
  if (cnt < 5) return;
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
#pragma unroll
  for (int k = 0; k < 9; ++k) s[RS_K + k] = cam.K[k];
  const int sel[5] = {i0, i1, i2, i3, i4};
#pragma unroll
  for (int i = 0; i < 5; ++i) {
#pragma unroll
    for (int k = 0; k < 3; ++k) s[RS_PW + 3 * i + k] = Ms[3 * sel[i] + k];
#pragma unroll
    for (int k = 0; k < 2; ++k) s[RS_PX + 2 * i + k] = ms[2 * sel[i] + k];
  }
  // control points: the centroid and the principal axes
  double c0[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double a = s[RS_PW + k];
    for (int i = 1; i < 5; ++i) a = a + s[RS_PW + 3 * i + k];
    c0[k] = a / 5.0;
  }
  {
    double Cv[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) Cv[q] = 0.0;
    for (int i = 0; i < 5; ++i) {
      double D[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) D[k] = s[RS_PW + 3 * i + k] - c0[k];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) Cv[3 * a + b] += D[a] * D[b];
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) s[RS_A + q] = Cv[q];
  }
  jacobi_sym(s + RS_A, s + RS_V, 3, RANSAC_SWEEPS3);
  const double l0 = s[RS_A], l1 = s[RS_A + 4], l2 = s[RS_A + 8];
  int o[3];
  o[0] = (l0 >= l1 && l0 >= l2) ? 0 : (l1 >= l2 ? 1 : 2);
  {
    const int a = o[0] == 0 ? 1 : 0, b = o[0] == 2 ? 1 : 2;
    const double la = a == 0 ? l0 : l1, lb = b == 1 ? l1 : l2;
    o[1] = la >= lb ? a : b;
    o[2] = la >= lb ? b : a;
  }
  double lam[3], E[9];  // E[3 k + j]: component k of axis j
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    lam[j] = o[j] == 0 ? l0 : o[j] == 1 ? l1 : l2;
#pragma unroll
    for (int k = 0; k < 3; ++k) E[3 * k + j] = s[RS_V + 3 * k + o[j]];
  }
  if (!finite_all(lam, 3) || !(lam[2] >= RANSAC_PCA_MIN * lam[0]) || !(lam[0] > 0)) return;
  double sc[3], cw[12];
#pragma unroll
  for (int j = 0; j < 3; ++j) sc[j] = sqrt(lam[j] / 5.0);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    cw[k] = c0[k];
#pragma unroll
    for (int j = 0; j < 3; ++j) cw[3 * (j + 1) + k] = c0[k] + sc[j] * E[3 * k + j];
  }
  for (int i = 0; i < 5; ++i) {
    const double D0 = s[RS_PW + 3 * i] - c0[0], D1 = s[RS_PW + 3 * i + 1] - c0[1], D2 = s[RS_PW + 3 * i + 2] - c0[2];
    double a[4];
#pragma unroll
    for (int j = 0; j < 3; ++j) a[j + 1] = (D0 * E[j] + D1 * E[3 + j] + D2 * E[6 + j]) / sc[j];
    a[0] = 1.0 - a[1] - a[2] - a[3];
#pragma unroll
    for (int j = 0; j < 4; ++j) s[RS_AL + 4 * i + j] = a[j];
  }
  {
    const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const double d0 = cw[3 * pa[r]] - cw[3 * pb[r]], d1 = cw[3 * pa[r] + 1] - cw[3 * pb[r] + 1],
                   d2 = cw[3 * pa[r] + 2] - cw[3 * pb[r] + 2];
      s[RS_RHO + r] = d0 * d0 + d1 * d1 + d2 * d2;
    }
  }
  // M^T M of the 10 x 12 M, rows accumulated in order
  for (int q = 0; q < 144; ++q) s[RS_A + q] = 0.0;
  for (int i = 0; i < 5; ++i)
    for (int r = 0; r < 2; ++r) {
      const double x = s[RS_PX + 2 * i + r];
      double row[12];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < 3; ++k) row[3 * j + k] = s[RS_AL + 4 * i + j] * (s[RS_K + 3 * r + k] - x * s[RS_K + 6 + k]);
#pragma unroll
      for (int b = 0; b < 12; ++b) s[RS_PC + b] = row[b];  // the camera-point section is free until the betas
#pragma unroll
      for (int a = 0; a < 12; ++a)
#pragma unroll 1
        for (int b = 0; b < 12; ++b) s[RS_A + 12 * a + b] = s[RS_A + 12 * a + b] + row[a] * s[RS_PC + b];
    }
  jacobi_sym(s + RS_A, s + RS_V, 12, RANSAC_SWEEPS12);
  // the eigenvectors of the 4 smallest eigenvalues, ties to the lower index
  int ev[4];
  {
    unsigned taken = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int best = -1;
      double bv = 0;
      for (int k = 0; k < 12; ++k) {
        const double d = s[RS_A + 13 * k];
        if (!isfinite(d)) return;
        if (!(taken >> k & 1u) && (best < 0 || d < bv)) {
          best = k;
          bv = d;
        }
      }
      taken |= 1u << best;
      ev[r] = best;
    }
  }
  // L_6x10 (the MtM section is free now)
  {
    const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
    for (int r = 0; r < 6; ++r) {
      double dv[4][3];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k)
          dv[i][k] = s[RS_V + 12 * (3 * pa[r] + k) + ev[i]] - s[RS_V + 12 * (3 * pb[r] + k) + ev[i]];
#define RDOT(a, b) (dv[a][0] * dv[b][0] + dv[a][1] * dv[b][1] + dv[a][2] * dv[b][2])
      s[RS_L + 10 * r + 0] = RDOT(0, 0);
      s[RS_L + 10 * r + 1] = 2.0 * RDOT(0, 1);
      s[RS_L + 10 * r + 2] = RDOT(1, 1);
      s[RS_L + 10 * r + 3] = 2.0 * RDOT(0, 2);
      s[RS_L + 10 * r + 4] = 2.0 * RDOT(1, 2);
      s[RS_L + 10 * r + 5] = RDOT(2, 2);
      s[RS_L + 10 * r + 6] = 2.0 * RDOT(0, 3);
      s[RS_L + 10 * r + 7] = 2.0 * RDOT(1, 3);
      s[RS_L + 10 * r + 8] = 2.0 * RDOT(2, 3);
      s[RS_L + 10 * r + 9] = RDOT(3, 3);
#undef RDOT
    }
  }
  double bestErr = CUDART_INF;
#pragma unroll 1
  for (int N = 1; N <= 3; ++N) {
    double b[4] = {0, 0, 0, 0};
    if (N == 1) {
      betas_lstsq(s, 4);
      const double x0 = s[RS_LSX];
      const bool neg = x0 < 0;
      b[0] = sqrt(neg ? -x0 : x0);
      for (int k = 1; k < 4; ++k) b[k] = (neg ? -s[RS_LSX + k] : s[RS_LSX + k]) / b[0];
    } else {
      betas_lstsq(s, N == 2 ? 3 : 5);
      const double x0 = s[RS_LSX], x1 = s[RS_LSX + 1], x2 = s[RS_LSX + 2];
      if (x0 < 0) {
        b[0] = sqrt(-x0);
        b[1] = x2 < 0 ? sqrt(-x2) : 0.0;
      } else {
        b[0] = sqrt(x0);
        b[1] = x2 > 0 ? sqrt(x2) : 0.0;
      }
      if (x1 < 0) b[0] = -b[0];
      if (N == 3) b[2] = s[RS_LSX + 3] / b[0];
    }
    for (int it = 0; it < RANSAC_GN; ++it) {  // Gauss-Newton on the 4 betas
      for (int i = 0; i < 6; ++i) {
        double l[10];
#pragma unroll
        for (int q = 0; q < 10; ++q) l[q] = s[RS_L + 10 * i + q];
        s[RS_LSA + 4 * i + 0] = 2.0 * l[0] * b[0] + l[1] * b[1] + l[3] * b[2] + l[6] * b[3];
        s[RS_LSA + 4 * i + 1] = l[1] * b[0] + 2.0 * l[2] * b[1] + l[4] * b[2] + l[7] * b[3];
        s[RS_LSA + 4 * i + 2] = l[3] * b[0] + l[4] * b[1] + 2.0 * l[5] * b[2] + l[8] * b[3];
        s[RS_LSA + 4 * i + 3] = l[6] * b[0] + l[7] * b[1] + l[8] * b[2] + 2.0 * l[9] * b[3];
        s[RS_LSB + i] = s[RS_RHO + i] - (l[0] * b[0] * b[0] + l[1] * b[0] * b[1] + l[2] * b[1] * b[1] +
                                         l[3] * b[0] * b[2] + l[4] * b[1] * b[2] + l[5] * b[2] * b[2] +
                                         l[6] * b[0] * b[3] + l[7] * b[1] * b[3] + l[8] * b[2] * b[3] +
                                         l[9] * b[3] * b[3]);
      }
      lstsq6(s + RS_LSA, s + RS_LSB, s + RS_LSX, 4);
#pragma unroll
      for (int k = 0; k < 4; ++k) b[k] = b[k] + s[RS_LSX + k];
    }
    double R[9], t[3];
    const double err = epnp_pose(s, ev, b, R, t);
    if (err < bestErr) {
      bestErr = err;
#pragma unroll
      for (int k = 0; k < 9; ++k) s[RS_BEST + k] = R[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) s[RS_BEST + 9 + k] = t[k];
    }
  }
  if (!isfinite(bestErr)) return;
  for (int k = 0; k < 12; ++k) out[k] = s[RS_BEST + k];
  out[12] = 1.0;
}

// Inlier count and sum of squared errors of pose (R, t) at one point: depth > 0 and sqrt(du^2 + dv^2) < thr.
__device__ __forceinline__ void ransac_point(const double K[9], const double R[9], const double t[3], const double* M,
                                            const double* m, double thr, bool& inl, double& e2) {
  const double c0 = R[0] * M[0] + R[1] * M[1] + R[2] * M[2] + t[0];
  const double c1 = R[3] * M[0] + R[4] * M[1] + R[5] * M[2] + t[1];
  const double c2 = R[6] * M[0] + R[7] * M[1] + R[8] * M[2] + t[2];
  const double u = K[0] * c0 + K[1] * c1 + K[2] * c2;
  const double v = K[3] * c0 + K[4] * c1 + K[5] * c2;
  const double w = K[6] * c0 + K[7] * c1 + K[8] * c2;
  const double du = m[0] - u / w, dv = m[1] - v / w;
  e2 = du * du + dv * dv;
  inl = c2 > 0 && sqrt(e2) < thr;
}

// Slot k of camera c (blockIdx.y) is the caller's R0, t0 for k = 0 and hypothesis k - 1 after; each thread scores
// one slot over the camera's points, staged through shared memory in tiles.  cnt = -1 (sse 0) for a degenerate
// hypothesis and for every hypothesis of a camera that draws none.
__global__ void __launch_bounds__(RANSAC_SCORE_THREADS)
ransac_score_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll,
                    const double* __restrict__ msAll, const unsigned char* __restrict__ use, int nHyp,
                    const double* __restrict__ hyp, double thr, int* __restrict__ cnt, double* __restrict__ sse) {
  __shared__ double s_pt[RANSAC_SCORE_THREADS * 5];
  const int c = blockIdx.y;
  const int k = blockIdx.x * RANSAC_SCORE_THREADS + threadIdx.x;
  const PoseCam& cam = cams[c];
  const int n = cam.npts;
  const bool draws = use[c] && n >= 5;
  int* oc = cnt + (size_t)c * (nHyp + 1);
  double* os = sse + (size_t)c * (nHyp + 1);
  if (!draws && blockIdx.x > 0) {  // uniform over the CTA
    if (k <= nHyp) {
      oc[k] = -1;
      os[k] = 0.0;
    }
    return;
  }
  double K[9], R[9], t[3];
  bool live = k <= nHyp;
#pragma unroll
  for (int q = 0; q < 9; ++q) K[q] = cam.K[q];
  if (k == 0) {
#pragma unroll
    for (int q = 0; q < 9; ++q) R[q] = cam.R0[q];
#pragma unroll
    for (int q = 0; q < 3; ++q) t[q] = cam.t0[q];
  } else if (live) {
    const double* r = hyp + RANSAC_HYP * ((size_t)c * nHyp + (k - 1));
    live = draws && r[12] != 0.0;
#pragma unroll
    for (int q = 0; q < 9; ++q) R[q] = r[q];
#pragma unroll
    for (int q = 0; q < 3; ++q) t[q] = r[9 + q];
  }
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
  int ni = 0;
  double acc = 0.0;
  for (int i0 = 0; i0 < n; i0 += RANSAC_SCORE_THREADS) {
    const int m = min(RANSAC_SCORE_THREADS, n - i0);
    __syncthreads();
    for (int q = threadIdx.x; q < 3 * m; q += RANSAC_SCORE_THREADS) s_pt[q] = Ms[3 * i0 + q];
    for (int q = threadIdx.x; q < 2 * m; q += RANSAC_SCORE_THREADS) s_pt[3 * RANSAC_SCORE_THREADS + q] = ms[2 * i0 + q];
    __syncthreads();
    if (live)
      for (int i = 0; i < m; ++i) {
        bool inl;
        double e2;
        ransac_point(K, R, t, s_pt + 3 * i, s_pt + 3 * RANSAC_SCORE_THREADS + 2 * i, thr, inl, e2);
        if (inl) {
          ++ni;
          acc = acc + e2;
        }
      }
  }
  if (k <= nHyp) {
    oc[k] = live ? ni : -1;
    os[k] = live ? acc : 0.0;
  }
}

// Slot a ranks before slot b: more inliers, then less sse, then the lower slot (slot 0, R0, is h = -1).
__device__ __forceinline__ bool ransac_before(int ca, double sa, int a, int cb, double sb, int b) {
  if (ca != cb) return ca > cb;
  if (sa != sb) return sa < sb;
  return a < b;
}

// One CTA per camera: the best slot by a reduction over a total order (so the result does not depend on thread
// order), the status, the start pose (written into the record when a hypothesis replaces R0, t0), the result record
// res[c] and the start pose's inlier flag of every point.
__global__ void __launch_bounds__(RANSAC_SEL_THREADS)
ransac_select_kernel(PoseCam* __restrict__ cams, const double* __restrict__ MsAll, const double* __restrict__ msAll,
                     const unsigned char* __restrict__ use, int nHyp, const double* __restrict__ hyp,
                     const int* __restrict__ cnt, const double* __restrict__ sse, double thr, int minInl,
                     double* __restrict__ res, unsigned char* __restrict__ inl) {
  __shared__ int s_k[RANSAC_SEL_THREADS], s_c[RANSAC_SEL_THREADS];
  __shared__ double s_s[RANSAC_SEL_THREADS];
  __shared__ double s_pose[12];
  const int c = blockIdx.x;
  PoseCam& cam = cams[c];
  const int n = cam.npts;
  const bool draws = use[c] && n >= 5;
  const int slots = draws ? nHyp + 1 : 1;
  const int* oc = cnt + (size_t)c * (nHyp + 1);
  const double* os = sse + (size_t)c * (nHyp + 1);
  int bk = 0, bc = oc[0];
  double bs = os[0];
  for (int k = threadIdx.x; k < slots; k += RANSAC_SEL_THREADS)
    if (ransac_before(oc[k], os[k], k, bc, bs, bk)) {
      bk = k;
      bc = oc[k];
      bs = os[k];
    }
  s_k[threadIdx.x] = bk;
  s_c[threadIdx.x] = bc;
  s_s[threadIdx.x] = bs;
  __syncthreads();
  for (int w = RANSAC_SEL_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      const int o = threadIdx.x + w;
      if (ransac_before(s_c[o], s_s[o], s_k[o], s_c[threadIdx.x], s_s[threadIdx.x], s_k[threadIdx.x])) {
        s_k[threadIdx.x] = s_k[o];
        s_c[threadIdx.x] = s_c[o];
        s_s[threadIdx.x] = s_s[o];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    bk = s_k[0];
    const int status = !use[c] ? 3 : n < 5 ? 1 : bk == 0 ? 4 : s_c[0] < minInl ? 2 : 0;
    const double* src = status == 0 ? hyp + RANSAC_HYP * ((size_t)c * nHyp + (bk - 1)) : nullptr;
    double* r = res + RANSAC_RES * (size_t)c;
    for (int q = 0; q < 9; ++q) s_pose[q] = src ? src[q] : cam.R0[q];
    for (int q = 0; q < 3; ++q) s_pose[9 + q] = src ? src[9 + q] : cam.t0[q];
    for (int q = 0; q < 12; ++q) r[q] = s_pose[q];
    r[12] = status;
    r[13] = s_c[0];
    r[14] = s_s[0];
    r[15] = bk - 1;
    if (status == 0) {
      for (int q = 0; q < 9; ++q) cam.R0[q] = s_pose[q];
      for (int q = 0; q < 3; ++q) cam.t0[q] = s_pose[9 + q];
    }
  }
  __syncthreads();
  double K[9], R[9], t[3];
#pragma unroll
  for (int q = 0; q < 9; ++q) {
    K[q] = cam.K[q];
    R[q] = s_pose[q];
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) t[q] = s_pose[9 + q];
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
  for (int i = threadIdx.x; i < n; i += RANSAC_SEL_THREADS) {
    bool f;
    double e2;
    ransac_point(K, R, t, Ms + 3 * i, ms + 2 * i, thr, f, e2);
    inl[cam.off + i] = f ? 1 : 0;
  }
}


// Checks of one solve's inputs shared by the batch call and cosl_pose_solver_submit; *tot = points over all
// cameras.
int check_cameras(const char* fn, int C, const int* npts, const double* const* Ms, const double* const* ms,
                  const cosl_pose_opt* opts, long long* tot) {
  long long n = 0;
  for (int c = 0; c < C; ++c) {
    if (npts[c] < 0 || (npts[c] && (!Ms[c] || !ms[c])))
      return set_error(COSL_E_INVALID, "%s: bad camera %d", fn, c);
    n += npts[c];
  }
  if (n > INT_MAX) return set_error(COSL_E_INVALID, "%s: %lld points exceed one solve", fn, n);
  // all opts share the solver settings of opts[0] except lambda0, which is per camera in the
  // reference (carried across calls by the caller); kernel cfg takes opts[0], lambda0 is uniform
  for (int c = 1; c < C; ++c)
    if (opts[c].lambda0 != opts[0].lambda0 || opts[c].maxIterLM != opts[0].maxIterLM ||
        opts[c].maxIterRW != opts[0].maxIterRW || opts[c].epsErrorChangeLM != opts[0].epsErrorChangeLM ||
        opts[c].epsParamChangeLM != opts[0].epsParamChangeLM ||
        opts[c].epsErrorChangeRW != opts[0].epsErrorChangeRW)
      return set_error(COSL_E_INVALID, "batched pose solve needs identical options per camera");
  *tot = n;
  return COSL_OK;
}

// The whitening factor of one measurement covariance c = [a b; b c'] (row-major, px^2): the upper-triangular
// L = {sqrt(c'/det), -b/sqrt(c' det), 1/sqrt(c')} with L^T L = c^-1, det = a c' - b^2.  False unless c is finite,
// exactly symmetric, a > 0, det > 0 and L comes out finite.
bool cov_factor(const double* c, double L[3]) {
  if (!std::isfinite(c[0]) || !std::isfinite(c[1]) || !std::isfinite(c[2]) || !std::isfinite(c[3])) return false;
  if (c[1] != c[2] || !(c[0] > 0)) return false;
  const double det = c[0] * c[3] - c[1] * c[1];
  if (!(det > 0)) return false;
  L[0] = std::sqrt(c[3] / det);
  L[1] = -c[1] / std::sqrt(c[3] * det);
  L[2] = 1.0 / std::sqrt(c[3]);
  return std::isfinite(L[0]) && std::isfinite(L[1]) && std::isfinite(L[2]) && L[0] > 0 && L[2] > 0;
}

// A measurement covariance c (row-major 2x2, nullable) as staged for the devices: (xx, xy, yy), or pixel_var I when c
// is nullptr.
void pack_cov2(const double* c, double pixel_var, double out[3]) {
  out[0] = c ? c[0] : pixel_var;
  out[1] = c ? c[1] : 0.0;
  out[2] = c ? c[3] : pixel_var;
}

// Checks every covariance of covx (nullable, as covx[c]) against cov_factor, naming the first bad one.
int check_covx(const char* fn, int C, const int* npts, const double* const* covx) {
  if (!covx) return COSL_OK;
  for (int c = 0; c < C; ++c) {
    if (!covx[c]) continue;
    for (int i = 0; i < npts[c]; ++i) {
      double L[3];
      const double* v = covx[c] + 4 * (size_t)i;
      if (!cov_factor(v, L))
        return set_error(COSL_E_INVALID,
                         "%s: covariance of camera %d point %d [%g %g; %g %g] is not finite, symmetric and positive "
                         "definite",
                         fn, c, i, v[0], v[1], v[2], v[3]);
    }
  }
  return COSL_OK;
}

// Cholesky A = G G^T of a symmetric positive definite 6x6 (row-major; G lower, row-major); false on a pivot that is
// not positive and finite.
bool chol6(const double* A, double* G) {
  for (int i = 0; i < 36; ++i) G[i] = 0.0;
  for (int j = 0; j < 6; ++j) {
    double d = A[7 * j];
    for (int k = 0; k < j; ++k) d -= G[6 * j + k] * G[6 * j + k];
    if (!(d > 0.0) || !std::isfinite(d)) return false;
    G[7 * j] = std::sqrt(d);
    for (int i = j + 1; i < 6; ++i) {
      double v = A[6 * i + j];
      for (int k = 0; k < j; ++k) v -= G[6 * i + k] * G[6 * j + k];
      G[6 * i + j] = v / G[7 * j];
    }
  }
  return true;
}

// S = 0.5 (P + P^T) of a 6x6 P (row-major)
void sym6(const double* P, double S[36]) {
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) S[6 * a + b] = 0.5 * (P[6 * a + b] + P[6 * b + a]);
}

// Checks camera c's prior record p (R_p[9] row-major | t_p[3] | P[36] row-major in the order (w, dt)) and, when out is
// not nullptr, writes its POSE_PRIOR_REC doubles: the upper-triangular L with L^T L = P^-1 packed by rows, R_p, t_p.
// R_p must be a rotation (|R_p^T R_p - I|_max <= 1e-9, det > 0), every value finite, P symmetric to 1e-12 of its
// largest diagonal entry and positive definite; otherwise COSL_E_INVALID names camera c.
int prior_factor(const char* fn, int c, const double* p, double* out) {
  const double *Rp = p, *tp = p + 9, *P = p + 12;
  for (int i = 0; i < 48; ++i)
    if (!std::isfinite(p[i])) return set_error(COSL_E_INVALID, "%s: prior of camera %d is not finite", fn, c);
  double orth = 0.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      const double g = Rp[a] * Rp[b] + Rp[3 + a] * Rp[3 + b] + Rp[6 + a] * Rp[6 + b] - (a == b ? 1.0 : 0.0);
      orth = std::max(orth, std::fabs(g));
    }
  const double det = Rp[0] * (Rp[4] * Rp[8] - Rp[5] * Rp[7]) - Rp[1] * (Rp[3] * Rp[8] - Rp[5] * Rp[6]) +
                     Rp[2] * (Rp[3] * Rp[7] - Rp[4] * Rp[6]);
  if (orth > 1e-9 || !(det > 0.0))
    return set_error(COSL_E_INVALID, "%s: R of camera %d's prior is not a rotation (|R^T R - I| %.3g, det %.17g)", fn,
                     c, orth, det);
  double pmax = 0.0;
  for (int i = 0; i < 6; ++i) pmax = std::max(pmax, std::fabs(P[7 * i]));
  for (int a = 0; a < 6; ++a)
    for (int b = a + 1; b < 6; ++b)
      if (std::fabs(P[6 * a + b] - P[6 * b + a]) > 1e-12 * pmax)
        return set_error(COSL_E_INVALID, "%s: P of camera %d's prior is not symmetric (%d, %d)", fn, c, a, b);
  // P = G G^T, P^-1 = G^-T G^-1 = C C^T and L = C^T
  double S[36], G[36], Gi[36] = {}, Pi[36], C[36];
  sym6(P, S);
  if (!chol6(S, G)) return set_error(COSL_E_INVALID, "%s: P of camera %d's prior is not positive definite", fn, c);
  for (int k = 0; k < 6; ++k)  // G^-1, lower, by forward substitution of the unit columns
    for (int i = k; i < 6; ++i) {
      double a = i == k ? 1.0 : 0.0;
      for (int q = k; q < i; ++q) a -= G[6 * i + q] * Gi[6 * q + k];
      Gi[6 * i + k] = a / G[6 * i + i];
    }
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) {
      double u = 0.0;
      for (int q = std::max(a, b); q < 6; ++q) u += Gi[6 * q + a] * Gi[6 * q + b];
      Pi[6 * a + b] = u;
    }
  if (!chol6(Pi, C)) return set_error(COSL_E_INVALID, "%s: P of camera %d's prior is not positive definite", fn, c);
  if (!out) return COSL_OK;
  int q = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) out[q++] = C[6 * b + a];
  for (int i = 0; i < 9; ++i) out[21 + i] = Rp[i];
  for (int i = 0; i < 3; ++i) out[30 + i] = tp[i];
  return COSL_OK;
}

// Checks every prior of prior (nullable, as prior[c]) with prior_factor, naming the first bad camera; *any = some
// camera has one.
int check_priors(const char* fn, int C, const double* const* prior, bool* any) {
  *any = false;
  if (!prior) return COSL_OK;
  for (int c = 0; c < C; ++c) {
    if (!prior[c]) continue;
    COSL_TRY(prior_factor(fn, c, prior[c], nullptr));
    *any = true;
  }
  return COSL_OK;
}

// The map points of cosl_pose_solver_submit_mappts, as passed
struct MapPtsArgs {
  const int* n;
  const double* const* X;
  const double* const* P;
  const double* const* m;
  const double* const* cov;  // nullable, as cov[c]
  double gate;
};

// True when the 3x3 covariance P (row-major) is finite, symmetric to 1e-12 of its largest diagonal entry and positive
// definite; S gets its symmetrised upper triangle (xx xy xz yy yz zz).
bool point_cov(const double* P, double S[6]) {
  double pmax = 0.0;
  for (int i = 0; i < 9; ++i)
    if (!std::isfinite(P[i])) return false;
  for (int i = 0; i < 3; ++i) pmax = std::max(pmax, std::fabs(P[4 * i]));
  for (int a = 0; a < 3; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (std::fabs(P[3 * a + b] - P[3 * b + a]) > 1e-12 * pmax) return false;
  int k = 0;
  for (int a = 0; a < 3; ++a)
    for (int b = a; b < 3; ++b) S[k++] = 0.5 * (P[3 * a + b] + P[3 * b + a]);
  // Cholesky pivots of S
  const double d0 = S[0];
  if (!(d0 > 0)) return false;
  const double l10 = S[1] / std::sqrt(d0), l20 = S[2] / std::sqrt(d0);
  const double d1 = S[3] - l10 * l10;
  if (!(d1 > 0)) return false;
  const double l21 = (S[4] - l20 * l10) / std::sqrt(d1);
  const double d2 = S[5] - l20 * l20 - l21 * l21;
  return d2 > 0 && std::isfinite(d2);
}

// A symmetric 3x3 packed as (xx xy xz yy yz zz), unpacked into P (row-major)
void unpack_sym3(const double* S, double P[9]) {
  P[0] = S[0];
  P[1] = P[3] = S[1];
  P[2] = P[6] = S[2];
  P[4] = S[3];
  P[5] = P[7] = S[4];
  P[8] = S[5];
}

// Checks the map points of one submit, naming the first bad camera and point; *tot = map points over all cameras.
int check_mappts(const char* fn, int C, int cap, const MapPtsArgs& mp, long long* tot) {
  if (!mp.n || !mp.X || !mp.P || !mp.m) return set_error(COSL_E_INVALID, "%s: null map-point argument", fn);
  if (!std::isfinite(mp.gate) || !(mp.gate > 0))
    return set_error(COSL_E_INVALID, "%s: gate %g is not a finite value > 0", fn, mp.gate);
  long long n = 0;
  for (int c = 0; c < C; ++c) {
    if (mp.n[c] < 0 || (mp.n[c] && (!mp.X[c] || !mp.P[c] || !mp.m[c])))
      return set_error(COSL_E_INVALID, "%s: bad map points of camera %d", fn, c);
    n += mp.n[c];
  }
  if (n > cap) return set_error(COSL_E_INVALID, "%s: %lld map points exceed the %d reserved", fn, n, cap);
  for (int c = 0; c < C; ++c)
    for (int i = 0; i < mp.n[c]; ++i) {
      const double* X = mp.X[c] + 3 * (size_t)i;
      const double* m = mp.m[c] + 2 * (size_t)i;
      if (!std::isfinite(X[0]) || !std::isfinite(X[1]) || !std::isfinite(X[2]) || !std::isfinite(m[0]) ||
          !std::isfinite(m[1]))
        return set_error(COSL_E_INVALID, "%s: map point %d of camera %d: X or m is not finite", fn, i, c);
      double S[6];
      if (!point_cov(mp.P[c] + 9 * (size_t)i, S))
        return set_error(COSL_E_INVALID,
                         "%s: map point %d of camera %d: P is not finite, symmetric and positive definite", fn, i, c);
      double L[3];
      if (mp.cov && mp.cov[c] && !cov_factor(mp.cov[c] + 4 * (size_t)i, L))
        return set_error(COSL_E_INVALID,
                         "%s: map point %d of camera %d: covm is not finite, symmetric and positive definite", fn, i,
                         c);
    }
  *tot = n;
  return COSL_OK;
}

// The section at byte offset `off` of a staging buffer or of its device copy
template <class T>
T* section(unsigned char* base, size_t off) {
  return reinterpret_cast<T*>(base + off);
}

// The sections of a pose solve's staging buffer and its device copy: PoseCam[C] | M[3 tot] | m[2 tot] | prevErrs[tot]
// | L[3 tot] | prior[C][POSE_PRIOR_REC] | hasPrior[C] | map[nmap][MAPPT_IN] | blk[nblk] (tot = points of the solve).
// The whitening factors L are carried by the submits with covariances, the priors by a submit with some prior, and
// the map points and the CTA table of pose_mappt_kernel by cosl_pose_solver_submit_mappts.  A section a submit does
// not carry takes 0 bytes, so its one copy of `bytes` stops within 255 bytes of the end of the last one it carries.
struct PoseLayout {
  size_t cams, M, m, prev, L, rec, has, map, blk, bytes;
};

PoseLayout pose_layout(int C, long long tot, bool obsCov, bool prior, long long nmap, int nblk) {
  SlabLayout S;
  PoseLayout o;
  o.cams = S.take(sizeof(PoseCam) * C);
  o.M = S.take(sizeof(double) * 3 * tot);
  o.m = S.take(sizeof(double) * 2 * tot);
  o.prev = S.take(sizeof(double) * tot);
  o.L = S.take(obsCov ? sizeof(double) * 3 * tot : 0);
  o.rec = S.take(prior ? sizeof(double) * POSE_PRIOR_REC * C : 0);
  o.has = S.take(prior ? sizeof(int) * C : 0);
  o.map = S.take(sizeof(double) * MAPPT_IN * nmap);
  o.blk = S.take(sizeof(int4) * nblk);
  o.bytes = S.bytes;
  return o;
}

}  // namespace

// A pose solver handle.  The inputs of one solve travel in one copy from a pinned staging buffer laid out by
// pose_layout; the PoseOuts come back into pinned memory.  Capacity is fixed at create: everything is allocated once,
// the covariance stage's buffers (laid out as res[C][POSE_COV_STRIDE] | err[tot]) when the handle is first armed, and
// the map-point sections and results (mres[nmap][MAPPT_OUT]) by cosl_pose_solver_reserve_mappts, which reallocates the
// staging buffers.
struct cosl_pose_solver {
  int device = 0, maxCams = 0, maxPts = 0;
  RequestStream rq;
  unsigned char* h_in = nullptr;
  unsigned char* d_in = nullptr;
  double* d_W = nullptr;
  PoseOut* d_out = nullptr;
  PoseOut* h_out = nullptr;
  int C = 0;           // cameras of the solve in flight
  long long tot = 0;   // points of the solve in flight
  PoseLayout lay = {}; // its staged sections
  double pixelVar = 0; // > 0: armed
  double* d_cov = nullptr;
  double* h_cov = nullptr;
  bool covReady = false;  // the last submitted solve was armed
  bool obsCov = false;    // the solve in flight carries measurement covariances
  bool prior = false;     // the solve in flight carries pose priors
  int maxMap = 0;         // map points reserved per submit
  double* d_mres = nullptr;
  double* h_mres = nullptr;
  bool map = false;       // the solve in flight carries map points
  bool mapReady = false;  // the last submit was a cosl_pose_solver_submit_mappts
  long long nmap = 0;     // map points of that submit
  int nblk = 0;           // CTAs of its pose_mappt_kernel
  double gate = 0;
  // PnP RANSAC (cosl_pose_solver_set_ransac): the armed setting (rC = 0: disarmed), its buffers, allocated by
  // set_ransac for rCap hypotheses per camera and laid out as hyp[maxCams][rCap][RANSAC_HYP], smp[maxCams][rCap][5],
  // cnt and sse[maxCams][rCap + 1], and the results res[C][RANSAC_RES] | inl[tot], copied back in one piece
  int rC = 0, rHyp = 0, rMinInl = 0, rCap = 0;
  double rThr = 0;
  unsigned long long rSeed = 0;
  unsigned char* d_ruse = nullptr;
  double* d_rhyp = nullptr;
  int* d_rsmp = nullptr;
  int* d_rcnt = nullptr;
  double* d_rsse = nullptr;
  unsigned char* d_rres = nullptr;
  unsigned char* h_rres = nullptr;
  bool ransac = false;       // the solve in flight runs RANSAC
  bool ransacReady = false;  // the last submit ran it
  bool ransacHyps = false;   // the hypothesis buffers still hold the last submit's
  int rHypRun = 0;           // nHyp of the last submit that ran it
};

namespace {

// the staging buffers' size: every section at the handle's maxima, with maxMap map points and a bound on their CTAs
// (sum_c ceil(n_c / MAPPT_THREADS), none without points)
size_t pose_capacity(const cosl_pose_solver* s, int maxMap) {
  const int maxBlk = (int)std::min<long long>(maxMap, maxMap / MAPPT_THREADS + s->maxCams);
  return pose_layout(s->maxCams, s->maxPts, true, true, maxMap, maxBlk).bytes;
}

void free_pose_solver(cosl_pose_solver* s) {
  cudaSetDevice(s->device);
  s->rq.destroy();
  if (s->h_in) cudaFreeHost(s->h_in);
  if (s->h_out) cudaFreeHost(s->h_out);
  if (s->h_cov) cudaFreeHost(s->h_cov);
  if (s->h_mres) cudaFreeHost(s->h_mres);
  cudaFree(s->d_in);
  cudaFree(s->d_W);
  cudaFree(s->d_out);
  cudaFree(s->d_cov);
  cudaFree(s->d_mres);
  if (s->h_rres) cudaFreeHost(s->h_rres);
  cudaFree(s->d_ruse);
  cudaFree(s->d_rhyp);
  cudaFree(s->d_rsmp);
  cudaFree(s->d_rcnt);
  cudaFree(s->d_rsse);
  cudaFree(s->d_rres);
  delete s;
}

size_t cov_doubles(int C, long long tot) { return (size_t)POSE_COV_STRIDE * C + tot; }

int alloc_pose_solver(cosl_pose_solver* s) {
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.create());
  const size_t in = pose_capacity(s, s->maxMap);
  COSL_CUDA(cudaHostAlloc(&s->h_in, in, cudaHostAllocPortable));
  COSL_CUDA(cudaHostAlloc(&s->h_out, sizeof(PoseOut) * s->maxCams, cudaHostAllocPortable));
  COSL_CUDA(cudaMalloc(&s->d_in, in));
  COSL_CUDA(cudaMalloc(&s->d_W, sizeof(double) * std::max(s->maxPts, 1)));
  COSL_CUDA(cudaMalloc(&s->d_out, sizeof(PoseOut) * s->maxCams));
  return COSL_OK;
}

size_t ransac_res_bytes(int C, long long tot) { return sizeof(double) * RANSAC_RES * C + tot; }
size_t ransac_hyp_smem() { return sizeof(double) * RS_N * RANSAC_HYP_THREADS; }

// PnP RANSAC of the armed cameras on the staged inputs: hypotheses, scores, selection (which rewrites the records'
// R0, t0 it replaces), and the results' read-back.  Enqueued after the inputs' copy and before the solve.
int enqueue_ransac(cosl_pose_solver* s, int C, long long tot) {
  PoseCam* d_cams = section<PoseCam>(s->d_in, s->lay.cams);
  const double* d_M = section<const double>(s->d_in, s->lay.M);
  const double* d_m = section<const double>(s->d_in, s->lay.m);
  cudaStream_t st = s->rq.stream;
  const int nh = s->rHyp;
  double* d_res = reinterpret_cast<double*>(s->d_rres);
  unsigned char* d_inl = s->d_rres + sizeof(double) * RANSAC_RES * C;
  COSL_LAUNCH(ransac_hyp_kernel, dim3((nh + RANSAC_HYP_THREADS - 1) / RANSAC_HYP_THREADS, C), RANSAC_HYP_THREADS,
              ransac_hyp_smem(), st, d_cams, d_M, d_m, s->d_ruse, nh, s->rSeed, s->d_rhyp, s->d_rsmp);
  COSL_CUDA(cudaGetLastError());
  COSL_LAUNCH(ransac_score_kernel, dim3(nh / RANSAC_SCORE_THREADS + 1, C), RANSAC_SCORE_THREADS, 0, st, d_cams, d_M,
              d_m, s->d_ruse, nh, s->d_rhyp, s->rThr, s->d_rcnt, s->d_rsse);
  COSL_CUDA(cudaGetLastError());
  COSL_LAUNCH(ransac_select_kernel, C, RANSAC_SEL_THREADS, 0, st, d_cams, d_M, d_m, s->d_ruse, nh, s->d_rhyp,
              s->d_rcnt, s->d_rsse, s->rThr, s->rMinInl, d_res, d_inl);
  COSL_CUDA(cudaGetLastError());
  COSL_CUDA(cudaMemcpyAsync(s->h_rres, s->d_rres, ransac_res_bytes(C, tot), cudaMemcpyDeviceToHost, st));
  return COSL_OK;
}

// The staged inputs of C cameras and tot points (the sections of s->lay): copy, kernels, read-backs.  s->obsCov
// selects the whitened instantiations, s->prior the PRIOR ones.
int enqueue_solve(cosl_pose_solver* s, int C, long long tot, const PoseCfg& cfg) {
  const PoseLayout& lay = s->lay;
  const PoseCam* d_cams = section<const PoseCam>(s->d_in, lay.cams);
  const double* d_M = section<const double>(s->d_in, lay.M);
  const double* d_m = section<const double>(s->d_in, lay.m);
  const double* d_p = section<const double>(s->d_in, lay.prev);
  const double* d_L = section<const double>(s->d_in, lay.L);
  const PosePriorDev pr{section<const double>(s->d_in, lay.rec), section<const int>(s->d_in, lay.has)};
  cudaStream_t st = s->rq.stream;
  COSL_CUDA(cudaMemcpyAsync(s->d_in, s->h_in, lay.bytes, cudaMemcpyHostToDevice, st));
  if (s->ransac) COSL_TRY(enqueue_ransac(s, C, tot));
  const auto solve = s->obsCov ? (s->prior ? pose_intracam_kernel<true, true> : pose_intracam_kernel<true, false>)
                               : (s->prior ? pose_intracam_kernel<false, true> : pose_intracam_kernel<false, false>);
  COSL_LAUNCH(solve, C, POSE_THREADS, 0, st, d_cams, d_M, d_m, d_p, s->d_W, cfg, s->d_out, d_L, pr);
  COSL_CUDA(cudaGetLastError());
  COSL_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(PoseOut) * C, cudaMemcpyDeviceToHost, st));
  if (s->pixelVar > 0) {
    double* d_res = s->d_cov;
    double* d_err = s->d_cov + POSE_COV_STRIDE * C;
    const auto stage = s->obsCov ? (s->prior ? pose_cov_kernel<true, true> : pose_cov_kernel<true, false>)
                                 : (s->prior ? pose_cov_kernel<false, true> : pose_cov_kernel<false, false>);
    COSL_LAUNCH(stage, C, POSE_THREADS, 0, st, d_cams, d_M, d_m, s->d_out, cfg.tau, s->pixelVar, d_res, d_err, d_L,
                pr);
    COSL_CUDA(cudaGetLastError());
    COSL_CUDA(cudaMemcpyAsync(s->h_cov, s->d_cov, sizeof(double) * cov_doubles(C, tot), cudaMemcpyDeviceToHost, st));
    if (s->map && s->nblk > 0) {  // submit_mappts requires an armed handle
      COSL_LAUNCH(pose_mappt_kernel, s->nblk, MAPPT_THREADS, 0, st, section<const int4>(s->d_in, lay.blk),
                  section<const double>(s->d_in, lay.map), d_cams, s->d_out, d_res, s->gate, s->d_mres);
      COSL_CUDA(cudaGetLastError());
      COSL_CUDA(cudaMemcpyAsync(s->h_mres, s->d_mres, sizeof(double) * MAPPT_OUT * s->nmap, cudaMemcpyDeviceToHost,
                                st));
    }
  }
  return COSL_OK;
}

// cosl_pose_solver_submit (covx == prior == mp == nullptr), cosl_pose_solver_submit_cov (prior == mp == nullptr),
// cosl_pose_solver_submit_prior (mp == nullptr) and cosl_pose_solver_submit_mappts; fn names the caller in messages.
int submit_solve(const char* fn, cosl_pose_solver* s, int C, const double* K9, const double* R0, const double* t0,
                 const int* npts, const double* const* Ms, const double* const* ms, const double* const* covx,
                 const double* const* prior, const double* const* prevErrs, double tau, const cosl_pose_opt* opts,
                 const MapPtsArgs* mp = nullptr) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle(fn));
  if (C < 1 || !K9 || !R0 || !t0 || !npts || !Ms || !ms || !opts)
    return set_error(COSL_E_INVALID, "%s: null argument", fn);
  if (C > s->maxCams)
    return set_error(COSL_E_INVALID, "%s: %d cameras exceed the handle's %d", fn, C, s->maxCams);
  long long tot = 0;
  if (s->rC > 0 && C != s->rC)
    return set_error(COSL_E_INVALID, "%s: %d cameras, but RANSAC is armed for %d (set_ransac)", fn, C, s->rC);
  COSL_TRY(check_cameras(fn, C, npts, Ms, ms, opts, &tot));
  if (tot > s->maxPts)
    return set_error(COSL_E_INVALID, "%s: %lld points exceed the handle's %d", fn, tot, s->maxPts);
  COSL_TRY(check_covx(fn, C, npts, covx));
  bool anyPrior = false;
  COSL_TRY(check_priors(fn, C, prior, &anyPrior));
  long long nmap = 0;
  if (mp) {
    if (!(s->pixelVar > 0)) return set_error(COSL_E_STATE, "%s: the handle is not armed (set_covariance)", fn);
    if (s->maxMap < 1) return set_error(COSL_E_STATE, "%s: no map points reserved (reserve_mappts)", fn);
    COSL_TRY(check_mappts(fn, C, s->maxMap, *mp, &nmap));
  }
  COSL_CUDA(cudaSetDevice(s->device));
  int nblk = 0;  // one CTA of pose_mappt_kernel per MAPPT_THREADS map points of a camera
  if (mp)
    for (int c = 0; c < C; ++c) nblk += div_up(mp->n[c], MAPPT_THREADS);
  const PoseLayout lay = pose_layout(C, tot, covx != nullptr, anyPrior, nmap, nblk);
  // nothing is in flight, so no copy reads the staging buffer any more
  PoseCam* cams = section<PoseCam>(s->h_in, lay.cams);
  double* hM = section<double>(s->h_in, lay.M);
  double* hm = section<double>(s->h_in, lay.m);
  double* hp = section<double>(s->h_in, lay.prev);
  double* hL = section<double>(s->h_in, lay.L);
  long long off = 0;
  for (int c = 0; c < C; ++c) {
    std::memcpy(cams[c].K, K9 + 9 * c, sizeof(double) * 9);
    std::memcpy(cams[c].R0, R0 + 9 * c, sizeof(double) * 9);
    std::memcpy(cams[c].t0, t0 + 3 * c, sizeof(double) * 3);
    cams[c].npts = npts[c];
    cams[c].hasPrev = (prevErrs && prevErrs[c]) ? 1 : 0;
    cams[c].off = off;
    if (npts[c]) {
      std::memcpy(hM + 3 * off, Ms[c], sizeof(double) * 3 * npts[c]);
      std::memcpy(hm + 2 * off, ms[c], sizeof(double) * 2 * npts[c]);
      // a camera without prevErrs leaves its slice unset: the kernel does not read it
      if (cams[c].hasPrev) std::memcpy(hp + off, prevErrs[c], sizeof(double) * npts[c]);
      // a camera without covariances gets the identity factor {1, -0, 1}, whitening it bit for bit to nothing
      if (covx)
        for (int i = 0; i < npts[c]; ++i) {
          double* L = hL + 3 * (off + i);
          if (covx[c]) {
            cov_factor(covx[c] + 4 * (size_t)i, L);
          } else {
            L[0] = 1.0;
            L[1] = -0.0;
            L[2] = 1.0;
          }
        }
    }
    off += npts[c];
  }
  if (anyPrior) {
    double* hq = section<double>(s->h_in, lay.rec);
    int* hh = section<int>(s->h_in, lay.has);
    for (int c = 0; c < C; ++c) {
      hh[c] = prior[c] ? 1 : 0;
      // a camera without a prior leaves its record unset: the kernels do not read it
      if (prior[c]) prior_factor(fn, c, prior[c], hq + POSE_PRIOR_REC * (size_t)c);
    }
  }
  if (mp) {  // records camera-major, then the CTA table
    double* hr = section<double>(s->h_in, lay.map);
    int4* hb = section<int4>(s->h_in, lay.blk);
    long long j = 0;
    int b = 0;
    for (int c = 0; c < C; ++c) {
      for (int i = 0; i < mp->n[c]; ++i) {
        double* r = hr + (size_t)MAPPT_IN * (j + i);
        std::memcpy(r, mp->X[c] + 3 * (size_t)i, sizeof(double) * 3);
        const double* P = mp->P[c] + 9 * (size_t)i;  // symmetrised, as point_cov checked it
        r[3] = P[0];
        r[4] = 0.5 * (P[1] + P[3]);
        r[5] = 0.5 * (P[2] + P[6]);
        r[6] = P[4];
        r[7] = 0.5 * (P[5] + P[7]);
        r[8] = P[8];
        std::memcpy(r + 9, mp->m[c] + 2 * (size_t)i, sizeof(double) * 2);
        pack_cov2((mp->cov && mp->cov[c]) ? mp->cov[c] + 4 * (size_t)i : nullptr, s->pixelVar, r + 11);
      }
      for (int i = 0; i < mp->n[c]; i += MAPPT_THREADS)
        hb[b++] = make_int4(c, (int)(j + i), (int)(j + std::min(i + MAPPT_THREADS, mp->n[c])), 0);
      j += mp->n[c];
    }
  }
  PoseCfg cfg;
  cfg.maxIterLM = opts[0].maxIterLM;
  cfg.maxIterRW = opts[0].maxIterRW;
  cfg.epsErr = opts[0].epsErrorChangeLM;
  cfg.epsParam = opts[0].epsParamChangeLM;
  cfg.epsRW = opts[0].epsErrorChangeRW;
  cfg.lambda0 = opts[0].lambda0;
  cfg.tau = tau;
  s->C = C;
  s->tot = tot;
  s->lay = lay;
  s->covReady = false;
  s->obsCov = covx != nullptr;
  s->prior = anyPrior;
  s->map = mp != nullptr;
  s->mapReady = false;
  s->nmap = nmap;
  s->nblk = nblk;
  s->gate = mp ? mp->gate : 0.0;
  s->ransac = s->rC > 0;
  s->ransacReady = false;
  if (s->ransac) {
    s->ransacHyps = true;
    s->rHypRun = s->rHyp;
  }
  COSL_TRY(s->rq.submit(fn, [&]() { return enqueue_solve(s, C, tot, cfg); }));
  s->covReady = s->pixelVar > 0;
  s->mapReady = s->map;
  s->ransacReady = s->ransac;
  return COSL_OK;
}

}  // namespace

// A triangulation handle (cosl_tri_solver).  The inputs of one submit travel in one copy from a pinned staging buffer
// in the sections of tri_layout, TriCam[nCams] | views[nViews][TRI_VIEW] | viewOff[nPts + 1] | viewCam[nViews];
// TRI_OUT doubles per point come back into pinned memory.  Everything, the per-view scratch included, is allocated by
// create for at most maxCams camera entries, maxPts points and maxViews views per submit.
struct cosl_tri_solver {
  int device = 0, maxCams = 0, maxPts = 0, maxViews = 0;
  RequestStream rq;
  unsigned char* h_in = nullptr;
  unsigned char* d_in = nullptr;
  double* d_scratch = nullptr;
  double* d_out = nullptr;
  double* h_out = nullptr;
  int* seen = nullptr;  // [maxCams]: the last point that used each camera entry, for the repeated-camera check
  int nPts = 0;         // points of the submit in flight or last collected
};

namespace {

// The sections of a triangulation submit's staging buffer and its device copy
struct TriLayout {
  size_t cams, views, viewOff, viewCam, bytes;
};

TriLayout tri_layout(int nCams, int nPts, int nViews) {
  SlabLayout S;
  TriLayout o;
  o.cams = S.take(sizeof(TriCam) * nCams);
  o.views = S.take(sizeof(double) * TRI_VIEW * nViews);
  o.viewOff = S.take(sizeof(int) * ((size_t)nPts + 1));
  o.viewCam = S.take(sizeof(int) * (size_t)nViews);
  o.bytes = S.bytes;
  return o;
}

void free_tri_solver(cosl_tri_solver* s) {
  cudaSetDevice(s->device);
  s->rq.destroy();
  if (s->h_in) cudaFreeHost(s->h_in);
  if (s->h_out) cudaFreeHost(s->h_out);
  cudaFree(s->d_in);
  cudaFree(s->d_scratch);
  cudaFree(s->d_out);
  delete[] s->seen;
  delete s;
}

int alloc_tri_solver(cosl_tri_solver* s) {
  s->seen = new (std::nothrow) int[s->maxCams];
  if (!s->seen) return set_error(COSL_E_NOMEM, "cosl_tri_solver_create: out of host memory");
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.create());
  const size_t in = tri_layout(s->maxCams, s->maxPts, s->maxViews).bytes;
  const size_t outb = sizeof(double) * TRI_OUT * s->maxPts;
  COSL_CUDA(cudaHostAlloc(&s->h_in, in, cudaHostAllocPortable));
  COSL_CUDA(cudaHostAlloc(&s->h_out, outb, cudaHostAllocPortable));
  COSL_CUDA(cudaMalloc(&s->d_in, in));
  COSL_CUDA(cudaMalloc(&s->d_scratch, sizeof(double) * TRI_SCRATCH * s->maxViews));
  COSL_CUDA(cudaMalloc(&s->d_out, outb));
  return COSL_OK;
}

// Checks a camera table of the triangulation and registration handles: K, R and t finite, R a rotation and camCov[c]
// (nullable, as camCov[c]) symmetric and positive definite, the rules of a pose prior (R, t, P), naming the first bad
// camera.
int check_cam_table(const char* fn, int nCams, const double* K9, const double* R, const double* t,
                    const double* const* camCov) {
  for (int c = 0; c < nCams; ++c) {
    for (int k = 0; k < 9; ++k)
      if (!std::isfinite(K9[9 * c + k]) || !std::isfinite(R[9 * c + k]) || (k < 3 && !std::isfinite(t[3 * c + k])))
        return set_error(COSL_E_INVALID, "%s: K, R or t of camera %d is not finite", fn, c);
    // R a rotation and camCov symmetric and positive definite: the rules of a pose prior (R, t, P)
    double rec[48] = {};
    std::memcpy(rec, R + 9 * c, sizeof(double) * 9);
    std::memcpy(rec + 9, t + 3 * c, sizeof(double) * 3);
    if (camCov && camCov[c]) std::memcpy(rec + 12, camCov[c], sizeof(double) * 36);
    else for (int k = 0; k < 6; ++k) rec[12 + 7 * k] = 1.0;
    COSL_TRY(prior_factor(fn, c, rec, nullptr));
  }
  return COSL_OK;
}

// Checks one submit on the calling thread, naming the first bad camera, point or view.
int check_tri(const char* fn, cosl_tri_solver* s, int nCams, const double* K9, const double* R, const double* t,
              const double* const* camCov, int nPts, const int* viewOff, const int* viewCam, const double* m,
              const double* covm, double pixel_var, double max_err) {
  if (nCams < 0 || nPts < 0) return set_error(COSL_E_INVALID, "%s: nCams %d or nPts %d < 0", fn, nCams, nPts);
  if (nCams > s->maxCams)
    return set_error(COSL_E_INVALID, "%s: %d cameras exceed the handle's %d", fn, nCams, s->maxCams);
  if (nPts > s->maxPts)
    return set_error(COSL_E_INVALID, "%s: %d points exceed the handle's %d", fn, nPts, s->maxPts);
  if (!viewOff || (nCams > 0 && (!K9 || !R || !t)) || (nPts > 0 && (!viewCam || !m)))
    return set_error(COSL_E_INVALID, "%s: null argument", fn);
  if (!std::isfinite(pixel_var) || !(pixel_var > 0))
    return set_error(COSL_E_INVALID, "%s: pixel_var %g is not a finite value > 0", fn, pixel_var);
  if (!(max_err > 0)) return set_error(COSL_E_INVALID, "%s: max_err %g is not > 0", fn, max_err);
  COSL_TRY(check_cam_table(fn, nCams, K9, R, t, camCov));
  if (viewOff[0] != 0) return set_error(COSL_E_INVALID, "%s: viewOff[0] = %d is not 0", fn, viewOff[0]);
  for (int c = 0; c < nCams; ++c) s->seen[c] = -1;
  for (int j = 0; j < nPts; ++j) {
    const int n = viewOff[j + 1] - viewOff[j];
    if (viewOff[j + 1] < viewOff[j] || n < 2 || n > TRI_MAX_VIEWS)
      return set_error(COSL_E_INVALID, "%s: point %d has %d views, not 2 to %d", fn, j, n, TRI_MAX_VIEWS);
    if (viewOff[j + 1] > s->maxViews)
      return set_error(COSL_E_INVALID, "%s: point %d: %d views exceed the handle's %d", fn, j, viewOff[j + 1],
                       s->maxViews);
    for (int v = viewOff[j]; v < viewOff[j + 1]; ++v) {
      const int c = viewCam[v];
      if (c < 0 || c >= nCams)
        return set_error(COSL_E_INVALID, "%s: view %d of point %d: camera %d is not in [0, %d)", fn, v, j, c, nCams);
      if (s->seen[c] == j)
        return set_error(COSL_E_INVALID, "%s: view %d of point %d: camera %d is used twice", fn, v, j, c);
      s->seen[c] = j;
      if (!std::isfinite(m[2 * (size_t)v]) || !std::isfinite(m[2 * (size_t)v + 1]))
        return set_error(COSL_E_INVALID, "%s: view %d of point %d: m is not finite", fn, v, j);
      double L[3];
      if (covm && !cov_factor(covm + 4 * (size_t)v, L))
        return set_error(COSL_E_INVALID, "%s: view %d of point %d: covm is not finite, symmetric and positive definite",
                         fn, v, j);
    }
  }
  return COSL_OK;
}

// Stages a checked submit and enqueues the copy, tri_kernel and the read-back.
int stage_tri(cosl_tri_solver* s, int nCams, const double* K9, const double* R, const double* t,
              const double* const* camCov, int nPts, const int* viewOff, const int* viewCam, const double* m,
              const double* covm, double pixel_var, double max_err) {
  const int nViews = viewOff[nPts];
  const TriLayout lay = tri_layout(nCams, nPts, nViews);
  TriCam* hc = section<TriCam>(s->h_in, lay.cams);
  double* hv = section<double>(s->h_in, lay.views);
  for (int c = 0; c < nCams; ++c) {
    TriCam& e = hc[c];
    const double* k = K9 + 9 * c;
    std::memcpy(e.K, k, sizeof(double) * 9);
    std::memcpy(e.R, R + 9 * c, sizeof(double) * 9);
    std::memcpy(e.t, t + 3 * c, sizeof(double) * 3);
    // K^-1 by the adjugate; a singular K gives non-finite rays and status 4
    const double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) +
                       k[2] * (k[3] * k[7] - k[4] * k[6]);
    const double adj[9] = {k[4] * k[8] - k[5] * k[7], k[2] * k[7] - k[1] * k[8], k[1] * k[5] - k[2] * k[4],
                           k[5] * k[6] - k[3] * k[8], k[0] * k[8] - k[2] * k[6], k[2] * k[3] - k[0] * k[5],
                           k[3] * k[7] - k[4] * k[6], k[1] * k[6] - k[0] * k[7], k[0] * k[4] - k[1] * k[3]};
    for (int i = 0; i < 9; ++i) e.Ki[i] = adj[i] / det;
    e.hasP = camCov && camCov[c] ? 1 : 0;
    e.pad = 0;
    if (e.hasP) sym6(camCov[c], e.P);  // symmetrised, as prior_factor checked it
  }
  for (int v = 0; v < nViews; ++v) {
    double* q = hv + (size_t)TRI_VIEW * v;
    q[0] = m[2 * (size_t)v];
    q[1] = m[2 * (size_t)v + 1];
    pack_cov2(covm ? covm + 4 * (size_t)v : nullptr, pixel_var, q + 2);
  }
  std::memcpy(section<int>(s->h_in, lay.viewOff), viewOff, sizeof(int) * ((size_t)nPts + 1));
  if (nViews) std::memcpy(section<int>(s->h_in, lay.viewCam), viewCam, sizeof(int) * (size_t)nViews);
  s->nPts = nPts;
  cudaStream_t st = s->rq.stream;
  return s->rq.submit("cosl_tri_solver_submit", [&]() -> int {
    COSL_CUDA(cudaMemcpyAsync(s->d_in, s->h_in, lay.bytes, cudaMemcpyHostToDevice, st));
    if (nPts > 0) {
      COSL_LAUNCH(tri_kernel, div_up(nPts, TRI_THREADS), TRI_THREADS, 0, st, section<const TriCam>(s->d_in, lay.cams),
                  section<const double>(s->d_in, lay.views), section<const int>(s->d_in, lay.viewOff),
                  section<const int>(s->d_in, lay.viewCam), nPts, max_err, s->d_scratch, s->d_out);
      COSL_CUDA(cudaGetLastError());
      COSL_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * TRI_OUT * nPts, cudaMemcpyDeviceToHost, st));
    }
    return COSL_OK;
  });
}

}  // namespace

// A registration handle (cosl_assoc_solver).  The inputs of one submit travel in one copy from a pinned staging buffer
// in the sections of assoc_layout, AssocCam[nCams] | pts[nPts][ASSOC_PT] | feats[nFeats][ASSOC_FEAT] | trkM[nTrk][2] |
// featOff[nCams + 1] | cell[nFeats] | owned[nFeats] | trkOff[nFeats + 1] | trkCam[nTrk] | qPt[nQ] | qCam[nQ];
// ASSOC_OUT doubles per query pair come back into pinned memory.  The grid (count and start per cell, the features
// sorted by cell) and the claim keys live on the device only.  Everything is allocated by create for at most maxCams
// camera entries, maxPts points, maxQueries query pairs, maxFeats features and maxTrackObs track observations per
// submit.
struct cosl_assoc_solver {
  int device = 0, maxCams = 0, maxPts = 0, maxQueries = 0, maxFeats = 0, maxTrackObs = 0;
  RequestStream rq;
  unsigned char* h_in = nullptr;
  unsigned char* d_in = nullptr;
  int* d_count = nullptr;   // [maxCams * ASSOC_MAX_CELLS]
  int* d_start = nullptr;   // [maxCams * ASSOC_MAX_CELLS + 1]
  int* d_sorted = nullptr;  // [maxFeats]
  unsigned long long* d_key = nullptr;  // [maxFeats]: pass one of the claims, the least d2 bits per feature
  unsigned int* d_win = nullptr;        // [maxFeats]: pass two, the least point index among those holding it
  double* d_out = nullptr;
  double* h_out = nullptr;
  int* seen = nullptr;  // [maxCams]: the last point that queried each camera entry, for the repeated-entry check
  int nQ = 0;           // query pairs of the submit in flight or last collected
};

namespace {

// The sections of a registration submit's staging buffer and its device copy
struct AssocLayout {
  size_t cams, pts, feats, trkM, featOff, cell, owned, trkOff, trkCam, qPt, qCam, bytes;
};

AssocLayout assoc_layout(int nCams, int nPts, int nFeats, int nTrk, int nQ) {
  SlabLayout S;
  AssocLayout o;
  o.cams = S.take(sizeof(AssocCam) * nCams);
  o.pts = S.take(sizeof(double) * ASSOC_PT * nPts);
  o.feats = S.take(sizeof(double) * ASSOC_FEAT * nFeats);
  o.trkM = S.take(sizeof(double) * 2 * nTrk);
  o.featOff = S.take(sizeof(int) * ((size_t)nCams + 1));
  o.cell = S.take(sizeof(int) * nFeats);
  o.owned = S.take(sizeof(int) * nFeats);
  o.trkOff = S.take(sizeof(int) * ((size_t)nFeats + 1));
  o.trkCam = S.take(sizeof(int) * nTrk);
  o.qPt = S.take(sizeof(int) * nQ);
  o.qCam = S.take(sizeof(int) * nQ);
  o.bytes = S.bytes;
  return o;
}

void free_assoc_solver(cosl_assoc_solver* s) {
  cudaSetDevice(s->device);
  s->rq.destroy();
  if (s->h_in) cudaFreeHost(s->h_in);
  if (s->h_out) cudaFreeHost(s->h_out);
  cudaFree(s->d_in);
  cudaFree(s->d_count);
  cudaFree(s->d_start);
  cudaFree(s->d_sorted);
  cudaFree(s->d_key);
  cudaFree(s->d_win);
  cudaFree(s->d_out);
  delete[] s->seen;
  delete s;
}

int alloc_assoc_solver(cosl_assoc_solver* s) {
  s->seen = new (std::nothrow) int[s->maxCams];
  if (!s->seen) return set_error(COSL_E_NOMEM, "cosl_assoc_solver_create: out of host memory");
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.create());
  const size_t in = assoc_layout(s->maxCams, s->maxPts, s->maxFeats, s->maxTrackObs, s->maxQueries).bytes;
  const size_t outb = sizeof(double) * ASSOC_OUT * s->maxQueries;
  const size_t cells = (size_t)s->maxCams * ASSOC_MAX_CELLS;
  COSL_CUDA(cudaHostAlloc(&s->h_in, in, cudaHostAllocPortable));
  COSL_CUDA(cudaHostAlloc(&s->h_out, outb, cudaHostAllocPortable));
  COSL_CUDA(cudaMalloc(&s->d_in, in));
  COSL_CUDA(cudaMalloc(&s->d_count, sizeof(int) * cells));
  COSL_CUDA(cudaMalloc(&s->d_start, sizeof(int) * (cells + 1)));
  COSL_CUDA(cudaMalloc(&s->d_sorted, sizeof(int) * s->maxFeats));
  COSL_CUDA(cudaMalloc(&s->d_key, sizeof(unsigned long long) * s->maxFeats));
  COSL_CUDA(cudaMalloc(&s->d_win, sizeof(unsigned int) * s->maxFeats));
  COSL_CUDA(cudaMalloc(&s->d_out, outb));
  return COSL_OK;
}

// The arguments of one cosl_assoc_solver_submit
struct AssocArgs {
  int nCams;
  const double *K9, *R, *t;
  const double* const* camCov;
  const int* wh;
  const int* featOff;
  const double *mf, *covf;
  const int* owned;
  const int *trkOff, *trkCam;
  const double* trkM;
  int nPts;
  const double *X, *PX;
  const int *qOff, *qCam;
  double pixel_var, gate, track_gate;
};

// Checks one submit on the calling thread, naming the first bad camera, feature, track observation, point or query.
int check_assoc(const char* fn, cosl_assoc_solver* s, const AssocArgs& a) {
  const int nCams = a.nCams, nPts = a.nPts;
  if (nCams < 0 || nPts < 0) return set_error(COSL_E_INVALID, "%s: nCams %d or nPts %d < 0", fn, nCams, nPts);
  if (nCams > s->maxCams)
    return set_error(COSL_E_INVALID, "%s: %d cameras exceed the handle's %d", fn, nCams, s->maxCams);
  if (nPts > s->maxPts)
    return set_error(COSL_E_INVALID, "%s: %d points exceed the handle's %d", fn, nPts, s->maxPts);
  if (!a.featOff || !a.qOff || (nCams > 0 && (!a.K9 || !a.R || !a.t || !a.wh)) || (nPts > 0 && (!a.X || !a.PX)))
    return set_error(COSL_E_INVALID, "%s: null argument", fn);
  if (!std::isfinite(a.pixel_var) || !(a.pixel_var > 0))
    return set_error(COSL_E_INVALID, "%s: pixel_var %g is not a finite value > 0", fn, a.pixel_var);
  if (!(a.gate > 0)) return set_error(COSL_E_INVALID, "%s: gate %g is not > 0", fn, a.gate);
  if (!(a.track_gate > 0)) return set_error(COSL_E_INVALID, "%s: track_gate %g is not > 0", fn, a.track_gate);
  COSL_TRY(check_cam_table(fn, nCams, a.K9, a.R, a.t, a.camCov));
  for (int c = 0; c < nCams; ++c)
    if (a.wh[2 * c] < 1 || a.wh[2 * c] > ASSOC_MAX_SIDE || a.wh[2 * c + 1] < 1 || a.wh[2 * c + 1] > ASSOC_MAX_SIDE)
      return set_error(COSL_E_INVALID, "%s: image size %d x %d of camera %d is not in [1, %d]", fn, a.wh[2 * c],
                       a.wh[2 * c + 1], c, ASSOC_MAX_SIDE);
  if (a.featOff[0] != 0) return set_error(COSL_E_INVALID, "%s: featOff[0] = %d is not 0", fn, a.featOff[0]);
  for (int c = 0; c < nCams; ++c)
    if (a.featOff[c + 1] < a.featOff[c])
      return set_error(COSL_E_INVALID, "%s: camera %d has %d features", fn, c, a.featOff[c + 1] - a.featOff[c]);
  const int nF = a.featOff[nCams];
  if (nF > s->maxFeats)
    return set_error(COSL_E_INVALID, "%s: %d features exceed the handle's %d", fn, nF, s->maxFeats);
  if (nF > 0 && !a.mf) return set_error(COSL_E_INVALID, "%s: null argument", fn);
  if (a.trkOff) {
    if (a.trkOff[0] != 0) return set_error(COSL_E_INVALID, "%s: trkOff[0] = %d is not 0", fn, a.trkOff[0]);
    for (int f = 0; f < nF; ++f)
      if (a.trkOff[f + 1] < a.trkOff[f])
        return set_error(COSL_E_INVALID, "%s: feature %d has %d track observations", fn, f,
                         a.trkOff[f + 1] - a.trkOff[f]);
    if (a.trkOff[nF] > s->maxTrackObs)
      return set_error(COSL_E_INVALID, "%s: %d track observations exceed the handle's %d", fn, a.trkOff[nF],
                       s->maxTrackObs);
    if (a.trkOff[nF] > 0 && (!a.trkCam || !a.trkM)) return set_error(COSL_E_INVALID, "%s: null argument", fn);
  }
  for (int f = 0; f < nF; ++f) {
    if (!std::isfinite(a.mf[2 * (size_t)f]) || !std::isfinite(a.mf[2 * (size_t)f + 1]))
      return set_error(COSL_E_INVALID, "%s: feature %d: m is not finite", fn, f);
    double L[3];
    if (a.covf && !cov_factor(a.covf + 4 * (size_t)f, L))
      return set_error(COSL_E_INVALID, "%s: feature %d: covf is not finite, symmetric and positive definite", fn, f);
    if (a.owned && a.owned[f] != 0 && a.owned[f] != 1)
      return set_error(COSL_E_INVALID, "%s: feature %d: owned %d is not 0 or 1", fn, f, a.owned[f]);
    for (int k = a.trkOff ? a.trkOff[f] : 0; a.trkOff && k < a.trkOff[f + 1]; ++k) {
      const int c = a.trkCam[k];
      if (c < 0 || c >= nCams)
        return set_error(COSL_E_INVALID, "%s: track observation %d of feature %d: camera %d is not in [0, %d)", fn,
                         k, f, c, nCams);
      if (!std::isfinite(a.trkM[2 * (size_t)k]) || !std::isfinite(a.trkM[2 * (size_t)k + 1]))
        return set_error(COSL_E_INVALID, "%s: track observation %d of feature %d: m is not finite", fn, k, f);
    }
  }
  for (int j = 0; j < nPts; ++j) {
    const double* X = a.X + 3 * (size_t)j;
    if (!std::isfinite(X[0]) || !std::isfinite(X[1]) || !std::isfinite(X[2]))
      return set_error(COSL_E_INVALID, "%s: point %d: X is not finite", fn, j);
    double S[6];
    if (!point_cov(a.PX + 9 * (size_t)j, S))
      return set_error(COSL_E_INVALID, "%s: point %d: P is not finite, symmetric and positive definite", fn, j);
  }
  if (a.qOff[0] != 0) return set_error(COSL_E_INVALID, "%s: qOff[0] = %d is not 0", fn, a.qOff[0]);
  for (int c = 0; c < nCams; ++c) s->seen[c] = -1;
  for (int j = 0; j < nPts; ++j) {
    const int n = a.qOff[j + 1] - a.qOff[j];
    if (a.qOff[j + 1] < a.qOff[j] || n > ASSOC_MAX_QUERIES)
      return set_error(COSL_E_INVALID, "%s: point %d has %d queries, not 0 to %d", fn, j, n, ASSOC_MAX_QUERIES);
    if (a.qOff[j + 1] > s->maxQueries)
      return set_error(COSL_E_INVALID, "%s: point %d: %d queries exceed the handle's %d", fn, j, a.qOff[j + 1],
                       s->maxQueries);
    if (n > 0 && !a.qCam) return set_error(COSL_E_INVALID, "%s: null argument", fn);
    for (int q = a.qOff[j]; q < a.qOff[j + 1]; ++q) {
      const int c = a.qCam[q];
      if (c < 0 || c >= nCams)
        return set_error(COSL_E_INVALID, "%s: query %d of point %d: camera %d is not in [0, %d)", fn, q, j, c, nCams);
      if (s->seen[c] == j)
        return set_error(COSL_E_INVALID, "%s: query %d of point %d: camera %d is queried twice", fn, q, j, c);
      s->seen[c] = j;
    }
  }
  return COSL_OK;
}

// Stages a checked submit and enqueues the copy, the binning, the search, the claims and the read-back.
int stage_assoc(cosl_assoc_solver* s, const AssocArgs& a) {
  const int nCams = a.nCams, nPts = a.nPts, nF = a.featOff[nCams];
  const int nTrk = a.trkOff ? a.trkOff[nF] : 0, nQ = a.qOff[nPts];
  const AssocLayout lay = assoc_layout(nCams, nPts, nF, nTrk, nQ);
  AssocCam* hc = section<AssocCam>(s->h_in, lay.cams);
  double* hp = section<double>(s->h_in, lay.pts);
  double* hf = section<double>(s->h_in, lay.feats);
  int* hcell = section<int>(s->h_in, lay.cell);
  int* hown = section<int>(s->h_in, lay.owned);
  int* htoff = section<int>(s->h_in, lay.trkOff);
  int* hqpt = section<int>(s->h_in, lay.qPt);
  int cells = 0;
  for (int c = 0; c < nCams; ++c) {
    AssocCam& e = hc[c];
    std::memcpy(e.K, a.K9 + 9 * c, sizeof(double) * 9);
    std::memcpy(e.R, a.R + 9 * c, sizeof(double) * 9);
    std::memcpy(e.t, a.t + 3 * c, sizeof(double) * 3);
    e.hasP = a.camCov && a.camCov[c] ? 1 : 0;
    if (e.hasP) sym6(a.camCov[c], e.P);  // symmetrised, as prior_factor checked it
    e.W = a.wh[2 * c];
    e.H = a.wh[2 * c + 1];
    e.nx = (a.wh[2 * c] + ASSOC_CELL - 1) / ASSOC_CELL;
    e.ny = (a.wh[2 * c + 1] + ASSOC_CELL - 1) / ASSOC_CELL;
    e.cell0 = cells;
    cells += e.nx * e.ny;
    // the features: m_f, Sigma_f (pixel_var I without covf), the cell and lam = the largest lambda_max(Sigma_f)
    double lam = 0.0;
    for (int f = a.featOff[c]; f < a.featOff[c + 1]; ++f) {
      double* q = hf + (size_t)ASSOC_FEAT * f;
      q[0] = a.mf[2 * (size_t)f];
      q[1] = a.mf[2 * (size_t)f + 1];
      pack_cov2(a.covf ? a.covf + 4 * (size_t)f : nullptr, a.pixel_var, q + 2);
      const double h = 0.5 * (q[2] - q[4]);
      lam = std::max(lam, 0.5 * (q[2] + q[4]) + std::sqrt(h * h + q[3] * q[3]));
      const double cx = std::max(0.0, std::min(e.nx - 1.0, std::floor(q[0] / ASSOC_CELL)));
      const double cy = std::max(0.0, std::min(e.ny - 1.0, std::floor(q[1] / ASSOC_CELL)));
      hcell[f] = e.cell0 + (int)cy * e.nx + (int)cx;
    }
    e.lam = lam;
  }
  for (int j = 0; j < nPts; ++j) {
    double* p = hp + (size_t)ASSOC_PT * j;
    std::memcpy(p, a.X + 3 * (size_t)j, sizeof(double) * 3);
    point_cov(a.PX + 9 * (size_t)j, p + 3);  // symmetrised, as check_assoc accepted it
    for (int q = a.qOff[j]; q < a.qOff[j + 1]; ++q) hqpt[q] = j;
  }
  if (nTrk) std::memcpy(section<double>(s->h_in, lay.trkM), a.trkM, sizeof(double) * 2 * (size_t)nTrk);
  std::memcpy(section<int>(s->h_in, lay.featOff), a.featOff, sizeof(int) * ((size_t)nCams + 1));
  for (int f = 0; f < nF; ++f) hown[f] = a.owned ? a.owned[f] : 0;
  if (a.trkOff) std::memcpy(htoff, a.trkOff, sizeof(int) * ((size_t)nF + 1));
  else std::fill(htoff, htoff + nF + 1, 0);
  if (nTrk) std::memcpy(section<int>(s->h_in, lay.trkCam), a.trkCam, sizeof(int) * (size_t)nTrk);
  if (nQ) std::memcpy(section<int>(s->h_in, lay.qCam), a.qCam, sizeof(int) * (size_t)nQ);
  s->nQ = nQ;
  cudaStream_t st = s->rq.stream;
  const double pv = a.pixel_var, gate = a.gate, tg = a.track_gate;
  return s->rq.submit("cosl_assoc_solver_submit", [&]() -> int {
    COSL_CUDA(cudaMemcpyAsync(s->d_in, s->h_in, lay.bytes, cudaMemcpyHostToDevice, st));
    if (nQ == 0) return COSL_OK;
    const AssocCam* d_cams = section<const AssocCam>(s->d_in, lay.cams);
    const int* d_cell = section<const int>(s->d_in, lay.cell);
    const int* d_qpt = section<const int>(s->d_in, lay.qPt);
    // the grid: count, a per-entry exclusive scan, scatter
    COSL_CUDA(cudaMemsetAsync(s->d_count, 0, sizeof(int) * (size_t)cells, st));
    if (nF) COSL_LAUNCH(assoc_count_kernel, div_up(nF, ASSOC_BIN_THREADS), ASSOC_BIN_THREADS, 0, st, d_cell, nF,
                        s->d_count);
    COSL_LAUNCH(assoc_scan_kernel, nCams, ASSOC_SCAN_THREADS, 0, st, d_cams, section<const int>(s->d_in, lay.featOff),
                nCams, s->d_count, s->d_start);
    if (nF) {
      COSL_LAUNCH(assoc_scatter_kernel, div_up(nF, ASSOC_BIN_THREADS), ASSOC_BIN_THREADS, 0, st, d_cell, nF,
                  s->d_start, s->d_count, s->d_sorted);
      COSL_CUDA(cudaMemsetAsync(s->d_key, 0xff, sizeof(unsigned long long) * (size_t)nF, st));
      COSL_CUDA(cudaMemsetAsync(s->d_win, 0xff, sizeof(unsigned int) * (size_t)nF, st));
    }
    // the search with pass one of the claims, pass two, and the statuses
    COSL_LAUNCH(assoc_search_kernel, div_up(nQ, ASSOC_THREADS), ASSOC_THREADS, 0, st, d_cams,
                section<const double>(s->d_in, lay.pts), section<const double>(s->d_in, lay.feats),
                section<const int>(s->d_in, lay.owned), section<const int>(s->d_in, lay.trkOff),
                section<const int>(s->d_in, lay.trkCam), section<const double>(s->d_in, lay.trkM), d_qpt,
                section<const int>(s->d_in, lay.qCam), nQ, s->d_start, s->d_sorted, pv, gate, tg, s->d_key, s->d_out);
    COSL_LAUNCH(assoc_claim_kernel, div_up(nQ, ASSOC_BIN_THREADS), ASSOC_BIN_THREADS, 0, st, d_qpt, nQ, s->d_key,
                s->d_win, s->d_out);
    COSL_LAUNCH(assoc_final_kernel, div_up(nQ, ASSOC_BIN_THREADS), ASSOC_BIN_THREADS, 0, st, d_qpt, nQ, s->d_key,
                s->d_win, s->d_out);
    COSL_CUDA(cudaGetLastError());
    COSL_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(double) * ASSOC_OUT * (size_t)nQ, cudaMemcpyDeviceToHost,
                              st));
    return COSL_OK;
  });
}

}  // namespace

extern "C" {

void cosl_pose_opt_default(cosl_pose_opt* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->maxIterLM = 100;
  o->maxIterRW = 5;
  o->epsErrorChangeLM = 1e-7;
  o->epsParamChangeLM = 1e-6;
  o->epsErrorChangeRW = 1e-6;
  o->lambda0 = 1e-3;
}

int cosl_pose_solver_create(int device, int maxCams, int maxPts, cosl_pose_solver** out) {
  if (!out || device < 0 || maxCams < 1 || maxPts < 0)
    return set_error(COSL_E_INVALID, "cosl_pose_solver_create: bad argument");
  *out = nullptr;
  COSL_TRY(check_device(device));
  cosl_pose_solver* s = new (std::nothrow) cosl_pose_solver;
  if (!s) return set_error(COSL_E_NOMEM, "cosl_pose_solver_create: out of host memory");
  s->device = device;
  s->maxCams = maxCams;
  s->maxPts = maxPts;
  const int rc = alloc_pose_solver(s);
  if (rc != COSL_OK) {
    free_pose_solver(s);
    return rc;
  }
  *out = s;
  return COSL_OK;
}

int cosl_pose_solver_destroy(cosl_pose_solver* s) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  free_pose_solver(s);
  return COSL_OK;
}

int cosl_pose_solver_submit(cosl_pose_solver* s, int C, const double* K9, const double* R0, const double* t0,
                            const int* npts, const double* const* Ms, const double* const* ms,
                            const double* const* prevErrs, double tau, const cosl_pose_opt* opts) {
  return submit_solve("cosl_pose_solver_submit", s, C, K9, R0, t0, npts, Ms, ms, nullptr, nullptr, prevErrs, tau,
                      opts);
}

int cosl_pose_solver_submit_cov(cosl_pose_solver* s, int C, const double* K9, const double* R0, const double* t0,
                                const int* npts, const double* const* Ms, const double* const* ms,
                                const double* const* covx, const double* const* prevErrs, double tau,
                                const cosl_pose_opt* opts) {
  return submit_solve("cosl_pose_solver_submit_cov", s, C, K9, R0, t0, npts, Ms, ms, covx, nullptr, prevErrs, tau,
                      opts);
}

int cosl_pose_solver_submit_prior(cosl_pose_solver* s, int C, const double* K9, const double* R0, const double* t0,
                                  const int* npts, const double* const* Ms, const double* const* ms,
                                  const double* const* covx, const double* const* prior,
                                  const double* const* prevErrs, double tau, const cosl_pose_opt* opts) {
  return submit_solve("cosl_pose_solver_submit_prior", s, C, K9, R0, t0, npts, Ms, ms, covx, prior, prevErrs, tau,
                      opts);
}

int cosl_pose_solver_reserve_mappts(cosl_pose_solver* s, int maxMapPts) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  if (maxMapPts < 0) return set_error(COSL_E_INVALID, "cosl_pose_solver_reserve_mappts: maxMapPts %d < 0", maxMapPts);
  COSL_TRY(s->rq.idle("cosl_pose_solver_reserve_mappts"));
  if (maxMapPts == s->maxMap) return COSL_OK;
  COSL_CUDA(cudaSetDevice(s->device));
  // the new buffers first, so a failed allocation leaves the handle as it was
  const size_t in = pose_capacity(s, maxMapPts);
  unsigned char *h_in = nullptr, *d_in = nullptr;
  double *h_mres = nullptr, *d_mres = nullptr;
  const size_t nres = sizeof(double) * MAPPT_OUT * (size_t)maxMapPts;
  cudaError_t e = cudaHostAlloc(&h_in, in, cudaHostAllocPortable);
  if (e == cudaSuccess) e = cudaMalloc(&d_in, in);
  if (e == cudaSuccess && nres) e = cudaHostAlloc(&h_mres, nres, cudaHostAllocPortable);
  if (e == cudaSuccess && nres) e = cudaMalloc(&d_mres, nres);
  if (e != cudaSuccess) {
    if (h_in) cudaFreeHost(h_in);
    if (h_mres) cudaFreeHost(h_mres);
    cudaFree(d_in);
    cudaFree(d_mres);
    return set_error(COSL_E_NOMEM, "cosl_pose_solver_reserve_mappts: %d map points: %s", maxMapPts,
                     cudaGetErrorString(e));
  }
  cudaFreeHost(s->h_in);
  cudaFree(s->d_in);
  if (s->h_mres) cudaFreeHost(s->h_mres);
  cudaFree(s->d_mres);
  s->h_in = h_in;
  s->d_in = d_in;
  s->h_mres = h_mres;
  s->d_mres = d_mres;
  s->maxMap = maxMapPts;
  s->mapReady = false;
  return COSL_OK;
}

int cosl_pose_solver_submit_mappts(cosl_pose_solver* s, int C, const double* K9, const double* R0, const double* t0,
                                   const int* npts, const double* const* Ms, const double* const* ms,
                                   const double* const* covx, const double* const* prior,
                                   const double* const* prevErrs, double tau, const cosl_pose_opt* opts,
                                   const int* nmap, const double* const* Xmap, const double* const* Pmap,
                                   const double* const* mmap, const double* const* covm, double gate) {
  const MapPtsArgs mp{nmap, Xmap, Pmap, mmap, covm, gate};
  return submit_solve("cosl_pose_solver_submit_mappts", s, C, K9, R0, t0, npts, Ms, ms, covx, prior, prevErrs, tau,
                      opts, &mp);
}

int cosl_pose_solver_download_mappts(cosl_pose_solver* s, double* X, double* P, double* stat, int* status) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle("cosl_pose_solver_download_mappts"));
  if (!s->mapReady)
    return set_error(COSL_E_STATE, "cosl_pose_solver_download_mappts: the last submit was not a submit_mappts");
  for (long long j = 0; j < s->nmap; ++j) {
    const double* r = s->h_mres + (size_t)MAPPT_OUT * j;
    if (X) std::memcpy(X + 3 * j, r, sizeof(double) * 3);
    if (P) unpack_sym3(r + 3, P + 9 * j);
    if (stat) std::memcpy(stat + 3 * j, r + 9, sizeof(double) * 3);
    if (status) status[j] = (int)r[12];
  }
  return COSL_OK;
}

int cosl_pose_solver_set_ransac(cosl_pose_solver* s, int C, const uint8_t* use, int nHyp, double err_thres,
                                int min_inliers, uint64_t seed) {
  static const char* fn = "cosl_pose_solver_set_ransac";
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle(fn));
  if (!use) {
    s->rC = 0;
    return COSL_OK;
  }
  if (C < 1 || C > s->maxCams)
    return set_error(COSL_E_INVALID, "%s: %d cameras, the handle takes 1 to %d", fn, C, s->maxCams);
  if (nHyp < 1 || nHyp > (1 << 20)) return set_error(COSL_E_INVALID, "%s: nHyp %d is not in [1, 2^20]", fn, nHyp);
  if (!std::isfinite(err_thres) || !(err_thres > 0))
    return set_error(COSL_E_INVALID, "%s: err_thres %g is not a finite value > 0", fn, err_thres);
  if (min_inliers < 5) return set_error(COSL_E_INVALID, "%s: min_inliers %d < 5", fn, min_inliers);
  COSL_CUDA(cudaSetDevice(s->device));
  if (!s->d_rres) {  // the first arming: all of it or nothing, as below
    COSL_CUDA(cudaFuncSetAttribute(ransac_hyp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)ransac_hyp_smem()));
    const size_t nres = ransac_res_bytes(s->maxCams, s->maxPts);
    unsigned char *ruse = nullptr, *h_res = nullptr, *d_res = nullptr;
    cudaError_t e = cudaMalloc(&ruse, s->maxCams);
    if (e == cudaSuccess) e = cudaHostAlloc(&h_res, nres, cudaHostAllocPortable);
    if (e == cudaSuccess) e = cudaMalloc(&d_res, nres);
    if (e != cudaSuccess) {
      cudaFree(ruse);
      if (h_res) cudaFreeHost(h_res);
      cudaFree(d_res);
      return set_error(COSL_E_NOMEM, "%s: result buffers for %d cameras and %d points: %s", fn, s->maxCams,
                       s->maxPts, cudaGetErrorString(e));
    }
    s->d_ruse = ruse;
    s->h_rres = h_res;
    s->d_rres = d_res;
  }
  if (nHyp > s->rCap) {  // the new buffers first, so a failed allocation leaves the handle as it was
    const size_t nc = (size_t)s->maxCams;
    double *hyp = nullptr, *sse = nullptr;
    int *smp = nullptr, *cnt = nullptr;
    cudaError_t e = cudaMalloc(&hyp, sizeof(double) * RANSAC_HYP * nc * nHyp);
    if (e == cudaSuccess) e = cudaMalloc(&smp, sizeof(int) * 5 * nc * nHyp);
    if (e == cudaSuccess) e = cudaMalloc(&cnt, sizeof(int) * nc * (nHyp + 1));
    if (e == cudaSuccess) e = cudaMalloc(&sse, sizeof(double) * nc * (nHyp + 1));
    if (e != cudaSuccess) {
      cudaFree(hyp);
      cudaFree(smp);
      cudaFree(cnt);
      cudaFree(sse);
      return set_error(COSL_E_NOMEM, "%s: %d hypotheses for %d cameras: %s", fn, nHyp, s->maxCams,
                       cudaGetErrorString(e));
    }
    cudaFree(s->d_rhyp);
    cudaFree(s->d_rsmp);
    cudaFree(s->d_rcnt);
    cudaFree(s->d_rsse);
    s->d_rhyp = hyp;
    s->d_rsmp = smp;
    s->d_rcnt = cnt;
    s->d_rsse = sse;
    s->rCap = nHyp;
    s->ransacHyps = false;
  }
  COSL_CUDA(cudaMemcpyAsync(s->d_ruse, use, C, cudaMemcpyHostToDevice, s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  s->rC = C;
  s->rHyp = nHyp;
  s->rThr = err_thres;
  s->rMinInl = min_inliers;
  s->rSeed = seed;
  return COSL_OK;
}

int cosl_pose_solver_download_ransac(cosl_pose_solver* s, double* R, double* t, double* stat, uint8_t* inl) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle("cosl_pose_solver_download_ransac"));
  if (!s->ransacReady)
    return set_error(COSL_E_STATE, "cosl_pose_solver_download_ransac: the last submit did not run RANSAC");
  const double* res = reinterpret_cast<const double*>(s->h_rres);
  for (int c = 0; c < s->C; ++c) {
    const double* r = res + RANSAC_RES * c;
    if (R) std::memcpy(R + 9 * c, r, sizeof(double) * 9);
    if (t) std::memcpy(t + 3 * c, r + 9, sizeof(double) * 3);
    if (stat) std::memcpy(stat + 4 * c, r + 12, sizeof(double) * 4);
  }
  if (inl) std::memcpy(inl, s->h_rres + sizeof(double) * RANSAC_RES * s->C, s->tot);
  return COSL_OK;
}

int cosl_pose_solver_download_ransac_hyps(cosl_pose_solver* s, int maxHyp, int* nHyp, int* idx, double* pose,
                                          int* inliers, double* sse) {
  static const char* fn = "cosl_pose_solver_download_ransac_hyps";
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle(fn));
  if (!s->ransacReady || !s->ransacHyps)
    return set_error(COSL_E_STATE, "%s: the buffers do not hold the last submit's hypotheses", fn);
  const int nh = s->rHypRun;
  if (nHyp) *nHyp = nh;
  if (!idx && !pose && !inliers && !sse) return COSL_OK;
  if (maxHyp < nh)
    return set_error(COSL_E_INVALID, "%s: room for %d hypotheses per camera, the last submit drew %d", fn, maxHyp, nh);
  COSL_CUDA(cudaSetDevice(s->device));
  const size_t C = s->C, cap = (size_t)maxHyp, n = (size_t)nh;
  if (idx)
    COSL_CUDA(cudaMemcpy2D(idx, sizeof(int) * 5 * cap, s->d_rsmp, sizeof(int) * 5 * n, sizeof(int) * 5 * n, C,
                           cudaMemcpyDeviceToHost));
  if (pose)
    for (size_t c = 0; c < C; ++c)
      COSL_CUDA(cudaMemcpy2D(pose + 12 * cap * c, sizeof(double) * 12, s->d_rhyp + RANSAC_HYP * n * c,
                             sizeof(double) * RANSAC_HYP, sizeof(double) * 12, n, cudaMemcpyDeviceToHost));
  if (inliers)
    COSL_CUDA(cudaMemcpy2D(inliers, sizeof(int) * cap, s->d_rcnt + 1, sizeof(int) * (n + 1), sizeof(int) * n, C,
                           cudaMemcpyDeviceToHost));
  if (sse)
    COSL_CUDA(cudaMemcpy2D(sse, sizeof(double) * cap, s->d_rsse + 1, sizeof(double) * (n + 1), sizeof(double) * n, C,
                           cudaMemcpyDeviceToHost));
  return COSL_OK;
}

int cosl_pose_solver_query(cosl_pose_solver* s, int* done) {
  if (!s || !done) return set_error(COSL_E_INVALID, "cosl_pose_solver_query: null argument");
  COSL_TRY(s->rq.pending("cosl_pose_solver_query"));
  COSL_CUDA(cudaSetDevice(s->device));
  return s->rq.query(done);
}

int cosl_pose_solver_collect(cosl_pose_solver* s, double* R_opt, double* t_opt, cosl_pose_opt* opts, int* ok,
                             double* device_ms) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.pending("cosl_pose_solver_collect"));
  if (!R_opt || !t_opt || !opts) return set_error(COSL_E_INVALID, "cosl_pose_solver_collect: null argument");
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.wait(device_ms));
  const PoseOut* outs = s->h_out;
  for (int c = 0; c < s->C; ++c) {
    std::memcpy(R_opt + 9 * c, outs[c].R, sizeof(double) * 9);
    std::memcpy(t_opt + 3 * c, outs[c].t, sizeof(double) * 3);
    opts[c].lambda0 = outs[c].lambda0;
    opts[c].lambda = outs[c].lambda;
    opts[c].err0 = outs[c].err0;
    opts[c].err = outs[c].err;
    opts[c].errRW = outs[c].errRW;
    opts[c].retTypeLM = outs[c].retTypeLM;
    opts[c].npts = outs[c].npts;
    opts[c].nIterLM = outs[c].nIterLM;
    opts[c].nIterRW = outs[c].nIterRW;
    if (ok) ok[c] = outs[c].ok;
  }
  return COSL_OK;
}

void* cosl_pose_solver_stream(cosl_pose_solver* s) { return s ? (void*)s->rq.stream : nullptr; }

int cosl_pose_solver_set_covariance(cosl_pose_solver* s, double pixel_var) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  if (!(pixel_var >= 0) || !std::isfinite(pixel_var))
    return set_error(COSL_E_INVALID, "cosl_pose_solver_set_covariance: pixel_var %g is not a finite value >= 0",
                     pixel_var);
  COSL_TRY(s->rq.idle("cosl_pose_solver_set_covariance"));
  if (pixel_var > 0) {
    COSL_CUDA(cudaSetDevice(s->device));
    const size_t n = cov_doubles(s->maxCams, s->maxPts);
    if (!s->h_cov) COSL_CUDA(cudaHostAlloc(&s->h_cov, sizeof(double) * n, cudaHostAllocPortable));
    if (!s->d_cov) COSL_CUDA(cudaMalloc(&s->d_cov, sizeof(double) * n));
  }
  s->pixelVar = pixel_var;
  return COSL_OK;
}

int cosl_pose_solver_download_covariance(cosl_pose_solver* s, double* cov, double* err, double* out) {
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle("cosl_pose_solver_download_covariance"));
  if (!out) return set_error(COSL_E_INVALID, "cosl_pose_solver_download_covariance: null out");
  if (!s->covReady)
    return set_error(COSL_E_STATE, "cosl_pose_solver_download_covariance: the last solve was not armed");
  for (int c = 0; c < s->C; ++c) {
    const double* r = s->h_cov + POSE_COV_STRIDE * c;
    if (cov) std::memcpy(cov + 36 * c, r, sizeof(double) * 36);
    std::memcpy(out + 4 * c, r + 36, sizeof(double) * 4);
  }
  if (err) std::memcpy(err, s->h_cov + POSE_COV_STRIDE * s->C, sizeof(double) * s->tot);
  return COSL_OK;
}

int cosl_pose_intracam_batch(int C, const double* K9, const double* R0, const double* t0,
                             const int* npts, const double* const* Ms, const double* const* ms,
                             const double* const* prevErrs, double tau, double* R_opt,
                             double* t_opt, cosl_pose_opt* opts, int* ok, int device) {
  if (C < 1 || !K9 || !R0 || !t0 || !npts || !Ms || !ms || !R_opt || !t_opt || !opts)
    return set_error(COSL_E_INVALID, "cosl_pose_intracam_batch: null argument");
  COSL_TRY(check_device(device));
  long long tot = 0;
  COSL_TRY(check_cameras("cosl_pose_intracam_batch", C, npts, Ms, ms, opts, &tot));
  // one library-owned handle per device, reused across calls (the solve is latency-bound: an allocation per
  // call would cost more than the kernel); it is replaced by a larger one when a call does not fit.  The lock
  // serialises the callers of these shared handles only.
  static std::mutex mtx;
  static std::map<int, cosl_pose_solver*> shared;
  std::lock_guard<std::mutex> lock(mtx);
  cosl_pose_solver*& s = shared[device];
  if (!s || s->maxCams < C || s->maxPts < tot) {
    const int capC = std::max(C, s ? s->maxCams : 16);
    const int capP = (int)std::max<long long>(tot, s ? s->maxPts : 4096);
    if (s) cosl_pose_solver_destroy(s);
    s = nullptr;
    COSL_TRY(cosl_pose_solver_create(device, capC, capP, &s));
  }
  COSL_TRY(cosl_pose_solver_submit(s, C, K9, R0, t0, npts, Ms, ms, prevErrs, tau, opts));
  return cosl_pose_solver_collect(s, R_opt, t_opt, opts, ok, nullptr);
}

int cosl_pose_intracam(const double K[9], const double R0[9], const double t0[3], int npts,
                       const double* prevErrs, const double* Ms, const double* ms, double tau,
                       double R_opt[9], double t_opt[3], cosl_pose_opt* opt, int* ok) {
  const double* Msp[1] = {Ms};
  const double* msp[1] = {ms};
  const double* pep[1] = {prevErrs};
  int device = 0;
  cudaGetDevice(&device);
  return cosl_pose_intracam_batch(1, K, R0, t0, &npts, Msp, msp, prevErrs ? pep : nullptr, tau,
                                  R_opt, t_opt, opt, ok, device);
}

int cosl_tri_solver_create(int device, int maxCams, int maxPts, int maxViews, cosl_tri_solver** out) {
  if (!out || device < 0 || maxCams < 1 || maxPts < 1 || maxViews < 2)
    return set_error(COSL_E_INVALID, "cosl_tri_solver_create: bad argument");
  *out = nullptr;
  COSL_TRY(check_device(device));
  cosl_tri_solver* s = new (std::nothrow) cosl_tri_solver;
  if (!s) return set_error(COSL_E_NOMEM, "cosl_tri_solver_create: out of host memory");
  s->device = device;
  s->maxCams = maxCams;
  s->maxPts = maxPts;
  s->maxViews = maxViews;
  const int rc = alloc_tri_solver(s);
  if (rc != COSL_OK) {
    free_tri_solver(s);
    return rc;
  }
  *out = s;
  return COSL_OK;
}

int cosl_tri_solver_destroy(cosl_tri_solver* s) {
  if (!s) return set_error(COSL_E_INVALID, "null triangulation handle");
  free_tri_solver(s);
  return COSL_OK;
}

int cosl_tri_solver_submit(cosl_tri_solver* s, int nCams, const double* K9, const double* R, const double* t,
                           const double* const* camCov, int nPts, const int* viewOff, const int* viewCam,
                           const double* m, const double* covm, double pixel_var, double max_err) {
  const char* fn = "cosl_tri_solver_submit";
  if (!s) return set_error(COSL_E_INVALID, "null triangulation handle");
  COSL_TRY(s->rq.idle(fn));
  COSL_TRY(check_tri(fn, s, nCams, K9, R, t, camCov, nPts, viewOff, viewCam, m, covm, pixel_var, max_err));
  COSL_CUDA(cudaSetDevice(s->device));
  return stage_tri(s, nCams, K9, R, t, camCov, nPts, viewOff, viewCam, m, covm, pixel_var, max_err);
}

int cosl_tri_solver_query(cosl_tri_solver* s, int* done) {
  if (!s || !done) return set_error(COSL_E_INVALID, "cosl_tri_solver_query: null argument");
  COSL_TRY(s->rq.pending("cosl_tri_solver_query"));
  COSL_CUDA(cudaSetDevice(s->device));
  return s->rq.query(done);
}

int cosl_tri_solver_collect(cosl_tri_solver* s, double* X, double* P, double* stat, int* status, double* device_ms) {
  if (!s) return set_error(COSL_E_INVALID, "null triangulation handle");
  COSL_TRY(s->rq.pending("cosl_tri_solver_collect"));
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.wait(device_ms));
  for (int j = 0; j < s->nPts; ++j) {
    const double* r = s->h_out + (size_t)TRI_OUT * j;
    if (X) std::memcpy(X + 3 * (size_t)j, r, sizeof(double) * 3);
    if (P) unpack_sym3(r + 3, P + 9 * (size_t)j);
    if (stat) std::memcpy(stat + 4 * (size_t)j, r + 9, sizeof(double) * 4);
    if (status) status[j] = (int)r[13];
  }
  return COSL_OK;
}

void* cosl_tri_solver_stream(cosl_tri_solver* s) { return s ? (void*)s->rq.stream : nullptr; }

int cosl_assoc_solver_create(int device, int maxCams, int maxPts, int maxQueries, int maxFeats, int maxTrackObs,
                             cosl_assoc_solver** out) {
  if (!out || device < 0 || maxCams < 1 || maxPts < 1 || maxQueries < 1 || maxFeats < 1 || maxTrackObs < 0)
    return set_error(COSL_E_INVALID, "cosl_assoc_solver_create: bad argument");
  *out = nullptr;
  COSL_TRY(check_device(device));
  cosl_assoc_solver* s = new (std::nothrow) cosl_assoc_solver;
  if (!s) return set_error(COSL_E_NOMEM, "cosl_assoc_solver_create: out of host memory");
  s->device = device;
  s->maxCams = maxCams;
  s->maxPts = maxPts;
  s->maxQueries = maxQueries;
  s->maxFeats = maxFeats;
  s->maxTrackObs = maxTrackObs;
  const int rc = alloc_assoc_solver(s);
  if (rc != COSL_OK) {
    free_assoc_solver(s);
    return rc;
  }
  *out = s;
  return COSL_OK;
}

int cosl_assoc_solver_destroy(cosl_assoc_solver* s) {
  if (!s) return set_error(COSL_E_INVALID, "null registration handle");
  free_assoc_solver(s);
  return COSL_OK;
}

int cosl_assoc_solver_submit(cosl_assoc_solver* s, int nCams, const double* K9, const double* R, const double* t,
                             const double* const* camCov, const int* wh, const int* featOff, const double* mf,
                             const double* covf, const int* owned, const int* trkOff, const int* trkCam,
                             const double* trkM, int nPts, const double* X, const double* PX, const int* qOff,
                             const int* qCam, double pixel_var, double gate, double track_gate) {
  const char* fn = "cosl_assoc_solver_submit";
  if (!s) return set_error(COSL_E_INVALID, "null registration handle");
  COSL_TRY(s->rq.idle(fn));
  const AssocArgs a{nCams, K9, R, t, camCov, wh, featOff, mf, covf, owned, trkOff, trkCam, trkM, nPts, X, PX, qOff,
                    qCam, pixel_var, gate, track_gate};
  COSL_TRY(check_assoc(fn, s, a));
  COSL_CUDA(cudaSetDevice(s->device));
  return stage_assoc(s, a);
}

int cosl_assoc_solver_query(cosl_assoc_solver* s, int* done) {
  if (!s || !done) return set_error(COSL_E_INVALID, "cosl_assoc_solver_query: null argument");
  COSL_TRY(s->rq.pending("cosl_assoc_solver_query"));
  COSL_CUDA(cudaSetDevice(s->device));
  return s->rq.query(done);
}

int cosl_assoc_solver_collect(cosl_assoc_solver* s, int* status, int* feat, double* d2, double* pred,
                              double* device_ms) {
  if (!s) return set_error(COSL_E_INVALID, "null registration handle");
  COSL_TRY(s->rq.pending("cosl_assoc_solver_collect"));
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.wait(device_ms));
  for (int q = 0; q < s->nQ; ++q) {
    const double* r = s->h_out + (size_t)ASSOC_OUT * q;
    if (status) status[q] = (int)r[0];
    if (feat) feat[q] = (int)r[1];
    if (d2) std::memcpy(d2 + 2 * (size_t)q, r + 2, sizeof(double) * 2);
    if (pred) std::memcpy(pred + 5 * (size_t)q, r + 4, sizeof(double) * 5);
  }
  return COSL_OK;
}

void* cosl_assoc_solver_stream(cosl_assoc_solver* s) { return s ? (void*)s->rq.stream : nullptr; }

}  // extern "C"
