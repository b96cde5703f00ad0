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
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <mutex>
#include <new>

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

__device__ double weighted_cost(const double K[9], const double R[9], const double t[3], int n,
                                const double* Ws, const double* Ms, const double* ms,
                                double* s_red) {
  double err[1] = {0};
  for (int i = threadIdx.x; i < n; i += POSE_THREADS) {
    double rm[2];
    project(K, R, t, Ms + 3 * i, rm);
    const double dx = ms[2 * i] - rm[0], dy = ms[2 * i + 1] - rm[1];
    err[0] += (dx * dx + dy * dy) * Ws[i];
  }
  block_sum<1>(err, s_red);
  return err[0];
}

// intraCamWeightedLMStep (:259-303)
__device__ void weighted_step(const double K[9], const double R[9], const double t[3], int n,
                              const double* Ws, const double* Ms, const double* ms,
                              double param[6], double lambda, const double dRk[3][9],
                              double* s_red) {
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
    const double w = Ws[i];
#pragma unroll
    for (int k = 0; k < 12; ++k) J[k] = w * J[k];
    const double r0 = (-rm0[0] + ms[2 * i]) * w;
    const double r1 = (-rm0[1] + ms[2 * i + 1]) * w;
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

__global__ void __launch_bounds__(POSE_THREADS)
pose_intracam_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll,
                     const double* __restrict__ msAll, const double* __restrict__ prevAll,
                     double* __restrict__ WsAll, PoseCfg cfg, PoseOut* __restrict__ outs) {
  __shared__ double s_red[(POSE_THREADS / 32) * 27];
  const PoseCam cam = cams[blockIdx.x];
  const int n = cam.npts;
  const double* Ms = MsAll + 3 * cam.off;
  const double* ms = msAll + 2 * cam.off;
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
    err0 = weighted_cost(K, R, t, n, Ws, Ms, ms, s_red);
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
      weighted_step(K, Rlm, tlm, n, Ws, Ms, ms, param, lambda, dRk, s_red);
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
      err = weighted_cost(K, R_opt, t_opt, n, Ws, Ms, ms, s_red);
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
__global__ void __launch_bounds__(POSE_THREADS)
pose_cov_kernel(const PoseCam* __restrict__ cams, const double* __restrict__ MsAll,
                const double* __restrict__ msAll, const PoseOut* __restrict__ outs, double tau, double pixel_var,
                double* __restrict__ res, double* __restrict__ errAll) {
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
      int q = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int b = a; b < 6; ++b) acc[q++] += w * (J[a] * J[b] + J[6 + a] * J[6 + b]);
      }
      acc[21] += w * (e * e);
      acc[22] += 1;
    }
  }
  block_sum<23>(acc, s_red);
  if (threadIdx.x != 0) return;
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

}  // namespace

// A pose solver handle.  The inputs of one solve travel in one copy from a pinned staging buffer laid out as
// PoseCam[C] | M[3 tot] | m[2 tot] | prevErrs[tot] (tot = points of the solve); the PoseOuts come back into
// pinned memory.  Capacity is fixed at create: everything is allocated once, the covariance stage's buffers
// (laid out as res[C][POSE_COV_STRIDE] | err[tot]) when the handle is first armed.
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
  double pixelVar = 0; // > 0: armed
  double* d_cov = nullptr;
  double* h_cov = nullptr;
  bool covReady = false;  // the last submitted solve was armed
};

namespace {

size_t input_bytes(int C, long long tot) { return sizeof(PoseCam) * C + sizeof(double) * 6 * tot; }

void free_pose_solver(cosl_pose_solver* s) {
  cudaSetDevice(s->device);
  s->rq.destroy();
  if (s->h_in) cudaFreeHost(s->h_in);
  if (s->h_out) cudaFreeHost(s->h_out);
  if (s->h_cov) cudaFreeHost(s->h_cov);
  cudaFree(s->d_in);
  cudaFree(s->d_W);
  cudaFree(s->d_out);
  cudaFree(s->d_cov);
  delete s;
}

size_t cov_doubles(int C, long long tot) { return (size_t)POSE_COV_STRIDE * C + tot; }

int alloc_pose_solver(cosl_pose_solver* s) {
  COSL_CUDA(cudaSetDevice(s->device));
  COSL_TRY(s->rq.create());
  const size_t in = input_bytes(s->maxCams, s->maxPts);
  COSL_CUDA(cudaHostAlloc(&s->h_in, in, cudaHostAllocPortable));
  COSL_CUDA(cudaHostAlloc(&s->h_out, sizeof(PoseOut) * s->maxCams, cudaHostAllocPortable));
  COSL_CUDA(cudaMalloc(&s->d_in, in));
  COSL_CUDA(cudaMalloc(&s->d_W, sizeof(double) * std::max(s->maxPts, 1)));
  COSL_CUDA(cudaMalloc(&s->d_out, sizeof(PoseOut) * s->maxCams));
  return COSL_OK;
}

// The staged inputs of C cameras and tot points: copy, kernel, read-back.
int enqueue_solve(cosl_pose_solver* s, int C, long long tot, const PoseCfg& cfg) {
  const PoseCam* d_cams = reinterpret_cast<const PoseCam*>(s->d_in);
  const double* d_M = reinterpret_cast<const double*>(s->d_in + sizeof(PoseCam) * C);
  const double* d_m = d_M + 3 * tot;
  const double* d_p = d_m + 2 * tot;
  cudaStream_t st = s->rq.stream;
  COSL_CUDA(cudaMemcpyAsync(s->d_in, s->h_in, input_bytes(C, tot), cudaMemcpyHostToDevice, st));
  COSL_LAUNCH(pose_intracam_kernel, C, POSE_THREADS, 0, st, d_cams, d_M, d_m, d_p, s->d_W, cfg, s->d_out);
  COSL_CUDA(cudaGetLastError());
  COSL_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, sizeof(PoseOut) * C, cudaMemcpyDeviceToHost, st));
  if (s->pixelVar > 0) {
    COSL_LAUNCH(pose_cov_kernel, C, POSE_THREADS, 0, st, d_cams, d_M, d_m, s->d_out, cfg.tau, s->pixelVar, s->d_cov,
                s->d_cov + POSE_COV_STRIDE * C);
    COSL_CUDA(cudaGetLastError());
    COSL_CUDA(cudaMemcpyAsync(s->h_cov, s->d_cov, sizeof(double) * cov_doubles(C, tot), cudaMemcpyDeviceToHost, st));
  }
  return COSL_OK;
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
  if (!s) return set_error(COSL_E_INVALID, "null pose solver handle");
  COSL_TRY(s->rq.idle("cosl_pose_solver_submit"));
  if (C < 1 || !K9 || !R0 || !t0 || !npts || !Ms || !ms || !opts)
    return set_error(COSL_E_INVALID, "cosl_pose_solver_submit: null argument");
  if (C > s->maxCams)
    return set_error(COSL_E_INVALID, "cosl_pose_solver_submit: %d cameras exceed the handle's %d", C, s->maxCams);
  long long tot = 0;
  COSL_TRY(check_cameras("cosl_pose_solver_submit", C, npts, Ms, ms, opts, &tot));
  if (tot > s->maxPts)
    return set_error(COSL_E_INVALID, "cosl_pose_solver_submit: %lld points exceed the handle's %d", tot, s->maxPts);
  COSL_CUDA(cudaSetDevice(s->device));
  // nothing is in flight, so no copy reads the staging buffer any more
  PoseCam* cams = reinterpret_cast<PoseCam*>(s->h_in);
  double* hM = reinterpret_cast<double*>(s->h_in + sizeof(PoseCam) * C);
  double* hm = hM + 3 * tot;
  double* hp = hm + 2 * tot;
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
    }
    off += npts[c];
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
  s->covReady = false;
  COSL_TRY(s->rq.submit("cosl_pose_solver_submit", [&]() { return enqueue_solve(s, C, tot, cfg); }));
  s->covReady = s->pixelVar > 0;
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

}  // extern "C"
