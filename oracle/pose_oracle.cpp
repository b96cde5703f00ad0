/*
 * pose_oracle.cpp -- CPU restatement of the reference's per-frame 6-DoF pose refinement
 * (TEST INFRASTRUCTURE, see oracle.h).  PARITY PINNED: the unmodified reference file
 * slam/SL_IntraCamPose.cpp is compiled here into oracle/_ref/libintracam_ref.so (oracle/Makefile
 * target `ref`; only the 7 LibVisualSLAM primitives project/matATB/matAB/matInv/mat33AB/
 * reprojError2/doubleArrCopy are supplied by oracle/ref_stubs/primitives.cpp, restated from their
 * use) and this restatement reproduces its intraCamEstimate BIT FOR BIT: 40 seeded live cases +
 * the committed reference-generated vectors tests/golden/pose_ref.npz (tests/test_pose_ref.py).
 *
 * Follows /root/reference/src/slam/SL_IntraCamPose.cpp:
 *   so3_exp            getSO3ExpMap                 :10-39
 *   jac_numeric        _perspectiveSO3JacobiNum     :43-84,  _perspectiveTJacobiNum :89-117
 *   weighted_step      intraCamWeightedLMStep       :259-303
 *   update_pose        intraCamUpdatePose           :367-380
 *   weighted_cost      reprojError2Weighted         :439-456
 *   weighted_lm        intraCamWeightedLMProc       :475-549
 *   orc_pose_intracam  intraCamEstimate             :626-709
 * Choices: matInv(6) = Gauss-Jordan with partial pivoting; R_tmp/t_tmp (read uninitialised by the
 * reference when the very first LM steps all fail, :540-543) start at R0/t0, and so do R_opt/t_opt
 * (never written by the reference when maxIterRW = 0 or maxIterLM = 0).
 *
 * Compiled with -ffp-contract=off so the forward differences (eps = 1e-8) see the same roundings
 * as the CUDA kernel, which uses explicit non-fused fp64 operations for them.
 */
#include "oracle.h"

#include <cmath>
#include <cstring>
#include <vector>

extern "C" void orc_so3_exp(const double w[3], double R[9]) {
  const double th = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (th == 0) {
    for (int i = 0; i < 9; ++i) R[i] = 0;
    R[0] = R[4] = R[8] = 1.0;
    return;
  }
  const double a0 = w[0] / th, a1 = w[1] / th, a2 = w[2] / th;
  const double s = std::sin(th), c1 = 1 - std::cos(th);
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

extern "C" void orc_project(const double K[9], const double R[9], const double t[3],
                            const double M[3], double m[2]) {
  // x = K (R M + t), m = x_{1,2} / x_3   (inferred from use, SL_IntraCamPose.cpp:60,234)
  const double c0 = R[0] * M[0] + R[1] * M[1] + R[2] * M[2] + t[0];
  const double c1 = R[3] * M[0] + R[4] * M[1] + R[5] * M[2] + t[1];
  const double c2 = R[6] * M[0] + R[7] * M[1] + R[8] * M[2] + t[2];
  const double u = K[0] * c0 + K[1] * c1 + K[2] * c2;
  const double v = K[3] * c0 + K[4] * c1 + K[5] * c2;
  const double w = K[6] * c0 + K[7] * c1 + K[8] * c2;
  m[0] = u / w;
  m[1] = v / w;
}

namespace {

inline void mat33(const double A[9], const double B[9], double C[9]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// forward differences, eps = 1e-8; J rows: [d m0 / d(w,t) ; d m1 / d(w,t)]
void jac_numeric(const double K[9], const double R[9], const double t[3], const double M[3],
                 const double rm0[2], double J[12]) {
  const double eps = 1e-8;
  double rm[2], dR[9], R1[9];
  for (int k = 0; k < 3; ++k) {
    double w[3] = {0, 0, 0};
    w[k] = eps;
    orc_so3_exp(w, dR);
    mat33(R, dR, R1);
    orc_project(K, R1, t, M, rm);
    J[k] = (rm[0] - rm0[0]) / eps;
    J[6 + k] = (rm[1] - rm0[1]) / eps;
  }
  for (int k = 0; k < 3; ++k) {
    double t1[3] = {t[0], t[1], t[2]};
    t1[k] = t[k] + eps;
    orc_project(K, R, t1, M, rm);
    J[3 + k] = (rm[0] - rm0[0]) / eps;
    J[9 + k] = (rm[1] - rm0[1]) / eps;
  }
}

// inverse by Gauss-Jordan elimination with partial pivoting; returns false if singular
bool inv6(const double A[36], double Ainv[36]) {
  double a[6][12];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      a[i][j] = A[6 * i + j];
      a[i][6 + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < 6; ++c) {
    int p = c;
    double best = std::fabs(a[c][c]);
    for (int r = c + 1; r < 6; ++r)
      if (std::fabs(a[r][c]) > best) {
        best = std::fabs(a[r][c]);
        p = r;
      }
    if (best == 0.0) return false;
    if (p != c)
      for (int j = 0; j < 12; ++j) std::swap(a[c][j], a[p][j]);
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

void weighted_step(const double K[9], const double R[9], const double t[3], int n,
                   const double* Ws, const double* Ms, const double* ms, double param[6],
                   double lambda) {
  double sA[36], sB[6];
  std::memset(sA, 0, sizeof(sA));
  std::memset(sB, 0, sizeof(sB));
  for (int i = 0; i < n; ++i) {
    double rm[2], J[12];
    orc_project(K, R, t, Ms + 3 * i, rm);
    jac_numeric(K, R, t, Ms + 3 * i, rm, J);
    for (int k = 0; k < 12; ++k) J[k] = Ws[i] * J[k];
    const double r0 = (-rm[0] + ms[2 * i]) * Ws[i];
    const double r1 = (-rm[1] + ms[2 * i + 1]) * Ws[i];
    for (int a = 0; a < 6; ++a) {
      for (int b = 0; b < 6; ++b) sA[6 * a + b] += J[a] * J[b] + J[6 + a] * J[6 + b];
      sB[a] += J[a] * r0 + J[6 + a] * r1;
    }
  }
  for (int a = 0; a < 6; ++a) sA[7 * a] += lambda;
  double inv[36];
  if (!inv6(sA, inv)) {
    for (int a = 0; a < 6; ++a) param[a] = 0;
    return;
  }
  for (int a = 0; a < 6; ++a) {
    double s = 0;
    for (int b = 0; b < 6; ++b) s += inv[6 * a + b] * sB[b];
    param[a] = s;
  }
}

void update_pose(const double R[9], const double t[3], const double p[6], double Rn[9],
                 double tn[3]) {
  double dR[9];
  orc_so3_exp(p, dR);
  mat33(R, dR, Rn);
  tn[0] = t[0] + p[3];
  tn[1] = t[1] + p[4];
  tn[2] = t[2] + p[5];
}

double weighted_cost(const double K[9], const double R[9], const double t[3], int n,
                     const double* Ws, const double* Ms, const double* ms) {
  double err = 0;
  for (int i = 0; i < n; ++i) {
    double rm[2];
    orc_project(K, R, t, Ms + 3 * i, rm);
    const double dx = ms[2 * i] - rm[0], dy = ms[2 * i + 1] - rm[1];
    err += (dx * dx + dy * dy) * Ws[i];
  }
  return err;
}

bool weighted_lm(const double K[9], const double R0[9], const double t0[3], int n,
                 const double* Ws, const double* Ms, const double* ms, double R_opt[9],
                 double t_opt[3], cosl_pose_opt* opt) {
  double param[6];
  opt->npts = n;
  opt->lambda = opt->lambda0;
  opt->err0 = weighted_cost(K, R0, t0, n, Ws, Ms, ms);
  opt->err = opt->err0;
  double R[9], t[3], R_tmp[9], t_tmp[3];
  std::memcpy(R, R0, sizeof(R));
  std::memcpy(t, t0, sizeof(t));
  std::memcpy(R_tmp, R0, sizeof(R));
  std::memcpy(t_tmp, t0, sizeof(t));
  opt->retTypeLM = 1;
  int i = 0;
  double err = opt->err0;
  for (; i < opt->maxIterLM; ++i) {
    weighted_step(K, R, t, n, Ws, Ms, ms, param, opt->lambda);
    update_pose(R, t, param, R_opt, t_opt);
    double p2 = 0;
    for (int k = 0; k < 6; ++k) p2 += param[k] * param[k];
    if (p2 < opt->epsParamChangeLM) {
      std::memcpy(R, R_opt, sizeof(R));
      std::memcpy(t, t_opt, sizeof(t));
      opt->retTypeLM = 0;
      break;
    }
    err = weighted_cost(K, R_opt, t_opt, n, Ws, Ms, ms);
    if (std::fabs(err - opt->err) < opt->epsErrorChangeLM) {
      opt->retTypeLM = 0;
      break;
    }
    if (err <= opt->err) {
      std::memcpy(R, R_opt, sizeof(R));
      std::memcpy(t, t_opt, sizeof(t));
      std::memcpy(R_tmp, R_opt, sizeof(R));
      std::memcpy(t_tmp, t_opt, sizeof(t));
      opt->err = err;
      opt->lambda /= 10;
    } else {
      opt->lambda *= 10;
      if (opt->lambda > 1e+18) {
        opt->retTypeLM = -1;
        break;
      }
    }
  }
  if (opt->retTypeLM == -1) {
    std::memcpy(R_opt, R_tmp, sizeof(R));
    std::memcpy(t_opt, t_tmp, sizeof(t));
  }
  opt->err = err;
  opt->nIterLM = i;
  return opt->retTypeLM >= 0;
}

inline double tukey(double e, double tau) {
  if (e >= tau) return 0;
  e /= tau;
  e = 1 - e * e;
  return e * e;
}

}  // namespace

extern "C" int orc_pose_intracam(const double K[9], const double R0[9], const double t0[3],
                                 int npts, const double* prevErrs, const double* Ms,
                                 const double* ms, double tau, double R_opt[9], double t_opt[3],
                                 cosl_pose_opt* opt) {
  std::vector<double> Ws(npts > 0 ? npts : 1);
  for (int i = 0; i < npts; ++i) Ws[i] = prevErrs ? tukey(std::fabs(prevErrs[i]), tau) : 1.0;
  double R[9], t[3];
  std::memcpy(R, R0, sizeof(R));
  std::memcpy(t, t0, sizeof(t));
  // the reference leaves R_opt / t_opt unwritten with maxIterRW = 0 and, with maxIterLM = 0, reads them
  // back as the next round's pose; like the kernel, they start at R0 / t0
  std::memcpy(R_opt, R0, sizeof(R));
  std::memcpy(t_opt, t0, sizeof(t));
  bool ret = true;
  int k = 0;
  opt->errRW = -1;
  for (; k < opt->maxIterRW; ++k) {
    if (!weighted_lm(K, R, t, npts, Ws.data(), Ms, ms, R_opt, t_opt, opt)) {
      ret = false;
      break;
    }
    opt->lambda0 = opt->lambda;
    if (opt->errRW < 0)
      opt->errRW = opt->err;
    else {
      if (std::fabs(opt->err - opt->errRW) < opt->epsErrorChangeRW) {
        ret = true;
        break;
      }
      opt->errRW = opt->err;
    }
    std::memcpy(R, R_opt, sizeof(R));
    std::memcpy(t, t_opt, sizeof(t));
    for (int i = 0; i < npts; ++i) {
      double rm[2];
      orc_project(K, R, t, Ms + 3 * i, rm);
      const double dx = rm[0] - ms[2 * i], dy = rm[1] - ms[2 * i + 1];
      Ws[i] = tukey(std::sqrt(dx * dx + dy * dy), tau);
    }
  }
  opt->nIterRW = k;
  return ret ? 1 : 0;
}
