/*
 * ba_oracle.cpp -- CPU restatement of the reference's multi-camera bundle adjustment
 * (TEST INFRASTRUCTURE, see oracle.h).  PARITY UNPINNED.
 *
 * The arithmetic of this path lives in a third-party dependency that is NOT under /root/reference:
 *   danping/LibVisualSLAM (version unpinned: find_package(VisualSLAM REQUIRED), CMakeLists.txt:7)
 *     geometry/SL_BundleAdjust.{h,cpp}   bundleAdjustRobust, Meas2D, Point3d
 *     geometry/SL_BundleHelper.{h,cpp}   img_projsKRTS_x, img_projsKRTS_jac_x, sbaGlobs
 *     extern/sba-1.6 (Lourakis & Argyros)  sba_motstr_levmar_x
 * What is restated here:
 *   - parameterisation, options and unpacking from the in-tree adapter
 *     app/SL_CoSLAMBA.cpp:290-378 (packing, opts = {1e-3*1e-4,1e-12,1e-12,0,1e-16}),
 *     :473-509 (R = quat2mat(dq (x) q0));
 *   - one LM iteration = the published SBA algorithm (Lourakis & Argyros, ACM TOMS 36(1), 2009,
 *     "sba_motstr_levmar_x"): Schur complement on the point blocks, dense Cholesky of the reduced
 *     camera system, Nielsen damping update, stop tests eps1..eps4; constants as published;
 *   - the robust wrapper bundleAdjustRobust is INFERRED from its call sites
 *     (app/SL_CoSLAMRobustBA.cpp:174, app/SL_InterCamPoseEstimator.cpp:95,
 *      app/SL_MergeCameraGroup.cpp:646-647) and from the Tukey biweight used everywhere else in
 *     the tree (slam/SL_IntraCamPose.cpp:641-655): maxIter rounds of
 *     {w = (1-(|e|/maxErr)^2)^2 if |e|<maxErr else 0; weighted LM with itmax = nInnerMaxIter},
 *     then Meas2D::outlier = (|e| >= maxErr).
 * All parity claims of the CUDA path are relative to this restatement.
 */
#include "oracle.h"

#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

int orc_threads();

/* ---------------------------------------------------------------- LAPACK (optional) */
typedef void (*dpotrf_t)(const char*, const int*, double*, const int*, int*);
typedef void (*dpotrs_t)(const char*, const int*, const int*, const double*, const int*, double*,
                         const int*, int*);
typedef void (*setthr_t)(int);
static dpotrf_t g_dpotrf = nullptr;
static dpotrs_t g_dpotrs = nullptr;
static setthr_t g_setthr = nullptr;

extern "C" int orc_set_lapack(const char* path) {
  void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!h) return -1;
  g_dpotrf = (dpotrf_t)dlsym(h, "scipy_dpotrf_");
  g_dpotrs = (dpotrs_t)dlsym(h, "scipy_dpotrs_");
  g_setthr = (setthr_t)dlsym(h, "scipy_openblas_set_num_threads");
  if (!g_dpotrf) g_dpotrf = (dpotrf_t)dlsym(h, "dpotrf_");
  if (!g_dpotrs) g_dpotrs = (dpotrs_t)dlsym(h, "dpotrs_");
  if (!g_setthr) g_setthr = (setthr_t)dlsym(h, "openblas_set_num_threads");
  return (g_dpotrf && g_dpotrs) ? 0 : -2;
}

/* ---------------------------------------------------------------- quaternions */
extern "C" void orc_quat2mat(const double q[4], double R[9]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = w * w + x * x - y * y - z * z;
  R[1] = 2 * (x * y - w * z);
  R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z);
  R[4] = w * w - x * x + y * y - z * z;
  R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y);
  R[7] = 2 * (y * z + w * x);
  R[8] = w * w - x * x - y * y + z * z;
}

extern "C" void orc_mat2quat(const double R[9], double q[4]) {
  // Shepperd's method, result normalised with w >= 0
  const double tr = R[0] + R[4] + R[8];
  double w, x, y, z;
  if (tr > 0) {
    double s = std::sqrt(tr + 1.0) * 2;
    w = 0.25 * s;
    x = (R[7] - R[5]) / s;
    y = (R[2] - R[6]) / s;
    z = (R[3] - R[1]) / s;
  } else if (R[0] > R[4] && R[0] > R[8]) {
    double s = std::sqrt(1.0 + R[0] - R[4] - R[8]) * 2;
    w = (R[7] - R[5]) / s;
    x = 0.25 * s;
    y = (R[1] + R[3]) / s;
    z = (R[2] + R[6]) / s;
  } else if (R[4] > R[8]) {
    double s = std::sqrt(1.0 + R[4] - R[0] - R[8]) * 2;
    w = (R[2] - R[6]) / s;
    x = (R[1] + R[3]) / s;
    y = 0.25 * s;
    z = (R[5] + R[7]) / s;
  } else {
    double s = std::sqrt(1.0 + R[8] - R[0] - R[4]) * 2;
    w = (R[3] - R[1]) / s;
    x = (R[2] + R[6]) / s;
    y = (R[5] + R[7]) / s;
    z = 0.25 * s;
  }
  double nrm = std::sqrt(w * w + x * x + y * y + z * z);
  if (w < 0) nrm = -nrm;
  q[0] = w / nrm;
  q[1] = x / nrm;
  q[2] = y / nrm;
  q[3] = z / nrm;
}

static inline void quat_mul(const double a[4], const double b[4], double p[4]) {
  p[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  p[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  p[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  p[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

static inline void cross(const double a[3], const double b[3], double c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

/* ---------------------------------------------------------------- camera model
 * x = pi(K (R(dq(v)) R(q0) X + t)), dq = (sqrt(1-|v|^2), v)   (app/SL_CoSLAMBA.cpp:337-354,483-490)
 * K = [fx s cx; 0 fy cy; 0 0 1] (only K0,K1,K2,K4,K5 are read, as BundleRTS packs them).
 * A = d x / d (v, t) (2x6 row-major), B = d x / d X (2x3 row-major). */
extern "C" void orc_ba_project(const double K[9], const double q0[4], const double v[3],
                               const double t[3], const double X[3], double xy[2], double A[12],
                               double B[6]) {
  double R0[9];
  orc_quat2mat(q0, R0);
  const double Y[3] = {R0[0] * X[0] + R0[1] * X[1] + R0[2] * X[2],
                       R0[3] * X[0] + R0[4] * X[1] + R0[5] * X[2],
                       R0[6] * X[0] + R0[7] * X[1] + R0[8] * X[2]};
  const double w = std::sqrt(1.0 - (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
  double vxY[3], vxvxY[3];
  cross(v, Y, vxY);
  cross(v, vxY, vxvxY);
  const double P[3] = {Y[0] + 2 * w * vxY[0] + 2 * vxvxY[0] + t[0],
                       Y[1] + 2 * w * vxY[1] + 2 * vxvxY[1] + t[1],
                       Y[2] + 2 * w * vxY[2] + 2 * vxvxY[2] + t[2]};
  const double iz = 1.0 / P[2];
  const double un = K[0] * P[0] + K[1] * P[1];
  xy[0] = un * iz + K[2];
  xy[1] = K[4] * P[1] * iz + K[5];
  if (!A && !B) return;
  // d xy / d P
  const double Jp[6] = {K[0] * iz, K[1] * iz, -un * iz * iz, 0.0, K[4] * iz, -K[4] * P[1] * iz * iz};
  if (A) {
    for (int k = 0; k < 3; ++k) {
      double e[3] = {0, 0, 0};
      e[k] = 1.0;
      double exY[3], exvxY[3], vxexY[3];
      cross(e, Y, exY);
      cross(e, vxY, exvxY);
      cross(v, exY, vxexY);
      const double dw = -v[k] / w;
      double dP[3];
      for (int c = 0; c < 3; ++c)
        dP[c] = 2 * dw * vxY[c] + 2 * w * exY[c] + 2 * exvxY[c] + 2 * vxexY[c];
      A[k] = Jp[0] * dP[0] + Jp[1] * dP[1] + Jp[2] * dP[2];
      A[6 + k] = Jp[3] * dP[0] + Jp[4] * dP[1] + Jp[5] * dP[2];
    }
    for (int k = 0; k < 3; ++k) {
      A[3 + k] = Jp[k];
      A[9 + k] = Jp[3 + k];
    }
  }
  if (B) {
    // R_full = R(dq) R0
    const double dq[4] = {w, v[0], v[1], v[2]};
    double Rd[9], Rf[9];
    orc_quat2mat(dq, Rd);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        Rf[3 * i + j] = Rd[3 * i] * R0[j] + Rd[3 * i + 1] * R0[3 + j] + Rd[3 * i + 2] * R0[6 + j];
    for (int k = 0; k < 3; ++k) {
      B[k] = Jp[0] * Rf[k] + Jp[1] * Rf[3 + k] + Jp[2] * Rf[6 + k];
      B[3 + k] = Jp[3] * Rf[k] + Jp[4] * Rf[3 + k] + Jp[5] * Rf[6 + k];
    }
  }
}

namespace {

inline double tukey(double e, double s) {
  if (e >= s) return 0;
  e /= s;
  e = 1 - e * e;
  return e * e;
}

// 3x3 symmetric positive definite inverse via cofactors; V = [v00 v01 v02 v11 v12 v22]
inline bool inv3sym(const double V[6], double I[6]) {
  const double a = V[0], b = V[1], c = V[2], d = V[3], e = V[4], f = V[5];
  const double A = d * f - e * e, B = c * e - b * f, C = b * e - c * d;
  const double det = a * A + b * B + c * C;
  if (!(det > 0) || !std::isfinite(det)) return false;
  const double r = 1.0 / det;
  I[0] = A * r;
  I[1] = B * r;
  I[2] = C * r;
  I[3] = (a * f - c * c) * r;
  I[4] = (b * c - a * e) * r;
  I[5] = (a * d - b * b) * r;
  return true;
}

// dense SPD solve S x = b; S row-major, upper triangle valid (== column-major lower)
bool chol_solve(std::vector<double>& S, std::vector<double>& b, int n) {
  if (g_dpotrf && g_dpotrs) {
    if (g_setthr) g_setthr(orc_threads());
    int info = 0, one = 1;
    g_dpotrf("L", &n, S.data(), &n, &info);
    if (info != 0) return false;
    g_dpotrs("L", &n, &one, S.data(), &n, b.data(), &n, &info);
    return info == 0;
  }
  // fallback: row-major upper U^T U factorisation, blocked over rows for OpenMP
  for (int k = 0; k < n; ++k) {
    double d = S[(size_t)k * n + k];
    if (!(d > 0)) return false;
    d = std::sqrt(d);
    S[(size_t)k * n + k] = d;
    const double r = 1.0 / d;
    for (int j = k + 1; j < n; ++j) S[(size_t)k * n + j] *= r;
#pragma omp parallel for num_threads(orc_threads()) schedule(static) if (n - k > 256)
    for (int i = k + 1; i < n; ++i) {
      const double f = S[(size_t)k * n + i];
      if (f == 0) continue;
      double* row = &S[(size_t)i * n];
      const double* rk = &S[(size_t)k * n];
      for (int j = i; j < n; ++j) row[j] -= f * rk[j];
    }
  }
  // U^T y = b ; U x = y
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= S[(size_t)k * n + i] * b[k];
    b[i] = s / S[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int k = i + 1; k < n; ++k) s -= S[(size_t)i * n + k] * b[k];
    b[i] = s / S[(size_t)i * n + i];
  }
  return true;
}

struct BA {
  int m, n, mcon, ncon, mf;
  int64_t N;
  const double* K;
  const int64_t* ptr;
  const int32_t* cam;
  const double* xy;
  std::vector<double> q0;      // m x 4
  std::vector<double> pa;      // m x 6  (v, t)
  std::vector<double> pb;      // n x 3
  std::vector<double> wgt;     // N observation weights
  std::vector<int32_t> pt_of;  // N
  // camera-major lists
  std::vector<int64_t> cptr;   // m+1
  std::vector<int64_t> cobs;   // N obs ids grouped by camera
  // linearisation
  std::vector<double> Aw, Bw, ew;  // N x 12, N x 6, N x 2 (already scaled by sqrt(w))
  std::vector<double> U, ea;       // m x 36 (row-major full), m x 6
  std::vector<double> V, eb;       // n x 6 (sym), n x 3
  std::vector<double> Wm, Ym;      // N x 18 (6x3 row-major)
  std::vector<double> S, rhs;
  std::vector<double> dpa, dpb;
  int nfev = 0, njev = 0, nlss = 0;

  void init(const cosl_ba_problem* p) {
    m = p->m;
    n = p->n;
    N = p->nobs;
    mcon = p->m_con;
    ncon = p->n_con;
    mf = m - mcon;
    K = p->K;
    ptr = p->ptr;
    cam = p->cam;
    xy = p->xy;
    q0.resize((size_t)m * 4);
    pa.assign((size_t)m * 6, 0.0);
    pb.assign(p->X, p->X + (size_t)n * 3);
    for (int j = 0; j < m; ++j) {
      orc_mat2quat(p->R + 9 * j, &q0[4 * j]);
      for (int k = 0; k < 3; ++k) pa[6 * j + 3 + k] = p->t[3 * j + k];
    }
    wgt.assign(N, 1.0);
    pt_of.resize(N);
    for (int i = 0; i < n; ++i)
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) pt_of[o] = i;
    cptr.assign(m + 1, 0);
    for (int64_t o = 0; o < N; ++o) cptr[cam[o] + 1]++;
    for (int j = 0; j < m; ++j) cptr[j + 1] += cptr[j];
    cobs.resize(N);
    std::vector<int64_t> fill(cptr.begin(), cptr.end() - 1);
    for (int64_t o = 0; o < N; ++o) cobs[fill[cam[o]]++] = o;
    Aw.resize((size_t)N * 12);
    Bw.resize((size_t)N * 6);
    ew.resize((size_t)N * 2);
    U.resize((size_t)m * 36);
    ea.resize((size_t)m * 6);
    V.resize((size_t)n * 6);
    eb.resize((size_t)n * 3);
    Wm.resize((size_t)N * 18);
    Ym.resize((size_t)N * 18);
    S.resize((size_t)(6 * mf) * (6 * mf));
    rhs.resize((size_t)6 * mf);
    dpa.assign((size_t)m * 6, 0.0);
    dpb.assign((size_t)n * 3, 0.0);
  }

  // residual norms per observation at (pa_, pb_): out[o] = |e_o| (unweighted)
  void residual_norms(const std::vector<double>& pa_, const std::vector<double>& pb_,
                      std::vector<double>& out) const {
    out.resize(N);
#pragma omp parallel for num_threads(orc_threads()) schedule(static)
    for (int i = 0; i < n; ++i)
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) {
        const int j = cam[o];
        double h[2];
        orc_ba_project(K + 9 * j, &q0[4 * j], &pa_[6 * j], &pa_[6 * j + 3], &pb_[3 * i], h,
                       nullptr, nullptr);
        const double dx = xy[2 * o] - h[0], dy = xy[2 * o + 1] - h[1];
        out[o] = std::sqrt(dx * dx + dy * dy);
      }
  }

  double cost(const std::vector<double>& pa_, const std::vector<double>& pb_) {
    ++nfev;
    double tot = 0;
#pragma omp parallel for num_threads(orc_threads()) schedule(static) reduction(+ : tot)
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) {
        const int j = cam[o];
        double h[2];
        orc_ba_project(K + 9 * j, &q0[4 * j], &pa_[6 * j], &pa_[6 * j + 3], &pb_[3 * i], h,
                       nullptr, nullptr);
        const double dx = xy[2 * o] - h[0], dy = xy[2 * o + 1] - h[1];
        s += wgt[o] * (dx * dx + dy * dy);
      }
      tot += s;
    }
    return tot;
  }

  // Jacobians, U, V, W, ea, eb at (pa, pb); returns |g|_inf over free params and max diag
  void linearize(double& ginf, double& maxdiag) {
    ++njev;
#pragma omp parallel for num_threads(orc_threads()) schedule(static)
    for (int i = 0; i < n; ++i) {
      double Vi[6] = {0, 0, 0, 0, 0, 0}, ebi[3] = {0, 0, 0};
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) {
        const int j = cam[o];
        double h[2];
        double* A = &Aw[(size_t)o * 12];
        double* B = &Bw[(size_t)o * 6];
        orc_ba_project(K + 9 * j, &q0[4 * j], &pa[6 * j], &pa[6 * j + 3], &pb[3 * i], h, A, B);
        const double sw = std::sqrt(wgt[o]);
        const double e0 = (xy[2 * o] - h[0]) * sw, e1 = (xy[2 * o + 1] - h[1]) * sw;
        ew[2 * o] = e0;
        ew[2 * o + 1] = e1;
        for (int k = 0; k < 12; ++k) A[k] *= sw;
        for (int k = 0; k < 6; ++k) B[k] *= sw;
        if (i >= ncon) {
          Vi[0] += B[0] * B[0] + B[3] * B[3];
          Vi[1] += B[0] * B[1] + B[3] * B[4];
          Vi[2] += B[0] * B[2] + B[3] * B[5];
          Vi[3] += B[1] * B[1] + B[4] * B[4];
          Vi[4] += B[1] * B[2] + B[4] * B[5];
          Vi[5] += B[2] * B[2] + B[5] * B[5];
          for (int c = 0; c < 3; ++c) ebi[c] += B[c] * e0 + B[3 + c] * e1;
        }
        if (i >= ncon && j >= mcon) {
          double* W = &Wm[(size_t)o * 18];
          for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 3; ++c) W[3 * r + c] = A[r] * B[c] + A[6 + r] * B[3 + c];
        }
      }
      for (int k = 0; k < 6; ++k) V[(size_t)6 * i + k] = Vi[k];
      for (int k = 0; k < 3; ++k) eb[(size_t)3 * i + k] = ebi[k];
    }
#pragma omp parallel for num_threads(orc_threads()) schedule(dynamic, 1)
    for (int j = mcon; j < m; ++j) {
      double Uj[36], eaj[6];
      std::memset(Uj, 0, sizeof(Uj));
      std::memset(eaj, 0, sizeof(eaj));
      for (int64_t q = cptr[j]; q < cptr[j + 1]; ++q) {
        const int64_t o = cobs[q];
        const double* A = &Aw[(size_t)o * 12];
        for (int r = 0; r < 6; ++r) {
          for (int c = 0; c < 6; ++c) Uj[6 * r + c] += A[r] * A[c] + A[6 + r] * A[6 + c];
          eaj[r] += A[r] * ew[2 * o] + A[6 + r] * ew[2 * o + 1];
        }
      }
      std::memcpy(&U[(size_t)36 * j], Uj, sizeof(Uj));
      std::memcpy(&ea[(size_t)6 * j], eaj, sizeof(eaj));
    }
    ginf = 0;
    maxdiag = 0;
    for (int j = mcon; j < m; ++j)
      for (int r = 0; r < 6; ++r) {
        ginf = std::max(ginf, std::fabs(ea[6 * j + r]));
        maxdiag = std::max(maxdiag, U[36 * j + 7 * r]);
      }
    for (int i = ncon; i < n; ++i) {
      for (int r = 0; r < 3; ++r) ginf = std::max(ginf, std::fabs(eb[3 * i + r]));
      maxdiag = std::max(maxdiag, std::max(V[6 * i], std::max(V[6 * i + 3], V[6 * i + 5])));
    }
  }

  // Schur complement + dense solve + back substitution for damping mu; false if not solvable
  bool solve(double mu) {
    ++nlss;
    const int ns = 6 * mf;
    std::vector<double> Vinv((size_t)n * 6);
    bool ok = true;
#pragma omp parallel for num_threads(orc_threads()) schedule(static)
    for (int i = ncon; i < n; ++i) {
      double Vs[6] = {V[6 * i] + mu, V[6 * i + 1], V[6 * i + 2], V[6 * i + 3] + mu, V[6 * i + 4],
                      V[6 * i + 5] + mu};
      double Iv[6];
      if (!inv3sym(Vs, Iv)) {
#pragma omp atomic write
        ok = false;
        for (int k = 0; k < 6; ++k) Iv[k] = 0;
      }
      for (int k = 0; k < 6; ++k) Vinv[(size_t)6 * i + k] = Iv[k];
      const double M[9] = {Iv[0], Iv[1], Iv[2], Iv[1], Iv[3], Iv[4], Iv[2], Iv[4], Iv[5]};
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) {
        if (cam[o] < mcon) continue;
        const double* W = &Wm[(size_t)o * 18];
        double* Y = &Ym[(size_t)o * 18];
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 3; ++c)
            Y[3 * r + c] = W[3 * r] * M[c] + W[3 * r + 1] * M[3 + c] + W[3 * r + 2] * M[6 + c];
      }
    }
    if (!ok) return false;
    if (ns > 0) {
      std::fill(S.begin(), S.end(), 0.0);
      // row block j of S (upper part) is owned by one thread
#pragma omp parallel for num_threads(orc_threads()) schedule(dynamic, 1)
      for (int j = mcon; j < m; ++j) {
        const int jr = 6 * (j - mcon);
        double rj[6];
        for (int r = 0; r < 6; ++r) {
          for (int c = 0; c < 6; ++c) S[(size_t)(jr + r) * ns + jr + c] = U[36 * j + 6 * r + c];
          S[(size_t)(jr + r) * ns + jr + r] += mu;
          rj[r] = ea[6 * j + r];
        }
        for (int64_t q = cptr[j]; q < cptr[j + 1]; ++q) {
          const int64_t o = cobs[q];
          const int i = pt_of[o];
          if (i < ncon) continue;
          const double* Y = &Ym[(size_t)o * 18];
          for (int r = 0; r < 6; ++r)
            rj[r] -= Y[3 * r] * eb[3 * i] + Y[3 * r + 1] * eb[3 * i + 1] + Y[3 * r + 2] * eb[3 * i + 2];
          for (int64_t o2 = ptr[i]; o2 < ptr[i + 1]; ++o2) {
            const int k = cam[o2];
            if (k < j) continue;  // cam sorted within a point; only upper blocks (k >= j)
            const int kc = 6 * (k - mcon);
            const double* W = &Wm[(size_t)o2 * 18];
            for (int r = 0; r < 6; ++r)
              for (int c = 0; c < 6; ++c)
                S[(size_t)(jr + r) * ns + kc + c] -=
                    Y[3 * r] * W[3 * c] + Y[3 * r + 1] * W[3 * c + 1] + Y[3 * r + 2] * W[3 * c + 2];
          }
        }
        for (int r = 0; r < 6; ++r) rhs[jr + r] = rj[r];
      }
      if (!chol_solve(S, rhs, ns)) return false;
    }
    std::fill(dpa.begin(), dpa.end(), 0.0);
    for (int j = mcon; j < m; ++j)
      for (int r = 0; r < 6; ++r) dpa[6 * j + r] = rhs[6 * (j - mcon) + r];
    std::fill(dpb.begin(), dpb.end(), 0.0);
#pragma omp parallel for num_threads(orc_threads()) schedule(static)
    for (int i = ncon; i < n; ++i) {
      double t3[3] = {eb[3 * i], eb[3 * i + 1], eb[3 * i + 2]};
      for (int64_t o = ptr[i]; o < ptr[i + 1]; ++o) {
        const int j = cam[o];
        if (j < mcon) continue;
        const double* W = &Wm[(size_t)o * 18];
        for (int c = 0; c < 3; ++c)
          for (int r = 0; r < 6; ++r) t3[c] -= W[3 * r + c] * dpa[6 * j + r];
      }
      const double* Iv = &Vinv[(size_t)6 * i];
      dpb[3 * i] = Iv[0] * t3[0] + Iv[1] * t3[1] + Iv[2] * t3[2];
      dpb[3 * i + 1] = Iv[1] * t3[0] + Iv[3] * t3[1] + Iv[4] * t3[2];
      dpb[3 * i + 2] = Iv[2] * t3[0] + Iv[4] * t3[1] + Iv[5] * t3[2];
    }
    return true;
  }

  /* Weighted SBA LM (sba_motstr_levmar_x with fixed per-observation weights).
   * fixed_trials > 0: benchmark mode, run exactly that many linear solves, no stop tests. */
  int levmar(int itmax, const double opts[5], double info[10], int fixed_trials, int verbose) {
    const double tau = opts[0], eps1 = opts[1], eps2 = opts[2], eps2_sq = opts[2] * opts[2],
                 eps3 = opts[3], eps4 = opts[4];
    const double EPS_SQ = 1e-24;  // SBA_EPSILON_SQ
    double mu = 0, nu = 2;
    int stop = 0, itno = 0;
    nfev = njev = nlss = 0;
    double p_eL2 = cost(pa, pb);
    const double init_eL2 = p_eL2;
    double ginf = 0, maxdiag = 0, dp_L2 = 0;
    std::vector<double> na(pa.size()), nb(pb.size());
    if (!std::isfinite(p_eL2)) stop = 7;
    for (itno = 0; itno < itmax && !stop; ++itno) {
      linearize(ginf, maxdiag);
      double p_L2 = 0;
      for (int j = mcon; j < m; ++j)
        for (int r = 0; r < 6; ++r) p_L2 += pa[6 * j + r] * pa[6 * j + r];
      for (int i = ncon; i < n; ++i)
        for (int r = 0; r < 3; ++r) p_L2 += pb[3 * i + r] * pb[3 * i + r];
      if (!fixed_trials && ginf <= eps1) {
        stop = 1;
        break;
      }
      if (itno == 0) mu = tau * maxdiag;
      while (true) {
        bool solved = solve(mu);
        bool accepted = false;
        if (solved) {
          dp_L2 = 0;
          double dL = 0;
          for (int j = mcon; j < m; ++j)
            for (int r = 0; r < 6; ++r) {
              const double d = dpa[6 * j + r];
              dp_L2 += d * d;
              dL += d * (mu * d + ea[6 * j + r]);
              na[6 * j + r] = pa[6 * j + r] + d;
            }
          for (int j = 0; j < mcon; ++j)
            for (int r = 0; r < 6; ++r) na[6 * j + r] = pa[6 * j + r];
          for (int i = 0; i < n; ++i)
            for (int r = 0; r < 3; ++r) {
              const double d = (i >= ncon) ? dpb[3 * i + r] : 0.0;
              dp_L2 += d * d;
              if (i >= ncon) dL += d * (mu * d + eb[3 * i + r]);
              nb[3 * i + r] = pb[3 * i + r] + d;
            }
          if (!fixed_trials) {
            if (dp_L2 <= eps2_sq * p_L2) {
              stop = 2;
              break;
            }
            if (dp_L2 >= (p_L2 + eps2) / EPS_SQ) {
              stop = 4;
              break;
            }
          }
          const double pdp_eL2 = cost(na, nb);
          if (!std::isfinite(pdp_eL2)) {
            stop = 7;
            break;
          }
          const double dF = p_eL2 - pdp_eL2;
          if (verbose)
            std::printf("  [orc LM %d] mu %.3e cost %.9g -> %.9g dL %.3e\n", itno, mu, p_eL2,
                        pdp_eL2, dL);
          if (dF > 0 && dL > 0) {
            double tmp = 2 * dF / dL - 1;
            tmp = 1 - tmp * tmp * tmp;
            mu = mu * std::max(tmp, 1.0 / 3.0);
            nu = 2;
            if (!fixed_trials && (std::sqrt(p_eL2) - std::sqrt(pdp_eL2)) < eps4 * std::sqrt(p_eL2))
              stop = 6;
            pa = na;
            pb = nb;
            p_eL2 = pdp_eL2;
            accepted = true;
          }
        }
        if (fixed_trials && nlss >= fixed_trials) {
          stop = 3;
          break;
        }
        if (accepted) break;
        mu *= nu;
        const double nu2 = nu * 2;
        if (!(nu2 > nu) || !std::isfinite(mu)) {
          stop = 5;
          break;
        }
        nu = nu2;
      }
      if (!fixed_trials && p_eL2 <= eps3) stop = 3;
    }
    if (itno >= itmax && !stop) stop = 3;
    if (info) {
      info[0] = init_eL2;
      info[1] = p_eL2;
      info[2] = ginf;
      info[3] = dp_L2;
      info[4] = maxdiag > 0 ? mu / maxdiag : 0;
      info[5] = itno;
      info[6] = stop;
      info[7] = nfev;
      info[8] = njev;
      info[9] = nlss;
    }
    return itno;
  }

  void write_back(cosl_ba_problem* p) const {
    for (int j = 0; j < m; ++j) {
      const double* v = &pa[6 * j];
      const double dq[4] = {std::sqrt(1.0 - (v[0] * v[0] + v[1] * v[1] + v[2] * v[2])), v[0], v[1],
                            v[2]};
      double q[4];
      quat_mul(dq, &q0[4 * j], q);
      const double nr = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      for (int k = 0; k < 4; ++k) q[k] /= nr;
      if (j >= mcon) {
        orc_quat2mat(q, p->R + 9 * j);
        for (int k = 0; k < 3; ++k) p->t[3 * j + k] = pa[6 * j + 3 + k];
      }
    }
    for (int i = ncon; i < n; ++i)
      for (int k = 0; k < 3; ++k) p->X[3 * i + k] = pb[3 * i + k];
  }
};

// a camera observes a point at most once (sba's vmask cannot say more); the library refuses the rest
bool observations_valid(const cosl_ba_problem* p) {
  std::vector<int> seen((size_t)p->m, -1);
  for (int i = 0; i < p->n; ++i)
    for (int64_t o = p->ptr[i]; o < p->ptr[i + 1]; ++o) {
      const int j = p->cam[o];
      if (j < 0 || j >= p->m || seen[j] == i) return false;
      seen[j] = i;
    }
  return true;
}

int run_robust(cosl_ba_problem* prob, const cosl_ba_options* opt, int fixed_trials,
               double info[COSL_BA_INFOSZ]) {
  if (!prob || !opt || prob->m < 1 || prob->n < 0 || !observations_valid(prob)) return COSL_E_INVALID;
  BA ba;
  ba.init(prob);
  double sinfo[10] = {0};
  double first_e0 = -1;
  int total_trials = 0;
  std::vector<double> rn;
  auto t0 = std::chrono::steady_clock::now();
  const int rounds = fixed_trials ? 1 : std::max(1, opt->outer_iters);
  for (int r = 0; r < rounds; ++r) {
    if (opt->max_err > 0) {
      ba.residual_norms(ba.pa, ba.pb, rn);
      for (int64_t o = 0; o < ba.N; ++o) ba.wgt[o] = tukey(rn[o], opt->max_err);
    }
    ba.levmar(fixed_trials ? (1 << 30) : opt->inner_iters, opt->opts, sinfo, fixed_trials,
              opt->verbose);
    if (first_e0 < 0) first_e0 = sinfo[0];
    total_trials += (int)sinfo[9];
  }
  auto t1 = std::chrono::steady_clock::now();
  ba.write_back(prob);
  int nout = 0;
  if (opt->max_err > 0) {
    ba.residual_norms(ba.pa, ba.pb, rn);
    for (int64_t o = 0; o < ba.N; ++o) {
      const int f = rn[o] >= opt->max_err;
      nout += f;
      if (prob->outlier) prob->outlier[o] = (uint8_t)f;
    }
  } else if (prob->outlier) {
    std::memset(prob->outlier, 0, (size_t)ba.N);
  }
  if (info) {
    for (int k = 0; k < COSL_BA_INFOSZ; ++k) info[k] = 0;
    for (int k = 0; k < 10; ++k) info[k] = sinfo[k];
    info[0] = first_e0;
    info[10] = total_trials;
    info[11] = std::chrono::duration<double>(t1 - t0).count();
    info[12] = sinfo[1];
    info[13] = nout;
  }
  return COSL_OK;
}

}  // namespace

extern "C" int orc_ba_solve(cosl_ba_problem* prob, const cosl_ba_options* opt,
                            double info[COSL_BA_INFOSZ]) {
  return run_robust(prob, opt, 0, info);
}

extern "C" int orc_ba_run_fixed(cosl_ba_problem* prob, const cosl_ba_options* opt, int trials,
                                double info[COSL_BA_INFOSZ]) {
  return run_robust(prob, opt, trials < 1 ? 1 : trials, info);
}

extern "C" double orc_ba_cost(const cosl_ba_problem* prob) {
  BA ba;
  ba.init(prob);
  return ba.cost(ba.pa, ba.pb);
}

/* sba_motstr_levmar_x(n, ncon, m, mcon, vmask, p, cnp, pnp, x, covx=0, mnp, proj, projac, globs,
 * itmax, verbose, opts, info) specialised to img_projsKRTS_x (app/SL_CoSLAMBA.cpp:360-363).
 * p = [m x (fx,cx,cy,ar,s, q1,q2,q3, t1,t2,t3) | n x 3]; rot0params = sbaGlobs::rot0params. */
extern "C" int orc_sba_motstr_levmar_x(int n, int ncon, int m, int mcon, const char* vmask,
                                       double* p, int cnp, int pnp, const double* x, int mnp,
                                       const double* rot0params, int itmax, int verbose,
                                       const double opts[5], double info[10]) {
  if (cnp != 11 || pnp != 3 || mnp != 2) return COSL_E_INVALID;
  std::vector<double> K((size_t)m * 9, 0.0), R((size_t)m * 9), t((size_t)m * 3), X((size_t)n * 3);
  for (int j = 0; j < m; ++j) {
    const double* c = p + (size_t)cnp * j;
    double* k = &K[9 * j];
    k[0] = c[0];
    k[1] = c[4];
    k[2] = c[1];
    k[4] = c[3] * c[0];
    k[5] = c[2];
    k[8] = 1.0;
    // current rotation = quat(sqrt(1-|v|^2), v) (x) rot0  -> start the solver from it
    const double dq[4] = {std::sqrt(1.0 - (c[5] * c[5] + c[6] * c[6] + c[7] * c[7])), c[5], c[6],
                          c[7]};
    double q[4];
    quat_mul(dq, rot0params + 4 * j, q);
    orc_quat2mat(q, &R[9 * j]);
    for (int a = 0; a < 3; ++a) t[3 * j + a] = c[8 + a];
  }
  std::memcpy(X.data(), p + (size_t)cnp * m, sizeof(double) * 3 * n);
  std::vector<int64_t> ptr(n + 1, 0);
  std::vector<int32_t> cam;
  for (int i = 0; i < n; ++i) {
    for (int j = 0; j < m; ++j)
      if (vmask[(size_t)i * m + j]) cam.push_back(j);
    ptr[i + 1] = (int64_t)cam.size();
  }
  cosl_ba_problem pr;
  std::memset(&pr, 0, sizeof(pr));
  pr.m = m;
  pr.n = n;
  pr.nobs = (int64_t)cam.size();
  pr.m_con = mcon;
  pr.n_con = ncon;
  pr.K = K.data();
  pr.R = R.data();
  pr.t = t.data();
  pr.X = X.data();
  pr.ptr = ptr.data();
  pr.cam = cam.data();
  pr.xy = x;
  cosl_ba_options o;
  std::memset(&o, 0, sizeof(o));
  o.max_err = 0;
  o.outer_iters = 1;
  o.inner_iters = itmax;
  for (int k = 0; k < 5; ++k) o.opts[k] = opts[k];
  o.verbose = verbose;
  double inf[COSL_BA_INFOSZ];
  int rc = run_robust(&pr, &o, 0, inf);
  if (rc != COSL_OK) return rc;
  if (info)
    for (int k = 0; k < 10; ++k) info[k] = inf[k];
  // repack: local quaternion relative to rot0
  for (int j = mcon; j < m; ++j) {
    double q[4], q0c[4] = {rot0params[4 * j], -rot0params[4 * j + 1], -rot0params[4 * j + 2],
                           -rot0params[4 * j + 3]};
    double qn[4];
    orc_mat2quat(&R[9 * j], q);
    quat_mul(q, q0c, qn);
    if (qn[0] < 0)
      for (int a = 0; a < 4; ++a) qn[a] = -qn[a];
    double* c = p + (size_t)cnp * j;
    c[5] = qn[1];
    c[6] = qn[2];
    c[7] = qn[3];
    for (int a = 0; a < 3; ++a) c[8 + a] = t[3 * j + a];
  }
  std::memcpy(p + (size_t)cnp * m + 3 * (size_t)ncon, X.data() + 3 * (size_t)ncon,
              sizeof(double) * 3 * (size_t)(n - ncon));
  return (int)inf[5];
}
