// klt_undist.cuh -- undistorted pixel position and covariance of every KLT slot (cosl_klt_set_undistortion,
// DESIGN.md section 3.5).  Runs after the last writer of the feature table of an armed frame; it reads that
// table and the frame's position covariances (klt_cov.cuh) and changes nothing the tracker or the detector
// reads.
#pragma once
#include "klt_kernels.cuh"

namespace coslam {

// Camera c's lens: K2 = [[fx, s], [0, fy]], principal point (cx, cy), Bouguet's k_c = (k1, k2, p1, p2, k3),
// and the camera's own extent W x H, which turns the table's normalised positions into pixels.
struct KltUndistCam {
  double fx, s, cx, fy, cy;
  double k1, k2, p1, p2, k3;
  int W, H;
};

// Bouguet's / OpenCV's forward model d(x) at the normalised point (x, y) and its Jacobian J = dd/dx:
//   r2 = x^2 + y^2, a = 1 + k1 r2 + k2 r2^2 + k3 r2^3
//   d = (a x + 2 p1 x y + p2 (r2 + 2 x^2),  a y + p1 (r2 + 2 y^2) + 2 p2 x y)
__device__ __forceinline__ void klt_distort(const KltUndistCam& m, double x, double y, double& dx, double& dy,
                                            double& j00, double& j01, double& j10, double& j11) {
  const double r2 = x * x + y * y;
  const double a = 1.0 + r2 * (m.k1 + r2 * (m.k2 + r2 * m.k3));
  const double b = m.k1 + r2 * (2.0 * m.k2 + 3.0 * r2 * m.k3);  // da / d(r2)
  dx = a * x + 2.0 * m.p1 * x * y + m.p2 * (r2 + 2.0 * x * x);
  dy = a * y + m.p1 * (r2 + 2.0 * y * y) + 2.0 * m.p2 * x * y;
  const double c = 2.0 * x * y * b + 2.0 * m.p1 * x + 2.0 * m.p2 * y;
  j00 = a + 2.0 * x * x * b + 2.0 * m.p1 * y + 6.0 * m.p2 * x;
  j01 = c;
  j10 = c;
  j11 = a + 2.0 * y * y * b + 6.0 * m.p1 * y + 2.0 * m.p2 * x;
}

// One thread per slot, grid (div_up(F, 128), C), 128 threads.  Slot i of camera c:
//   (u_d, v_d) = (pos.x W_c, pos.y H_c), x_d = K2^-1 (u_d - cx, v_d - cy)
//   Newton from x = x_d, at most 20 steps x -= J^-1 (d(x) - x_d), stopping as soon as
//   |K2 (d(x) - x_d)|_inf <= 1e-9 px; fails when that is not met after 20 steps, when det J <= 0 at an
//   iterate or at the answer, or on a non-finite value
//   pos[c][i] = K2 x* + (cx, cy); with cov (the frame's position covariances, nullptr: not armed)
//   ucov[c][i] = A Sigma_d A^T, A = K2 J(x*)^-1 K2^-1, as (xx, xy, yy)
// NaN for a slot with status < 0, a failed inverse, and (ucov) a NaN entry of cov.
__global__ void __launch_bounds__(128)
klt_undistort(const cosl_klt_feature* __restrict__ feat, const float* __restrict__ cov,
              const KltUndistCam* __restrict__ cams, double* __restrict__ pos, float* __restrict__ ucov, int F) {
  const int cam = blockIdx.y;
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= F) return;
  const size_t k = (size_t)cam * F + slot;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const float nanf = __int_as_float(0x7fffffff);
  const KltUndistCam m = cams[cam];
  const cosl_klt_feature f = feat[k];
  const double ud = (double)f.pos[0] * m.W, vd = (double)f.pos[1] * m.H;
  const double yd = (vd - m.cy) / m.fy;
  const double xd = (ud - m.cx - m.s * yd) / m.fx;
  double x = xd, y = yd, j00 = 0.0, j01 = 0.0, j10 = 0.0, j11 = 0.0;
  bool ok = f.status >= 0 && isfinite(xd) && isfinite(yd);
  for (int it = 0; ok; ++it) {
    double dx, dy;
    klt_distort(m, x, y, dx, dy, j00, j01, j10, j11);
    const double det = j00 * j11 - j01 * j10;
    const double r0 = dx - xd, r1 = dy - yd;
    if (!(det > 0.0) || !isfinite(det) || !isfinite(r0) || !isfinite(r1)) {
      ok = false;
      break;
    }
    if (fmax(fabs(m.fx * r0 + m.s * r1), fabs(m.fy * r1)) <= 1e-9) break;
    if (it == 20) {
      ok = false;
      break;
    }
    x -= (j11 * r0 - j01 * r1) / det;
    y -= (j00 * r1 - j10 * r0) / det;
  }
  const double u = m.fx * x + m.s * y + m.cx, v = m.fy * y + m.cy;
  ok = ok && isfinite(u) && isfinite(v);
  pos[2 * k] = ok ? u : nan;
  pos[2 * k + 1] = ok ? v : nan;
  if (!cov) return;
  const double sxx = cov[3 * k], sxy = cov[3 * k + 1], syy = cov[3 * k + 2];
  // A = K2 J^-1 K2^-1, J^-1 = [[j11, -j01], [-j10, j00]] / det, K2^-1 = [[1/fx, -s/(fx fy)], [0, 1/fy]]
  const double det = j00 * j11 - j01 * j10;
  const double i00 = j11 / det, i01 = -j01 / det, i10 = -j10 / det, i11 = j00 / det;
  const double b00 = m.fx * i00 + m.s * i10, b01 = m.fx * i01 + m.s * i11;  // K2 J^-1
  const double b10 = m.fy * i10, b11 = m.fy * i11;
  const double q00 = 1.0 / m.fx, q01 = -m.s / (m.fx * m.fy), q11 = 1.0 / m.fy;
  const double a00 = b00 * q00, a01 = b00 * q01 + b01 * q11;
  const double a10 = b10 * q00, a11 = b10 * q01 + b11 * q11;
  // A Sigma A^T, Sigma = [[sxx, sxy], [sxy, syy]]
  const double t00 = a00 * sxx + a01 * sxy, t01 = a00 * sxy + a01 * syy;
  const double t10 = a10 * sxx + a11 * sxy, t11 = a10 * sxy + a11 * syy;
  const double cxx = t00 * a00 + t01 * a01, cxy = t00 * a10 + t01 * a11, cyy = t10 * a10 + t11 * a11;
  const bool cok = ok && isfinite(cxx) && isfinite(cxy) && isfinite(cyy);
  ucov[3 * k] = cok ? (float)cxx : nanf;
  ucov[3 * k + 1] = cok ? (float)cxy : nanf;
  ucov[3 * k + 2] = cok ? (float)cyy : nanf;
}

}  // namespace coslam
