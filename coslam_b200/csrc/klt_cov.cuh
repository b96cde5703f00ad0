// klt_cov.cuh -- position covariance of every tracked KLT slot (cosl_klt_set_covariance, DESIGN.md
// section 3.4).  Runs after the tracker of an armed group, on the pyramids and the start table the
// tracker read and the table it returned; it changes nothing the tracker or the detector reads.
#pragma once
#include "klt_track.cuh"

namespace coslam {

// One warp per slot, grid (div_up(F, 8), C), 256 threads.  Level `level` of both pyramids (offset
// `off`, rows `pitch` texels apart) is the tracker's last.  Camera c's entry of `cams` gives its
// extent and, on a step's table, whether it was tracked.  The window is the tracker's own:
//   gain  taps one texel of the level apart around the centre (klt_centre, as klt_gain_*)
//   2x2   taps 2^level / W_c apart in normalised coordinates, each sampled on its own (klt_track_2x2)
// Slot i's normal matrix at the returned (x1, beta) is accumulated in fp32 and inverted in fp64:
//   gain  J = (jx, jy, -I0), M = J J^T, M[2][2] = sum (I0^2 + lambda |grad I0|^2) + 8 delta npx
//   2x2   J = (jx, jy), beta = 1
// with jx = (beta Ix0 + Ix1) W_c / 2, jy = (beta Iy0 + Iy1) H_c / 2.  The residual variance is
// noiseVar, or SSD / (npx - k) when noiseVar == 0 (k = 3 gain, 2).  cov[c][i] = (xx, xy, yy) of
// sigma^2 diag(W_c, H_c) [M^-1]_pos diag(W_c, H_c), level-0 pixels^2; NaN for a slot the tracker
// lost or did not start, a camera outside the tracker stage, or a singular M.
__global__ void __launch_bounds__(256)
klt_cov(const float4* __restrict__ pyr0, const float4* __restrict__ pyr1, long long pyrStride, long long off,
        int pitch, int level, const KltCam* __restrict__ cams, const float4* __restrict__ X0buf,
        const float4* __restrict__ res, float* __restrict__ cov, int F, int hw, int gain, float lambda,
        float delta, float noiseVar) {
  const int cam = blockIdx.y;
  const int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (slot >= F) return;
  const size_t k = (size_t)cam * F + slot;
  const float nan = __int_as_float(0x7fffffff);
  const float4 x0 = X0buf[k], r = res[k];
  if (!(__ldg(&cams[cam].stages) & KLT_STAGE_TRACK) || x0.x < 0.f || r.x < 0.f) {
    if (lane < 3) cov[3 * k + lane] = nan;
    return;
  }
  const int Wc = __ldg(&cams[cam].W), Hc = __ldg(&cams[cam].H);
  const int w = Wc >> level, h = Hc >> level;
  const float4* L0 = pyr0 + (size_t)cam * pyrStride + off;
  const float4* L1 = pyr1 + (size_t)cam * pyrStride + off;
  const float Wf = (float)Wc, Hf = (float)Hc;
  const float beta = gain ? r.z : 1.0f;
  const int fwid = 2 * hw + 1, npx = fwid * fwid;
  // gain: the window centres; 2x2: the normalised tap step
  const KltCentre c0 = klt_centre(w, h, x0.x, x0.y), c1 = klt_centre(w, h, r.x, r.y);
  const float dsx = (1.0f / Wf) * (float)(1 << level), dsy = (1.0f / Hf) * (float)(1 << level);
  float a = 0.f, b = 0.f, c = 0.f, p = 0.f, q = 0.f, m = 0.f, s = 0.f;
  for (int i = lane; i < npx; i += 32) {
    const int iy = i / fwid, ix = i - iy * fwid;
    float3 I0, I1;
    if (gain) {
      I0 = klt_fetch_global(L0, pitch, w, h, c0.xi + ix - hw, c0.yi + iy - hw, c0.ax, c0.ay);
      I1 = klt_fetch_global(L1, pitch, w, h, c1.xi + ix - hw, c1.yi + iy - hw, c1.ax, c1.ay);
    } else {
      const float fx = (float)(ix - hw), fy = (float)(iy - hw);
      I0 = klt_sample(L0, pitch, w, h, x0.x + fx * dsx, x0.y + fy * dsy);
      I1 = klt_sample(L1, pitch, w, h, r.x + fx * dsx, r.y + fy * dsy);
    }
    const float e = beta * I0.x - I1.x;
    const float jx = (beta * I0.y + I1.y) * Wf * 0.5f;
    const float jy = (beta * I0.z + I1.z) * Hf * 0.5f;
    a += jx * jx;
    b += jx * jy;
    c += jy * jy;
    p += jx * I0.x;
    q += jy * I0.x;
    m += I0.x * I0.x + lambda * (I0.y * I0.y + I0.z * I0.z);
    s += e * e;
  }
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  p = warp_sum(p);
  q = warp_sum(q);
  m = warp_sum(m);
  s = warp_sum(s);
  if (lane != 0) return;
  const double A = a, B = b, Cc = c;
  double det, i00, i01, i11;
  if (gain) {  // M = [[A, B, -P], [B, C, -Q], [-P, -Q, M22]]: the position block of its adjugate
    const double P = p, Q = q, M22 = (double)m + 8.0 * (double)delta * npx;
    i00 = Cc * M22 - Q * Q;
    i01 = P * Q - B * M22;
    i11 = A * M22 - P * P;
    det = A * i00 + B * i01 - P * (Cc * P - B * Q);
  } else {
    i00 = Cc;
    i01 = -B;
    i11 = A;
    det = A * Cc - B * B;
  }
  const int dof = npx - (gain ? 3 : 2);
  const double var = noiseVar > 0.f ? (double)noiseVar : dof > 0 ? (double)s / dof : nan;
  const double f = var / det;
  const double xx = f * i00 * Wf * Wf, xy = f * i01 * Wf * Hf, yy = f * i11 * Hf * Hf;
  const bool ok = det > 0.0 && isfinite(xx) && isfinite(xy) && isfinite(yy);
  cov[3 * k] = ok ? (float)xx : nan;
  cov[3 * k + 1] = ok ? (float)xy : nan;
  cov[3 * k + 2] = ok ? (float)yy : nan;
}

}  // namespace coslam
