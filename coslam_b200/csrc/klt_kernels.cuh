// klt_kernels.cuh -- device code of the pyramidal KLT tracker (sm_90a).
//
// Data layout in HBM (per tracker group, C cameras, camera-major).  W x H is the group's largest
// geometry (the maximum width and the maximum height over its cameras); every camera's slice is laid
// out at it, and camera c's data occupies the top-left W_c x H_c (level l: (W_c >> l) x (H_c >> l))
// of its slice.  Nothing reads the rest (KltCam):
//   image    u8   [C][H][imgPitch]
//   pyramid  float4 (I, Ix, Iy, 0) [2 buffers][C][sum_l w_l*h_l]   level l at offset lvOff[l], rows
//                                                                   w_l = W >> l texels apart
//   cornerness float [C][H][W]
//   feature buffers float4 (x, y, gain, _) [C][F]: src (X0), dst (provided), ping/pong/res
//   candidates u64 keys [C][candCap]: (~cornerness_bits << 32) | y << 16 | x  (ascending sort ==
//                                      cornerness desc, y asc, x asc)
//   dest     cosl_klt_feature [C][F]
//
// Arithmetic follows SURVEY.md Appendix A (reference shader citations in each kernel).  Pyramid and
// detector use explicitly non-fused IEEE operations in the oracle's order, so they are bit-exact
// against oracle/klt_oracle.cpp; the LK solve uses FMAs and warp-tree reductions (tolerance parity).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/coslam_b200.h"

namespace coslam {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// A copy of v the compiler cannot see through: what is derived from it is computed where it is
// used instead of being hoisted out of a loop and held in registers (or spilled) across it.
__device__ __forceinline__ int klt_opaque(int v) {
  asm volatile("" : "+r"(v));
  return v;
}

// One camera of a group whose cameras differ in size (cosl_klt_group_create_sizes): its level-0
// extent (level l is (W >> l) x (H >> l)) and its detector window.  Every kernel clamps its accesses
// to the camera's own level border, so the padding of a smaller camera's slice is never read as data.
//
// Each kernel that needs an extent is instantiated twice, selected by the group's sizes:
//   MIXED = false  the cameras are of one size: the kernel reads it from scalar kernel parameters (the
//                  group's W, H, detector window, validRegion), as for a single camera;
//   MIXED = true   the kernel reads its camera's entry of the table in global memory (the camera index
//                  may differ between the lane groups of a warp: a parameter array indexed with it
//                  would compile to chains of predicated constant loads).
// A table of kernel parameters indexed per block was measured too: its size slowed the launches of
// the uniform case, and a table read in every kernel added a memory round trip to each block.
struct KltCam {
  int W, H;
  int ixlo, ixhi, iylo, iyhi;  // detector window: pixels whose centre lies inside the margins
  int stages;                  // KLT_STAGE_* bits this camera takes part in (cosl_klt_group_step)
};

// Stages of a frame, per camera.  The group's own table has every bit set; cosl_klt_group_step
// runs the MIXED instantiations on a table of its own in which each camera carries the stages of
// its op (FIRST = PYR | DETECT, TRACK = PYR | TRACK, NEXT = all three, SKIP = none), and every
// kernel's blocks of a camera that does not take part in its stage exit.
enum { KLT_STAGE_PYR = 1, KLT_STAGE_TRACK = 2, KLT_STAGE_DETECT = 4, KLT_STAGE_ALL = 7 };

// MIXED: camera `cam` takes part in the stages `bits` (all of them); always true otherwise
template <bool MIXED>
__device__ __forceinline__ bool klt_in_stage(const KltCam* __restrict__ cams, int cam, int bits) {
  return !MIXED || (__ldg(&cams[cam].stages) & bits) == bits;
}

// extent of camera `cam`: its table entry, or the group's W x H when all cameras share it
template <bool MIXED>
__device__ __forceinline__ int2 klt_extent(const KltCam* __restrict__ cams, int cam, int W, int H) {
  if (MIXED) return make_int2(__ldg(&cams[cam].W), __ldg(&cams[cam].H));
  return make_int2(W, H);
}

// [1 3 3 1] / 8 tap of the pyramid levels l >= 1 (pyramid_with_derivative_pass2.cg:1-15, host
// v3d_gpupyramid.cpp:402-420), applied vertically then horizontally with decimation by 2 on all three
// channels by klt_front (level 1) and klt_pyr_down_tma (levels >= 2).
__device__ __forceinline__ float tap1331(float a, float b, float c, float d) {
  float r = __fadd_rn(a, __fmul_rn(3.0f, b));
  r = __fadd_rn(r, __fmul_rn(3.0f, c));
  r = __fadd_rn(r, d);
  return __fmul_rn(r, 0.125f);  // == r / 8 exactly
}

// ------------------------------------------------------------------------------------------
// Bilinear sampling of a pyramid level with clamp-to-edge (SURVEY Appendix A.3).
// ------------------------------------------------------------------------------------------
// pitch: row pitch of the level in texels; w x h: the camera's extent of the level
__device__ __forceinline__ float3 klt_sample(const float4* __restrict__ lv, int pitch, int w, int h,
                                             float s, float t) {
  float u = s * (float)w - 0.5f;
  float v = t * (float)h - 0.5f;
  u = fminf(fmaxf(u, -2.0f), (float)w + 1.0f);
  v = fminf(fmaxf(v, -2.0f), (float)h + 1.0f);
  const float fu = floorf(u), fv = floorf(v);
  const float ax = u - fu, ay = v - fv;
  const int xi = (int)fu, yi = (int)fv;
  const int x0 = clampi(xi, 0, w - 1), x1 = clampi(xi + 1, 0, w - 1);
  const int y0 = clampi(yi, 0, h - 1), y1 = clampi(yi + 1, 0, h - 1);
  const float4 p00 = __ldg(&lv[(size_t)y0 * pitch + x0]);
  const float4 p10 = __ldg(&lv[(size_t)y0 * pitch + x1]);
  const float4 p01 = __ldg(&lv[(size_t)y1 * pitch + x0]);
  const float4 p11 = __ldg(&lv[(size_t)y1 * pitch + x1]);
  float3 r;
  {
    const float top = p00.x + ax * (p10.x - p00.x), bot = p01.x + ax * (p11.x - p01.x);
    r.x = top + ay * (bot - top);
  }
  {
    const float top = p00.y + ax * (p10.y - p00.y), bot = p01.y + ax * (p11.y - p01.y);
    r.y = top + ay * (bot - top);
  }
  {
    const float top = p00.z + ax * (p10.z - p00.z), bot = p01.z + ax * (p11.z - p01.z);
    r.z = top + ay * (bot - top);
  }
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// W, H, vr*: the group's (MIXED = false); a mixed group's kernels use the camera's extent and derive
// the strict validRegion from `margin` (klt_vr_lo / klt_vr_hi)
struct KltTrackParams {
  int W, H, F, halfWidth;
  float sqrConv, ssdThr;
  float vr0, vr1, vr2, vr3;  // validRegion
  float lambda, delta;
  int strict;    // this set holds the strict validRegion (not the lax one, -1 .. 2)
  float margin;  // trackBorderMargin (pixels)
};

// validRegion of a strict pass for a camera of n pixels along the axis: margin / n and
// 1 - margin / n, the same correctly rounded fp32 values the host computes (v3d_gpuklt.cpp:266-270)
__device__ __forceinline__ float klt_vr_lo(float margin, int n) { return __fdiv_rn(margin, (float)n); }
__device__ __forceinline__ float klt_vr_hi(float margin, int n) {
  return __fsub_rn(1.0f, __fdiv_rn(margin, (float)n));
}

// w, h: the group's level sizes (largest camera), also the row pitch of the level in texels
struct KltLevels {
  int n;             // number of levels visited
  int level[8];
  int w[8], h[8];
  long long off[8];
  float mult[8];
};

// ------------------------------------------------------------------------------------------
// 2x2 LK (klt_tracker.cg:24-132): all levels and iterations inside one kernel, one warp per
// feature.  Output (X1.x, X1.y, X0.x) or -1.
// ------------------------------------------------------------------------------------------

template <bool MIXED>
__global__ void __launch_bounds__(256)
klt_track_2x2(const float4* __restrict__ pyr0, const float4* __restrict__ pyr1, long long pyrStride,
              KltLevels LV, const KltCam* __restrict__ cams, const float4* __restrict__ X0buf,
              float4* __restrict__ out, KltTrackParams P, int nIter) {
  const int cam = blockIdx.y;
  if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) return;
  const int2 ext = klt_extent<MIXED>(cams, cam, P.W, P.H);
  const int Wc = ext.x, Hc = ext.y;
  const int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (slot >= P.F) return;
  const size_t fb = (size_t)cam * P.F;
  const float4 x0 = X0buf[fb + slot];
  const float X0x = x0.x, X0y = x0.y;
  float X1x = X0x, X1y = X0y;
  bool invalid = (X1x < 0.f);
  const int hw = P.halfWidth, fwid = 2 * hw + 1, npx = fwid * fwid;
  const float Wf = (float)Wc, Hf = (float)Hc;
  const float dsx = 1.0f / Wf, dsy = 1.0f / Hf;
  float sqrLen = 0.f, ssd = 0.f;
  for (int li = 0; li < LV.n; ++li) {
    const float4* L0 = pyr0 + (size_t)cam * pyrStride + LV.off[li];
    const float4* L1 = pyr1 + (size_t)cam * pyrStride + LV.off[li];
    const int pitch = LV.w[li];
    const int w = MIXED ? Wc >> LV.level[li] : LV.w[li], h = MIXED ? Hc >> LV.level[li] : LV.h[li];
    const float dx = dsx * LV.mult[li], dy = dsy * LV.mult[li];
    for (int it = 0; it < nIter; ++it) {
      float a = 0, b = 0, c = 0, r0 = 0, r1 = 0;
      ssd = 0;
      for (int p = lane; p < npx; p += 32) {
        const int py = p / fwid, px = p - py * fwid;
        const float fx = (float)(px - hw), fy = (float)(py - hw);
        const float3 I0 = klt_sample(L0, pitch, w, h, X0x + fx * dx, X0y + fy * dy);
        const float3 I1 = klt_sample(L1, pitch, w, h, X1x + fx * dx, X1y + fy * dy);
        const float e = I0.x - I1.x;
        const float Jx = (I0.y + I1.y) * Wf * 0.5f;
        const float Jy = (I0.z + I1.z) * Hf * 0.5f;
        a += Jx * Jx;
        b += Jx * Jy;
        c += Jy * Jy;
        r0 += e * Jx;
        r1 += e * Jy;
        ssd += e * e;
      }
      a = warp_sum(a);
      b = warp_sum(b);
      c = warp_sum(c);
      r0 = warp_sum(r0);
      r1 = warp_sum(r1);
      ssd = warp_sum(ssd);
      const float det = a * c - b * b;
      invalid = invalid || (det < 0.00001f);
      const float rdet = 1.0f / det;
      float ux = rdet * (c * r0 - b * r1);
      float uy = rdet * (-b * r0 + a * r1);
      X1x += ux;
      X1y += uy;
      ux *= Wf;
      uy *= Hf;
      sqrLen = ux * ux + uy * uy;
    }
    invalid = invalid || (sqrLen > P.sqrConv);
    invalid = invalid || (ssd > P.ssdThr);
  }
  if (MIXED)
    invalid = invalid || (X1x < klt_vr_lo(P.margin, Wc) || X1y < klt_vr_lo(P.margin, Hc)) ||
              (X1x > klt_vr_hi(P.margin, Wc) || X1y > klt_vr_hi(P.margin, Hc));
  else
    invalid = invalid || (X1x < P.vr0 || X1y < P.vr1) || (X1x > P.vr2 || X1y > P.vr3);
  if (lane == 0)
    out[fb + slot] = invalid ? make_float4(-1.f, -1.f, -1.f, 0.f) : make_float4(X1x, X1y, X0x, 0.f);
}

// ------------------------------------------------------------------------------------------
// KLT_SequenceTracker::track host loop (v3d_gpuklt.cpp:872-888) on the device: tracker output ->
// dest entries + per-camera count of present features.  counters[cam*8 + 0] = nPresent.
// MIXED: only the cameras of the tracker stage (cams, KltCam::stages).
// ------------------------------------------------------------------------------------------
template <bool MIXED>
__global__ void klt_status(const float4* __restrict__ res, cosl_klt_feature* __restrict__ dest,
                           int* __restrict__ counters, int F, const KltCam* __restrict__ cams) {
  const int cam = blockIdx.y;
  if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool live = false;
  if (i < F) {
    const float4 r = res[(size_t)cam * F + i];
    cosl_klt_feature f;
    if (r.x >= 0.f) {
      f.status = 0;
      f.pos[0] = r.x;
      f.pos[1] = r.y;
      f.gain = r.z;
      live = true;
    } else {
      f.status = -1;
      f.pos[0] = f.pos[1] = -1.0f;
      f.gain = 1.0f;
    }
    f.fed = -1;
    dest[(size_t)cam * F + i] = f;
  }
  const unsigned m = __ballot_sync(0xffffffffu, live);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&counters[cam * 8 + 0], __popc(m));
}

// Suppress detection at the pixel of every live point (presentFeaturesShader, v3d_gpuklt.cpp:475-500).
// pts: float4 (x, y, .., ..) per slot, x < 0 == dead (clipped).  Camera c reads nPer[c] points when
// nPer is given (present lists of different lengths), else n.
// The cornerness map of camera c: rows `pitch` floats apart, `cornStride` floats per camera.
// MIXED: only the cameras that take part in all of the stages `bits`.
template <bool MIXED>
__global__ void klt_suppress(const float4* __restrict__ pts, int n, const int* __restrict__ nPer,
                             int ptsStride, float* __restrict__ corn, int pitch, long long cornStride,
                             const KltCam* __restrict__ cams, int W, int H, int bits) {
  const int cam = blockIdx.y;
  if (!klt_in_stage<MIXED>(cams, cam, bits)) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (nPer ? nPer[cam] : n)) return;
  const float4 p = pts[(size_t)cam * ptsStride + i];
  if (!(p.x >= 0.0f && p.x < 1.0f && p.y >= 0.0f && p.y < 1.0f)) return;
  if (MIXED) {
    W = __ldg(&cams[cam].W);
    H = __ldg(&cams[cam].H);
  }
  const int ix = (int)floorf(__fmul_rn(p.x, (float)W)), iy = (int)floorf(__fmul_rn(p.y, (float)H));
  if (ix >= 0 && ix < W && iy >= 0 && iy < H) corn[(size_t)cam * cornStride + (size_t)iy * pitch + ix] = -1e30f;
}

// ------------------------------------------------------------------------------------------
// Non-max suppression + compaction (klt_detector_nonmax.cg:12-26, run by the reference as a
// horizontal then a vertical pass with the sign trick "m = c if |c| > max|n| else -max|n|").
// The two passes leave a positive value exactly at pixels with c > 0 whose value is STRICTLY
// larger than |v| of every other texel v of their (2r+1)^2 window (klt_suppress marks live points
// with -1e30, which therefore clears their whole neighbourhood), the window being read with
// CLAMP_TO_EDGE (so a pixel on the image border, whose window contains a clamped copy of itself,
// never survives).  That predicate is evaluated directly, candidate driven:
//   klt_nm_prefilter  one streaming pass: pixels with c > 0 that beat |.| of their (2p+1)^2
//                     neighbourhood, p = min(r, 3) -- a necessary condition, at most one pixel per
//                     2x2 block passes -> prelim list
//   klt_nm_verify     one warp per prelim pixel checks the remaining window texels (L2 resident)
//                     and appends the survivors' sort keys
// The cornerness map is mostly zero after thresholding, so the second kernel touches a few
// percent of the pixels; the map is read from HBM once (4 B/px).
// counters[cam*8+4] = prelim count, counters[cam*8+1] = candidate count.
// ------------------------------------------------------------------------------------------
constexpr int NP_ROWS = 16;  // rows per warp in klt_nm_prefilter

// PR = prefilter radius (1..3, <= the suppression radius r): lanes PR .. 31-PR produce outputs.
template <int PR, bool MIXED>
__global__ void __launch_bounds__(256)
klt_nm_prefilter(const float* __restrict__ corn, int pitch, long long cornStride,
                 const KltCam* __restrict__ cams, int W, int H, unsigned* __restrict__ prelim,
                 int prelimCap, int* __restrict__ counters) {
  constexpr int NCOLS = 32 - 2 * PR, NR = 2 * PR + 1;
  const int cam = blockIdx.z;
  if (MIXED) {
    W = __ldg(&cams[cam].W);
    H = __ldg(&cams[cam].H);
    if ((int)blockIdx.x * NCOLS >= W) return;  // the block's output columns lie outside this camera
    if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_DETECT)) return;
  }
  const float* cm = corn + (size_t)cam * cornStride;
  const int lane = threadIdx.x & 31;
  const int x = blockIdx.x * NCOLS - PR + lane;                        // unclamped column
  const int y0 = (blockIdx.y * 8 + (threadIdx.x >> 5)) * NP_ROWS;      // first output row
  if (y0 >= H) return;
  const int cx = clampi(x, 0, W - 1);
  // all NP_ROWS + 2 PR rows of this column in flight at once
  float v[NP_ROWS + 2 * PR];
#pragma unroll
  for (int k = 0; k < NP_ROWS + 2 * PR; ++k)
    v[k] = fabsf(__ldg(&cm[(size_t)clampi(y0 - PR + k, 0, H - 1) * pitch + cx]));
  // The clamped loads make the window of a pixel near the image border contain copies of the edge
  // texels, which is exactly what the reference's CLAMP_TO_EDGE window contains there.
  const bool colOK = (lane >= PR) && (lane < PR + NCOLS) && (x < W);
  // horizontal maxima of |.| over columns x-PR .. x+PR: with the centre (incl) and without (excl)
  auto hmax = [&](float c, float& incl, float& excl) {
    float m = 0.f;  // |.| >= 0: neutral
#pragma unroll
    for (int d = 1; d <= PR; ++d)
      m = fmaxf(m, fmaxf(__shfl_up_sync(0xffffffffu, c, d), __shfl_down_sync(0xffffffffu, c, d)));
    excl = m;
    incl = fmaxf(m, c);
  };
  float hm[NR], hx[NR];  // rows y-PR .. y+PR of the row under test
#pragma unroll
  for (int q = 1; q < NR; ++q) hmax(v[q - 1], hm[q], hx[q]);
  unsigned mine = 0;  // bit k: this lane's pixel of row y0 + k is a preliminary candidate
#pragma unroll
  for (int k = 0; k < NP_ROWS; ++k) {
    // rows y-PR .. y+PR are v[k] .. v[k+2PR]: slide, then add the new bottom row
#pragma unroll
    for (int q = 0; q + 1 < NR; ++q) {
      hm[q] = hm[q + 1];
      hx[q] = hx[q + 1];
    }
    hmax(v[k + 2 * PR], hm[NR - 1], hx[NR - 1]);
    const int y = y0 + k;
    // |c| == c for a positive candidate; a suppressed centre (-1e30) has |c| = 1e30 and passes here,
    // but klt_nm_verify re-reads the signed value and drops it
    const float c = v[k + PR];
    float others = hx[PR];
#pragma unroll
    for (int q = 0; q < NR; ++q)
      if (q != PR) others = fmaxf(others, hm[q]);
    if (colOK && (y < H) && (c > 0.f) && (c > others)) mine |= 1u << k;
  }
  // one atomic per warp: exclusive prefix of the per-lane counts, then every lane writes its own
  if (!__any_sync(0xffffffffu, mine != 0)) return;
  const int cnt = __popc(mine);
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  int base = 0;
  if (lane == 31) base = atomicAdd(&counters[cam * 8 + 4], incl);
  base = __shfl_sync(0xffffffffu, base, 31);
  int idx = base + incl - cnt;
  while (mine) {
    const int k = __ffs(mine) - 1;
    mine &= mine - 1;
    if (idx < prelimCap) prelim[(size_t)cam * prelimCap + idx] = ((unsigned)(y0 + k) << 16) | (unsigned)x;
    ++idx;
  }
}

constexpr int NV_BATCH = 4;  // candidates a warp examines together (independent loads in flight)

template <bool MIXED>
__global__ void __launch_bounds__(256)
klt_nm_verify(const float* __restrict__ corn, int pitch, long long cornStride,
              const KltCam* __restrict__ cams, int W, int H, int r, const unsigned* __restrict__ prelim,
              int prelimCap, unsigned long long* __restrict__ cand, int candCap, int* __restrict__ counters) {
  const int cam = blockIdx.y;
  if (MIXED) {
    if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_DETECT)) return;
    W = __ldg(&cams[cam].W);
    H = __ldg(&cams[cam].H);
  }
  // Launched as a programmatic dependent of the kernel ahead of it on the group's stream: the
  // prefilter on a detect frame, the tracker or klt_suppress on a re-detect frame.  Above, only the
  // camera table is read, which work ahead of that kernel wrote.  The prelim list, its count and
  // the cornerness map (its centre values and windows marked by the tracker) are read after the
  // wait, which returns once that grid has completed and its stores are visible.  The trigger
  // follows the wait, so klt_select_refill, which reads the tracker's feature table before its own
  // wait, starts only after a wait here has returned.  A CTA of a camera outside the detector stage
  // exits above, which counts as a trigger; its camera's select CTA exits before it reads anything.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const float* cm = corn + (size_t)cam * cornStride;
  const int lane = threadIdx.x & 31;
  const int warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int n = min(counters[cam * 8 + 4], prelimCap);
  const int side = 2 * r + 1, nwin = side * side;
  // window texel k (rows from the centre outwards: 0, -1, +1, -2, ...)
  auto beaten_by = [&](int k, int x, int y, float c) -> bool {
    if (k >= nwin) return false;
    const int ri = k / side, dx = k - ri * side - r;
    const int dy = (ri & 1) ? -((ri + 1) >> 1) : (ri >> 1);
    const float v = __ldg(&cm[(size_t)clampi(y + dy, 0, H - 1) * pitch + clampi(x + dx, 0, W - 1)]);
    return ((dx | dy) != 0) && !(c > fabsf(v));
  };
  for (int i0 = warp * NV_BATCH; i0 < n; i0 += nwarps * NV_BATCH) {
    unsigned p[NV_BATCH];
    float c[NV_BATCH];
    bool b[NV_BATCH];
#pragma unroll
    for (int j = 0; j < NV_BATCH; ++j) p[j] = (i0 + j < n) ? prelim[(size_t)cam * prelimCap + i0 + j] : 0u;
#pragma unroll
    for (int j = 0; j < NV_BATCH; ++j)  // signed value: negative if suppressed meanwhile
      c[j] = (i0 + j < n) ? __ldg(&cm[(size_t)(p[j] >> 16) * pitch + (p[j] & 0xffffu)]) : -1.0f;
    // first 32 texels (the centre row and most of the one above) of every candidate of the batch in
    // one memory round trip; the few candidates that are still unbeaten walk the rest of their
    // window 32 texels at a time and leave at the first larger value (reading whole windows
    // unconditionally was measured slower: the kernel is bound by L1 requests, not by latency)
#pragma unroll
    for (int j = 0; j < NV_BATCH; ++j) b[j] = beaten_by(lane, (int)(p[j] & 0xffffu), (int)(p[j] >> 16), c[j]);
#pragma unroll
    for (int j = 0; j < NV_BATCH; ++j) {
      bool beaten = !(c[j] > 0.f) || __any_sync(0xffffffffu, b[j]);
      const int x = (int)(p[j] & 0xffffu), y = (int)(p[j] >> 16);
      for (int k0 = 32; k0 < nwin && !beaten; k0 += 32)
        beaten = __any_sync(0xffffffffu, beaten_by(k0 + lane, x, y, c[j]));
      if (!beaten && lane == 0) {
        const int idx = atomicAdd(&counters[cam * 8 + 1], 1);
        if (idx < candCap) {
          const unsigned cb = ~__float_as_uint(c[j]);
          cand[(size_t)cam * candCap + idx] =
              ((unsigned long long)cb << 32) | ((unsigned long long)y << 16) | (unsigned long long)x;
        }
      }
    }
  }
}

constexpr int KLT_MAX_SMEM_KEYS = 16384;  // keys sorted in shared memory; more sort in global memory

// Exclusive prefix over the block of v (one value per thread), and the block's sum in total.  s_w
// holds 33 ints; it is free again when the call returns.
__device__ __forceinline__ int klt_block_excl_scan(int v, int* s_w, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_w[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const int w = (lane < (int)(blockDim.x >> 5)) ? s_w[lane] : 0;
    int wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    s_w[lane] = wi - w;  // exclusive prefix of the warp totals
    if (lane == 31) s_w[32] = wi;
  }
  __syncthreads();
  const int r = s_w[wid] + inc - v;
  total = s_w[32];
  __syncthreads();
  return r;
}

// The largest key T such that exactly k of the n distinct keys ck[0..n) are <= T (1 <= k < n): a
// radix select from the most significant byte down.  Each pass histograms the byte below the prefix
// found so far over the keys that carry that prefix; the bin holding the k-th key becomes the new
// prefix, and the select ends at the first pass where the k-th key is the last of its bin, so T is the
// largest key with that prefix.  The keys are distinct, so that happens at the last byte at the latest.
// s_hist holds 256 ints, s_sel 3.
__device__ __forceinline__ unsigned long long klt_select_threshold(const unsigned long long* __restrict__ ck, int n, int k,
                                                   int* s_hist, int* s_sel) {
  const int lane = threadIdx.x & 31;
  unsigned long long prefix = 0, pmask = 0;
  for (int shift = 56;; shift -= 8) {
    if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long key = ck[i];
      if ((key & pmask) == prefix) atomicAdd(&s_hist[(unsigned)(key >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {  // warp 0: lane l owns bins 8l .. 8l+7
      int h[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        h[j] = s_hist[8 * lane + j];
        sum += h[j];
      }
      int inc = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      int before = inc - sum;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (before < k && k <= before + h[j]) {  // exactly one bin of one lane
          s_sel[0] = 8 * lane + j;
          s_sel[1] = k - before;
          s_sel[2] = (k - before) == h[j];
        }
        before += h[j];
      }
    }
    __syncthreads();
    const int digit = s_sel[0], kr = s_sel[1], closes = s_sel[2];
    prefix |= (unsigned long long)digit << shift;
    pmask |= 0xffull << shift;
    if (closes) return prefix | ~pmask;  // the k-th key is the last of its bin
    k = kr;
    // s_sel and s_hist are rewritten only after the next pass's first barrier
  }
}

// ------------------------------------------------------------------------------------------
// Single-CTA per camera: the strongest candidates in increasing key order, then the slot logic of
// KLT_SequenceTracker::{detect, redetect} (v3d_gpuklt.cpp:651-805) on the device:
//   mode 0 (detect):   slots [0, nDet) <- strongest corners, [nDet, nDet+nPresent) <- present pts
//                      (nPresent = nPresentExt[cam], 0 when nPresentExt is null)
//   mode 1 (redetect): dead slots, in increasing slot index, <- strongest corners
//   mode 2 (MIXED):    per camera, 1 for a camera of the tracker stage, else 0
//                      (cosl_klt_group_step; the cameras outside the detector stage exit)
// and "provide" the new feature table (dst buffer).  counters[cam*8+2] = returned count
// (nDetected / nNewFeatures as the reference defines them), [3] = raw candidate count.
//
// Only the first nSel = min(nCand, plCap, free slots) keys of the sorted list are used.  The keys
// (~cornerness | y | x) are distinct, so those are one set in one order: a radix select finds the
// nSel-th key, the keys at or below it are compacted into shared memory and only they are sorted
// (bitonic, next_pow2(nSel) <= next_pow2(F) keys).  Only a group with more than KLT_MAX_SMEM_KEYS
// slots can have more winners than shared memory holds; it sorts every key in global memory.
// COSL_KLT_COMPAT_HISTOPYR needs the whole candidate list in Morton order and sorts all of it.
//
// Dynamic shared memory: smemKeys keys, then one int per 32 slots (the dead slots ahead of them).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void bitonic_sort(unsigned long long* k, int n2) {
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (n2 >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));  // index with bit `stride` cleared
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = k[lo], b = k[hi];
        if ((a > b) == up) {
          k[lo] = b;
          k[hi] = a;
        }
      }
    }
  }
  __syncthreads();
}

// Morton code with x in the even bits: the extraction order of the reference's HistoPyramid traversal
// (klt_detector_traverse_histpyr.cg:33-50 visits the children (x,y), (x+1,y), (x,y+1), (x+1,y+1) in that
// order at every level; the 2x2 taps of the base level have the same order, v3d_gpuklt.cpp:42-57)
__device__ __forceinline__ unsigned klt_part1by1(unsigned v) {
  v &= 0xffffu;
  v = (v | (v << 8)) & 0x00ff00ffu;
  v = (v | (v << 4)) & 0x0f0f0f0fu;
  v = (v | (v << 2)) & 0x33333333u;
  v = (v | (v << 1)) & 0x55555555u;
  return v;
}
__device__ __forceinline__ unsigned klt_compact1by1(unsigned v) {
  v &= 0x55555555u;
  v = (v | (v >> 1)) & 0x33333333u;
  v = (v | (v >> 2)) & 0x0f0f0f0fu;
  v = (v | (v >> 4)) & 0x00ff00ffu;
  v = (v | (v >> 8)) & 0x0000ffffu;
  return v;
}

// (1024, 1): with the block count left open ptxas kept the kernel at 32 registers, and it spilled
template <bool MIXED>
__global__ void __launch_bounds__(1024, 1)
klt_select_refill(unsigned long long* __restrict__ cand, int candCap, int plCap,
                  int* __restrict__ counters, cosl_klt_feature* __restrict__ dest,
                  float4* __restrict__ dstbuf, float4* __restrict__ alsoSrc,
                  const float4* __restrict__ present, const int* __restrict__ nPresentPer,
                  int F, const KltCam* __restrict__ cams, int W, int H, int mode, int withGain,
                  int smemKeys, int histo) {
  extern __shared__ unsigned long long s_keys[];
  __shared__ int s_w[33];
  __shared__ int s_hist[256];
  __shared__ int s_sel[3];
  __shared__ int s_nWin, s_nDead;
  const int cam = blockIdx.x;
  if (MIXED) {
    const int stages = __ldg(&cams[cam].stages);
    if (!(stages & KLT_STAGE_DETECT)) return;
    if (mode == 2) mode = (stages & KLT_STAGE_TRACK) ? 1 : 0;  // per camera: re-detect after a track
  }
  const int lane = threadIdx.x & 31;
  cosl_klt_feature* d = dest + (size_t)cam * F;
  int* s_dead = reinterpret_cast<int*>(s_keys + smemKeys);  // dead slots ahead of each 32-slot group
  if (mode == 1) {
    // Launched as a programmatic dependent of klt_nm_verify, whose CTAs trigger only after their own
    // griddepcontrol.wait returned, i.e. after the grid ahead of verify completed.  That is the
    // tracker (the fused gain tracker writes the feature table itself), klt_status or klt_suppress,
    // each behind the table's last writer on the same stream, so the table read here is complete
    // and visible.  Nothing this CTA reads or writes in global memory before its own wait is touched
    // by verify.  This scan is what the refill would do after the wait: dead slots get ranks in
    // increasing slot index.
    const int nGroups = (F + 31) >> 5;
    for (int gi = threadIdx.x >> 5; gi < nGroups; gi += blockDim.x >> 5) {
      const int i = gi * 32 + lane;
      const unsigned bal = __ballot_sync(0xffffffffu, i < F && d[i].status < 0);
      if (lane == 0) s_dead[gi] = __popc(bal);
    }
    __syncthreads();
    int nDead = 0;
    for (int s = 0; s < nGroups; s += blockDim.x) {
      const int gi = s + threadIdx.x;
      int tot;
      const int ex = klt_block_excl_scan(gi < nGroups ? s_dead[gi] : 0, s_w, tot);
      if (gi < nGroups) s_dead[gi] = nDead + ex;
      nDead += tot;
    }
    if (threadIdx.x == 0) s_nDead = nDead;  // read by the same thread after the wait
  }
  // Everything below reads what verify (the candidate keys and their count) or the work ahead of it
  // wrote.  Triggering after the wait lets the stream's next kernel, if it is a programmatic launch,
  // be placed while this one runs; it waits for this grid to complete before it reads.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  int* cnt = counters + cam * 8;
  unsigned long long* ck = cand + (size_t)cam * candCap;
  const int nCand = min(cnt[1], candCap);
  // the present counts are read again after the selection, so that they are not live across it
  const int freeSlots = F - ((mode == 0) ? (nPresentPer ? nPresentPer[cam] : 0) : cnt[0]);
  unsigned long long* keys = s_keys;
  int nSel;
  if (histo) {
    // COSL_KLT_COMPAT_HISTOPYR: the reference's candidate list.  (1) the discriminator pass covers W/2 x H/2
    // texels of 2x2 pixels (v3d_gpuklt.cpp:519-523): a last odd row / column is never seen; (2) the first
    // plCap candidates in HistoPyramid extraction order (= Morton order) are read back (:752-757);
    // (3) only if they exceed the free slots they are ordered by cornerness (:759-768), else they fill
    // the slots in extraction order.
    if (MIXED) {
      W = __ldg(&cams[cam].W);
      H = __ldg(&cams[cam].H);
    }
    int n2 = 1;
    while (n2 < nCand) n2 <<= 1;
    if (n2 <= smemKeys) {
      for (int i = threadIdx.x; i < n2; i += blockDim.x) keys[i] = (i < nCand) ? ck[i] : ~0ull;
    } else {
      keys = ck;  // sort in place in global memory (candCap is a power of two >= n2)
      for (int i = nCand + threadIdx.x; i < n2; i += blockDim.x) keys[i] = ~0ull;
    }
    __syncthreads();
    __shared__ int s_nvalid;
    const unsigned Wc = 2u * (unsigned)(W / 2), Hc = 2u * (unsigned)(H / 2);
    if (threadIdx.x == 0) s_nvalid = 0;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
      unsigned long long k = keys[i];
      if (k != ~0ull) {
        const unsigned x = (unsigned)(k & 0xffff), y = (unsigned)((k >> 16) & 0xffff);
        if (x >= Wc || y >= Hc)
          k = ~0ull;
        else
          k = ((unsigned long long)(klt_part1by1(x) | (klt_part1by1(y) << 1)) << 32) | (k >> 32);
      }
      keys[i] = k;
    }
    __syncthreads();
    if (nCand > 1) bitonic_sort(keys, n2);
    for (int i = threadIdx.x; i < n2; i += blockDim.x)
      if (keys[i] != ~0ull && (i + 1 == n2 || keys[i + 1] == ~0ull)) s_nvalid = i + 1;
    __syncthreads();
    const int nCandEff = min(s_nvalid, plCap);
    const bool wantSort = nCandEff > freeSlots;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
      unsigned long long k = keys[i];
      if (i < nCandEff) {
        const unsigned mc = (unsigned)(k >> 32);
        const unsigned x = klt_compact1by1(mc), y = klt_compact1by1(mc >> 1);
        k = ((k & 0xffffffffull) << 32) | ((unsigned long long)y << 16) | x;
      } else {
        k = ~0ull;
      }
      keys[i] = k;
    }
    __syncthreads();
    if (nCand > 1 && wantSort) bitonic_sort(keys, n2);
    nSel = max(0, min(nCandEff, freeSlots));
  } else {
    nSel = max(0, min(min(nCand, plCap), freeSlots));
    int n2 = 1;
    while (n2 < nSel) n2 <<= 1;
    if (n2 <= smemKeys) {
      if (nSel > 0) {
        const unsigned long long T = (nSel < nCand) ? klt_select_threshold(ck, nCand, nSel, s_hist, s_sel) : ~0ull;
        if (threadIdx.x == 0) s_nWin = 0;
        __syncthreads();
        // exactly nSel keys are <= T; one shared-memory atomic per warp and round
        for (int s = 0; s < nCand; s += blockDim.x) {
          const int i = s + threadIdx.x;
          const unsigned long long key = (i < nCand) ? ck[i] : ~0ull;
          const bool win = (i < nCand) && key <= T;
          const unsigned bal = __ballot_sync(0xffffffffu, win);
          int base = 0;
          if (lane == 0 && bal) base = atomicAdd(&s_nWin, __popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (win) keys[base + __popc(bal & ((1u << lane) - 1))] = key;
        }
      }
      for (int i = nSel + threadIdx.x; i < n2; i += blockDim.x) keys[i] = ~0ull;
      __syncthreads();
      if (nSel > 1) bitonic_sort(keys, n2);
    } else {
      // more winners than shared memory holds (more than KLT_MAX_SMEM_KEYS slots): sort every key in place
      n2 = 1;
      while (n2 < nCand) n2 <<= 1;
      keys = ck;
      for (int i = nCand + threadIdx.x; i < n2; i += blockDim.x) keys[i] = ~0ull;
      __syncthreads();
      if (nCand > 1) bitonic_sort(keys, n2);
    }
  }
  const int nPresentExt = (mode == 0 && nPresentPer) ? nPresentPer[cam] : 0;
  // written ahead of the refill so that no count stays live across it
  if (threadIdx.x == 0) {
    const int nCandRaw = cnt[1];
    cnt[2] = (mode == 0) ? nSel + nPresentExt : min(nSel, s_nDead) + cnt[0];
    cnt[3] = nCandRaw;
  }
  if (MIXED) {  // read here rather than at the top, so that they are not live across the selection
    W = __ldg(&cams[cam].W);
    H = __ldg(&cams[cam].H);
  }
  const float Wf = (float)W, Hf = (float)H;
  float4* pb = dstbuf + (size_t)cam * F;
  float4* ps = alsoSrc ? alsoSrc + (size_t)cam * F : nullptr;  // advanceFrame copy folded in
  if (mode == 0) {
    const int nDet = nSel;
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
      cosl_klt_feature f;
      float4 p;
      if (i < nDet) {
        const unsigned long long key = keys[i];
        const float c = __uint_as_float(~(unsigned)(key >> 32));
        const int py = (int)((key >> 16) & 0xffff), px = (int)(key & 0xffff);
        f.status = 1;
        f.pos[0] = __fdiv_rn(__fadd_rn((float)px, 0.5f), Wf);
        f.pos[1] = __fdiv_rn(__fadd_rn((float)py, 0.5f), Hf);
        f.gain = withGain ? 1.0f : c;
        f.fed = -1;
        p = make_float4(f.pos[0], f.pos[1], f.gain, 0.f);
      } else if (i < nDet + nPresentExt) {
        const float4 q = present[(size_t)cam * F + (i - nDet)];
        f.status = 1;
        f.pos[0] = q.x;
        f.pos[1] = q.y;
        f.gain = 1.0f;
        f.fed = i - nDet;
        p = make_float4(q.x, q.y, 1.0f, 0.f);
      } else {
        f.status = -1;
        f.pos[0] = f.pos[1] = -1.0f;
        f.gain = 1.0f;
        f.fed = -1;
        p = make_float4(-1.f, -1.f, 1.f, 0.f);
      }
      d[i] = f;
      pb[i] = p;
      if (ps) ps[i] = p;
    }
  } else {
    const int nNew = nSel;
    // dead slot i gets corner k = its rank among the dead slots (the scan before the wait); a warp
    // covers one 32-slot group per round (blockDim.x is a multiple of 32), so the round's ballot
    // gives the rank within the group
    for (int s = 0; s < F; s += blockDim.x) {
      const int i = s + threadIdx.x;
      const bool dead = (i < F) && (d[i].status < 0);
      const unsigned bal = __ballot_sync(0xffffffffu, dead);
      if (i < F) {
        float4 p;
        if (dead) {
          const int rank = s_dead[i >> 5] + __popc(bal & ((1u << lane) - 1));
          if (rank < nNew) {
            const unsigned long long key = keys[rank];
            const float c = __uint_as_float(~(unsigned)(key >> 32));
            const int py = (int)((key >> 16) & 0xffff), px = (int)(key & 0xffff);
            cosl_klt_feature f;
            f.status = 1;
            f.pos[0] = __fdiv_rn(__fadd_rn((float)px, 0.5f), Wf);
            f.pos[1] = __fdiv_rn(__fadd_rn((float)py, 0.5f), Hf);
            f.gain = c;  // v3d_gpuklt.cpp:780 copies the cornerness into gain
            f.fed = -1;
            d[i] = f;
            p = make_float4(f.pos[0], f.pos[1], 1.0f, 0.f);
          } else {
            p = make_float4(-1.f, -1.f, 1.f, 0.f);
          }
        } else {
          const cosl_klt_feature f = d[i];
          p = make_float4(f.pos[0], f.pos[1], 1.0f, 0.f);
        }
        pb[i] = p;
        if (ps) ps[i] = p;
      }
    }
  }
}

// "provide" after a plain track(): dst <- tracker result
__global__ void klt_copy_f4(const float4* __restrict__ a, float4* __restrict__ b, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = a[i];
}

struct KltCamList {
  int n;
  int cam[64];
};

// "provide" and advanceFrame of the tracked-only cameras of a cosl_klt_group_step: dst and src
// <- tracker result for the cameras of the list.  grid (div_up(F, blockDim.x), n).
__global__ void klt_provide_cams(const float4* __restrict__ res, float4* __restrict__ dst,
                                 float4* __restrict__ src, int F, KltCamList L) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const size_t k = (size_t)L.cam[blockIdx.y] * F + i;
  const float4 v = res[k];
  dst[k] = v;
  src[k] = v;
}

// ------------------------------------------------------------------------------------------
// feedExternFeaturePoints (v3d_gpuklt.cpp:808-855): (1) kill KLT points within normalised
// distance^2 < 1e-4 of any fed point, (2) place fed points into dead slots in increasing index.
// One launch serves every addressed camera of a group: the points of list k (camera cam[k]) are
// pts3[3 * off[k], 3 * off[k + 1]), their slots go to trackIds[off[k] + j] and the count of placed
// points to nFed[k].
// ------------------------------------------------------------------------------------------
struct KltFeedList {
  int n;         // addressed cameras
  int cam[64];
  int off[65];   // point offsets, off[n] = total
};

// grid (div_up(F, blockDim.x), n).  stride = 3 (default) or 2 (COSL_KLT_COMPAT_FEED_STRIDE2: the
// reference's reads at :826-827, within the camera's own list)
__global__ void klt_feed_kill(float4* __restrict__ buf, int F, const float* __restrict__ pts3,
                              KltFeedList L, int stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const int k0 = L.off[blockIdx.y], npts = L.off[blockIdx.y + 1] - k0;
  const float* p = pts3 + 3 * (size_t)k0;
  float4* b = buf + (size_t)L.cam[blockIdx.y] * F;
  float4 c = b[i];
  if (c.x < 0.f) return;
  for (int k = 0; k < npts; ++k) {
    const double dx = (double)(p[stride * k] - c.x), dy = (double)(p[stride * k + 1] - c.y);
    if (dx * dx + dy * dy < 1e-4) {
      c.x = -1.0f;
      b[i] = c;
      return;
    }
  }
}

// grid n, one warp per camera: sequential scan semantics via a warp-stride loop of ballots
__global__ void __launch_bounds__(32) klt_feed_place(float4* __restrict__ buf, int F,
                                                     const float* __restrict__ pts3, KltFeedList L,
                                                     int* __restrict__ trackIds, int* __restrict__ nFed) {
  const int k0 = L.off[blockIdx.x], npts = L.off[blockIdx.x + 1] - k0;
  const float* p = pts3 + 3 * (size_t)k0;
  float4* b = buf + (size_t)L.cam[blockIdx.x] * F;
  int* ids = trackIds + k0;
  const int lane = threadIdx.x;
  int base = 0;  // fed points placed so far (warp-uniform)
  for (int start = 0; start < F && base < npts; start += 32) {
    const int i = start + lane;
    const bool dead = (i < F) && (b[i].x < 0.f);
    const unsigned bal = __ballot_sync(0xffffffffu, dead);
    const int k = base + __popc(bal & ((1u << lane) - 1));
    if (dead && k < npts) {
      b[i] = make_float4(p[3 * k], p[3 * k + 1], 1.0f, 0.f);
      ids[k] = i;
    }
    base = min(npts, base + __popc(bal));
  }
  if (lane == 0) nFed[blockIdx.x] = base;
}

// ------------------------------------------------------------------------------------------
// advanceFrame (v3d_gpuklt.h:252-259) for a strict subset of a group's cameras: the O(1) flip of
// the pyramid buffers cannot apply to part of a group, so the cameras' slices of the two buffers
// are exchanged (an exchange, not a copy: a second advance swaps them back, as the reference's
// double swap does) and their feature slice is copied dst -> src (F = 0: pyramids only).
// grid (any, n).
// ------------------------------------------------------------------------------------------
__global__ void klt_advance_cams(float4* __restrict__ pyrA, float4* __restrict__ pyrB, long long pyrStride,
                                 const float4* __restrict__ dst, float4* __restrict__ src, int F,
                                 KltCamList L) {
  const int cam = L.cam[blockIdx.y];
  float4* a = pyrA + (size_t)cam * pyrStride;
  float4* b = pyrB + (size_t)cam * pyrStride;
  const long long step = (long long)gridDim.x * blockDim.x;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * step < pyrStride; i += 4 * step) {  // 8 loads in flight per thread
    float4 ta[4], tb[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      ta[u] = a[i + u * step];
      tb[u] = b[i + u * step];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      a[i + u * step] = tb[u];
      b[i + u * step] = ta[u];
    }
  }
  for (; i < pyrStride; i += step) {
    const float4 t = a[i];
    a[i] = b[i];
    b[i] = t;
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < F; i += step)
    src[(size_t)cam * F + i] = dst[(size_t)cam * F + i];
}

}  // namespace coslam
