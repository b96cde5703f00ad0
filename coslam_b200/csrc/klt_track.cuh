// klt_track.cuh -- the 3x3 Lucas-Kanade solve with gain (klt_tracker_with_gain.cg:42-148, host loop
// v3d_gpuklt.cpp:205-305) for sm_90a.
//
// Mapping: one QUARTER-WARP (KLT_G = 8 lanes) per feature slot, four slots per warp.  The (2hw+1)^2
// window pixels are spread over the 8 lanes in ROUNDS rounds: for the live hw = 3, lane gl < 7 owns
// window column gl and walks its 7 rows (lane 7 idles, 87.5 % lane use), so the horizontal stage of
// the bilinear sample is shared by two vertically adjacent pixels; for any other width the pixels
// p = gl + 8r are taken in row-major order.  The running sums are reduced with width-8 butterfly
// shuffles and every lane solves the 3x3 system in closed form (adjugate), so control flow is
// uniform.  The per-pass overhead (neighbour wait, reduction, solve, publish) is paid once per
// warp, i.e. shared by four slots.
//
// Window sampling.  The window samples of a level are one texel apart (ds = 1 / w_level), so all
// (2hw+1)^2 bilinear taps of a window share the fractional offsets of the window centre and their
// integer texel coordinates are centre + (dx, dy).  The kernels evaluate the centre once per pass
// (same expression as the oracle's sample(): u = s*w - 0.5, clamped, floor) and address the taps
// as centre + offset; the oracle evaluates u per pixel in fp32, which differs from centre + offset
// by at most one ulp of u (~3e-5 texel) -- far below the 1/256-texel weights of the GL hardware the
// reference ran on, and covered by the tolerance of the LK parity tests.
//
// Two drivers share the same arithmetic (bit-identical results, checked by
// tests/test_gpu_klt.py::test_fused_gain_tracker_equals_pass_kernels):
//   klt_gain_pass   one launch per (level, iteration) pass, like the reference's draw calls
//   klt_gain_fused  ALL passes in one persistent cooperative launch:
//     * per level, the I0 window samples (constant over the iterations of a level) are computed
//       once and kept in registers together with the I0-only sum of the normal matrix, and a
//       12x12-texel tile of the current-frame pyramid around the feature is staged in shared memory
//       (clamped 128-bit loads; TMA box loads cannot reproduce CLAMP_TO_EDGE, and at the coarse
//       levels most windows straddle the border) -- the iterations then sample from shared memory;
//       a window that drifts out of its tile gets the tile re-centred on it;
//     * the only coupling between slots, the gain-smoothness term that reads beta of <= 8
//       neighbour slots from the PREVIOUS pass, is synchronised without grid barriers and without
//       fences: each slot publishes (pass number, beta) as ONE naturally atomic 8-byte word into a
//       parity double buffer; a slot starts pass p once every slot in its wait set (neighbours +
//       reverse neighbours) has published p-1, and gets the neighbour gains with the poll itself.
//       Waiting also on the reverse neighbours makes overwriting the p-1 record (when publishing
//       p+1) safe on non-square slot grids whose neighbour relation is not symmetric.  Warps own
//       their items for the whole launch and walk the passes in order, so the least advanced item
//       can always run (cooperative launch guarantees co-residency).
#pragma once
#include "klt_kernels.cuh"

namespace coslam {

constexpr int KLT_TW = 12;      // staged I1 tile side (texels): 2*hw + 2 + 2*margin with hw = 3
// Row pitch of the tile in shared memory.  On the hw = 3 path the lanes of a group read 7
// consecutive texels of one tile row per LDS.128, which is conflict-free at any pitch.  The
// any-width path reads 8 consecutive window pixels in row-major order per LDS.128; for a 7-wide
// window (p = 7*py + px) that is float4 index p + py*(pitch - 7), which pitch 15 makes p (mod 8):
// the 8 lanes of a quarter-warp hit 8 distinct 16-byte bank groups (pitch 12 gave 2-way conflicts).
constexpr int KLT_TP = 15;
constexpr int KLT_G = 8;        // lanes per feature slot
constexpr int KLT_ROUNDS = 7;   // window pixels per lane on the fast path (<= 56 pixels)

// Texel (a, b) = (column, row) of the I1 tile that lane gl of a group loads in load u (0..8) of a
// tile half (rows 0..5 or 6..11): each load covers two rows x four columns, so the indices are
// constants plus (gl >> 2, gl & 3) and cost no registers across the passes.
static_assert(KLT_TW == 12 && KLT_G == 8, "tile load mapping: 3 x 3 loads of 2 rows x 4 columns per half");
__device__ __forceinline__ int2 klt_tile_texel(int gl, int half, int u) {
  return make_int2(4 * (u % 3) + (gl & 3), half * (KLT_TW / 2) + 2 * (u / 3) + (gl >> 2));
}

// L2 prefetch of the texels (x .. x + n - 1, y) of a level, clamped to the camera's w x h of the
// level like the loads that will read them (one bulk prefetch: a row segment is contiguous)
__device__ __forceinline__ void klt_prefetch_row(const float4* lv, int pitch, int w, int h, int x, int y,
                                                 int n) {
  const int xa = clampi(x, 0, w - 1), xb = clampi(x + n - 1, 0, w - 1);
  const float4* p = lv + (size_t)clampi(y, 0, h - 1) * pitch + xa;
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"((xb - xa + 1) * 16) : "memory");
}

struct KltCentre {
  float ax, ay;  // bilinear weights shared by the whole window
  int xi, yi;    // unclamped integer texel coordinates of the centre's top-left tap
};

__device__ __forceinline__ KltCentre klt_centre(int w, int h, float s, float t) {
  float u = __fmaf_rn(s, (float)w, -0.5f);
  float v = __fmaf_rn(t, (float)h, -0.5f);
  u = fminf(fmaxf(u, -2.0f), (float)w + 1.0f);
  v = fminf(fmaxf(v, -2.0f), (float)h + 1.0f);
  const float fu = floorf(u), fv = floorf(v);
  KltCentre p;
  p.ax = __fsub_rn(u, fu);
  p.ay = __fsub_rn(v, fv);
  p.xi = (int)fu;
  p.yi = (int)fv;
  return p;
}

// All LK arithmetic below is written with explicit fma/mul/add intrinsics: the two drivers inline
// these helpers into different surroundings, and only a fixed operation sequence keeps their
// results bit-identical (the compiler is otherwise free to contract a*b+c differently per site).
__device__ __forceinline__ float lerp1(float p0, float p1, float a) {
  return __fmaf_rn(a, __fsub_rn(p1, p0), p0);
}

// The two stages of the bilinear sample: along a tap row, then between two tap rows.  The hw = 3
// window walks share one horizontal stage between the two pixels above and below a tap row; every
// sample is still lerp1(lerp1(p00, p10, ax), lerp1(p01, p11, ax), ay), bit for bit.
__device__ __forceinline__ float3 klt_hlerp(const float4 p0, const float4 p1, float ax) {
  return make_float3(lerp1(p0.x, p1.x, ax), lerp1(p0.y, p1.y, ax), lerp1(p0.z, p1.z, ax));
}

__device__ __forceinline__ float3 klt_vlerp(const float3 h0, const float3 h1, float ay) {
  return make_float3(lerp1(h0.x, h1.x, ay), lerp1(h0.y, h1.y, ay), lerp1(h0.z, h1.z, ay));
}

__device__ __forceinline__ float3 klt_lerp4(const float4 p00, const float4 p10, const float4 p01,
                                            const float4 p11, float ax, float ay) {
  return klt_vlerp(klt_hlerp(p00, p10, ax), klt_hlerp(p01, p11, ax), ay);
}

// tap (xi, yi) of a level (rows `pitch` texels apart) with clamp-to-edge at the camera's w x h,
// weights (ax, ay)
__device__ __forceinline__ float3 klt_fetch_global(const float4* __restrict__ lv, int pitch, int w, int h,
                                                   int xi, int yi, float ax, float ay) {
  const int x0 = clampi(xi, 0, w - 1), x1 = clampi(xi + 1, 0, w - 1);
  const int y0 = clampi(yi, 0, h - 1), y1 = clampi(yi + 1, 0, h - 1);
  return klt_lerp4(__ldg(&lv[(size_t)y0 * pitch + x0]), __ldg(&lv[(size_t)y0 * pitch + x1]),
                   __ldg(&lv[(size_t)y1 * pitch + x0]), __ldg(&lv[(size_t)y1 * pitch + x1]), ax, ay);
}

__device__ __forceinline__ float grp_sum(float v) {
#pragma unroll
  for (int o = KLT_G / 2; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o, KLT_G));
  return v;
}

// sqrt.approx.ftz: one MUFU, no denormal rescaling (gradient magnitudes here are 0 or >> 1e-38)
__device__ __forceinline__ float klt_sqrt(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

struct KltAcc {
  float a0, a1, a2, d0, d1, r0, r1, r2, ssd;
};

// the I0-only entry of the normal matrix (constant over the iterations of a level)
__device__ __forceinline__ float klt_d2_term(const float3 I0, float lambda, float delta) {
  const float g0 = klt_sqrt(__fmaf_rn(I0.y, I0.y, __fmul_rn(I0.z, I0.z)));
  return __fmaf_rn(delta, 8.0f, __fmaf_rn(__fmul_rn(lambda, g0), g0, __fmul_rn(I0.x, I0.x)));
}

// halfW = 0.5 * W, halfH = 0.5 * H (the factor 0.5 is exact, so (x * W) * 0.5 == x * (0.5 W))
// The neighbour term delta * nbterm of klt_tracker_with_gain.cg:111 is the same for every window
// pixel; it is added once, as npx * (delta * nbterm), in klt_gain_finish (the shader adds it per
// pixel -- a rounding-level difference, inside the LK parity tolerance), so the pixel loop does
// not depend on the neighbours' gains.
__device__ __forceinline__ void klt_acc_pixel(KltAcc& A, const float3 I0, const float3 I1, float beta,
                                              float halfW, float halfH, float lambda) {
  const float e = __fmaf_rn(beta, I0.x, -I1.x);
  const float Jx = __fmul_rn(__fmaf_rn(beta, I0.y, I1.y), halfW);
  const float Jy = __fmul_rn(__fmaf_rn(beta, I0.z, I1.z), halfH);
  const float n0 = __fmaf_rn(I0.y, I0.y, __fmul_rn(I0.z, I0.z));
  const float n1 = __fmaf_rn(I1.y, I1.y, __fmul_rn(I1.z, I1.z));
  const float g0 = klt_sqrt(n0);
  const float g1 = klt_sqrt(n1);
  A.a0 = __fmaf_rn(Jx, Jx, A.a0);
  A.a1 = __fmaf_rn(Jx, Jy, A.a1);
  A.a2 = __fmaf_rn(Jx, -I0.x, A.a2);
  A.d0 = __fmaf_rn(Jy, Jy, A.d0);
  A.d1 = __fmaf_rn(Jy, -I0.x, A.d1);
  A.r0 = __fmaf_rn(e, Jx, A.r0);
  A.r1 = __fmaf_rn(e, Jy, A.r1);
  const float t = __fmaf_rn(__fmul_rn(lambda, g0), __fmaf_rn(-beta, g0, g1), __fmul_rn(-e, I0.x));
  A.r2 = __fadd_rn(A.r2, t);
  A.ssd = __fmaf_rn(e, e, A.ssd);
}

// The tracker parameters klt_gain_finish reads, held by value.  The fused kernel picks the lax or
// strict threshold field by field on the warp-uniform `strict`: a reference to one of two by-value
// kernel-parameter structs (strict ? Pstrict : Plax) cannot be formed as a pointer, so every field
// read through it compiled to a chain of predicated constant loads over all candidate offsets.
struct KltFinishParams {
  float delta, W, H;         // the same in the lax and the strict set; W, H: the slot's camera
  float ssdThr, sqrConv;
  float vr0, vr1, vr2, vr3;  // validRegion
};

// c ? a : b as a bit mask, with the mask opaque to the compiler: a plain select of two
// kernel parameters compiles to a load of one and a predicated constant load of the other
__device__ __forceinline__ float klt_select(bool c, float a, float b) {
  const unsigned m = (unsigned)klt_opaque(-(int)c);
  return __uint_as_float((__float_as_uint(a) & m) | (__float_as_uint(b) & ~m));
}

// MIXED: the slot's camera is Wc x Hc (the lane groups of a warp may serve two cameras), and the
// strict validRegion is derived from it; otherwise every field comes from the parameter sets
template <bool MIXED>
__device__ __forceinline__ KltFinishParams klt_finish_params(const KltTrackParams& lax,
                                                             const KltTrackParams& str, bool strict,
                                                             int Wc, int Hc) {
  KltFinishParams T;
  T.delta = lax.delta;
  T.W = (float)(MIXED ? Wc : lax.W);
  T.H = (float)(MIXED ? Hc : lax.H);
  T.ssdThr = klt_select(strict, str.ssdThr, lax.ssdThr);
  T.sqrConv = klt_select(strict, str.sqrConv, lax.sqrConv);
  if (MIXED) {
    T.vr0 = klt_select(strict, klt_vr_lo(str.margin, Wc), lax.vr0);
    T.vr1 = klt_select(strict, klt_vr_lo(str.margin, Hc), lax.vr1);
    T.vr2 = klt_select(strict, klt_vr_hi(str.margin, Wc), lax.vr2);
    T.vr3 = klt_select(strict, klt_vr_hi(str.margin, Hc), lax.vr3);
  } else {
    T.vr0 = klt_select(strict, str.vr0, lax.vr0);
    T.vr1 = klt_select(strict, str.vr1, lax.vr1);
    T.vr2 = klt_select(strict, str.vr2, lax.vr2);
    T.vr3 = klt_select(strict, str.vr3, lax.vr3);
  }
  return T;
}

// reduce over the lane group, solve, test (klt_tracker_with_gain.cg:12-40,124-147)
// f = group sum of klt_d2_term over the window
__device__ __forceinline__ float4 klt_gain_finish(KltAcc A, float f, float nbterm, float npxf,
                                                  float X1x, float X1y, float beta,
                                                  const KltFinishParams P) {
  const float a = grp_sum(A.a0), b = grp_sum(A.a1), c = grp_sum(A.a2);
  const float d = grp_sum(A.d0), e = grp_sum(A.d1);
  const float r0 = grp_sum(A.r0), r1 = grp_sum(A.r1);
  const float r2 = __fmaf_rn(npxf, __fmul_rn(P.delta, nbterm), grp_sum(A.r2));
  const float ssd = grp_sum(A.ssd);
  // det3x3symm: a*d*f + 2*b*c*e - (a*e*e + b*b*f + c*c*d)
  const float detp = __fmaf_rn(__fmul_rn(2.0f, __fmul_rn(b, c)), e, __fmul_rn(__fmul_rn(a, d), f));
  const float detm = __fmaf_rn(__fmul_rn(c, c), d, __fmaf_rn(__fmul_rn(b, b), f, __fmul_rn(__fmul_rn(a, e), e)));
  const float det = __fsub_rn(detp, detm);
  const float rdet = __fdividef(1.0f, det);
  const float Aa = __fmaf_rn(d, f, -__fmul_rn(e, e)), Bb = __fmaf_rn(c, e, -__fmul_rn(b, f));
  const float Cc = __fmaf_rn(b, e, -__fmul_rn(c, d)), Dd = __fmaf_rn(a, f, -__fmul_rn(c, c));
  const float Ee = __fmaf_rn(b, c, -__fmul_rn(a, e)), Ff = __fmaf_rn(a, d, -__fmul_rn(b, b));
  float ux = __fmul_rn(__fmaf_rn(Cc, r2, __fmaf_rn(Bb, r1, __fmul_rn(Aa, r0))), rdet);
  float uy = __fmul_rn(__fmaf_rn(Ee, r2, __fmaf_rn(Dd, r1, __fmul_rn(Bb, r0))), rdet);
  const float ub = __fmul_rn(__fmaf_rn(Ff, r2, __fmaf_rn(Ee, r1, __fmul_rn(Cc, r0))), rdet);
  X1x = __fadd_rn(X1x, ux);
  X1y = __fadd_rn(X1y, uy);
  ux = __fmul_rn(ux, P.W);
  uy = __fmul_rn(uy, P.H);
  const float sqrLen = __fmaf_rn(ux, ux, __fmul_rn(uy, uy));
  bool invalid = (det < 0.00001f);
  invalid = invalid || (ssd > P.ssdThr);
  invalid = invalid || (sqrLen > P.sqrConv);
  invalid = invalid || (X1x < P.vr0 || X1y < P.vr1) || (X1x > P.vr2 || X1y > P.vr3);
  return invalid ? make_float4(-1.f, -1.f, -1.f, 0.f)
                 : make_float4(X1x, X1y, __fadd_rn(beta, ub), 0.f);
}

// dot(float4(1), betaN1 + betaN2 - 2*beta) of klt_tracker_with_gain.cg:111 from the eight
// neighbour gains held by the 8 lanes of the group (bn); invalid (< 0) neighbours count as own beta
__device__ __forceinline__ float klt_nbterm(float bn, float beta, int gl, int grpBase) {
  bn = (bn < 0.f) ? beta : bn;
  const float hi = __shfl_sync(0xffffffffu, bn, grpBase + (gl & 3) + 4);
  const float s4 = __fsub_rn(__fadd_rn(bn, hi), __fmul_rn(2.0f, beta));
  const float s0 = __shfl_sync(0xffffffffu, s4, grpBase + 0);
  const float s1 = __shfl_sync(0xffffffffu, s4, grpBase + 1);
  const float s2 = __shfl_sync(0xffffffffu, s4, grpBase + 2);
  const float s3 = __shfl_sync(0xffffffffu, s4, grpBase + 3);
  return __fadd_rn(__fadd_rn(__fadd_rn(s0, s1), s2), s3);
}


// Both gain-tracker drivers are instantiated for a window half-width known at compile time (HWC,
// the live CoSLAM setting hw = 3) and for any width (HWC = 0: P.halfWidth at run time).  With the
// width fixed, the window size, the pixel guards and the fast-path test fold to constants, and the
// window is walked column per lane (see the top of the file); the arithmetic of a pixel is the same
// in both instantiations.  Every path of both drivers walks a window in the same lane assignment
// and order, so that their sums round alike.
constexpr int KLT_HW_LIVE = 3;
static_assert(2 * KLT_HW_LIVE + 1 <= KLT_G && 2 * KLT_HW_LIVE + 1 <= KLT_ROUNDS,
              "hw = 3 walk: one window column per lane, one row per round");

// A window walked with clamped global loads (the per-pass kernel; the fused kernel's items without
// a tile): adds every pixel to A and returns this lane's sum of klt_d2_term, in the lane
// assignment and order of the tile path
template <int HWC>
__device__ __forceinline__ float klt_window_global(KltAcc& A, const float4* __restrict__ L0,
                                                   const float4* __restrict__ L1, int pitch, int w, int h,
                                                   const KltCentre c0, const KltCentre c1, int gl, int hw,
                                                   float beta, float halfW, float halfH, float lambda,
                                                   float delta) {
  const int fwid = 2 * hw + 1, npx = fwid * fwid;
  float d2 = 0.f;
  auto pixel = [&](int px, int py) {
    const int dx = px - hw, dy = py - hw;
    const float3 I0 = klt_fetch_global(L0, pitch, w, h, c0.xi + dx, c0.yi + dy, c0.ax, c0.ay);
    const float3 I1 = klt_fetch_global(L1, pitch, w, h, c1.xi + dx, c1.yi + dy, c1.ax, c1.ay);
    d2 = __fadd_rn(d2, klt_d2_term(I0, lambda, delta));
    klt_acc_pixel(A, I0, I1, beta, halfW, halfH, lambda);
  };
  if constexpr (HWC == KLT_HW_LIVE) {
    // a trip count known only at run time, like the any-width loop: fully unrolled, the loads of
    // 7 rows in flight push the fused kernel past its register budget
    const int rows = gl < fwid ? fwid : 0;
    for (int py = 0; py < rows; ++py) pixel(gl, py);
  } else {
    for (int p = gl; p < npx; p += KLT_G) {
      const int py = p / fwid;
      pixel(p - py * fwid, py);
    }
  }
  return d2;
}

// ------------------------------------------------------------------------------------------
// One pass per launch (diagnostic / fallback).  Grid: x = ceil(F / 32) blocks of 256 threads
// (32 lane groups), y = camera.  level, lvOff, pitch: the pyramid level of the pass.
// ------------------------------------------------------------------------------------------
template <int HWC, bool MIXED>
__global__ void __launch_bounds__(256)
klt_gain_pass(const float4* __restrict__ pyr0, const float4* __restrict__ pyr1, long long pyrStride,
              long long lvOff, int level, int pitch, const KltCam* __restrict__ cams,
              const float4* __restrict__ X0buf, const float4* __restrict__ in, float4* __restrict__ out,
              const int* __restrict__ nbr, KltTrackParams P, int firstPass) {
  const int cam = blockIdx.y;
  if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) return;
  const int2 ext = klt_extent<MIXED>(cams, cam, P.W, P.H);
  const int Wc = ext.x, Hc = ext.y;
  const int w = Wc >> level, h = Hc >> level;
  const int gl = threadIdx.x & (KLT_G - 1), grpBase = threadIdx.x & (32 - KLT_G);
  int slot = blockIdx.x * (blockDim.x / KLT_G) + (threadIdx.x / KLT_G);
  const bool active = slot < P.F;
  if (!active) slot = P.F - 1;  // keep the whole warp in the shuffles; result is discarded
  const float4* L0 = pyr0 + (size_t)cam * pyrStride + lvOff;
  const float4* L1 = pyr1 + (size_t)cam * pyrStride + lvOff;
  const size_t fb = (size_t)cam * P.F;
  const float4 x0 = X0buf[fb + slot];
  float4 cur = in[fb + slot];
  if (firstPass) cur.z = 1.0f;  // gain cleared to 1 before the first pass (v3d_gpuklt.cpp:223-227)
  const float beta = cur.z;
  const float bn = firstPass ? 1.0f : in[fb + nbr[slot * 8 + gl]].z;
  const float nbterm = klt_nbterm(bn, beta, gl, grpBase);
  const bool pre_invalid = (cur.x < 0.f) || (x0.x < 0.f);
  const int hw = HWC > 0 ? HWC : P.halfWidth, fwid = 2 * hw + 1, npx = fwid * fwid;
  const float halfW = 0.5f * (float)Wc, halfH = 0.5f * (float)Hc;
  const KltCentre c0 = klt_centre(w, h, x0.x, x0.y);
  const KltCentre c1 = klt_centre(w, h, cur.x, cur.y);
  KltAcc A = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const float d2 = klt_window_global<HWC>(A, L0, L1, pitch, w, h, c0, c1, gl, hw, beta, halfW, halfH,
                                          P.lambda, P.delta);
  // the host chose P per pass: its validRegion is the strict or the lax one as P.strict says
  float4 res = klt_gain_finish(A, grp_sum(d2), nbterm, (float)npx, cur.x, cur.y, beta,
                               klt_finish_params<MIXED>(P, P, P.strict != 0, Wc, Hc));
  if (pre_invalid) res = make_float4(-1.f, -1.f, -1.f, 0.f);
  if (gl == 0 && active) out[fb + slot] = res;
}

// ------------------------------------------------------------------------------------------
// All passes in one persistent cooperative launch.
//   rec[2][T] u64 = (pass number << 32) | float_bits(beta): value and version travel in ONE naturally
//   atomic 8-byte word, so publishing needs no fence and a reader gets beta with the poll itself;
//   state[T] float4 holds (x, y, beta) of items that are not register-resident
//   waitset[F][16]: first 8 = neighbours (values + versions), last 8 = reverse neighbours or -1
// Work item = (camera, slot); lane group q (global index) owns items q, q + Q, ...; the first item
// of a group is "resident": its invariants, I0 samples and state live in registers and its I1 tile
// in shared memory; further items (only when T > Q) take the global path.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// same load without the compiler-level memory barrier: a hint whose result is re-validated
__device__ __forceinline__ unsigned long long ld_hint_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Optional tail of the last pass: what klt_status (feature table + live count) and klt_suppress
// (-1e30 at the pixel of every live track) would do in two more launches.  dest == nullptr: off.
struct KltTail {
  cosl_klt_feature* dest;
  int* counters;
  float* corn;
  long long cornStride;  // floats per camera; rows are `pitch` floats apart
  int pitch, suppress;
};

constexpr int KLT_FUSED_THREADS = 128;  // 16 lane groups per CTA
constexpr int KLT_FUSED_MINBLOCKS = 4;
constexpr int KLT_GPB = KLT_FUSED_THREADS / KLT_G;

// X0 of an item of klt_gain_fused.  MIXED: an item of a camera outside the tracker stage reads as a
// dead slot (x < 0), so it stages, loads and accumulates nothing; it also neither waits for nor
// publishes records and writes no result (the stage is re-read there, see below).
template <bool MIXED>
__device__ __forceinline__ float4 klt_fused_x0(const float4* __restrict__ X0buf, const KltCam* __restrict__ cams,
                                               int item, int cam) {
  float4 x0 = X0buf[item];
  if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) x0.x = -1.0f;
  return x0;
}

template <int HWC, bool MIXED>
__global__ void __launch_bounds__(KLT_FUSED_THREADS, KLT_FUSED_MINBLOCKS)
klt_gain_fused(const float4* __restrict__ pyr0, const float4* __restrict__ pyr1,
               long long pyrStride, KltLevels LV, const KltCam* __restrict__ cams, int nIter,
               const float4* __restrict__ X0buf,
               float4* __restrict__ state, unsigned long long* __restrict__ rec,
               const int* __restrict__ waitset,
               float4* __restrict__ out, int C, KltTrackParams Plax, KltTrackParams Pstrict,
               int verBase, KltTail tail) {
  __shared__ float4 s_tile[KLT_GPB][KLT_TW * KLT_TP];  // one tile per lane group
  const int gl = threadIdx.x & (KLT_G - 1), grpBase = threadIdx.x & (32 - KLT_G);
  const int grpInBlock = threadIdx.x / KLT_G;
  const int q = blockIdx.x * KLT_GPB + grpInBlock;
  const int Q = gridDim.x * KLT_GPB;
  const int F = Plax.F;
  const int T = C * F;
  const int hw = HWC > 0 ? HWC : Plax.halfWidth, fwid = 2 * hw + 1, npx = fwid * fwid;
  const bool fast = (npx <= KLT_G * KLT_ROUNDS) && (2 * hw + 2 + 2 <= KLT_TW) && (2 * hw + 2 <= 8);
  float4* tile = s_tile[grpInBlock];
  // all groups of a warp must execute the same number of outer iterations (full-mask shuffles)
  const int nOwn = (T + Q - 1) / Q;

  // ---- invariants of the resident item
  const bool active0 = q < T;
  const int item0 = active0 ? q : T - 1;
  const int cam0 = item0 / F, slot0 = item0 - cam0 * F;
  const float4 x00 = klt_fused_x0<MIXED>(X0buf, cams, item0, cam0);
  const int wsA0 = waitset[slot0 * 16 + gl], wsB0 = waitset[slot0 * 16 + 8 + gl];
  // MIXED: the resident item's camera, packed W | H << 16 into one register
  const unsigned wh0 = MIXED ? (unsigned)__ldg(&cams[cam0].W) | ((unsigned)__ldg(&cams[cam0].H) << 16) : 0u;
  float3 I0r[KLT_ROUNDS];
  float f0 = 0.f;  // group sum of klt_d2_term of the resident item at the current level
  float4 cur0 = make_float4(-1.f, -1.f, -1.f, 0.f);
  int tx0 = 0, ty0 = 0;

  // The I0 block of every level depends only on X0: all of them are requested into L2 now, so the
  // per-level staging below finds them there (lane gl: row gl of each 8x8 block)
  if (fast && active0 && x00.x >= 0.f) {
    for (int li = 0; li < LV.n; ++li) {
      const int w = MIXED ? (int)(wh0 & 0xffffu) >> LV.level[li] : LV.w[li];
      const int h = MIXED ? (int)(wh0 >> 16) >> LV.level[li] : LV.h[li];
      const KltCentre c0 = klt_centre(w, h, x00.x, x00.y);
      klt_prefetch_row(pyr0 + (size_t)cam0 * pyrStride + LV.off[li], LV.w[li], w, h, c0.xi - hw,
                       c0.yi - hw + gl, 8);
    }
  }
  int pass = 0;
  for (int li = 0; li < LV.n; ++li) {
    const int pitch = LV.w[li], level = LV.level[li];
    for (int it = 1; it <= nIter; ++it) {
      ++pass;
      // thresholds are lax except on the last iteration of a level (v3d_gpuklt.cpp:266-279)
      const bool strict = (it == nIter) && (it != 1);
      const int rd = (pass - 1) & 1, wr = pass & 1;
      for (int own = 0; own < nOwn; ++own) {
        const bool staged = fast && (own == 0);
        int item = item0, cam = cam0, wsA = wsA0, wsB = wsB0;
        bool active = active0;
        float4 x0 = x00;
        if (own != 0) {
          item = q + own * Q;
          active = item < T;
          if (!active) item = T - 1;
          cam = item / F;
          const int slot = item - cam * F;
          x0 = klt_fused_x0<MIXED>(X0buf, cams, item, cam);
          wsA = waitset[slot * 16 + gl];
          wsB = waitset[slot * 16 + 8 + gl];
        }
        // the item's camera: the lane groups of a warp may serve two cameras (F % 4 != 0)
        int Wc = Plax.W, Hc = Plax.H, w = pitch, h = LV.h[li];
        if (MIXED) {
          const unsigned wh =
              (own == 0) ? wh0 : (unsigned)__ldg(&cams[cam].W) | ((unsigned)__ldg(&cams[cam].H) << 16);
          Wc = wh & 0xffffu;
          Hc = wh >> 16;
          w = Wc >> level;
          h = Hc >> level;
        }
        // own state; the neighbours' gains are needed only after the pixel loop (klt_gain_finish)
        float4 cur;
        if (pass == 1)
          cur = make_float4(x0.x, x0.y, 1.0f, 0.f);  // X1 <- X0, gain cleared to 1 (:223-227)
        else
          cur = (staged) ? cur0 : __ldcg(&state[item]);
        // records of pass p-1 of everything this slot reads (first 8 entries: they also deliver
        // the neighbour gains) or is read by (last 8, may be -1); wsA is always a valid slot
        const unsigned long long* ra = rec + (size_t)rd * T + (size_t)cam * F + wsA;
        const unsigned long long* rb = rec + (size_t)rd * T + (size_t)cam * F + (wsB >= 0 ? wsB : wsA);
        const int need = verBase + pass - 1;
        unsigned long long va = 0, vb = 0;  // version 0 < need for every pass >= 2
        const float beta = cur.z;
        const bool pre_invalid = (cur.x < 0.f) || (x0.x < 0.f);
        const KltCentre c1 = klt_centre(w, h, cur.x, cur.y);
        // last iteration of a level: request the next level's I1 tile around the current estimate
        // into L2 (rows gl and gl + 8), so its staging does not wait on HBM
        if (staged && it == nIter && li + 1 < LV.n && !pre_invalid) {
          const int pn = LV.w[li + 1];
          const int wn = MIXED ? Wc >> LV.level[li + 1] : pn, hn = MIXED ? Hc >> LV.level[li + 1] : LV.h[li + 1];
          const KltCentre cn = klt_centre(wn, hn, cur.x, cur.y);
          const float4* Ln = pyr1 + (size_t)cam * pyrStride + LV.off[li + 1];
          klt_prefetch_row(Ln, pn, wn, hn, cn.xi - hw - 2, cn.yi - hw - 2 + gl, KLT_TW);
          if (gl + KLT_G < KLT_TW) klt_prefetch_row(Ln, pn, wn, hn, cn.xi - hw - 2, cn.yi - hw - 2 + gl + KLT_G, KLT_TW);
        }
        // ---- per-level staging (first iteration of a level): I0 samples + I1 tile.
        // Three memory round trips with all loads of a trip in flight together: (A) the 8x8 texels
        // under the I0 window and the upper half of the I1 tile, (B) the I0 samples interpolated
        // from shared memory (the I0 texels borrow the lower tile rows), (C) the lower tile half.
        if (staged && it == 1) {
          const float4* L0 = pyr0 + (size_t)cam * pyrStride + LV.off[li];
          const float4* L1 = pyr1 + (size_t)cam * pyrStride + LV.off[li];
          const KltCentre c0 = klt_centre(w, h, x0.x, x0.y);
          constexpr int NLD = KLT_TW * KLT_TW / KLT_G / 2;  // 9 tile texels per lane and half
          constexpr int I0B = (KLT_TW / 2) * KLT_TP;        // I0 texels: tile rows 6.., pitch 8
          static_assert(I0B + 64 <= KLT_TW * KLT_TP, "I0 staging area must fit the lower tile half");
          tx0 = c1.xi - hw - 2;
          ty0 = c1.yi - hw - 2;
          // every __syncwarp below is executed by the whole warp: only the memory operations are
          // predicated on the slot being alive (the four slots of a warp differ in that)
          float d2 = 0.f;
          if (!pre_invalid) {
            float4 t0[8], tv[NLD];
#pragma unroll
            for (int u = 0; u < 8; ++u)  // lane gl loads column gl of the 8x8 block
              t0[u] = __ldg(&L0[(size_t)clampi(c0.yi - hw + u, 0, h - 1) * pitch + clampi(c0.xi - hw + gl, 0, w - 1)]);
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int2 ba = klt_tile_texel(gl, 0, u);
              const int b = ba.y, a = ba.x;
              tv[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) tile[I0B + u * 8 + gl] = t0[u];
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int2 ba = klt_tile_texel(gl, 0, u);
              const int b = ba.y, a = ba.x;
              tile[b * KLT_TP + a] = tv[u];
            }
          }
          __syncwarp();
          // I0r is written on every path (a dead slot never reads it), so the previous level's
          // samples are not live across the loads above
          if constexpr (HWC == KLT_HW_LIVE) {
            // I0r[r] = pixel (gl, r): lane gl walks column gl of the 8x8 block, one tap row per row
            if (!pre_invalid && gl < fwid) {
              const float4* t4 = tile + I0B + gl;
              float3 hp = klt_hlerp(t4[0], t4[1], c0.ax);
#pragma unroll
              for (int r = 0; r < KLT_ROUNDS; ++r) {
                const float3 hn = klt_hlerp(t4[8 * (r + 1)], t4[8 * (r + 1) + 1], c0.ax);
                I0r[r] = klt_vlerp(hp, hn, c0.ay);
                d2 = __fadd_rn(d2, klt_d2_term(I0r[r], Plax.lambda, Plax.delta));
                hp = hn;
              }
            } else {
#pragma unroll
              for (int r = 0; r < KLT_ROUNDS; ++r) I0r[r] = make_float3(0.f, 0.f, 0.f);
            }
          } else {
#pragma unroll
            for (int r = 0; r < KLT_ROUNDS; ++r) {
              const int p = gl + KLT_G * r;
              if (!pre_invalid && p < npx) {
                const int py = p / fwid, px = p - py * fwid;
                const float4* t4 = tile + I0B + py * 8 + px;
                I0r[r] = klt_lerp4(t4[0], t4[1], t4[8], t4[9], c0.ax, c0.ay);
                d2 = __fadd_rn(d2, klt_d2_term(I0r[r], Plax.lambda, Plax.delta));
              } else {
                I0r[r] = make_float3(0.f, 0.f, 0.f);
              }
            }
          }
          __syncwarp();
          if (!pre_invalid) {
            float4 tw[NLD];
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int2 ba = klt_tile_texel(gl, 1, u);
              const int b = ba.y, a = ba.x;
              tw[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
            }
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int2 ba = klt_tile_texel(gl, 1, u);
              const int b = ba.y, a = ba.x;
              tile[b * KLT_TP + a] = tw[u];
            }
          }
          f0 = grp_sum(d2);
          __syncwarp();
        }
        // ---- the iteration
        KltAcc A = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        float f = f0;
        const float halfW = 0.5f * (float)Wc, halfH = 0.5f * (float)Hc;
        // tile[b * KLT_TP + a] == level[clamp(ty0 + b)][clamp(tx0 + a)]: indexing with the
        // unclamped tap coordinates reproduces the clamped fetches exactly
        int a0 = c1.xi - tx0, b0 = c1.yi - ty0;
        // A window that drifted out of its tile gets the tile re-centred (two batches of loads)
        // rather than paying clamped global loads for the rest of the level; the slow warp would
        // otherwise hold up every slot that waits on it.
        if (staged && it != 1) {
          const bool inTile = (a0 - hw >= 0) && (a0 + hw + 1 < KLT_TW) && (b0 - hw >= 0) && (b0 + hw + 1 < KLT_TW);
          const bool need = !pre_invalid && !inTile;
          if (__any_sync(0xffffffffu, need)) {
            if (need) {
              const float4* L1 = pyr1 + (size_t)cam * pyrStride + LV.off[li];
              tx0 = c1.xi - hw - 2;
              ty0 = c1.yi - hw - 2;
              constexpr int NLD = KLT_TW * KLT_TW / KLT_G / 2;
#pragma unroll
              for (int half = 0; half < 2; ++half) {
                float4 tv[NLD];
#pragma unroll
                for (int u = 0; u < NLD; ++u) {
                  const int2 ba = klt_tile_texel(gl, half, u);
                  const int b = ba.y, a = ba.x;
                  tv[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
                }
#pragma unroll
                for (int u = 0; u < NLD; ++u) {
                  const int2 ba = klt_tile_texel(gl, half, u);
                  const int b = ba.y, a = ba.x;
                  tile[b * KLT_TP + a] = tv[u];
                }
              }
              a0 = c1.xi - tx0;  // the window now lies in the tile: 2 * hw + 2 + 2 <= KLT_TW when staged
              b0 = c1.yi - ty0;
            }
            __syncwarp();
          }
        }
        if (!pre_invalid) {
          // a staged window is in its tile here: the tile was staged around it on the first
          // iteration of the level or re-centred on it above
          if (staged && HWC == KLT_HW_LIVE) {
            // lane gl < 7: window column gl.  Tap row j (taps (gl, j) and (gl + 1, j): 7 lanes read
            // 8 consecutive texels of one tile row) is interpolated along x once and serves the
            // pixels of rows j - 1 and j: 16 LDS.128 and 45 lerps per lane for 7 pixels
            const float4* tc = tile + (b0 - hw) * KLT_TP + (a0 - hw) + gl;
            const bool col = gl < fwid;
            constexpr int JP = 5;  // tap rows 0..4 (pixel rows 0..3), the record poll, tap rows 5..7
            float3 hp;
            if (col) {
              hp = klt_hlerp(tc[0], tc[1], c1.ax);
#pragma unroll
              for (int j = 1; j < JP; ++j) {
                const float3 hn = klt_hlerp(tc[j * KLT_TP], tc[j * KLT_TP + 1], c1.ax);
                klt_acc_pixel(A, I0r[j - 1], klt_vlerp(hp, hn, c1.ay), beta, halfW, halfH, Plax.lambda);
                hp = hn;
              }
            }
            if (pass > 1 && active) {
              // early, non-binding look at the records: usually published by now, and the L2
              // round trip overlaps the rest of the window
              va = ld_hint_u64(ra);
              vb = ld_hint_u64(rb);
            }
            if (col) {
#pragma unroll
              for (int j = JP; j <= 2 * KLT_HW_LIVE + 1; ++j) {
                const float3 hn = klt_hlerp(tc[j * KLT_TP], tc[j * KLT_TP + 1], c1.ax);
                klt_acc_pixel(A, I0r[j - 1], klt_vlerp(hp, hn, c1.ay), beta, halfW, halfH, Plax.lambda);
                hp = hn;
              }
            }
          } else if (staged) {
            const float4* tc = tile + b0 * KLT_TP + a0;
            // the tap offsets of this lane are recomputed every pass: held across the passes,
            // they do not fit the register budget of 4 CTAs per SM
            const int glp = klt_opaque(gl);
#pragma unroll
            for (int r = 0; r < KLT_ROUNDS; ++r) {
              if (r == KLT_ROUNDS / 2 && pass > 1 && active) {
                // early, non-binding look at the records: usually published by now, and the L2
                // round trip overlaps the remaining rounds
                va = ld_hint_u64(ra);
                vb = ld_hint_u64(rb);
              }
              if (gl + KLT_G * r < npx) {
                const int p = glp + KLT_G * r, py = p / fwid, px = p - py * fwid;
                const float4* t4 = tc + ((py - hw) * KLT_TP + (px - hw));
                const float3 I1 = klt_lerp4(t4[0], t4[1], t4[KLT_TP], t4[KLT_TP + 1], c1.ax, c1.ay);
                klt_acc_pixel(A, I0r[r], I1, beta, halfW, halfH, Plax.lambda);
              }
            }
          } else {
            const float4* L0 = pyr0 + (size_t)cam * pyrStride + LV.off[li];
            const float4* L1 = pyr1 + (size_t)cam * pyrStride + LV.off[li];
            const KltCentre c0 = klt_centre(w, h, x0.x, x0.y);
            f = klt_window_global<HWC>(A, L0, L1, pitch, w, h, c0, c1, gl, hw, beta, halfW, halfH,
                                       Plax.lambda, Plax.delta);
          }
        }
        if (!staged) f = grp_sum(f);  // warp-uniform branch: staged depends on own only
        // ---- wait for the pass-(p-1) records, get the neighbour gains with the poll itself
        float bn = 1.0f;
        if (pass > 1) {
          bn = -1.0f;
          // an item of a camera outside the tracker stage (MIXED) neither waits nor writes; the
          // stage is read where it is needed, not held in a register across the pixel loop
          if (active && klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) {
            while ((int)(va >> 32) < need) {
              va = ld_relaxed_u64(ra);
              if ((int)(va >> 32) >= need) break;
              __nanosleep(20);
            }
            while ((int)(vb >> 32) < need) {
              vb = ld_relaxed_u64(rb);
              if ((int)(vb >> 32) >= need) break;
              __nanosleep(20);
            }
            bn = __uint_as_float((unsigned)va);
          }
          __syncwarp();
        }
        const float nbterm = klt_nbterm(bn, beta, gl, grpBase);
        float4 res = klt_gain_finish(A, f, nbterm, (float)npx, cur.x, cur.y, beta,
                                     klt_finish_params<MIXED>(Plax, Pstrict, strict, Wc, Hc));
        if (pre_invalid) res = make_float4(-1.f, -1.f, -1.f, 0.f);
        if (staged) cur0 = res;
        if (gl == 0 && active && klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) {
          if (pass == LV.n * nIter) {
            out[item] = res;
            if (tail.dest) {  // v3d_gpuklt.cpp:872-888 and :475-500, see klt_status / klt_suppress
              cosl_klt_feature f;
              const bool live = res.x >= 0.f;
              f.status = live ? 0 : -1;
              f.pos[0] = live ? res.x : -1.0f;
              f.pos[1] = live ? res.y : -1.0f;
              f.gain = live ? res.z : 1.0f;
              f.fed = -1;
              tail.dest[item] = f;
              if (live) {
                atomicAdd(&tail.counters[cam * 8 + 0], 1);
                if (tail.suppress && res.x < 1.0f && res.y >= 0.0f && res.y < 1.0f) {
                  const int ix = (int)floorf(__fmul_rn(res.x, (float)Wc));
                  const int iy = (int)floorf(__fmul_rn(res.y, (float)Hc));
                  if (ix >= 0 && ix < Wc && iy >= 0 && iy < Hc)
                    tail.corn[(size_t)cam * tail.cornStride + (size_t)iy * tail.pitch + ix] = -1e30f;
                }
              }
            }
          }
          if (!staged) __stcg(&state[item], res);
          st_relaxed_u64(rec + (size_t)wr * T + item,
                         ((unsigned long long)(unsigned)(verBase + pass) << 32) |
                             (unsigned long long)__float_as_uint(res.z));
        }
        __syncwarp();
      }
    }
  }
}

}  // namespace coslam

namespace coslam {

// ------------------------------------------------------------------------------------------
// 2x2 LK (klt_tracker.cg:35-131, host loop v3d_gpuklt.cpp:99-161) with the memory structure of
// klt_gain_fused: 8 lanes per slot, per level the I0 samples in registers and a 12x12 tile of the
// current frame in shared memory (re-centred if the window leaves it).  Slots do not interact, so
// this is a plain launch: grid = (ceil(F / 16), cameras), 128 threads.  Same control flow as
// klt_track_2x2 (thresholds from the last iteration of every level, validity region at the end);
// used when the window fits the tile (hw <= 3), klt_track_2x2 otherwise.
// ------------------------------------------------------------------------------------------
template <bool MIXED>
__global__ void __launch_bounds__(128)
klt_track_2x2_tiled(const float4* __restrict__ pyr0, const float4* __restrict__ pyr1,
                    long long pyrStride, KltLevels LV, const KltCam* __restrict__ cams,
                    const float4* __restrict__ X0buf, float4* __restrict__ out, KltTrackParams P,
                    int nIter) {
  __shared__ float4 s_tile[16][KLT_TW * KLT_TP];
  const int gl = threadIdx.x & (KLT_G - 1);
  const int grp = threadIdx.x / KLT_G;
  const int cam = blockIdx.y;
  if (!klt_in_stage<MIXED>(cams, cam, KLT_STAGE_TRACK)) return;
  int slot = blockIdx.x * 16 + grp;
  const bool active = slot < P.F;
  if (!active) slot = P.F - 1;  // keep the warp complete for the shuffles
  float4* tile = s_tile[grp];
  const size_t fb = (size_t)cam * P.F;
  const float4 x0 = X0buf[fb + slot];
  float X1x = x0.x, X1y = x0.y;
  bool invalid = (x0.x < 0.f);
  const bool dead = invalid;  // no samples are fetched for a dead slot
  const int hw = P.halfWidth, fwid = 2 * hw + 1, npx = fwid * fwid;
  const int2 ext = klt_extent<MIXED>(cams, cam, P.W, P.H);
  const int Wc = ext.x, Hc = ext.y;
  const float halfW = 0.5f * (float)Wc, halfH = 0.5f * (float)Hc;
  int toff[KLT_ROUNDS];
#pragma unroll
  for (int r = 0; r < KLT_ROUNDS; ++r) {
    const int p = min(gl + KLT_G * r, npx - 1);
    const int py = p / fwid, px = p - py * fwid;
    toff[r] = (py - hw) * KLT_TP + (px - hw);
  }
  float3 I0r[KLT_ROUNDS];
  float sqrLen = 0.f, ssd = 0.f;
  for (int li = 0; li < LV.n; ++li) {
    const int pitch = LV.w[li];
    const int w = MIXED ? Wc >> LV.level[li] : LV.w[li], h = MIXED ? Hc >> LV.level[li] : LV.h[li];
    const float4* L0 = pyr0 + (size_t)cam * pyrStride + LV.off[li];
    const float4* L1 = pyr1 + (size_t)cam * pyrStride + LV.off[li];
    constexpr int NLD = KLT_TW * KLT_TW / KLT_G / 2;
    constexpr int I0B = (KLT_TW / 2) * KLT_TP;
    int tx0, ty0;
    {
      // ---- staging, as in klt_gain_fused: I0 block + upper tile half, I0 samples, lower tile half
      const KltCentre c0 = klt_centre(w, h, x0.x, x0.y);
      const KltCentre c1 = klt_centre(w, h, X1x, X1y);
      tx0 = c1.xi - hw - 2;
      ty0 = c1.yi - hw - 2;
      if (!dead) {
        float4 t0[8], tv[NLD];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          t0[u] = __ldg(&L0[(size_t)clampi(c0.yi - hw + u, 0, h - 1) * pitch + clampi(c0.xi - hw + gl, 0, w - 1)]);
#pragma unroll
        for (int u = 0; u < NLD; ++u) {
          const int i = gl + KLT_G * u;
          const int b = i / KLT_TW, a = i - b * KLT_TW;
          tv[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) tile[I0B + u * 8 + gl] = t0[u];
#pragma unroll
        for (int u = 0; u < NLD; ++u) {
          const int i = gl + KLT_G * u;
          const int b = i / KLT_TW, a = i - b * KLT_TW;
          tile[b * KLT_TP + a] = tv[u];
        }
      }
      __syncwarp();
      if (!dead) {
#pragma unroll
        for (int r = 0; r < KLT_ROUNDS; ++r) {
          const int p = gl + KLT_G * r;
          if (p < npx) {
            const int py = p / fwid, px = p - py * fwid;
            const float4* t4 = tile + I0B + py * 8 + px;
            I0r[r] = klt_lerp4(t4[0], t4[1], t4[8], t4[9], c0.ax, c0.ay);
          } else {
            I0r[r] = make_float3(0.f, 0.f, 0.f);
          }
        }
      }
      __syncwarp();
      if (!dead) {
        float4 tw[NLD];
#pragma unroll
        for (int u = 0; u < NLD; ++u) {
          const int i = gl + KLT_G * (u + NLD);
          const int b = i / KLT_TW, a = i - b * KLT_TW;
          tw[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
        }
#pragma unroll
        for (int u = 0; u < NLD; ++u) {
          const int i = gl + KLT_G * (u + NLD);
          const int b = i / KLT_TW, a = i - b * KLT_TW;
          tile[b * KLT_TP + a] = tw[u];
        }
      }
      __syncwarp();
    }
    for (int it = 0; it < nIter; ++it) {
      const KltCentre c1 = klt_centre(w, h, X1x, X1y);
      int a0 = c1.xi - tx0, b0 = c1.yi - ty0;
      const bool inTile = (a0 - hw >= 0) && (a0 + hw + 1 < KLT_TW) && (b0 - hw >= 0) && (b0 + hw + 1 < KLT_TW);
      const bool need = !dead && !inTile;
      if (__any_sync(0xffffffffu, need)) {  // re-centre the tile (warp-uniform branch)
        if (need) {
          tx0 = c1.xi - hw - 2;
          ty0 = c1.yi - hw - 2;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            float4 tv[NLD];
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int i = gl + KLT_G * (u + half * NLD);
              const int b = i / KLT_TW, a = i - b * KLT_TW;
              tv[u] = __ldg(&L1[(size_t)clampi(ty0 + b, 0, h - 1) * pitch + clampi(tx0 + a, 0, w - 1)]);
            }
#pragma unroll
            for (int u = 0; u < NLD; ++u) {
              const int i = gl + KLT_G * (u + half * NLD);
              const int b = i / KLT_TW, a = i - b * KLT_TW;
              tile[b * KLT_TP + a] = tv[u];
            }
          }
          a0 = c1.xi - tx0;
          b0 = c1.yi - ty0;
        }
        __syncwarp();
      }
      float a = 0.f, b = 0.f, c = 0.f, r0 = 0.f, r1 = 0.f, sd = 0.f;
      if (!dead) {
        const float4* tc = tile + b0 * KLT_TP + a0;
#pragma unroll
        for (int r = 0; r < KLT_ROUNDS; ++r) {
          if (gl + KLT_G * r < npx) {
            const float4* t4 = tc + toff[r];
            const float3 I1 = klt_lerp4(t4[0], t4[1], t4[KLT_TP], t4[KLT_TP + 1], c1.ax, c1.ay);
            const float3 I0 = I0r[r];
            const float e = __fsub_rn(I0.x, I1.x);
            const float Jx = __fmul_rn(__fadd_rn(I0.y, I1.y), halfW);
            const float Jy = __fmul_rn(__fadd_rn(I0.z, I1.z), halfH);
            a = __fmaf_rn(Jx, Jx, a);
            b = __fmaf_rn(Jx, Jy, b);
            c = __fmaf_rn(Jy, Jy, c);
            r0 = __fmaf_rn(e, Jx, r0);
            r1 = __fmaf_rn(e, Jy, r1);
            sd = __fmaf_rn(e, e, sd);
          }
        }
      }
      a = grp_sum(a);
      b = grp_sum(b);
      c = grp_sum(c);
      r0 = grp_sum(r0);
      r1 = grp_sum(r1);
      ssd = grp_sum(sd);
      const float det = __fmaf_rn(a, c, -__fmul_rn(b, b));
      invalid = invalid || (det < 0.00001f);
      const float rdet = __fdividef(1.0f, det);
      float ux = __fmul_rn(rdet, __fmaf_rn(c, r0, -__fmul_rn(b, r1)));
      float uy = __fmul_rn(rdet, __fmaf_rn(a, r1, -__fmul_rn(b, r0)));
      X1x = __fadd_rn(X1x, ux);
      X1y = __fadd_rn(X1y, uy);
      ux = __fmul_rn(ux, (float)Wc);
      uy = __fmul_rn(uy, (float)Hc);
      sqrLen = __fmaf_rn(ux, ux, __fmul_rn(uy, uy));
    }
    invalid = invalid || (sqrLen > P.sqrConv);
    invalid = invalid || (ssd > P.ssdThr);
  }
  if (MIXED)
    invalid = invalid || (X1x < klt_vr_lo(P.margin, Wc) || X1y < klt_vr_lo(P.margin, Hc)) ||
              (X1x > klt_vr_hi(P.margin, Wc) || X1y > klt_vr_hi(P.margin, Hc));
  else
    invalid = invalid || (X1x < P.vr0 || X1y < P.vr1) || (X1x > P.vr2 || X1y > P.vr3);
  if (gl == 0 && active)
    out[fb + slot] = invalid ? make_float4(-1.f, -1.f, -1.f, 0.f) : make_float4(X1x, X1y, x0.x, 0.f);
}

}  // namespace coslam
