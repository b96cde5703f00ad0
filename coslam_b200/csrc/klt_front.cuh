// klt_front.cuh -- fused front end of a KLT frame: from the u8 image, ONE kernel produces
//   * pyramid level 0 (I, Ix, Iy)          [pyramid_with_derivative_pass1v.cg + pass1h.cg]
//   * pyramid level 1 ([1 3 3 1]^2 / 64)   [pyramid_with_derivative_pass2.cg]
//   * the detector's cornerness map        [klt_detector_pass1.cg + klt_detector_pass2.cg]
// so the 16 B/px level-0 texels are written once and never re-read from HBM by the pyramid or the
// detector.  When nothing will read level 0 (STORE_L0 = false: a tracking frame whose cornerness
// is fused here and whose tracker skips level 0), it is not written at all.  Every output is
// computed with the same operations, in the same order, as the oracle (oracle/klt_oracle.cpp):
// bit-exact.
// (The level-0 taps 1/8, 1/4, 1/2 are powers of two, so fma(k, x, acc) rounds exactly like
// acc + k*x; the [1 3 3 1] taps and the structure-tensor sums keep separate mul / add.)
//
// Register-blocked streaming design, no shared memory: one WARP owns a strip of 64 level-0 columns
// (lane l holds columns X0 + 2l and X0 + 2l + 1) and walks down a chunk of rows.  All vertical
// filters (5-tap smooth / derivative, the [1 3 3 1] taps, the 7-row structure-tensor sums) slide
// through registers; all horizontal filters fetch the neighbour columns with warp shuffles.  The
// strip has a halo of 6 columns on either side, so 52 of the 64 columns produce outputs; a chunk
// of R rows needs R + 6 level-0 rows (R + 10 image rows).
//
// CLAMP_TO_EDGE of every pass is reproduced by construction: lanes / rows outside the image hold
// the values of the clamped coordinate (u8 loads are clamped; level-0 values of out-of-image
// columns are replaced by those of column 0 / W-1, out-of-image rows re-use row 0 / H-1).  W x H is
// the camera's own extent (MIXED: its KltCam entry); the grid covers the group's largest camera and
// the warps past a smaller camera's strips and chunks exit.
#pragma once
#include "klt_kernels.cuh"

namespace coslam {

constexpr int FS_SW = 52;  // output columns per strip
constexpr int FS_HL = 6;   // strip halo (columns)
#ifndef FS_ROWS
#define FS_ROWS 36         // rows per chunk: even, (FS_ROWS + 6) % 7 == 0
#endif
constexpr int FS_R = FS_ROWS;
static_assert(FS_R % 2 == 0 && (FS_R + 6) % 7 == 0, "chunk height");
constexpr int FS_WARPS = 4;  // warps per CTA (independent of each other)
#ifndef FS_MINB
#define FS_MINB 4
#endif
#ifndef FS_PF
#define FS_PF 3           // image rows in flight ahead of the row loop
#endif

constexpr int KLT_CORN_PER_CAM = 2;  // FrontParams::wantCorn: each camera of the detector stage (MIXED)

struct FrontParams {
  const uint8_t* img;
  size_t imgPitch, imgStride;
  float4* pyr;
  long long pyrStride, lv1Off;
  float* corn;
  long long cornStride;  // floats per camera; rows are W floats apart
  int W, H, nStrips, nChunks, wantL1, wantCorn;  // W x H: the group's (largest) geometry
  int camBase;  // first camera of this launch (per-camera launches pipeline with the uploads)
  float minC;
  int ixlo, ixhi, iylo, iyhi;  // detector window (pixels whose centre lies inside the margins)
  const KltCam* cams;          // MIXED: every camera's extent and detector window
};

// STORE_L0 = false: level 0 is computed (every other output derives from it) but not written
template <bool STORE_L0, bool MIXED>
__global__ void __launch_bounds__(32 * FS_WARPS, FS_MINB)
klt_front(const FrontParams P) {
  const int lane = threadIdx.x & 31;
  const int wid = blockIdx.x * FS_WARPS + (threadIdx.x >> 5);
  const int cam = blockIdx.y + P.camBase;
  if (!klt_in_stage<MIXED>(P.cams, cam, KLT_STAGE_PYR)) return;
  const int2 ext = klt_extent<MIXED>(P.cams, cam, P.W, P.H);
  const int W = ext.x, H = ext.y;
  const int nStrips = MIXED ? (W + FS_SW - 1) / FS_SW : P.nStrips;
  if (wid >= nStrips * (MIXED ? (H + FS_R - 1) / FS_R : P.nChunks)) return;
  const int chunk = wid / nStrips, strip = wid - chunk * nStrips;
  const int X0 = strip * FS_SW - FS_HL;
  const int xa = X0 + 2 * lane, xb = xa + 1;
  const int r0 = chunk * FS_R, r1 = min(H, r0 + FS_R);
  const bool edge = (X0 < 0) || (X0 + 63 >= W);
  const int cxa = clampi(xa, 0, W - 1), cxb = clampi(xb, 0, W - 1);
  // lane / component that holds the clamped column (edge strips only)
  const int la = (cxa - X0) >> 1, ca = (cxa - X0) & 1;
  const int lb = (cxb - X0) >> 1, cb = (cxb - X0) & 1;
  const bool owner = (lane >= FS_HL / 2) && (lane < (FS_HL + FS_SW) / 2);
  const bool wa = owner && xa < W, wb = owner && xb < W;  // this lane writes column xa / xb
  const uint8_t* im = P.img + (size_t)cam * P.imgStride;
  float4* out0 = P.pyr + (size_t)cam * P.pyrStride;
  float4* out1 = out0 + P.lv1Off;
  float* outc = P.corn + (size_t)cam * P.cornStride;
  const int dh = H >> 1;
  const int j0 = r0 >> 1, j1 = min(dh, (r0 + FS_R) >> 1);  // level-1 rows of this chunk
  const bool w1 = owner && (xa >> 1) < (W >> 1);            // this lane writes a level-1 column

  float ga[5], gb[5];  // image rows yc-2 .. yc+2 (clamped) at columns xa, xb
  // raw pixel pair (xa | xb << 8) of a clamped image row
  auto load_raw = [&](int y) -> unsigned {
    const uint8_t* rp = im + (size_t)clampi(y, 0, H - 1) * P.imgPitch;
    if (!edge)  // xa is even and the pitch a multiple of 16: aligned 16-bit load
      return __ldg(reinterpret_cast<const unsigned short*>(rp + xa));
    return (unsigned)__ldg(rp + cxa) | ((unsigned)__ldg(rp + cxb) << 8);
  };
  // the image row a level-0 row needs last (yc + 2) is fetched FS_PF rows ahead of its use, so
  // the row loop never waits on global memory
  unsigned q[FS_PF];
  {
    const int yc0 = clampi(r0 - 3, 0, H - 1);
    unsigned h4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) h4[k] = load_raw(yc0 - 2 + k);
#pragma unroll
    for (int k = 0; k < FS_PF; ++k) q[k] = load_raw(yc0 + 2 + k);
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // slides into rows yc0-2 .. yc0+1
      ga[k + 1] = (float)(h4[k] & 0xff);
      gb[k + 1] = (float)(h4[k] >> 8);
    }
  }
  float A[3] = {0.f, 0.f, 0.f}, B[3] = {0.f, 0.f, 0.f};  // level-0 (I, Ix, Iy) of the current row
  float pA[3] = {0.f, 0.f, 0.f}, pB[3] = {0.f, 0.f, 0.f};  // previous row
  float eA[3] = {0.f, 0.f, 0.f}, eB[3] = {0.f, 0.f, 0.f};  // running [1 3 3 1] column taps
  float prod[7][6];                                        // ring: gx^2, gx gy, gy^2 at xa, xb
  int ycPrev = -0x7fffffff;

  for (int base = 0; base < FS_R + 6; base += 7) {
#pragma unroll
    for (int u = 0; u < 7; ++u) {
      const int yy = r0 - 3 + base + u;  // unclamped level-0 row
      const int yc = clampi(yy, 0, H - 1);
      if (yc != ycPrev) {  // warp-uniform: a new image row enters, otherwise the edge row repeats
        ycPrev = yc;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ga[k] = ga[k + 1];
          gb[k] = gb[k + 1];
        }
        ga[4] = (float)(q[0] & 0xff);
        gb[4] = (float)(q[0] >> 8);
#pragma unroll
        for (int k = 0; k + 1 < FS_PF; ++k) q[k] = q[k + 1];
        q[FS_PF - 1] = load_raw(yc + 2 + FS_PF);
        // vertical [1 2 1]/4 and [-1 -2 0 2 1]/8 (pyramid_with_derivative_pass1v.cg)
        const float va = __fmaf_rn(0.25f, ga[3], __fmaf_rn(0.5f, ga[2], __fmul_rn(0.25f, ga[1])));
        const float vb = __fmaf_rn(0.25f, gb[3], __fmaf_rn(0.5f, gb[2], __fmul_rn(0.25f, gb[1])));
        const float da = __fmaf_rn(0.125f, ga[4], __fmaf_rn(0.25f, ga[3], __fmaf_rn(-0.25f, ga[1], __fmul_rn(-0.125f, ga[0]))));
        const float db = __fmaf_rn(0.125f, gb[4], __fmaf_rn(0.25f, gb[3], __fmaf_rn(-0.25f, gb[1], __fmul_rn(-0.125f, gb[0]))));
        // horizontal pass (pass1h.cg): columns xa-2 .. xb+2 of v, xa-1 .. xb+1 of dv
        const float vLa = __shfl_up_sync(0xffffffffu, va, 1), vLb = __shfl_up_sync(0xffffffffu, vb, 1);
        const float vRa = __shfl_down_sync(0xffffffffu, va, 1), vRb = __shfl_down_sync(0xffffffffu, vb, 1);
        const float dLb = __shfl_up_sync(0xffffffffu, db, 1), dRa = __shfl_down_sync(0xffffffffu, da, 1);
        A[0] = __fmaf_rn(0.25f, vb, __fmaf_rn(0.5f, va, __fmul_rn(0.25f, vLb)));
        B[0] = __fmaf_rn(0.25f, vRa, __fmaf_rn(0.5f, vb, __fmul_rn(0.25f, va)));
        A[1] = __fmaf_rn(0.125f, vRa, __fmaf_rn(0.25f, vb, __fmaf_rn(-0.25f, vLb, __fmul_rn(-0.125f, vLa))));
        B[1] = __fmaf_rn(0.125f, vRb, __fmaf_rn(0.25f, vRa, __fmaf_rn(-0.25f, va, __fmul_rn(-0.125f, vLb))));
        A[2] = __fmaf_rn(0.25f, db, __fmaf_rn(0.5f, da, __fmul_rn(0.25f, dLb)));
        B[2] = __fmaf_rn(0.25f, dRa, __fmaf_rn(0.5f, db, __fmul_rn(0.25f, da)));
        if (edge) {  // out-of-image columns take the values of column 0 / W-1
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float a_a = __shfl_sync(0xffffffffu, A[c], la), a_b = __shfl_sync(0xffffffffu, B[c], la);
            const float b_a = __shfl_sync(0xffffffffu, A[c], lb), b_b = __shfl_sync(0xffffffffu, B[c], lb);
            A[c] = ca ? a_b : a_a;
            B[c] = cb ? b_b : b_a;
          }
        }
      }
      // ---- level 0 out
      if (STORE_L0 && yy >= r0 && yy < r1) {
        float4* o = out0 + (size_t)yy * P.W + xa;
        if (wa) o[0] = make_float4(A[0], A[1], A[2], 0.0f);
        if (wb) o[1] = make_float4(B[0], B[1], B[2], 0.0f);
      }
      // ---- level 1: column taps a + 3b + 3c + d over rows 2j-1 .. 2j+2 (pass2.cg), then the row taps
      if (P.wantL1) {
        if ((yy & 1) == 0) {
          const int j = (yy >> 1) - 1;  // the level-1 row whose last tap is this row
          if (j >= j0 && j < j1) {
            float r[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const float ta = __fmul_rn(__fadd_rn(eA[c], A[c]), 0.125f);
              const float tb = __fmul_rn(__fadd_rn(eB[c], B[c]), 0.125f);
              const float tl = __shfl_up_sync(0xffffffffu, tb, 1);    // column xa - 1
              const float tr = __shfl_down_sync(0xffffffffu, ta, 1);  // column xb + 1
              r[c] = tap1331(tl, ta, tb, tr);
            }
            const int i = xa >> 1;
            if (w1) out1[(size_t)j * (P.W >> 1) + i] = make_float4(r[0], r[1], r[2], 0.0f);
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            eA[c] = __fadd_rn(pA[c], __fmul_rn(3.0f, A[c]));
            eB[c] = __fadd_rn(pB[c], __fmul_rn(3.0f, B[c]));
          }
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            eA[c] = __fadd_rn(eA[c], __fmul_rn(3.0f, A[c]));
            eB[c] = __fadd_rn(eB[c], __fmul_rn(3.0f, B[c]));
          }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          pA[c] = A[c];
          pB[c] = B[c];
        }
      }
      // ---- cornerness of row yy - 3 (klt_detector_pass1.cg / pass2.cg)
      // MIXED, wantCorn == KLT_CORN_PER_CAM: the cameras of the detector stage (re-read per row for
      // the register limit, see below)
      if (MIXED ? (P.wantCorn == KLT_CORN_PER_CAM
                       ? klt_in_stage<MIXED>(P.cams, klt_opaque((int)blockIdx.y) + P.camBase, KLT_STAGE_DETECT)
                       : P.wantCorn != 0)
                : P.wantCorn != 0) {
        prod[u][0] = __fmul_rn(A[1], A[1]);
        prod[u][1] = __fmul_rn(A[1], A[2]);
        prod[u][2] = __fmul_rn(A[2], A[2]);
        prod[u][3] = __fmul_rn(B[1], B[1]);
        prod[u][4] = __fmul_rn(B[1], B[2]);
        prod[u][5] = __fmul_rn(B[2], B[2]);
        const int yo = yy - 3;
        if (yo >= r0 && yo < r1) {  // implies 7 rows in the ring
          float s[6];
#pragma unroll
          for (int c = 0; c < 6; ++c) {
            float t = 0.f;
#pragma unroll
            for (int k = 0; k < 7; ++k) t = __fadd_rn(t, prod[(u + 1 + k) % 7][c]);  // top row first
            s[c] = t;
          }
          // a mixed group's detector window, read here rather than held across the row loop,
          // which is at the register limit (the camera index is re-read for the same reason)
          int ixlo = P.ixlo, ixhi = P.ixhi, iylo = P.iylo, iyhi = P.iyhi;
          if (MIXED) {
            const KltCam* K = P.cams + klt_opaque((int)blockIdx.y) + P.camBase;
            ixlo = __ldg(&K->ixlo);
            ixhi = __ldg(&K->ixhi);
            iylo = __ldg(&K->iylo);
            iyhi = __ldg(&K->iyhi);
          }
          float cs[2];
          float h[2][3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float sa = s[c], sb = s[c + 3];
            const float l2b = __shfl_up_sync(0xffffffffu, sb, 2);
            const float l1a = __shfl_up_sync(0xffffffffu, sa, 1), l1b = __shfl_up_sync(0xffffffffu, sb, 1);
            const float r1a = __shfl_down_sync(0xffffffffu, sa, 1), r1b = __shfl_down_sync(0xffffffffu, sb, 1);
            const float r2a = __shfl_down_sync(0xffffffffu, sa, 2);
            float t = __fadd_rn(0.f, l2b);  // columns xa-3 .. xa+3, left to right
            t = __fadd_rn(t, l1a);
            t = __fadd_rn(t, l1b);
            t = __fadd_rn(t, sa);
            t = __fadd_rn(t, sb);
            t = __fadd_rn(t, r1a);
            h[0][c] = __fadd_rn(t, r1b);
            t = __fadd_rn(0.f, l1a);  // columns xb-3 .. xb+3
            t = __fadd_rn(t, l1b);
            t = __fadd_rn(t, sa);
            t = __fadd_rn(t, sb);
            t = __fadd_rn(t, r1a);
            t = __fadd_rn(t, r1b);
            h[1][c] = __fadd_rn(t, r2a);
          }
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const float a = h[q][0], b = h[q][1], c = h[q][2];
            const float amc = __fsub_rn(a, c);
            const float rad = __fadd_rn(__fmul_rn(amc, amc), __fmul_rn(4.0f, __fmul_rn(b, b)));
            float v = __fmul_rn(0.5f, __fsub_rn(__fadd_rn(a, c), __fsqrt_rn(rad)));
            v = fmaxf(__fsub_rn(v, P.minC), 0.0f);
            const int gx = xa + q;
            const bool inside = (gx >= ixlo && gx <= ixhi) && (yo >= iylo && yo <= iyhi);
            cs[q] = inside ? v : 0.0f;
          }
          float* o = outc + (size_t)yo * P.W + xa;
          if (wa) o[0] = cs[0];
          if (wb) o[1] = cs[1];
        }
      }
    }
    if (r0 - 3 + base + 7 > r1 + 2) break;  // the rows that remain feed nothing of this chunk
  }
  // Level 2 of the pyramid tail is a programmatic dependent launch of this kernel: it is scheduled
  // once every CTA has a warp here or has exited, and its griddepcontrol.wait still waits for the
  // whole grid.  Not at kernel start: this pass shares the SMs with the previous frame's detector,
  // and level-2 CTAs launched then would sit in their wait through the whole pass, holding slots
  // and shared memory the detector could use.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

}  // namespace coslam
