// klt_pyr_tma.cuh -- pyramid levels >= 2 with the source tile staged into shared memory by TMA.
//
// [1 3 3 1] / 8 vertically, then horizontally with decimation by 2 (tap1331;
// pyramid_with_derivative_pass2.cg, host CGKLT/v3d_gpupyramid.cpp:402-420), in the oracle's order:
// bit-exact.  The data movement is TMA:
//   * the (2*TW+2) x (2*TH+2) source tile of float4 texels arrives through ONE
//     cp.async.bulk.tensor.3d (SASS: UTMALDG) issued by one thread and completes on an mbarrier; no
//     thread computes addresses or clamps coordinates for the load.  The tensor map describes one
//     pyramid level of the whole camera group (x: texels as pairs of 8-byte elements, y: rows,
//     z: cameras).
//   * CLAMP_TO_EDGE: TMA zero-fills texels outside the level, and the box origin may be negative;
//     the kernel never reads those texels -- it indexes the tile with the CLAMPED coordinate, which
//     always lies inside the box.
//   * the TW x TH output tile is written back with a TMA store (SASS: UTMASTG), which clips the
//     tile at the level border by itself.
// In a group of cameras of different sizes the tensor maps describe the group's largest level, and
// the kernel clamps to the camera's own source level (sw x sh = the camera's extent of level - 1): the
// box may cover padding of a smaller camera's slice, but only clamped coordinates are read.  The
// store clips at the largest level, so a tile that straddles the camera's border also writes into
// its padding (values derived from clamped data, never read); blocks wholly outside the camera exit.
#pragma once
#include <cuda.h>

#include "klt_kernels.cuh"

namespace coslam {

constexpr int PT_TW = 32, PT_TH = 8;
constexpr int PT_SW = 2 * PT_TW + 2, PT_SH = 2 * PT_TH + 2;  // source tile (texels)

__device__ __forceinline__ unsigned smem_u32(const void* p) {
  return (unsigned)__cvta_generic_to_shared(p);
}

// sw x sh: the source level of the group's cameras (MIXED: of the largest; each block reads its own
// camera's from `cams`); level: the destination level
template <bool MIXED>
__global__ void __launch_bounds__(256)
klt_pyr_down_tma(const __grid_constant__ CUtensorMap srcMap, const __grid_constant__ CUtensorMap dstMap,
                 int sw, int sh, const KltCam* __restrict__ cams, int level) {
  __shared__ __align__(128) float4 s_in[PT_SH][PT_SW];
  __shared__ __align__(128) float4 s_out[PT_TH][PT_TW];
  __shared__ float4 s_t[PT_TH][PT_SW];
  __shared__ __align__(8) unsigned long long s_bar;
  const int cam = blockIdx.z;
  const int ox = blockIdx.x * PT_TW, oy = blockIdx.y * PT_TH;
  if (MIXED) {
    const int Wc = __ldg(&cams[cam].W), Hc = __ldg(&cams[cam].H);
    if (ox >= (Wc >> level) || oy >= (Hc >> level) || !klt_in_stage<MIXED>(cams, cam, KLT_STAGE_PYR)) return;
    sw = Wc >> (level - 1);
    sh = Hc >> (level - 1);
  }
  const int tid = threadIdx.x;
  const int x0 = 2 * ox - 1, y0 = 2 * oy - 1;  // tile origin in the source level (may be -1)
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&srcMap) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&dstMap) : "memory");
  }
  __syncthreads();
  // Launched as a programmatic dependent of the kernel that writes the source level (klt_front or
  // the level above), whose CTAs may still run: everything above reads only the tensor maps and the
  // camera table.  The wait returns once that grid has completed and its stores, TMA stores
  // included, are visible; nothing of this level is read or written before it.  The level-0 flag,
  // the mixed-group clamping and the zero-fill reasoning above do not depend on it.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // The next level may be scheduled once every CTA of this one has passed here: by then all of them
  // hold their slots, so its CTAs (which wait above) take only slots this level does not need.
  // Triggering here rather than after the store gets them resident ahead of the side stream's
  // prefilter, which otherwise fills the SMs as level 2 drains and delays level 3 by about 4 us.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) {
    constexpr unsigned bytes = PT_SH * PT_SW * sizeof(float4);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&s_bar)), "r"(bytes)
                 : "memory");
    // coordinates: x in 8-byte elements (two per texel), y in rows, z = camera
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(&s_in[0][0])), "l"(&srcMap), "r"(2 * x0), "r"(y0), "r"(cam), "r"(smem_u32(&s_bar))
        : "memory");
  }
  {  // all threads wait for the tile (phase 0)
    unsigned done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(smem_u32(&s_bar))
          : "memory");
    }
  }
  // vertical [1 3 3 1] / 8 on rows 2j-1 .. 2j+2 (clamped), then horizontal with decimation
  for (int i = tid; i < PT_TH * PT_SW; i += 256) {
    const int ty = i / PT_SW, tx = i - ty * PT_SW;
    const int cx = clampi(x0 + tx, 0, sw - 1) - x0;
    const int yb = y0 + 2 * ty;
    const float4 a = s_in[clampi(yb, 0, sh - 1) - y0][cx], b = s_in[clampi(yb + 1, 0, sh - 1) - y0][cx],
                 c = s_in[clampi(yb + 2, 0, sh - 1) - y0][cx], d = s_in[clampi(yb + 3, 0, sh - 1) - y0][cx];
    s_t[ty][tx] = make_float4(tap1331(a.x, b.x, c.x, d.x), tap1331(a.y, b.y, c.y, d.y),
                              tap1331(a.z, b.z, c.z, d.z), 0.0f);
  }
  __syncthreads();
  {
    const int ty = tid / PT_TW, tx = tid - ty * PT_TW;
    const float4 a = s_t[ty][2 * tx], b = s_t[ty][2 * tx + 1], c = s_t[ty][2 * tx + 2], d = s_t[ty][2 * tx + 3];
    s_out[ty][tx] = make_float4(tap1331(a.x, b.x, c.x, d.x), tap1331(a.y, b.y, c.y, d.y),
                                tap1331(a.z, b.z, c.z, d.z), 0.0f);
  }
  // generic-proxy writes of s_out -> visible to the async proxy, then one TMA store of the tile
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (tid == 0) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&dstMap),
                 "r"(2 * ox), "r"(oy), "r"(cam), "r"(smem_u32(&s_out[0][0]))
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem may be released after the read
  }
}

}  // namespace coslam
