// klt.cu -- host side of the KLT tracker group + its C-ABI (see include/coslam_b200.h).
// Replaces V3D_GPU::KLT_SequenceTracker (tracking/CGKLT/v3d_gpuklt.{h,cpp}) and its GL/Cg runtime.
// All sequencing (status mapping, top-N selection, slot refill, provide) runs on the device; a
// frame costs one H2D copy per camera, one D2H copy of the feature table and one synchronise.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "klt_kernels.cuh"
#include "klt_track.cuh"
#include "klt_front.cuh"
#include "klt_pyr_tma.cuh"
#include "klt_cov.cuh"

using namespace coslam;

// Everything that differs between the frames run_frame enqueues: plan_frame decides it for a frame of
// one kind, plan_step for a step whose cameras have different ops.
struct FramePlan {
  const KltCam* cams;   // the camera table the kernels read: the group's, or a step's (stages)
  bool mixed;           // the kernels' MIXED instantiation runs (reads `cams`)
  bool tracked;         // the tracker runs (for some camera)
  int cornMode;         // FrontParams::wantCorn: 0, 1, or KLT_CORN_PER_CAM (a step)
  bool wantCorn;        // klt_front also produces the detector's cornerness map, and the detector runs
                        // (for some camera)
  bool storeL0;         // klt_front stores pyramid level 0
  bool lv0[64];         // the record of camera c's slice of the buffer the front pass writes (lv0Stored)
  bool earlyPrefilter;  // the detector's prefilter runs on auxStream right after klt_front
  bool trackerTail;     // the tracker writes the feature table (klt_status) and, with wantCorn, the
                        // suppression marks of the live tracks (klt_suppress) itself
  bool foldAdvance;     // klt_select_refill also writes the provided set to d_src (the advance copy),
                        // and the frame ends with the pyramid half of the advance
  int detectMode = 0;   // run_detector's mode
  int maxPresent = 0;   // detect: the longest present list (upload_present)
  bool provideAll = false;  // track: the tracked set becomes every camera's feature table (klt_copy_f4)
  KltCamList provide{};     // a step's TRACK cameras: their tracked sets go to both feature buffers
  // a step's only (plan_step)
  const uint8_t* ops = nullptr;  // the cameras with COSL_KLT_OP_SKIP are neither uploaded nor built
  int tab = -1;                  // its op table: h_stepCams[tab] -> d_stepCams[tab] == cams
  bool intoP1 = false;           // the front pass writes p1, not the third buffer, and so does the next
  bool flip = false;             // intoP1: p0 and p1 change roles at the end of the frame
  KltCamList exchangeEarly{};    // slices of p0 and p1 exchanged ahead of the front pass
  KltCamList exchangeLate{};     // ... after the tracker, or after the detector when nothing is tracked
};

// A frame whose image half cosl_klt_group_prefetch has enqueued and whose dependent half has not run
// (run_frame): what the second half needs of the first.  Until the frame is consumed, the handle's
// par, nxt, p1 and level-0 records stay those of the last consumed frame, so feeds, advances, fetch
// and the debug reads in between see the group as if nothing had been prefetched.
struct KltPrefetch {
  bool pending = false;
  FramePlan plan;
  uint8_t ops[64];            // the frame's ops (all NEXT when none were given); plan.ops points here
  bool step = false;          // ops were given: the frame is a step, as cosl_klt_group_step runs it
  bool advanceAfter = false;  // every camera TRACK: advance() follows the frame (run_step)
  int par = 0;                // the counter set next_par moved the frame to
  int buf = 0;                // the pyramid buffer its front pass wrote: p1 once consumed
};

struct cosl_klt {
  cosl_klt_config cfg;
  // W x H: the group's largest geometry (maximum width, maximum height); every buffer slice is laid
  // out at it and camera c uses the top-left hcam[c].W x hcam[c].H of its slice (klt_kernels.cuh)
  int C = 1, W = 0, H = 0, L = 0, fw = 0, fh = 0, F = 0, plCap = 0, device = 0;
  bool mixed = false;        // the cameras differ in size: kernels read the per-camera table
  bool pitchZeroOK = false;  // made by cosl_klt_group_create_sizes: pitch 0 = each camera's own width
  KltCam hcam[64];           // per camera: extent and detector window (camera 0's: the uniform case)
  KltCam* d_cams = nullptr;  // device copy of hcam, read by the kernels of a mixed group
  // cosl_klt_group_step: hcam with each camera's stages, written to one of three pinned tables and
  // copied to the device table of the same index, in turn (the front pass of a step may run while
  // the detectors of the two steps before it still read their tables); evStepTab[t] follows the last
  // copy from table t, evStepFence[t] the last group-stream reader of device table t
  KltCam* h_stepCams[3] = {nullptr, nullptr, nullptr};
  KltCam* d_stepCams[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t evStepTab[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t evStepFence[3] = {nullptr, nullptr, nullptr};
  int stepTab = 0;
  // the ops of the last frame call when it was a step: what cosl_klt_group_fetch hands back
  uint8_t stepOps[64];
  bool stepOpsValid = false;
  int levelSkip = 1, halfWidth = 3;
  float trackMargin = 4.f, conv = 0.1f, ssd = 5000.f, detectMargin = 10.f;
  cudaStream_t stream = nullptr;
  // image copies, klt_front and the pyramid tail run on the front stream, so that frame n+1's
  // pyramid is built while frames n and n-1 still run on `stream`.  Before a frame, the front stream
  // waits for the fence of each buffer it writes (evPyr, evPar, evStepFence), which `stream` records
  // behind the last stage that reads or writes that buffer (run_frame), and for evCams when
  // update_cameras has rewritten d_cams since; `stream` waits for evTail before the frame's tracker
  // or detector.
  cudaStream_t frontStream = nullptr;
  cudaEvent_t evPyr[3] = {nullptr, nullptr, nullptr}, evPar[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t evCams = nullptr, evTail = nullptr;
  bool camsDirty = false;
  // host uploads run on their own stream, one event per camera, so that klt_front of camera c
  // overlaps the copy of camera c+1 (cosl_klt_group_next path)
  cudaStream_t copyStream = nullptr;
  cudaEvent_t evImg[64] = {};
  cudaEvent_t evFront = nullptr;
  bool imgPerCam = false, frontRecorded = false;
  // the detector's prefilter needs only the cornerness map: on the re-detect path it runs on a side
  // stream next to the coarse pyramid levels and the tracker (valid on the unsuppressed map: the
  // suppression marks can only remove candidates, and klt_nm_verify reads the marked map)
  cudaStream_t auxStream = nullptr;
  cudaEvent_t evPre = nullptr;
  // geometry
  int lvW[8], lvH[8];
  long long lvOff[8];
  long long pyrStride = 0;  // float4 elements per camera
  size_t imgPitch = 0, imgStride = 0;
  int candCap = 0, smemKeys = 0;
  // device memory
  uint8_t* d_img = nullptr;
  // Three pyramid buffers.  p0 holds the previous frame's pyramid (the tracker's P0) and p1 the
  // current one (P1), as in the reference's two-buffer tracker; `nxt` is the buffer the next front
  // pass writes, p1 itself or, after an advance, the third buffer.  An advance makes p1 the new p0
  // and the old p0 the new p1 (the reference's swap), and points nxt at the third buffer, whose last
  // reader is the tracker of two frames back: so frame n+1's pyramid is built while frame n's tracker
  // runs.  A front pass writes nxt, and the frame's dependent half then sets p1 = nxt (run_frame).
  float4* d_pyr[3] = {nullptr, nullptr, nullptr};
  int p0 = 0, p1 = 1, nxt = 1;
  // level 0 of camera c's slice of d_pyr[b] holds its frame (see build_pyramid); per camera because
  // cosl_klt_group_advance_cams exchanges single cameras' slices between the buffers
  bool lv0Stored[3][64];
  // Three sets of what the front stream of frame n+1 writes while the detectors of frames n and n-1
  // may still read it: cornerness map, prelim list and counters.  A frame with a cornerness map
  // moves on to the next set; `par` is the set of the last frame (the one fetch and the debug reads
  // see).
  int par = 0;
  float* d_corn[3] = {nullptr, nullptr, nullptr};
  float4 *d_src = nullptr, *d_dst = nullptr, *d_ping = nullptr, *d_pong = nullptr, *d_res = nullptr;
  float4* d_present = nullptr;
  int* d_nPresent = nullptr;  // [C] lengths of the present lists in d_present
  int* d_nbr = nullptr;
  unsigned long long* d_cand = nullptr;
  unsigned* d_prelim[3] = {nullptr, nullptr, nullptr};  // [C][prelimCap] packed (y << 16 | x) of 3x3 maxima
  int prelimCap = 0;
  // [C][8]: [0] live tracks, [1] candidates, [2] returned count, [3] raw candidates, [4] prelim
  // (klt_kernels.cuh).  `stream` zeroes [0..3] of a frame; [4] belongs to the prefilter, which may
  // count before `stream` gets to the frame, so the front stream zeroes it.
  int* d_counters[3] = {nullptr, nullptr, nullptr};
  cosl_klt_feature* d_feat = nullptr;
  // fed points (3 floats each), then their slots and the per-camera placed counts (ints)
  void* d_feedbuf = nullptr;
  size_t feedCap = 0;  // bytes
  // pinned host mirrors
  cosl_klt_feature* h_feat = nullptr;
  int* h_counters = nullptr;
  float4* h_present = nullptr;
  int* h_nPresent = nullptr;
  // frame-pipelined ingest (cosl_klt_group_submit / _submit_step / _collect): two result slots,
  // completion events, and the ops of the frame each slot holds (all NEXT for a submit)
  cosl_klt_feature* h_featQ[2] = {nullptr, nullptr};
  int* h_cntQ[2] = {nullptr, nullptr};
  cudaEvent_t evDone[2] = {nullptr, nullptr};
  uint8_t opsQ[2][64];
  unsigned subSeq = 0;
  int nInFlight = 0;
  bool havePrev = false;
  KltPrefetch pf;
  // position covariances of the tracked slots (cosl_klt_set_covariance, klt_cov.cuh).  covNoise < 0:
  // disarmed, nothing below is allocated or launched.  d_cov [C][F][3] holds the last frame run_frame
  // computed it for (covFrame); it is read back with the feature table, into h_cov for the synchronous
  // calls and into h_covQ[slot] for a submitted frame (covQ[slot]: that frame was armed), and copy_out
  // hands the addressed cameras' entries to covOut, what cosl_klt_group_download_covariance returns
  // (covHanded: the last frame handed out was armed)
  float covNoise = -1.f;
  bool covFrame = false, covHanded = false;
  bool covQ[2] = {false, false};
  float* d_cov = nullptr;
  float* h_cov = nullptr;
  float* h_covQ[2] = {nullptr, nullptr};
  std::vector<float> covOut;
  // persistent fused gain tracker (klt_gain_fused)
  float4* d_state = nullptr;             // [C*F]
  unsigned long long* d_ver = nullptr;   // [2][C*F] (pass << 32 | beta bits)
  int* d_waitset = nullptr;   // [F][16]
  bool fusedOK = false;
  int fusedBlocks = 0;
  int fusedBlocksMixed = 0;  // of the MIXED instantiation, which steps run on every group
  int numSM = 132;
  int verBase = 0;
  // TMA descriptors of every pyramid level of the three buffers: [buffer][level], load box (source
  // of level + 1) and store box (destination of level - 1 -> level); klt_pyr_tma.cuh
  CUtensorMap tmLoad[3][8], tmStore[3][8];
  SectionTimer timer;
  int secPyr = 0, secTrack = 0, secDetect = 0, secSelect = 0;
};

namespace {

// Detector window of every camera, then hcam -> d_cams on the group's stream (the margin can change
// between frames).
// Detector window (klt_detector_pass2.cg: the pixel centre (i + 0.5) / n must lie inside
// [margin / n, 1 - margin / n]); evaluated with the fp32 expressions the oracle's margin mask
// evaluates per pixel (sx = (x + 0.5f) / W against margin / W and 1 - margin / W,
// oracle/klt_oracle.cpp), so the integer bounds select exactly the same pixels.
static int update_cameras(cosl_klt* g) {
  const float mg = g->detectMargin;
  auto bounds = [](int n, float lo, float hi, int& i0, int& i1) {
    const float nf = (float)n;
    i0 = n;
    i1 = -1;
    for (int i = 0; i < n; ++i) {
      const float sc = ((float)i + 0.5f) / nf;
      if (sc >= lo && sc <= hi) {
        i0 = std::min(i0, i);
        i1 = std::max(i1, i);
      }
    }
  };
  for (int c = 0; c < g->C; ++c) {
    KltCam& K = g->hcam[c];
    const float Wf = (float)K.W, Hf = (float)K.H;
    bounds(K.W, mg / Wf, 1.0f - mg / Wf, K.ixlo, K.ixhi);
    bounds(K.H, mg / Hf, 1.0f - mg / Hf, K.iylo, K.iyhi);
    K.stages = KLT_STAGE_ALL;
  }
  // pageable source: the copy is staged before the call returns, so hcam may change again
  COSL_CUDA(cudaMemcpyAsync(g->d_cams, g->hcam, sizeof(KltCam) * g->C, cudaMemcpyHostToDevice, g->stream));
  // the next frame's front pass reads d_cams
  COSL_CUDA(cudaEventRecord(g->evCams, g->stream));
  g->camsDirty = true;
  return COSL_OK;
}

// the pyramid buffer b's fence: its last group-stream reader or writer so far
static int fence_pyr(cosl_klt* g, int b) {
  COSL_CUDA(cudaEventRecord(g->evPyr[b], g->stream));
  return COSL_OK;
}

// The front stream's waits ahead of a frame whose front pass writes pyramid buffer nxt, the
// counter set par (wantCorn) and, for a step, op table tab (-1: none).
static int front_waits(cosl_klt* g, bool wantCorn, int tab) {
  COSL_CUDA(cudaStreamWaitEvent(g->frontStream, g->evPyr[g->nxt], 0));
  if (wantCorn) COSL_CUDA(cudaStreamWaitEvent(g->frontStream, g->evPar[g->par], 0));
  if (tab >= 0) COSL_CUDA(cudaStreamWaitEvent(g->frontStream, g->evStepFence[tab], 0));
  if (g->camsDirty) {
    COSL_CUDA(cudaStreamWaitEvent(g->frontStream, g->evCams, 0));
    g->camsDirty = false;
  }
  return COSL_OK;
}

// A frame with a cornerness map moves on to the next counter set; the set it leaves is fenced behind
// everything enqueued on `stream` so far, which includes the read-back of the frame before.
static int next_par(cosl_klt* g) {
  COSL_CUDA(cudaEventRecord(g->evPar[g->par], g->stream));
  g->par = (g->par + 1) % 3;
  return COSL_OK;
}

// the gain tracker's instantiation for this group's window (compile-time width when it is the live one)
using FusedFn = void (*)(const float4*, const float4*, long long, KltLevels, const KltCam*, int, const float4*,
                         float4*, unsigned long long*, const int*, float4*, int, KltTrackParams, KltTrackParams,
                         int, KltTail);
using PassFn = void (*)(const float4*, const float4*, long long, long long, int, int, const KltCam*,
                        const float4*, const float4*, float4*, const int*, KltTrackParams, int);
static FusedFn fused_kernel(const cosl_klt* g, bool mixed) {
  if (mixed) return g->halfWidth == KLT_HW_LIVE ? klt_gain_fused<KLT_HW_LIVE, true> : klt_gain_fused<0, true>;
  return g->halfWidth == KLT_HW_LIVE ? klt_gain_fused<KLT_HW_LIVE, false> : klt_gain_fused<0, false>;
}
static PassFn pass_kernel(const cosl_klt* g, bool mixed) {
  if (mixed) return g->halfWidth == KLT_HW_LIVE ? klt_gain_pass<KLT_HW_LIVE, true> : klt_gain_pass<0, true>;
  return g->halfWidth == KLT_HW_LIVE ? klt_gain_pass<KLT_HW_LIVE, false> : klt_gain_pass<0, false>;
}
// the instantiation of a kernel that reads the camera table (mixed) or not (klt_kernels.cuh, KltCam)
#define KLT_SIZED(mixed, ...) ((mixed) ? __VA_ARGS__<true> : __VA_ARGS__<false>)

int alloc_group(cosl_klt* g) {
  const int C = g->C, W = g->W, H = g->H, F = g->F;
  COSL_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
  COSL_CUDA(cudaStreamCreateWithFlags(&g->frontStream, cudaStreamNonBlocking));
  for (int b = 0; b < 3; ++b) {
    COSL_CUDA(cudaEventCreateWithFlags(&g->evPyr[b], cudaEventDisableTiming));
    COSL_CUDA(cudaEventCreateWithFlags(&g->evPar[b], cudaEventDisableTiming));
  }
  COSL_CUDA(cudaEventCreateWithFlags(&g->evCams, cudaEventDisableTiming));
  COSL_CUDA(cudaEventCreateWithFlags(&g->evTail, cudaEventDisableTiming));
  COSL_CUDA(cudaStreamCreateWithFlags(&g->copyStream, cudaStreamNonBlocking));
  COSL_CUDA(cudaEventCreateWithFlags(&g->evFront, cudaEventDisableTiming));
  for (int c = 0; c < C; ++c) COSL_CUDA(cudaEventCreateWithFlags(&g->evImg[c], cudaEventDisableTiming));
  COSL_CUDA(cudaStreamCreateWithFlags(&g->auxStream, cudaStreamNonBlocking));
  COSL_CUDA(cudaEventCreateWithFlags(&g->evPre, cudaEventDisableTiming));
  long long off = 0;
  for (int l = 0; l < g->L; ++l) {
    g->lvW[l] = W >> l;
    g->lvH[l] = H >> l;
    g->lvOff[l] = off;
    off += (long long)g->lvW[l] * g->lvH[l];
  }
  g->pyrStride = off;
  g->imgPitch = ((size_t)W + 15) & ~(size_t)15;
  g->imgStride = g->imgPitch * H;
  COSL_CUDA(cudaMalloc(&g->d_cams, sizeof(KltCam) * C));
  for (int t = 0; t < 3; ++t) {
    COSL_CUDA(cudaMalloc(&g->d_stepCams[t], sizeof(KltCam) * C));
    COSL_CUDA(cudaMallocHost(&g->h_stepCams[t], sizeof(KltCam) * C));
    COSL_CUDA(cudaEventCreateWithFlags(&g->evStepTab[t], cudaEventDisableTiming));
    COSL_CUDA(cudaEventCreateWithFlags(&g->evStepFence[t], cudaEventDisableTiming));
  }
  // candidate capacity: a strict (2r+1)^2 maximum admits at most one survivor per (r+1)^2 pixels
  // (of the largest camera, which bounds every camera's count)
  const int r = std::max(1, g->cfg.minDistance);
  long long maxCand = ((long long)(W + r) / (r + 1) + 1) * ((long long)(H + r) / (r + 1) + 1);
  int cap = 1024;
  while (cap < maxCand) cap <<= 1;
  g->candCap = cap;
  g->smemKeys = std::min(cap, KLT_MAX_SMEM_KEYS);
  COSL_CUDA(cudaMalloc(&g->d_img, g->imgStride * C));
  std::fill(&g->lv0Stored[0][0], &g->lv0Stored[0][0] + 3 * 64, true);
  for (int b = 0; b < 3; ++b) {
    COSL_CUDA(cudaMalloc(&g->d_pyr[b], sizeof(float4) * g->pyrStride * C));
    COSL_CUDA(cudaMemsetAsync(g->d_pyr[b], 0, sizeof(float4) * g->pyrStride * C, g->stream));
  }
  for (int b = 0; b < 3; ++b) COSL_CUDA(cudaMalloc(&g->d_corn[b], sizeof(float) * (size_t)W * H * C));
  const size_t fbytes = sizeof(float4) * (size_t)F * C;
  float4** bufs[] = {&g->d_src, &g->d_dst, &g->d_ping, &g->d_pong, &g->d_res, &g->d_present};
  std::vector<float4> init((size_t)F * C, make_float4(-1.f, -1.f, 1.f, 0.f));
  for (auto pb : bufs) {
    COSL_CUDA(cudaMalloc(pb, fbytes));
    COSL_CUDA(cudaMemcpy(*pb, init.data(), fbytes, cudaMemcpyHostToDevice));
  }
  COSL_CUDA(cudaMalloc(&g->d_cand, sizeof(unsigned long long) * (size_t)cap * C));
  // strict 3x3 maxima cannot be 8-adjacent: at most one per 2x2 block
  g->prelimCap = ((W + 1) / 2) * ((H + 1) / 2);
  for (int b = 0; b < 3; ++b) {
    COSL_CUDA(cudaMalloc(&g->d_prelim[b], sizeof(unsigned) * (size_t)g->prelimCap * C));
    COSL_CUDA(cudaMalloc(&g->d_counters[b], sizeof(int) * 8 * C));
    COSL_CUDA(cudaMemset(g->d_counters[b], 0, sizeof(int) * 8 * C));
  }
  COSL_CUDA(cudaMalloc(&g->d_feat, sizeof(cosl_klt_feature) * (size_t)F * C));
  COSL_CUDA(cudaMallocHost(&g->h_feat, sizeof(cosl_klt_feature) * (size_t)F * C));
  COSL_CUDA(cudaMallocHost(&g->h_counters, sizeof(int) * 8 * C));
  COSL_CUDA(cudaMallocHost(&g->h_present, fbytes));
  COSL_CUDA(cudaMalloc(&g->d_nPresent, sizeof(int) * C));
  COSL_CUDA(cudaMallocHost(&g->h_nPresent, sizeof(int) * C));
  // neighbour slots of the gain smoothness term (klt_tracker_with_gain.cg:64-75): NEAREST,
  // CLAMP_TO_EDGE lookups in the featW x featH slot texture at st0 +- ds0; betaN1 adds the SCALAR
  // ds0.x (resp. ds0.y) to both coordinates.
  std::vector<int> nbr((size_t)F * 8);
  const double fw = g->fw, fh = g->fh;
  for (int sy = 0; sy < g->fh; ++sy)
    for (int sx = 0; sx < g->fw; ++sx) {
      const double cx = sx + 0.5, cy = sy + 0.5;
      const double offs[8][2] = {{+1.0, +fh / fw}, {-1.0, -fh / fw}, {+fw / fh, +1.0},
                                 {-fw / fh, -1.0}, {+1.0, 0.0},      {-1.0, 0.0},
                                 {0.0, +1.0},      {0.0, -1.0}};
      for (int k = 0; k < 8; ++k) {
        const int nx = std::min(std::max((int)std::floor(cx + offs[k][0]), 0), g->fw - 1);
        const int ny = std::min(std::max((int)std::floor(cy + offs[k][1]), 0), g->fh - 1);
        nbr[(size_t)(sy * g->fw + sx) * 8 + k] = ny * g->fw + nx;
      }
    }
  COSL_CUDA(cudaMalloc(&g->d_nbr, sizeof(int) * nbr.size()));
  COSL_CUDA(cudaMemcpy(g->d_nbr, nbr.data(), sizeof(int) * nbr.size(), cudaMemcpyHostToDevice));
  // wait sets of the persistent gain tracker: 8 neighbours + up to 8 reverse neighbours (slots
  // that read this slot but are not among its neighbours are enough; duplicates are harmless)
  {
    std::vector<int> ws((size_t)F * 16, -1);
    std::vector<int> nrev(F, 0);
    bool ok = true;
    for (int i = 0; i < F; ++i)
      for (int k = 0; k < 8; ++k) ws[(size_t)i * 16 + k] = nbr[(size_t)i * 8 + k];
    for (int i = 0; i < F && ok; ++i)
      for (int k = 0; k < 8 && ok; ++k) {
        const int j = nbr[(size_t)i * 8 + k];  // i reads j  ->  j must wait for i
        bool have = false;
        for (int q = 0; q < 8 + nrev[j]; ++q)
          if (ws[(size_t)j * 16 + q] == i) have = true;
        if (have) continue;
        if (nrev[j] >= 8) {
          ok = false;
          break;
        }
        ws[(size_t)j * 16 + 8 + nrev[j]++] = i;
      }
    int dev = 0, coop = 0, nsm = 0, perSM = 0, perSMMixed = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    g->numSM = std::max(1, nsm);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fused_kernel(g, g->mixed), KLT_FUSED_THREADS, 0);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSMMixed, fused_kernel(g, true), KLT_FUSED_THREADS, 0);
    g->fusedOK = ok && coop && perSM > 0 && perSMMixed > 0 && !(g->cfg.compat & COSL_KLT_PASS_KERNELS);
    const int T = F * C;
    g->fusedBlocks = std::max(1, std::min(div_up(T, KLT_GPB), nsm * perSM));
    g->fusedBlocksMixed = std::max(1, std::min(div_up(T, KLT_GPB), nsm * perSMMixed));
    COSL_CUDA(cudaMalloc(&g->d_waitset, sizeof(int) * ws.size()));
    COSL_CUDA(cudaMemcpy(g->d_waitset, ws.data(), sizeof(int) * ws.size(), cudaMemcpyHostToDevice));
    COSL_CUDA(cudaMalloc(&g->d_state, sizeof(float4) * 2 * (size_t)T));
    COSL_CUDA(cudaMalloc(&g->d_ver, sizeof(unsigned long long) * 2 * (size_t)T));
    COSL_CUDA(cudaMemset(g->d_ver, 0, sizeof(unsigned long long) * 2 * (size_t)T));
    g->verBase = 0;
  }
  // tensor maps for the TMA pyramid kernel (driver entry point through the runtime: no -lcuda)
  if (g->L > 2) {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                 const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn ||
        qr != cudaDriverEntryPointSuccess)
      return set_error(COSL_E_CUDA, "KLT pyramid: cuTensorMapEncodeTiled is not available");
    for (int b = 0; b < 3; ++b)
      for (int l = 1; l < g->L; ++l) {
        // a level of the whole camera group: x = texels as pairs of 8-byte elements, y, camera
        const cuuint64_t dims[3] = {2ull * g->lvW[l], (cuuint64_t)g->lvH[l], (cuuint64_t)C};
        const cuuint64_t strides[2] = {16ull * g->lvW[l], 16ull * (cuuint64_t)g->pyrStride};
        const cuuint32_t es[3] = {1, 1, 1};
        const cuuint32_t boxL[3] = {2 * PT_SW, PT_SH, 1}, boxS[3] = {2 * PT_TW, PT_TH, 1};
        void* base = (void*)(g->d_pyr[b] + g->lvOff[l]);
        if (((EncodeFn)fn)(&g->tmLoad[b][l], CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, base, dims, strides, boxL, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS ||
            ((EncodeFn)fn)(&g->tmStore[b][l], CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, base, dims, strides, boxS, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
          return set_error(COSL_E_CUDA, "KLT pyramid: cannot encode the tensor maps of level %d (%dx%d)", l,
                           g->lvW[l], g->lvH[l]);
      }
  }
  // dynamic shared memory opt-in: the attribute belongs to the kernel, not to this group, so it is
  // the largest any group uses (a group created later must not lower it below an earlier one's)
  for (const bool mixed : {false, true})
    COSL_CUDA(cudaFuncSetAttribute(KLT_SIZED(mixed, klt_select_refill), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   KLT_MAX_SMEM_KEYS * (int)sizeof(unsigned long long)));
  COSL_TRY(update_cameras(g));
  g->secPyr = g->timer.section("klt_pyramid");
  g->secTrack = g->timer.section("klt_track");
  g->secDetect = g->timer.section("klt_detect");
  g->secSelect = g->timer.section("klt_select");
  COSL_CUDA(cudaStreamSynchronize(g->stream));
  return COSL_OK;
}

void free_group(cosl_klt* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  // a pending prefetch is not joined into `stream` (cosl_klt_group_prefetch)
  for (cudaStream_t st : {g->copyStream, g->frontStream, g->auxStream})
    if (st) cudaStreamSynchronize(st);
  g->timer.destroy();
  cudaFree(g->d_img);
  cudaFree(g->d_cams);
  for (int t = 0; t < 3; ++t) {
    cudaFree(g->d_stepCams[t]);
    if (g->h_stepCams[t]) cudaFreeHost(g->h_stepCams[t]);
    if (g->evStepTab[t]) cudaEventDestroy(g->evStepTab[t]);
    if (g->evStepFence[t]) cudaEventDestroy(g->evStepFence[t]);
    cudaFree(g->d_pyr[t]);
    cudaFree(g->d_corn[t]);
    cudaFree(g->d_prelim[t]);
    cudaFree(g->d_counters[t]);
    if (g->evPyr[t]) cudaEventDestroy(g->evPyr[t]);
    if (g->evPar[t]) cudaEventDestroy(g->evPar[t]);
  }
  cudaFree(g->d_src);
  cudaFree(g->d_dst);
  cudaFree(g->d_ping);
  cudaFree(g->d_pong);
  cudaFree(g->d_res);
  cudaFree(g->d_present);
  cudaFree(g->d_nPresent);
  cudaFree(g->d_nbr);
  if (g->auxStream) cudaStreamDestroy(g->auxStream);
  if (g->evPre) cudaEventDestroy(g->evPre);
  if (g->frontStream) cudaStreamDestroy(g->frontStream);
  if (g->evCams) cudaEventDestroy(g->evCams);
  if (g->evTail) cudaEventDestroy(g->evTail);
  if (g->copyStream) cudaStreamDestroy(g->copyStream);
  if (g->evFront) cudaEventDestroy(g->evFront);
  for (int c = 0; c < 64; ++c)
    if (g->evImg[c]) cudaEventDestroy(g->evImg[c]);
  cudaFree(g->d_cand);
  cudaFree(g->d_feat);
  cudaFree(g->d_feedbuf);
  cudaFree(g->d_state);
  cudaFree(g->d_ver);
  cudaFree(g->d_waitset);
  cudaFreeHost(g->h_feat);
  cudaFreeHost(g->h_counters);
  cudaFreeHost(g->h_present);
  cudaFreeHost(g->h_nPresent);
  for (int i = 0; i < 2; ++i) {
    if (g->h_featQ[i]) cudaFreeHost(g->h_featQ[i]);
    if (g->h_cntQ[i]) cudaFreeHost(g->h_cntQ[i]);
    if (g->evDone[i]) cudaEventDestroy(g->evDone[i]);
    if (g->h_covQ[i]) cudaFreeHost(g->h_covQ[i]);
  }
  cudaFree(g->d_cov);
  if (g->h_cov) cudaFreeHost(g->h_cov);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
}

// ---- stages (all asynchronous; the streams of each are in run_frame) ----

// camera c's image: hcam[c].W x hcam[c].H bytes, rows `pitch` bytes apart (0: hcam[c].W, pitch_ok);
// on the front stream, or for a multi-camera host upload on the copy stream.  ops (a step, else
// nullptr): the cameras with COSL_KLT_OP_SKIP are not copied; their events are still recorded, so
// the front pass can wait for any camera's.
int upload_images(cosl_klt* g, const uint8_t* const* imgs, size_t pitch, cudaMemcpyKind kind,
                  const uint8_t* ops) {
  if (kind == cudaMemcpyHostToDevice && g->C > 1) {
    // the previous frame's front pass must have consumed d_img before it is overwritten
    if (g->frontRecorded) COSL_CUDA(cudaStreamWaitEvent(g->copyStream, g->evFront, 0));
    for (int c = 0; c < g->C; ++c) {
      if (ops && ops[c] == COSL_KLT_OP_SKIP) {
        COSL_CUDA(cudaEventRecord(g->evImg[c], g->copyStream));
        continue;
      }
      const size_t w = (size_t)g->hcam[c].W, sp = pitch ? pitch : w;
      if (sp == w && g->imgPitch == w)  // one contiguous block
        COSL_CUDA(cudaMemcpyAsync(g->d_img + (size_t)c * g->imgStride, imgs[c], w * g->hcam[c].H, kind,
                                  g->copyStream));
      else
        COSL_CUDA(cudaMemcpy2DAsync(g->d_img + (size_t)c * g->imgStride, g->imgPitch, imgs[c], sp, w,
                                    g->hcam[c].H, kind, g->copyStream));
      COSL_CUDA(cudaEventRecord(g->evImg[c], g->copyStream));
    }
    g->imgPerCam = true;
    return COSL_OK;
  }
  for (int c = 0; c < g->C; ++c)
    if (!ops || ops[c] != COSL_KLT_OP_SKIP)
      COSL_CUDA(cudaMemcpy2DAsync(g->d_img + (size_t)c * g->imgStride, g->imgPitch, imgs[c],
                                  pitch ? pitch : (size_t)g->hcam[c].W, g->hcam[c].W, g->hcam[c].H, kind,
                                  g->frontStream));
  return COSL_OK;
}

// klt_nm_prefilter on `st` (prefilter radius = min(minDistance, 3))
static void launch_prefilter(cosl_klt* g, cudaStream_t st, bool mixed, const KltCam* cams) {
  const int pr = std::min(std::max(1, g->cfg.minDistance), 3);
  dim3 gp(div_up(g->W, 32 - 2 * pr), div_up(g->H, 8 * NP_ROWS), g->C);
  const long long cs = (long long)g->W * g->H;
  const auto kern = pr == 3 ? (mixed ? klt_nm_prefilter<3, true> : klt_nm_prefilter<3, false>)
                  : pr == 2 ? (mixed ? klt_nm_prefilter<2, true> : klt_nm_prefilter<2, false>)
                            : (mixed ? klt_nm_prefilter<1, true> : klt_nm_prefilter<1, false>);
  COSL_LAUNCH(kern, gp, 256, 0, st, g->d_corn[g->par], g->W, cs, cams, g->W, g->H, g->d_prelim[g->par],
              g->prelimCap, g->d_counters[g->par]);
}

// The tracker's level list: L-1, L-1-levelSkip, ... down to >= 0.  scaled: the 2x2 tracker's
// window step at each level (2^level); 1 for the gain trackers.
static KltLevels tracker_levels(const cosl_klt* g, bool scaled) {
  KltLevels LV;
  LV.n = 0;
  float mult = scaled ? (float)(1 << (g->L - 1)) : 1.0f;
  for (int level = g->L - 1; level >= 0; level -= g->levelSkip) {
    LV.level[LV.n] = level;
    LV.w[LV.n] = g->lvW[level];
    LV.h[LV.n] = g->lvH[level];
    LV.off[LV.n] = g->lvOff[level];
    LV.mult[LV.n] = mult;
    if (scaled) mult /= (float)(1 << g->levelSkip);
    ++LV.n;
  }
  return LV;
}

// true when the tracker's level list contains level 0
static bool tracker_reads_level0(const cosl_klt* g) { return (g->L - 1) % g->levelSkip == 0; }

// the persistent gain tracker (klt_gain_fused) runs, not the per-pass kernels or the 2x2 tracker
static bool fused_tracker(const cosl_klt* g) { return g->cfg.trackWithGain && g->fusedOK; }

// PyramidWithDerivativesCreator::buildPyramidForGrayscaleImage (v3d_gpupyramid.cpp:366-429), on the
// front stream
int build_pyramid(cosl_klt* g, const FramePlan& p) {
  cudaStream_t st = g->frontStream;
  float4* P = g->d_pyr[g->nxt];
  g->timer.begin(g->secPyr, st);
  // level 0 + level 1 + (optionally) the detector's cornerness map in one pass over the image
  FrontParams fp;
  fp.img = g->d_img;
  fp.imgPitch = g->imgPitch;
  fp.imgStride = g->imgStride;
  fp.pyr = P;
  fp.pyrStride = g->pyrStride;
  fp.lv1Off = g->L > 1 ? g->lvOff[1] : 0;
  fp.corn = g->d_corn[g->par];
  fp.cornStride = (long long)g->W * g->H;
  fp.W = g->W;
  fp.H = g->H;
  fp.nStrips = div_up(g->W, FS_SW);
  fp.nChunks = div_up(g->H, FS_R);
  fp.wantL1 = g->L > 1 ? 1 : 0;
  const auto front = p.storeL0 ? (p.mixed ? klt_front<true, true> : klt_front<true, false>)
                                : (p.mixed ? klt_front<false, true> : klt_front<false, false>);
  fp.wantCorn = p.cornMode;
  fp.minC = g->cfg.minCornerness;
  fp.ixlo = g->hcam[0].ixlo;
  fp.ixhi = g->hcam[0].ixhi;
  fp.iylo = g->hcam[0].iylo;
  fp.iyhi = g->hcam[0].iyhi;
  fp.cams = p.cams;
  // the grid covers the largest camera; a smaller camera's surplus warps exit
  const int nWarps = fp.nStrips * fp.nChunks;
  if (g->imgPerCam) {
    // two half-groups: the front pass of the first half overlaps the upload of the second (a launch
    // per camera would leave the SMs mostly empty: 500 warps per 1280x720 camera)
    g->imgPerCam = false;
    const int half = (g->C + 1) / 2;
    for (int c0 = 0; c0 < g->C; c0 += half) {
      const int nc = std::min(half, g->C - c0);
      COSL_CUDA(cudaStreamWaitEvent(st, g->evImg[c0 + nc - 1], 0));
      fp.camBase = c0;
      dim3 g1(div_up(nWarps, FS_WARPS), nc);
      COSL_LAUNCH(front, g1, 32 * FS_WARPS, 0, st, fp);
    }
  } else {
    fp.camBase = 0;
    dim3 g0(div_up(nWarps, FS_WARPS), g->C);
    COSL_LAUNCH(front, g0, 32 * FS_WARPS, 0, st, fp);
  }
  COSL_CUDA(cudaEventRecord(g->evFront, st));
  g->frontRecorded = true;
  if (p.earlyPrefilter) {
    COSL_CUDA(cudaStreamWaitEvent(g->auxStream, g->evFront, 0));
    launch_prefilter(g, g->auxStream, p.mixed, p.cams);
    COSL_CUDA(cudaEventRecord(g->evPre, g->auxStream));
  }
  // source tile by TMA load, destination tile by TMA store (klt_pyr_tma.cuh).  Each level is a
  // programmatic dependent launch of the kernel before it (klt_front, then the level above): its
  // CTAs are scheduled before that kernel ends and wait in the kernel for the source level.
  // The front passes themselves are plain launches: they read the image copies and the counter
  // reset ahead of them on this stream and have no grid-dependency wait.
  for (int l = 2; l < g->L; ++l) {
    dim3 gl(div_up(g->lvW[l], PT_TW), div_up(g->lvH[l], PT_TH), g->C);
    COSL_LAUNCH_PDL(KLT_SIZED(p.mixed, klt_pyr_down_tma), gl, 256, 0, st, g->tmLoad[g->nxt][l - 1],
                    g->tmStore[g->nxt][l], g->lvW[l - 1], g->lvH[l - 1], p.cams, l);
  }
  g->timer.end(st);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// W, H, vr*: camera 0's, which are every camera's unless the group is mixed (klt_vr_lo / _hi)
KltTrackParams track_params(const cosl_klt* g, bool strict) {
  KltTrackParams P;
  P.W = g->hcam[0].W;
  P.H = g->hcam[0].H;
  P.F = g->F;
  P.halfWidth = g->halfWidth;
  P.strict = strict ? 1 : 0;
  P.margin = g->trackMargin;
  const float Wf = (float)P.W, Hf = (float)P.H, m = g->trackMargin;
  if (strict) {
    P.sqrConv = g->conv * g->conv;
    P.ssdThr = g->ssd;
    P.vr0 = m / Wf;
    P.vr1 = m / Hf;
    P.vr2 = 1.0f - m / Wf;
    P.vr3 = 1.0f - m / Hf;
  } else {  // v3d_gpuklt.cpp:246-248, 266-270
    P.sqrConv = 1000000.0f;
    P.ssdThr = 1000000.0f;
    P.vr0 = -1.0f;
    P.vr1 = -1.0f;
    P.vr2 = 2.0f;
    P.vr3 = 2.0f;
  }
  P.lambda = 1.0f;
  P.delta = 200.0f;
  return P;
}

// KLT_TrackerWithGain::trackFeaturesAndGain (v3d_gpuklt.cpp:205-305) /
// KLT_Tracker::trackFeatures (:99-161); result -> d_res.  The caller fences both buffers after it.
int run_tracker(cosl_klt* g, const FramePlan& p) {
  const float4* P0 = g->d_pyr[g->p0];
  const float4* P1 = g->d_pyr[g->p1];
  const int wpb = 8;  // warps per block (2x2 tracker: one warp per slot)
  dim3 grid(div_up(g->F, wpb), g->C);
  dim3 gridHalf(div_up(g->F, 256 / KLT_G), g->C);  // gain tracker: one lane group per slot
  KltLevels LV = tracker_levels(g, !g->cfg.trackWithGain);
  g->timer.begin(g->secTrack, g->stream);
  if (fused_tracker(g)) {
    int nIter = g->cfg.nIterations, C = g->C;
    const int nPass = LV.n * nIter;
    if (g->verBase > 2000000000 - 2 * nPass) {  // version wrap: restart the counters
      COSL_CUDA(cudaMemsetAsync(g->d_ver, 0, sizeof(unsigned long long) * 2 * (size_t)g->F * g->C,
                                g->stream));
      g->verBase = 0;
    }
    long long pyrStride = g->pyrStride;
    KltTrackParams Plax = track_params(g, false), Pstrict = track_params(g, true);
    int verBase = g->verBase;
    // the feature table and, when this frame produced a cornerness map, its suppression marks
    KltTail tail = {g->d_feat, g->d_counters[g->par], g->d_corn[g->par], (long long)g->W * g->H, g->W,
                    p.wantCorn ? 1 : 0};
    void* args[] = {(void*)&P0,          (void*)&P1,       (void*)&pyrStride,  (void*)&LV,
                    (void*)&p.cams,      (void*)&nIter,    (void*)&g->d_src,   (void*)&g->d_state,
                    (void*)&g->d_ver,    (void*)&g->d_waitset, (void*)&g->d_res, (void*)&C,
                    (void*)&Plax,        (void*)&Pstrict,  (void*)&verBase,    (void*)&tail};
    COSL_CUDA(cudaLaunchCooperativeKernel((const void*)fused_kernel(g, p.mixed),
                                          dim3(p.mixed ? g->fusedBlocksMixed : g->fusedBlocks),
                                          dim3(KLT_FUSED_THREADS), args, 0, g->stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    g->verBase += nPass;
  } else if (g->cfg.trackWithGain) {
    const float4* in = g->d_src;
    float4* bufs[2] = {g->d_ping, g->d_pong};
    const PassFn pass = pass_kernel(g, p.mixed);
    int which = 0, first = 1;
    bool strict = false;
    for (int li = 0; li < LV.n; ++li) {
      for (int iter = 1; iter <= g->cfg.nIterations; ++iter) {
        if (iter == 1)
          strict = false;
        else if (iter == g->cfg.nIterations)
          strict = true;
        const bool last = (li == LV.n - 1) && (iter == g->cfg.nIterations);
        float4* out = last ? g->d_res : bufs[which];
        COSL_LAUNCH(pass, gridHalf, 256, 0, g->stream, P0, P1, g->pyrStride, LV.off[li], LV.level[li],
                    LV.w[li], p.cams, g->d_src, in, out, g->d_nbr, track_params(g, strict), first);
        in = out;
        which ^= 1;
        first = 0;
      }
    }
  } else {
    const int nIter = (g->cfg.compat & COSL_KLT_COMPAT_ITER5) ? 5 : g->cfg.nIterations;
    const int hw2 = g->halfWidth, npx2 = (2 * hw2 + 1) * (2 * hw2 + 1);
    const bool tiled = (npx2 <= KLT_G * KLT_ROUNDS) && (2 * hw2 + 4 <= KLT_TW) && (2 * hw2 + 2 <= 8) &&
                       !(g->cfg.compat & COSL_KLT_PASS_KERNELS);
    if (tiled) {
      dim3 gt(div_up(g->F, 16), g->C);
      COSL_LAUNCH(KLT_SIZED(p.mixed, klt_track_2x2_tiled), gt, 128, 0, g->stream, P0, P1, g->pyrStride, LV, p.cams,
                  g->d_src, g->d_res, track_params(g, true), nIter);
    } else {
      COSL_LAUNCH(KLT_SIZED(p.mixed, klt_track_2x2), grid, wpb * 32, 0, g->stream, P0, P1, g->pyrStride, LV, p.cams,
                  g->d_src, g->d_res, track_params(g, true), nIter);
    }
  }
  g->timer.end(g->stream);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// The position covariances of an armed frame (klt_cov.cuh) into d_cov.  After a tracker it reads the
// pyramids, the start table d_src and the result d_res that tracker read and wrote, at its last level,
// so it runs before the fences of p0 / p1 (it is their last reader), before a step's exchange of
// their slices and before provide or the refill rewrite d_src.  A frame without a tracker leaves
// every camera NaN.
static int run_covariance(cosl_klt* g, const FramePlan& p) {
  if (!p.tracked) {
    COSL_CUDA(cudaMemsetAsync(g->d_cov, 0xff, sizeof(float) * 3 * g->F * g->C, g->stream));  // NaN
    return COSL_OK;
  }
  const KltLevels LV = tracker_levels(g, false);
  const int li = LV.n - 1;
  const KltTrackParams P = track_params(g, true);
  COSL_LAUNCH(klt_cov, dim3(div_up(g->F, 8), g->C), 256, 0, g->stream, g->d_pyr[g->p0], g->d_pyr[g->p1],
              g->pyrStride, LV.off[li], LV.w[li], LV.level[li], p.cams, g->d_src, g->d_res, g->d_cov, g->F,
              g->halfWidth, g->cfg.trackWithGain ? 1 : 0, P.lambda, P.delta, g->covNoise);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// KLT_Detector::detectCorners + extractCorners (v3d_gpuklt.cpp:423-588) and the slot logic of
// detect/redetect (:651-805) on the cornerness map klt_front produced for this frame.  p.detectMode
// 0: detect (present = the external points of upload_present, p.maxPresent = the longest list),
// 1: redetect, 2: per camera of a step (klt_select_refill).
int run_detector(cosl_klt* g, const FramePlan& p) {
  const int mode = p.detectMode, maxPresent = p.maxPresent;
  g->timer.begin(g->secDetect, g->stream);
  const long long cs = (long long)g->W * g->H;
  float* corn = g->d_corn[g->par];
  int* counters = g->d_counters[g->par];
  if (mode != 0 && p.tracked && !p.trackerTail) {  // the live tracks of the re-detecting cameras
    dim3 gs(div_up(g->F, 256), g->C);
    COSL_LAUNCH(KLT_SIZED(p.mixed, klt_suppress), gs, 256, 0, g->stream, g->d_res, g->F, (const int*)nullptr, g->F,
                corn, g->W, cs, p.cams, g->W, g->H, KLT_STAGE_TRACK | KLT_STAGE_DETECT);
  } else if (mode == 0 && maxPresent > 0) {
    dim3 gs(div_up(maxPresent, 256), g->C);
    COSL_LAUNCH(KLT_SIZED(p.mixed, klt_suppress), gs, 256, 0, g->stream, g->d_present, 0, g->d_nPresent, g->F,
                corn, g->W, cs, p.cams, g->W, g->H, KLT_STAGE_DETECT);
  }
  const int r = std::max(1, g->cfg.minDistance);
  if (p.earlyPrefilter)
    COSL_CUDA(cudaStreamWaitEvent(g->stream, g->evPre, 0));
  else
    launch_prefilter(g, g->stream, p.mixed, p.cams);
  dim3 gv(2 * g->numSM, g->C);
  COSL_LAUNCH(KLT_SIZED(p.mixed, klt_nm_verify), gv, 256, 0, g->stream, corn, g->W, cs, p.cams, g->W, g->H, r,
              g->d_prelim[g->par], g->prelimCap, g->d_cand, g->candCap, counters);
  g->timer.end(g->stream);
  g->timer.begin(g->secSelect, g->stream);
  COSL_LAUNCH(KLT_SIZED(p.mixed, klt_select_refill), g->C, 1024, g->smemKeys * sizeof(unsigned long long), g->stream,
              g->d_cand, g->candCap, g->plCap, counters, g->d_feat, g->d_dst,
              p.foldAdvance ? g->d_src : (float4*)nullptr, g->d_present,
              maxPresent > 0 ? g->d_nPresent : (const int*)nullptr, g->F, p.cams, g->W, g->H, mode,
              g->cfg.trackWithGain ? 1 : 0, g->smemKeys, (g->cfg.compat & COSL_KLT_COMPAT_HISTOPYR) ? 1 : 0);
  g->timer.end(g->stream);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

int fetch_results(cosl_klt* g) {
  COSL_CUDA(cudaMemcpyAsync(g->h_feat, g->d_feat, sizeof(cosl_klt_feature) * (size_t)g->F * g->C,
                            cudaMemcpyDeviceToHost, g->stream));
  COSL_CUDA(cudaMemcpyAsync(g->h_counters, g->d_counters[g->par], sizeof(int) * 8 * g->C,
                            cudaMemcpyDeviceToHost, g->stream));
  if (g->covFrame)
    COSL_CUDA(cudaMemcpyAsync(g->h_cov, g->d_cov, sizeof(float) * 3 * g->F * g->C, cudaMemcpyDeviceToHost,
                              g->stream));
  COSL_CUDA(cudaStreamSynchronize(g->stream));
  return COSL_OK;
}

// The pyramid half of advanceFrame: p1 becomes p0, and the old p0 becomes p1, as the reference swaps
// its two pyramids.  The next front pass writes the third buffer, not p1, so it does not wait for
// the tracker that read p0 and p1 (whose last frame might still be running).
static void advance_pyramids(cosl_klt* g) {
  std::swap(g->p0, g->p1);
  g->nxt = 3 - g->p0 - g->p1;
}

int advance(cosl_klt* g) {
  // swapFeatureBuffers + swap pyramids (v3d_gpuklt.h:252-259); the feature buffer is copied, not
  // swapped, so a later feed() still sees the provided set (see DESIGN.md, quirk list)
  const size_t n = (size_t)g->F * g->C;
  COSL_LAUNCH(klt_copy_f4, (unsigned)div_up64(n, 256), 256, 0, g->stream, g->d_dst, g->d_src, n);
  advance_pyramids(g);
  return COSL_OK;
}

// Exchange the cameras' slices of p0 and p1 (and their level-0 records) and copy their provided
// feature sets to d_src (nFeat = F; 0: no copy), on g->stream; both buffers are fenced after it.
static int exchange_slices(cosl_klt* g, const KltCamList& L, int nFeat) {
  if (L.n == 0) return COSL_OK;
  dim3 grid((unsigned)std::min<long long>(div_up64(g->pyrStride, 256), 2 * g->numSM), L.n);
  COSL_LAUNCH(klt_advance_cams, grid, 256, 0, g->stream, g->d_pyr[g->p0], g->d_pyr[g->p1], g->pyrStride,
              g->d_dst, g->d_src, nFeat, L);
  for (int k = 0; k < L.n; ++k) std::swap(g->lv0Stored[g->p0][L.cam[k]], g->lv0Stored[g->p1][L.cam[k]]);
  COSL_TRY(fence_pyr(g, g->p0));
  return fence_pyr(g, g->p1);
}

// advance() for the cameras with cams[c] != 0 only.  A strict subset cannot move the buffer
// indices: the cameras' slices of p0 and p1 are exchanged instead (klt_advance_cams), as advance()
// exchanges the roles of the two buffers.  nxt stays: the third buffer holds nothing any camera keeps.
int advance_cams(cosl_klt* g, const uint8_t* cams) {
  KltCamList L;
  L.n = 0;
  for (int c = 0; c < g->C; ++c)
    if (cams[c]) L.cam[L.n++] = c;
  if (L.n == g->C) return advance(g);
  return exchange_slices(g, L, g->F);
}

// The present lists of a detect: camera c's nPresent[c] points (x, y, ignored) -> d_present[c][.],
// the lengths -> d_nPresent.  *maxPresent = the longest list (0: nothing uploaded).
int upload_present(cosl_klt* g, const int* nPresent, const float* const* present3, int* maxPresent) {
  int mx = 0;
  size_t n4 = 0;  // float4s up to the end of the last non-empty list
  for (int c = 0; c < g->C; ++c) {
    const int n = nPresent[c];
    for (int i = 0; i < n; ++i)
      g->h_present[(size_t)c * g->F + i] = make_float4(present3[c][3 * i], present3[c][3 * i + 1], 0.f, 0.f);
    g->h_nPresent[c] = n;
    if (n > 0) n4 = (size_t)c * g->F + n;
    mx = std::max(mx, n);
  }
  *maxPresent = mx;
  if (mx == 0) return COSL_OK;
  COSL_CUDA(cudaMemcpyAsync(g->d_present, g->h_present, sizeof(float4) * n4, cudaMemcpyHostToDevice, g->stream));
  COSL_CUDA(cudaMemcpyAsync(g->d_nPresent, g->h_nPresent, sizeof(int) * g->C, cudaMemcpyHostToDevice, g->stream));
  return COSL_OK;
}

// feedExternFeaturePoints (v3d_gpuklt.cpp:808-855) for every camera with npts[c] >= 0, into d_dst:
// one launch of klt_feed_kill and klt_feed_place for all cameras with points, one H2D copy, one D2H
// copy, one synchronise.  No advance.
int feed_cams(cosl_klt* g, const int* npts, const float* const* pts3, int* const* trackIds, int* nFed) {
  KltFeedList L;
  L.n = 0;
  L.off[0] = 0;
  long long total = 0;
  for (int c = 0; c < g->C; ++c) {
    if (npts[c] >= 0) nFed[c] = 0;
    if (npts[c] <= 0) continue;
    total += npts[c];
    if (total > (1 << 26)) return set_error(COSL_E_INVALID, "feed: too many points (%lld)", total);
    L.cam[L.n] = c;
    L.off[++L.n] = (int)total;
  }
  if (L.n == 0) return COSL_OK;
  const size_t ptsBytes = sizeof(float) * 3 * total, idsCount = (size_t)total + L.n;
  const size_t bytes = ptsBytes + sizeof(int) * idsCount;
  if (bytes > g->feedCap) {
    cudaFree(g->d_feedbuf);
    g->d_feedbuf = nullptr;
    g->feedCap = 0;
    COSL_CUDA(cudaMalloc(&g->d_feedbuf, bytes));
    g->feedCap = bytes;
  }
  std::vector<float> pts((size_t)3 * total);
  for (int k = 0; k < L.n; ++k)
    std::memcpy(pts.data() + (size_t)3 * L.off[k], pts3[L.cam[k]], sizeof(float) * 3 * (L.off[k + 1] - L.off[k]));
  float* d_pts = (float*)g->d_feedbuf;
  int* d_ids = (int*)((char*)g->d_feedbuf + ptsBytes);
  COSL_CUDA(cudaMemcpyAsync(d_pts, pts.data(), ptsBytes, cudaMemcpyHostToDevice, g->stream));
  COSL_CUDA(cudaMemsetAsync(d_ids, 0xff, sizeof(int) * idsCount, g->stream));
  COSL_LAUNCH(klt_feed_kill, dim3(div_up(g->F, 256), L.n), 256, 0, g->stream, g->d_dst, g->F, d_pts, L,
              (g->cfg.compat & COSL_KLT_COMPAT_FEED_STRIDE2) ? 2 : 3);
  COSL_LAUNCH(klt_feed_place, L.n, 32, 0, g->stream, g->d_dst, g->F, d_pts, L, d_ids, d_ids + total);
  std::vector<int> ids(idsCount);
  COSL_CUDA(cudaMemcpyAsync(ids.data(), d_ids, sizeof(int) * idsCount, cudaMemcpyDeviceToHost, g->stream));
  COSL_CUDA(cudaStreamSynchronize(g->stream));
  for (int k = 0; k < L.n; ++k) {
    const int c = L.cam[k];
    std::memcpy(trackIds[c], ids.data() + L.off[k], sizeof(int) * (L.off[k + 1] - L.off[k]));
    nFed[c] = ids[total + k];
  }
  return COSL_OK;
}

enum FrameKind {
  FRAME_DETECT,    // detect, first: pyramid with the cornerness map, detector, slot refill
  FRAME_TRACK,     // track: pyramid, tracker; the tracked set becomes the next frame's table
  FRAME_REDETECT,  // redetect, next, next_dev, submit: as FRAME_TRACK, then the detector refills
};

// The plan of a frame of one kind for every camera.  maxPresent: the longest present list of a
// detect (upload_present).  foldAdvance (detector kinds): advanceFrame follows the frame, and
// klt_select_refill writes the provided set to both feature buffers, so the advance is the pyramid
// flip alone.
static FramePlan plan_frame(const cosl_klt* g, FrameKind kind, int maxPresent, bool foldAdvance) {
  FramePlan p;
  p.cams = g->d_cams;
  p.mixed = g->mixed;
  p.tracked = kind != FRAME_DETECT;
  p.wantCorn = kind != FRAME_TRACK;
  p.cornMode = p.wantCorn ? 1 : 0;
  // A re-detect frame has its cornerness fused into the front pass, so nothing but a tracker that
  // visits level 0 reads that level.  It is stored only then: at 16 B/px it is larger than the L2,
  // and writing it would evict the pyramid levels the tracker that follows reads.
  p.storeL0 = kind != FRAME_REDETECT || tracker_reads_level0(g);
  std::fill(p.lv0, p.lv0 + g->C, p.storeL0);
  p.earlyPrefilter = kind == FRAME_REDETECT;
  p.trackerTail = fused_tracker(g);
  p.foldAdvance = foldAdvance;
  p.detectMode = kind == FRAME_REDETECT ? 1 : 0;
  p.maxPresent = maxPresent;
  p.provideAll = kind == FRAME_TRACK;
  return p;
}

// the stages of a cosl_klt_group_step op (KltCam::stages)
static int op_stages(int op) {
  return op == COSL_KLT_OP_FIRST   ? KLT_STAGE_PYR | KLT_STAGE_DETECT
         : op == COSL_KLT_OP_TRACK ? KLT_STAGE_PYR | KLT_STAGE_TRACK
         : op == COSL_KLT_OP_NEXT  ? KLT_STAGE_ALL
                                   : 0;
}

// The plan of a step whose cameras do not all have the same op, and its op table: the group's table
// with each camera's stages, written to h_stepCams[tab].  The kernels are the MIXED instantiations on
// that table, so each launch covers the group and a camera's blocks exit in the stages its op does
// not have:
//   pyramid (front pass, tail)       FIRST, TRACK, NEXT
//   tracker, status                  TRACK, NEXT
//   cornerness, non-max, selection   FIRST, NEXT      (klt_select_refill: mode per camera)
//   provide (klt_provide_cams)       TRACK
// The folds are those of the union of the ops: the front pass stores level 0 when one of its cameras
// needs it (each camera's record is what its single tracker records), the prefilter runs early, and
// a step with a detecting camera moves on to the next counter set.
//
// Advance of a strict subset: the pyramid slices of either the skipped or the addressed cameras
// are exchanged, whichever are fewer.  Skipped ones: p0 and p1 change roles for the group and their
// slices are exchanged ahead of the front pass (nothing of the step touches them); addressed ones:
// the roles stay and their slices are exchanged after the tracker.  Such a step builds into p1, as
// the two-buffer tracker does, not into the third buffer: then the skipped cameras would need their
// slices of all three buffers rotated, where one exchange of two buffers moves the same bytes.  So
// it waits for the tracker before it, and the next step for its own.  The feature-buffer half of the
// advance is folded into klt_select_refill and klt_provide_cams.
static FramePlan plan_step(cosl_klt* g, const uint8_t* ops, int tab) {
  FramePlan p;
  p.cams = g->d_stepCams[tab];
  p.mixed = true;
  p.tracked = p.wantCorn = p.storeL0 = false;
  KltCamList addr, skip;
  addr.n = skip.n = 0;
  KltCam* hstep = g->h_stepCams[tab];
  for (int c = 0; c < g->C; ++c) {
    const int st = op_stages(ops[c]);
    hstep[c] = g->hcam[c];
    hstep[c].stages = st;
    if (!st) {
      skip.cam[skip.n++] = c;
      continue;
    }
    addr.cam[addr.n++] = c;
    if (ops[c] == COSL_KLT_OP_TRACK) p.provide.cam[p.provide.n++] = c;
    p.tracked = p.tracked || (st & KLT_STAGE_TRACK);
    p.wantCorn = p.wantCorn || (st & KLT_STAGE_DETECT);
    p.lv0[c] = ops[c] != COSL_KLT_OP_NEXT || tracker_reads_level0(g);
    p.storeL0 = p.storeL0 || p.lv0[c];
  }
  p.cornMode = p.wantCorn ? KLT_CORN_PER_CAM : 0;
  p.earlyPrefilter = p.wantCorn;
  p.trackerTail = fused_tracker(g);
  p.foldAdvance = true;
  p.detectMode = 2;
  p.ops = ops;
  p.tab = tab;
  p.intoP1 = true;
  p.flip = skip.n <= addr.n;
  if (p.flip)
    p.exchangeEarly = skip;
  else
    p.exchangeLate = addr;
  return p;
}

// The halves of a frame in run_frame.  The image half depends on the frame's images alone: upload,
// front pass (levels 0 / 1, cornerness map), pyramid tail and early prefilter, on the copy, front and
// aux streams.  The dependent half reads the feature tables and p0 / p1 as the calls before it left
// them: tracker, provide, detector and refill on g->stream, which first joins the image half.
enum FrameHalf { HALF_IMAGES = 1, HALF_DEPENDENT = 2, HALF_BOTH = 3 };

// One frame through its stages, asynchronous on g->stream and, joined into it before the call
// returns, the front stream (image copies, klt_front, pyramid tail) and auxStream (the early
// prefilter).  Every entry point that processes a frame, the per-camera steps included, enqueues it
// here; what differs between frames is decided before, in the plan (plan_frame, plan_step).  imgs,
// pitch, copyKind: the frame's images (upload_images).  Nothing of the plan outlives the call, unless
// the halves run in two calls (cosl_klt_group_prefetch): then the image half leaves g->par and g->nxt
// on the set and the buffer it wrote, the caller keeps them with the plan (KltPrefetch) and puts them
// back before the dependent half.  Run back to back, the halves enqueue exactly the undivided frame.
//
// Frame n+1's image copies wait only for frame n's front pass.  Its front pass and pyramid tail wait
// only for the fences of the buffers they write, each recorded on g->stream behind that buffer's
// last reader or writer there.  Between frames that advance, that is frame n-1's tracker, so the
// steady state of back-to-back frames is
//   tracker(n-1) | front(n+1) next to detector(n-1) | tracker(n) next to tail(n+1) | front(n+2) ...
// What the front stream writes, its ring and its fence:
//   d_img                    one; read by the front passes only (same stream; copy stream: evFront)
//   d_pyr[nxt]               three (p0, p1, nxt; a step's nxt is p1); evPyr[b], recorded after each
//                            tracker for the two buffers it reads and after each exchange of slices
//   d_corn, d_prelim,        three sets; the tracker's marks, klt_suppress, verify, select and the
//   d_counters[.][8c + 4]    read-backs use set `par`.  A frame with a cornerness map moves on to the
//                            next set and records the fence evPar of the set it leaves (next_par)
//   d_stepCams[tab]          three, a step's op table: copied from h_stepCams[tab] after the waits
//                            (evStepTab[tab] follows the copy); evStepFence[tab], recorded at the end
//                            of the step
// and it reads d_cams, which update_cameras rewrites on g->stream (evCams).  A step exchanges pyramid
// slices of p0 and p1 (klt_advance_cams, which fences both) on g->stream: exchangeEarly is enqueued
// after the front stream's waits, which must not wait for it (the front pass writes the other
// cameras' slices only); exchangeLate takes the place of the tracker's fences, or follows the
// detector when nothing is tracked.
int run_frame(cosl_klt* g, const FramePlan& p, const uint8_t* const* imgs, size_t pitch, cudaMemcpyKind copyKind,
              int halves = HALF_BOTH) {
  if (halves & HALF_IMAGES) {
    if (p.wantCorn) COSL_TRY(next_par(g));
    int* counters = g->d_counters[g->par];
    // counters [0..3] of every camera, zeroed first on every kind; [4] on the front stream below.  A
    // prefetched frame zeroes them at consume: a frame without a cornerness map keeps the last
    // frame's set, whose counts group_fetch still returns until then
    if (halves & HALF_DEPENDENT)
      COSL_CUDA(cudaMemset2DAsync(counters, 8 * sizeof(int), 0, 4 * sizeof(int), g->C, g->stream));
    // the images ahead of the fences: d_img is read by the front passes alone, so they run under the
    // previous frame's tracker
    COSL_TRY(upload_images(g, imgs, pitch, copyKind, p.ops));
    if (p.intoP1) g->nxt = g->p1;
    COSL_TRY(front_waits(g, p.wantCorn, p.tab));
    COSL_TRY(exchange_slices(g, p.exchangeEarly, 0));
    if (p.tab >= 0) {
      COSL_CUDA(cudaMemcpyAsync(g->d_stepCams[p.tab], g->h_stepCams[p.tab], sizeof(KltCam) * g->C,
                                cudaMemcpyHostToDevice, g->frontStream));
      COSL_CUDA(cudaEventRecord(g->evStepTab[p.tab], g->frontStream));
    }
    if (p.wantCorn)
      COSL_CUDA(cudaMemset2DAsync(counters + 4, 8 * sizeof(int), 0, sizeof(int), g->C, g->frontStream));
    COSL_TRY(build_pyramid(g, p));
    COSL_CUDA(cudaEventRecord(g->evTail, g->frontStream));
  }
  if (!(halves & HALF_DEPENDENT)) return COSL_OK;
  g->stepOpsValid = false;
  int* counters = g->d_counters[g->par];
  if (!(halves & HALF_IMAGES))
    COSL_CUDA(cudaMemset2DAsync(counters, 8 * sizeof(int), 0, 4 * sizeof(int), g->C, g->stream));
  for (int c = 0; c < g->C; ++c)
    if (!p.ops || p.ops[c] != COSL_KLT_OP_SKIP) g->lv0Stored[g->nxt][c] = p.lv0[c];
  g->p1 = g->nxt;
  COSL_CUDA(cudaStreamWaitEvent(g->stream, g->evTail, 0));
  g->covFrame = g->covNoise >= 0.f;
  if (p.tracked) {
    COSL_TRY(run_tracker(g, p));
    if (g->covFrame) COSL_TRY(run_covariance(g, p));
    if (p.exchangeLate.n) {
      COSL_TRY(exchange_slices(g, p.exchangeLate, 0));
    } else {
      COSL_TRY(fence_pyr(g, g->p0));
      COSL_TRY(fence_pyr(g, g->p1));
    }
    if (!p.trackerTail) {
      // on a step's table the cameras outside the tracker stage exit
      const auto status = p.tab < 0 ? klt_status<false> : klt_status<true>;
      dim3 grid(div_up(g->F, 256), g->C);
      COSL_LAUNCH(status, grid, 256, 0, g->stream, g->d_res, g->d_feat, counters, g->F, p.cams);
    }
  } else if (g->covFrame) {
    COSL_TRY(run_covariance(g, p));
  }
  // provide: the tracked set becomes the feature table of the next frame
  if (p.provideAll) {
    const size_t n = (size_t)g->F * g->C;
    COSL_LAUNCH(klt_copy_f4, (unsigned)div_up64(n, 256), 256, 0, g->stream, g->d_res, g->d_dst, n);
  }
  if (p.provide.n)
    COSL_LAUNCH(klt_provide_cams, dim3(div_up(g->F, 256), p.provide.n), 256, 0, g->stream, g->d_res, g->d_dst,
                g->d_src, g->F, p.provide);
  if (p.wantCorn) COSL_TRY(run_detector(g, p));
  if (!p.tracked) COSL_TRY(exchange_slices(g, p.exchangeLate, 0));
  if (p.tab >= 0) COSL_CUDA(cudaEventRecord(g->evStepFence[p.tab], g->stream));
  if (p.intoP1) {
    if (p.flip) std::swap(g->p0, g->p1);
    g->nxt = g->p1;
  } else if (p.foldAdvance) {
    advance_pyramids(g);
  }
  return COSL_OK;
}

// The frame of a step (cosl_klt_group_step): camera c gets ops[c] followed by advanceFrame, or
// nothing.  Every camera with the same op: the frame of that kind, exactly as group_first /
// group_next / track + advance run it (*advanceAfter: the advance after track).  Otherwise
// plan_step's plan, on the next op table.  *any = false: every camera skips, and nothing runs.
static int plan_ops(cosl_klt* g, const uint8_t* ops, FramePlan* p, bool* advanceAfter, bool* any) {
  const int C = g->C;
  int nOp[4] = {0, 0, 0, 0};
  for (int c = 0; c < C; ++c) ++nOp[ops[c]];
  *advanceAfter = false;
  *any = nOp[COSL_KLT_OP_SKIP] < C;
  if (nOp[COSL_KLT_OP_NEXT] == C) {
    *p = plan_frame(g, FRAME_REDETECT, 0, true);
  } else if (nOp[COSL_KLT_OP_FIRST] == C) {
    *p = plan_frame(g, FRAME_DETECT, 0, true);
  } else if (nOp[COSL_KLT_OP_TRACK] == C) {
    *p = plan_frame(g, FRAME_TRACK, 0, false);
    *advanceAfter = true;
  } else if (*any) {
    // the pinned table's previous copy was enqueued three steps ago: the host waits here only when
    // it runs more than two steps ahead of the front stream (cosl_klt_group_step_dev)
    const int tab = g->stepTab = (g->stepTab + 1) % 3;
    COSL_CUDA(cudaEventSynchronize(g->evStepTab[tab]));
    *p = plan_step(g, ops, tab);
  }
  return COSL_OK;
}

// One step of cosl_klt_group_step
int run_step(cosl_klt* g, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch, cudaMemcpyKind copyKind) {
  FramePlan p;
  bool advanceAfter = false, any = false;
  COSL_TRY(plan_ops(g, ops, &p, &advanceAfter, &any));
  if (any) COSL_TRY(run_frame(g, p, imgs, pitch, copyKind));
  if (advanceAfter) COSL_TRY(advance(g));
  std::memcpy(g->stepOps, ops, g->C);
  g->stepOpsValid = true;
  return COSL_OK;
}

// The dependent half of the prefetched frame (cosl_klt_group_prefetch), on the feature tables and
// p0 / p1 the feeds and advances since have left, then what run_step or group_next does after it.
static int consume_prefetch(cosl_klt* g) {
  KltPrefetch& f = g->pf;
  f.pending = false;
  g->par = f.par;
  g->nxt = f.buf;
  COSL_TRY(run_frame(g, f.plan, nullptr, 0, cudaMemcpyHostToDevice, HALF_DEPENDENT));
  if (f.advanceAfter) COSL_TRY(advance(g));
  if (f.step) {
    std::memcpy(g->stepOps, f.ops, g->C);
    g->stepOpsValid = true;
  }
  return COSL_OK;
}

// Waits on the host for everything a dropped prefetch enqueued: its upload, which still reads the
// caller's image buffers, and its prefilter on auxStream, which may still write the counter set the
// next frame moves to.  A discard is rare (a camera restarts), so it need not return early.
static int drop_prefetch(cosl_klt* g) {
  g->pf.pending = false;
  for (cudaStream_t st : {g->copyStream, g->frontStream, g->auxStream}) COSL_CUDA(cudaStreamSynchronize(st));
  return COSL_OK;
}

// Camera c's table of `feat` -> dest[c] and its count counters[8c + 2] -> n[c], each where given.
// ops: the step the tables come from (nullptr: a frame of one kind for every camera): the addressed
// cameras only, a tracked-only camera's count being its live tracks (counters[8c + 0], what track()
// returns).  cov: the frame's covariances (nullptr: it was not armed), which the addressed cameras'
// entries of covOut take, as dest[c] takes the table.
void copy_out(cosl_klt* g, const cosl_klt_feature* feat, const int* counters, const float* cov,
              const uint8_t* ops, cosl_klt_feature* const* dest, int* n) {
  bool any = false;
  for (int c = 0; c < g->C; ++c) {
    const int op = ops ? ops[c] : COSL_KLT_OP_NEXT;
    if (op == COSL_KLT_OP_SKIP) continue;
    any = true;
    if (dest && dest[c]) std::memcpy(dest[c], feat + (size_t)c * g->F, sizeof(cosl_klt_feature) * g->F);
    if (n) n[c] = counters[8 * c + (op == COSL_KLT_OP_TRACK ? 0 : 2)];
    if (cov) {
      const size_t o = (size_t)3 * c * g->F;
      std::memcpy(g->covOut.data() + o, cov + o, sizeof(float) * 3 * g->F);
    }
  }
  if (any) g->covHanded = cov != nullptr;
}

// the synchronous calls' covariances (fetch_results): those of the last frame run, if it was armed
const float* sync_cov(const cosl_klt* g) { return g->covFrame ? g->h_cov : nullptr; }

}  // namespace

/* ================================================================ C-ABI */
extern "C" {

void cosl_klt_config_default(cosl_klt_config* c) {
  if (!c) return;
  c->nIterations = 12;
  c->nLevels = 3;
  c->levelSkip = 2;
  c->windowWidth = 5;
  c->trackBorderMargin = 4.0f;
  c->convergenceThreshold = 0.1f;
  c->SSD_Threshold = 5000.0f;
  c->trackWithGain = 0;
  c->minDistance = 8;
  c->minCornerness = 1000.0f;
  c->detectBorderMargin = 4.0f;
  c->compat = COSL_KLT_COMPAT_ITER5;
}

int cosl_klt_group_create_sizes(const cosl_klt_config* cfg, int nCams, const int* widths,
                                const int* heights, int nLevels, int featW, int featH, int plW, int plH,
                                int device, cosl_klt** out) {
  if (!cfg || !out || !widths || !heights) return set_error(COSL_E_INVALID, "null argument");
  *out = nullptr;
  if (nCams < 1 || nCams > 64 || nLevels < 1 || nLevels > 8 || featW < 1 || featH < 1)
    return set_error(COSL_E_INVALID, "bad tracker geometry L=%d feat=%dx%d C=%d", nLevels, featW, featH, nCams);
  int maxW = 0, maxH = 0;
  for (int c = 0; c < nCams; ++c) {
    const int width = widths[c], height = heights[c];
    if (width < 16 || height < 16 || width > 65535 || height > 65535 || (width >> (nLevels - 1)) < 2 ||
        (height >> (nLevels - 1)) < 2)
      return set_error(COSL_E_INVALID, "bad tracker geometry of camera %d: %dx%d L=%d", c, width, height,
                       nLevels);
    maxW = std::max(maxW, width);
    maxH = std::max(maxH, height);
  }
  if (cfg->windowWidth < 1 || cfg->windowWidth > 31 || cfg->minDistance < 1 ||
      cfg->minDistance > 32 || cfg->nIterations < 1)
    return set_error(COSL_E_INVALID, "bad tracker config");
  COSL_TRY(check_device(device));
  COSL_CUDA(cudaSetDevice(device));
  cosl_klt* g = new (std::nothrow) cosl_klt();
  if (!g) return set_error(COSL_E_NOMEM, "host allocation failed");
  g->cfg = *cfg;
  g->cfg.nLevels = nLevels;
  g->C = nCams;
  g->W = maxW;
  g->H = maxH;
  for (int c = 0; c < nCams; ++c) {
    g->hcam[c].W = widths[c];
    g->hcam[c].H = heights[c];
    g->mixed = g->mixed || widths[c] != widths[0] || heights[c] != heights[0];
  }
  g->L = nLevels;
  g->fw = featW;
  g->fh = featH;
  g->F = featW * featH;
  if (plW <= 0) plW = 2 * featW;
  if (plH <= 0) plH = 2 * featH;
  g->plCap = plW * plH;
  g->device = device;
  g->pitchZeroOK = true;
  g->levelSkip = cfg->levelSkip > 0 ? cfg->levelSkip : (nLevels - 1);
  if (g->levelSkip < 1) g->levelSkip = 1;
  g->halfWidth = cfg->windowWidth / 2;
  g->trackMargin = cfg->trackBorderMargin;
  g->conv = cfg->convergenceThreshold;
  g->ssd = cfg->SSD_Threshold;
  g->detectMargin = 10.0f;  // KLT_Detector::_margin default (v3d_gpuklt.h:113-114)
  int rc = alloc_group(g);
  if (rc != COSL_OK) {
    free_group(g);
    return rc;
  }
  *out = g;
  return COSL_OK;
}

int cosl_klt_group_create(const cosl_klt_config* cfg, int nCams, int width, int height,
                          int nLevels, int featW, int featH, int plW, int plH, int device,
                          cosl_klt** out) {
  if (!out) return set_error(COSL_E_INVALID, "null argument");
  *out = nullptr;
  if (nCams < 1 || nCams > 64)
    return set_error(COSL_E_INVALID, "bad tracker geometry %dx%d L=%d feat=%dx%d C=%d", width, height, nLevels,
                     featW, featH, nCams);
  int widths[64], heights[64];
  std::fill(widths, widths + nCams, width);
  std::fill(heights, heights + nCams, height);
  COSL_TRY(cosl_klt_group_create_sizes(cfg, nCams, widths, heights, nLevels, featW, featH, plW, plH, device, out));
  (*out)->pitchZeroOK = false;  // the images of an equal-size group are always given a pitch
  return COSL_OK;
}

int cosl_klt_create(const cosl_klt_config* cfg, int width, int height, int nLevels, int featW,
                    int featH, int plW, int plH, int device, cosl_klt** out) {
  return cosl_klt_group_create(cfg, 1, width, height, nLevels, featW, featH, plW, plH, device, out);
}

int cosl_klt_destroy(cosl_klt* h) {
  free_group(h);
  return COSL_OK;
}

#define KLT_ENTER(h)                                              \
  if (!(h)) return set_error(COSL_E_INVALID, "null tracker handle"); \
  COSL_CUDA(cudaSetDevice((h)->device));

// Row pitch of the images a call takes: at least the widest camera's width, or 0 on a group made with
// cosl_klt_group_create_sizes (camera c's rows are its own width apart)
static bool pitch_ok(const cosl_klt* g, size_t pitch) { return pitch ? pitch >= (size_t)g->W : g->pitchZeroOK; }

// the calls that process a frame of their own, and set_margin (the margin enters the cornerness map
// the prefetched front pass already made), wait until a prefetched frame is consumed or discarded
#define KLT_NOT_PREFETCHED(h, name) \
  if ((h)->pf.pending) return set_error(COSL_E_STATE, name ": a prefetched frame is pending");

#define KLT_SINGLE(h) \
  KLT_ENTER(h)        \
  if ((h)->C != 1) return set_error(COSL_E_STATE, "single-camera call on a %d-camera group", (h)->C);

int cosl_klt_detect(cosl_klt* h, const uint8_t* img, size_t pitch, int nPresent,
                    const float* present3, cosl_klt_feature* dest, int* nDetected) {
  KLT_SINGLE(h)
  KLT_NOT_PREFETCHED(h, "cosl_klt_detect")
  if (!img || !dest || !nDetected || nPresent < 0 || nPresent > h->F || (nPresent && !present3) ||
      !pitch_ok(h, pitch))
    return set_error(COSL_E_INVALID, "cosl_klt_detect: bad argument");
  int maxPresent = 0;
  COSL_TRY(upload_present(h, &nPresent, &present3, &maxPresent));
  const uint8_t* imgs[1] = {img};
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_DETECT, maxPresent, false), imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), nullptr, &dest, nDetected);
  return COSL_OK;
}

int cosl_klt_redetect(cosl_klt* h, const uint8_t* img, size_t pitch, cosl_klt_feature* dest,
                      int* nNewFeatures) {
  KLT_SINGLE(h)
  KLT_NOT_PREFETCHED(h, "cosl_klt_redetect")
  if (!img || !dest || !nNewFeatures || !pitch_ok(h, pitch))
    return set_error(COSL_E_INVALID, "cosl_klt_redetect: bad argument");
  const uint8_t* imgs[1] = {img};
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_REDETECT, 0, false), imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), nullptr, &dest, nNewFeatures);
  return COSL_OK;
}

int cosl_klt_track(cosl_klt* h, const uint8_t* img, size_t pitch, cosl_klt_feature* dest,
                   int* nPresent) {
  KLT_SINGLE(h)
  KLT_NOT_PREFETCHED(h, "cosl_klt_track")
  if (!img || !dest || !nPresent || !pitch_ok(h, pitch))
    return set_error(COSL_E_INVALID, "cosl_klt_track: bad argument");
  const uint8_t* imgs[1] = {img};
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_TRACK, 0, false), imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), nullptr, &dest, nullptr);
  *nPresent = h->h_counters[0];
  return COSL_OK;
}

int cosl_klt_feed(cosl_klt* h, int npts, const float* pts3, int* trackIds, int* nFed) {
  KLT_SINGLE(h)
  if (npts < 0 || (npts && (!pts3 || !trackIds)) || !nFed)
    return set_error(COSL_E_INVALID, "cosl_klt_feed: bad argument");
  return feed_cams(h, &npts, &pts3, &trackIds, nFed);
}

int cosl_klt_advance(cosl_klt* h) {
  KLT_ENTER(h)
  COSL_TRY(advance(h));
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

int cosl_klt_set_margin(cosl_klt* h, float m) {  // tracker AND detector (v3d_gpuklt.h:217-224)
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "cosl_klt_set_margin")
  h->trackMargin = m;
  h->detectMargin = m;
  return update_cameras(h);
}
int cosl_klt_set_conv(cosl_klt* h, float t) {
  KLT_ENTER(h)
  h->conv = t;
  return COSL_OK;
}
int cosl_klt_set_ssd(cosl_klt* h, float t) {
  KLT_ENTER(h)
  h->ssd = t;
  return COSL_OK;
}

// The buffers are made on the first arming and kept when the group is disarmed.
int cosl_klt_set_covariance(cosl_klt* h, float noise_var) {
  KLT_ENTER(h)
  if (!std::isfinite(noise_var)) return set_error(COSL_E_INVALID, "set_covariance: noise_var is not finite");
  if (noise_var >= 0.f && !h->d_cov) {
    const size_t n = (size_t)3 * h->F * h->C;
    COSL_CUDA(cudaMalloc(&h->d_cov, sizeof(float) * n));
    COSL_CUDA(cudaMallocHost(&h->h_cov, sizeof(float) * n));
    for (int i = 0; i < 2; ++i) COSL_CUDA(cudaMallocHost(&h->h_covQ[i], sizeof(float) * n));
    h->covOut.assign(n, std::nanf(""));
  }
  h->covNoise = noise_var >= 0.f ? noise_var : -1.f;
  return COSL_OK;
}

int cosl_klt_group_download_covariance(cosl_klt* h, float* const* cov) {
  KLT_ENTER(h)
  if (!cov) return set_error(COSL_E_INVALID, "group_download_covariance: null argument");
  if (!h->covHanded)
    return set_error(COSL_E_STATE, "group_download_covariance: the last frame handed out was not armed "
                                   "(cosl_klt_set_covariance)");
  for (int c = 0; c < h->C; ++c)
    if (cov[c])
      std::memcpy(cov[c], h->covOut.data() + (size_t)3 * c * h->F, sizeof(float) * 3 * h->F);
  return COSL_OK;
}

#define KLT_NOT_IN_FLIGHT(h, name) \
  if ((h)->nInFlight > 0) return set_error(COSL_E_STATE, name ": submitted frames not yet collected");

// batched GPUKLT::first(f, img[, present, ips]) (tracking/GPUKLT.cpp:111-135): detect + advanceFrame;
// nPresent == nullptr: no present lists
static int group_first(cosl_klt* h, const uint8_t* const* imgs, size_t pitch, const int* nPresent,
                       const float* const* present3, cosl_klt_feature* const* dest, int* nDetected) {
  int maxPresent = 0;
  if (nPresent) COSL_TRY(upload_present(h, nPresent, present3, &maxPresent));
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_DETECT, maxPresent, true), imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), nullptr, dest, nDetected);
  return COSL_OK;
}

int cosl_klt_group_first(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                         cosl_klt_feature* const* dest, int* nDetected) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_first")
  if (!imgs || !pitch_ok(h, pitch)) return set_error(COSL_E_INVALID, "group_first: bad argument");
  return group_first(h, imgs, pitch, nullptr, nullptr, dest, nDetected);
}

int cosl_klt_group_first_present(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                                 const int* nPresent, const float* const* present3,
                                 cosl_klt_feature* const* dest, int* nDetected) {
  KLT_ENTER(h)
  KLT_NOT_IN_FLIGHT(h, "group_first_present")
  KLT_NOT_PREFETCHED(h, "group_first_present")
  if (!imgs || !pitch_ok(h, pitch) || !nPresent)
    return set_error(COSL_E_INVALID, "group_first_present: bad argument");
  for (int c = 0; c < h->C; ++c)
    if (nPresent[c] < 0 || nPresent[c] > h->F || (nPresent[c] > 0 && (!present3 || !present3[c])))
      return set_error(COSL_E_INVALID, "group_first_present: bad present list of camera %d", c);
  return group_first(h, imgs, pitch, nPresent, present3, dest, nDetected);
}

int cosl_klt_group_feed(cosl_klt* h, const int* npts, const float* const* pts3, int* const* trackIds,
                        int* nFed) {
  KLT_ENTER(h)
  KLT_NOT_IN_FLIGHT(h, "group_feed")
  if (!npts || !nFed) return set_error(COSL_E_INVALID, "group_feed: bad argument");
  for (int c = 0; c < h->C; ++c)
    if (npts[c] > 0 && (!pts3 || !pts3[c] || !trackIds || !trackIds[c]))
      return set_error(COSL_E_INVALID, "group_feed: null point or id list for camera %d", c);
  return feed_cams(h, npts, pts3, trackIds, nFed);
}

int cosl_klt_group_advance_cams(cosl_klt* h, const uint8_t* cams) {
  KLT_ENTER(h)
  KLT_NOT_IN_FLIGHT(h, "group_advance_cams")
  if (!cams) return set_error(COSL_E_INVALID, "group_advance_cams: null camera mask");
  COSL_TRY(advance_cams(h, cams));
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

int cosl_klt_group_next(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                        cosl_klt_feature* const* dest, int* nNew) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_next")
  if (!imgs || !pitch_ok(h, pitch)) return set_error(COSL_E_INVALID, "group_next: bad argument");
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_REDETECT, 0, true), imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), nullptr, dest, nNew);
  return COSL_OK;
}

int cosl_klt_group_next_dev(cosl_klt* h, const uint8_t* const* dimgs, size_t pitch) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_next_dev")
  if (!dimgs || !pitch_ok(h, pitch))
    return set_error(COSL_E_INVALID, "group_next_dev: bad argument");
  return run_frame(h, plan_frame(h, FRAME_REDETECT, 0, true), dimgs, pitch, cudaMemcpyDeviceToDevice);
}

// ops[c] in COSL_KLT_OP_*, an image for every addressed camera
static int check_step(const cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch,
                      const char* name) {
  if (!ops || !imgs || !pitch_ok(h, pitch)) return set_error(COSL_E_INVALID, "%s: bad argument", name);
  for (int c = 0; c < h->C; ++c) {
    if (ops[c] > COSL_KLT_OP_NEXT) return set_error(COSL_E_INVALID, "%s: bad op %d of camera %d", name, ops[c], c);
    if (ops[c] != COSL_KLT_OP_SKIP && !imgs[c])
      return set_error(COSL_E_INVALID, "%s: no image for camera %d", name, c);
  }
  return COSL_OK;
}

int cosl_klt_group_step(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch,
                        cosl_klt_feature* const* dest, int* n) {
  KLT_ENTER(h)
  KLT_NOT_IN_FLIGHT(h, "group_step")
  KLT_NOT_PREFETCHED(h, "group_step")
  COSL_TRY(check_step(h, ops, imgs, pitch, "group_step"));
  COSL_TRY(run_step(h, ops, imgs, pitch, cudaMemcpyHostToDevice));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), ops, dest, n);
  return COSL_OK;
}

int cosl_klt_group_step_dev(cosl_klt* h, const uint8_t* ops, const uint8_t* const* dimgs, size_t pitch) {
  KLT_ENTER(h)
  KLT_NOT_IN_FLIGHT(h, "group_step_dev")
  KLT_NOT_PREFETCHED(h, "group_step_dev")
  COSL_TRY(check_step(h, ops, dimgs, pitch, "group_step_dev"));
  return run_step(h, ops, dimgs, pitch, cudaMemcpyDeviceToDevice);
}

int cosl_klt_group_fetch(cosl_klt* h, cosl_klt_feature* const* dest, int* nNew) {
  KLT_ENTER(h)
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), h->stepOpsValid ? h->stepOps : nullptr, dest, nNew);
  return COSL_OK;
}

// Frame-pipelined ingest (SURVEY.md 8f-4, the upload half): submit() enqueues the H2D copy of frame
// n + 1, its kernels and the D2H copy of its feature table and returns; collect() waits for the OLDEST
// submitted frame.  With submit(n+1) called before collect(n), the image upload of frame n + 1 runs on
// the copy stream under the tracker / detector kernels of frame n (it only waits for frame n's front
// pass, which is the last reader of the image buffer), and its pyramid under frame n's detector
// (run_frame).  submit_step() does the same for a step (run_step); both share the two slots and the
// FIFO, and the slot keeps the frame's ops for collect().
//
// The result slot of the next submitted frame, allocated on first use.
static int submit_slot(cosl_klt* h, const char* name, int* slot) {
  if (h->nInFlight >= 2) return set_error(COSL_E_STATE, "%s: two frames in flight, collect one first", name);
  const int s = (int)(h->subSeq & 1u);
  if (!h->h_featQ[s]) {
    COSL_CUDA(cudaMallocHost(&h->h_featQ[s], sizeof(cosl_klt_feature) * (size_t)h->F * h->C));
    COSL_CUDA(cudaMallocHost(&h->h_cntQ[s], sizeof(int) * 8 * h->C));
    COSL_CUDA(cudaEventCreateWithFlags(&h->evDone[s], cudaEventDisableTiming));
  }
  *slot = s;
  return COSL_OK;
}

// The read-back of the frame just enqueued into `slot` (whose opsQ is set) and its place in the
// FIFO.  An all-SKIP step has nothing to read back: its event alone keeps the order.
static int submit_readback(cosl_klt* h, int slot) {
  bool any = false;
  for (int c = 0; c < h->C; ++c) any = any || h->opsQ[slot][c] != COSL_KLT_OP_SKIP;
  if (any) {
    COSL_CUDA(cudaMemcpyAsync(h->h_featQ[slot], h->d_feat, sizeof(cosl_klt_feature) * (size_t)h->F * h->C,
                              cudaMemcpyDeviceToHost, h->stream));
    COSL_CUDA(cudaMemcpyAsync(h->h_cntQ[slot], h->d_counters[h->par], sizeof(int) * 8 * h->C,
                              cudaMemcpyDeviceToHost, h->stream));
  }
  h->covQ[slot] = any && h->covFrame;
  if (h->covQ[slot])
    COSL_CUDA(cudaMemcpyAsync(h->h_covQ[slot], h->d_cov, sizeof(float) * 3 * h->F * h->C, cudaMemcpyDeviceToHost,
                              h->stream));
  COSL_CUDA(cudaEventRecord(h->evDone[slot], h->stream));
  ++h->subSeq;
  ++h->nInFlight;
  return COSL_OK;
}

int cosl_klt_group_submit(cosl_klt* h, const uint8_t* const* imgs, size_t pitch) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_submit")
  if (!imgs || !pitch_ok(h, pitch)) return set_error(COSL_E_INVALID, "group_submit: bad argument");
  int slot = 0;
  COSL_TRY(submit_slot(h, "group_submit", &slot));
  COSL_TRY(run_frame(h, plan_frame(h, FRAME_REDETECT, 0, true), imgs, pitch, cudaMemcpyHostToDevice));
  std::memset(h->opsQ[slot], COSL_KLT_OP_NEXT, h->C);
  return submit_readback(h, slot);
}

// A step's op table comes from one of three pinned host tables (run_step); the host waits for the
// copy out of the table it reuses, made three mixed steps earlier.  At most two frames are in flight,
// so when that step was submitted it has been collected (the copy is done); only a step_dev can leave
// it pending, and its copy is already enqueued.
int cosl_klt_group_submit_step(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_submit_step")
  COSL_TRY(check_step(h, ops, imgs, pitch, "group_submit_step"));
  int slot = 0;
  COSL_TRY(submit_slot(h, "group_submit_step", &slot));
  COSL_TRY(run_step(h, ops, imgs, pitch, cudaMemcpyHostToDevice));
  std::memcpy(h->opsQ[slot], ops, h->C);
  return submit_readback(h, slot);
}

int cosl_klt_group_collect(cosl_klt* h, cosl_klt_feature* const* dest, int* nNew) {
  KLT_ENTER(h)
  if (h->nInFlight <= 0) return set_error(COSL_E_STATE, "group_collect: nothing submitted");
  const int slot = (int)((h->subSeq - (unsigned)h->nInFlight) & 1u);
  COSL_CUDA(cudaEventSynchronize(h->evDone[slot]));
  --h->nInFlight;
  copy_out(h, h->h_featQ[slot], h->h_cntQ[slot], h->covQ[slot] ? h->h_covQ[slot] : nullptr, h->opsQ[slot], dest,
           nNew);
  return COSL_OK;
}

// The image half of a frame now, its dependent half later (cosl_klt_group_run_prefetched /
// _submit_prefetched), with feeds and advances in between.  The front pass writes the third buffer,
// the one neither p0 nor p1 holds, which no feed or advance touches; an advance only exchanges p0 and
// p1 (or slices of them).  A step whose ops differ would build into p1 (plan_step); without skipped
// cameras nothing of p1 needs keeping, so it builds into the third buffer like a frame of one kind.
int cosl_klt_group_prefetch(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch) {
  KLT_ENTER(h)
  KLT_NOT_PREFETCHED(h, "group_prefetch")
  if (!imgs || !pitch_ok(h, pitch)) return set_error(COSL_E_INVALID, "group_prefetch: bad argument");
  for (int c = 0; c < h->C; ++c) {
    if (ops && (ops[c] == COSL_KLT_OP_SKIP || ops[c] > COSL_KLT_OP_NEXT))
      return set_error(COSL_E_INVALID, "group_prefetch: op %d of camera %d (SKIP cannot be prefetched)", ops[c], c);
    if (!imgs[c]) return set_error(COSL_E_INVALID, "group_prefetch: no image for camera %d", c);
  }
  KltPrefetch& f = h->pf;
  f.step = ops != nullptr;
  if (ops)
    std::memcpy(f.ops, ops, h->C);
  else
    std::memset(f.ops, COSL_KLT_OP_NEXT, h->C);
  bool any = true;
  COSL_TRY(plan_ops(h, f.ops, &f.plan, &f.advanceAfter, &any));
  f.plan.intoP1 = f.plan.flip = false;
  const int par = h->par, nxt = h->nxt;
  h->nxt = 3 - h->p0 - h->p1;
  const int rc = run_frame(h, f.plan, imgs, pitch, cudaMemcpyHostToDevice, HALF_IMAGES);
  f.par = h->par;
  f.buf = h->nxt;
  h->par = par;
  h->nxt = nxt;
  if (rc != COSL_OK) {
    drop_prefetch(h);
    return rc;
  }
  f.pending = true;
  return COSL_OK;
}

int cosl_klt_group_run_prefetched(cosl_klt* h, cosl_klt_feature* const* dest, int* n) {
  KLT_ENTER(h)
  if (!h->pf.pending) return set_error(COSL_E_STATE, "group_run_prefetched: nothing prefetched");
  if (h->pf.step) KLT_NOT_IN_FLIGHT(h, "group_run_prefetched")
  COSL_TRY(consume_prefetch(h));
  COSL_TRY(fetch_results(h));
  copy_out(h, h->h_feat, h->h_counters, sync_cov(h), h->pf.step ? h->pf.ops : nullptr, dest, n);
  return COSL_OK;
}

int cosl_klt_group_submit_prefetched(cosl_klt* h) {
  KLT_ENTER(h)
  if (!h->pf.pending) return set_error(COSL_E_STATE, "group_submit_prefetched: nothing prefetched");
  int slot = 0;
  COSL_TRY(submit_slot(h, "group_submit_prefetched", &slot));
  COSL_TRY(consume_prefetch(h));
  std::memcpy(h->opsQ[slot], h->pf.ops, h->C);
  return submit_readback(h, slot);
}

int cosl_klt_group_discard_prefetch(cosl_klt* h) {
  KLT_ENTER(h)
  if (!h->pf.pending) return set_error(COSL_E_STATE, "group_discard_prefetch: nothing prefetched");
  return drop_prefetch(h);
}

int cosl_klt_group_sync(cosl_klt* h) {
  KLT_ENTER(h)
  COSL_CUDA(cudaStreamSynchronize(h->stream));
  if (h->pf.pending) {
    COSL_CUDA(cudaStreamSynchronize(h->frontStream));
    COSL_CUDA(cudaStreamSynchronize(h->auxStream));
  }
  return COSL_OK;
}

void* cosl_klt_stream(cosl_klt* h) { return h ? (void*)h->stream : nullptr; }

int cosl_klt_debug_pyramid(cosl_klt* h, int cam, int which, int level, float* out3, int* w,
                           int* ht) {
  KLT_ENTER(h)
  if (cam < 0 || cam >= h->C || level < 0 || level >= h->L)
    return set_error(COSL_E_INVALID, "debug_pyramid: bad argument");
  const int lw = h->hcam[cam].W >> level, lh = h->hcam[cam].H >> level;
  if (w) *w = lw;
  if (ht) *ht = lh;
  if (!out3) return COSL_OK;
  const int buf = which ? h->p1 : h->p0;
  if (level == 0 && !h->lv0Stored[buf][cam])
    return set_error(COSL_E_INVALID,
                     "debug_pyramid: level 0 of this pyramid was not stored (a tracked frame keeps only "
                     "the levels its tracker visits; detect() and first() store every level)");
  std::vector<float4> tmp((size_t)lw * lh);
  const float4* src = h->d_pyr[buf] + (size_t)cam * h->pyrStride + h->lvOff[level];
  COSL_CUDA(cudaStreamSynchronize(h->stream));
  COSL_CUDA(cudaMemcpy2D(tmp.data(), sizeof(float4) * lw, src, sizeof(float4) * h->lvW[level], sizeof(float4) * lw,
                         lh, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < tmp.size(); ++i) {
    out3[3 * i] = tmp[i].x;
    out3[3 * i + 1] = tmp[i].y;
    out3[3 * i + 2] = tmp[i].z;
  }
  return COSL_OK;
}

int cosl_klt_debug_cornerness(cosl_klt* h, int cam, float* out) {
  KLT_ENTER(h)
  if (cam < 0 || cam >= h->C || !out) return set_error(COSL_E_INVALID, "debug_cornerness");
  COSL_CUDA(cudaStreamSynchronize(h->stream));
  COSL_CUDA(cudaMemcpy2D(out, sizeof(float) * h->hcam[cam].W, h->d_corn[h->par] + (size_t)cam * h->W * h->H,
                         sizeof(float) * h->W, sizeof(float) * h->hcam[cam].W, h->hcam[cam].H,
                         cudaMemcpyDeviceToHost));
  return COSL_OK;
}

int cosl_klt_debug_num_candidates(cosl_klt* h, int cam) {
  if (!h || cam < 0 || cam >= h->C) return -1;
  return h->h_counters[8 * cam + 3];
}

double cosl_klt_algorithmic_bytes(cosl_klt* h) {
  if (!h) return 0;
  // SURVEY.md 8(d): B_frame = C * (25 W H + 4640 F); the 4640 B/feature generalise to
  // n_lvl * 2 * (w+1)^2 * 12 + 32 for other window sizes / level sets
  const int nlv = tracker_levels(h, false).n;
  const double w1 = 2 * h->halfWidth + 2;
  double pyr = 1.0;
  for (int l = 0; l < h->L; ++l) pyr += 12.0 / (double)(1 << (2 * l));
  const double perFeat = nlv * 2.0 * w1 * w1 * 12.0 + 32.0;
  double px = 0.0;  // pixels of all cameras (exact)
  for (int c = 0; c < h->C; ++c) px += (double)h->hcam[c].W * h->hcam[c].H;
  return (double)h->C * ((pyr + 8.0) * (px / h->C) + perFeat * h->F);
}

int cosl_klt_profile_enable(cosl_klt* h, int on) {
  KLT_ENTER(h)
  COSL_CUDA(cudaStreamSynchronize(h->stream));
  h->timer.reset();
  h->timer.enabled = on != 0;
  return COSL_OK;
}

const char* cosl_klt_profile_get(cosl_klt* h, int idx, double* ms, int* calls) {
  if (!h || idx < 0 || idx >= h->timer.nsec) return nullptr;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  h->timer.flush();
  if (ms) *ms = h->timer.ms[idx];
  if (calls) *calls = h->timer.calls[idx];
  return h->timer.names[idx];
}

}  // extern "C"
