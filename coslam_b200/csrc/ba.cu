// ba.cu -- host side of the bundle-adjustment solver + its C-ABI (see include/coslam_b200.h).
// Replaces bundleAdjustRobust (LibVisualSLAM, call app/SL_CoSLAMRobustBA.cpp:174) and
// sba_motstr_levmar_x (sba-1.6, call app/SL_CoSLAMBA.cpp:360-363).  The LM control flow (ba_lm.cuh)
// mirrors oracle/ba_oracle.cpp:levmar line by line; every arithmetic step runs in the kernels of
// ba_kernels.cuh.  Multi-GPU: points (with all their observations) are sharded over the ranks,
// cameras are replicated; per LM trial one NCCL all-reduce (sum) of the packed buffer
// [S | rhs] and one of a handful of scalars; per linearisation one of [U | ea] and one max-reduce.
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <sched.h>
#include <thread>
#include <unordered_map>
#include <vector>

#include "ba_ctl.cuh"
#include "ba_kernels.cuh"
#include "ba_tile.cuh"
#include "common.cuh"
#include "tile_solve.h"

using namespace coslam;

/* ---------------------------------------------------------------- tile solve set-up and launch (tile_solve.h) */
namespace coslam {

TileLaunch tile_launch_plan(const BaPlan& P) {
  TileLaunch L;
  std::vector<BaTask>& order = L.order;
  // two ticket lists (each keeps the critical-path-first order, hence stays topological)
  for (const BaTask& t : P.tasks)
    if (t.type == BA_T_POTRF || t.type == BA_T_BWD) order.push_back(t);
  L.nA = (int)order.size();
  for (const BaTask& t : P.tasks)
    if (!(t.type == BA_T_POTRF || t.type == BA_T_BWD)) order.push_back(t);
  // hot successors of every POTRF(k): TRSM(j, k) and the diagonal UPD(j, j, k) of j = first block
  // of struct(k) -- the next pivot of the dependency chain (ba_tile.cuh)
  std::vector<int> firstTrsm(P.nb, -1), firstRow(P.nb, 1 << 30);
  for (int t = 0; t < (int)order.size(); ++t) {
    const BaTask& k = order[t];
    if (k.type == BA_T_TRSM && k.i < firstRow[k.k]) {
      firstRow[k.k] = k.i;
      firstTrsm[k.k] = t;
    }
  }
  std::vector<int> diagUpd(P.nb, -1);
  for (int t = 0; t < (int)order.size(); ++t) {
    const BaTask& k = order[t];
    if (k.type == BA_T_UPD && (k.flags & 1) && firstTrsm[k.k] >= 0 && k.i == firstRow[k.k]) diagUpd[k.k] = t;
  }
  for (BaTask& k : order)
    if (k.type == BA_T_POTRF) {
      k.l0 = firstTrsm[k.k];
      k.l1 = diagUpd[k.k];
    }
  // Systems of one or two blocks (local BA) are solved by one resident CTA: for the 72 x 72 system of
  // the c3 local BA, ba_tile_two needs 26 us per LM trial and the task kernel 42 us (H100 80GB HBM3, 400 W).
  if (P.nb >= 1 && P.nb <= 2) {
    L.t00 = P.tileIdx[0];
    L.t10 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 0] : -1;
    L.t11 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 1] : -1;
    L.two = L.t00 >= 0 && (P.nb == 1 || L.t11 >= 0);
  }
  return L;
}

int tile_launch_device(TileLaunch& L) {
  static std::mutex mu;
  static std::vector<int> smCount;  // per device, 0 until the attributes are set there
  int device = 0, nsm = 0;
  COSL_CUDA(cudaGetDevice(&device));
  {
    std::lock_guard<std::mutex> lk(mu);
    if ((int)smCount.size() <= device) smCount.resize(device + 1, 0);
    if (!smCount[device]) {
      COSL_CUDA(cudaFuncSetAttribute(ba_tile_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_TILE_SMEM));
      COSL_CUDA(cudaFuncSetAttribute(ba_tile_two, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_TILE_SMEM));
      COSL_CUDA(cudaFuncSetAttribute(ba_selinv_two, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_SEL2_SMEM));
      COSL_CUDA(cudaFuncSetAttribute(ba_selinv_xinv, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_SELX_SMEM));
      COSL_CUDA(cudaFuncSetAttribute(ba_selinv_step, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_SELS_SMEM));
      int perSm = 0;
      COSL_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
      COSL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, ba_tile_solve, BA_NTHREADS, BA_TILE_SMEM));
      if (perSm < 1) return set_error(COSL_E_CUDA, "tile solve: the kernel does not fit on a multiprocessor");
      smCount[device] = std::max(1, nsm);
    }
    nsm = smCount[device];
  }
  // one CTA per multiprocessor, at most one per task plus one
  L.grid = std::max(2, std::min(nsm, (int)L.order.size() + 1));
  L.nSpecial = std::max(1, std::min(std::min(24, std::max(1, L.grid / 6)), L.grid - 1));
  return COSL_OK;
}

TileImage tile_image(const BaPlan& P, const TileLaunch& L) {
  TileImage I;
  SlabLayout S;
  auto put = [&](size_t bytes) { return S.take(std::max<size_t>(bytes, 1)); };
  I.tasks = put(sizeof(BaTask) * L.order.size());
  I.bwd = put(sizeof(BaBwdEntry) * P.bwdList.size());
  I.sum = put(sizeof(BaSumEntry) * P.sumList.size());
  I.blkRows = put(sizeof(int) * P.blkRows.size());
  I.blkCam0 = put(sizeof(int) * P.blkCam0.size());
  I.order = put(sizeof(int) * P.order.size());
  I.diagBlk = put(sizeof(int) * std::max(1, P.nTiles));
  I.diagTile = put(sizeof(int) * std::max(1, P.nb));
  I.bytes = S.bytes;
  return I;
}

void tile_image_write(const BaPlan& P, const TileLaunch& L, const TileImage& I, unsigned char* dst) {
  std::vector<int> diagBlk(std::max(1, P.nTiles), -1), diagTile(std::max(1, P.nb), 0);
  for (int k = 0; k < P.nb; ++k) {
    diagTile[k] = P.tileIdx[(size_t)k * P.nb + k];
    diagBlk[diagTile[k]] = k;
  }
  auto pack = [&](size_t off, const void* src, size_t bytes) {
    if (bytes) std::memcpy(dst + off, src, bytes);
  };
  pack(I.tasks, L.order.data(), sizeof(BaTask) * L.order.size());
  pack(I.bwd, P.bwdList.data(), sizeof(BaBwdEntry) * P.bwdList.size());
  pack(I.sum, P.sumList.data(), sizeof(BaSumEntry) * P.sumList.size());
  pack(I.blkRows, P.blkRows.data(), sizeof(int) * P.blkRows.size());
  pack(I.blkCam0, P.blkCam0.data(), sizeof(int) * P.blkCam0.size());
  pack(I.order, P.order.data(), sizeof(int) * P.order.size());
  pack(I.diagBlk, diagBlk.data(), sizeof(int) * diagBlk.size());
  pack(I.diagTile, diagTile.data(), sizeof(int) * diagTile.size());
}

TileLists tile_lists(const TileImage& I, const void* base) {
  const unsigned char* b = static_cast<const unsigned char*>(base);
  TileLists t;
  t.tasks = reinterpret_cast<const BaTask*>(b + I.tasks);
  t.bwd = reinterpret_cast<const BaBwdEntry*>(b + I.bwd);
  t.sum = reinterpret_cast<const BaSumEntry*>(b + I.sum);
  t.blkRows = reinterpret_cast<const int*>(b + I.blkRows);
  t.blkCam0 = reinterpret_cast<const int*>(b + I.blkCam0);
  t.order = reinterpret_cast<const int*>(b + I.order);
  t.diagBlk = reinterpret_cast<const int*>(b + I.diagBlk);
  t.diagTile = reinterpret_cast<const int*>(b + I.diagTile);
  return t;
}

BaTileDev tile_dev(const BaPlan& P, const TileLaunch& L, const TileLists& lists) {
  BaTileDev td = {};
  td.tasks = lists.tasks;
  td.bwd = lists.bwd;
  td.sum = lists.sum;
  td.blkRows = lists.blkRows;
  td.nTasks = (int)L.order.size();
  td.nA = L.nA;
  td.nb = P.nb;
  td.nTiles = P.nTiles;
  td.nCounters = P.nCounters;
  td.nSpecial = L.nSpecial;
  td.xdoneBase = P.nTiles + P.nScratch;
  return td;
}

int tile_solve_enqueue(const TileLaunch& L, const BaTileDev& td, cudaStream_t s) {
  if (L.two)
    COSL_LAUNCH(ba_tile_two, 1, BA_NTHREADS, BA_TILE_SMEM, s, td, L.t00, L.t10, L.t11);
  else
    COSL_LAUNCH(ba_tile_solve, L.grid, BA_NTHREADS, BA_TILE_SMEM, s, td);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// Z = S^-1 on the tile pattern of the plan (S in td.tiles; the dataflow factorisation leaves its factor there).
// Systems of one or two blocks: one resident CTA (ba_selinv_two).  Otherwise the diagonal of S is kept for the
// pivot test, ba_tile_solve factors (its substitutions run on whatever rhs holds), then X_k = L_kk^-T for every
// block and one launch per step of the plan.  Pivot break-down lands in td.sc[td.scFail], the blocks' minimum
// relative pivots in sd.piv.  sd.cnt must be zero.
int selinv_launch(const TileLaunch& L, const BaSelPlan& SP, const BaTileDev& td, const BaSelDev& sd,
                  cudaStream_t st) {
  if (td.nb <= 0) return COSL_OK;
  if (L.two) {
    COSL_LAUNCH(ba_selinv_two, 1, BA_NTHREADS, BA_SEL2_SMEM, st, td.tiles, td.blkRows, L.t00, L.t10, L.t11, sd.Z,
                sd.piv, td.sc + td.scFail);
  } else {
    COSL_LAUNCH(ba_cov_sdiag, td.nb, BA_TB, 0, st, td.tiles, sd.diagTile, sd.sdiag);
    COSL_LAUNCH(ba_tile_solve, L.grid, BA_NTHREADS, BA_TILE_SMEM, st, td);
    COSL_LAUNCH(ba_selinv_xinv, td.nb, BA_NTHREADS, BA_SELX_SMEM, st, sd);
    for (int q = 0; q + 1 < (int)SP.stepBegin.size(); ++q) {
      const int t0 = SP.stepBegin[q], nOff = SP.stepBegin[q + 1] - t0 - 1;
      COSL_LAUNCH(ba_selinv_step, std::max(1, nOff), BA_NTHREADS, BA_SELS_SMEM, st, sd, q, t0, nOff);
    }
  }
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// The device copy of a selected-inversion plan: [tasks | ops]
std::vector<unsigned char> selinv_index(const BaSelPlan& SP, size_t* oOps) {
  SlabLayout S;
  S.take(sizeof(BaSelTask) * std::max<size_t>(1, SP.tasks.size()));
  *oOps = S.take(sizeof(BaSelOp) * std::max<size_t>(1, SP.ops.size()));
  std::vector<unsigned char> h(S.bytes, 0);
  if (!SP.tasks.empty()) std::memcpy(h.data(), SP.tasks.data(), sizeof(BaSelTask) * SP.tasks.size());
  if (!SP.ops.empty()) std::memcpy(h.data() + *oOps, SP.ops.data(), sizeof(BaSelOp) * SP.ops.size());
  return h;
}

}  // namespace coslam

/* ---------------------------------------------------------------- NCCL through dlopen */
namespace {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSum = 0, ncclMax = 2, ncclUint8 = 1, ncclFloat64 = 8 };

struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};

NcclApi& nccl() {
  static NcclApi api;
  if (api.handle) return api;
  // an already-loaded libnccl (e.g. the one torch bundles) wins: same SONAME
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (api.handle) break;
  }
  if (!api.handle) return api;
  api.GetUniqueId = (int (*)(ncclUniqueId*))dlsym(api.handle, "ncclGetUniqueId");
  api.CommInitRank =
      (int (*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(api.handle, "ncclCommInitRank");
  api.CommDestroy = (int (*)(ncclComm_t))dlsym(api.handle, "ncclCommDestroy");
  api.AllReduce = (int (*)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(
      api.handle, "ncclAllReduce");
  api.GetErrorString = (const char* (*)(int))dlsym(api.handle, "ncclGetErrorString");
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce;
  return api;
}

}  // namespace

struct cosl_ba_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1, device = 0;
};

/* ---------------------------------------------------------------- solver state */
struct cosl_ba_solver {
  cosl_ba_options opt;
  cosl_ba_comm* comm = nullptr;
  int device = 0;
  RequestStream rq;  // the solver's stream: every call enqueues there, cosl_ba_solver_submit as one request
  BaDev d;
  // host copies needed for write-back
  int m = 0, n = 0, mcon = 0, ncon = 0, mf = 0, ns = 0;
  long long N = 0, Nc = 0;
  std::vector<double> q0;  // m x 4
  // device buffers: every allocation is in `cap` (bytes), kept while a loaded problem fits in it
  std::unordered_map<void*, size_t> cap;
  // the read-only arrays of the loaded problem, uploaded as one block (load_problem): ptr, cam, xy, camK,
  // the Schur work items and the solve plan's lists point into d_in
  unsigned char* d_in = nullptr;
  const double* d_camK = nullptr;
  double* d_camR0 = nullptr;
  double *d_pa = nullptr, *d_na = nullptr, *d_dpa = nullptr;
  double *d_pb = nullptr, *d_nb = nullptr, *d_dpb = nullptr;
  const int* d_cam = nullptr;
  int *d_pt = nullptr, *d_cobs = nullptr, *d_ccam = nullptr;
  const double* d_xy = nullptr;
  double* d_wgt = nullptr;
  const long long* d_ptr = nullptr;
  unsigned *d_hist = nullptr, *d_pcnt = nullptr;  // set-up scratch of the index kernels
  // pinned staging buffer of the uploads: [R0 | pa | X] (upload_params) then the block of d_in; evStaged
  // marks the end of the last copy out of it
  unsigned char* h_stage = nullptr;
  size_t stageBytes = 0;
  cudaEvent_t evStaged = nullptr;
  double *d_W = nullptr, *d_V = nullptr, *d_eb = nullptr;
  double* d_Uea = nullptr;   // [U (m x 21) | ea (m x 6)] contiguous for one all-reduce
  // reduced camera system: [rhs (nb*64) | tiles]; the leading part [rhs | Schur-structure tiles]
  // is the payload of the one all-reduce per LM trial (ba_tile.cuh)
  BaPlan plan;
  double* d_S = nullptr;
  long long reduceCount = 0;  // doubles in the all-reduce payload
  double *d_Linv = nullptr, *d_y = nullptr, *d_x = nullptr;
  int* d_cnt = nullptr;
  double* d_rhsS = nullptr;
  const int* d_solIdx = nullptr;
  TileLaunch tile;  // of the loaded plan
  TileLists tl;     // the plan's lists in d_in
  BaTileDev td;
  unsigned long long* d_trace = nullptr;
  int numSM = 1;  // of the solver's device
  double factorFlops = 0.0;
  double* d_sc = nullptr;
  unsigned char* d_outlier = nullptr;
  const BaPairItem* d_items = nullptr;
  double* d_Vinv = nullptr;
  unsigned long long scSeq = 0;  // sequence number of the last scalar read-back (ba_publish_sc)
  int4* d_entries = nullptr;
  int nItems = 0;
  long long nEntries = 0;
  double* h_sc = nullptr;  // pinned
  SectionTimer timer;
  int secLin = 0, secSchur = 0, secSolve = 0, secBack = 0, secCost = 0, secComm = 0;
  // submitted robust loop (cosl_ba_solver_submit): the graph with the device-side LM control and the
  // parameter buffers it was built for
  BaCtl* d_ctl = nullptr;
  cudaGraphExec_t graphExec = nullptr;
  bool graphStale = false;  // a load changed the problem since the graph was built
  const double *graphPa = nullptr, *graphNa = nullptr, *graphPb = nullptr, *graphNb = nullptr;
  // stop / progress (cosl_ba_solver_stop / _progress), the calls another thread may make while one is inside
  // run / submit / collect.  Every run and submit takes the next request number; a stop names the current one.
  BaCtlLink* d_link = nullptr;        // request number, stop word and progress record of the submitted loop
  cudaStream_t sideStream = nullptr;  // the copies of stop and progress
  std::mutex sideMu;                  // the side stream and its pinned slots (h_sc + BA_PIN_*)
  std::atomic<unsigned long long> reqNo{0}, stopReq{0};
  std::atomic<int> reqKind{0};     // of the last request: 0 none, 1 run (host loop), 2 submit (graph)
  std::atomic<int> hostRunning{0}, submitted{0};
  unsigned long long loopReq = 0;  // the request the host loop runs; 0: not stoppable (run_fixed, cosl_ba_solve)
  std::mutex hostProgMu;
  BaProgress hostProg = {};  // the host driver's progress record
  // covariance stage (cosl_ba_solver_set_covariance, DESIGN.md 4.6)
  double covVar = 0.0;       // pixel variance; 0: disarmed
  bool covReady = false;     // the selected-inversion plan and the stage's buffers exist for the loaded problem
  bool covValid = false;     // the stage ran on the resident parameters
  double graphCovVar = 0.0;  // covVar the submitted graph was built with
  BaSelPlan sel;
  BaSelDev sdev = {};
  double *d_covWgt = nullptr, *d_covZ = nullptr, *d_covX = nullptr, *d_covSdiag = nullptr, *d_covPiv = nullptr;
  double *d_covT = nullptr, *d_covCam = nullptr, *d_covPt = nullptr, *d_covSc = nullptr;
  unsigned char *d_covUnc = nullptr, *d_covIdx = nullptr;
  int* d_covCnt = nullptr;
  // measurement covariances (cosl_ba_solver_set_obs_cov, DESIGN.md 4.7): d.obsL is d_obsL while they are set and
  // nullptr otherwise; the kernels that read it are launched as their OBSCOV instantiations then
  double* d_obsL = nullptr;
  const double* graphObsL = nullptr;  // d.obsL the submitted graph was built with
};

namespace {

void quat2mat(const double q[4], double R[9]) {
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

// mat2quat of LibVisualSLAM geometry/SL_Quaternion.h is not in the tree; Shepperd's method,
// normalised, w >= 0 (same as the oracle)
void mat2quat(const double R[9], double q[4]) {
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

void quat_mul(const double a[4], const double b[4], double p[4]) {
  p[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  p[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  p[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  p[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

// Pinned slots for the per-trial scalar read-back.  cudaMallocHost / cudaFreeHost cost milliseconds
// each; a drop-in call creates and destroys a solver, so the slots are pooled.
enum {
  BA_PIN_REQ = 20,   // the request number the submit copies to the device
  BA_PIN_STOP = 24,  // the stop word cosl_ba_solver_stop copies to the device
  BA_PIN_PROG = 32,  // two copies of the progress record (8 doubles each)
  BA_PIN_SLOT = 48   // doubles per slot
};
static_assert(sizeof(BaProgress) == 8 * sizeof(double), "progress record size");
struct PinnedSlots {
  std::mutex mu;
  std::vector<double*> free_;
  double* get() {
    std::lock_guard<std::mutex> lk(mu);
    if (!free_.empty()) {
      double* p = free_.back();
      free_.pop_back();
      return p;
    }
    double* p = nullptr;
    // 16 scalars + the sequence flag of ba_publish_sc; mapped + portable: every device of the process writes
    // its scalars straight into this host memory (UVA: the host pointer is the device pointer).  Then the
    // sources and targets of the request-number, stop and progress copies (BA_PIN_*).
    if (cudaHostAlloc(&p, sizeof(double) * BA_PIN_SLOT, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
      return nullptr;
    std::memset(p, 0, sizeof(double) * BA_PIN_SLOT);
    return p;
  }
  void put(double* p) {
    std::lock_guard<std::mutex> lk(mu);
    free_.push_back(p);
  }
};
static PinnedSlots& pinned_slots() {
  static PinnedSlots* p = new PinnedSlots();  // never destroyed: outlives the CUDA context teardown order
  return *p;
}

template <typename T>
int dev_alloc(cudaStream_t st, T** p, size_t count) {
  COSL_CUDA(cudaMallocAsync((void**)p, sizeof(T) * (count ? count : 1), st));
  return COSL_OK;
}

// worker threads for host-side index building: affinity and cgroup quota (shared between the
// local ranks), at most 16; COSLAM_B200_THREADS overrides
static thread_local int t_rank_share = 1;  // ranks driven by threads of this process (cosl_ba_solve_multi)
static int host_threads_all() {
  static const int n = [] {
    int c = 1;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) c = CPU_COUNT(&set);
    if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
      char q[64];
      long long per = 0;
      if (std::fscanf(f, "%63s %lld", q, &per) == 2 && std::strcmp(q, "max") != 0 && per > 0) {
        const long long quota = std::atoll(q);
        if (quota > 0) c = std::min<long long>(c, (quota + per - 1) / per);
      }
      std::fclose(f);
    }
    // several ranks on one host (torchrun exports LOCAL_WORLD_SIZE) share the quota
    if (const char* lws = std::getenv("LOCAL_WORLD_SIZE")) {
      const int n = std::atoi(lws);
      if (n > 1) c = std::max(1, c / n);
    }
    if (const char* ov = std::getenv("COSLAM_B200_THREADS")) {
      const int n = std::atoi(ov);
      if (n >= 1) c = n;
    }
    return std::max(1, std::min(c, 16));
  }();
  return n;
}
static int host_threads() { return std::max(1, host_threads_all() / std::max(1, t_rank_share)); }

static bool ba_timing() {
  static const bool on = std::getenv("COSL_BA_TIMING") != nullptr;
  return on;
}
static double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ptr monotone from 0, camera indices in range, and no (point, camera) pair twice.  The Schur
// contraction relies on the last: its pair lists hold one entry per ordered pair of a point's
// observations with the second camera >= the first, which covers each pair of cameras once only
// when a point has at most one observation per camera (sba's vmask cannot express more either).
int check_observations(const cosl_ba_problem* p) {
  if (p->n && p->ptr[0] != 0) return set_error(COSL_E_INVALID, "ptr[0] != 0");
  std::vector<int> seen((size_t)p->m, -1);  // last point that camera j observed
  for (int i = 0; i < p->n; ++i) {
    if (p->ptr[i + 1] < p->ptr[i]) return set_error(COSL_E_INVALID, "ptr not monotone at %d", i);
    for (long long o = p->ptr[i]; o < p->ptr[i + 1]; ++o) {
      const int j = p->cam[o];
      if (j < 0 || j >= p->m) return set_error(COSL_E_INVALID, "camera index out of range");
      if (seen[j] == i)
        return set_error(COSL_E_INVALID, "point %d is observed twice by camera %d (one observation per pair)", i, j);
      seen[j] = i;
    }
  }
  return COSL_OK;
}

// Library-owned pinned staging buffers: a load copies every array it uploads into one first, so that
// the uploads are asynchronous whatever memory the caller's arrays live in.  cudaHostAlloc costs
// milliseconds and cosl_ba_solve creates a solver per call, so released buffers are pooled.
struct PinnedStaging {
  std::mutex mu;
  std::vector<std::pair<unsigned char*, size_t>> free_;
  // a buffer of at least `bytes`: the largest pooled one, replaced by a new one when it is too small
  int get(size_t bytes, unsigned char** p, size_t* size) {
    std::pair<unsigned char*, size_t> b(nullptr, 0);
    {
      std::lock_guard<std::mutex> lk(mu);
      auto it = std::max_element(free_.begin(), free_.end(),
                                 [](const std::pair<unsigned char*, size_t>& a,
                                    const std::pair<unsigned char*, size_t>& c) { return a.second < c.second; });
      if (it != free_.end()) {
        b = *it;
        free_.erase(it);
      }
    }
    if (b.first && b.second < bytes) {
      cudaFreeHost(b.first);
      b = {nullptr, 0};
    }
    if (!b.first) {
      const size_t sz = std::max<size_t>(bytes + bytes / 4, (size_t)1 << 20);
      void* q = nullptr;
      if (cudaHostAlloc(&q, sz, cudaHostAllocPortable) != cudaSuccess)
        return set_error(COSL_E_NOMEM, "pinned staging buffer of %zu bytes", sz);
      b = {(unsigned char*)q, sz};
    }
    *p = b.first;
    *size = b.second;
    return COSL_OK;
  }
  void put(unsigned char* p, size_t size) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(mu);
    free_.emplace_back(p, size);
  }
};
static PinnedStaging& pinned_staging() {
  static PinnedStaging* p = new PinnedStaging();  // never destroyed, as pinned_slots()
  return *p;
}

// A device buffer of at least `count` elements: kept while it is large enough, otherwise replaced by a
// stream-ordered allocation with some headroom.  Neither waits for the device.
template <typename T>
int grow(cosl_ba_solver* s, T** p, size_t count) {
  const size_t bytes = sizeof(T) * std::max<size_t>(count, 1);
  if (*p) {
    auto it = s->cap.find((void*)*p);
    if (it != s->cap.end() && it->second >= bytes) return COSL_OK;
    s->cap.erase((void*)*p);
    COSL_CUDA(cudaFreeAsync((void*)*p, s->rq.stream));
    *p = nullptr;
  }
  const size_t want = bytes + bytes / 4;
  COSL_CUDA(cudaMallocAsync((void**)p, want, s->rq.stream));
  s->cap[(void*)*p] = want;
  return COSL_OK;
}

inline bool multi(const cosl_ba_solver* s) { return s->comm && s->comm->nranks > 1; }
inline int rank_of(const cosl_ba_solver* s) { return s->comm ? s->comm->rank : 0; }

// R, t, X -> camR0, pa, pb through the parameter part of the staging buffer.  The caller has waited for
// evStaged (the staging buffer is free) and records it after its own copies.
int upload_params(cosl_ba_solver* s, const cosl_ba_problem* p) {
  const int m = s->m;
  double* R0 = reinterpret_cast<double*>(s->h_stage);
  double* pa = R0 + 9 * (size_t)m;
  double* X = pa + 6 * (size_t)m;
  s->q0.resize((size_t)m * 4);
  for (int j = 0; j < m; ++j) {
    mat2quat(p->R + 9 * j, &s->q0[4 * j]);
    quat2mat(&s->q0[4 * j], &R0[9 * j]);
    for (int k = 0; k < 3; ++k) {
      pa[6 * j + k] = 0.0;
      pa[6 * j + 3 + k] = p->t[3 * j + k];
    }
  }
  if (s->n) std::memcpy(X, p->X, sizeof(double) * 3 * (size_t)s->n);
  COSL_CUDA(cudaMemcpyAsync(s->d_camR0, R0, sizeof(double) * 9 * m, cudaMemcpyHostToDevice, s->rq.stream));
  COSL_CUDA(cudaMemcpyAsync(s->d_pa, pa, sizeof(double) * 6 * m, cudaMemcpyHostToDevice, s->rq.stream));
  if (s->n)
    COSL_CUDA(cudaMemcpyAsync(s->d_pb, X, sizeof(double) * 3 * (size_t)s->n, cudaMemcpyHostToDevice, s->rq.stream));
  return COSL_OK;
}

void free_solver(cosl_ba_solver* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  if (s->rq.stream) cudaStreamSynchronize(s->rq.stream);
  if (s->sideStream) {
    cudaStreamSynchronize(s->sideStream);
    cudaStreamDestroy(s->sideStream);
  }
  s->timer.destroy();
  if (s->graphExec) cudaGraphExecDestroy(s->graphExec);
  if (s->evStaged) cudaEventDestroy(s->evStaged);
  for (const auto& b : s->cap) cudaFreeAsync(b.first, s->rq.stream);
  s->rq.destroy();  // waits for the frees above
  if (s->h_sc) pinned_slots().put(s->h_sc);
  pinned_staging().put(s->h_stage, s->stageBytes);
  delete s;
}

// temporaries of the solver set-up: handed back to the pool on every exit path
struct TmpDeviceBufs {
  cudaStream_t st;
  std::vector<void*> bufs;
  explicit TmpDeviceBufs(cudaStream_t s) : st(s) {}
  ~TmpDeviceBufs() {
    for (void* b : bufs)
      if (b) cudaFreeAsync(b, st);
  }
  template <typename T>
  int alloc(T** p, size_t count) {
    const int rc = dev_alloc(st, p, count);
    if (rc == COSL_OK) bufs.push_back(*p);
    return rc;
  }
};

// The arguments of a problem (cosl_ba_solver_create / _load)
int check_problem(const cosl_ba_problem* prob, const char* what) {
  if (!prob) return set_error(COSL_E_INVALID, "%s: null problem", what);
  if (prob->m < 1 || prob->n < 0 || prob->nobs < 0 || prob->m_con < 0 || prob->m_con > prob->m ||
      prob->n_con < 0 || prob->n_con > prob->n || !prob->K || !prob->R || !prob->t ||
      (prob->n && (!prob->X || !prob->ptr)) || (prob->nobs && (!prob->cam || !prob->xy)) ||
      prob->nobs >= (1ll << 31))
    return set_error(COSL_E_INVALID, "%s: bad problem", what);
  if (prob->n && prob->ptr[prob->n] != prob->nobs) return set_error(COSL_E_INVALID, "ptr[n] != nobs");
  return check_observations(prob);
}

// Measurement covariances covx[N][2][2] (px^2, row-major): finite, symmetric to 1e-12 relative and positive
// definite.  On success L[N][3] holds (s00, s01, s11) for ba_obscov_factor; otherwise the first bad observation is
// named.
int check_obs_cov(const double* covx, long long N, std::vector<double>& L, const char* what) {
  L.resize(3 * (size_t)N);
  for (long long o = 0; o < N; ++o) {
    const double* c = covx + 4 * (size_t)o;
    const double a = c[0], b = c[1], b2 = c[2], d = c[3];
    if (!std::isfinite(a) || !std::isfinite(b) || !std::isfinite(b2) || !std::isfinite(d))
      return set_error(COSL_E_INVALID, "%s: covariance of observation %lld is not finite", what, o);
    if (std::fabs(b - b2) > 1e-12 * std::max(std::fabs(a), std::fabs(d)))
      return set_error(COSL_E_INVALID, "%s: covariance of observation %lld is not symmetric (%.17g, %.17g)", what, o,
                       b, b2);
    const double s01 = 0.5 * (b + b2), det = a * d - s01 * s01;
    if (!(a > 0.0) || !(d > 0.0) || !(det > 0.0) || !std::isfinite(d / det))
      return set_error(COSL_E_INVALID, "%s: covariance of observation %lld is not positive definite", what, o);
    L[3 * (size_t)o] = a;
    L[3 * (size_t)o + 1] = s01;
    L[3 * (size_t)o + 2] = d;
  }
  return COSL_OK;
}

// Sets (covx != NULL, checked by check_obs_cov into L) or clears the measurement covariances of the loaded problem:
// the upload and the factorisation are enqueued on the solver's stream, nothing is waited for.
int set_obs_cov(cosl_ba_solver* s, const std::vector<double>* L) {
  if (!L) {
    s->d.obsL = nullptr;
    return COSL_OK;
  }
  COSL_TRY(grow(s, &s->d_obsL, 3 * (size_t)s->N));
  // from pageable memory: the call returns once the source has been staged
  if (s->N) {
    COSL_CUDA(cudaMemcpyAsync(s->d_obsL, L->data(), sizeof(double) * 3 * (size_t)s->N, cudaMemcpyHostToDevice,
                              s->rq.stream));
    COSL_LAUNCH(ba_obscov_factor, (unsigned)div_up64(s->N, 256), 256, 0, s->rq.stream, s->d_obsL, s->N);
    COSL_CUDA(cudaGetLastError());
  }
  s->d.obsL = s->d_obsL;
  return COSL_OK;
}

// What the host derives from the observation lists (validated by check_problem) to plan a problem
// without a device round trip: the start of each free camera in the camera-major list and the start of
// each camera-pair bucket (ja <= jb, row-major over mf x mf) in the Schur pair entries.
struct BaIndex {
  long long Nc = 0, nEntries = 0;
  std::vector<unsigned> camStart;  // mf + 1
  std::vector<unsigned> poff;      // mf * mf + 1
};

int index_problem(const cosl_ba_problem* p, BaIndex& x) {
  const int mcon = p->m_con, mf = p->m - p->m_con, n = p->n, ncon = p->n_con;
  std::vector<long long> perCam((size_t)mf, 0);
  long long ne = 0;
  for (int i = 0; i < n; ++i) {
    long long k = 0;
    for (long long o = p->ptr[i]; o < p->ptr[i + 1]; ++o)
      if (p->cam[o] >= mcon) {
        ++perCam[p->cam[o] - mcon];
        ++k;
      }
    // ba_pairs_build: a free point with k free-camera observations gives k (k + 1) / 2 entries
    if (i >= ncon) ne += k * (k + 1) / 2;
  }
  if (ne > INT_MAX)
    return set_error(COSL_E_INVALID, "%lld Schur pair entries: more than the solver's 32-bit offsets can address", ne);
  x.nEntries = ne;
  x.camStart.assign((size_t)mf + 1, 0u);
  for (int j = 0; j < mf; ++j) x.camStart[j + 1] = x.camStart[j] + (unsigned)perCam[j];
  x.Nc = x.camStart[mf];
  // entries per bucket; large problems (the c4 global BA) split the points over a few threads
  const size_t nBuckets = (size_t)mf * mf;
  auto count = [&](int i0, int i1, unsigned* c) {
    std::vector<int> js;
    for (int i = i0; i < i1; ++i) {
      js.clear();
      for (long long o = p->ptr[i]; o < p->ptr[i + 1]; ++o)
        if (p->cam[o] >= mcon) js.push_back(p->cam[o] - mcon);
      for (size_t a = 0; a < js.size(); ++a)
        for (size_t b = a; b < js.size(); ++b) ++c[(size_t)std::min(js[a], js[b]) * mf + std::max(js[a], js[b])];
    }
  };
  std::vector<unsigned> cnt(nBuckets, 0u);
  const int T = (int)std::min<long long>({(long long)host_threads(), 1 + ne / (1 << 20), (long long)std::max(1, n - ncon)});
  if (T <= 1) {
    count(ncon, n, cnt.data());
  } else {
    std::vector<std::vector<unsigned>> part(T);
    std::vector<std::thread> th;
    for (int t = 0; t < T; ++t)
      th.emplace_back([&, t] {
        part[t].assign(nBuckets, 0u);
        count(ncon + (int)((long long)(n - ncon) * t / T), ncon + (int)((long long)(n - ncon) * (t + 1) / T),
              part[t].data());
      });
    for (auto& h : th) h.join();
    th.clear();
    for (int t = 0; t < T; ++t)
      th.emplace_back([&, t] {
        const size_t b0 = nBuckets * t / T, b1 = nBuckets * (t + 1) / T;
        for (int u = 0; u < T; ++u)
          for (size_t b = b0; b < b1; ++b) cnt[b] += part[u][b];
      });
    for (auto& h : th) h.join();
  }
  x.poff.assign(nBuckets + 1, 0u);
  for (size_t b = 0; b < nBuckets; ++b) x.poff[b + 1] = x.poff[b] + cnt[b];
  return COSL_OK;
}

int cov_prepare(cosl_ba_solver* s);

// Replace the solver's problem with `p` (validated by check_problem, indexed by index_problem).  The
// host plans the reduced-system solve and the Schur work items from the bucket counts, copies everything
// the device needs into the staging buffer and enqueues the rest on the solver's stream: the upload, the
// observation index kernels (ba_index_*) and the pair entries (ba_pairs_build).  Waits for nothing on the
// device except, for a multi-rank solver, the all-reduce of the co-visibility bitmap.
int load_problem(cosl_ba_solver* s, const cosl_ba_problem* p, const BaIndex& x) {
  const double tLoad0 = now_s();
  const int m = p->m, n = p->n, mcon = p->m_con, ncon = p->n_con, mf = m - mcon;
  const long long N = p->nobs, Nc = x.Nc, nEntries = x.nEntries;
  const size_t nBuckets = (size_t)mf * mf;
  // camera co-visibility (which pairs of free cameras share a free point) -> plan of the reduced-system
  // solve (ordering, tiles, task DAG) and the work lists of the Schur contraction.  In the multi-GPU case
  // every rank must derive the SAME structure although it only sees the pairs of its own point shard:
  // the presence bitmap is all-reduced (max) first.
  std::vector<uint8_t> adj(nBuckets, 0);
  for (int ja = 0; ja < mf; ++ja)
    for (int jb = ja; jb < mf; ++jb)
      if (x.poff[(size_t)ja * mf + jb + 1] > x.poff[(size_t)ja * mf + jb]) adj[(size_t)ja * mf + jb] = adj[(size_t)jb * mf + ja] = 1;
  if (multi(s) && mf > 0) {
    TmpDeviceBufs tmp(s->rq.stream);
    uint8_t* d_adj = nullptr;
    COSL_TRY(tmp.alloc(&d_adj, adj.size()));
    COSL_CUDA(cudaMemcpyAsync(d_adj, adj.data(), adj.size(), cudaMemcpyHostToDevice, s->rq.stream));
    const int rc = nccl().AllReduce(d_adj, d_adj, adj.size(), ncclUint8, ncclMax, s->comm->comm, s->rq.stream);
    if (rc != 0) return set_error(COSL_E_NCCL, "ncclAllReduce (co-visibility) failed (%d)", rc);
    COSL_CUDA(cudaMemcpyAsync(adj.data(), d_adj, adj.size(), cudaMemcpyDeviceToHost, s->rq.stream));
    COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  }
  const double tPlan0 = now_s();
  BaPlan P = ba_make_plan(mf, adj);
  if (ba_timing()) std::fprintf(stderr, "[ba timing] plan %.1f ms\n", 1e3 * (now_s() - tPlan0));
  if (P.nb < 0) return set_error(COSL_E_INVALID, "solve plan: dependency cycle (internal error)");
  // destination of the 6x6 block of camera pair (ja <= jb) in the tile storage: the lower
  // triangle of the permuted system, i.e. the later camera (block, offset) gives the row
  auto pair_dst = [&](int ja, int jb, int& dst, int& rOff, int& cOff, int& trans) {
    const int bA = P.camBlk[ja], oA = P.camOff[ja], bB = P.camBlk[jb], oB = P.camOff[jb];
    const bool bLater = (bB > bA) || (bB == bA && oB >= oA);
    const int tile = bLater ? P.tileIdx[(size_t)bB * P.nb + bA] : P.tileIdx[(size_t)bA * P.nb + bB];
    if (tile < 0 || tile >= P.nTilesOrig) return false;
    dst = tile * BA_TILE;
    trans = bLater ? 0 : 1;
    cOff = bLater ? oA : oB;
    rOff = bLater ? oB : oA;
    return true;
  };
  // pair lists: one bucket per camera pair; a work item is a run of <= 512 entries of one bucket; the
  // entries themselves are placed by ba_pairs_build.  Fewer entries per item when the problem is small
  // (local BA: a few dozen camera pairs with thousands of entries each), so that the grid still fills
  // the GPU; ba_schur_pairs_st works in batches of 32 entries and sums 32 lanes per item: multiples of
  // 32, >= 128
  std::vector<BaPairItem> items;
  const int chunk = (int)(32 * std::max<long long>(4, std::min<long long>(16, nEntries / (4096 * 32))));
  for (int ja = 0; ja < mf; ++ja)
    for (int jb = ja; jb < mf; ++jb) {
      const long long b0 = x.poff[(size_t)ja * mf + jb], b1 = x.poff[(size_t)ja * mf + jb + 1];
      if (b1 == b0) continue;
      BaPairItem it;
      std::memset(&it, 0, sizeof(it));
      it.rowCam = ja;
      it.colCam = jb;
      if (!pair_dst(ja, jb, it.dst, it.rOff, it.cOff, it.trans))
        return set_error(COSL_E_INVALID, "solve plan: missing tile");
      it.rhsIdx = P.camBlk[ja] * BA_TB + P.camOff[ja];
      for (long long b = b0; b < b1; b += chunk) {
        it.begin = (int)b;
        it.end = (int)std::min(b1, b + chunk);
        items.push_back(it);
      }
    }
  TileLaunch tile = tile_launch_plan(P);
  COSL_TRY(tile_launch_device(tile));
  const TileImage img = tile_image(P, tile);
  const int nb = std::max(1, P.nb), nTiles = std::max(1, P.nTiles);
  std::vector<int> h_solIdx(std::max(1, mf), 0);
  for (int j = 0; j < mf; ++j) h_solIdx[j] = P.camBlk[j] * BA_TB + P.camOff[j];
  // intrinsics: only K0,K1,K2,K4,K5 are used (as BundleRTS packs them, app/SL_CoSLAMBA.cpp:337-343)
  std::vector<double> camK((size_t)m * 5);
  for (int j = 0; j < m; ++j) {
    const double* K = p->K + 9 * j;
    camK[5 * j] = K[0];
    camK[5 * j + 1] = K[1];
    camK[5 * j + 2] = K[2];
    camK[5 * j + 3] = K[4];
    camK[5 * j + 4] = K[5];
  }
  // the block of read-only arrays that becomes d_in: sections of whole 256-byte lines
  struct Sec {
    const void* src;
    size_t bytes, off;
  };
  std::vector<Sec> secs;
  size_t inBytes = 0;
  auto sec = [&](const void* src, size_t bytes) {
    secs.push_back({src, bytes, inBytes});
    inBytes += std::max<size_t>(256, (bytes + 255) & ~(size_t)255);
    return secs.back().off;
  };
  const long long zeroPtr = 0;
  const size_t oPtr = sec(n ? (const void*)p->ptr : (const void*)&zeroPtr, sizeof(long long) * ((size_t)n + 1));
  const size_t oCam = sec(p->cam, sizeof(int) * (size_t)N);
  const size_t oXy = sec(p->xy, sizeof(double) * 2 * (size_t)N);
  const size_t oK = sec(camK.data(), sizeof(double) * camK.size());
  const size_t oItems = sec(items.data(), sizeof(BaPairItem) * items.size());
  const size_t oPlan = sec(nullptr, img.bytes);  // tile_image_write
  const size_t oSol = sec(h_solIdx.data(), sizeof(int) * h_solIdx.size());
  const size_t oCamStart = sec(x.camStart.data(), sizeof(unsigned) * x.camStart.size());
  const size_t oPoff = sec(x.poff.data(), sizeof(unsigned) * x.poff.size());
  const size_t parBytes = (sizeof(double) * (15 * (size_t)m + 3 * (size_t)n) + 255) & ~(size_t)255;
  // the staging buffer is free once the last copy out of it has run (at once, unless a load was
  // enqueued behind other work and is loaded over right away)
  if (s->evStaged) COSL_CUDA(cudaEventSynchronize(s->evStaged));
  if (parBytes + inBytes > s->stageBytes) {
    pinned_staging().put(s->h_stage, s->stageBytes);
    s->h_stage = nullptr;
    s->stageBytes = 0;
    COSL_TRY(pinned_staging().get(parBytes + inBytes, &s->h_stage, &s->stageBytes));
  }
  for (const Sec& q : secs)
    if (q.src && q.bytes) std::memcpy(s->h_stage + parBytes + q.off, q.src, q.bytes);
  tile_image_write(P, tile, img, s->h_stage + parBytes + oPlan);
  // from here on the handle holds the new problem
  s->m = m;
  s->n = n;
  s->mcon = mcon;
  s->ncon = ncon;
  s->mf = mf;
  s->ns = 6 * mf;
  s->N = N;
  s->Nc = Nc;
  s->nEntries = nEntries;
  s->nItems = (int)items.size();
  s->plan = std::move(P);
  s->tile = std::move(tile);
  const BaPlan& PL = s->plan;
  s->reduceCount = (long long)nb * BA_TB + (long long)PL.nTilesOrig * BA_TILE;
  s->factorFlops = PL.flops;
  s->graphStale = true;
  COSL_TRY(grow(s, &s->d_in, inBytes));
  COSL_CUDA(cudaMemcpyAsync(s->d_in, s->h_stage + parBytes, inBytes, cudaMemcpyHostToDevice, s->rq.stream));
  s->d_ptr = reinterpret_cast<const long long*>(s->d_in + oPtr);
  s->d_cam = reinterpret_cast<const int*>(s->d_in + oCam);
  s->d_xy = reinterpret_cast<const double*>(s->d_in + oXy);
  s->d_camK = reinterpret_cast<const double*>(s->d_in + oK);
  s->d_items = reinterpret_cast<const BaPairItem*>(s->d_in + oItems);
  s->tl = tile_lists(img, s->d_in + oPlan);
  s->d_solIdx = reinterpret_cast<const int*>(s->d_in + oSol);
  const unsigned* d_camStart = reinterpret_cast<const unsigned*>(s->d_in + oCamStart);
  const unsigned* d_poff = reinterpret_cast<const unsigned*>(s->d_in + oPoff);
  // the buffers the solver writes
  COSL_TRY(grow(s, &s->d_camR0, (size_t)m * 9));
  COSL_TRY(grow(s, &s->d_pa, (size_t)m * 6));
  COSL_TRY(grow(s, &s->d_na, (size_t)m * 6));
  COSL_TRY(grow(s, &s->d_dpa, (size_t)m * 6));
  COSL_TRY(grow(s, &s->d_pb, (size_t)n * 3));
  COSL_TRY(grow(s, &s->d_nb, (size_t)n * 3));
  COSL_TRY(grow(s, &s->d_dpb, (size_t)n * 3));
  COSL_TRY(grow(s, &s->d_pt, (size_t)N));
  COSL_TRY(grow(s, &s->d_cobs, (size_t)Nc));
  COSL_TRY(grow(s, &s->d_ccam, (size_t)Nc));
  COSL_TRY(grow(s, &s->d_wgt, (size_t)N));
  COSL_TRY(grow(s, &s->d_W, (size_t)N * 18));
  // [V (n x 6) | e_b (n x 3) | U (m x 21) | e_a (m x 6)] in one slab: one memset per linearisation
  COSL_TRY(grow(s, &s->d_V, (size_t)n * 9 + (size_t)m * 27));
  s->d_eb = s->d_V + (size_t)n * 6;
  s->d_Uea = s->d_eb + (size_t)n * 3;
  const size_t rhsLen = (size_t)nb * BA_TB;
  COSL_TRY(grow(s, &s->d_S, rhsLen + ((size_t)nTiles + PL.nScratch) * BA_TILE));
  COSL_TRY(grow(s, &s->d_rhsS, (size_t)std::max(1, PL.nScratch) * BA_TB));
  COSL_TRY(grow(s, &s->d_Linv, (size_t)nb * BA_TILE));
  COSL_TRY(grow(s, &s->d_y, rhsLen));
  COSL_TRY(grow(s, &s->d_x, rhsLen));
  COSL_TRY(grow(s, &s->d_cnt, (size_t)PL.nCounters + 2 + PL.tasks.size()));
  COSL_TRY(grow(s, &s->d_outlier, (size_t)N));
  COSL_TRY(grow(s, &s->d_Vinv, (size_t)n * 6));
  COSL_TRY(grow(s, &s->d_entries, (size_t)nEntries));
  COSL_TRY(upload_params(s, p));
  COSL_CUDA(cudaEventRecord(s->evStaged, s->rq.stream));
  // observation index lists and Schur pair entries
  if (n) COSL_LAUNCH(ba_index_points, div_up(n, 256), 256, 0, s->rq.stream, s->d_ptr, n, s->d_pt);
  if (Nc) {
    const int chunk = (int)std::max<long long>(256, 32 * div_up64(div_up64(N, 256), 32));
    const int nChunks = (int)div_up64(N, chunk);
    COSL_TRY(grow(s, &s->d_hist, (size_t)nChunks * mf));
    COSL_CUDA(cudaMemsetAsync(s->d_hist, 0, sizeof(unsigned) * (size_t)nChunks * mf, s->rq.stream));
    const unsigned gW = (unsigned)div_up64(32LL * nChunks, 256);
    COSL_LAUNCH(ba_index_cams<false>, gW, 256, 0, s->rq.stream, s->d_cam, N, mcon, mf, chunk, s->d_hist, s->d_cobs,
                s->d_ccam);
    COSL_LAUNCH(ba_index_cam_base, div_up(mf, 256), 256, 0, s->rq.stream, s->d_hist, nChunks, mf, d_camStart);
    COSL_LAUNCH(ba_index_cams<true>, gW, 256, 0, s->rq.stream, s->d_cam, N, mcon, mf, chunk, s->d_hist, s->d_cobs,
                s->d_ccam);
  }
  BaDev& d = s->d;
  d.m = m;
  d.n = n;
  d.mcon = mcon;
  d.ncon = ncon;
  d.mf = mf;
  d.ns = s->ns;
  d.N = N;
  d.Nc = Nc;
  d.camK = s->d_camK;
  d.camR0 = s->d_camR0;
  d.cam = s->d_cam;
  d.pt = s->d_pt;
  d.xy = s->d_xy;
  d.wgt = s->d_wgt;
  d.obsL = nullptr;  // a new problem has new observations: its covariances are unset
  d.ptr = s->d_ptr;
  d.cobs = s->d_cobs;
  d.ccam = s->d_ccam;
  d.W = s->d_W;
  d.V = s->d_V;
  d.eb = s->d_eb;
  d.U = s->d_Uea;
  d.ea = s->d_Uea + (size_t)m * 21;
  d.rhs = s->d_S;
  d.tiles = s->d_S + rhsLen;
  d.solIdx = s->d_solIdx;
  d.sc = s->d_sc;
  if (nEntries) {
    COSL_TRY(grow(s, &s->d_pcnt, nBuckets + 1));
    COSL_CUDA(cudaMemsetAsync(s->d_pcnt, 0, sizeof(unsigned) * (nBuckets + 1), s->rq.stream));
    COSL_LAUNCH(ba_pairs_build<true>, (unsigned)div_up64(Nc, 256), 256, 0, s->rq.stream, d, s->d_pcnt, d_poff,
                s->d_entries);
  }
  COSL_CUDA(cudaGetLastError());
  BaTileDev& td = s->td;
  td = tile_dev(PL, s->tile, s->tl);
  td.rhs = d.rhs;
  td.tiles = d.tiles;
  td.rhsS = s->d_rhsS;
  td.Linv = s->d_Linv;
  td.y = s->d_y;
  td.x = s->d_x;
  td.cnt = s->d_cnt;
  td.sc = s->d_sc;
  td.scFail = (int)SC_FAIL;
  s->covReady = s->covValid = false;
  if (s->covVar > 0) COSL_TRY(cov_prepare(s));
  if (ba_timing())
    std::fprintf(stderr, "[ba timing] load: host %.2f ms (%lld pair entries, %d items)\n", 1e3 * (now_s() - tLoad0),
                 nEntries, s->nItems);
  return COSL_OK;
}

// A solver handle without a problem on the current device: stream, scalar slots, the kernel attribute of the
// Schur contraction.  *out is set once the handle exists, also when a later step fails.
int make_handle(const cosl_ba_options* opt, cosl_ba_comm* comm, cosl_ba_solver** out) {
  cosl_ba_solver* s = new (std::nothrow) cosl_ba_solver();
  if (!s) return set_error(COSL_E_NOMEM, "host allocation failed");
  s->opt = *opt;
  s->comm = comm;
  s->device = opt->device;
  *out = s;
  COSL_TRY(s->rq.create());
  keep_pool(opt->device);
  static_assert(SC_NTOT <= 16, "pinned slot size");
  s->h_sc = pinned_slots().get();
  if (!s->h_sc) return set_error(COSL_E_NOMEM, "pinned host allocation failed");
  *reinterpret_cast<volatile unsigned long long*>(s->h_sc + SC_NTOT) = 0;  // a pooled slot keeps its last flag
  s->scSeq = 0;
  COSL_CUDA(cudaEventCreateWithFlags(&s->evStaged, cudaEventDisableTiming));
  COSL_TRY(grow(s, &s->d_sc, (size_t)SC_NTOT));
  COSL_CUDA(cudaStreamCreateWithFlags(&s->sideStream, cudaStreamNonBlocking));
  COSL_TRY(grow(s, &s->d_link, 1));
  COSL_CUDA(cudaMemsetAsync(s->d_link, 0, sizeof(BaCtlLink), s->rq.stream));  // request numbers start at 1
  COSL_CUDA(cudaFuncSetAttribute(ba_schur_pairs_st, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_ST_SMEM));
  int nsm = 0;
  COSL_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, s->device));
  s->numSM = std::max(1, nsm);
  s->secLin = s->timer.section("ba_linearize");
  s->secSchur = s->timer.section("ba_schur");
  s->secSolve = s->timer.section("ba_solve");
  s->secBack = s->timer.section("ba_backsub");
  s->secCost = s->timer.section("ba_cost");
  s->secComm = s->timer.section("ba_allreduce");
  return COSL_OK;
}

/* ---------------------------------------------------------------- device steps */

int allreduce(cosl_ba_solver* s, double* buf, size_t count, int op) {
  if (!multi(s)) return COSL_OK;
  s->timer.begin(s->secComm, s->rq.stream);
  const int rc = nccl().AllReduce(buf, buf, count, ncclFloat64, op, s->comm->comm, s->rq.stream);
  s->timer.end(s->rq.stream);
  if (rc != 0)
    return set_error(COSL_E_NCCL, "ncclAllReduce: %s",
                     nccl().GetErrorString ? nccl().GetErrorString(rc) : "?");
  return COSL_OK;
}

// clear the scalar slots of `mask` (ba_lm_cleared): one memset per run of adjacent slots
int clear_sc(cosl_ba_solver* s, unsigned mask) {
  for (int k = 0; k < SC_NTOT; ++k) {
    if (!(mask >> k & 1u)) continue;
    int e = k + 1;
    while (e < SC_NTOT && (mask >> e & 1u)) ++e;
    COSL_CUDA(cudaMemsetAsync(s->d_sc + k, 0, sizeof(double) * (e - k), s->rq.stream));
    k = e;
  }
  return COSL_OK;
}

// Scalars of a trial -> host.  Instead of a copy-engine transfer + stream synchronise (microseconds of latency per
// LM trial), a 32-thread kernel stores the 16 scalars into MAPPED pinned host memory, fences, and stores a
// sequence number; the host spins on that word.  Falls back to a stream synchronise if the flag does not
// arrive (error on the stream).
__global__ void ba_publish_sc(const double* __restrict__ sc, volatile double* host, unsigned long long seq) {
  if (threadIdx.x < SC_NTOT) host[threadIdx.x] = sc[threadIdx.x];
  __threadfence_system();
  __syncwarp();
  if (threadIdx.x == 0) {
    __threadfence_system();
    *reinterpret_cast<volatile unsigned long long*>(host + SC_NTOT) = seq;
  }
}

int read_sc(cosl_ba_solver* s) {
  // multi-GPU on a crowded host (fewer than 3 usable cores per rank, e.g. 8 ranks in a 16-thread cgroup): a
  // copy-engine read-back + stream synchronise (N ranks polling mapped memory compete with NCCL's proxy
  // threads for the cores; with enough cores per rank the polling read-back wins)
  const bool crowded = multi(s) && host_threads_all() < 3 * s->comm->nranks;
  if (crowded) {
    COSL_CUDA(cudaMemcpyAsync(s->h_sc, s->d_sc, sizeof(double) * SC_NTOT, cudaMemcpyDeviceToHost,
                              s->rq.stream));
    COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
    return COSL_OK;
  }
  const unsigned long long seq = ++s->scSeq;
  COSL_LAUNCH(ba_publish_sc, 1, 32, 0, s->rq.stream, s->d_sc, s->h_sc, seq);
  volatile unsigned long long* flag = reinterpret_cast<volatile unsigned long long*>(s->h_sc + SC_NTOT);
  for (long long spin = 0; *flag != seq; ++spin) {
    if ((spin & 0xfff) == 0xfff) {
      const cudaError_t q = cudaStreamQuery(s->rq.stream);
      if (q == cudaSuccess) break;  // everything ran: the stores are visible after the query
      if (q != cudaErrorNotReady)
        return set_error(COSL_E_CUDA, "scalar read-back: %s", cudaGetErrorString(q));
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (*flag != seq) {  // left through the query: make sure the stores have landed
    COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
    if (*flag != seq) return set_error(COSL_E_CUDA, "scalar read-back: flag missing after synchronise");
  }
  return COSL_OK;
}

// sum w |e|^2 (w |L e|^2 with measurement covariances) at (pa, pb) into d.sc[SC_COST]
int launch_cost(const BaDev& d, const double* pa, const double* pb, unsigned gN, cudaStream_t st) {
  if (d.obsL)
    COSL_LAUNCH(ba_residual_kernel<true>, gN, 256, 0, st, d, pa, pb, 0, 0.0, nullptr);
  else
    COSL_LAUNCH(ba_residual_kernel<false>, gN, 256, 0, st, d, pa, pb, 0, 0.0, nullptr);
  return COSL_OK;
}

// the two linearisation kernels at (d_pa, d_pb) into d's V, eb, W, U, ea (zeroed before)
int launch_linearize(const cosl_ba_solver* s, const BaDev& d, cudaStream_t st) {
  const unsigned gN = (unsigned)div_up64(s->N, 256), gC = (unsigned)div_up64(s->Nc, 128);
  if (d.obsL) {
    if (s->N) COSL_LAUNCH(ba_linearize_points<true>, gN, 256, 0, st, d, s->d_pa, s->d_pb);
    if (s->Nc) COSL_LAUNCH(ba_linearize_cams<true>, gC, 128, 0, st, d, s->d_pa, s->d_pb);
  } else {
    if (s->N) COSL_LAUNCH(ba_linearize_points<false>, gN, 256, 0, st, d, s->d_pa, s->d_pb);
    if (s->Nc) COSL_LAUNCH(ba_linearize_cams<false>, gC, 128, 0, st, d, s->d_pa, s->d_pb);
  }
  return COSL_OK;
}

// The kernels of one stage of the robust loop, enqueued on st (the solver's stream, or the capture of the
// submitted graph), with the stage's multi-rank all-reduces.  dctl: the control block of the submitted loop,
// from which the trial kernels read mu (and the prep kernel doStats) when they run; without it they take mu
// and doStats from the host driver.  doStats: the stage computes |g|_inf / max diag for the eps1 test
// (BaCtl::statsPending).
int enqueue_stage(cosl_ba_solver* s, cudaStream_t st, int stage, const BaCtl* dctl, double mu, int doStats) {
  const unsigned gN = (unsigned)div_up64(s->N, 256);
  const int r0 = rank_of(s) == 0 ? 1 : 0;
  const bool oc = s->d.obsL != nullptr;
  SectionTimer& T = s->timer;
  if (stage == BA_STAGE_ROUND) {  // the round's Tukey weights (on the pixel distance), then its initial cost
    if (s->N) {
      if (s->opt.max_err > 0)
        COSL_LAUNCH(ba_residual_kernel<false>, gN, 256, 0, st, s->d, s->d_pa, s->d_pb, 1, s->opt.max_err, nullptr);
      else
        COSL_LAUNCH(ba_fill_f64, std::min<unsigned>(gN, 1024), 256, 0, st, s->d_wgt, s->N, 1.0);
    }
    T.begin(s->secCost, st);
    if (s->N) COSL_TRY(launch_cost(s->d, s->d_pa, s->d_pb, gN, st));
    T.end(st);
  } else if (stage == BA_STAGE_LIN0 || stage == BA_STAGE_LIN) {  // Jacobians, U, V, W, ea, eb at (pa, pb)
    const long long nV = 9LL * s->n + 27LL * s->m;  // [V | eb | U | ea]
    T.begin(s->secLin, st);
    COSL_LAUNCH(ba_fill_f64, (unsigned)std::min<long long>(div_up64(nV, 256), 1024), 256, 0, st, s->d_V, nV, 0.0);
    COSL_TRY(launch_linearize(s, s->d, st));
    T.end(st);
    COSL_TRY(allreduce(s, s->d_Uea, (size_t)27 * s->m, ncclSum));
    // at itno > 0 the prep kernel of the next trial computes the statistics, unless there is none
    if (stage == BA_STAGE_LIN0 || (!s->ns && doStats)) {
      COSL_LAUNCH(ba_stats_kernel, (unsigned)div_up64((long long)s->n + s->m, 256), 256, 0, st, s->d);
      COSL_TRY(allreduce(s, s->d_sc + SC_NSUM, 2, ncclMax));
    }
  } else if (s->ns) {  // a trial: Schur complement + dense solve + back substitution for mu, and its cost
    const int nTilesInit = std::max(1, s->plan.nTiles);
    T.begin(s->secSchur, st);
    // also clears the scalars of this trial (|dp|^2, dL, |p|^2, fail, cost, non-finite), the task counters
    // of the solve and the accumulator of the point back-substitution (d_dpb)
    COSL_LAUNCH(ba_prep_kernel, nTilesInit + (unsigned)div_up64((long long)s->n + s->m, 256), 256, 0, st, s->d, dctl,
                mu, r0, s->tl.diagBlk, s->tl.blkCam0, s->tl.order, s->d_cnt, s->td.nCounters + 2 + s->td.nTasks,
                nTilesInit, s->d_Vinv, doStats, s->d_dpb, 3LL * s->n);
    if (doStats) COSL_TRY(allreduce(s, s->d_sc + SC_NSUM, 2, ncclMax));
    if (s->nItems)
      COSL_LAUNCH(ba_schur_pairs_st, div_up(s->nItems, BA_ST_WARPS), 32 * BA_ST_WARPS, BA_ST_SMEM, st, s->d,
                  s->d_items, s->nItems, s->d_entries, s->d_Vinv);
    T.end(st);
    // the one exchange of an LM trial: [rhs | Schur-structure tiles] is contiguous, no packing
    COSL_TRY(allreduce(s, s->d_S, (size_t)s->reduceCount, ncclSum));
    T.begin(s->secSolve, st);  // reduced camera system -> d_x (block padded, permuted)
    COSL_TRY(tile_solve_enqueue(s->tile, s->td, st));
    T.end(st);
    // back substitution + trial cost in two launches (ba_kernels.cuh); V*^-1 is the one the contraction used
    const int nCamBlocks = div_up(6 * s->m, 256);
    T.begin(s->secBack, st);
    COSL_LAUNCH(ba_back_cams_points, nCamBlocks + gN, 256, 0, st, s->d, dctl, s->d_pa, s->d_x, s->d_dpa, s->d_na, mu,
                r0, nCamBlocks, s->d_dpb);
    T.end(st);
    T.begin(s->secCost, st);
    if (s->N + s->n) {  // a problem without points never reaches a trial (|g| = 0 stops it), but is captured
      const unsigned gF = (unsigned)div_up64(s->N + (long long)s->n, 256);
      if (oc)
        COSL_LAUNCH(ba_finish_cost<true>, gF, 256, 0, st, s->d, dctl, s->d_na, s->d_pb, s->d_nb, s->d_dpb, s->d_Vinv, mu);
      else
        COSL_LAUNCH(ba_finish_cost<false>, gF, 256, 0, st, s->d, dctl, s->d_na, s->d_pb, s->d_nb, s->d_dpb, s->d_Vinv,
                    mu);
    }
    T.end(st);
  } else {  // a trial without free cameras
    T.begin(s->secBack, st);
    // (also zeroes the accumulator of the point back-substitution, d_nb)
    COSL_LAUNCH(ba_cam_update,
                std::max(div_up(6 * s->m, 256), (int)std::min<long long>(s->numSM, div_up64(3LL * s->n, 1024))), 256,
                0, st, s->d, dctl, s->d_pa, s->d_x, s->d_dpa, s->d_na, mu, r0, s->d_nb, 3LL * s->n);
    if (s->N) COSL_LAUNCH(ba_back_subst, gN, 256, 0, st, s->d, s->d_dpa, s->d_nb);
    if (s->n)
      COSL_LAUNCH(ba_back_finish, (unsigned)div_up64(s->n, 256), 256, 0, st, s->d, dctl, s->d_pb, s->d_nb, s->d_dpb,
                  mu);
    T.end(st);
    T.begin(s->secCost, st);
    if (s->N) COSL_TRY(launch_cost(s->d, s->d_na, s->d_nb, gN, st));
    T.end(st);
  }
  if (stage == BA_STAGE_ROUND || stage == BA_STAGE_TRIAL) COSL_TRY(allreduce(s, s->d_sc, SC_NSUM, ncclSum));
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// The outlier pass after the loop, at its final parameters: the flags, and their number over all ranks in
// sc[SC_COST] (cleared by the loop's last decision).  The same branch on every rank (options are global).
int enqueue_outliers(cosl_ba_solver* s, cudaStream_t st) {
  if (s->opt.max_err > 0) {
    if (s->N)
      COSL_LAUNCH(ba_residual_kernel<false>, (unsigned)div_up64(s->N, 256), 256, 0, st, s->d, s->d_pa, s->d_pb, 2,
                  s->opt.max_err, s->d_outlier);
    COSL_TRY(allreduce(s, s->d_sc, SC_NSUM, ncclSum));
  } else {
    COSL_CUDA(cudaMemsetAsync(s->d_outlier, 0, (size_t)s->N ? (size_t)s->N : 1, st));
  }
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// fixedTrials > 0: cosl_ba_solver_run_fixed (one round of that many trials)
BaLmParams lm_params(const cosl_ba_solver* s, int fixedTrials) {
  BaLmParams P = {};
  const double* o = s->opt.opts;
  P.tau = o[0];
  P.eps1 = o[1];
  P.eps2 = o[2];
  P.eps3 = o[3];
  P.eps4 = o[4];
  P.rounds = fixedTrials ? 1 : std::max(1, s->opt.outer_iters);
  P.itmax = fixedTrials ? (1 << 30) : s->opt.inner_iters;
  P.ns = s->ns;
  P.hasObs = s->N > 0;
  P.outliers = s->opt.max_err > 0;
  P.fixedTrials = fixedTrials;
  return P;
}

// info[] of a finished loop (include/coslam_b200.h): the levmar fields of its last round, the first round's
// initial cost, the trials of all rounds, the time it took and the outliers of the pass after it
void fill_info(double info[COSL_BA_INFOSZ], const BaCtl& c, double seconds, double nout, bool outliers) {
  if (!info) return;
  for (int k = 0; k < COSL_BA_INFOSZ; ++k) info[k] = 0;
  info[0] = c.first_e0;
  info[1] = c.p_eL2;
  info[2] = c.ginf;
  info[3] = c.dp_L2;
  info[4] = c.maxdiag > 0 ? c.mu / c.maxdiag : 0;
  info[5] = c.itno;
  info[6] = c.stop;
  info[7] = c.nfev;
  info[8] = c.njev;
  info[9] = c.nlss;
  info[10] = c.totalTrials;
  info[11] = seconds;
  info[12] = c.p_eL2;
  info[13] = outliers ? nout : 0.0;
}

// The host driver of the robust loop (run, run_fixed and the handle-less entry points): after each stage the
// scalars it needs are read back and ba_lm_decide picks the next stage, the decisions ba_ctl_step takes on the
// device for submit.  Through the handle (s->loopReq) it stops when the caller asks and keeps the progress
// record.  info[11]: wall time.
int run_host(cosl_ba_solver* s, int fixedTrials, double info[COSL_BA_INFOSZ]) {
  const BaLmParams P = lm_params(s, fixedTrials);
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  const auto t0 = std::chrono::steady_clock::now();
  BaCtl c;
  ba_lm_start(c);
  while (true) {
    COSL_TRY(clear_sc(s, ba_lm_cleared(c, P)));
    if (c.done) break;
    const int stage = c.stage, itno = c.itno;
    const double mu = c.mu, p_eL2 = c.p_eL2;
    COSL_TRY(enqueue_stage(s, s->rq.stream, stage, nullptr, mu, c.statsPending));
    // a linearisation at itno > 0 is decided without its statistics: they arrive with the next trial's
    if (stage != BA_STAGE_LIN) COSL_TRY(read_sc(s));
    ba_lm_decide(c, s->h_sc, P, s->loopReq && s->stopReq.load(std::memory_order_relaxed) == s->loopReq);
    if (c.rated && s->opt.verbose && rank_of(s) == 0)
      std::printf("  [gpu LM %d] mu %.3e cost %.9g -> %.9g dL %.3e\n", itno, mu, p_eL2, s->h_sc[SC_COST],
                  s->h_sc[SC_DL]);
    if (c.copy) {
      std::swap(s->d_pa, s->d_na);
      std::swap(s->d_pb, s->d_nb);
    }
    if (s->loopReq) {
      std::lock_guard<std::mutex> lk(s->hostProgMu);
      BaProgress& g = s->hostProg;
      g.seq0 = g.seq1 = g.seq1 + 1;
      g.req = s->loopReq;
      ba_lm_progress(c, g);
    }
  }
  COSL_TRY(enqueue_outliers(s, s->rq.stream));
  COSL_TRY(read_sc(s));
  const double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  fill_info(info, c, seconds, s->h_sc[SC_COST], P.outliers);
  return COSL_OK;
}

int download(cosl_ba_solver* s, cosl_ba_problem* p) {
  const int m = s->m;
  std::vector<double> pa((size_t)m * 6);
  COSL_CUDA(cudaMemcpyAsync(pa.data(), s->d_pa, sizeof(double) * 6 * m, cudaMemcpyDeviceToHost,
                            s->rq.stream));
  std::vector<double> X((size_t)s->n * 3);
  COSL_CUDA(cudaMemcpyAsync(X.data(), s->d_pb, sizeof(double) * 3 * (size_t)s->n,
                            cudaMemcpyDeviceToHost, s->rq.stream));
  if (p->outlier && s->N)
    COSL_CUDA(cudaMemcpyAsync(p->outlier, s->d_outlier, (size_t)s->N, cudaMemcpyDeviceToHost,
                              s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  for (int j = s->mcon; j < m; ++j) {
    const double* v = &pa[6 * j];
    const double dq[4] = {std::sqrt(1.0 - (v[0] * v[0] + v[1] * v[1] + v[2] * v[2])), v[0], v[1],
                          v[2]};
    double q[4];
    quat_mul(dq, &s->q0[4 * j], q);
    const double nr = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int k = 0; k < 4; ++k) q[k] /= nr;
    quat2mat(q, p->R + 9 * j);
    for (int k = 0; k < 3; ++k) p->t[3 * j + k] = pa[6 * j + 3 + k];
  }
  for (int i = s->ncon; i < s->n; ++i)
    for (int k = 0; k < 3; ++k) p->X[3 * (size_t)i + k] = X[3 * (size_t)i + k];
  return COSL_OK;
}

/* ---------------------------------------------------------------- covariance stage (DESIGN.md 4.6) */
// The selected-inversion plan of the loaded problem and the stage's buffers (arming, or a load while armed:
// never inside run / submit).  Z has the factor's tile layout.
int cov_prepare(cosl_ba_solver* s) {
  const BaPlan& P = s->plan;
  s->sel = ba_make_selinv_plan(P);
  size_t oOps = 0;
  const std::vector<unsigned char> idx = selinv_index(s->sel, &oOps);
  const size_t nb = (size_t)std::max(1, P.nb), n = (size_t)s->n, m = (size_t)s->m;
  COSL_TRY(grow(s, &s->d_covIdx, idx.size()));
  COSL_TRY(grow(s, &s->d_covWgt, (size_t)s->N));
  COSL_TRY(grow(s, &s->d_covZ, (size_t)std::max(1, P.nTiles) * BA_TILE));
  COSL_TRY(grow(s, &s->d_covX, nb * BA_TILE));
  COSL_TRY(grow(s, &s->d_covSdiag, nb * BA_TB));
  COSL_TRY(grow(s, &s->d_covPiv, nb));
  COSL_TRY(grow(s, &s->d_covCnt, nb));
  COSL_TRY(grow(s, &s->d_covT, 6 * n));
  COSL_TRY(grow(s, &s->d_covUnc, n));
  COSL_TRY(grow(s, &s->d_covCam, 36 * m));
  COSL_TRY(grow(s, &s->d_covPt, 9 * n));
  COSL_TRY(grow(s, &s->d_covSc, (size_t)COV_NTOT));
  // from pageable memory: the call returns once the source has been staged
  COSL_CUDA(cudaMemcpyAsync(s->d_covIdx, idx.data(), idx.size(), cudaMemcpyHostToDevice, s->rq.stream));
  BaSelDev& sd = s->sdev;
  sd.L = s->d.tiles;
  sd.Linv = s->d_Linv;
  sd.sdiag = s->d_covSdiag;
  sd.Z = s->d_covZ;
  sd.X = s->d_covX;
  sd.piv = s->d_covPiv;
  sd.diagTile = s->tl.diagTile;
  sd.tasks = reinterpret_cast<const BaSelTask*>(s->d_covIdx);
  sd.ops = reinterpret_cast<const BaSelOp*>(s->d_covIdx + oOps);
  sd.blkRows = s->tl.blkRows;
  sd.cnt = s->d_covCnt;
  s->covReady = true;
  return COSL_OK;
}

// The covariance stage at the resident parameters (d_pa, d_pb), enqueued on st (the solver's stream, or the
// capture of the submitted graph): undamped re-linearisation with Tukey weights at those parameters through
// the LM loop's kernels, Schur contraction, factorisation + selected inversion, camera and point blocks,
// scalars.  Its weights and scalars are its own; the other buffers it writes (W, V, U, S, V^-1, the factor
// work space) are rebuilt by the LM loop before it reads them.
int enqueue_cov(cosl_ba_solver* s, cudaStream_t st) {
  BaDev cd = s->d;
  cd.wgt = s->d_covWgt;
  cd.sc = s->d_covSc;
  BaTileDev td = s->td;
  td.sc = s->d_covSc;
  td.scFail = (int)SC_FAIL;
  td.trace = nullptr;
  const unsigned gN = (unsigned)div_up64(s->N, 256);
  const int n = s->n, m = s->m, nb = std::max(0, s->plan.nb);
  const double var = s->covVar;
  COSL_LAUNCH(ba_cov_begin, (unsigned)std::max<long long>(1, std::min<long long>(1024, div_up64(6LL * n, 256))), 256,
              0, st, s->d_covSc, s->d_covT, 6LL * n, s->d_covCnt, nb);
  if (s->N) {
    if (s->opt.max_err > 0)
      COSL_LAUNCH(ba_residual_kernel<false>, gN, 256, 0, st, cd, s->d_pa, s->d_pb, 1, s->opt.max_err, nullptr);
    else
      COSL_LAUNCH(ba_fill_f64, std::min<unsigned>(gN, 1024), 256, 0, st, s->d_covWgt, s->N, 1.0);
  }
  if (n) COSL_LAUNCH(ba_cov_mask, div_up(n, 256), 256, 0, st, cd, s->d_covUnc);
  const long long nV = 9LL * n + 27LL * m;
  COSL_LAUNCH(ba_fill_f64, (unsigned)std::min<long long>(div_up64(nV, 256), 1024), 256, 0, st, s->d_V, nV, 0.0);
  COSL_TRY(launch_linearize(s, cd, st));
  // mu = 0: S and V^-1 of the undamped system (and the cleared scalars and task counters)
  const int nTilesInit = std::max(1, s->plan.nTiles);
  COSL_LAUNCH(ba_prep_kernel, nTilesInit + (unsigned)div_up64((long long)n + m, 256), 256, 0, st, cd, nullptr, 0.0, 1,
              s->tl.diagBlk, s->tl.blkCam0, s->tl.order, s->d_cnt, s->td.nCounters + 2 + s->td.nTasks, nTilesInit,
              s->d_Vinv, 0, nullptr, 0LL);
  if (s->N) COSL_TRY(launch_cost(cd, s->d_pa, s->d_pb, gN, st));
  if (n) COSL_LAUNCH(ba_cov_vfix, div_up(n, 256), 256, 0, st, s->d_covUnc, s->d_Vinv, n);
  if (s->ns) {
    if (s->nItems)
      COSL_LAUNCH(ba_schur_pairs_st, div_up(s->nItems, BA_ST_WARPS), 32 * BA_ST_WARPS, BA_ST_SMEM, st, cd, s->d_items,
                  s->nItems, s->d_entries, s->d_Vinv);
    COSL_TRY(selinv_launch(s->tile, s->sel, td, s->sdev, st));
  }
  COSL_LAUNCH(ba_cov_cams, div_up(m, 128), 128, 0, st, cd, s->d_pa, s->d_covZ, s->sdev.diagTile, var, s->d_covCam);
  if (s->ns && s->nItems)
    COSL_LAUNCH(ba_cov_pairs, div_up(s->nItems, 4), 128, 0, st, cd, s->d_items, s->nItems, s->d_entries, s->d_covZ,
                s->d_covT);
  if (n) COSL_LAUNCH(ba_cov_points, div_up(n, 256), 256, 0, st, n, s->ncon, s->d_Vinv, s->d_covT, s->d_covUnc, var,
                     s->d_covPt);
  COSL_LAUNCH(ba_cov_end, 1, 32, 0, st, s->d_covSc, s->d_covPiv, nb, s->mf, var);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// run's covariance stage: after the robust loop, on the solver's stream, waited for
int run_cov(cosl_ba_solver* s) {
  COSL_TRY(enqueue_cov(s, s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  s->covValid = true;
  return COSL_OK;
}

/* ---------------------------------------------------------------- submitted robust loop (ba_ctl.cuh) */
// Add a conditional node after the current capture position of `cs`; the capture continues behind it.
int capture_conditional(cudaStream_t cs, cudaGraphConditionalHandle h, cudaGraphConditionalNodeType type,
                        cudaGraph_t* body) {
  cudaStreamCaptureStatus st;
  cudaGraph_t cg = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t nd = 0;
  COSL_CUDA(cudaStreamGetCaptureInfo(cs, &st, nullptr, &cg, &deps, &nd));
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = h;
  np.conditional.type = type;
  np.conditional.size = 1;
  cudaGraphNode_t node;
  COSL_CUDA(cudaGraphAddNode(&node, cg, deps, nd, &np));
  *body = np.conditional.phGraph_out[0];
  COSL_CUDA(cudaStreamUpdateCaptureDependencies(cs, &node, 1, cudaStreamSetCaptureDependencies));
  return COSL_OK;
}

// capture into `g` on cs, leaving an empty node in a body that has no kernel (e.g. no observations)
template <typename F>
int capture_into(cudaStream_t cs, cudaGraph_t g, F&& enqueue) {
  COSL_CUDA(cudaStreamBeginCaptureToGraph(cs, g, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaGraph_t out = nullptr;
  const cudaError_t e = cudaStreamEndCapture(cs, &out);
  COSL_TRY(rc);
  if (e != cudaSuccess) return set_error(COSL_E_CUDA, "graph capture: %s", cudaGetErrorString(e));
  size_t nn = 0;
  COSL_CUDA(cudaGraphGetNodes(g, nullptr, &nn));
  if (nn == 0) {
    cudaGraphNode_t empty;
    COSL_CUDA(cudaGraphAddEmptyNode(&empty, g, nullptr, 0));
  }
  return COSL_OK;
}

// The graph of the submitted robust loop:
//   ba_ctl_init -> WHILE(loop) { IF(round) -> IF(lin0) -> IF(lin) -> IF(trial) -> ba_ctl_step -> ba_ctl_accept }
//   -> outlier pass -> covariance stage (when armed)
int build_graph_nodes(cosl_ba_solver* s, cudaStream_t cs, cudaGraph_t g) {
  BaCtlParams P = {};
  P.lm = lm_params(s, 0);
  P.link = s->d_link;
  COSL_CUDA(cudaGraphConditionalHandleCreate(&P.hLoop, g, 1, cudaGraphCondAssignDefault));
  for (int k = 0; k < BA_NSTAGES; ++k)
    COSL_CUDA(cudaGraphConditionalHandleCreate(&P.hStage[k], g, k == BA_STAGE_ROUND ? 1 : 0, cudaGraphCondAssignDefault));
  cudaGraph_t loopBody = nullptr, stageBody[BA_NSTAGES] = {};
  COSL_TRY(capture_into(cs, g, [&]() -> int {
    COSL_LAUNCH(ba_ctl_init, 1, 32, 0, cs, s->d_ctl, s->d_sc, P.lm);
    COSL_TRY(capture_conditional(cs, P.hLoop, cudaGraphCondTypeWhile, &loopBody));
    COSL_TRY(enqueue_outliers(s, cs));
    if (s->covVar > 0) COSL_TRY(enqueue_cov(s, cs));
    COSL_CUDA(cudaGetLastError());
    return COSL_OK;
  }));
  COSL_TRY(capture_into(cs, loopBody, [&]() -> int {
    for (int k = 0; k < BA_NSTAGES; ++k) COSL_TRY(capture_conditional(cs, P.hStage[k], cudaGraphCondTypeIf, &stageBody[k]));
    COSL_LAUNCH(ba_ctl_step, 1, 32, 0, cs, s->d_ctl, s->d_sc, P);
    const long long nA = 6LL * s->m, nB = 3LL * s->n;
    COSL_LAUNCH(ba_ctl_accept, (unsigned)std::max<long long>(1, std::min<long long>(4LL * s->numSM, div_up64(nA + nB, 256))),
                256, 0, cs, s->d_ctl, s->d_pa, s->d_na, nA, s->d_pb, s->d_nb, nB);
    COSL_CUDA(cudaGetLastError());
    return COSL_OK;
  }));
  // the trial kernels read mu and doStats from the control block; a submitted loop always wants the statistics
  for (int k = 0; k < BA_NSTAGES; ++k)
    COSL_TRY(capture_into(cs, stageBody[k], [&]() { return enqueue_stage(s, cs, k, s->d_ctl, 0.0, 1); }));
  return COSL_OK;
}

// (Re)builds the graph for the loaded problem.  An existing executable graph is updated in place when
// the driver accepts the new topology, and instantiated afresh otherwise; neither waits for the device
// (an executable graph that is destroyed while it runs is released when it completes).
int build_graph(cosl_ba_solver* s) {
  const double t0 = now_s();
  int drv = 0;
  COSL_CUDA(cudaDriverGetVersion(&drv));
  if (drv < 12040)
    return set_error(COSL_E_CUDA,
                     "cosl_ba_solver_submit: the CUDA driver (version %d) has no conditional graph nodes (12.4 or "
                     "newer is needed)", drv);
  COSL_TRY(grow(s, &s->d_ctl, 1));
  cudaStream_t cs = nullptr;
  COSL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaGraphCreate(&g, 0);
  const bool timing = s->timer.enabled;
  s->timer.enabled = false;  // the section timers time the host driver's stages, not a capture
  int rc = e == cudaSuccess ? build_graph_nodes(s, cs, g) : set_error(COSL_E_CUDA, "cudaGraphCreate: %s", cudaGetErrorString(e));
  s->timer.enabled = timing;
  const double t1 = now_s();
  bool updated = false;
  if (rc == COSL_OK && s->graphExec) {
    cudaGraphExecUpdateResultInfo ui;
    updated = cudaGraphExecUpdate(s->graphExec, g, &ui) == cudaSuccess;
    if (!updated) {
      cudaGetLastError();  // a refused update is not an error: instantiate instead
      cudaGraphExecDestroy(s->graphExec);
      s->graphExec = nullptr;
    }
  }
  if (rc == COSL_OK && !updated) {
    e = cudaGraphInstantiate(&s->graphExec, g, 0);
    if (e != cudaSuccess) {
      s->graphExec = nullptr;
      rc = set_error(COSL_E_CUDA, "cosl_ba_solver_submit: graph instantiation failed: %s", cudaGetErrorString(e));
    }
  }
  if (g) cudaGraphDestroy(g);
  cudaStreamDestroy(cs);
  if (rc != COSL_OK) return rc;
  if (ba_timing())
    std::fprintf(stderr, "[ba timing] graph: capture %.2f ms, %s %.2f ms\n", 1e3 * (t1 - t0),
                 updated ? "exec update" : "instantiate", 1e3 * (now_s() - t1));
  s->graphStale = false;
  s->graphPa = s->d_pa;
  s->graphNa = s->d_na;
  s->graphPb = s->d_pb;
  s->graphNb = s->d_nb;
  s->graphCovVar = s->covVar;
  s->graphObsL = s->d.obsL;
  return COSL_OK;
}

/* ---------------------------------------------------------------- debug entry points */
// The device side of a debug solve of the dense SPD system S (6 mf x 6 mf) in one block from `tmp`, enqueued on
// `st`: the lower triangle of S placed as load_problem's pair_dst places the Schur blocks (the camera later in
// the elimination order owns the rows; fill and padding stay zero), b or zeros as the block-padded rhs, the
// plan's lists, the solve's work buffers (scratch tiles and their rhs parts start as NaN: their first update must
// overwrite them), zeroed counters and failure flag (td.sc[0]), and `extraBytes` more at *extra.
int debug_tile_setup(const BaPlan& P, const TileLaunch& L, int mf, const uint8_t* adj, const double* S,
                     const double* b, size_t extraBytes, TmpDeviceBufs& tmp, cudaStream_t st, BaTileDev& td,
                     TileLists& tl, unsigned char** extra) {
  const int nb = P.nb;
  const size_t ns = 6 * (size_t)mf, nScratch = (size_t)std::max(1, P.nScratch);
  const size_t nCnt = (size_t)P.nCounters + 2 + L.order.size();
  std::vector<double> hTiles((size_t)P.nTiles * BA_TILE, 0.0), hRhs((size_t)nb * BA_TB, 0.0);
  for (int a = 0; a < mf; ++a)
    for (int c = 0; c < mf; ++c) {
      if (a != c && !adj[(size_t)a * mf + c] && !adj[(size_t)c * mf + a]) continue;
      const int bA = P.camBlk[a], bC = P.camBlk[c];
      if (bA < bC || (bA == bC && P.camOff[a] < P.camOff[c])) continue;
      double* T = &hTiles[(size_t)P.tileIdx[(size_t)bA * nb + bC] * BA_TILE];
      for (int r = 0; r < 6; ++r)
        for (int q = 0; q < 6; ++q) {
          if (a == c && q > r) continue;
          const size_t i = 6 * (size_t)a + r, j = 6 * (size_t)c + q;
          T[(size_t)(P.camOff[c] + q) * BA_TB + P.camOff[a] + r] = i >= j ? S[i * ns + j] : S[j * ns + i];
        }
    }
  if (b)
    for (int a = 0; a < mf; ++a)
      for (int r = 0; r < 6; ++r) hRhs[(size_t)P.camBlk[a] * BA_TB + P.camOff[a] + r] = b[6 * a + r];
  const TileImage img = tile_image(P, L);
  SlabLayout W;
  const size_t oImg = W.take(img.bytes), oRhs = W.take(8 * hRhs.size());
  const size_t oTiles = W.take(8 * ((size_t)P.nTiles + P.nScratch) * BA_TILE), oRhsS = W.take(8 * nScratch * BA_TB);
  const size_t oLinv = W.take(8 * (size_t)nb * BA_TILE), oY = W.take(8 * hRhs.size()), oX = W.take(8 * hRhs.size());
  const size_t oSc = W.take(8), oCnt = W.take(4 * nCnt), oExtra = W.take(extraBytes);
  unsigned char* d = nullptr;
  COSL_TRY(tmp.alloc(&d, W.bytes));
  tl = tile_lists(img, d + oImg);
  td = tile_dev(P, L, tl);
  td.rhs = reinterpret_cast<double*>(d + oRhs);
  td.tiles = reinterpret_cast<double*>(d + oTiles);
  td.rhsS = reinterpret_cast<double*>(d + oRhsS);
  td.Linv = reinterpret_cast<double*>(d + oLinv);
  td.y = reinterpret_cast<double*>(d + oY);
  td.x = reinterpret_cast<double*>(d + oX);
  td.cnt = reinterpret_cast<int*>(d + oCnt);
  td.sc = reinterpret_cast<double*>(d + oSc);
  td.scFail = 0;
  *extra = d + oExtra;
  std::vector<unsigned char> hImg(img.bytes);
  tile_image_write(P, L, img, hImg.data());
  COSL_CUDA(cudaMemcpyAsync(d + oImg, hImg.data(), hImg.size(), cudaMemcpyHostToDevice, st));
  COSL_CUDA(cudaMemcpyAsync(td.rhs, hRhs.data(), 8 * hRhs.size(), cudaMemcpyHostToDevice, st));
  COSL_CUDA(cudaMemcpyAsync(td.tiles, hTiles.data(), 8 * hTiles.size(), cudaMemcpyHostToDevice, st));
  COSL_CUDA(cudaMemsetAsync(td.tiles + hTiles.size(), 0xff, 8 * (size_t)P.nScratch * BA_TILE, st));
  COSL_CUDA(cudaMemsetAsync(td.rhsS, 0xff, 8 * nScratch * BA_TB, st));
  COSL_CUDA(cudaMemsetAsync(td.cnt, 0, 4 * nCnt, st));
  COSL_CUDA(cudaMemsetAsync(td.sc, 0, 8, st));
  return COSL_OK;
}

}  // namespace

/* ================================================================ C-ABI */
extern "C" {

void cosl_ba_options_default(cosl_ba_options* o) {
  if (!o) return;
  o->max_err = 6.0;  // RobustBundleRTSParameter defaults (app/SL_CoSLAMRobustBA.h:33-38)
  o->outer_iters = 5;
  o->inner_iters = 10;
  o->opts[0] = 1e-3 * 1e-4;  // app/SL_CoSLAMBA.cpp:323-328
  o->opts[1] = 1e-12;
  o->opts[2] = 1e-12;
  o->opts[3] = 0;
  o->opts[4] = 1e-16;
  o->device = 0;
  o->verbose = 0;
}

int cosl_nccl_unique_id(uint8_t id[128]) {
  if (!id) return set_error(COSL_E_INVALID, "null id");
  if (!nccl().ok) return set_error(COSL_E_NCCL, "libnccl.so.2 could not be loaded");
  ncclUniqueId u;
  const int rc = nccl().GetUniqueId(&u);
  if (rc != 0) return set_error(COSL_E_NCCL, "ncclGetUniqueId failed (%d)", rc);
  std::memcpy(id, u.internal, 128);
  return COSL_OK;
}

int cosl_ba_comm_create(const uint8_t id[128], int rank, int nranks, int device,
                        cosl_ba_comm** out) {
  if (!id || !out || rank < 0 || rank >= nranks)
    return set_error(COSL_E_INVALID, "cosl_ba_comm_create: bad argument");
  *out = nullptr;
  if (!nccl().ok) return set_error(COSL_E_NCCL, "libnccl.so.2 could not be loaded");
  COSL_CUDA(cudaSetDevice(device));
  cosl_ba_comm* c = new (std::nothrow) cosl_ba_comm();
  if (!c) return set_error(COSL_E_NOMEM, "host allocation failed");
  ncclUniqueId u;
  std::memcpy(u.internal, id, 128);
  const int rc = nccl().CommInitRank(&c->comm, nranks, u, rank);
  if (rc != 0) {
    delete c;
    return set_error(COSL_E_NCCL, "ncclCommInitRank: %s",
                     nccl().GetErrorString ? nccl().GetErrorString(rc) : "?");
  }
  c->rank = rank;
  c->nranks = nranks;
  c->device = device;
  *out = c;
  return COSL_OK;
}

int cosl_ba_comm_destroy(cosl_ba_comm* c) {
  if (!c) return COSL_OK;
  if (c->comm) nccl().CommDestroy(c->comm);
  delete c;
  return COSL_OK;
}

int cosl_ba_solver_create(const cosl_ba_problem* prob, const cosl_ba_options* opt,
                          cosl_ba_comm* comm, cosl_ba_solver** out) {
  if (!prob || !opt || !out) return set_error(COSL_E_INVALID, "null argument");
  *out = nullptr;
  COSL_TRY(check_problem(prob, "cosl_ba_solver_create"));
  const double t0 = now_s();
  BaIndex x;
  COSL_TRY(index_problem(prob, x));
  if (ba_timing()) std::fprintf(stderr, "[ba timing] index %.2f ms\n", 1e3 * (now_s() - t0));
  COSL_TRY(check_device(opt->device));
  COSL_CUDA(cudaSetDevice(opt->device));
  cosl_ba_solver* s = nullptr;
  int rc = make_handle(opt, comm, &s);
  if (rc == COSL_OK) rc = load_problem(s, prob, x);
  if (rc == COSL_OK && cudaStreamSynchronize(s->rq.stream) != cudaSuccess)
    rc = set_error(COSL_E_CUDA, "cosl_ba_solver_create: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc != COSL_OK) {
    free_solver(s);
    return rc;
  }
  *out = s;
  return COSL_OK;
}

#define BA_ENTER(s)                                               \
  if (!(s)) return set_error(COSL_E_INVALID, "null solver handle"); \
  COSL_CUDA(cudaSetDevice((s)->device));

int cosl_ba_solver_reset(cosl_ba_solver* s, const cosl_ba_problem* prob) {
  BA_ENTER(s)
  COSL_TRY(s->rq.idle("cosl_ba_solver_reset"));
  if (!prob || prob->m != s->m || prob->n != s->n)
    return set_error(COSL_E_INVALID, "cosl_ba_solver_reset: problem shape changed");
  s->timer.reset();
  s->covValid = false;
  COSL_CUDA(cudaEventSynchronize(s->evStaged));
  COSL_TRY(upload_params(s, prob));
  COSL_CUDA(cudaEventRecord(s->evStaged, s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  return COSL_OK;
}

int cosl_ba_solver_load(cosl_ba_solver* s, const cosl_ba_problem* prob) {
  BA_ENTER(s)
  if (multi(s))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_load: a multi-rank solver plans over all ranks; create one");
  COSL_TRY(s->rq.idle("cosl_ba_solver_load"));
  COSL_TRY(check_problem(prob, "cosl_ba_solver_load"));
  BaIndex x;
  COSL_TRY(index_problem(prob, x));
  s->timer.reset();
  return load_problem(s, prob, x);
}

int cosl_ba_solver_run(cosl_ba_solver* s, double info[COSL_BA_INFOSZ]) {
  BA_ENTER(s)
  COSL_TRY(s->rq.idle("cosl_ba_solver_run"));
  s->loopReq = s->reqNo.load() + 1;
  s->reqKind.store(1);
  s->hostRunning.store(1);
  s->reqNo.store(s->loopReq);
  s->covValid = false;
  int rc = run_host(s, 0, info);
  if (rc == COSL_OK && s->covVar > 0) rc = run_cov(s);
  s->hostRunning.store(0);
  s->loopReq = 0;
  return rc;
}

int cosl_ba_solver_run_fixed(cosl_ba_solver* s, int trials, double info[COSL_BA_INFOSZ]) {
  BA_ENTER(s)
  COSL_TRY(s->rq.idle("cosl_ba_solver_run_fixed"));
  s->covValid = false;
  return run_host(s, trials < 1 ? 1 : trials, info);
}

int cosl_ba_solver_download(cosl_ba_solver* s, cosl_ba_problem* prob) {
  BA_ENTER(s)
  COSL_TRY(s->rq.idle("cosl_ba_solver_download"));
  if (!prob || prob->m != s->m || prob->n != s->n)
    return set_error(COSL_E_INVALID, "cosl_ba_solver_download: problem shape changed");
  return download(s, prob);
}

int cosl_ba_solver_submit(cosl_ba_solver* s) {
  BA_ENTER(s)
  if (multi(s))
    return set_error(COSL_E_INVALID,
                     "cosl_ba_solver_submit: a multi-rank solver exchanges over NCCL between host-ordered steps; "
                     "use cosl_ba_solver_run");
  COSL_TRY(s->rq.idle("cosl_ba_solver_submit"));
  // the synchronous path swaps d_pa / d_na (d_pb / d_nb) on every accepted trial; the graph holds pointers
  if (!s->graphExec || s->graphStale || s->graphPa != s->d_pa || s->graphNa != s->d_na || s->graphPb != s->d_pb ||
      s->graphNb != s->d_nb || s->graphCovVar != s->covVar || s->graphObsL != s->d.obsL)
    COSL_TRY(build_graph(s));
  // the request number goes to the device ahead of the graph, on the solver's stream: a stop made before the
  // graph starts names it too (the pinned source is not rewritten before this request is collected)
  const unsigned long long req = s->reqNo.load() + 1;
  *reinterpret_cast<volatile unsigned long long*>(s->h_sc + BA_PIN_REQ) = req;
  COSL_CUDA(cudaMemcpyAsync(&s->d_link->req, s->h_sc + BA_PIN_REQ, sizeof(req), cudaMemcpyHostToDevice,
                            s->rq.stream));
  s->reqKind.store(2);
  s->reqNo.store(req);
  const int rc = s->rq.submit("cosl_ba_solver_submit", [&]() {
    COSL_CUDA(cudaGraphLaunch(s->graphExec, s->rq.stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return (int)COSL_OK;
  });
  if (rc == COSL_OK) s->submitted.store(1);
  s->covValid = rc == COSL_OK && s->covVar > 0;  // readable once collected
  return rc;
}

int cosl_ba_solver_query(cosl_ba_solver* s, int* done) {
  BA_ENTER(s)
  if (!done) return set_error(COSL_E_INVALID, "cosl_ba_solver_query: null argument");
  COSL_TRY(s->rq.pending("cosl_ba_solver_query"));
  return s->rq.query(done);
}

int cosl_ba_solver_collect(cosl_ba_solver* s, double info[COSL_BA_INFOSZ]) {
  BA_ENTER(s)
  COSL_TRY(s->rq.pending("cosl_ba_solver_collect"));
  double ms = 0;
  const int waited = s->rq.wait(&ms);
  s->submitted.store(0);
  if (waited != COSL_OK) s->covValid = false;
  COSL_TRY(waited);
  BaCtl c;
  double nout = 0;
  COSL_CUDA(cudaMemcpyAsync(&c, s->d_ctl, sizeof(c), cudaMemcpyDeviceToHost, s->rq.stream));
  COSL_CUDA(cudaMemcpyAsync(&nout, s->d_sc + SC_COST, sizeof(double), cudaMemcpyDeviceToHost, s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  fill_info(info, c, 1e-3 * ms, nout, s->opt.max_err > 0);
  return COSL_OK;
}

int cosl_ba_solver_stop(cosl_ba_solver* s) {
  BA_ENTER(s)
  if (multi(s))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_stop: each rank of a multi-rank solver would stop at a "
                     "different trial");
  std::lock_guard<std::mutex> lk(s->sideMu);
  const unsigned long long req = s->reqNo.load();
  s->stopReq.store(req);  // the host loop's stop word
  if (!req) return COSL_OK;
  // the submitted loop's: a copy on the side stream, never behind the solver's stream.  A copy still queued
  // from an earlier stop reads the newer number, which names a request that was asked to stop as well.
  *reinterpret_cast<volatile unsigned long long*>(s->h_sc + BA_PIN_STOP) = req;
  COSL_CUDA(cudaMemcpyAsync(&s->d_link->stop, s->h_sc + BA_PIN_STOP, sizeof(req), cudaMemcpyHostToDevice,
                            s->sideStream));
  return COSL_OK;
}

int cosl_ba_solver_progress(cosl_ba_solver* s, double out[8]) {
  BA_ENTER(s)
  if (!out) return set_error(COSL_E_INVALID, "cosl_ba_solver_progress: null argument");
  const int kind = s->reqKind.load();
  const unsigned long long req = s->reqNo.load();
  BaProgress g = {};
  int running = 0;
  if (kind == 1) {
    std::lock_guard<std::mutex> lk(s->hostProgMu);
    g = s->hostProg;
    running = s->hostRunning.load();
  } else if (kind == 2) {
    if (s->submitted.load()) {
      const cudaError_t q = cudaEventQuery(s->rq.evDone);
      if (q != cudaSuccess && q != cudaErrorNotReady)
        return set_error(COSL_E_CUDA, "cosl_ba_solver_progress: %s", cudaGetErrorString(q));
      running = q == cudaErrorNotReady;
    }
    // two copies of the record, one after the other: taken when both agree and neither raced a write
    std::lock_guard<std::mutex> lk(s->sideMu);
    BaProgress* h = reinterpret_cast<BaProgress*>(s->h_sc + BA_PIN_PROG);
    for (int attempt = 0;; ++attempt) {
      COSL_CUDA(cudaMemcpyAsync(h, &s->d_link->prog, sizeof(BaProgress), cudaMemcpyDeviceToHost,
                                s->sideStream));
      COSL_CUDA(cudaMemcpyAsync(h + 1, &s->d_link->prog, sizeof(BaProgress), cudaMemcpyDeviceToHost,
                                s->sideStream));
      COSL_CUDA(cudaStreamSynchronize(s->sideStream));
      if (h[0].seq0 == h[0].seq1 && !std::memcmp(&h[0], &h[1], sizeof(BaProgress))) break;
      if (attempt == 1000)
        return set_error(COSL_E_CUDA, "cosl_ba_solver_progress: no consistent copy of the progress record");
    }
    g = h[0];
  }
  for (int k = 0; k < 8; ++k) out[k] = 0.0;
  out[0] = running;
  if (kind && g.req == req) {  // otherwise the request has not reached its first decision
    out[1] = g.round;
    out[2] = g.itno;
    out[3] = g.trials;
    out[4] = g.p_eL2;
    out[5] = g.init_eL2;
    out[6] = g.mu;
  }
  out[7] = (req && s->stopReq.load() == req) ? 1.0 : 0.0;
  return COSL_OK;
}

int cosl_ba_solver_set_covariance(cosl_ba_solver* s, double pixel_var) {
  BA_ENTER(s)
  if (multi(s))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_set_covariance: the multi-rank solver has no covariance stage");
  if (!(pixel_var >= 0.0) || !std::isfinite(pixel_var))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_set_covariance: pixel_var must be finite and >= 0");
  COSL_TRY(s->rq.idle("cosl_ba_solver_set_covariance"));
  if (pixel_var > 0 && !s->covReady) COSL_TRY(cov_prepare(s));
  s->covVar = pixel_var;
  return COSL_OK;
}

int cosl_ba_solver_set_obs_cov(cosl_ba_solver* s, const double* covx) {
  BA_ENTER(s)
  if (multi(s))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_set_obs_cov: a multi-rank solver has no measurement covariances");
  COSL_TRY(s->rq.idle("cosl_ba_solver_set_obs_cov"));
  if (!covx) return set_obs_cov(s, nullptr);
  std::vector<double> L;
  COSL_TRY(check_obs_cov(covx, s->N, L, "cosl_ba_solver_set_obs_cov"));
  return set_obs_cov(s, &L);
}

int cosl_ba_solver_download_covariance(cosl_ba_solver* s, double* camCov, double* ptCov, double out[8]) {
  BA_ENTER(s)
  COSL_TRY(s->rq.idle("cosl_ba_solver_download_covariance"));
  if (!s->covValid)
    return set_error(COSL_E_STATE, "cosl_ba_solver_download_covariance: no covariance for the resident parameters "
                     "(no armed run or collect since the last create, load, reset, run_fixed or unarmed BA)");
  double sc[COV_NTOT];
  COSL_CUDA(cudaMemcpyAsync(sc, s->d_covSc, sizeof(sc), cudaMemcpyDeviceToHost, s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  if (sc[COV_SING] != 0.0)
    return set_error(COSL_E_NUMERIC,
                     "cosl_ba_solver_download_covariance: the information matrix is singular in the gauge (%s; "
                     "smallest relative pivot %.3e, threshold %.0e): fix cameras or points, or drop free cameras "
                     "without weighted observations",
                     sc[SC_FAIL] != 0.0 ? "pivot break-down" : "small pivot", sc[COV_OUT + 5], BA_COV_MIN_PIVOT);
  if (camCov && s->m)
    COSL_CUDA(cudaMemcpyAsync(camCov, s->d_covCam, sizeof(double) * 36 * (size_t)s->m, cudaMemcpyDeviceToHost,
                              s->rq.stream));
  if (ptCov && s->n)
    COSL_CUDA(cudaMemcpyAsync(ptCov, s->d_covPt, sizeof(double) * 9 * (size_t)s->n, cudaMemcpyDeviceToHost,
                              s->rq.stream));
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  if (out)
    for (int k = 0; k < 8; ++k) out[k] = sc[COV_OUT + k];
  return COSL_OK;
}

int cosl_ba_solver_destroy(cosl_ba_solver* s) {
  free_solver(s);  // waits for a submitted solve that is still in flight
  return COSL_OK;
}

void* cosl_ba_solver_stream(cosl_ba_solver* s) { return s ? (void*)s->rq.stream : nullptr; }

int cosl_ba_solver_stats(cosl_ba_solver* s, double out[8]) {
  if (!s || !out) return set_error(COSL_E_INVALID, "cosl_ba_solver_stats: null argument");
  for (int k = 0; k < 8; ++k) out[k] = 0.0;
  out[0] = (double)s->ns;
  out[1] = (double)s->reduceCount;
  out[2] = 0.5 * s->factorFlops;
  out[5] = (double)s->plan.nb;
  out[6] = (double)s->plan.nTiles;
  out[7] = (double)s->plan.tasks.size();
  out[3] = (double)s->nEntries;
  out[4] = (double)s->nItems;
  return COSL_OK;
}

int cosl_ba_solver_plan_info(cosl_ba_solver* s, int out[8]) {
  if (!s || !out) return set_error(COSL_E_INVALID, "cosl_ba_solver_plan_info: null argument");
  out[0] = s->plan.nb;
  out[1] = s->plan.nTilesOrig;
  out[2] = s->plan.nTiles;
  out[3] = (int)s->plan.tasks.size();
  out[4] = s->plan.ndDepth;
  out[5] = s->plan.criticalPathTasks;
  out[6] = s->tile.grid;
  out[7] = s->tile.two ? 1 : 0;
  return COSL_OK;
}

// diagnostic: per-task timeline of the LAST persistent solve launch.  enable -> run -> get.
// out: [nTasks][8] = sm id, globaltimer ns at ticket / operands ready / done, 4 phase stamps; meta: [nTasks][3] =
// task type, pivot block k, row block i.
int cosl_ba_solver_trace(cosl_ba_solver* s, int enable, uint64_t* out, int32_t* meta, int cap) {
  BA_ENTER(s)
  const int nt = (int)s->plan.tasks.size();
  if (enable) {
    COSL_TRY(grow(s, &s->d_trace, (size_t)std::max(1, nt) * 8));
    COSL_CUDA(cudaMemsetAsync(s->d_trace, 0, sizeof(unsigned long long) * 8 * std::max(1, nt), s->rq.stream));
    s->td.trace = s->d_trace;
    return nt;
  }
  if (out && s->d_trace) {
    const int n = std::min(cap, nt);
    COSL_CUDA(cudaMemcpyAsync(out, s->d_trace, sizeof(uint64_t) * 8 * n, cudaMemcpyDeviceToHost, s->rq.stream));
    COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
    if (meta)
      for (int t = 0; t < n; ++t) {
        meta[3 * t] = s->tile.order[t].type;
        meta[3 * t + 1] = s->tile.order[t].k;
        meta[3 * t + 2] = s->tile.order[t].i;
      }
  }
  s->td.trace = nullptr;
  return nt;
}

// diagnostic: the task list of the solve plan, 16 ints per task (BaTask of ba_plan.h), and the
// BACKWARD / SUM wait lists flattened as (counter index, required value) pairs in `lists`, with
// tasks[.].l0/l1 of those two task types rewritten to index into it.  Returns the task count.
int cosl_ba_solver_tasks(cosl_ba_solver* s, int32_t* tasks, int cap, int32_t* lists, int listCap) {
  if (!s) return set_error(COSL_E_INVALID, "null solver handle");
  const BaPlan& P = s->plan;
  const int nt = (int)P.tasks.size();
  int nl = 0;
  for (int t = 0; t < nt && t < cap; ++t) {
    BaTask k = s->tile.order[t];
    if (k.type == BA_T_BWD || k.type == BA_T_SUM) {
      const int l0 = nl;
      for (int e = k.l0; e < k.l1; ++e) {
        if (lists && nl < listCap) {
          lists[2 * nl] = (k.type == BA_T_BWD) ? P.nTiles + P.nScratch + P.bwdList[e].blk : P.sumList[e].tile;
          lists[2 * nl + 1] = (k.type == BA_T_BWD) ? 1 : P.sumList[e].count;
        }
        ++nl;
      }
      k.l0 = l0;
      k.l1 = nl;
    }
    if (tasks) std::memcpy(tasks + 16 * (size_t)t, &k, sizeof(BaTask));
  }
  return nt;
}

// diagnostic: one solve of a dense SPD system with the reduced-camera-system solve of the BA, from the
// plan to the unpermuted solution, so that the tile kernels can be checked against a dense reference
int cosl_ba_debug_tile_solve(int mf, const uint8_t* adj, int nd_depth, const double* S, const double* b,
                             double* x, int* fail, int out[8]) {
  if (mf < 1 || !adj || !S || !b || !x || !fail || !out)
    return set_error(COSL_E_INVALID, "cosl_ba_debug_tile_solve: bad argument");
  const BaPlan P = ba_make_plan(mf, std::vector<uint8_t>(adj, adj + (size_t)mf * mf), nd_depth);
  if (P.nb <= 0) return set_error(COSL_E_INVALID, "cosl_ba_debug_tile_solve: planning failed");
  TileLaunch L = tile_launch_plan(P);
  COSL_TRY(tile_launch_device(L));
  cudaStream_t s = cudaStreamPerThread;
  TmpDeviceBufs tmp(s);
  BaTileDev td;
  TileLists tl;
  unsigned char* extra = nullptr;
  COSL_TRY(debug_tile_setup(P, L, mf, adj, S, b, 0, tmp, s, td, tl, &extra));
  COSL_TRY(tile_solve_enqueue(L, td, s));
  std::vector<double> hX((size_t)P.nb * BA_TB);
  double hFail = 0.0;
  COSL_CUDA(cudaMemcpyAsync(hX.data(), td.x, 8 * hX.size(), cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaMemcpyAsync(&hFail, td.sc, 8, cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaStreamSynchronize(s));
  for (int a = 0; a < mf; ++a)
    for (int r = 0; r < 6; ++r) x[6 * a + r] = hX[(size_t)P.camBlk[a] * BA_TB + P.camOff[a] + r];
  *fail = hFail != 0.0 ? 1 : 0;
  out[0] = P.nb;
  out[1] = P.nTilesOrig;
  out[2] = P.nTiles;
  out[3] = (int)P.tasks.size();
  out[4] = P.ndDepth;
  out[5] = P.criticalPathTasks;
  out[6] = L.two ? 1 : L.grid;
  out[7] = L.two ? 1 : 0;
  return COSL_OK;
}

// diagnostic: Z = S^-1 on the tile pattern with the covariance stage's factorisation and selected inversion
int cosl_ba_debug_tile_selinv(int mf, const uint8_t* adj, int nd_depth, const double* S, double* Z, int* fail,
                              int out[8]) {
  if (mf < 1 || !adj || !S || !Z || !fail || !out)
    return set_error(COSL_E_INVALID, "cosl_ba_debug_tile_selinv: bad argument");
  const BaPlan P = ba_make_plan(mf, std::vector<uint8_t>(adj, adj + (size_t)mf * mf), nd_depth);
  if (P.nb <= 0) return set_error(COSL_E_INVALID, "cosl_ba_debug_tile_selinv: planning failed");
  const BaSelPlan SP = ba_make_selinv_plan(P);
  TileLaunch L = tile_launch_plan(P);
  COSL_TRY(tile_launch_device(L));
  const int nb = P.nb;
  const size_t ns = 6 * (size_t)mf;
  size_t oOps = 0;
  const std::vector<unsigned char> idx = selinv_index(SP, &oOps);
  // the stage's buffers: [plan | Z | X | sdiag | piv | cnt]
  SlabLayout E;
  const size_t oIdx = E.take(idx.size()), oZ = E.take(8 * (size_t)P.nTiles * BA_TILE);
  const size_t oXk = E.take(8 * (size_t)nb * BA_TILE), oSdiag = E.take(8 * (size_t)nb * BA_TB);
  const size_t oPiv = E.take(8 * (size_t)nb), oCnt = E.take(4 * (size_t)nb);
  cudaStream_t s = cudaStreamPerThread;
  TmpDeviceBufs tmp(s);
  BaTileDev td;
  TileLists tl;
  unsigned char* e = nullptr;
  COSL_TRY(debug_tile_setup(P, L, mf, adj, S, nullptr, E.bytes, tmp, s, td, tl, &e));
  BaSelDev sd = {};
  sd.L = td.tiles;
  sd.Linv = td.Linv;
  sd.sdiag = reinterpret_cast<double*>(e + oSdiag);
  sd.Z = reinterpret_cast<double*>(e + oZ);
  sd.X = reinterpret_cast<double*>(e + oXk);
  sd.piv = reinterpret_cast<double*>(e + oPiv);
  sd.diagTile = tl.diagTile;
  sd.tasks = reinterpret_cast<const BaSelTask*>(e + oIdx);
  sd.ops = reinterpret_cast<const BaSelOp*>(e + oIdx + oOps);
  sd.blkRows = tl.blkRows;
  sd.cnt = reinterpret_cast<int*>(e + oCnt);
  COSL_CUDA(cudaMemcpyAsync(e + oIdx, idx.data(), idx.size(), cudaMemcpyHostToDevice, s));
  COSL_CUDA(cudaMemsetAsync(sd.cnt, 0, 4 * (size_t)nb, s));
  COSL_TRY(selinv_launch(L, SP, td, sd, s));
  std::vector<double> hZ((size_t)P.nTiles * BA_TILE), hPiv(nb);
  double hFail = 0.0;
  COSL_CUDA(cudaMemcpyAsync(hZ.data(), sd.Z, 8 * hZ.size(), cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaMemcpyAsync(hPiv.data(), sd.piv, 8 * (size_t)nb, cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaMemcpyAsync(&hFail, td.sc, 8, cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaStreamSynchronize(s));
  double minPiv = 1e300;
  for (double v : hPiv) minPiv = std::min(minPiv, v);
  *fail = (hFail != 0.0 || !(minPiv >= BA_COV_MIN_PIVOT)) ? 1 : 0;
  // the lower camera blocks (a >= c) whose tile is in the pattern
  std::memset(Z, 0, sizeof(double) * ns * ns);
  for (int a = 0; a < mf; ++a)
    for (int c = 0; c <= a; ++c) {
      const int bA = P.camBlk[a], bC = P.camBlk[c];
      const int t = bA >= bC ? P.tileIdx[(size_t)bA * nb + bC] : P.tileIdx[(size_t)bC * nb + bA];
      if (t < 0) continue;
      const double* T = &hZ[(size_t)t * BA_TILE];
      for (int r = 0; r < 6; ++r)
        for (int q = 0; q < 6; ++q) {
          const int ra = P.camOff[a] + r, qc = P.camOff[c] + q;
          // element (row of a, column of c) of the lower tile: transposed when c's block comes later
          Z[(6 * (size_t)a + r) * ns + 6 * (size_t)c + q] = bA >= bC ? T[(size_t)qc * BA_TB + ra] : T[(size_t)ra * BA_TB + qc];
        }
    }
  out[0] = P.nb;
  out[1] = P.nTilesOrig;
  out[2] = P.nTiles;
  out[3] = (int)SP.tasks.size();
  out[4] = P.ndDepth;
  out[5] = (int)SP.stepBegin.size() - 1;
  out[6] = L.two ? 1 : L.grid;
  out[7] = L.two ? 1 : 0;
  return COSL_OK;
}

int cosl_ba_solver_profile_enable(cosl_ba_solver* s, int on) {
  BA_ENTER(s)
  COSL_CUDA(cudaStreamSynchronize(s->rq.stream));
  s->timer.reset();
  s->timer.enabled = on != 0;
  return COSL_OK;
}

const char* cosl_ba_solver_timer(cosl_ba_solver* s, int idx, double* ms, int* calls) {
  if (!s || idx < 0 || idx >= s->timer.nsec) return nullptr;
  cudaSetDevice(s->device);
  cudaStreamSynchronize(s->rq.stream);
  s->timer.flush();
  if (ms) *ms = s->timer.ms[idx];
  if (calls) *calls = s->timer.calls[idx];
  return s->timer.names[idx];
}

}  // extern "C"

namespace {
// cosl_ba_solve, with the measurement covariances L (check_obs_cov's output) when it is given
int solve_once(cosl_ba_problem* prob, const cosl_ba_options* opt, const std::vector<double>* L,
               double info[COSL_BA_INFOSZ]) {
  cosl_ba_solver* s = nullptr;
  const double t0 = now_s();
  COSL_TRY(cosl_ba_solver_create(prob, opt, nullptr, &s));
  const double t1 = now_s();
  int rc = L ? set_obs_cov(s, L) : COSL_OK;
  if (rc == COSL_OK) rc = run_host(s, 0, info);
  const double t2 = now_s();
  if (rc == COSL_OK) rc = download(s, prob);
  const double t3 = now_s();
  if (rc == COSL_OK && info && prob->outlier) {
    long long c = 0;
    for (long long o = 0; o < prob->nobs; ++o) c += prob->outlier[o] ? 1 : 0;
    info[13] = (double)c;
  }
  free_solver(s);
  if (ba_timing())
    std::fprintf(stderr, "[ba timing] cosl_ba_solve: create %.1f  run %.1f  download %.1f  destroy %.1f ms\n",
                 1e3 * (t1 - t0), 1e3 * (t2 - t1), 1e3 * (t3 - t2), 1e3 * (now_s() - t3));
  return rc;
}
}  // namespace

extern "C" {

int cosl_ba_solve(cosl_ba_problem* prob, const cosl_ba_options* opt, double info[COSL_BA_INFOSZ]) {
  return solve_once(prob, opt, nullptr, info);
}

// Single-process multi-GPU drop-in (SURVEY.md 8b: the reference's BA pthread is ONE process,
// app/SL_CoSLAM.cpp:1702-1729): one host thread per device, points sharded by sum(k^2 + 8k) like
// the multi-process path, NCCL communicator created here.  Same results as cosl_ba_solve.
int cosl_ba_solve_multi(cosl_ba_problem* prob, const cosl_ba_options* opt, int n_gpus,
                        const int* devices, double info[COSL_BA_INFOSZ]) {
  if (!prob || !opt) return set_error(COSL_E_INVALID, "null argument");
  if (n_gpus <= 1) {
    cosl_ba_options o = *opt;
    if (devices) o.device = devices[0];
    return cosl_ba_solve(prob, &o, info);
  }
  if (!nccl().ok) return set_error(COSL_E_NCCL, "libnccl.so.2 could not be loaded");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < n_gpus)
    return set_error(COSL_E_CUDA, "%d GPUs requested, %d visible", n_gpus, ndev);
  const int R = n_gpus, n = prob->n;
  // contiguous point ranges balanced by sum(k^2 + 8 k)
  std::vector<int> bound(R + 1, 0);
  {
    std::vector<double> w((size_t)n + 1, 0.0);
    for (int i = 0; i < n; ++i) {
      const double k = (double)(prob->ptr[i + 1] - prob->ptr[i]);
      w[i + 1] = w[i] + k * k + 8.0 * k;
    }
    for (int r = 1; r < R; ++r)
      bound[r] = (int)(std::lower_bound(w.begin() + 1, w.end(), w[n] * r / R) - (w.begin() + 1));
    bound[R] = n;
    for (int r = 1; r <= R; ++r) bound[r] = std::max(bound[r], bound[r - 1]);
  }
  ncclUniqueId uid;
  if (nccl().GetUniqueId(&uid) != 0) return set_error(COSL_E_NCCL, "ncclGetUniqueId failed");
  std::vector<int> rc(R, COSL_OK);
  std::vector<std::string> err(R);
  std::vector<std::vector<double>> infos(R, std::vector<double>(COSL_BA_INFOSZ, 0.0));
  std::vector<std::vector<double>> Rr(R), tr(R);
  auto worker = [&](int r) {
    t_rank_share = R;
    const int dev = devices ? devices[r] : r;
    const int lo = bound[r], hi = bound[r + 1];
    const int64_t o0 = prob->ptr[lo], o1 = prob->ptr[hi];
    std::vector<int64_t> ptr((size_t)(hi - lo) + 1);
    for (int i = lo; i <= hi; ++i) ptr[i - lo] = prob->ptr[i] - o0;
    // cameras are replicated: every rank works on its own copy of R, t
    Rr[r].assign(prob->R, prob->R + 9 * (size_t)prob->m);
    tr[r].assign(prob->t, prob->t + 3 * (size_t)prob->m);
    cosl_ba_problem sp = *prob;
    sp.n = hi - lo;
    sp.nobs = o1 - o0;
    sp.n_con = std::max(0, std::min(prob->n_con - lo, hi - lo));
    sp.R = Rr[r].data();
    sp.t = tr[r].data();
    sp.X = prob->X + 3 * (size_t)lo;
    sp.ptr = ptr.data();
    sp.cam = prob->cam + o0;
    sp.xy = prob->xy + 2 * o0;
    sp.outlier = prob->outlier ? prob->outlier + o0 : nullptr;
    cosl_ba_options o = *opt;
    o.device = dev;
    cosl_ba_comm* comm = nullptr;
    cosl_ba_solver* sv = nullptr;
    int c = cosl_ba_comm_create((const uint8_t*)uid.internal, r, R, dev, &comm);
    if (c == COSL_OK) c = cosl_ba_solver_create(&sp, &o, comm, &sv);
    if (c == COSL_OK) c = cosl_ba_solver_run(sv, infos[r].data());
    if (c == COSL_OK) c = cosl_ba_solver_download(sv, &sp);
    if (c != COSL_OK) err[r] = last_error_ref();
    if (sv) cosl_ba_solver_destroy(sv);
    if (comm) cosl_ba_comm_destroy(comm);
    rc[r] = c;
  };
  std::vector<std::thread> th;
  for (int r = 1; r < R; ++r) th.emplace_back(worker, r);
  worker(0);
  for (auto& x : th) x.join();
  t_rank_share = 1;
  for (int r = 0; r < R; ++r)
    if (rc[r] != COSL_OK) return set_error(rc[r], "rank %d: %s", r, err[r].c_str());
  std::memcpy(prob->R, Rr[0].data(), sizeof(double) * 9 * (size_t)prob->m);
  std::memcpy(prob->t, tr[0].data(), sizeof(double) * 3 * (size_t)prob->m);
  if (info) {
    for (int k = 0; k < COSL_BA_INFOSZ; ++k) info[k] = infos[0][k];
    if (prob->outlier) {
      long long c = 0;
      for (long long o = 0; o < prob->nobs; ++o) c += prob->outlier[o] ? 1 : 0;
      info[13] = (double)c;
    }
  }
  return COSL_OK;
}

int cosl_sba_motstr_levmar_x(int n, int ncon, int m, int mcon, const char* vmask, double* p,
                             int cnp, int pnp, const double* x, int mnp,
                             const double* rot0params, int itmax, int verbose,
                             const double opts[5], double info[10], int device) {
  return cosl_sba_motstr_levmar_x_cov(n, ncon, m, mcon, vmask, p, cnp, pnp, x, nullptr, mnp, rot0params, itmax,
                                      verbose, opts, info, device);
}

int cosl_sba_motstr_levmar_x_cov(int n, int ncon, int m, int mcon, const char* vmask, double* p,
                                 int cnp, int pnp, const double* x, const double* covx, int mnp,
                                 const double* rot0params, int itmax, int verbose,
                                 const double opts[5], double info[10], int device) {
  if (cnp != 11 || pnp != 3 || mnp != 2 || !vmask || !p || !x || !rot0params || !opts)
    return set_error(COSL_E_INVALID, "cosl_sba_motstr_levmar_x: only cnp=11, pnp=3, mnp=2");
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
    const double dq[4] = {std::sqrt(1.0 - (c[5] * c[5] + c[6] * c[6] + c[7] * c[7])), c[5], c[6],
                          c[7]};
    double q[4];
    quat_mul(dq, rot0params + 4 * j, q);
    quat2mat(q, &R[9 * j]);
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
  // covx follows x: sba's point-major measurement order, which is the order of cam above
  std::vector<double> L;
  if (covx) COSL_TRY(check_obs_cov(covx, pr.nobs, L, "cosl_sba_motstr_levmar_x_cov"));
  cosl_ba_options o;
  cosl_ba_options_default(&o);
  o.max_err = 0;
  o.outer_iters = 1;
  o.inner_iters = itmax;
  for (int k = 0; k < 5; ++k) o.opts[k] = opts[k];
  o.verbose = verbose;
  o.device = device;
  double inf[COSL_BA_INFOSZ];
  COSL_TRY(solve_once(&pr, &o, covx ? &L : nullptr, inf));
  if (info)
    for (int k = 0; k < 10; ++k) info[k] = inf[k];
  for (int j = mcon; j < m; ++j) {
    double q[4], qn[4];
    const double q0c[4] = {rot0params[4 * j], -rot0params[4 * j + 1], -rot0params[4 * j + 2],
                           -rot0params[4 * j + 3]};
    mat2quat(&R[9 * j], q);
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

}  // extern "C"
