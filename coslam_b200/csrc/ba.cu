// ba.cu -- host side of the bundle-adjustment solver + its C-ABI (see include/coslam_b200.h).
// Replaces bundleAdjustRobust (LibVisualSLAM, call app/SL_CoSLAMRobustBA.cpp:174) and
// sba_motstr_levmar_x (sba-1.6, call app/SL_CoSLAMBA.cpp:360-363).  The LM control flow mirrors
// oracle/ba_oracle.cpp:levmar line by line; every arithmetic step runs in the kernels of
// ba_kernels.cuh.  Multi-GPU: points (with all their observations) are sharded over the ranks,
// cameras are replicated; per LM trial one NCCL all-reduce (sum) of the packed buffer
// [S | rhs] and one of a handful of scalars; per linearisation one of [U | ea] and one max-reduce.
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <sched.h>
#include <thread>
#include <vector>

#include "ba_kernels.cuh"
#include "ba_tile.cuh"
#include "common.cuh"
#include "tile_solve.h"

using namespace coslam;

/* ---------------------------------------------------------------- the tile solve for other callers */
namespace coslam {

int tile_task_order(const BaPlan& P, std::vector<BaTask>& order) {
  // two ticket lists (each keeps the critical-path-first order, hence stays topological)
  order.clear();
  for (const BaTask& t : P.tasks)
    if (t.type == BA_T_POTRF || t.type == BA_T_BWD) order.push_back(t);
  const int nA = (int)order.size();
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
  return nA;
}

int tile_solve_launch(const BaPlan& P, int nA, const TileSolveBufs& b, int device, cudaStream_t s, int* gridOut) {
  if (gridOut) *gridOut = 0;
  if (P.nb <= 0) return COSL_OK;
  BaTileDev td = {};
  td.rhs = b.rhs;
  td.tiles = b.tiles;
  td.rhsS = b.rhsS;
  td.Linv = b.Linv;
  td.y = b.y;
  td.x = b.x;
  td.cnt = b.cnt;
  td.tasks = b.tasks;
  td.bwd = b.bwd;
  td.sum = b.sum;
  td.blkRows = b.blkRows;
  td.nTasks = (int)P.tasks.size();
  td.nA = nA;
  td.nb = P.nb;
  td.nTiles = P.nTiles;
  td.nCounters = P.nCounters;
  td.xdoneBase = P.nTiles + P.nScratch;
  td.sc = b.fail;
  td.scFail = 0;
  td.trace = nullptr;
  const int t00 = P.tileIdx[0];
  const int t10 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 0] : -1;
  const int t11 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 1] : -1;
  if (P.nb <= 2 && t00 >= 0 && (P.nb == 1 || t11 >= 0)) {
    COSL_CUDA(cudaFuncSetAttribute(ba_tile_two, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_TILE_SMEM));
    COSL_LAUNCH(ba_tile_two, 1, BA_NTHREADS, BA_TILE_SMEM, s, td, t00, t10, t11);
    if (gridOut) *gridOut = 1;
  } else {
    // same grid rule as the BA solver: never more CTAs than can be co-resident (the tickets spin)
    COSL_CUDA(cudaFuncSetAttribute(ba_tile_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_TILE_SMEM));
    int nsm = 0, perSm = 0;
    COSL_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    COSL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, ba_tile_solve, BA_NTHREADS, BA_TILE_SMEM));
    if (perSm < 1) return set_error(COSL_E_CUDA, "tile solve: the kernel does not fit on a multiprocessor");
    const int grid = std::max(2, std::min(std::max(1, nsm), td.nTasks + 1));
    td.nSpecial = std::max(1, std::min(std::min(24, std::max(1, grid / 6)), grid - 1));
    COSL_LAUNCH(ba_tile_solve, grid, BA_NTHREADS, BA_TILE_SMEM, s, td);
    if (gridOut) *gridOut = grid;
  }
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
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
  cudaStream_t stream = nullptr;
  BaDev d;
  // host copies needed for write-back
  int m = 0, n = 0, mcon = 0, ncon = 0, mf = 0, ns = 0;
  long long N = 0, Nc = 0;
  std::vector<double> q0;  // m x 4
  // device buffers
  double *d_camK = nullptr, *d_camR0 = nullptr;
  double *d_pa = nullptr, *d_na = nullptr, *d_dpa = nullptr;
  double *d_pb = nullptr, *d_nb = nullptr, *d_dpb = nullptr;
  int *d_cam = nullptr, *d_pt = nullptr, *d_cobs = nullptr, *d_ccam = nullptr;
  double *d_xy = nullptr, *d_wgt = nullptr;
  long long* d_ptr = nullptr;
  double *d_W = nullptr, *d_V = nullptr, *d_eb = nullptr;
  double* d_Uea = nullptr;   // [U (m x 21) | ea (m x 6)] contiguous for one all-reduce
  // reduced camera system: [rhs (nb*64) | tiles]; the leading part [rhs | Schur-structure tiles]
  // is the payload of the one all-reduce per LM trial (ba_tile.cuh)
  BaPlan plan;
  double* d_S = nullptr;
  long long reduceCount = 0;  // doubles in the all-reduce payload
  double *d_Linv = nullptr, *d_y = nullptr, *d_x = nullptr;
  int* d_cnt = nullptr;
  BaTask* d_tasks = nullptr;
  BaBwdEntry* d_bwd = nullptr;
  BaSumEntry* d_sum = nullptr;
  double* d_rhsS = nullptr;
  int *d_blkRows = nullptr, *d_diagBlk = nullptr,
      *d_blkCam0 = nullptr, *d_order = nullptr, *d_solIdx = nullptr;
  BaTileDev td;
  std::vector<BaTask> taskOrder;  // as uploaded: [POTRF / BACKWARD | TRSM / UPDATE / SUM]
  unsigned long long* d_trace = nullptr;
  int solveGrid = 1;
  int numSM = 1;  // of the solver's device
  double factorFlops = 0.0;
  double* d_sc = nullptr;
  unsigned char* d_outlier = nullptr;
  BaPairItem* d_items = nullptr;
  double* d_Vinv = nullptr;
  bool costDone = false;         // solve_trial already evaluated the trial cost (ba_finish_cost)
  bool statsPending = false;     // |g|_inf / max diag of the last linearisation still to be computed (prep kernel)
  unsigned long long scSeq = 0;  // sequence number of the last scalar read-back (ba_publish_sc)
  int4* d_entries = nullptr;
  int nItems = 0;
  long long nEntries = 0;
  double* h_sc = nullptr;  // pinned
  bool twoSolve = false;  // <= 2 blocks: single-CTA resident solve (ba_tile_two)
  int two00 = -1, two10 = -1, two11 = -1;
  SectionTimer timer;
  int secLin = 0, secSchur = 0, secSolve = 0, secBack = 0, secCost = 0, secComm = 0;
  // statistics
  int nfev = 0, njev = 0, nlss = 0;
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

// Solver buffers come from the device's stream-ordered memory pool with an unlimited release
// threshold: cosl_ba_solve creates and destroys a solver per call, and after the first call the
// ~30 buffers (0.7 GB at c4) are handed out again without touching the driver's allocator.
static void pool_keep(int device) {
  static std::mutex mu;
  static bool done[64] = {};
  std::lock_guard<std::mutex> lk(mu);
  if (device < 0 || device >= 64 || done[device]) return;
  done[device] = true;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
}

// Pinned 128-byte slots for the per-trial scalar read-back.  cudaMallocHost / cudaFreeHost cost
// milliseconds each; a drop-in call creates and destroys a solver, so the slots are pooled.
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
    // its scalars straight into this host memory (UVA: the host pointer is the device pointer)
    if (cudaHostAlloc(&p, sizeof(double) * 32, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess)
      return nullptr;
    std::memset(p, 0, sizeof(double) * 32);
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

int upload_params(cosl_ba_solver* s, const cosl_ba_problem* p) {
  const int m = s->m;
  std::vector<double> R0((size_t)m * 9), pa((size_t)m * 6, 0.0);
  s->q0.resize((size_t)m * 4);
  for (int j = 0; j < m; ++j) {
    mat2quat(p->R + 9 * j, &s->q0[4 * j]);
    quat2mat(&s->q0[4 * j], &R0[9 * j]);
    for (int k = 0; k < 3; ++k) pa[6 * j + 3 + k] = p->t[3 * j + k];
  }
  COSL_CUDA(cudaMemcpyAsync(s->d_camR0, R0.data(), sizeof(double) * 9 * m, cudaMemcpyHostToDevice,
                            s->stream));
  COSL_CUDA(cudaMemcpyAsync(s->d_pa, pa.data(), sizeof(double) * 6 * m, cudaMemcpyHostToDevice,
                            s->stream));
  COSL_CUDA(cudaMemcpyAsync(s->d_pb, p->X, sizeof(double) * 3 * (size_t)s->n,
                            cudaMemcpyHostToDevice, s->stream));
  COSL_CUDA(cudaStreamSynchronize(s->stream));
  return COSL_OK;
}

void free_solver(cosl_ba_solver* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  s->timer.destroy();
  void* bufs[] = {s->d_camK, s->d_camR0, s->d_pa, s->d_na, s->d_dpa, s->d_pb, s->d_nb, s->d_dpb,
                  s->d_cam, s->d_pt, s->d_cobs, s->d_ccam, s->d_xy, s->d_wgt, s->d_ptr, s->d_W,
                  s->d_V, s->d_S, s->d_y, s->d_x, s->d_sc, s->d_outlier,
                  s->d_items, s->d_entries, s->d_Linv, s->d_cnt, s->d_tasks, s->d_bwd, s->d_blkRows,
                  s->d_diagBlk, s->d_blkCam0, s->d_order, s->d_solIdx,
                  s->d_trace, s->d_sum, s->d_rhsS, s->d_Vinv};
  for (void* b : bufs)
    if (b) cudaFreeAsync(b, s->stream);
  if (s->stream) cudaStreamSynchronize(s->stream);
  if (s->h_sc) pinned_slots().put(s->h_sc);
  if (s->stream) cudaStreamDestroy(s->stream);
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

int build_solver(cosl_ba_solver* s, const cosl_ba_problem* p) {
  TmpDeviceBufs tmp(s->stream);
  const double tBuild0 = now_s();
  const int m = p->m, n = p->n, mcon = p->m_con, ncon = p->n_con;
  const long long N = p->nobs;
  s->m = m;
  s->n = n;
  s->mcon = mcon;
  s->ncon = ncon;
  s->mf = m - mcon;
  s->ns = 6 * s->mf;
  s->N = N;
  // host-side index structures (the observation lists were validated by check_observations)
  std::vector<int> pt((size_t)N), cam((size_t)N);
  for (int i = 0; i < n; ++i)
    for (long long o = p->ptr[i]; o < p->ptr[i + 1]; ++o) pt[o] = i;
  for (long long o = 0; o < N; ++o) cam[o] = p->cam[o];
  // camera-major list of the free-camera observations
  std::vector<long long> cptr(m + 1, 0);
  for (long long o = 0; o < N; ++o)
    if (cam[o] >= mcon) cptr[cam[o] + 1]++;
  for (int j = 0; j < m; ++j) cptr[j + 1] += cptr[j];
  const long long Nc = cptr[m];
  s->Nc = Nc;
  std::vector<int> cobs((size_t)Nc), ccam((size_t)Nc);
  {
    std::vector<long long> fill(cptr.begin(), cptr.end() - 1);
    for (long long o = 0; o < N; ++o)
      if (cam[o] >= mcon) {
        const long long q = fill[cam[o]]++;
        cobs[q] = (int)o;
        ccam[q] = cam[o];
      }
  }
  if (ba_timing()) std::fprintf(stderr, "[ba timing] observation index lists %.1f ms\n", 1e3 * (now_s() - tBuild0));
  // camera co-visibility (which pairs of free cameras share a free point) -> plan of the
  // reduced-system solve (ordering, tiles, task DAG) and the work lists of the Schur contraction.
  // In the multi-GPU case every rank must derive the SAME structure although it only sees the
  // pairs of its own point shard: the presence bitmap is all-reduced (max) first.
  const int mf = s->mf;
  const double tPair0 = now_s();
  // the observation index arrays go to the device first: the pair buckets are counted there
  COSL_TRY(dev_alloc(s->stream, &s->d_cam, (size_t)N));
  COSL_TRY(dev_alloc(s->stream, &s->d_pt, (size_t)N));
  COSL_TRY(dev_alloc(s->stream, &s->d_ptr, (size_t)n + 1));
  COSL_TRY(dev_alloc(s->stream, &s->d_cobs, (size_t)Nc));
  COSL_TRY(dev_alloc(s->stream, &s->d_ccam, (size_t)Nc));
  const size_t nBuckets = (size_t)mf * mf;
  unsigned *d_pcnt = nullptr, *d_poff = nullptr;
  COSL_TRY(tmp.alloc(&d_pcnt, nBuckets + 1));
  COSL_TRY(tmp.alloc(&d_poff, nBuckets + 1));
  COSL_CUDA(cudaMemcpyAsync(s->d_cam, cam.data(), sizeof(int) * (size_t)N, cudaMemcpyHostToDevice, s->stream));
  COSL_CUDA(cudaMemcpyAsync(s->d_pt, pt.data(), sizeof(int) * (size_t)N, cudaMemcpyHostToDevice, s->stream));
  COSL_CUDA(cudaMemcpyAsync(s->d_ptr, p->ptr, sizeof(long long) * ((size_t)n + 1), cudaMemcpyHostToDevice, s->stream));
  if (Nc) {
    COSL_CUDA(cudaMemcpyAsync(s->d_cobs, cobs.data(), sizeof(int) * (size_t)Nc, cudaMemcpyHostToDevice, s->stream));
    COSL_CUDA(cudaMemcpyAsync(s->d_ccam, ccam.data(), sizeof(int) * (size_t)Nc, cudaMemcpyHostToDevice, s->stream));
  }
  BaDev db;  // just what ba_pairs_build reads
  std::memset(&db, 0, sizeof(db));
  db.mcon = mcon;
  db.ncon = ncon;
  db.mf = mf;
  db.Nc = Nc;
  db.cam = s->d_cam;
  db.pt = s->d_pt;
  db.ptr = s->d_ptr;
  db.cobs = s->d_cobs;
  std::vector<unsigned> poff(nBuckets + 1, 0u);
  COSL_CUDA(cudaMemsetAsync(d_pcnt, 0, sizeof(unsigned) * (nBuckets + 1), s->stream));
  if (Nc && mf) {
    COSL_LAUNCH(ba_pairs_build<false>, (unsigned)div_up64(Nc, 256), 256, 0, s->stream, db, d_pcnt, d_poff, nullptr);
    COSL_LAUNCH(ba_scan_u32, 1, 1024, 0, s->stream, d_pcnt, d_poff, (long long)nBuckets);
    COSL_CUDA(cudaMemcpyAsync(poff.data(), d_poff, sizeof(unsigned) * (nBuckets + 1), cudaMemcpyDeviceToHost, s->stream));
  }
  COSL_CUDA(cudaStreamSynchronize(s->stream));
  std::vector<uint8_t> adj(nBuckets, 0);
  for (int ja = 0; ja < mf; ++ja)
    for (int jb = ja; jb < mf; ++jb)
      if (poff[(size_t)ja * mf + jb + 1] > poff[(size_t)ja * mf + jb]) adj[(size_t)ja * mf + jb] = adj[(size_t)jb * mf + ja] = 1;
  if (s->comm && s->comm->nranks > 1 && mf > 0) {
    uint8_t* d_adj = nullptr;
    COSL_TRY(tmp.alloc(&d_adj, adj.size()));
    COSL_CUDA(cudaMemcpyAsync(d_adj, adj.data(), adj.size(), cudaMemcpyHostToDevice, s->stream));
    const int rc = nccl().AllReduce(d_adj, d_adj, adj.size(), ncclUint8, ncclMax, s->comm->comm, s->stream);
    if (rc != 0) return set_error(COSL_E_NCCL, "ncclAllReduce (co-visibility) failed (%d)", rc);
    COSL_CUDA(cudaMemcpyAsync(adj.data(), d_adj, adj.size(), cudaMemcpyDeviceToHost, s->stream));
    COSL_CUDA(cudaStreamSynchronize(s->stream));
  }
  {
    const double tPlan0 = now_s();
    s->plan = ba_make_plan(mf, adj);
    if (ba_timing()) std::fprintf(stderr, "[ba timing] plan %.1f ms\n", 1e3 * (now_s() - tPlan0));
    if (s->plan.nb < 0) return set_error(COSL_E_INVALID, "solve plan: dependency cycle (internal error)");
  }
  const BaPlan& P = s->plan;
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
  // pair lists: one bucket per camera pair (offsets counted on the device above); a work item is
  // a run of <= 512 entries of one bucket; the entries themselves are placed by ba_pairs_build.
  // Fewer entries per item when the problem is small (local BA: a few dozen camera pairs with
  // thousands of entries each), so that the grid still fills the GPU; ba_schur_pairs_st works in
  // batches of 32 entries and sums 32 lanes per item: multiples of 32, >= 128
  std::vector<BaPairItem> items;
  const long long nEntries = poff[nBuckets];
  const int chunk = (int)(32 * std::max<long long>(4, std::min<long long>(16, nEntries / (4096 * 32))));
  for (int ja = 0; ja < mf; ++ja)
    for (int jb = ja; jb < mf; ++jb) {
      const long long b0 = poff[(size_t)ja * mf + jb], b1 = poff[(size_t)ja * mf + jb + 1];
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
  COSL_TRY(dev_alloc(s->stream, &s->d_entries, (size_t)nEntries));
  COSL_CUDA(cudaMemsetAsync(d_pcnt, 0, sizeof(unsigned) * (nBuckets + 1), s->stream));
  if (nEntries)
    COSL_LAUNCH(ba_pairs_build<true>, (unsigned)div_up64(Nc, 256), 256, 0, s->stream, db, d_pcnt, d_poff, s->d_entries);
  s->nEntries = nEntries;
  s->nItems = (int)items.size();
  if (ba_timing())
    std::fprintf(stderr, "[ba timing] co-visibility + Schur work lists %.1f ms (%lld pair entries, %d threads)\n",
                 1e3 * (now_s() - tPair0), nEntries, host_threads());
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
  // device allocations
  COSL_TRY(dev_alloc(s->stream, &s->d_camK, (size_t)m * 5));
  COSL_TRY(dev_alloc(s->stream, &s->d_camR0, (size_t)m * 9));
  COSL_TRY(dev_alloc(s->stream, &s->d_pa, (size_t)m * 6));
  COSL_TRY(dev_alloc(s->stream, &s->d_na, (size_t)m * 6));
  COSL_TRY(dev_alloc(s->stream, &s->d_dpa, (size_t)m * 6));
  COSL_TRY(dev_alloc(s->stream, &s->d_pb, (size_t)n * 3));
  COSL_TRY(dev_alloc(s->stream, &s->d_nb, (size_t)n * 3));
  COSL_TRY(dev_alloc(s->stream, &s->d_dpb, (size_t)n * 3));
  COSL_TRY(dev_alloc(s->stream, &s->d_xy, (size_t)N * 2));
  COSL_TRY(dev_alloc(s->stream, &s->d_wgt, (size_t)N));
  COSL_TRY(dev_alloc(s->stream, &s->d_W, (size_t)N * 18));
  // [V (n x 6) | e_b (n x 3) | U (m x 21) | e_a (m x 6)] in one slab: one memset per linearisation
  COSL_TRY(dev_alloc(s->stream, &s->d_V, (size_t)n * 9 + (size_t)m * 27));
  s->d_eb = s->d_V + (size_t)n * 6;
  s->d_Uea = s->d_eb + (size_t)n * 3;
  const double tAlloc0 = now_s();
  const int nb = std::max(1, P.nb), nTiles = std::max(1, P.nTiles);
  const size_t rhsLen = (size_t)nb * BA_TB;
  s->reduceCount = (long long)rhsLen + (long long)P.nTilesOrig * BA_TILE;
  s->factorFlops = P.flops;
  COSL_TRY(dev_alloc(s->stream, &s->d_S, rhsLen + ((size_t)nTiles + P.nScratch) * BA_TILE));
  COSL_TRY(dev_alloc(s->stream, &s->d_rhsS, (size_t)std::max(1, P.nScratch) * BA_TB));
  COSL_TRY(dev_alloc(s->stream, &s->d_sum, P.sumList.size()));
  COSL_TRY(dev_alloc(s->stream, &s->d_Linv, (size_t)nb * BA_TILE));
  COSL_TRY(dev_alloc(s->stream, &s->d_y, rhsLen));
  COSL_TRY(dev_alloc(s->stream, &s->d_x, rhsLen));
  COSL_TRY(dev_alloc(s->stream, &s->d_cnt, (size_t)P.nCounters + 2 + P.tasks.size()));
  COSL_TRY(dev_alloc(s->stream, &s->d_tasks, P.tasks.size()));
  COSL_TRY(dev_alloc(s->stream, &s->d_bwd, P.bwdList.size()));
  COSL_TRY(dev_alloc(s->stream, &s->d_blkRows, (size_t)nb));
  COSL_TRY(dev_alloc(s->stream, &s->d_diagBlk, (size_t)nTiles));
  COSL_TRY(dev_alloc(s->stream, &s->d_blkCam0, (size_t)nb + 1));
  COSL_TRY(dev_alloc(s->stream, &s->d_order, (size_t)std::max(1, mf)));
  COSL_TRY(dev_alloc(s->stream, &s->d_solIdx, (size_t)std::max(1, mf)));
  std::vector<int> h_diagBlk(nTiles, -1), h_solIdx(std::max(1, mf), 0);
  for (int k = 0; k < P.nb; ++k) h_diagBlk[P.tileIdx[(size_t)k * P.nb + k]] = k;
  for (int j = 0; j < mf; ++j) h_solIdx[j] = P.camBlk[j] * BA_TB + P.camOff[j];
  COSL_TRY(dev_alloc(s->stream, &s->d_sc, (size_t)SC_NTOT));
  COSL_TRY(dev_alloc(s->stream, &s->d_outlier, (size_t)N));
  COSL_TRY(dev_alloc(s->stream, &s->d_items, items.size()));
  COSL_TRY(dev_alloc(s->stream, &s->d_Vinv, (size_t)n * 6));
  static_assert(SC_NTOT <= 16, "pinned slot size");
  s->h_sc = pinned_slots().get();
  if (!s->h_sc) return set_error(COSL_E_NOMEM, "pinned host allocation failed");
  *reinterpret_cast<volatile unsigned long long*>(s->h_sc + SC_NTOT) = 0;  // a pooled slot keeps its last flag
  s->scSeq = 0;
#define UP(dst, src, bytes) \
  COSL_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s->stream))
  UP(s->d_camK, camK.data(), sizeof(double) * 5 * m);
  UP(s->d_xy, p->xy, sizeof(double) * 2 * (size_t)N);
  if (!items.empty()) UP(s->d_items, items.data(), sizeof(BaPairItem) * items.size());
  const int nA = tile_task_order(P, s->taskOrder);
  if (!s->taskOrder.empty()) UP(s->d_tasks, s->taskOrder.data(), sizeof(BaTask) * s->taskOrder.size());
  if (!P.bwdList.empty()) UP(s->d_bwd, P.bwdList.data(), sizeof(BaBwdEntry) * P.bwdList.size());
  if (!P.sumList.empty()) UP(s->d_sum, P.sumList.data(), sizeof(BaSumEntry) * P.sumList.size());
  if (P.nb) {
    UP(s->d_blkRows, P.blkRows.data(), sizeof(int) * P.nb);
    UP(s->d_blkCam0, P.blkCam0.data(), sizeof(int) * (P.nb + 1));
    UP(s->d_order, P.order.data(), sizeof(int) * mf);
  }
  UP(s->d_diagBlk, h_diagBlk.data(), sizeof(int) * nTiles);
  UP(s->d_solIdx, h_solIdx.data(), sizeof(int) * std::max(1, mf));
#undef UP
  COSL_CUDA(cudaStreamSynchronize(s->stream));
  if (ba_timing()) std::fprintf(stderr, "[ba timing] allocations + uploads %.1f ms\n", 1e3 * (now_s() - tAlloc0));
  BaDev& d = s->d;
  d.m = m;
  d.n = n;
  d.mcon = mcon;
  d.ncon = ncon;
  d.mf = s->mf;
  d.ns = s->ns;
  d.N = N;
  d.Nc = Nc;
  d.camK = s->d_camK;
  d.camR0 = s->d_camR0;
  d.cam = s->d_cam;
  d.pt = s->d_pt;
  d.xy = s->d_xy;
  d.wgt = s->d_wgt;
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
  BaTileDev& td = s->td;
  td.rhs = d.rhs;
  td.tiles = d.tiles;
  td.Linv = s->d_Linv;
  td.y = s->d_y;
  td.x = s->d_x;
  td.cnt = s->d_cnt;
  td.tasks = s->d_tasks;
  td.bwd = s->d_bwd;
  td.sum = s->d_sum;
  td.rhsS = s->d_rhsS;
  td.xdoneBase = P.nTiles + P.nScratch;
  td.blkRows = s->d_blkRows;
  td.nTasks = (int)P.tasks.size();
  td.nA = nA;
  td.nb = P.nb;
  td.nTiles = P.nTiles;
  td.nCounters = P.nCounters;
  td.sc = s->d_sc;
  td.scFail = (int)SC_FAIL;
  td.trace = nullptr;
  // Systems of one or two blocks (local BA) are solved by one resident CTA: for the 72 x 72 system of
  // the c3 local BA, ba_tile_two needs 26 us per LM trial and the task kernel 42 us (H100 80GB HBM3, 400 W).
  if (P.nb >= 1 && P.nb <= 2) {
    s->twoSolve = true;
    s->two00 = P.tileIdx[0];
    s->two10 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 0] : -1;
    s->two11 = P.nb == 2 ? P.tileIdx[(size_t)1 * P.nb + 1] : -1;
    if (s->two00 < 0 || (P.nb == 2 && s->two11 < 0)) s->twoSolve = false;
  }
  COSL_CUDA(cudaFuncSetAttribute(ba_tile_solve, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 BA_TILE_SMEM));
  COSL_CUDA(cudaFuncSetAttribute(ba_tile_two, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_TILE_SMEM));
  COSL_CUDA(cudaFuncSetAttribute(ba_schur_pairs_st, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_ST_SMEM));
  {
    // persistent grid: never more CTAs than can be co-resident (the ticket scheduler spins)
    int nsm = 0, perSm = 0;
    COSL_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, s->device));
    s->numSM = std::max(1, nsm);
    COSL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, ba_tile_solve, BA_NTHREADS,
                                                            BA_TILE_SMEM));
    const int grid = nsm * std::max(1, std::min(perSm, 1));
    s->solveGrid = std::max(2, std::min(grid, td.nTasks + 1));
    // CTAs that only ever run the diagonal-block tasks (see BaTileDev::nSpecial)
    const int nsp = std::min(24, std::max(1, s->solveGrid / 6));
    td.nSpecial = std::max(1, std::min(nsp, s->solveGrid - 1));
  }
  s->secLin = s->timer.section("ba_linearize");
  s->secSchur = s->timer.section("ba_schur");
  s->secSolve = s->timer.section("ba_solve");
  s->secBack = s->timer.section("ba_backsub");
  s->secCost = s->timer.section("ba_cost");
  s->secComm = s->timer.section("ba_allreduce");
  return upload_params(s, p);
}

/* ---------------------------------------------------------------- device steps */
inline bool multi(const cosl_ba_solver* s) { return s->comm && s->comm->nranks > 1; }
inline int rank_of(const cosl_ba_solver* s) { return s->comm ? s->comm->rank : 0; }

int allreduce(cosl_ba_solver* s, double* buf, size_t count, int op) {
  if (!multi(s)) return COSL_OK;
  s->timer.begin(s->secComm, s->stream);
  const int rc = nccl().AllReduce(buf, buf, count, ncclFloat64, op, s->comm->comm, s->stream);
  s->timer.end(s->stream);
  if (rc != 0)
    return set_error(COSL_E_NCCL, "ncclAllReduce: %s",
                     nccl().GetErrorString ? nccl().GetErrorString(rc) : "?");
  return COSL_OK;
}

int zero_sc(cosl_ba_solver* s, int first, int count) {
  COSL_CUDA(cudaMemsetAsync(s->d_sc + first, 0, sizeof(double) * count, s->stream));
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
                              s->stream));
    COSL_CUDA(cudaStreamSynchronize(s->stream));
    return COSL_OK;
  }
  const unsigned long long seq = ++s->scSeq;
  COSL_LAUNCH(ba_publish_sc, 1, 32, 0, s->stream, s->d_sc, s->h_sc, seq);
  volatile unsigned long long* flag = reinterpret_cast<volatile unsigned long long*>(s->h_sc + SC_NTOT);
  for (long long spin = 0; *flag != seq; ++spin) {
    if ((spin & 0xfff) == 0xfff) {
      const cudaError_t q = cudaStreamQuery(s->stream);
      if (q == cudaSuccess) break;  // everything ran: the stores are visible after the query
      if (q != cudaErrorNotReady)
        return set_error(COSL_E_CUDA, "scalar read-back: %s", cudaGetErrorString(q));
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (*flag != seq) {  // left through the query: make sure the stores have landed
    COSL_CUDA(cudaStreamSynchronize(s->stream));
    if (*flag != seq) return set_error(COSL_E_CUDA, "scalar read-back: flag missing after synchronise");
  }
  return COSL_OK;
}

// weighted cost of a parameter set -> *out (all ranks)
int eval_cost(cosl_ba_solver* s, const double* pa, const double* pb, double* out, bool* finite) {
  ++s->nfev;
  COSL_TRY(zero_sc(s, SC_COST, 1));
  COSL_TRY(zero_sc(s, SC_NONFINITE, 1));
  s->timer.begin(s->secCost, s->stream);
  if (s->N)
    COSL_LAUNCH(ba_residual_kernel, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d, pa, pb,
                0, 0.0, nullptr);
  s->timer.end(s->stream);
  COSL_TRY(allreduce(s, s->d_sc, SC_NSUM, ncclSum));
  COSL_TRY(read_sc(s));
  *out = s->h_sc[SC_COST];
  *finite = std::isfinite(*out) && s->h_sc[SC_NONFINITE] == 0.0;
  return COSL_OK;
}

int compute_weights(cosl_ba_solver* s) {
  if (s->opt.max_err > 0) {
    if (s->N)
      COSL_LAUNCH(ba_residual_kernel, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d,
                  s->d_pa, s->d_pb, 1, s->opt.max_err, nullptr);
  } else {
    std::vector<double> ones((size_t)s->N, 1.0);
    COSL_CUDA(cudaMemcpyAsync(s->d_wgt, ones.data(), sizeof(double) * (size_t)s->N,
                              cudaMemcpyHostToDevice, s->stream));
    COSL_CUDA(cudaStreamSynchronize(s->stream));
  }
  return COSL_OK;
}

// Jacobians, U, V, W, ea, eb at (pa, pb); ginf / maxdiag land in h_sc
// statsNow: |g|_inf / max diag are wanted before the next solve (first iteration: mu0); otherwise they are
// computed by the prep kernel of the next trial (solve_trial) and arrive with that trial's scalars
int linearize(cosl_ba_solver* s, bool statsNow, bool statsLater) {
  ++s->njev;
  s->timer.begin(s->secLin, s->stream);
  COSL_CUDA(cudaMemsetAsync(s->d_V, 0, sizeof(double) * (9 * (size_t)s->n + 27 * (size_t)s->m), s->stream));
  if (s->N)
    COSL_LAUNCH(ba_linearize_points, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d,
                s->d_pa, s->d_pb);
  if (s->Nc)
    COSL_LAUNCH(ba_linearize_cams, (unsigned)div_up64(s->Nc, 128), 128, 0, s->stream, s->d,
                s->d_pa, s->d_pb);
  s->timer.end(s->stream);
  COSL_TRY(allreduce(s, s->d_Uea, (size_t)27 * s->m, ncclSum));
  if (!s->N) COSL_TRY(zero_sc(s, SC_GINF, 2));  // otherwise ba_linearize_points cleared them
  s->statsPending = false;
  if (statsNow || (statsLater && !s->ns)) {
    COSL_LAUNCH(ba_stats_kernel, (unsigned)div_up64((long long)s->n + s->m, 256), 256, 0, s->stream,
                s->d);
    COSL_TRY(allreduce(s, s->d_sc + SC_NSUM, 2, ncclMax));
  } else if (statsLater) {
    s->statsPending = true;
  }
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// reduced camera system -> d_x (block padded, permuted): one persistent dataflow launch
int dense_solve(cosl_ba_solver* s) {
  const int ns = s->ns;
  if (ns == 0) return COSL_OK;
  s->timer.begin(s->secSolve, s->stream);
  if (s->twoSolve) {
    COSL_LAUNCH(ba_tile_two, 1, BA_NTHREADS, BA_TILE_SMEM, s->stream, s->td, s->two00, s->two10, s->two11);
  } else {
    COSL_LAUNCH(ba_tile_solve, s->solveGrid, BA_NTHREADS, BA_TILE_SMEM, s->stream, s->td);
  }
  s->timer.end(s->stream);
  COSL_CUDA(cudaGetLastError());
  return COSL_OK;
}

// Schur complement + dense solve + back substitution for damping mu; trial parameters -> na, nb;
// scalars (dp_L2, dL, p_L2, fail) -> h_sc
int solve_trial(cosl_ba_solver* s, double mu, bool* solved) {
  ++s->nlss;
  const bool r0 = rank_of(s) == 0;
  const long long ns = s->ns;
  if (!ns) {  // no free camera: nothing launches ba_tile_init, which clears the trial's scalars otherwise
    COSL_TRY(zero_sc(s, SC_DP_L2, 3));
    COSL_TRY(zero_sc(s, SC_FAIL, 1));
    COSL_TRY(zero_sc(s, SC_COST, 1));
    COSL_TRY(zero_sc(s, SC_NONFINITE, 1));
  }
  static const bool fineSchur = std::getenv("COSL_BA_TIMING_FINE") != nullptr;  // diagnostic: init / contraction apart
  const int secInit = fineSchur ? s->timer.section("ba_schur_init") : s->secSchur;
  s->timer.begin(secInit, s->stream);
  if (ns) {
    // also clears the scalars of this trial (|dp|^2, dL, |p|^2, fail, cost, non-finite) and the task
    // counters of the solve: five memset nodes less per trial
    const int nTilesInit = std::max(1, s->plan.nTiles);
    const bool doStats = s->statsPending;
    s->statsPending = false;
    COSL_LAUNCH(ba_prep_kernel, nTilesInit + (unsigned)div_up64((long long)s->n + s->m, 256), 256, 0, s->stream, s->d,
                mu, r0 ? 1 : 0, s->d_diagBlk, s->d_blkCam0, s->d_order, s->d_cnt,
                s->td.nCounters + 2 + s->td.nTasks, nTilesInit, s->d_Vinv, doStats ? 1 : 0,
                s->d_dpb, 3LL * s->n);
    if (doStats) COSL_TRY(allreduce(s, s->d_sc + SC_NSUM, 2, ncclMax));
    if (fineSchur) {
      s->timer.end(s->stream);
      s->timer.begin(s->secSchur, s->stream);
    }
    if (s->nItems)
      COSL_LAUNCH(ba_schur_pairs_st, div_up(s->nItems, BA_ST_WARPS), 32 * BA_ST_WARPS, BA_ST_SMEM, s->stream,
                  s->d, s->d_items, s->nItems, s->d_entries, s->d_Vinv);
  }
  s->timer.end(s->stream);
  // the one exchange of an LM trial: [rhs | Schur-structure tiles] is contiguous, no packing
  if (ns && multi(s)) COSL_TRY(allreduce(s, s->d_S, (size_t)s->reduceCount, ncclSum));
  COSL_TRY(dense_solve(s));
  s->costDone = false;
  if (ns) {
    // back substitution + trial cost in two launches (ba_kernels.cuh): the accumulator d_dpb was zeroed by the
    // prep kernel, V*^-1 is the one the Schur contraction used
    const int nCamBlocks = div_up(6 * s->m, 256);
    s->timer.begin(s->secBack, s->stream);
    COSL_LAUNCH(ba_back_cams_points, nCamBlocks + (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d, s->d_pa,
                s->d_x, s->d_dpa, s->d_na, mu, r0 ? 1 : 0, nCamBlocks, s->d_dpb);
    s->timer.end(s->stream);
    s->timer.begin(s->secCost, s->stream);
    COSL_LAUNCH(ba_finish_cost, (unsigned)div_up64(s->N + (long long)s->n, 256), 256, 0, s->stream, s->d, s->d_na,
                s->d_pb, s->d_nb, s->d_dpb, s->d_Vinv, mu);
    s->timer.end(s->stream);
    s->costDone = true;
    COSL_CUDA(cudaGetLastError());
    *solved = true;
    return COSL_OK;
  }
  s->timer.begin(s->secBack, s->stream);
  // (also zeroes the accumulator of the point back-substitution, d_nb)
  COSL_LAUNCH(ba_cam_update, std::max(div_up(6 * s->m, 256), (int)std::min<long long>(s->numSM, div_up64(3LL * s->n, 1024))),
              256, 0, s->stream, s->d, s->d_pa, s->d_x, s->d_dpa, s->d_na, mu, r0 ? 1 : 0, s->d_nb, 3LL * s->n);
  if (s->N)
    COSL_LAUNCH(ba_back_subst, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d, s->d_dpa,
                s->d_nb);
  if (s->n)
    COSL_LAUNCH(ba_back_finish, (unsigned)div_up64(s->n, 256), 256, 0, s->stream, s->d, s->d_pb,
                s->d_nb, s->d_dpb, mu);
  s->timer.end(s->stream);
  COSL_CUDA(cudaGetLastError());
  // the scalar all-reduce of this trial is merged with the cost evaluation by the caller
  *solved = true;
  return COSL_OK;
}

/* Weighted SBA LM, control flow identical to oracle/ba_oracle.cpp:levmar */
int levmar(cosl_ba_solver* s, int itmax, const double opts[5], double info[10], int fixed_trials) {
  const double tau = opts[0], eps1 = opts[1], eps2 = opts[2], eps2_sq = opts[2] * opts[2],
               eps3 = opts[3], eps4 = opts[4];
  const double EPS_SQ = 1e-24;
  double mu = 0, nu = 2;
  int stop = 0, itno = 0;
  s->nfev = s->njev = s->nlss = 0;
  double p_eL2 = 0;
  bool finite = true;
  COSL_TRY(eval_cost(s, s->d_pa, s->d_pb, &p_eL2, &finite));
  const double init_eL2 = p_eL2;
  double ginf = 0, maxdiag = 0, dp_L2 = 0;
  if (!finite) stop = 7;
  for (itno = 0; itno < itmax && !stop; ++itno) {
    COSL_TRY(linearize(s, itno == 0, itno > 0 && !fixed_trials));
    // ginf / maxdiag are needed on the host for mu0 (first iteration) and for the eps1 stop test.  After
    // the first iteration the test is evaluated one read-back LATE: the scalars stay in d_sc (nothing
    // below touches SC_GINF / SC_MAXDIAG) and arrive with the read-back of the next trial, which is
    // discarded if the test fires -- it only wrote the trial buffers.  Same decisions and counters as
    // the oracle, one host synchronisation less per LM iteration.
    bool ginfPending = false;
    if (itno == 0) {
      COSL_TRY(read_sc(s));
      ginf = s->h_sc[SC_GINF];
      maxdiag = s->h_sc[SC_MAXDIAG];
    } else if (!fixed_trials) {
      ginfPending = true;
    }
    if (!fixed_trials && !ginfPending && ginf <= eps1) {
      stop = 1;
      break;
    }
    if (itno == 0) mu = tau * maxdiag;
    bool lateStop = false;
    while (true) {
      bool solved = false, accepted = false;
      COSL_TRY(solve_trial(s, mu, &solved));
      // trial cost, merged scalar all-reduce
      ++s->nfev;  // (cost / non-finite scalars were cleared by solve_trial)
      if (!s->costDone) {
        s->timer.begin(s->secCost, s->stream);
        if (s->N)
          COSL_LAUNCH(ba_residual_kernel, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d,
                      s->d_na, s->d_nb, 0, 0.0, nullptr);
        s->timer.end(s->stream);
      }
      COSL_TRY(allreduce(s, s->d_sc, SC_NSUM, ncclSum));
      COSL_TRY(read_sc(s));
      if (ginfPending) {
        ginfPending = false;
        ginf = s->h_sc[SC_GINF];
        maxdiag = s->h_sc[SC_MAXDIAG];
        if (ginf <= eps1) {  // the eps1 test of this iteration: the trial just run never happened
          --s->nlss;
          --s->nfev;
          stop = 1;
          lateStop = true;
          break;
        }
      }
      solved = (s->h_sc[SC_FAIL] == 0.0);
      if (solved) {
        dp_L2 = s->h_sc[SC_DP_L2];
        const double dL = s->h_sc[SC_DL], p_L2 = s->h_sc[SC_P_L2];
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
        const double pdp_eL2 = s->h_sc[SC_COST];
        if (!std::isfinite(pdp_eL2) || s->h_sc[SC_NONFINITE] != 0.0) {
          stop = 7;
          break;
        }
        const double dF = p_eL2 - pdp_eL2;
        if (s->opt.verbose && rank_of(s) == 0)
          std::printf("  [gpu LM %d] mu %.3e cost %.9g -> %.9g dL %.3e\n", itno, mu, p_eL2, pdp_eL2,
                      dL);
        if (dF > 0 && dL > 0) {
          double tmp = 2 * dF / dL - 1;
          tmp = 1 - tmp * tmp * tmp;
          mu = mu * std::max(tmp, 1.0 / 3.0);
          nu = 2;
          if (!fixed_trials && (std::sqrt(p_eL2) - std::sqrt(pdp_eL2)) < eps4 * std::sqrt(p_eL2))
            stop = 6;
          std::swap(s->d_pa, s->d_na);
          std::swap(s->d_pb, s->d_nb);
          p_eL2 = pdp_eL2;
          accepted = true;
        }
      }
      if (fixed_trials && s->nlss >= fixed_trials) {
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
    if (lateStop) break;
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
    info[7] = s->nfev;
    info[8] = s->njev;
    info[9] = s->nlss;
  }
  return COSL_OK;
}

int run_robust(cosl_ba_solver* s, int fixed_trials, double info[COSL_BA_INFOSZ]) {
  double sinfo[10] = {0};
  double first_e0 = -1;
  int total_trials = 0;
  COSL_CUDA(cudaStreamSynchronize(s->stream));
  const auto t0 = std::chrono::steady_clock::now();
  const int rounds = fixed_trials ? 1 : std::max(1, s->opt.outer_iters);
  for (int r = 0; r < rounds; ++r) {
    COSL_TRY(compute_weights(s));
    COSL_TRY(levmar(s, fixed_trials ? (1 << 30) : s->opt.inner_iters, s->opt.opts, sinfo,
                    fixed_trials));
    if (first_e0 < 0) first_e0 = sinfo[0];
    total_trials += (int)sinfo[9];
  }
  double nout = 0;
  if (s->opt.max_err > 0) {  // the same branch on every rank (options are global): collective inside
    COSL_TRY(zero_sc(s, SC_COST, 1));
    if (s->N)
      COSL_LAUNCH(ba_residual_kernel, (unsigned)div_up64(s->N, 256), 256, 0, s->stream, s->d, s->d_pa,
                  s->d_pb, 2, s->opt.max_err, s->d_outlier);
    COSL_TRY(allreduce(s, s->d_sc, SC_NSUM, ncclSum));
    COSL_TRY(read_sc(s));
    nout = s->h_sc[SC_COST];  // outliers over ALL ranks' observations
  } else {
    COSL_CUDA(cudaMemsetAsync(s->d_outlier, 0, (size_t)s->N ? (size_t)s->N : 1, s->stream));
    COSL_CUDA(cudaStreamSynchronize(s->stream));
  }
  const auto t1 = std::chrono::steady_clock::now();
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

int download(cosl_ba_solver* s, cosl_ba_problem* p) {
  const int m = s->m;
  std::vector<double> pa((size_t)m * 6);
  COSL_CUDA(cudaMemcpyAsync(pa.data(), s->d_pa, sizeof(double) * 6 * m, cudaMemcpyDeviceToHost,
                            s->stream));
  std::vector<double> X((size_t)s->n * 3);
  COSL_CUDA(cudaMemcpyAsync(X.data(), s->d_pb, sizeof(double) * 3 * (size_t)s->n,
                            cudaMemcpyDeviceToHost, s->stream));
  if (p->outlier && s->N)
    COSL_CUDA(cudaMemcpyAsync(p->outlier, s->d_outlier, (size_t)s->N, cudaMemcpyDeviceToHost,
                              s->stream));
  COSL_CUDA(cudaStreamSynchronize(s->stream));
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
  if (prob->m < 1 || prob->n < 0 || prob->nobs < 0 || prob->m_con < 0 || prob->m_con > prob->m ||
      prob->n_con < 0 || prob->n_con > prob->n || !prob->K || !prob->R || !prob->t ||
      (prob->n && (!prob->X || !prob->ptr)) || (prob->nobs && (!prob->cam || !prob->xy)) ||
      prob->nobs >= (1ll << 31))
    return set_error(COSL_E_INVALID, "cosl_ba_solver_create: bad problem");
  if (prob->n && prob->ptr[prob->n] != prob->nobs)
    return set_error(COSL_E_INVALID, "ptr[n] != nobs");
  COSL_TRY(check_observations(prob));
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || opt->device < 0 || opt->device >= ndev)
    return set_error(COSL_E_CUDA, "CUDA device %d not available", opt->device);
  COSL_CUDA(cudaSetDevice(opt->device));
  cosl_ba_solver* s = new (std::nothrow) cosl_ba_solver();
  if (!s) return set_error(COSL_E_NOMEM, "host allocation failed");
  s->opt = *opt;
  s->comm = comm;
  s->device = opt->device;
  cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete s;
    return set_error(COSL_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
  }
  pool_keep(opt->device);
  const double tBuild0 = now_s();
  const int rc = build_solver(s, prob);
  if (ba_timing()) std::fprintf(stderr, "[ba timing] build_solver %.1f ms\n", 1e3 * (now_s() - tBuild0));
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
  if (!prob || prob->m != s->m || prob->n != s->n)
    return set_error(COSL_E_INVALID, "cosl_ba_solver_reset: problem shape changed");
  s->timer.reset();
  return upload_params(s, prob);
}

int cosl_ba_solver_run(cosl_ba_solver* s, double info[COSL_BA_INFOSZ]) {
  BA_ENTER(s)
  return run_robust(s, 0, info);
}

int cosl_ba_solver_run_fixed(cosl_ba_solver* s, int trials, double info[COSL_BA_INFOSZ]) {
  BA_ENTER(s)
  return run_robust(s, trials < 1 ? 1 : trials, info);
}

int cosl_ba_solver_download(cosl_ba_solver* s, cosl_ba_problem* prob) {
  BA_ENTER(s)
  if (!prob || prob->m != s->m || prob->n != s->n)
    return set_error(COSL_E_INVALID, "cosl_ba_solver_download: problem shape changed");
  return download(s, prob);
}

int cosl_ba_solver_destroy(cosl_ba_solver* s) {
  free_solver(s);
  return COSL_OK;
}

void* cosl_ba_solver_stream(cosl_ba_solver* s) { return s ? (void*)s->stream : nullptr; }

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
  out[6] = s->solveGrid;
  out[7] = s->twoSolve ? 1 : 0;
  return COSL_OK;
}

// diagnostic: per-task timeline of the LAST persistent solve launch.  enable -> run -> get.
// out: [nTasks][8] = sm id, globaltimer ns at ticket / operands ready / done, 4 phase stamps; meta: [nTasks][3] =
// task type, pivot block k, row block i.
int cosl_ba_solver_trace(cosl_ba_solver* s, int enable, uint64_t* out, int32_t* meta, int cap) {
  BA_ENTER(s)
  const int nt = (int)s->plan.tasks.size();
  if (enable) {
    if (!s->d_trace) COSL_TRY(dev_alloc(s->stream, &s->d_trace, (size_t)std::max(1, nt) * 8));
    COSL_CUDA(cudaMemsetAsync(s->d_trace, 0, sizeof(unsigned long long) * 8 * std::max(1, nt), s->stream));
    s->td.trace = s->d_trace;
    return nt;
  }
  if (out && s->d_trace) {
    const int n = std::min(cap, nt);
    COSL_CUDA(cudaMemcpyAsync(out, s->d_trace, sizeof(uint64_t) * 8 * n, cudaMemcpyDeviceToHost, s->stream));
    COSL_CUDA(cudaStreamSynchronize(s->stream));
    if (meta)
      for (int t = 0; t < n; ++t) {
        meta[3 * t] = s->taskOrder[t].type;
        meta[3 * t + 1] = s->taskOrder[t].k;
        meta[3 * t + 2] = s->taskOrder[t].i;
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
    BaTask k = s->taskOrder[t];
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
  std::vector<BaTask> tasks;
  const int nA = tile_task_order(P, tasks);
  const int nb = P.nb;
  const size_t ns = 6 * (size_t)mf, nScratch = (size_t)std::max(1, P.nScratch);
  const size_t nCnt = (size_t)P.nCounters + 2 + tasks.size();
  // the lower triangle of the permuted system, placed as build_solver's pair_dst places the Schur
  // blocks: the camera later in the elimination order owns the rows; fill and padding stay zero
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
  for (int a = 0; a < mf; ++a)
    for (int r = 0; r < 6; ++r) hRhs[(size_t)P.camBlk[a] * BA_TB + P.camOff[a] + r] = b[6 * a + r];
  int device = 0;
  COSL_CUDA(cudaGetDevice(&device));
  cudaStream_t s = cudaStreamPerThread;
  TmpDeviceBufs tmp(s);
  double *dRhs, *dTiles, *dRhsS, *dLinv, *dY, *dX, *dFail;
  int *dCnt, *dBlkRows;
  BaTask* dTasks;
  BaBwdEntry* dBwd;
  BaSumEntry* dSum;
  COSL_TRY(tmp.alloc(&dRhs, (size_t)nb * BA_TB));
  COSL_TRY(tmp.alloc(&dTiles, ((size_t)P.nTiles + P.nScratch) * BA_TILE));
  COSL_TRY(tmp.alloc(&dRhsS, nScratch * BA_TB));
  COSL_TRY(tmp.alloc(&dLinv, (size_t)nb * BA_TILE));
  COSL_TRY(tmp.alloc(&dY, (size_t)nb * BA_TB));
  COSL_TRY(tmp.alloc(&dX, (size_t)nb * BA_TB));
  COSL_TRY(tmp.alloc(&dFail, 1));
  COSL_TRY(tmp.alloc(&dCnt, nCnt));
  COSL_TRY(tmp.alloc(&dBlkRows, (size_t)nb));
  COSL_TRY(tmp.alloc(&dTasks, tasks.size()));
  COSL_TRY(tmp.alloc(&dBwd, P.bwdList.size()));
  COSL_TRY(tmp.alloc(&dSum, P.sumList.size()));
  COSL_CUDA(cudaMemcpyAsync(dRhs, hRhs.data(), 8 * hRhs.size(), cudaMemcpyHostToDevice, s));
  COSL_CUDA(cudaMemcpyAsync(dTiles, hTiles.data(), 8 * hTiles.size(), cudaMemcpyHostToDevice, s));
  // scratch tiles and their rhs parts start as NaN: their first update must overwrite them
  COSL_CUDA(cudaMemsetAsync(dTiles + (size_t)P.nTiles * BA_TILE, 0xff, 8 * (size_t)P.nScratch * BA_TILE, s));
  COSL_CUDA(cudaMemsetAsync(dRhsS, 0xff, 8 * nScratch * BA_TB, s));
  COSL_CUDA(cudaMemsetAsync(dCnt, 0, 4 * nCnt, s));
  COSL_CUDA(cudaMemsetAsync(dFail, 0, 8, s));
  COSL_CUDA(cudaMemcpyAsync(dBlkRows, P.blkRows.data(), 4 * (size_t)nb, cudaMemcpyHostToDevice, s));
  COSL_CUDA(cudaMemcpyAsync(dTasks, tasks.data(), sizeof(BaTask) * tasks.size(), cudaMemcpyHostToDevice, s));
  if (!P.bwdList.empty())
    COSL_CUDA(cudaMemcpyAsync(dBwd, P.bwdList.data(), sizeof(BaBwdEntry) * P.bwdList.size(), cudaMemcpyHostToDevice, s));
  if (!P.sumList.empty())
    COSL_CUDA(cudaMemcpyAsync(dSum, P.sumList.data(), sizeof(BaSumEntry) * P.sumList.size(), cudaMemcpyHostToDevice, s));
  const TileSolveBufs tb = {dRhs, dTiles, dRhsS, dLinv, dY, dX, dCnt, dTasks, dBwd, dSum, dBlkRows, dFail};
  int grid = 0;
  COSL_TRY(tile_solve_launch(P, nA, tb, device, s, &grid));
  std::vector<double> hX((size_t)nb * BA_TB);
  double hFail = 0.0;
  COSL_CUDA(cudaMemcpyAsync(hX.data(), dX, 8 * hX.size(), cudaMemcpyDeviceToHost, s));
  COSL_CUDA(cudaMemcpyAsync(&hFail, dFail, 8, cudaMemcpyDeviceToHost, s));
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
  out[6] = grid;
  out[7] = grid == 1 ? 1 : 0;
  return COSL_OK;
}

int cosl_ba_solver_profile_enable(cosl_ba_solver* s, int on) {
  BA_ENTER(s)
  COSL_CUDA(cudaStreamSynchronize(s->stream));
  s->timer.reset();
  s->timer.enabled = on != 0;
  return COSL_OK;
}

const char* cosl_ba_solver_timer(cosl_ba_solver* s, int idx, double* ms, int* calls) {
  if (!s || idx < 0 || idx >= s->timer.nsec) return nullptr;
  cudaSetDevice(s->device);
  cudaStreamSynchronize(s->stream);
  s->timer.flush();
  if (ms) *ms = s->timer.ms[idx];
  if (calls) *calls = s->timer.calls[idx];
  return s->timer.names[idx];
}

int cosl_ba_solve(cosl_ba_problem* prob, const cosl_ba_options* opt,
                  double info[COSL_BA_INFOSZ]) {
  cosl_ba_solver* s = nullptr;
  const double t0 = now_s();
  COSL_TRY(cosl_ba_solver_create(prob, opt, nullptr, &s));
  const double t1 = now_s();
  int rc = run_robust(s, 0, info);
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
  cosl_ba_options o;
  cosl_ba_options_default(&o);
  o.max_err = 0;
  o.outer_iters = 1;
  o.inner_iters = itmax;
  for (int k = 0; k < 5; ++k) o.opts[k] = opts[k];
  o.verbose = verbose;
  o.device = device;
  double inf[COSL_BA_INFOSZ];
  COSL_TRY(cosl_ba_solve(&pr, &o, inf));
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
