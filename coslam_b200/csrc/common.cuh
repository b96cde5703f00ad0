// common.cuh -- shared host/device helpers of libcoslam_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/coslam_b200.h"

namespace coslam {

// ---- error plumbing: the C-ABI never throws, every failure sets a thread-local message ----
std::string& last_error_ref();
int set_error(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define COSL_CUDA(expr)                                                                       \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return coslam::set_error(COSL_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                             __FILE__, __LINE__);                                             \
  } while (0)

#define COSL_TRY(expr)            \
  do {                            \
    int _rc = (expr);             \
    if (_rc != COSL_OK) return _rc; \
  } while (0)

// every kernel launch of this library goes through this macro so that gpu_launches is a count,
// not an estimate
#define COSL_LAUNCH(kernel, grid, block, smem, stream, ...)            \
  do {                                                                 \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);        \
    coslam::g_launches.fetch_add(1, std::memory_order_relaxed);          \
  } while (0)

// COSL_LAUNCH as a programmatic dependent launch: the kernel may be scheduled as soon as every CTA
// of the kernel before it on stream `strm` has executed griddepcontrol.launch_dependents or exited,
// so its launch and prologue overlap that kernel's drain.  The kernel must execute griddepcontrol.wait
// (it returns once the earlier grid has completed and its memory is visible) before it touches
// anything that grid or the work ahead of it on `strm` writes or reads.  Returns from the
// enclosing function on a launch error.
#define COSL_LAUNCH_PDL(kernel, grid, block, smem, strm, ...)                      \
  do {                                                                             \
    cudaLaunchAttribute _attr[1];                                                  \
    _attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;              \
    _attr[0].val.programmaticStreamSerializationAllowed = 1;                       \
    cudaLaunchConfig_t _cfg = {};                                                  \
    _cfg.gridDim = (grid);                                                         \
    _cfg.blockDim = (block);                                                       \
    _cfg.dynamicSmemBytes = (smem);                                                \
    _cfg.stream = (strm);                                                          \
    _cfg.attrs = _attr;                                                            \
    _cfg.numAttrs = 1;                                                             \
    coslam::g_launches.fetch_add(1, std::memory_order_relaxed);                    \
    COSL_CUDA(cudaLaunchKernelEx(&_cfg, kernel, __VA_ARGS__));                     \
  } while (0)

inline int div_up(int a, int b) { return (a + b - 1) / b; }
inline int64_t div_up64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// COSL_E_CUDA unless `device` is the ordinal of a visible CUDA device.
int check_device(int device);

// Gives the device's default memory pool an unlimited release threshold, once per device: after the first
// request, cudaMallocAsync hands out buffers again without a device synchronisation or a trip to the driver's
// allocator (cudaMalloc / cudaFree cost more than the kernels; cosl_ba_solve makes ~30 buffers, 0.7 GB at c4,
// per call).
void keep_pool(int device);

// One request in flight on a handle's own non-blocking stream: the pose, pose-graph and BA solver handles.
// evStart and evDone bracket the request's work.  The caller makes the handle's device current before
// create / destroy / submit / query / wait, and calls idle / pending where its checks put the state check.
struct RequestStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t evStart = nullptr, evDone = nullptr;
  bool inFlight = false;

  int create();    // on the current device; destroy() cleans up after a failure
  void destroy();  // waits for the stream first: a request in flight uses the handle's buffers
  int idle(const char* fn) const;     // COSL_E_STATE while a request is in flight
  int pending(const char* fn) const;  // COSL_E_STATE with nothing in flight
  int query(int* done);               // *done = 1 once the request has finished, without waiting
  int wait(double* device_ms);        // nothing is in flight afterwards; device_ms (nullable): evStart -> evDone

  // Records evStart, runs `enqueue` (a COSL_ status), records evDone.  On a failure the stream is drained (a
  // copy that was enqueued may still read a staging buffer) and nothing is in flight.
  template <class F>
  int submit(const char* fn, F enqueue) {
    int rc = COSL_OK;
    cudaError_t e = cudaEventRecord(evStart, stream);
    if (e == cudaSuccess) {
      rc = enqueue();
      if (rc == COSL_OK) e = cudaEventRecord(evDone, stream);
    }
    if (rc == COSL_OK && e != cudaSuccess)
      rc = set_error(COSL_E_CUDA, "%s: cudaEventRecord: %s", fn, cudaGetErrorString(e));
    if (rc != COSL_OK) cudaStreamSynchronize(stream);
    else inFlight = true;
    return rc;
  }
};

// simple per-stream section timer (CUDA events), used to report per-kernel-class device time
struct SectionTimer {
  static const int kMaxSections = 16;
  static const int kMaxPending = 4096;
  const char* names[kMaxSections];
  double ms[kMaxSections];
  int calls[kMaxSections];
  int nsec = 0;
  bool enabled = false;
  cudaEvent_t ev[kMaxPending][2];
  int pend_sec[kMaxPending];
  int npend = 0, nalloc = 0;
  int open_sec = -1;

  int section(const char* name) {
    for (int i = 0; i < nsec; ++i)
      if (!std::strcmp(names[i], name)) return i;
    if (nsec >= kMaxSections) return nsec - 1;
    names[nsec] = name;
    ms[nsec] = 0;
    calls[nsec] = 0;
    return nsec++;
  }
  void begin(int sec, cudaStream_t s) {
    if (!enabled) return;
    if (npend >= kMaxPending) flush();
    if (npend >= nalloc) {
      cudaEventCreate(&ev[nalloc][0]);
      cudaEventCreate(&ev[nalloc][1]);
      ++nalloc;
    }
    cudaEventRecord(ev[npend][0], s);
    pend_sec[npend] = sec;
    open_sec = sec;
  }
  void end(cudaStream_t s) {
    if (!enabled || open_sec < 0) return;
    cudaEventRecord(ev[npend][1], s);
    ++npend;
    open_sec = -1;
  }
  void flush() {  // requires the stream to be idle or will block on the last event
    for (int i = 0; i < npend; ++i) {
      cudaEventSynchronize(ev[i][1]);
      float t = 0;
      cudaEventElapsedTime(&t, ev[i][0], ev[i][1]);
      ms[pend_sec[i]] += t;
      calls[pend_sec[i]] += 1;
    }
    npend = 0;
  }
  void reset() {
    flush();
    for (int i = 0; i < nsec; ++i) {
      ms[i] = 0;
      calls[i] = 0;
    }
  }
  void destroy() {
    for (int i = 0; i < nalloc; ++i) {
      cudaEventDestroy(ev[i][0]);
      cudaEventDestroy(ev[i][1]);
    }
    nalloc = 0;
    npend = 0;
  }
};

}  // namespace coslam
