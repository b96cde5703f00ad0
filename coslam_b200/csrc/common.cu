// common.cu -- error plumbing, version, launch accounting and the solver handles' request stream of
// libcoslam_b200.
#include <mutex>

#include "common.cuh"

namespace coslam {

std::atomic<uint64_t> g_launches{0};

std::string& last_error_ref() {
  static thread_local std::string s;
  return s;
}

int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error_ref() = buf;
  return code;
}

int check_device(int device) {
  int ndev = 0;
  if (device < 0 || cudaGetDeviceCount(&ndev) != cudaSuccess || device >= ndev)
    return set_error(COSL_E_CUDA, "CUDA device %d not available", device);
  return COSL_OK;
}

void keep_pool(int device) {
  static std::mutex mu;
  static bool kept[64] = {};
  std::lock_guard<std::mutex> lk(mu);
  if (device < 0 || device >= 64 || kept[device]) return;
  kept[device] = true;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
}

int RequestStream::create() {
  COSL_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  COSL_CUDA(cudaEventCreate(&evStart));
  COSL_CUDA(cudaEventCreate(&evDone));
  return COSL_OK;
}

void RequestStream::destroy() {
  if (stream) cudaStreamSynchronize(stream);
  if (evStart) cudaEventDestroy(evStart);
  if (evDone) cudaEventDestroy(evDone);
  if (stream) cudaStreamDestroy(stream);
}

int RequestStream::idle(const char* fn) const {
  return inFlight ? set_error(COSL_E_STATE, "%s: a submitted solve is not collected yet", fn) : COSL_OK;
}

int RequestStream::pending(const char* fn) const {
  return inFlight ? COSL_OK : set_error(COSL_E_STATE, "%s: nothing submitted", fn);
}

int RequestStream::query(int* done) {
  const cudaError_t e = cudaEventQuery(evDone);
  if (e == cudaErrorNotReady) {
    *done = 0;
    return COSL_OK;
  }
  COSL_CUDA(e);
  *done = 1;
  return COSL_OK;
}

int RequestStream::wait(double* device_ms) {
  inFlight = false;
  COSL_CUDA(cudaEventSynchronize(evDone));
  if (device_ms) {
    float ms = 0.f;
    COSL_CUDA(cudaEventElapsedTime(&ms, evStart, evDone));
    *device_ms = ms;
  }
  return COSL_OK;
}

}  // namespace coslam

extern "C" {
const char* cosl_last_error(void) { return coslam::last_error_ref().c_str(); }
const char* cosl_version(void) { return "coslam_b200 0.1 (sm_90a)"; }
uint64_t cosl_kernel_launch_count(void) { return coslam::g_launches.load(); }
}
