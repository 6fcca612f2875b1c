// Error reporting / identification for libvidar_b200.so.
#include <stdarg.h>
#include <string.h>

#include <mutex>

#include "common.cuh"

namespace vidar {

std::atomic<int64_t> g_launches{0};

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

cudaError_t scratch_pool(cudaMemPool_t* pool) {
  static std::mutex mu;
  static cudaMemPool_t pools[128] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 128) return cudaErrorInvalidDevice;
  std::lock_guard<std::mutex> lock(mu);
  if (!pools[dev]) {
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t p = nullptr;
    e = cudaMemPoolCreate(&p, &props);
    if (e != cudaSuccess) return e;
    uint64_t keep = UINT64_MAX;
    e = cudaMemPoolSetAttribute(p, cudaMemPoolAttrReleaseThreshold, &keep);
    if (e != cudaSuccess) {
      cudaMemPoolDestroy(p);
      return e;
    }
    pools[dev] = p;
  }
  *pool = pools[dev];
  return cudaSuccess;
}

}  // namespace vidar

extern "C" const char* vidar_last_error(void) { return vidar::err_buf(); }
extern "C" const char* vidar_version(void) { return "vidar_b200 0.1 sm_90a"; }
extern "C" int64_t vidar_launch_count(void) {
  return vidar::g_launches.load(std::memory_order_relaxed);
}
