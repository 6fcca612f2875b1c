// Shared helpers for libvidar_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/vidar_b200.h"

namespace vidar {

// thread-local last-error text (vidar_last_error)
char* err_buf();
int set_error(int code, const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

// Stream-ordered scratch (cudaMallocFromPoolAsync / cudaFreeAsync) for the MSDA row order and the LatentRendering
// cell order comes from this memory pool of the library, one per device.  It keeps what it has allocated (release
// threshold = max): eager training does not pay a fresh physical allocation per backward, and the device's default
// pool, which the rest of the process may use, keeps its settings.  No host sync, and a CUDA graph captures the
// allocations as nodes, so the C signatures need no workspace argument.
cudaError_t scratch_pool(cudaMemPool_t* pool);

inline int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return set_error(VIDAR_E_CUDA, "%s: launch failed: %s", what, cudaGetErrorString(e));
  return VIDAR_OK;
}

#define VIDAR_REQUIRE(cond, ...)                                   \
  do {                                                             \
    if (!(cond)) return ::vidar::set_error(VIDAR_E_INVALID, __VA_ARGS__); \
  } while (0)

// SMs of the current device (132 on an H100 SXM): sizes the persistent grids.  Grid sizes only
// set how work is spread, never what is computed.
inline int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      n <= 0) {
    cudaGetLastError();
    return 132;
  }
  return n;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

// red.global.add.v4.f32 (sm_90+): one 16-byte vector reduction instead of four scalars.
__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}

__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// Segment of a flat index: the largest n with off[n] <= p, for off[0] <= p < off[N] (empty segments are skipped).
__device__ __forceinline__ int find_segment(const int64_t* __restrict__ off, int N, int64_t p) {
  int lo = 0, hi = N;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= p) lo = mid; else hi = mid;
  }
  return lo;
}

// Fixed-order fp64 sum over a block of kThreads threads (warp tree, then the warps in order); the result is valid
// in thread 0.  `red`: kThreads / 32 doubles of shared memory.
template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}

}  // namespace vidar
