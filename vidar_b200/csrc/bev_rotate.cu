// TemporalSelfAttention's value with ego motion (modules/transformer.py:137-150, modules/encoder.py:225-229): the
// previous BEV rotated by the frame's yaw change and stacked with the query, [bs, Q, C] x 2 -> [bs * 2, Q, C], in one
// pass.  The reference permutes each sample's previous BEV to [C, H, W], rotates it with torchvision's nearest
// `rotate`, permutes it back and stacks it with the query; that is a gather of whole channel rows, so here it is one.
//
// rows [bs, Q] int32 is the row map: output cell q of sample b copies source cell rows[b, q] of that sample's previous
// BEV, or zeros where rows[b, q] is outside [0, Q) (-1 in the maps vidar_b200/ego_motion.py builds from
// torchvision's own statements); no value of rows reads or writes outside the buffers.
//   forward   value[2b, q] = 0 <= rows[b, q] < Q ? prev[b, rows[b, q]] : 0,  value[2b + 1, q] = query[b, q]
//   backward  grad_prev[b, s] = sum of grad_value[2b, q] over the q with rows[b, q] = s, in ascending q,
//             grad_query[b, q] = grad_value[2b + 1, q]
// The backward's inverse map is a stable radix sort of (source, output) pairs: each source cell's outputs form one
// run in ascending q, so every source cell sums its (at most a few) rows in a fixed order, with no float atomics and
// bit-identical results from call to call.  C is a multiple of 4; one thread moves one float4 of one cell.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) bev_rotate_stack_fwd_kernel(const float* __restrict__ prev,
                                                                        const float* __restrict__ query,
                                                                        const int* __restrict__ rows,
                                                                        float* __restrict__ value, int Q, int C4,
                                                                        long long n) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;      // over bs * Q * C4
  if (t >= n) return;
  const int c = (int)(t % C4);
  const long long bq = t / C4;                                             // b * Q + q
  const long long b = bq / Q, q = bq - b * Q;
  const int src = __ldg(rows + bq);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (src >= 0 && src < Q) v = ldg4(prev + ((b * Q + src) * C4 + c) * 4);
  float4* out = reinterpret_cast<float4*>(value);
  out[((2 * b) * Q + q) * C4 + c] = v;
  out[((2 * b + 1) * Q + q) * C4 + c] = ldg4(query + (bq * C4 + c) * 4);
}

// keys: b * Q + rows[b, q] (bs * Q for a zero-filled cell -- rows outside [0, Q) -- sorted last), values: the output
// cell b * Q + q
__global__ void bev_rotate_keys_kernel(const int* __restrict__ rows, int Q, int n, unsigned* __restrict__ key,
                                       int* __restrict__ val) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const int src = rows[i];
  key[i] = src >= 0 && src < Q ? (unsigned)((i / Q) * Q + src) : (unsigned)n;
  val[i] = i;
}

// run bounds of each source cell in the sorted keys; begin / end are zeroed before (no run: empty)
__global__ void bev_rotate_runs_kernel(const unsigned* __restrict__ key, int n, int* __restrict__ begin,
                                       int* __restrict__ end) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const unsigned k = key[i];
  if (k >= (unsigned)n) return;
  if (i == 0 || key[i - 1] != k) begin[k] = i;
  if (i == n - 1 || key[i + 1] != k) end[k] = i + 1;
}

__global__ void __launch_bounds__(kThreads) bev_rotate_stack_bwd_kernel(const float* __restrict__ grad_value,
                                                                        const int* __restrict__ order,
                                                                        const int* __restrict__ begin,
                                                                        const int* __restrict__ end,
                                                                        float* __restrict__ grad_prev,
                                                                        float* __restrict__ grad_query, int Q, int C4,
                                                                        long long n) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;      // over bs * Q * C4
  if (t >= n) return;
  const int c = (int)(t % C4);
  const long long s = t / C4;                                              // b * Q + source cell
  const long long b = s / Q;
  const float4* g = reinterpret_cast<const float4*>(grad_value);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = begin[s]; i < end[s]; ++i) {
    const long long o = order[i];                                          // b * Q + q, ascending q
    const float4 v = __ldg(g + ((o + b * Q) * C4 + c));                    // row (2b) * Q + q
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  reinterpret_cast<float4*>(grad_prev)[s * C4 + c] = acc;
  reinterpret_cast<float4*>(grad_query)[s * C4 + c] = __ldg(g + ((s + (b + 1) * Q) * C4 + c));   // row (2b+1) * Q + q
}

int check_args(const char* who, int bs, int Q, int C, const void* a, const void* b, const void* c, const void* d,
               const void* e) {
  VIDAR_REQUIRE(bs > 0 && Q > 0 && C > 0 && C % 4 == 0, "%s: bad sizes (bs %d, Q %d, C %d; C must be a multiple of 4)",
                who, bs, Q, C);
  VIDAR_REQUIRE((long long)bs * Q < (1LL << 31) - 1, "%s: bs * Q = %lld cells is too many", who, (long long)bs * Q);
  VIDAR_REQUIRE(a && b && c && d && e, "%s: null pointer argument", who);
  VIDAR_REQUIRE(((uintptr_t)a | (uintptr_t)b | (uintptr_t)d | (uintptr_t)e) % 16 == 0 && (uintptr_t)c % 4 == 0,
                "%s: the float buffers must be 16-byte aligned, rows 4-byte aligned", who);
  return VIDAR_OK;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_bev_rotate_stack_forward(const float* prev, const float* query, const int32_t* rows, float* value,
                                              int bs, int Q, int C, void* stream) {
  const char* who = "bev_rotate_stack_forward";
  if (int rc = check_args(who, bs, Q, C, prev, query, rows, value, value)) return rc;
  const long long n = (long long)bs * Q * (C / 4);
  VIDAR_REQUIRE((n + kThreads - 1) / kThreads < (1LL << 31), "%s: too many cells", who);
  bev_rotate_stack_fwd_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      prev, query, rows, value, Q, C / 4, n);
  return check_launch(who);
}

extern "C" int vidar_bev_rotate_stack_backward(const float* grad_value, const int32_t* rows, float* grad_prev,
                                               float* grad_query, int bs, int Q, int C, void* stream) {
  const char* who = "bev_rotate_stack_backward";
  if (int rc = check_args(who, bs, Q, C, grad_value, grad_prev, rows, grad_query, grad_value)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int n = bs * Q;
  const long long m = (long long)n * (C / 4);
  VIDAR_REQUIRE((m + kThreads - 1) / kThreads < (1LL << 31), "%s: too many cells", who);
  int bits = 1;
  while ((1LL << bits) <= n) ++bits;                                       // keys 0 .. n
  size_t tmp = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, tmp, (const unsigned*)nullptr, (unsigned*)nullptr,
                                                  (const int*)nullptr, (int*)nullptr, n, 0, bits, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: source order: %s", who, cudaGetErrorString(e));
  const size_t off = ((sizeof(unsigned) + sizeof(int)) * 2 * (size_t)n + 2 * sizeof(int) * (size_t)n + 255) &
                     ~(size_t)255;
  cudaMemPool_t pool;
  e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, off + tmp, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  unsigned* k0 = reinterpret_cast<unsigned*>(s);
  unsigned* k1 = k0 + n;
  int* v0 = reinterpret_cast<int*>(k1 + n);
  int* v1 = v0 + n;
  int* begin = v1 + n;
  int* end = begin + n;
  const unsigned blocks = (unsigned)((n + kThreads - 1) / kThreads);
  e = cudaMemsetAsync(begin, 0, 2 * sizeof(int) * (size_t)n, st);
  if (e == cudaSuccess) {
    bev_rotate_keys_kernel<<<blocks, kThreads, 0, st>>>(rows, Q, n, k0, v0);
    e = cub::DeviceRadixSort::SortPairs(s + off, tmp, k0, k1, v0, v1, n, 0, bits, st);
  }
  if (e == cudaSuccess) {
    bev_rotate_runs_kernel<<<blocks, kThreads, 0, st>>>(k1, n, begin, end);
    bev_rotate_stack_bwd_kernel<<<(unsigned)((m + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        grad_value, v1, begin, end, grad_prev, grad_query, Q, C / 4, m);
  }
  const cudaError_t ef = cudaFreeAsync(s, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: source order: %s", who, cudaGetErrorString(e));
  if (ef != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(ef));
  return check_launch(who);
}
