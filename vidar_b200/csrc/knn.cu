// Nearest-neighbour (K = 1) search and its backward for the Chamfer distance, H100 (sm_90a).
//
// Reference: third_lib/chamfer_dist/chamferdist/chamferdist/knn.cu:21-260 (brute-force KNN,
// 256 blocks x 256 threads, every thread scans all of P2 from global memory), knn_cpu.cpp:7-106,
// used with K = 1 by ChamferDistance (chamfer.py:20-133) for ViDAR's evaluation metric
// (bevformer/utils/e2e_predictor_utils.py:163-183) -- SURVEY.md 8(f) item 2.
// dist = sum_d (p1 - p2)^2 accumulated in d order like the CPU reference; ties keep the
// smallest index (the CPU loop keeps the first strictly-smaller candidate).
//
// Mapping: a thread owns one p1 point; p2 streams through shared memory in 1024-point tiles
// (12 KB, read once per block instead of once per thread), and P2 is additionally split over
// blockIdx.y so 30k x 30k points fill all 132 SMs; partial results merge with one 64-bit
// atomicMin on (distance bits << 32 | index) -- non-negative floats order like unsigned ints.
#include "common.cuh"

namespace vidar {
namespace {

constexpr int kNnThreads = 256;
constexpr int kNnTile = 1024;

// The inner loop shared by the batched and the segmented search: scan `cnt` candidates of a shared-memory
// tile whose first point has index `base`, keeping the first strictly smaller squared distance.
template <int D>
__device__ __forceinline__ void nn_scan_tile(const float (&a)[D], const float* tile, int cnt, int base, float& bd,
                                             int& bi) {
  for (int j = 0; j < cnt; ++j) {
    float dist = 0.f;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      const float diff = a[d] - tile[j * D + d];
      dist = __fadd_rn(dist, __fmul_rn(diff, diff));     // `dist += diff * diff`, no contraction
    }
    if (dist < bd) { bd = dist; bi = base + j; }
  }
}

template <int D>
__global__ void __launch_bounds__(kNnThreads)
nn_forward_kernel(const float* __restrict__ p1, const float* __restrict__ p2,
                  const int64_t* __restrict__ len1, const int64_t* __restrict__ len2,
                  unsigned long long* __restrict__ best, int N, int P1, int P2, int splits) {
  __shared__ float tile[kNnTile * D];
  const int n = blockIdx.z;
  const int i = blockIdx.x * kNnThreads + threadIdx.x;
  const int L1 = len1 ? (int)len1[n] : P1;
  const int L2 = len2 ? (int)len2[n] : P2;
  const int chunk = (L2 + splits - 1) / splits;
  const int j0 = blockIdx.y * chunk, j1 = min(L2, j0 + chunk);
  if (j0 >= j1) return;
  float a[D];
  const bool live = i < L1;
#pragma unroll
  for (int d = 0; d < D; ++d) a[d] = live ? p1[((size_t)n * P1 + i) * D + d] : 0.f;
  float bd = INFINITY;
  int bi = 0;
  for (int t0 = j0; t0 < j1; t0 += kNnTile) {
    const int cnt = min(kNnTile, j1 - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * D; e += kNnThreads) tile[e] = p2[((size_t)n * P2 + t0) * D + e];
    __syncthreads();
    if (live) nn_scan_tile<D>(a, tile, cnt, t0, bd, bi);
  }
  if (live) {
    const unsigned long long key = ((unsigned long long)__float_as_uint(bd) << 32) | (unsigned)bi;
    atomicMin(best + (size_t)n * P1 + i, key);
  }
}

__global__ void nn_unpack_kernel(const unsigned long long* __restrict__ best, const int64_t* __restrict__ len1,
                                 const int64_t* __restrict__ len2, float* __restrict__ dists,
                                 int64_t* __restrict__ idx, int N, int P1, int P2) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * P1) return;
  const int n = (int)(t / P1), i = (int)(t % P1);
  const int L1 = len1 ? (int)len1[n] : P1;
  const int L2 = len2 ? (int)len2[n] : P2;
  const unsigned long long key = best[t];
  const bool ok = i < L1 && L2 > 0 && key != ~0ull;
  dists[t] = ok ? __uint_as_float((unsigned)(key >> 32)) : 0.f;     // zero padding like the reference
  idx[t] = ok ? (int64_t)(unsigned)(key & 0xffffffffu) : 0;
}

template <int D>
__global__ void nn_backward_kernel(const float* __restrict__ p1, const float* __restrict__ p2,
                                   const int64_t* __restrict__ len1, const int64_t* __restrict__ len2,
                                   const int64_t* __restrict__ idx, const float* __restrict__ grad_dists,
                                   float* __restrict__ grad_p1, float* __restrict__ grad_p2, int N, int P1,
                                   int P2) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * P1) return;
  const int n = (int)(t / P1), i = (int)(t % P1);
  const int L1 = len1 ? (int)len1[n] : P1;
  const int L2 = len2 ? (int)len2[n] : P2;
  if (i >= L1 || L2 < 1) return;
  const int64_t j = idx[t];
  const float g = grad_dists[t];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float diff = 2.0f * g * (p1[t * D + d] - p2[((size_t)n * P2 + j) * D + d]);
    grad_p1[t * D + d] = diff;                                 // caller-zeroed, one writer
    red_add_f32(grad_p2 + ((size_t)n * P2 + j) * D + d, -diff);
  }
}

// Segmented search: segment s pairs queries [q_off[s], q_off[s+1]) with candidates [c_off[s], c_off[s+1]),
// blockIdx.z = s, so ragged clouds of one call share a launch.  A masked candidate enters the tile as +inf and
// can never be strictly nearer than the running best (valid points are finite); a masked query writes nothing.
constexpr unsigned long long kNnNone = ~0ull;

__global__ void __launch_bounds__(kNnThreads)
nn_segments_kernel(const float* __restrict__ q, const float* __restrict__ c, const int64_t* __restrict__ q_off,
                   const int64_t* __restrict__ c_off, const unsigned char* __restrict__ q_mask,
                   const unsigned char* __restrict__ c_mask, unsigned long long* __restrict__ best, int splits) {
  __shared__ float tile[kNnTile * 3];
  const int s = blockIdx.z;
  const int64_t q0 = q_off[s], c0 = c_off[s];
  const int Lq = (int)(q_off[s + 1] - q0), Lc = (int)(c_off[s + 1] - c0);
  const int i = blockIdx.x * kNnThreads + threadIdx.x;
  if ((int)blockIdx.x * kNnThreads >= Lq) return;
  const int chunk = (Lc + splits - 1) / splits;
  const int j0 = blockIdx.y * chunk, j1 = min(Lc, j0 + chunk);
  if (j0 >= j1) return;
  float a[3];
  const bool live = i < Lq && (!q_mask || q_mask[q0 + i]);
  if (!__syncthreads_or(live)) return;      // a block of masked queries only: no tile to scan
#pragma unroll
  for (int d = 0; d < 3; ++d) a[d] = live ? q[(q0 + i) * 3 + d] : 0.f;
  float bd = INFINITY;
  int bi = 0;
  for (int t0 = j0; t0 < j1; t0 += kNnTile) {
    const int cnt = min(kNnTile, j1 - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * 3; e += kNnThreads) {
      const int64_t g = c0 + t0 + e / 3;
      tile[e] = (!c_mask || c_mask[g]) ? c[(c0 + t0) * 3 + e] : INFINITY;
    }
    __syncthreads();
    if (live) nn_scan_tile<3>(a, tile, cnt, t0, bd, bi);
  }
  if (live && bd < INFINITY) atomicMin(best + q0 + i, ((unsigned long long)__float_as_uint(bd) << 32) | (unsigned)bi);
}

__global__ void nn_segments_unpack_kernel(const unsigned long long* __restrict__ best,
                                          const unsigned char* __restrict__ q_mask, float* __restrict__ dists,
                                          int64_t* __restrict__ idx, long long Pq) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Pq) return;
  const unsigned long long key = best[t];
  const bool masked = q_mask && !q_mask[t];
  const bool ok = !masked && key != kNnNone;
  dists[t] = ok ? __uint_as_float((unsigned)(key >> 32)) : 0.f;
  idx[t] = ok ? (int64_t)(unsigned)(key & 0xffffffffu) : (masked ? VIDAR_NN_MASKED : VIDAR_NN_EMPTY);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_nn_segments_forward(const float* q, const float* c, const int64_t* q_off, const int64_t* c_off,
                                         const unsigned char* q_mask, const unsigned char* c_mask, float* dists,
                                         int64_t* idx, unsigned long long* scratch, int S, long long Pq,
                                         int max_q, int max_c, void* stream) {
  VIDAR_REQUIRE(q_off && c_off, "nn_segments: null pointer argument");
  VIDAR_REQUIRE(S > 0 && S <= 65535 && Pq >= 0 && max_q >= 0 && max_c >= 0,
                "nn_segments: bad sizes S=%d Pq=%lld max_q=%d max_c=%d", S, Pq, max_q, max_c);
  VIDAR_REQUIRE(Pq == 0 || (q && dists && idx && scratch), "nn_segments: null query / output buffer");
  VIDAR_REQUIRE(max_c == 0 || c, "nn_segments: null candidate buffer");
  if (Pq == 0) return VIDAR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0xff, sizeof(unsigned long long) * (size_t)Pq, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "nn_segments: memset: %s", cudaGetErrorString(e));
  if (max_q > 0 && max_c > 0) {
    const int bx = (max_q + kNnThreads - 1) / kNnThreads;
    // the same occupancy rule as vidar_nn_forward, with the longest segments standing for all of them
    int splits = (4 * num_sms() + bx * S - 1) / (bx * S);
    const int max_splits = (max_c + kNnTile - 1) / kNnTile;
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    nn_segments_kernel<<<dim3(bx, splits, S), kNnThreads, 0, st>>>(q, c, q_off, c_off, q_mask, c_mask, scratch, splits);
    int rc = check_launch("nn_segments");
    if (rc) return rc;
  }
  nn_segments_unpack_kernel<<<(unsigned)((Pq + 255) / 256), 256, 0, st>>>(scratch, q_mask, dists, idx, Pq);
  return check_launch("nn_segments(unpack)");
}

extern "C" int vidar_nn_forward(const float* p1, const float* p2, const int64_t* lengths1,
                                const int64_t* lengths2, float* dists, int64_t* idx,
                                unsigned long long* scratch, int N, int P1, int P2, int D, void* stream) {
  VIDAR_REQUIRE(p1 && p2 && dists && idx && scratch, "knn_points: null pointer argument");
  VIDAR_REQUIRE(N > 0 && P1 > 0 && P2 > 0, "knn_points: bad sizes N=%d P1=%d P2=%d", N, P1, P2);
  VIDAR_REQUIRE(D == 2 || D == 3 || D == 4, "knn_points: point dimension %d unsupported (2, 3 or 4)", D);
  VIDAR_REQUIRE(N <= 65535, "knn_points: batch too large");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(scratch, 0xff, sizeof(unsigned long long) * (size_t)N * P1, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "knn_points: memset: %s", cudaGetErrorString(e));
  const int bx = (P1 + kNnThreads - 1) / kNnThreads;
  // enough (block x split) pairs for ~4 waves of the device's SMs, at least one tile per split
  int splits = (4 * num_sms() + bx * N - 1) / (bx * N);
  const int max_splits = (P2 + kNnTile - 1) / kNnTile;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const dim3 grid(bx, splits, N);
  if (D == 3) nn_forward_kernel<3><<<grid, kNnThreads, 0, st>>>(p1, p2, lengths1, lengths2, scratch, N, P1, P2, splits);
  else if (D == 2) nn_forward_kernel<2><<<grid, kNnThreads, 0, st>>>(p1, p2, lengths1, lengths2, scratch, N, P1, P2, splits);
  else nn_forward_kernel<4><<<grid, kNnThreads, 0, st>>>(p1, p2, lengths1, lengths2, scratch, N, P1, P2, splits);
  int rc = check_launch("knn_points");
  if (rc) return rc;
  const long long total = (long long)N * P1;
  nn_unpack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(scratch, lengths1, lengths2, dists, idx, N, P1, P2);
  return check_launch("knn_points(unpack)");
}

extern "C" int vidar_nn_backward(const float* p1, const float* p2, const int64_t* lengths1,
                                 const int64_t* lengths2, const int64_t* idx, const float* grad_dists,
                                 float* grad_p1, float* grad_p2, int N, int P1, int P2, int D, void* stream) {
  VIDAR_REQUIRE(p1 && p2 && idx && grad_dists && grad_p1 && grad_p2, "knn_points_backward: null pointer argument");
  VIDAR_REQUIRE(N > 0 && P1 > 0 && P2 > 0, "knn_points_backward: bad sizes");
  VIDAR_REQUIRE(D == 2 || D == 3 || D == 4, "knn_points_backward: point dimension %d unsupported", D);
  const long long total = (long long)N * P1;
  const unsigned nb = (unsigned)((total + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 3) nn_backward_kernel<3><<<nb, 256, 0, st>>>(p1, p2, lengths1, lengths2, idx, grad_dists, grad_p1, grad_p2, N, P1, P2);
  else if (D == 2) nn_backward_kernel<2><<<nb, 256, 0, st>>>(p1, p2, lengths1, lengths2, idx, grad_dists, grad_p1, grad_p2, N, P1, P2);
  else nn_backward_kernel<4><<<nb, 256, 0, st>>>(p1, p2, lengths1, lengths2, idx, grad_dists, grad_p1, grad_p2, N, P1, P2);
  return check_launch("knn_points_backward");
}
