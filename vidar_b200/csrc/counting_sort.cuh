// Stable counting sort of rows by a small integer key, shared by the head's dense loss / GT alignment
// (dense_chamfer.cu) and the evaluation's cloud decode (eval_metrics.cu).
//
// Rows are cut into chunks of kSortChunk, one row per thread of a kSortChunk-thread block; every (segment, key) slot
// gets its rows in their original order.  counts[(seg * nkeys + key) * nchunk + chunk]: per-chunk row counts, turned
// into exclusive offsets inside the slot by sort_offsets.  All threads of the block call these.
#pragma once
#include "common.cuh"

namespace vidar {

constexpr int kSortChunk = 1024;      // rows per block of the counting sort, one per thread (32 warps)

// Per warp and key, the number of lanes holding that key, written by the lowest such lane into
// hist[warp * nkeys + key]; returns the lane's rank among them.  hist must be zeroed before.
__device__ __forceinline__ int warp_frame_rank(int f, int F, int* hist) {
  const unsigned peers = __match_any_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31;
  if (f >= 0 && lane == __ffs(peers) - 1) hist[(threadIdx.x >> 5) * F + f] = __popc(peers);
  return __popc(peers & ((1u << lane) - 1u));
}

// key of this thread's row (-1: none) -> the chunk's per-key counts
__device__ __forceinline__ void sort_count(int key, int nkeys, int seg, int c, int nchunk, int* hist,
                                           int* __restrict__ counts) {
  for (int e = threadIdx.x; e < 32 * nkeys; e += kSortChunk) hist[e] = 0;
  __syncthreads();
  warp_frame_rank(key, nkeys, hist);
  __syncthreads();
  for (int g = threadIdx.x; g < nkeys; g += kSortChunk) {
    int n = 0;
    for (int w = 0; w < 32; ++w) n += hist[w * nkeys + g];
    counts[((size_t)seg * nkeys + g) * nchunk + c] = n;
  }
}

// key of this thread's row -> its rank among the chunk's rows of that key (meaningless for key < 0)
__device__ __forceinline__ int sort_rank(int key, int nkeys, int* hist) {
  for (int e = threadIdx.x; e < 32 * nkeys; e += kSortChunk) hist[e] = 0;
  __syncthreads();
  int pos = warp_frame_rank(key, nkeys, hist);
  __syncthreads();
  if (key >= 0)
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pos += hist[w * nkeys + key];
  return pos;
}

// One block: chunk counts -> exclusive chunk offsets inside each of the S slots, and off[0..S] the exclusive
// slot offsets (off[S] = rows kept).
__device__ inline void sort_offsets(int S, int nchunk, int* __restrict__ counts, int64_t* __restrict__ off) {
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    int acc = 0;
    for (int c = 0; c < nchunk; ++c) {
      const int v = counts[(size_t)s * nchunk + c];
      counts[(size_t)s * nchunk + c] = acc;
      acc += v;
    }
    off[s + 1] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    off[0] = 0;
    for (int s = 0; s < S; ++s) { acc += off[s + 1]; off[s + 1] = acc; }
  }
  __syncthreads();
}

}  // namespace vidar
