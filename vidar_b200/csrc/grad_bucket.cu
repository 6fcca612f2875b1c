// One flat fp32 gradient bucket for the data-parallel all-reduce (vidar_b200/grad_bucket.py).
//
// pack:   bucket[offset_i + j] = grad_i[j] * scale_i   (grad_i NULL: 0)
// unpack: grad_i[j] = bucket[offset_i + j]
//
// The tensor table -- (pointer, numel, bucket offset, scale) per tensor -- travels as a __grid_constant__ kernel
// parameter, so a launch needs no upload and no scratch; a call with more tensors than one table holds is split
// into one launch per kTable tensors.  A launch's work is the concatenation of its tensors' elements (`start`, the
// prefix sum of their numels): block b copies elements [b * kTile, (b + 1) * kTile) of it, finds the tensor its
// first element belongs to by a binary search every thread of the block does alike (uniform reads of the parameter
// bank), then walks on through the tensors its tile spans.  Any numel, offset and 4-byte alignment: the copies are
// scalar and coalesced, kUnroll loads in flight per thread.  The product is one IEEE fp32 multiply, as
// `grad * scale` computes it in torch, so pack is bitwise `torch.cat([g.reshape(-1) * s ...])`.
#include "common.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kTile = kThreads * kUnroll * 2;   // elements per block
constexpr int kTable = 1024;                    // tensors per launch: 28 KB of kernel parameters (CUDA 12.1+ allow 32 KB)

struct Table {
  int64_t start[kTable + 1];     // prefix sum of the numels: tensor i is work [start[i], start[i + 1])
  int64_t offset[kTable];        // bucket offset of tensor i
  float* ptr[kTable];            // the gradient (pack: read, NULL = zeros; unpack: written)
  float scale[kTable];           // pack only
  int n;
};

template <bool kPack>
__global__ void __launch_bounds__(kThreads) bucket_kernel(const __grid_constant__ Table t, float* __restrict__ bucket) {
  const long long total = t.start[t.n];
  long long w = (long long)blockIdx.x * kTile;
  const long long wend = w + kTile < total ? w + kTile : total;
  int e = find_segment(t.start, t.n, w);
  for (; w < wend; ++e) {
    const long long seg_end = t.start[e + 1] < wend ? t.start[e + 1] : wend;
    const long long j0 = w - t.start[e], len = seg_end - w;
    float* g = t.ptr[e] ? t.ptr[e] + j0 : nullptr;
    float* b = bucket + t.offset[e] + j0;
    const float s = t.scale[e];
    for (long long i = threadIdx.x; i < len; i += kThreads * kUnroll) {
      float v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const long long k = i + (long long)u * kThreads;
        if (kPack) v[u] = (g && k < len) ? __fmul_rn(__ldg(g + k), s) : 0.f;
        else v[u] = k < len ? __ldg(b + k) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const long long k = i + (long long)u * kThreads;
        if (k < len) {
          if (kPack) b[k] = v[u];
          else g[k] = v[u];
        }
      }
    }
    w = seg_end;
  }
}

template <bool kPack>
int run(const char* who, const int64_t* ptr_host, const int64_t* numel_host, const int64_t* offset_host,
        const float* scale_host, int n, float* bucket, long long bucket_numel, cudaStream_t st) {
  VIDAR_REQUIRE(n >= 0 && bucket_numel >= 0, "%s: bad sizes (n %d, bucket_numel %lld)", who, n, bucket_numel);
  VIDAR_REQUIRE(n == 0 || (ptr_host && numel_host && offset_host && (!kPack || scale_host)),
                "%s: null pointer argument (table)", who);
  long long work = 0;
  for (int i = 0; i < n; ++i) {
    const long long m = numel_host[i], o = offset_host[i];
    VIDAR_REQUIRE(m >= 0 && o >= 0 && o <= bucket_numel - m,
                  "%s: tensor %d (numel %lld, offset %lld) does not fit the bucket of %lld", who, i, m, o, bucket_numel);
    VIDAR_REQUIRE(ptr_host[i] % 4 == 0, "%s: tensor %d is not 4-byte aligned", who, i);
    VIDAR_REQUIRE(kPack || m == 0 || ptr_host[i], "%s: null pointer argument (tensor %d)", who, i);
    work += m;
  }
  VIDAR_REQUIRE(work == 0 || bucket, "%s: null pointer argument (bucket)", who);
  VIDAR_REQUIRE((uintptr_t)bucket % 4 == 0, "%s: bucket is not 4-byte aligned", who);
  Table t;
  for (int i0 = 0; i0 < n; i0 += kTable) {
    t.n = n - i0 < kTable ? n - i0 : kTable;
    t.start[0] = 0;
    for (int i = 0; i < t.n; ++i) {
      t.start[i + 1] = t.start[i] + numel_host[i0 + i];
      t.offset[i] = offset_host[i0 + i];
      t.ptr[i] = (float*)(uintptr_t)ptr_host[i0 + i];
      t.scale[i] = kPack ? scale_host[i0 + i] : 0.f;
    }
    const long long blocks = (t.start[t.n] + kTile - 1) / kTile;
    if (blocks == 0) continue;
    VIDAR_REQUIRE(blocks < (1LL << 31), "%s: %lld elements in one launch is too many", who, t.start[t.n]);
    bucket_kernel<kPack><<<(unsigned)blocks, kThreads, 0, st>>>(t, bucket);
    const int rc = check_launch(who);
    if (rc != VIDAR_OK) return rc;
  }
  return VIDAR_OK;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_grad_bucket_pack(const int64_t* ptr_host, const int64_t* numel_host, const int64_t* offset_host,
                                      const float* scale_host, int n, float* bucket, long long bucket_numel,
                                      void* stream) {
  return run<true>("grad_bucket_pack", ptr_host, numel_host, offset_host, scale_host, n, bucket, bucket_numel,
                   (cudaStream_t)stream);
}

extern "C" int vidar_grad_bucket_unpack(const float* bucket, long long bucket_numel, const int64_t* ptr_host,
                                        const int64_t* numel_host, const int64_t* offset_host, int n, void* stream) {
  return run<false>("grad_bucket_unpack", ptr_host, numel_host, offset_host, nullptr, n, const_cast<float*>(bucket),
                    bucket_numel, (cudaStream_t)stream);
}
