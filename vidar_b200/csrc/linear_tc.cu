// Y = X W^T + b on the Hopper tensor cores, fp32-accurate (3xTF32), for H100 (sm_90a).
//
// The one dense contraction on the hot path (SURVEY.md 8f-4): MSDeformableAttention3D.value_proj over the
// flattened camera features, 6 x 30825 rows x 256 -> 256 (spatial_cross_attention.py:333; the operand is
// built at modules/transformer.py:159-179).  The reference runs it as an fp32 cuBLAS GEMM (TF32 is off by
// default for matmuls), so a plain TF32 tensor-core GEMM (10-bit mantissas, ~1e-3) would break the 1e-4
// parity bar.  3xTF32: x = x_hi + x_lo, w = w_hi + w_lo with tf32 parts,
//     x w  ~=  x_hi w_hi + x_hi w_lo + x_lo w_hi          (dropped term ~2^-22 relative)
// three wgmma.mma_async (tf32, m64n128k8) per K step accumulating in fp32 registers.
// The tensor core truncates every sum it accumulates (round toward zero), so one accumulator chained through all
// 3 K / 8 wgmma carries an error that does not cancel and grows like K (measured at K = 4608: 27x fp32 cuBLAS's RMS
// error).  Each K block is therefore summed in two fresh accumulators of 6 wgmma each, the small x_hi w_lo and
// x_lo w_hi products first, and added into the running sum by ordinary round-to-nearest FADDs.
//
// Kernel (one persistent CTA per SM, 3 warpgroups, mbarrier pipeline of kStages stages):
//   warp 0        TMA producer: per K block (32 floats = one 128-byte swizzle row) the raw X tile [128 x 32] and
//                 the pre-split W tiles W_hi / W_lo [128 x 32] -> shared memory (cp.async.bulk.tensor.2d, SWIZZLE_128B)
//   warpgroups 1-2  consumers, one per 64-row half of the tile: split their half of the raw X tile in place
//                 (x_hi to its own tile, x_lo over the raw values: the split is element-wise, so the TMA's swizzle
//                 pattern is preserved), fence.proxy.async, then 4 K steps x 3 products of wgmma m64n128k8
//                 with shared-memory descriptors (K-major, SWIZZLE_128B) into the block accumulators, which are then
//                 added to the tile's running sum; after the last K block, + bias and
//                 8-byte stores straight from the accumulator registers.  The producer runs ahead into the
//                 next tile while the consumers store, so loads overlap the epilogue.
// Tiles: (row block of 128) x (column block of 128); K = in_features is looped in blocks of 32.
// Registers: a consumer thread holds 3 x 64 accumulators, more than the 168 per thread __launch_bounds__(384, 1)
// allows, so the producer warpgroup drops to 40 (setmaxnreg) and the two consumer warpgroups take 232.
// Requires in_features % 32 == 0, out_features % 128 == 0; rows are arbitrary (TMA clips, stores are guarded).
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kTM = 128, kTN = 128, kTK = 32;        // tile: 128 rows x 128 cols, K block of 32 floats (128 bytes)
constexpr int kStages = 3;
constexpr int kTileBytes = kTM * kTK * 4;            // 16 KB: one [128 x 32] fp32 operand tile
// per stage: X raw (then x_lo), X hi, W hi, W lo
constexpr int kStageBytes = 4 * kTileBytes;
constexpr int kGemmThreads = 3 * 128;
constexpr int kConsumerWarps = 8;
constexpr size_t kGemmSmem = (size_t)kStages * kStageBytes + 1024 /* alignment slack */ + 256 /* barriers */;

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(unsigned long long* b, unsigned n) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(n));
}
__device__ __forceinline__ void mb_expect_tx(unsigned long long* b, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(unsigned long long* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory");
}
__device__ __forceinline__ void mb_wait(unsigned long long* b, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "W_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra D_%=;\n\t"
      "bra W_%=;\n\t"
      "D_%=:\n\t}" ::"r"(s32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_2d(void* dst, const CUtensorMap* m, int c0, int c1, unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(s32(dst)), "l"(m), "r"(c0), "r"(c1), "r"(s32(bar)) : "memory");
}
// K-major operand tile [rows x 32 floats], 128-byte rows, SWIZZLE_128B, 8-row groups 1024 bytes apart
// (wgmma matrix descriptor: start >> 4 | LBO(1, unused when swizzled) << 16 | SBO(1024 >> 4) << 32 | 128B swizzle << 62).
// The tile is 1024-byte aligned, so the base-offset field stays 0; a K step of 8 tf32 moves the start by 32 bytes.
__device__ __forceinline__ unsigned long long gmma_desc(const void* tile, int k_byte_offset) {
  const unsigned addr = s32(tile) + (unsigned)k_byte_offset;
  unsigned long long d = (unsigned long long)((addr >> 4) & 0x3fffu);
  d |= 1ull << 16;
  d |= (unsigned long long)(1024 >> 4) << 32;
  d |= 1ull << 62;
  return d;
}
// d[64x128] = (accumulate ? d : 0) + a[64x8] b[8x128]^T, tf32 operands from shared memory, fp32 accumulators in
// registers (thread layout: d[4j + 2h + e] is row 16 warp + lane / 4 + 8h, column 8j + 2 (lane % 4) + e).
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], unsigned long long a, unsigned long long b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// The accumulators are written asynchronously: pin them so no register access moves across issue / wait.
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ float to_tf32(float x) {
  unsigned r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

struct GemmDims {
  int M, N, K;
  int tiles_m, tiles_n;
};

__global__ void __launch_bounds__(kGemmThreads, 1)
linear_tf32x3_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_whi,
                     const __grid_constant__ CUtensorMap map_wlo, const float* __restrict__ bias, float* __restrict__ y,
                     GemmDims g) {
  extern __shared__ unsigned char gemm_smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(gemm_smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(smem + kStages * kStageBytes);
  unsigned long long* full = bars;                     // [kStages]  TMA -> consumers
  unsigned long long* empty = bars + kStages;          // [kStages]  consumers (wgmma done) -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k_blocks = g.K / kTK;
  const int n_tiles = g.tiles_m * g.tiles_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mb_init(&full[s], 1);
      mb_init(&empty[s], kConsumerWarps);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===== TMA producer =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      unsigned it = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int tm = t / g.tiles_n, tn = t % g.tiles_n;
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
          const int s = it % kStages;
          const unsigned ph = (it / kStages) & 1u;
          mb_wait(&empty[s], ph ^ 1u);                           // first pass: passes immediately
          unsigned char* st = smem + s * kStageBytes;
          mb_expect_tx(&full[s], 3 * kTileBytes);
          tma_2d(st, &map_x, kb * kTK, tm * kTM, &full[s]);                          // X raw
          tma_2d(st + 2 * kTileBytes, &map_whi, kb * kTK, tn * kTN, &full[s]);       // W hi
          tma_2d(st + 3 * kTileBytes, &map_wlo, kb * kTK, tn * kTN, &full[s]);       // W lo
        }
      }
    }
  } else if (warp >= 4) {
    // ===== consumers: warpgroup c owns rows [64 c, 64 c + 64) of the tile =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int c = (warp >> 2) - 1;
    const int tid = threadIdx.x & 127;
    const int half = c * (kTileBytes / 2);                       // byte offset of this half in an operand tile
    unsigned it = 0;
    float p0[64], p1[64];                                        // the K block's sums of k steps 0-1 and 2-3
#pragma unroll
    for (int i = 0; i < 64; ++i) p0[i] = p1[i] = 0.f;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const int tm = t / g.tiles_n, tn = t % g.tiles_n;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int kb = 0; kb < k_blocks; ++kb, ++it) {
        const int s = it % kStages;
        const unsigned ph = (it / kStages) & 1u;
        mb_wait(&full[s], ph);
        unsigned char* st = smem + s * kStageBytes;
        // x -> (tf32(x), tf32(x - tf32(x))) at the same swizzled positions; x_lo overwrites x
        float4* lo = reinterpret_cast<float4*>(st + half);
        float4* hi = reinterpret_cast<float4*>(st + kTileBytes + half);
#pragma unroll
        for (int i = 0; i < kTileBytes / 2 / 16 / 128; ++i) {    // 512 float4 per half tile, 128 threads
          const float4 v = lo[i * 128 + tid];
          float4 h, l;
          h.x = to_tf32(v.x); h.y = to_tf32(v.y); h.z = to_tf32(v.z); h.w = to_tf32(v.w);
          l.x = to_tf32(v.x - h.x); l.y = to_tf32(v.y - h.y); l.z = to_tf32(v.z - h.z); l.w = to_tf32(v.w - h.w);
          hi[i * 128 + tid] = h;
          lo[i * 128 + tid] = l;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> tensor-core reads
        asm volatile("bar.sync %0, 128;" ::"r"(1 + c) : "memory");      // the whole half is split
        const unsigned char* xlo = st + half;
        const unsigned char* xhi = st + kTileBytes + half;
        const unsigned char* whi = st + 2 * kTileBytes;
        const unsigned char* wlo = st + 3 * kTileBytes;
        fence_acc(p0);
        fence_acc(p1);
        wgmma_fence();
        // tf32: K = 8 per instruction = 32 bytes.  The first product of each accumulator overwrites it.
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_tf32(p0, gmma_desc(xhi, 32 * k), gmma_desc(wlo, 32 * k), k);
          wgmma_tf32(p0, gmma_desc(xlo, 32 * k), gmma_desc(whi, 32 * k), 1);
          wgmma_tf32(p1, gmma_desc(xhi, 32 * k + 64), gmma_desc(wlo, 32 * k + 64), k);
          wgmma_tf32(p1, gmma_desc(xlo, 32 * k + 64), gmma_desc(whi, 32 * k + 64), 1);
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_tf32(p0, gmma_desc(xhi, 32 * k), gmma_desc(whi, 32 * k), 1);
          wgmma_tf32(p1, gmma_desc(xhi, 32 * k + 64), gmma_desc(whi, 32 * k + 64), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_acc(p0);
        fence_acc(p1);
        __syncwarp();
        if (lane == 0) mb_arrive(&empty[s]);                     // this warp's reads of the stage are done
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] += p0[i] + p1[i];
      }
      // ===== epilogue: registers + bias -> global =====
      const int row0 = tm * kTM + c * 64 + (warp & 3) * 16 + (lane >> 2);
      const int col0 = tn * kTN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < kTN / 8; ++j) {
        const int col = col0 + 8 * j;
        const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row < g.M)
            *reinterpret_cast<float2*>(y + (size_t)row * g.N + col) = make_float2(d[4 * j + 2 * h] + b0, d[4 * j + 2 * h + 1] + b1);
        }
      }
    }
  }
}

// W -> (tf32(W), tf32(W - tf32(W))), once per call (out_features x in_features, 0.5 MB at 256 x 256)
__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = w[i];
  const float h = to_tf32(v);
  hi[i] = h;
  lo[i] = to_tf32(v - h);
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn encode_fn() {
  static const EncodeFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      f = nullptr;
    }
    return (EncodeFn)f;
  }();
  return fn;
}

// [rows, K] fp32 row-major, box [128 rows x 32 floats], 128-byte swizzle (what the wgmma descriptors expect)
bool make_operand_map(CUtensorMap* m, const float* base, long long rows, int K) {
  EncodeFn enc = encode_fn();
  if (!enc) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)K * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)kTK, (cuuint32_t)kTM};
  const cuuint32_t estr[2] = {1u, 1u};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

// y [M, N] = x [M, K] w[N, K]^T + bias [N]   (nn.Linear), fp32 in / out, 3xTF32 on wgmma.
// w_split: caller-provided scratch of 2 * N * K floats (the library never allocates).
extern "C" int vidar_linear_tf32x3(const float* x, const float* w, const float* bias, float* y, float* w_split, int M,
                                   int N, int K, void* stream) {
  const char* who = "linear_tf32x3";
  VIDAR_REQUIRE(x && w && y && w_split, "%s: null pointer argument", who);
  VIDAR_REQUIRE(M > 0 && N > 0 && K > 0, "%s: bad sizes M=%d N=%d K=%d", who, M, N, K);
  VIDAR_REQUIRE(K % kTK == 0 && N % kTN == 0, "%s: in_features must be a multiple of %d and out_features of %d (got %d, %d)",
                who, kTK, kTN, K, N);
  VIDAR_REQUIRE(((uintptr_t)x & 15u) == 0 && ((uintptr_t)y & 15u) == 0 && ((uintptr_t)w_split & 15u) == 0,
                "%s: x, y and w_split must be 16-byte aligned", who);
  cudaStream_t st = (cudaStream_t)stream;
  float* w_hi = w_split;
  float* w_lo = w_split + (size_t)N * K;
  const long long nw = (long long)N * K;
  split_tf32_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(w, w_hi, w_lo, nw);
  int rc = check_launch("linear_tf32x3(split W)");
  if (rc) return rc;
  CUtensorMap mx, mhi, mlo;
  VIDAR_REQUIRE(make_operand_map(&mx, x, M, K) && make_operand_map(&mhi, w_hi, N, K) && make_operand_map(&mlo, w_lo, N, K),
                "%s: cuTensorMapEncodeTiled unavailable or failed", who);
  GemmDims g;
  g.M = M; g.N = N; g.K = K;
  g.tiles_m = (M + kTM - 1) / kTM;
  g.tiles_n = N / kTN;
  const int tiles = g.tiles_m * g.tiles_n;
  const int sms = num_sms();
  const int grid = tiles < sms ? tiles : sms;
  if (cudaFuncSetAttribute(linear_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmem) != cudaSuccess)
    return set_error(VIDAR_E_CUDA, "%s: cannot opt in to %zu bytes of shared memory", who, kGemmSmem);
  linear_tf32x3_kernel<<<grid, kGemmThreads, kGemmSmem, st>>>(mx, mhi, mlo, bias, y, g);
  return check_launch(who);
}
