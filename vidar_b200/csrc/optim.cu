// The optimizer step of the pre-training configs (vidar_b200/optim.py): clip every gradient to a total 2-norm and
// step AdamW over every parameter, in two launches and with no host sync.
//
// norm:   partial[b] = sum of grad^2 over block b's tiles, in fp64 (kNormBlocks persistent blocks, fixed order)
// update: coef = clamp(max_norm / (norm + 1e-6), max=1) from every partial, summed alike in every block; then per
//         element, in the order of torch's single-tensor AdamW (torch.optim.adam._single_tensor_adam):
//           g  = grad * coef
//           p  = p * (1 - lr*wd)
//           m  = lerp(m, g, 1 - beta1)                      fma(w, g - m, m)
//           v  = v * beta2 + (1 - beta2) * (g * g)          fma(1 - beta2, g * g, v * beta2)
//           p  = p + (-lr/bc1) * (m / (sqrt(v) * (1/sqrt(bc2)) + eps))    fma(-lr/bc1, m / den, p)
//
// The tensor table is grad_bucket.cu's: (param, grad, per-tensor scalars) as a __grid_constant__ kernel parameter,
// a prefix sum of the numels, one uniform find_segment per tile and a walk through the tensors the tile spans.
// exp_avg and exp_avg_sq are two flat fp32 buffers in table order, so the table holds no pointers for them.  A tensor
// whose grad is NULL is skipped by both kernels: no decay, no state change, no share of the norm.  One launch of each
// kernel covers up to kTable tensors that share beta1, beta2 and eps; a longer list, or one whose hyperparameters
// change, is split into more launches of each.
//
// Determinism: every block of the norm kernel sums a fixed set of tiles in a fixed order (kNormBlocks does not
// depend on the device), the partials are summed in index order, and the update is elementwise, so the same
// gradients give bitwise the same parameters on every run and every rank.  Every rounding is written out (__fmul_rn,
// __fadd_rn, __fdiv_rn, __fmaf_rn) as torch's CUDA kernels round: one rounding per separate kernel, a fused
// multiply-add where its lerp, addcmul and addcdiv kernels compile to one, and the division by sqrt(bc2) as the
// multiplication by its fp32 reciprocal that torch makes of a division by a host scalar.
#include <math.h>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kTile = kThreads * kUnroll * 2;   // elements per tile
constexpr int kNormBlocks = 528;                // persistent blocks of the norm kernel: fixed, so its sums are too
constexpr int kTable = 896;                     // tensors per launch: 32 KB of kernel parameters (CUDA 12.1+)

struct Table {
  int64_t start[kTable + 1];   // prefix sum of the numels: tensor i is work and state [start[i], start[i + 1])
  float* param[kTable];
  const float* grad[kTable];   // NULL: the tensor has no gradient this step
  float decay[kTable];         // 1 - lr * wd
  float step[kTable];          // -lr / bc1
  float inv_bc2[kTable];       // 1 / sqrt(bc2), as torch's division by a host scalar computes it
  int n;
};

struct Hyper {                 // shared by every tensor of one launch
  float lerp_w;                // 1 - beta1
  float beta2, one_minus_beta2, eps;
};

static_assert(sizeof(Table) + sizeof(Hyper) + 64 <= 32764, "the table must fit the kernel parameter space");

__global__ void __launch_bounds__(kThreads) norm_kernel(const __grid_constant__ Table t, double* __restrict__ partial) {
  __shared__ double red[kThreads / 32];
  const long long total = t.start[t.n];
  double acc = 0.0;
  for (long long w0 = (long long)blockIdx.x * kTile; w0 < total; w0 += (long long)kNormBlocks * kTile) {
    long long w = w0;
    const long long wend = w0 + kTile < total ? w0 + kTile : total;
    int e = find_segment(t.start, t.n, w);
    for (; w < wend; ++e) {
      const long long seg_end = t.start[e + 1] < wend ? t.start[e + 1] : wend;
      if (t.grad[e]) {
        const float* g = t.grad[e] + (w - t.start[e]);
        const long long len = seg_end - w;
        for (long long i = threadIdx.x; i < len; i += kThreads * kUnroll) {
          float v[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const long long k = i + (long long)u * kThreads;
            v[u] = k < len ? __ldg(g + k) : 0.f;
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) acc = fma((double)v[u], (double)v[u], acc);
        }
      }
      w = seg_end;
    }
  }
  const double s = block_sum<kThreads>(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads)
update_kernel(const __grid_constant__ Table t, const Hyper h, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
              const double* __restrict__ partial, int nparts, float max_norm, float* __restrict__ grad_norm) {
  __shared__ double red[kThreads / 32];
  __shared__ float coef_s;
  float coef = 1.f;
  if (partial) {                       // clipping on: every block sums the partials alike
    double s = 0.0;
    for (int i = threadIdx.x; i < nparts; i += kThreads) s += partial[i];
    s = block_sum<kThreads>(s, red);
    if (threadIdx.x == 0) {
      const float norm = (float)sqrt(s);
      // torch: clip_coef = max_norm / (total_norm + 1e-6), i.e. reciprocal(total_norm + 1e-6) * max_norm, then
      // clamp(max=1).  `c > 1` is false for NaN, so a NaN norm gives a NaN coefficient as torch.clamp does.
      float c = __fmul_rn(__fdiv_rn(1.f, __fadd_rn(norm, 1e-6f)), max_norm);
      coef_s = c > 1.f ? 1.f : c;
      if (grad_norm && blockIdx.x == 0) *grad_norm = norm;
    }
    __syncthreads();
    coef = coef_s;
  }
  const long long total = t.start[t.n];
  const float one_minus_w = 1.f - h.lerp_w;
  const bool small_w = fabsf(h.lerp_w) < 0.5f;      // torch's lerp takes the form that keeps its weight below 0.5
  for (long long w0 = (long long)blockIdx.x * kTile; w0 < total; w0 += (long long)gridDim.x * kTile) {
    long long w = w0;
    const long long wend = w0 + kTile < total ? w0 + kTile : total;
    int e = find_segment(t.start, t.n, w);
    for (; w < wend; ++e) {
      const long long seg_end = t.start[e + 1] < wend ? t.start[e + 1] : wend;
      if (t.grad[e]) {
        const long long j0 = w - t.start[e], len = seg_end - w;
        const float* g = t.grad[e] + j0;
        float* p = t.param[e] + j0;
        float* m = exp_avg + w;
        float* v = exp_avg_sq + w;
        const float decay = t.decay[e], step = t.step[e], inv_bc2 = t.inv_bc2[e];
        for (long long i = threadIdx.x; i < len; i += kThreads * kUnroll) {
          float gr[kUnroll], pr[kUnroll], mr[kUnroll], vr[kUnroll];
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const long long k = i + (long long)u * kThreads;
            if (k < len) {
              gr[u] = __ldg(g + k);
              pr[u] = p[k];
              mr[u] = m[k];
              vr[u] = v[k];
            }
          }
#pragma unroll
          for (int u = 0; u < kUnroll; ++u) {
            const long long k = i + (long long)u * kThreads;
            if (k < len) {
              const float gg = __fmul_rn(gr[u], coef);
              const float pp = __fmul_rn(pr[u], decay);
              const float d = __fsub_rn(gg, mr[u]);
              const float mm = small_w ? __fmaf_rn(h.lerp_w, d, mr[u]) : __fmaf_rn(-d, one_minus_w, gg);
              const float vv = __fmaf_rn(h.one_minus_beta2, __fmul_rn(gg, gg), __fmul_rn(vr[u], h.beta2));
              const float den = __fadd_rn(__fmul_rn(sqrtf(vv), inv_bc2), h.eps);
              p[k] = __fmaf_rn(step, __fdiv_rn(mm, den), pp);
              m[k] = mm;
              v[k] = vv;
            }
          }
        }
      }
      w = seg_end;
    }
  }
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_adamw_step(const int64_t* param_host, const int64_t* grad_host, const int64_t* numel_host,
                                const float* scalar_host, int n, float* exp_avg, float* exp_avg_sq,
                                long long state_numel, int clip, float max_norm, float* grad_norm, void* stream) {
  const char* who = "adamw_step";
  cudaStream_t st = (cudaStream_t)stream;
  VIDAR_REQUIRE(n >= 0 && state_numel >= 0, "%s: bad sizes (n %d, state_numel %lld)", who, n, state_numel);
  VIDAR_REQUIRE(n == 0 || (param_host && grad_host && numel_host && scalar_host), "%s: null pointer argument (table)",
                who);
  VIDAR_REQUIRE(!clip || grad_norm, "%s: null pointer argument (grad_norm)", who);
  VIDAR_REQUIRE((uintptr_t)exp_avg % 4 == 0 && (uintptr_t)exp_avg_sq % 4 == 0 && (uintptr_t)grad_norm % 4 == 0,
                "%s: state buffers and grad_norm must be 4-byte aligned", who);
  // pass 1: validate, and cut the list into launches of at most kTable tensors with one (beta1, beta2, eps)
  long long work = 0;
  int launches = 0;
  for (int i = 0; i < n; ++i) {
    const long long m = numel_host[i];
    VIDAR_REQUIRE(m >= 0 && work <= state_numel - m, "%s: tensor %d (numel %lld at %lld) does not fit the state of %lld",
                  who, i, m, work, state_numel);
    VIDAR_REQUIRE(m == 0 || grad_host[i] == 0 || param_host[i], "%s: null pointer argument (parameter %d)", who, i);
    VIDAR_REQUIRE(param_host[i] % 4 == 0 && grad_host[i] % 4 == 0, "%s: tensor %d is not 4-byte aligned", who, i);
    work += m;
  }
  VIDAR_REQUIRE(work == 0 || (exp_avg && exp_avg_sq), "%s: null pointer argument (exp_avg / exp_avg_sq)", who);
  auto same_hyper = [&](int a, int b) {
    const float* x = scalar_host + 7LL * a;
    const float* y = scalar_host + 7LL * b;
    return x[3] == y[3] && x[4] == y[4] && x[5] == y[5] && x[6] == y[6];
  };
  auto chunk_end = [&](int i0) {
    int i1 = i0 + 1;
    while (i1 < n && i1 - i0 < kTable && same_hyper(i0, i1)) ++i1;
    return i1;
  };
  for (int i0 = 0; i0 < n; i0 = chunk_end(i0)) ++launches;
  if (launches == 0) {
    if (clip) {           // nothing has a gradient: the total norm is 0, as torch's clip_grad_norm_ of no tensors
      const cudaError_t e = cudaMemsetAsync(grad_norm, 0, sizeof(float), st);
      if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMemsetAsync: %s", who, cudaGetErrorString(e));
    }
    return VIDAR_OK;
  }

  double* partial = nullptr;
  const int nparts = launches * kNormBlocks;
  if (clip) {
    cudaMemPool_t pool;
    cudaError_t e = scratch_pool(&pool);
    if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch pool: %s", who, cudaGetErrorString(e));
    e = cudaMallocFromPoolAsync((void**)&partial, sizeof(double) * nparts, pool, st);
    if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  }
  const int update_blocks = 4 * num_sms();          // 48 registers: 4 blocks of 256 per SM, one resident wave
  int rc = VIDAR_OK;
  Table t;
  Hyper h;
  for (int pass = clip ? 0 : 1; pass < 2 && rc == VIDAR_OK; ++pass) {
    long long base = 0;
    int li = 0;
    for (int i0 = 0; i0 < n && rc == VIDAR_OK; ++li) {
      const int i1 = chunk_end(i0);
      t.n = i1 - i0;
      t.start[0] = 0;
      for (int i = 0; i < t.n; ++i) {
        const float* s = scalar_host + 7LL * (i0 + i);
        t.start[i + 1] = t.start[i] + numel_host[i0 + i];
        t.param[i] = (float*)(uintptr_t)param_host[i0 + i];
        t.grad[i] = (const float*)(uintptr_t)grad_host[i0 + i];
        t.decay[i] = s[0];
        t.step[i] = s[1];
        t.inv_bc2[i] = s[2];
      }
      const float* s = scalar_host + 7LL * i0;
      h.lerp_w = s[3];
      h.beta2 = s[4];
      h.one_minus_beta2 = s[5];
      h.eps = s[6];
      if (pass == 0) {
        norm_kernel<<<kNormBlocks, kThreads, 0, st>>>(t, partial + (long long)li * kNormBlocks);
        rc = check_launch("adamw_norm");
      } else {
        const long long tiles = (t.start[t.n] + kTile - 1) / kTile;
        const int blocks = (int)(tiles < update_blocks ? (tiles > 0 ? tiles : 1) : update_blocks);
        update_kernel<<<blocks, kThreads, 0, st>>>(t, h, exp_avg ? exp_avg + base : nullptr,
                                                   exp_avg_sq ? exp_avg_sq + base : nullptr, partial, nparts, max_norm,
                                                   li == 0 ? grad_norm : nullptr);
        rc = check_launch("adamw_update");
      }
      base += t.start[t.n];
      i0 = i1;
    }
  }
  if (partial) {
    const cudaError_t e = cudaFreeAsync(partial, st);
    if (e != cudaSuccess && rc == VIDAR_OK) rc = set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(e));
  }
  return rc;
}
