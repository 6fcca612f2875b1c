// LatentRendering's projections, fused (sm_90a).
//
// Reference: projects/mmdet3d_plugin/bevformer/modules/ray_operations/latent_rendering.py
//   :94   occ  = unsup_raymarching_head(embed)      (a single Linear E->D when num_pred_fcs == 0,
//                                                    the shipped config vidar_1_8_nusc_3future.py:159)
//   :134  feat = lora_a(embed)                      Linear E->A, A = E / reduction
//   :153  out  = lora_b(pooled)                     Linear A->E
//   :155  out  = out.view(.., D, E/D) * prob.view(.., D, 1)
// In PyTorch these are 3 skinny cuBLAS GEMMs forward, 6 backward (three of them reductions over
// all 40 000 rows into a [16..32, 256] weight gradient), 5 bias/elementwise kernels and ~0.6 GB of
// traffic for 82 MB (fwd) / 123 MB (bwd) of algorithmic bytes (SURVEY.md 8d, B7).  Here: one kernel
// per direction on each side of the ray-marching core, fp32 FMA (the GEMMs have N or K = 16..32: HBM-bound, tensor cores are irrelevant),
// `embed` / `grad_out` are read once, `out` / `grad_embed` written once.
//
//   proj_in_fwd   [occ | feat] = embed W^T + b            W = [w_occ ; w_feat]  (N1 = D + A <= 32 rows)
//   proj_in_bwd   grad_embed = [g_occ | g_feat] W ;  grad_W += [g_occ | g_feat]^T embed ; grad_b += sum
//   proj_out_fwd  out = (pooled Wb^T + bb) * prob[d(e)]
//   proj_out_bwd  gl = grad_out * prob[d(e)] ; grad_pooled = gl Wb ; grad_prob = sum_e-in-d grad_out*lin
//                 grad_Wb += gl^T pooled ; grad_bb += sum gl
// Mapping: a lane owns the float4 column chunks e = 128 j + 4 lane (j < E/128), so every global
// and shared access along E is a conflict-free 16-byte vector; weights live in shared memory;
// weight gradients are accumulated in registers across a persistent block's row tiles and
// flushed once with vector reductions (caller zero-fills, like the other backward ops).
#include "common.cuh"

namespace vidar {
namespace {

constexpr int kProjThreads = 256;          // 8 warps
constexpr int kTileRows = 32;              // rows per block tile in the backward kernels
constexpr int kMaxEC = 2;                  // E <= 256 (register budget of the backward kernels)

struct ProjDims {
  long long rows;
  int E, D, A, N1;        // N1 = D + A
};

__device__ __forceinline__ float4 f4_fma(float a, float4 w, float4 acc) {
  acc.x = fmaf(a, w.x, acc.x); acc.y = fmaf(a, w.y, acc.y);
  acc.z = fmaf(a, w.z, acc.z); acc.w = fmaf(a, w.w, acc.w);
  return acc;
}
__device__ __forceinline__ float f4_dot(float4 a, float4 b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}


// stage Wb [E][A] transposed into shared memory as WbT[A][E]: 16-byte reads along the rank,
// lanes along E so the four scalar stores are conflict-free
__device__ __forceinline__ void stage_wbt(float* WbT, const float* __restrict__ wb, int E, int A) {
  for (int idx = threadIdx.x; idx < E * (A >> 2); idx += kProjThreads) {
    const int e = idx % E, i = (idx / E) << 2;
    const float4 v = ldg4(wb + (size_t)e * A + i);
    WbT[(i + 0) * E + e] = v.x; WbT[(i + 1) * E + e] = v.y;
    WbT[(i + 2) * E + e] = v.z; WbT[(i + 3) * E + e] = v.w;
  }
}

// Sum N per-lane partials over the warp so that lane L ends up with the total of index L
// (N == 32) -- "transposed" butterfly: 16+8+4+2+1 shuffles instead of 32 x 5.
template <int N>
__device__ __forceinline__ void warp_transpose_reduce(float (&v)[N], int lane) {
  constexpr int H = N / 2;
  const bool up = (lane & H) != 0;
#pragma unroll
  for (int k = 0; k < H; ++k) {
    const float send = up ? v[k] : v[k + H], keep = up ? v[k + H] : v[k];
    v[k] = keep + __shfl_xor_sync(0xffffffffu, send, H);
  }
  if constexpr (H > 1) {
    float (&lo)[H] = reinterpret_cast<float (&)[H]>(v);
    warp_transpose_reduce<H>(lo, lane);
  }
}

// ------------------------------------------------------------------------------ proj_in forward
// smem: Wt[E][32] (column n of lane n, zero-padded to 32) + per-warp X tile [8][E].
constexpr int kInRows = 8;

__global__ void __launch_bounds__(kProjThreads)
proj_in_fwd_kernel(ProjDims P, const float* __restrict__ X, const float* __restrict__ w_occ,
                   const float* __restrict__ b_occ, const float* __restrict__ w_feat,
                   const float* __restrict__ b_feat, float* __restrict__ occ, float* __restrict__ feat) {
  extern __shared__ __align__(16) float smem[];
  const int E = P.E, EC = E >> 7;
  float* Wt = smem;                                    // [E][32]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* Xs = smem + (size_t)E * 32 + (size_t)warp * kInRows * E;   // [8][E]
  // stage W^T: thread reads a float4 of row n along k, writes 4 conflict-free scalars
  for (int idx = threadIdx.x; idx < 32 * (E >> 2); idx += kProjThreads) {
    const int n = idx & 31, k = (idx >> 5) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < P.D) v = ldg4(w_occ + (size_t)n * E + k);
    else if (n < P.N1) v = ldg4(w_feat + (size_t)(n - P.D) * E + k);
    Wt[(k + 0) * 32 + n] = v.x; Wt[(k + 1) * 32 + n] = v.y;
    Wt[(k + 2) * 32 + n] = v.z; Wt[(k + 3) * 32 + n] = v.w;
  }
  __syncthreads();
  const float bias = lane < P.D ? __ldg(b_occ + lane) : (lane < P.N1 ? __ldg(b_feat + lane - P.D) : 0.f);
  const long long ntiles = (P.rows + kInRows - 1) / kInRows;
  for (long long t = (long long)blockIdx.x * 8 + warp; t < ntiles; t += (long long)gridDim.x * 8) {
    const long long r0 = t * kInRows;
#pragma unroll
    for (int r = 0; r < kInRows; ++r) {
      const long long row = r0 + r;
      for (int j = 0; j < EC; ++j) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < P.rows) v = ldg4(X + row * E + 128 * j + 4 * lane);
        *reinterpret_cast<float4*>(Xs + r * E + 128 * j + 4 * lane) = v;
      }
    }
    __syncwarp();
    float acc[kInRows];
#pragma unroll
    for (int r = 0; r < kInRows; ++r) acc[r] = bias;
    for (int k = 0; k < E; k += 4) {
      const float w0 = Wt[(k + 0) * 32 + lane], w1 = Wt[(k + 1) * 32 + lane];
      const float w2 = Wt[(k + 2) * 32 + lane], w3 = Wt[(k + 3) * 32 + lane];
#pragma unroll
      for (int r = 0; r < kInRows; ++r) {
        const float4 x = *reinterpret_cast<const float4*>(Xs + r * E + k);   // broadcast
        acc[r] = fmaf(x.x, w0, acc[r]); acc[r] = fmaf(x.y, w1, acc[r]);
        acc[r] = fmaf(x.z, w2, acc[r]); acc[r] = fmaf(x.w, w3, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < kInRows; ++r) {
      const long long row = r0 + r;
      if (row < P.rows) {
        if (lane < P.D) occ[row * P.D + lane] = acc[r];
        else if (lane < P.N1) feat[row * P.A + (lane - P.D)] = acc[r];
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------ proj_in backward
// smem: W[32][E] (rows >= N1 zero) + Xs[32][E] + Gs[32][32].
template <int EC>
__global__ void __launch_bounds__(kProjThreads, 2)
proj_in_bwd_kernel(ProjDims P, const float* __restrict__ X, const float* __restrict__ w_occ,
                   const float* __restrict__ w_feat, const float* __restrict__ g_occ,
                   const float* __restrict__ g_feat, float* __restrict__ gX, float* __restrict__ gw_occ,
                   float* __restrict__ gb_occ, float* __restrict__ gw_feat, float* __restrict__ gb_feat) {
  extern __shared__ __align__(16) float smem[];
  constexpr int E = EC * 128;
  float* W = smem;                          // [32][E]
  float* Xs = W + 32 * E;                   // [32][E]
  float* Gs = Xs + kTileRows * E;           // [32][32]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int idx = threadIdx.x; idx < 32 * (E >> 2); idx += kProjThreads) {
    const int n = idx / (E >> 2), k = (idx % (E >> 2)) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < P.D) v = ldg4(w_occ + (size_t)n * E + k);
    else if (n < P.N1) v = ldg4(w_feat + (size_t)(n - P.D) * E + k);
    *reinterpret_cast<float4*>(W + n * E + k) = v;
  }
  // weight-gradient accumulators of this warp: rows n = 4 warp .. 4 warp + 3, this lane's columns
  float4 accw[4][EC];
  float accb[4];
#pragma unroll
  for (int nn = 0; nn < 4; ++nn) {
    accb[nn] = 0.f;
#pragma unroll
    for (int j = 0; j < EC; ++j) accw[nn][j] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const long long ntiles = (P.rows + kTileRows - 1) / kTileRows;
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const long long r0 = t * kTileRows;
    __syncthreads();                        // previous tile fully consumed (and W staged)
    for (int idx = threadIdx.x; idx < kTileRows * (E >> 2); idx += kProjThreads) {
      const int r = idx / (E >> 2), k = (idx % (E >> 2)) << 2;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < P.rows) v = ldg4(X + (r0 + r) * E + k);
      *reinterpret_cast<float4*>(Xs + r * E + k) = v;
    }
    for (int idx = threadIdx.x; idx < kTileRows * 32; idx += kProjThreads) {
      const int r = idx >> 5, n = idx & 31;
      float v = 0.f;
      if (r0 + r < P.rows) {
        if (n < P.D) v = __ldg(g_occ + (r0 + r) * P.D + n);
        else if (n < P.N1) v = __ldg(g_feat + (r0 + r) * P.A + (n - P.D));
      }
      Gs[idx] = v;
    }
    __syncthreads();
    // phase A: grad_embed rows 4 warp .. 4 warp + 3
    {
      float4 acc[4][EC];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int j = 0; j < EC; ++j) acc[r][j] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int n = 0; n < P.N1; n += 4) {
        float4 g[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) g[r] = *reinterpret_cast<const float4*>(Gs + (4 * warp + r) * 32 + n);
#pragma unroll
        for (int nn = 0; nn < 4; ++nn) {
#pragma unroll
          for (int j = 0; j < EC; ++j) {
            const float4 w = *reinterpret_cast<const float4*>(W + (n + nn) * E + 128 * j + 4 * lane);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              const float gv = nn == 0 ? g[r].x : nn == 1 ? g[r].y : nn == 2 ? g[r].z : g[r].w;
              acc[r][j] = f4_fma(gv, w, acc[r][j]);
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const long long row = r0 + 4 * warp + r;
        if (row < P.rows)
#pragma unroll
          for (int j = 0; j < EC; ++j)
            *reinterpret_cast<float4*>(gX + row * E + 128 * j + 4 * lane) = acc[r][j];
      }
    }
    // phase B: grad_W rows 4 warp .. 4 warp + 3 over all rows of the tile
    for (int r = 0; r < kTileRows; ++r) {
      const float4 g = *reinterpret_cast<const float4*>(Gs + r * 32 + 4 * warp);
      accb[0] += g.x; accb[1] += g.y; accb[2] += g.z; accb[3] += g.w;
#pragma unroll
      for (int j = 0; j < EC; ++j) {
        const float4 x = *reinterpret_cast<const float4*>(Xs + r * E + 128 * j + 4 * lane);
        accw[0][j] = f4_fma(g.x, x, accw[0][j]);
        accw[1][j] = f4_fma(g.y, x, accw[1][j]);
        accw[2][j] = f4_fma(g.z, x, accw[2][j]);
        accw[3][j] = f4_fma(g.w, x, accw[3][j]);
      }
    }
  }
#pragma unroll
  for (int nn = 0; nn < 4; ++nn) {
    const int n = 4 * warp + nn;
    if (n >= P.N1) continue;
    float* gw = n < P.D ? gw_occ + (size_t)n * E : gw_feat + (size_t)(n - P.D) * E;
#pragma unroll
    for (int j = 0; j < EC; ++j) red_add_v4(gw + 128 * j + 4 * lane, accw[nn][j]);
    if (lane == 0) red_add_f32(n < P.D ? gb_occ + n : gb_feat + (n - P.D), accb[nn]);
  }
}

// ------------------------------------------------------------------------------ proj_out forward
// smem: WbT[A][E] + per-warp pooled [4][A] and prob [4][D].
constexpr int kOutRows = 4;

template <int EC>
__global__ void __launch_bounds__(kProjThreads)
proj_out_fwd_kernel(ProjDims P, const float* __restrict__ pooled, const float* __restrict__ prob,
                    const float* __restrict__ wb, const float* __restrict__ bb, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  constexpr int E = EC * 128;
  const int A = P.A, D = P.D;
  float* WbT = smem;                                   // [A][E]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* Ps = smem + (size_t)A * E + (size_t)warp * kOutRows * (A + D);   // [4][A]
  float* Qs = Ps + kOutRows * A;                                          // [4][D]
  stage_wbt(WbT, wb, E, A);
  __syncthreads();
  float4 bias[EC];
  int dsel[EC];
  const int per = E / D;                               // channels per height, multiple of 4
#pragma unroll
  for (int j = 0; j < EC; ++j) {
    bias[j] = ldg4(bb + 128 * j + 4 * lane);
    dsel[j] = (128 * j + 4 * lane) / per;
  }
  const long long ntiles = (P.rows + kOutRows - 1) / kOutRows;
  for (long long t = (long long)blockIdx.x * 8 + warp; t < ntiles; t += (long long)gridDim.x * 8) {
    const long long r0 = t * kOutRows;
    for (int idx = lane; idx < kOutRows * A; idx += 32) {
      const long long row = r0 + idx / A;
      Ps[idx] = row < P.rows ? __ldg(pooled + row * A + idx % A) : 0.f;
    }
    for (int idx = lane; idx < kOutRows * D; idx += 32) {
      const long long row = r0 + idx / D;
      Qs[idx] = row < P.rows ? __ldg(prob + row * D + idx % D) : 0.f;
    }
    __syncwarp();
    float4 acc[kOutRows][EC];
#pragma unroll
    for (int r = 0; r < kOutRows; ++r)
#pragma unroll
      for (int j = 0; j < EC; ++j) acc[r][j] = bias[j];
    for (int i = 0; i < A; ++i) {
      float p[kOutRows];
#pragma unroll
      for (int r = 0; r < kOutRows; ++r) p[r] = Ps[r * A + i];
#pragma unroll
      for (int j = 0; j < EC; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(WbT + i * E + 128 * j + 4 * lane);
#pragma unroll
        for (int r = 0; r < kOutRows; ++r) acc[r][j] = f4_fma(p[r], w, acc[r][j]);
      }
    }
#pragma unroll
    for (int r = 0; r < kOutRows; ++r) {
      const long long row = r0 + r;
      if (row < P.rows)
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          const float q = Qs[r * D + dsel[j]];
          float4 o = acc[r][j];
          o.x *= q; o.y *= q; o.z *= q; o.w *= q;
          *reinterpret_cast<float4*>(out + row * E + 128 * j + 4 * lane) = o;
        }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------ proj_out backward
// smem: WbT[A][E] + GLs[32][E] + Ps[32][A] + Qs[32][D].  A == 16 (two rank columns per warp).
template <int EC>
__global__ void __launch_bounds__(kProjThreads, 2)
proj_out_bwd_kernel(ProjDims P, const float* __restrict__ gout, const float* __restrict__ pooled,
                    const float* __restrict__ prob, const float* __restrict__ wb,
                    const float* __restrict__ bb, float* __restrict__ g_pooled, float* __restrict__ g_prob,
                    float* __restrict__ gwb, float* __restrict__ gbb) {
  extern __shared__ __align__(16) float smem[];
  constexpr int E = EC * 128;
  constexpr int A = 16;
  const int D = P.D;
  float* WbT = smem;                        // [A][E]
  float* GLs = WbT + A * E;                 // [32][E]
  float* Ps = GLs + kTileRows * E;          // [32][A]
  float* Qs = Ps + kTileRows * A;           // [32][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  stage_wbt(WbT, wb, E, A);
  const int per = E / D;                    // multiple of 4, divides 128
  const int glanes = per >> 2;              // lanes that share one height group
  const int dlane = (4 * lane) / per, dchunk = 128 / per;   // height of chunk j: dlane + j * dchunk
  float4 accw[2][EC], accb[EC];             // grad_Wb columns i = 2 warp, 2 warp + 1 ; grad_bb (own rows)
#pragma unroll
  for (int j = 0; j < EC; ++j) {
    accw[0][j] = accw[1][j] = accb[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const long long ntiles = (P.rows + kTileRows - 1) / kTileRows;
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const long long r0 = t * kTileRows;
    __syncthreads();
    for (int idx = threadIdx.x; idx < kTileRows * A; idx += kProjThreads) {
      const long long row = r0 + idx / A;
      Ps[idx] = row < P.rows ? __ldg(pooled + row * A + idx % A) : 0.f;
    }
    for (int idx = threadIdx.x; idx < kTileRows * D; idx += kProjThreads) {
      const long long row = r0 + idx / D;
      Qs[idx] = row < P.rows ? __ldg(prob + row * D + idx % D) : 0.f;
    }
    __syncthreads();
    // phase A: rows 4 warp .. 4 warp + 3, two at a time (register budget)
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
      const int rl = 4 * warp + 2 * half;               // first local row of the pair
      float4 go[2][EC], lin[2][EC];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = r0 + rl + r;
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          go[r][j] = row < P.rows ? ldg4(gout + row * E + 128 * j + 4 * lane) : make_float4(0.f, 0.f, 0.f, 0.f);
          lin[r][j] = ldg4(bb + 128 * j + 4 * lane);
        }
      }
#pragma unroll
      for (int i = 0; i < A; ++i) {
        const float p0 = Ps[(rl + 0) * A + i], p1 = Ps[(rl + 1) * A + i];
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          const float4 w = *reinterpret_cast<const float4*>(WbT + i * E + 128 * j + 4 * lane);
          lin[0][j] = f4_fma(p0, w, lin[0][j]);
          lin[1][j] = f4_fma(p1, w, lin[1][j]);
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = r0 + rl + r;
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          // grad_prob[row][d] = sum over the group's channels of grad_out * lin
          float s = f4_dot(go[r][j], lin[r][j]);
          for (int off = 1; off < glanes; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
          if ((lane & (glanes - 1)) == 0 && row < P.rows) g_prob[row * D + dlane + j * dchunk] = s;
          const float q = Qs[(rl + r) * D + dlane + j * dchunk];
          float4 gl = go[r][j];
          gl.x *= q; gl.y *= q; gl.z *= q; gl.w *= q;
          go[r][j] = gl;
          *reinterpret_cast<float4*>(GLs + (rl + r) * E + 128 * j + 4 * lane) = gl;
          accb[j].x += gl.x; accb[j].y += gl.y; accb[j].z += gl.z; accb[j].w += gl.w;
        }
      }
      float part[2 * A];                    // this lane's share of grad_pooled[r][i], flat r*A + i
#pragma unroll
      for (int i = 0; i < A; ++i) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < EC; ++j) {
          const float4 w = *reinterpret_cast<const float4*>(WbT + i * E + 128 * j + 4 * lane);
          s0 += f4_dot(go[0][j], w);
          s1 += f4_dot(go[1][j], w);
        }
        part[i] = s0;
        part[A + i] = s1;
      }
      warp_transpose_reduce<2 * A>(part, lane);          // lane L now holds flat index L
      {
        const long long row = r0 + rl + (lane >> 4);
        if (row < P.rows) g_pooled[row * A + (lane & 15)] = part[0];
      }
    }
    __syncthreads();                         // GLs complete
    // phase B: grad_Wb[:, i] for i = 2 warp, 2 warp + 1 over the tile's rows
    for (int r = 0; r < kTileRows; ++r) {
      const float2 p = *reinterpret_cast<const float2*>(Ps + r * A + 2 * warp);
#pragma unroll
      for (int j = 0; j < EC; ++j) {
        const float4 gl = *reinterpret_cast<const float4*>(GLs + r * E + 128 * j + 4 * lane);
        accw[0][j] = f4_fma(p.x, gl, accw[0][j]);
        accw[1][j] = f4_fma(p.y, gl, accw[1][j]);
      }
    }
  }
  // flush: grad_Wb is [E][A]
#pragma unroll
  for (int j = 0; j < EC; ++j) {
    const int e = 128 * j + 4 * lane;
#pragma unroll
    for (int ii = 0; ii < 2; ++ii) {
      const int i = 2 * warp + ii;
      red_add_f32(gwb + (size_t)(e + 0) * A + i, accw[ii][j].x);
      red_add_f32(gwb + (size_t)(e + 1) * A + i, accw[ii][j].y);
      red_add_f32(gwb + (size_t)(e + 2) * A + i, accw[ii][j].z);
      red_add_f32(gwb + (size_t)(e + 3) * A + i, accw[ii][j].w);
    }
    red_add_v4(gbb + e, accb[j]);
  }
}

int check_proj(ProjDims& P, long long rows, int E, int D, int A, const char* what) {
  VIDAR_REQUIRE(rows >= 0 && E > 0 && D > 0 && A > 0, "%s: sizes must be positive", what);
  VIDAR_REQUIRE(E % 128 == 0 && E <= 128 * kMaxEC, "%s: embed_dims must be 128 or 256 (got %d)", what, E);
  VIDAR_REQUIRE(D + A <= 32 && (D + A) % 4 == 0, "%s: pred_height + rank must be a multiple of 4 and <= 32 (got %d + %d)", what, D, A);
  VIDAR_REQUIRE(E % D == 0 && (E / D) % 4 == 0 && 128 % (E / D) == 0,
                "%s: embed_dims / pred_height must be a multiple of 4 that divides 128 (got %d / %d)", what, E, D);
  P.rows = rows; P.E = E; P.D = D; P.A = A; P.N1 = D + A;
  return VIDAR_OK;
}

template <typename K>
int set_smem(K kernel, size_t bytes, const char* what) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: shared memory opt-in (%zu B): %s", what, bytes, cudaGetErrorString(e));
  return VIDAR_OK;
}

int grid_for(long long tiles, int per_sm) {
  const long long cap = (long long)num_sms() * per_sm;
  return (int)(tiles < cap ? (tiles > 0 ? tiles : 1) : cap);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

#define PROJ_EC_DISPATCH(KERNEL, ...)                                                       \
  do {                                                                                      \
    if (E == 128) { rc = set_smem(KERNEL<1>, smem, what); if (!rc) KERNEL<1><<<grid, kProjThreads, smem, st>>>(__VA_ARGS__); } \
    else { rc = set_smem(KERNEL<2>, smem, what); if (!rc) KERNEL<2><<<grid, kProjThreads, smem, st>>>(__VA_ARGS__); }          \
  } while (0)

extern "C" int vidar_latent_proj_in_forward(const float* embed, const float* w_occ, const float* b_occ,
                                            const float* w_feat, const float* b_feat, float* occ, float* feat,
                                            long long rows, int E, int D, int A, void* stream) {
  const char* what = "LatentRendering.proj_in_forward";
  ProjDims P;
  int rc = check_proj(P, rows, E, D, A, what);
  if (rc) return rc;
  if (rows == 0) return VIDAR_OK;
  VIDAR_REQUIRE(embed && w_occ && b_occ && w_feat && b_feat && occ && feat, "%s: null pointer argument", what);
  const size_t smem = sizeof(float) * ((size_t)E * 32 + (size_t)8 * kInRows * E);
  rc = set_smem(proj_in_fwd_kernel, smem, what);
  if (rc) return rc;
  const int grid = grid_for((rows + 8 * kInRows - 1) / (8 * kInRows), 2);
  proj_in_fwd_kernel<<<grid, kProjThreads, smem, (cudaStream_t)stream>>>(P, embed, w_occ, b_occ, w_feat, b_feat, occ, feat);
  return check_launch(what);
}

extern "C" int vidar_latent_proj_in_backward(const float* embed, const float* w_occ, const float* w_feat,
                                             const float* grad_occ, const float* grad_feat, float* grad_embed,
                                             float* grad_w_occ, float* grad_b_occ, float* grad_w_feat,
                                             float* grad_b_feat, long long rows, int E, int D, int A,
                                             void* stream) {
  const char* what = "LatentRendering.proj_in_backward";
  ProjDims P;
  int rc = check_proj(P, rows, E, D, A, what);
  if (rc) return rc;
  if (rows == 0) return VIDAR_OK;
  VIDAR_REQUIRE(embed && w_occ && w_feat && grad_occ && grad_feat && grad_embed && grad_w_occ && grad_b_occ &&
                grad_w_feat && grad_b_feat, "%s: null pointer argument", what);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = sizeof(float) * ((size_t)32 * E + (size_t)kTileRows * E + kTileRows * 32);
  const int grid = grid_for((rows + kTileRows - 1) / kTileRows, 2);
  PROJ_EC_DISPATCH(proj_in_bwd_kernel, P, embed, w_occ, w_feat, grad_occ, grad_feat, grad_embed, grad_w_occ,
                   grad_b_occ, grad_w_feat, grad_b_feat);
  if (rc) return rc;
  return check_launch(what);
}

extern "C" int vidar_latent_proj_out_forward(const float* pooled, const float* prob, const float* w, const float* b,
                                             float* out, long long rows, int E, int D, int A, void* stream) {
  const char* what = "LatentRendering.proj_out_forward";
  ProjDims P;
  int rc = check_proj(P, rows, E, D, A, what);
  if (rc) return rc;
  if (rows == 0) return VIDAR_OK;
  VIDAR_REQUIRE(pooled && prob && w && b && out, "%s: null pointer argument", what);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = sizeof(float) * ((size_t)A * E + (size_t)8 * kOutRows * (A + D));
  const int grid = grid_for((rows + 8 * kOutRows - 1) / (8 * kOutRows), 4);
  PROJ_EC_DISPATCH(proj_out_fwd_kernel, P, pooled, prob, w, b, out);
  if (rc) return rc;
  return check_launch(what);
}

extern "C" int vidar_latent_proj_out_backward(const float* grad_out, const float* pooled, const float* prob,
                                              const float* w, const float* b, float* grad_pooled, float* grad_prob,
                                              float* grad_w, float* grad_b, long long rows, int E, int D, int A,
                                              void* stream) {
  const char* what = "LatentRendering.proj_out_backward";
  ProjDims P;
  int rc = check_proj(P, rows, E, D, A, what);
  if (rc) return rc;
  VIDAR_REQUIRE(A == 16, "%s: rank (embed_dims / reduction) must be 16 (got %d)", what, A);
  if (rows == 0) return VIDAR_OK;
  VIDAR_REQUIRE(grad_out && pooled && prob && w && b && grad_pooled && grad_prob && grad_w && grad_b,
                "%s: null pointer argument", what);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = sizeof(float) * ((size_t)16 * E + (size_t)kTileRows * E + kTileRows * 16 + (size_t)kTileRows * D);
  const int grid = grid_for((rows + kTileRows - 1) / kTileRows, 2);
  PROJ_EC_DISPATCH(proj_out_bwd_kernel, P, grad_out, pooled, prob, w, b, grad_pooled, grad_prob, grad_w, grad_b);
  if (rc) return rc;
  return check_launch(what);
}
