// LatentRendering core (the paper's "latent rendering" operator) for H100 (sm_90a).
//
// Reference: projects/mmdet3d_plugin/bevformer/modules/ray_operations/latent_rendering.py:98-161
// -- pure PyTorch: 3 grid_sample launches + cumprod + masks that materialise
// [bs,16,40000,257] x3 and [bs,16,40000,256] x3 (about 4 GB of traffic and saved-for-backward
// state for 82 MB of algorithmic bytes, SURVEY.md B7).  Semantics (SURVEY.md A.3), per BEV
// cell u with centre c_u and unit direction r_u from the BEV centre:
//   waypoints  s_{u,k} = 1/2 + r_u (k+1/2) tstep, k < G ;  s_{u,G} = c_u ;  grid g = 2s-1
//   phase 1    a_k = act(bilerp(occ, g_k)) ; m_k = [|g_k| < |g_G|]
//              prob_u = a_G * prod_{k<G} (1 - a_k m_k)                        (per height d)
//   phase 2    b_k = [|g_k| < min(1/|r_x|, 1/|r_y|)]
//              pooled_{u,c} = sum_k bilerp(feat_c, g_k) * pg_k / (sum_k pg_k + eps),
//              pg_k = bilerp(prob_d, g_k) b_k,  c = d*g + j (channel group d <-> height d)
// Phase 2 samples the prob MAP that phase 1 produces for all cells, so the op is two kernels
// each way.  Everything else of the module (three Linear layers, the final product) stays
// in PyTorch.
//
// Layout: inputs are channel-LAST ([bs,Hb,Wb,D], [bs,Hb,Wb,D*g]) -- what the Linear layers
// emit -- so the D heights of one pixel are 64 contiguous bytes; the reference permutes to
// channel-first for grid_sample.
// Mapping: one warp per BEV cell; a lane is (waypoint slot, float4 of heights): LPW = D/4
// lanes cover one waypoint's heights with one 16-byte load per bilinear corner and
// 32/LPW waypoints are in flight per step; |g_k| grows linearly in k, so the march stops at
// the cell (phase 1) or at the BEV border (phase 2) instead of visiting all G waypoints
// behind a mask.  Products / sums over waypoints are finished with warp shuffles; only
// prob (D floats) and pooled (D*g floats) are written per cell.  Backward kernels recompute
// the forward quantities and scatter with vector reductions.
#include <math.h>

#include "common.cuh"

namespace vidar {
namespace {

struct LrDims {
  int bs, D, G, Hb, Wb, grid_num, act;   // G = feature channels per height
  float tstep, eps;
  long long cell0, ncells;               // this call handles cells [cell0, cell0 + ncells) of bs*Hb*Wb
};

struct Bil {
  int o[4];      // pixel index y*Wb+x, or -1 if outside
  float w[4];    // nw, ne, sw, se
};

__device__ __forceinline__ Bil bilinear_setup(float gx, float gy, int Hb, int Wb) {
  Bil b;
  // grid_sample: ((g + 1) * size - 1) / 2 ; the division by 2 is exact, so x 0.5 gives the same bits
  const float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)Wb), 1.f), 0.5f);
  const float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)Hb), 1.f), 0.5f);
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = (int)fx, y0 = (int)fy;
  const float wx1 = ix - fx, wy1 = iy - fy;
  const float wx0 = (fx + 1.f) - ix, wy0 = (fy + 1.f) - iy;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int xx = x0 + (j & 1), yy = y0 + (j >> 1);
    const bool in = xx >= 0 && xx < Wb && yy >= 0 && yy < Hb;
    b.o[j] = in ? yy * Wb + xx : -1;
    b.w[j] = ((j & 1) ? wx1 : wx0) * ((j & 2) ? wy1 : wy0);
  }
  return b;
}

struct Cell {
  float cgx, cgy, rnx, rny, lenG, boundary;
};

__device__ __forceinline__ Cell cell_geometry(const LrDims& L, int iy, int ix) {
  Cell c;
  const float cx = __fdiv_rn((float)ix + 0.5f, (float)L.Wb);
  const float cy = __fdiv_rn((float)iy + 0.5f, (float)L.Hb);
  const float rx = __fsub_rn(cx, 0.5f), ry = __fsub_rn(cy, 0.5f);
  const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry)));
  c.rnx = __fdiv_rn(rx, nrm);
  c.rny = __fdiv_rn(ry, nrm);
  if (c.rnx != c.rnx) c.rnx = 0.f;     // nan_to_num at the exact centre (:100-101)
  if (c.rny != c.rny) c.rny = 0.f;
  c.cgx = __fsub_rn(__fmul_rn(cx, 2.f), 1.f);
  c.cgy = __fsub_rn(__fmul_rn(cy, 2.f), 1.f);
  c.lenG = __fsqrt_rn(__fadd_rn(__fmul_rn(c.cgx, c.cgx), __fmul_rn(c.cgy, c.cgy)));
  c.boundary = fminf(__fdiv_rn(1.f, fabsf(c.rnx)), __fdiv_rn(1.f, fabsf(c.rny)));
  return c;
}

// grid position of waypoint k < grid_num; returns the reference's mask `|g_k| < limit`.
// |g_k| = 2*tstep*(k+0.5) up to ~1e-6 of rounding, so the IEEE square root is only evaluated for
// the waypoints within three steps of the limit (k >= kchk, see march_check): below that the
// comparison is true with a margin of 2.5 steps (0.025 at the shipped step), four orders of
// magnitude more than the rounding of |g_k|.
__device__ __forceinline__ bool waypoint(const LrDims& L, const Cell& c, int k, int kchk, float limit,
                                         float& gx, float& gy) {
  const float t = __fmul_rn((float)k + 0.5f, L.tstep);
  const float sx = __fadd_rn(0.5f, __fmul_rn(c.rnx, t));
  const float sy = __fadd_rn(0.5f, __fmul_rn(c.rny, t));
  gx = __fsub_rn(__fmul_rn(sx, 2.f), 1.f);
  gy = __fsub_rn(__fmul_rn(sy, 2.f), 1.f);
  if (k < kchk) return true;
  return __fsqrt_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))) < limit;
}

// |g_k| ~ 2*tstep*(k+0.5): first k that can fail `len < limit`, with slack for rounding
__device__ __forceinline__ int march_end(const LrDims& L, float limit) {
  if (!(limit < 1e30f)) return L.grid_num;
  const int k = (int)(limit / (2.f * L.tstep)) + 2;
  return k < L.grid_num ? k : L.grid_num;
}
// first k whose mask must be evaluated exactly (everything below is inside with margin)
__device__ __forceinline__ int march_check(const LrDims& L, float limit) {
  if (!(limit < 1e30f)) return 0;                 // NaN / inf limit: always evaluate
  const int k = (int)(limit / (2.f * L.tstep)) - 2;
  return k > 0 ? k : 0;
}

template <int VEC> struct V;
template <> struct V<4> {
  using T = float4;
  static __device__ __forceinline__ void ld(const float* p, float* v) { const float4 t = ldg4(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
  static __device__ __forceinline__ void st(float* p, const float* v) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
  static __device__ __forceinline__ void red(float* p, const float* v) { red_add_v4(p, make_float4(v[0], v[1], v[2], v[3])); }
};
template <> struct V<1> {
  static __device__ __forceinline__ void ld(const float* p, float* v) { v[0] = __ldg(p); }
  static __device__ __forceinline__ void st(float* p, const float* v) { p[0] = v[0]; }
  static __device__ __forceinline__ void red(float* p, const float* v) { red_add_f32(p, v[0]); }
};

// bilinear sample of VEC consecutive channels starting at channel ch of a channel-last map
template <int VEC>
__device__ __forceinline__ void sample(const float* __restrict__ map, int C, int ch, const Bil& b, float* out) {
#pragma unroll
  for (int v = 0; v < VEC; ++v) out[v] = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (b.o[j] >= 0) {
      float t[VEC];
      V<VEC>::ld(map + (size_t)b.o[j] * C + ch, t);
#pragma unroll
      for (int v = 0; v < VEC; ++v) out[v] += t[v] * b.w[j];   // nw, ne, sw, se like grid_sample
    }
  }
}

template <int VEC>
__device__ __forceinline__ void scatter(float* __restrict__ map, int C, int ch, const Bil& b, const float* g) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (b.o[j] >= 0) {
      float t[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) t[v] = g[v] * b.w[j];
      V<VEC>::red(map + (size_t)b.o[j] * C + ch, t);
    }
  }
}

__device__ __forceinline__ float activate(int act, float x) {
  // sigmoid: full-precision expf, reciprocal through the SFU (<= 2 ulp; the value feeds a smooth
  // product, no branch depends on it) instead of the ~10-instruction IEEE division
  if (act == 1) return __fdividef(1.f, 1.f + expf(-x));
  return 1.f - expf(-fmaxf(x, 0.f));                    // 1 - exp(-relu(x))
}
__device__ __forceinline__ float activate_grad(int act, float x, float a) {
  if (act == 1) return a * (1.f - a);
  return x > 0.f ? 1.f - a : 0.f;
}

constexpr int kCellsPerBlock = 8;

#define LR_PROLOGUE                                                                  \
  const int LPW = L.D / VEC;                 /* lanes per waypoint */               \
  const int WPI = 32 / LPW;                  /* waypoints per iteration */          \
  const int lane = threadIdx.x & 31;                                                 \
  const int slot = lane / LPW, ch = (lane % LPW) * VEC;                             \
  const long long cidx = (long long)blockIdx.x * kCellsPerBlock + (threadIdx.x >> 5); \
  const int HW = L.Hb * L.Wb;                                                        \
  if (cidx >= L.ncells) return;                                                      \
  const long long cell = L.cell0 + cidx;                                             \
  const int b = (int)(cell / HW), u = (int)(cell % HW);                             \
  const Cell c = cell_geometry(L, u / L.Wb, u % L.Wb);

// ---------------------------------------------------------------- phase 1 forward
template <int VEC>
__global__ void __launch_bounds__(kCellsPerBlock * 32)
latent_prob_fwd_kernel(LrDims L, const float* __restrict__ occ, float* __restrict__ prob,
                       float* __restrict__ aux_t, float* __restrict__ aux_nz) {
  LR_PROLOGUE
  const float* omap = occ + (size_t)b * HW * L.D;
  // product of the non-zero factors and the number of exactly-zero ones (saturated activation):
  // the backward needs "product of the other factors" without dividing by zero
  float tnz[VEC], nz[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) { tnz[v] = 1.f; nz[v] = 0.f; }
  const int kend = march_end(L, c.lenG), kchk = march_check(L, c.lenG);
  for (int k0 = 0; k0 < kend; k0 += WPI) {
    const int k = k0 + slot;
    if (k < kend) {
      float gx, gy;
      if (waypoint(L, c, k, kchk, c.lenG, gx, gy)) {
        float x[VEC];
        sample<VEC>(omap, L.D, ch, bilinear_setup(gx, gy, L.Hb, L.Wb), x);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          const float f = 1.f - activate(L.act, x[v]);
          if (f == 0.f) nz[v] += 1.f; else tnz[v] *= f;
        }
      }
    }
  }
#pragma unroll
  for (int v = 0; v < VEC; ++v)
    for (int off = LPW; off < 32; off <<= 1) {
      tnz[v] *= __shfl_xor_sync(0xffffffffu, tnz[v], off);
      nz[v] += __shfl_xor_sync(0xffffffffu, nz[v], off);
    }
  if (slot == 0) {
    float x[VEC], out[VEC];
    sample<VEC>(omap, L.D, ch, bilinear_setup(c.cgx, c.cgy, L.Hb, L.Wb), x);
#pragma unroll
    for (int v = 0; v < VEC; ++v) out[v] = (nz[v] > 0.f ? 0.f : tnz[v]) * activate(L.act, x[v]);
    const size_t o = ((size_t)b * HW + u) * L.D + ch;
    V<VEC>::st(prob + o, out);
    if (aux_t) {          // saved for the backward: no second march there
      V<VEC>::st(aux_t + o, tnz);
      V<VEC>::st(aux_nz + o, nz);
    }
  }
}

// ---------------------------------------------------------------- phase 1 backward
// grad_prob -> grad_occ.  d prob / d a_k = -a_G * prod_{j != k}(1 - a_j m_j); the product of
// the others is T / f_k unless a factor is exactly 0 (saturated activation), which is
// tracked by counting zero factors so nothing is divided by zero.
template <int VEC>
__global__ void __launch_bounds__(kCellsPerBlock * 32)
latent_prob_bwd_kernel(LrDims L, const float* __restrict__ occ, const float* __restrict__ grad_prob,
                       float* __restrict__ grad_occ, const float* __restrict__ aux_t,
                       const float* __restrict__ aux_nz) {
  LR_PROLOGUE
  const float* omap = occ + (size_t)b * HW * L.D;
  float* gmap = grad_occ + (size_t)b * HW * L.D;
  float tnz[VEC], nz[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) { tnz[v] = 1.f; nz[v] = 0.f; }
  const int kend = march_end(L, c.lenG), kchk = march_check(L, c.lenG);
  if (aux_t) {            // forward saved the products: skip the recomputation march
    V<VEC>::ld(aux_t + ((size_t)b * HW + u) * L.D + ch, tnz);
    V<VEC>::ld(aux_nz + ((size_t)b * HW + u) * L.D + ch, nz);
  }
  for (int k0 = 0; !aux_t && k0 < kend; k0 += WPI) {
    const int k = k0 + slot;
    if (k < kend) {
      float gx, gy;
      if (waypoint(L, c, k, kchk, c.lenG, gx, gy)) {
        float x[VEC];
        sample<VEC>(omap, L.D, ch, bilinear_setup(gx, gy, L.Hb, L.Wb), x);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          const float f = 1.f - activate(L.act, x[v]);
          if (f == 0.f) nz[v] += 1.f; else tnz[v] *= f;
        }
      }
    }
  }
  if (!aux_t) {
#pragma unroll
    for (int v = 0; v < VEC; ++v)
      for (int off = LPW; off < 32; off <<= 1) {
        tnz[v] *= __shfl_xor_sync(0xffffffffu, tnz[v], off);
        nz[v] += __shfl_xor_sync(0xffffffffu, nz[v], off);
      }
  }
  float g[VEC], xG[VEC], aG[VEC];
  V<VEC>::ld(grad_prob + ((size_t)b * HW + u) * L.D + ch, g);
  const Bil bG = bilinear_setup(c.cgx, c.cgy, L.Hb, L.Wb);
  sample<VEC>(omap, L.D, ch, bG, xG);
#pragma unroll
  for (int v = 0; v < VEC; ++v) aG[v] = activate(L.act, xG[v]);
  if (slot == 0) {   // the cell's own sample: d prob / d a_G = T
    float gx_[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v)
      gx_[v] = g[v] * (nz[v] > 0.f ? 0.f : tnz[v]) * activate_grad(L.act, xG[v], aG[v]);
    scatter<VEC>(gmap, L.D, ch, bG, gx_);
  }
  for (int k0 = 0; k0 < kend; k0 += WPI) {
    const int k = k0 + slot;
    if (k < kend) {
      float gx, gy;
      if (waypoint(L, c, k, kchk, c.lenG, gx, gy)) {
        const Bil bb = bilinear_setup(gx, gy, L.Hb, L.Wb);
        float x[VEC], gx_[VEC];
        sample<VEC>(omap, L.D, ch, bb, x);
        bool any = false;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          const float a = activate(L.act, x[v]);
          const float f = 1.f - a;
          float others;
          if (nz[v] == 0.f) others = __fdividef(tnz[v], f);
          else if (nz[v] == 1.f) others = (f == 0.f) ? tnz[v] : 0.f;
          else others = 0.f;
          gx_[v] = -g[v] * aG[v] * others * activate_grad(L.act, x[v], a);
          any |= gx_[v] != 0.f;
        }
        if (any) scatter<VEC>(gmap, L.D, ch, bb, gx_);
      }
    }
  }
}

// ---------------------------------------------------------------- phase 2 forward
template <int VEC, int G>
__device__ __forceinline__ void pool_accumulate(const LrDims& L, const Cell& c, const float* pmap,
                                                const float* fmap, int ch, int slot, int WPI,
                                                float* S, float* N) {
#pragma unroll
  for (int v = 0; v < VEC; ++v) S[v] = 0.f;
#pragma unroll
  for (int v = 0; v < VEC * G; ++v) N[v] = 0.f;
  const int kend = march_end(L, c.boundary), kchk = march_check(L, c.boundary);
  for (int k0 = 0; k0 < kend; k0 += WPI) {
    const int k = k0 + slot;
    if (k < kend) {
      float gx, gy;
      if (waypoint(L, c, k, kchk, c.boundary, gx, gy)) {
        const Bil bb = bilinear_setup(gx, gy, L.Hb, L.Wb);
        float pg[VEC];
        sample<VEC>(pmap, L.D, ch, bb, pg);
#pragma unroll
        for (int v = 0; v < VEC; ++v) S[v] += pg[v];
#pragma unroll
        for (int j = 0; j < G; ++j) {
          // channels (ch+v)*G + j, v < VEC: for G == 1 one vector, otherwise strided
          if (G == 1) {
            float f[VEC];
            sample<VEC>(fmap, L.D * G, ch, bb, f);
#pragma unroll
            for (int v = 0; v < VEC; ++v) N[v] += pg[v] * f[v];
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
              float f[1];
              sample<1>(fmap, L.D * G, (ch + v) * G + j, bb, f);
              N[v * G + j] += pg[v] * f[0];
            }
          }
        }
      }
    }
  }
}

template <int VEC, int G>
__global__ void __launch_bounds__(kCellsPerBlock * 32)
latent_pool_fwd_kernel(LrDims L, const float* __restrict__ prob, const float* __restrict__ feat,
                       float* __restrict__ pooled, float* __restrict__ aux_s) {
  LR_PROLOGUE
  const float* pmap = prob + (size_t)b * HW * L.D;
  const float* fmap = feat + (size_t)b * HW * L.D * G;
  float S[VEC], N[VEC * G];
  pool_accumulate<VEC, G>(L, c, pmap, fmap, ch, slot, WPI, S, N);
#pragma unroll
  for (int v = 0; v < VEC; ++v)
    for (int off = LPW; off < 32; off <<= 1) S[v] += __shfl_xor_sync(0xffffffffu, S[v], off);
#pragma unroll
  for (int v = 0; v < VEC * G; ++v)
    for (int off = LPW; off < 32; off <<= 1) N[v] += __shfl_xor_sync(0xffffffffu, N[v], off);
  if (slot == 0) {
    float* o = pooled + ((size_t)b * HW + u) * L.D * G;
#pragma unroll
    for (int v = 0; v < VEC; ++v)
#pragma unroll
      for (int j = 0; j < G; ++j) o[(ch + v) * G + j] = N[v * G + j] / (S[v] + L.eps);
    if (aux_s) V<VEC>::st(aux_s + ((size_t)b * HW + u) * L.D + ch, S);
  }
}

// ---------------------------------------------------------------- phase 2 backward
template <int VEC, int G>
__global__ void __launch_bounds__(kCellsPerBlock * 32)
latent_pool_bwd_kernel(LrDims L, const float* __restrict__ prob, const float* __restrict__ feat,
                       const float* __restrict__ grad_pooled, float* __restrict__ grad_prob_map,
                       float* __restrict__ grad_feat, const float* __restrict__ aux_s,
                       const float* __restrict__ pooled) {
  LR_PROLOGUE
  const float* pmap = prob + (size_t)b * HW * L.D;
  const float* fmap = feat + (size_t)b * HW * L.D * G;
  float* gpm = grad_prob_map + (size_t)b * HW * L.D;
  float* gfm = grad_feat + (size_t)b * HW * L.D * G;
  float S[VEC], N[VEC * G];
  if (aux_s) {            // forward saved S; N = pooled * (S + eps)
    V<VEC>::ld(aux_s + ((size_t)b * HW + u) * L.D + ch, S);
    const float* po = pooled + ((size_t)b * HW + u) * L.D * G;
#pragma unroll
    for (int v = 0; v < VEC; ++v)
#pragma unroll
      for (int j = 0; j < G; ++j) N[v * G + j] = __ldg(po + (ch + v) * G + j) * (S[v] + L.eps);
  } else {
    pool_accumulate<VEC, G>(L, c, pmap, fmap, ch, slot, WPI, S, N);
#pragma unroll
    for (int v = 0; v < VEC; ++v)
      for (int off = LPW; off < 32; off <<= 1) S[v] += __shfl_xor_sync(0xffffffffu, S[v], off);
#pragma unroll
    for (int v = 0; v < VEC * G; ++v)
      for (int off = LPW; off < 32; off <<= 1) N[v] += __shfl_xor_sync(0xffffffffu, N[v], off);
  }
  // pooled_c = N_c / (S_d + eps)
  float gN[VEC * G], gS[VEC];
  const float* gp = grad_pooled + ((size_t)b * HW + u) * L.D * G;
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    const float inv = 1.f / (S[v] + L.eps);
    gS[v] = 0.f;
#pragma unroll
    for (int j = 0; j < G; ++j) {
      const float gpc = __ldg(gp + (ch + v) * G + j);
      gN[v * G + j] = gpc * inv;
      gS[v] -= gpc * N[v * G + j] * inv * inv;
    }
  }
  const int kend = march_end(L, c.boundary), kchk = march_check(L, c.boundary);
  for (int k0 = 0; k0 < kend; k0 += WPI) {
    const int k = k0 + slot;
    if (k < kend) {
      float gx, gy;
      if (waypoint(L, c, k, kchk, c.boundary, gx, gy)) {
        const Bil bb = bilinear_setup(gx, gy, L.Hb, L.Wb);
        float pg[VEC], gpg[VEC];
        sample<VEC>(pmap, L.D, ch, bb, pg);
#pragma unroll
        for (int v = 0; v < VEC; ++v) gpg[v] = gS[v];
        if (G == 1) {
          float f[VEC], gf[VEC];
          sample<VEC>(fmap, L.D, ch, bb, f);
#pragma unroll
          for (int v = 0; v < VEC; ++v) { gpg[v] += gN[v] * f[v]; gf[v] = gN[v] * pg[v]; }
          scatter<VEC>(gfm, L.D, ch, bb, gf);
        } else {
#pragma unroll
          for (int v = 0; v < VEC; ++v)
#pragma unroll
            for (int j = 0; j < G; ++j) {
              float f[1], gf[1];
              sample<1>(fmap, L.D * G, (ch + v) * G + j, bb, f);
              gpg[v] += gN[v * G + j] * f[0];
              gf[0] = gN[v * G + j] * pg[v];
              scatter<1>(gfm, L.D * G, (ch + v) * G + j, bb, gf);
            }
        }
        scatter<VEC>(gpm, L.D, ch, bb, gpg);
      }
    }
  }
}

int check_lr(LrDims& L, int bs, int D, int G, int Hb, int Wb, int grid_num, float grid_step, float eps,
             int act, int& vec, const char* who, long long cell0, long long ncells) {
  VIDAR_REQUIRE(bs > 0 && D > 0 && G > 0 && Hb > 1 && Wb > 1 && grid_num > 0,
                "%s: bad sizes bs=%d D=%d G=%d Hb=%d Wb=%d grid_num=%d", who, bs, D, G, Hb, Wb, grid_num);
  VIDAR_REQUIRE(act == 0 || act == 1, "Only support exp or sigmoid activation_fn for now.");
  VIDAR_REQUIRE((D & (D - 1)) == 0 && D <= 32,
                "%s: pred_height=%d unsupported (power of two <= 32)", who, D);
  VIDAR_REQUIRE(G == 1 || G == 2 || G == 4 || G == 8 || G == 16,
                "%s: %d feature channels per height unsupported (1, 2, 4, 8 or 16)", who, G);
  VIDAR_REQUIRE((long long)Hb * Wb * D * G < (1LL << 31), "%s: BEV map too large", who);
  vec = (D % 4 == 0 && G <= 4) ? 4 : 1;   // a lane keeps VEC*G accumulators in registers
  const int half = (Hb < Wb ? Hb : Wb) / 2;
  const long long total = (long long)bs * Hb * Wb;
  VIDAR_REQUIRE(cell0 >= 0 && ncells >= 0 && cell0 <= total && ncells <= total - cell0,
                "%s: bad cell range [%lld, +%lld) of %lld", who, cell0, ncells, total);
  L = LrDims{bs, D, G, Hb, Wb, grid_num, act, (float)((double)grid_step / (double)half), eps, cell0, ncells};
  return VIDAR_OK;
}

inline unsigned lr_blocks(const LrDims& L) {
  return (unsigned)((L.ncells + kCellsPerBlock - 1) / kCellsPerBlock);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

#define LR_DISPATCH_VG(KERNEL, ...)                                                    \
  do {                                                                                 \
    const dim3 grid(lr_blocks(L)), block(kCellsPerBlock * 32);                         \
    if (vec == 4) {                                                                    \
      if (G == 1) KERNEL<4, 1><<<grid, block, 0, st>>>(__VA_ARGS__);                   \
      else if (G == 2) KERNEL<4, 2><<<grid, block, 0, st>>>(__VA_ARGS__);              \
      else KERNEL<4, 4><<<grid, block, 0, st>>>(__VA_ARGS__);                          \
    } else {                                                                           \
      if (G == 1) KERNEL<1, 1><<<grid, block, 0, st>>>(__VA_ARGS__);                   \
      else if (G == 2) KERNEL<1, 2><<<grid, block, 0, st>>>(__VA_ARGS__);              \
      else if (G == 4) KERNEL<1, 4><<<grid, block, 0, st>>>(__VA_ARGS__);              \
      else if (G == 8) KERNEL<1, 8><<<grid, block, 0, st>>>(__VA_ARGS__);              \
      else KERNEL<1, 16><<<grid, block, 0, st>>>(__VA_ARGS__);                         \
    }                                                                                  \
  } while (0)

// aux: optional [3, bs, Hb, Wb, D] floats written by the forward (product of non-zero factors,
// number of zero factors, sum of sampled probabilities) and read by the backward, which then skips
// its recomputation marches.  NULL = forward saves nothing / backward recomputes.
#define AUX_T(a) (a)
#define AUX_NZ(a, n) ((a) ? (a) + (n) : nullptr)
#define AUX_S(a, n) ((a) ? (a) + 2 * (n) : nullptr)

static int prob_fwd(const LrDims& L, int vec, const float* occ, float* prob, float* aux, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  const dim3 grid(lr_blocks(L)), block(kCellsPerBlock * 32);
  if (vec == 4) latent_prob_fwd_kernel<4><<<grid, block, 0, st>>>(L, occ, prob, AUX_T(aux), AUX_NZ(aux, n));
  else latent_prob_fwd_kernel<1><<<grid, block, 0, st>>>(L, occ, prob, AUX_T(aux), AUX_NZ(aux, n));
  return check_launch("LatentRendering.prob_forward");
}

static int pool_fwd(const LrDims& L, int vec, int G, const float* prob, const float* feat, float* pooled,
                    float* aux, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  LR_DISPATCH_VG(latent_pool_fwd_kernel, L, prob, feat, pooled, AUX_S(aux, n));
  return check_launch("LatentRendering.pool_forward");
}

static int pool_bwd(const LrDims& L, int vec, int G, const float* prob, const float* feat, const float* pooled,
                    const float* aux, const float* grad_pooled, float* grad_prob_map, float* grad_feat,
                    cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  const float* as = (aux && pooled) ? aux + 2 * n : nullptr;
  LR_DISPATCH_VG(latent_pool_bwd_kernel, L, prob, feat, grad_pooled, grad_prob_map, grad_feat, as, pooled);
  return check_launch("LatentRendering.pool_backward");
}

static int prob_bwd(const LrDims& L, int vec, const float* occ, const float* aux, const float* grad_prob_total,
                    float* grad_occ, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  const dim3 grid(lr_blocks(L)), block(kCellsPerBlock * 32);
  if (vec == 4) latent_prob_bwd_kernel<4><<<grid, block, 0, st>>>(L, occ, grad_prob_total, grad_occ, aux, aux ? aux + n : nullptr);
  else latent_prob_bwd_kernel<1><<<grid, block, 0, st>>>(L, occ, grad_prob_total, grad_occ, aux, aux ? aux + n : nullptr);
  return check_launch("LatentRendering.prob_backward");
}

extern "C" int vidar_latent_render_forward(const float* occ, const float* feat, float* prob, float* pooled,
                                           float* aux, int bs, int D, int G, int Hb, int Wb, int grid_num,
                                           float grid_step, float eps, int act, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, G, Hb, Wb, grid_num, grid_step, eps, act, vec, "LatentRendering.forward", 0,
                    (long long)bs * Hb * Wb);
  if (rc) return rc;
  VIDAR_REQUIRE(occ && feat && prob && pooled, "LatentRendering.forward: null pointer argument");
  rc = prob_fwd(L, vec, occ, prob, aux, (cudaStream_t)stream);
  if (rc) return rc;
  return pool_fwd(L, vec, G, prob, feat, pooled, aux, (cudaStream_t)stream);
}

extern "C" int vidar_latent_render_backward(const float* occ, const float* feat, const float* prob,
                                            const float* pooled, const float* aux, const float* grad_prob,
                                            const float* grad_pooled, float* grad_prob_total, float* grad_occ,
                                            float* grad_feat, int bs, int D, int G, int Hb, int Wb,
                                            int grid_num, float grid_step, float eps, int act, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, G, Hb, Wb, grid_num, grid_step, eps, act, vec, "LatentRendering.backward", 0,
                    (long long)bs * Hb * Wb);
  if (rc) return rc;
  VIDAR_REQUIRE(occ && feat && prob && grad_prob && grad_pooled && grad_prob_total && grad_occ && grad_feat,
                "LatentRendering.backward: null pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  // grad_prob_total starts as a copy of the upstream grad_prob; phase 2 adds the gradient that
  // reaches the prob map through the ray pooling; phase 1 consumes the sum.
  cudaError_t e = cudaMemcpyAsync(grad_prob_total, grad_prob, sizeof(float) * (size_t)bs * Hb * Wb * D,
                                  cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "LatentRendering.backward: memcpy: %s", cudaGetErrorString(e));
  rc = pool_bwd(L, vec, G, prob, feat, pooled, aux, grad_pooled, grad_prob_total, grad_feat, st);
  if (rc) return rc;
  return prob_bwd(L, vec, occ, aux, grad_prob_total, grad_occ, st);
}

// ---- phase-wise entry points on a cell range: lets the host put a collective between the
// phases when the BEV cells are sharded over GPUs (SURVEY.md 8e).
extern "C" int vidar_latent_prob_forward(const float* occ, float* prob, float* aux, int bs, int D, int Hb,
                                         int Wb, int grid_num, float grid_step, int act, long long cell0,
                                         long long ncells, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, 1, Hb, Wb, grid_num, grid_step, 0.f, act, vec, "LatentRendering.prob_forward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(occ && prob, "LatentRendering.prob_forward: null pointer argument");
  return prob_fwd(L, vec, occ, prob, aux, (cudaStream_t)stream);
}

extern "C" int vidar_latent_pool_forward(const float* prob, const float* feat, float* pooled, float* aux,
                                         int bs, int D, int G, int Hb, int Wb, int grid_num, float grid_step,
                                         float eps, long long cell0, long long ncells, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, G, Hb, Wb, grid_num, grid_step, eps, 1, vec, "LatentRendering.pool_forward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(prob && feat && pooled, "LatentRendering.pool_forward: null pointer argument");
  return pool_fwd(L, vec, G, prob, feat, pooled, aux, (cudaStream_t)stream);
}

extern "C" int vidar_latent_pool_backward(const float* prob, const float* feat, const float* pooled,
                                          const float* aux, const float* grad_pooled, float* grad_prob_map,
                                          float* grad_feat, int bs, int D, int G, int Hb, int Wb, int grid_num,
                                          float grid_step, float eps, long long cell0, long long ncells,
                                          void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, G, Hb, Wb, grid_num, grid_step, eps, 1, vec, "LatentRendering.pool_backward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(prob && feat && grad_pooled && grad_prob_map && grad_feat, "LatentRendering.pool_backward: null pointer argument");
  return pool_bwd(L, vec, G, prob, feat, pooled, aux, grad_pooled, grad_prob_map, grad_feat, (cudaStream_t)stream);
}

extern "C" int vidar_latent_prob_backward(const float* occ, const float* aux, const float* grad_prob_total,
                                          float* grad_occ, int bs, int D, int Hb, int Wb, int grid_num,
                                          float grid_step, int act, long long cell0, long long ncells,
                                          void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, 1, Hb, Wb, grid_num, grid_step, 0.f, act, vec, "LatentRendering.prob_backward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(occ && grad_prob_total && grad_occ, "LatentRendering.prob_backward: null pointer argument");
  return prob_bwd(L, vec, occ, aux, grad_prob_total, grad_occ, (cudaStream_t)stream);
}
