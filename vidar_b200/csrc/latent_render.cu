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
// behind a mask.  Products / sums over waypoints are finished with warp shuffles; per cell the
// forward writes prob (D floats), pooled (D*g floats) and its sums over the waypoints to aux
// (3*D floats).  Backward kernels read those sums and scatter with vector reductions.
// Backward dispatch, by shape: the phase 2 backward with VEC 4 and G 1 (every D in {4, 8, 16, 32} with one
// feature channel per height, the shipped configuration) runs in angular bundles that sum their scatter in
// shared memory (latent_pool_bwd_bundle_kernel); other VEC / G and the phase 1 backward use the per-cell kernels.
#include <limits.h>
#include <math.h>

#include <cub/device/device_radix_sort.cuh>

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

struct BilXY {
  int x0, y0;    // pixel of the nw corner (may lie outside the map)
  float w[4];    // nw, ne, sw, se
};

__device__ __forceinline__ BilXY bilinear_xy(float gx, float gy, int Hb, int Wb) {
  BilXY q;
  // grid_sample: ((g + 1) * size - 1) / 2 ; the division by 2 is exact, so x 0.5 gives the same bits
  const float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)Wb), 1.f), 0.5f);
  const float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)Hb), 1.f), 0.5f);
  const float fx = floorf(ix), fy = floorf(iy);
  q.x0 = (int)fx;
  q.y0 = (int)fy;
  const float wx1 = ix - fx, wy1 = iy - fy;
  const float wx0 = (fx + 1.f) - ix, wy0 = (fy + 1.f) - iy;
#pragma unroll
  for (int j = 0; j < 4; ++j) q.w[j] = ((j & 1) ? wx1 : wx0) * ((j & 2) ? wy1 : wy0);
  return q;
}

// corner j of a footprint: pixel index, or -1 outside the map
__device__ __forceinline__ int corner_pixel(int x0, int y0, int j, int Hb, int Wb) {
  const int xx = x0 + (j & 1), yy = y0 + (j >> 1);
  return (xx >= 0 && xx < Wb && yy >= 0 && yy < Hb) ? yy * Wb + xx : -1;
}

__device__ __forceinline__ Bil bilinear_setup(float gx, float gy, int Hb, int Wb) {
  const BilXY q = bilinear_xy(gx, gy, Hb, Wb);
  Bil b;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    b.o[j] = corner_pixel(q.x0, q.y0, j, Hb, Wb);
    b.w[j] = q.w[j];
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
    V<VEC>::st(aux_t + o, tnz);     // saved for the backward: no second march there
    V<VEC>::st(aux_nz + o, nz);
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
  const int kend = march_end(L, c.lenG), kchk = march_check(L, c.lenG);
  V<VEC>::ld(aux_t + ((size_t)b * HW + u) * L.D + ch, tnz);     // the forward's products
  V<VEC>::ld(aux_nz + ((size_t)b * HW + u) * L.D + ch, nz);
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
    V<VEC>::st(aux_s + ((size_t)b * HW + u) * L.D + ch, S);
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
  // forward saved S; N = pooled * (S + eps)
  V<VEC>::ld(aux_s + ((size_t)b * HW + u) * L.D + ch, S);
  const float* po = pooled + ((size_t)b * HW + u) * L.D * G;
#pragma unroll
  for (int v = 0; v < VEC; ++v)
#pragma unroll
    for (int j = 0; j < G; ++j) N[v * G + j] = __ldg(po + (ch + v) * G + j) * (S[v] + L.eps);
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

// ---------------------------------------------------------------- phase 2 backward in angular bundles (VEC 4, G 1)
// latent_pool_bwd_kernel sends one 16-byte reduction per (cell, waypoint, corner, float4, map): 18.3 M 64-byte
// lines per map at 200 x 200 with grid_num 256.  Every ray starts at the BEV centre and waypoint k of
// every ray lies ~k px from it, so the cells sorted by the direction of their ray and cut into bundles of
// kBundle consecutive cells put their kBundle footprints of one waypoint inside a kBox x kBox pixel box
// (a 4 x 4 box holds every bundle of 32 at 200 x 200).  A bundle kernel sums the bundle's contributions to
// each box pixel in shared memory, in a fixed cell order, and sends one reduction per touched pixel and map:
// 0.67 M lines per map at the bench shape.  A corner outside its box (bundles across the +-pi cut, the centre
// cell, small BEVs, a bundle's cells of a second batch element) is reduced straight to global memory as in the
// per-cell kernel.  The phase 1 backward keeps its per-cell kernel: its rays end at their own cell, so a
// bundle of cells at every radius along one direction spends most of its waypoints on finished cells, and the
// bundled form measured slower than the per-cell one (DESIGN.md 4.3).
constexpr int kBundle = 32;                                 // cells per bundle = lanes of a warp
constexpr int kBundleThreads = 256;
constexpr int kChunk = kBundleThreads / kBundle;            // waypoints staged in shared memory at a time
constexpr int kBox = 4;
constexpr int kAngleBits = 20;                              // angle bins of the cell order
constexpr int kNoCorner = -(1 << 29);                       // footprint slot of a (waypoint, cell) with no sample

// Cell order, key: batch element (relative to the range's first) above the angle bin of the cell's direction from
// the BEV centre, taken from its integer position so that it is exact on any BEV shape.
__global__ void __launch_bounds__(256) latent_order_key_kernel(LrDims L, unsigned long long* __restrict__ key,
                                                                int* __restrict__ idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.ncells) return;
  const int HW = L.Hb * L.Wb;
  const long long cell = L.cell0 + i;
  const int u = (int)(cell % HW), iy = u / L.Wb, ix = u % L.Wb;
  const float a = atan2f((float)(2 * iy + 1 - L.Hb), (float)(2 * ix + 1 - L.Wb));   // [-pi, pi]
  const float pi = 3.14159265358979f;
  const int bin = min(max((int)((a + pi) * ((float)(1 << kAngleBits) / (2.f * pi))), 0), (1 << kAngleBits) - 1);
  key[i] = ((unsigned long long)(cell / HW - L.cell0 / HW) << kAngleBits) | (unsigned)bin;
  idx[i] = (int)i;
}

// Shared memory of a bundle CTA: the fixed part, then per-height coefficient rows and the staged vectors.
struct BundleSmem {
  Cell cg[kBundle];
  int kend[kBundle], kchk[kBundle], bat[kBundle];   // bat: batch element, -1 past the range
  int2 xy[kChunk][kBundle];                         // nw corner pixel of (waypoint, cell); kNoCorner = no sample
  float4 w[kChunk][kBundle];                        // bilinear weights
  int2 box[kChunk];                                 // box origin of each waypoint; INT_MAX = empty
  unsigned who[kChunk][kBox * kBox];                // cells with a corner on each box pixel
  unsigned direct[kChunk];                          // cells with a corner the box does not cover
};
// then the gN, gS rows [2][kBundle][D] and the grad_feat, grad_prob_map vectors [2][kChunk][kBundle][D]
inline size_t bundle_smem_bytes(int D) {
  return sizeof(BundleSmem) + sizeof(float) * (size_t)D * kBundle * (2 + 2 * kChunk);
}

// latent_pool_bwd_kernel<4, 1> on the cells of `order`, one CTA per kBundle consecutive ones.  map0 = prob,
// grad_in = grad_pooled, out0 = grad_feat, out1 = grad_prob_map; aux0 / aux1 = the forward's S and pooled.
// prologue: a warp per cell forms gN and gS as latent_pool_bwd_kernel does.  Then per chunk of kChunk waypoints:
//   A1  thread = (waypoint, cell): waypoint, mask, bilinear footprint; the box origin is the warp's minimum
//       corner; ballots give each box pixel's cells and the cells with a corner outside the box.
//   A2  thread = (waypoint, cell, float4): gathers of prob and feat, gN pg and gS + gN f into shared memory.
//   B   corners outside the box are reduced to global memory; thread = (waypoint, box pixel, float4) sums the
//       pixel's cells in cell order and sends one reduction per touched pixel and map.
__global__ void __launch_bounds__(kBundleThreads, 4)
latent_pool_bwd_bundle_kernel(LrDims L, const int* __restrict__ order, const float* __restrict__ map0,
                              const float* __restrict__ feat, const float* __restrict__ grad_in,
                              float* __restrict__ out0, float* __restrict__ out1, const float* __restrict__ aux0,
                              const float* __restrict__ aux1) {
  constexpr int VEC = 4;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BundleSmem& sm = *reinterpret_cast<BundleSmem*>(smem_raw);
  float* rows = reinterpret_cast<float*>(smem_raw + sizeof(BundleSmem));   // [rows][kBundle][D]
  float* vec = rows + 2 * kBundle * L.D;                                    // [2][kChunk][kBundle][D]
  const int D = L.D, LPW = D / VEC, HW = L.Hb * L.Wb;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = lane / LPW, ch = (lane % LPW) * VEC;

  // ---- prologue: warp per cell
  for (int c = warp; c < kBundle; c += kBundleThreads / 32) {
    const long long pos = (long long)blockIdx.x * kBundle + c;
    if (pos >= L.ncells) {
      if (lane == 0) { sm.kend[c] = 0; sm.bat[c] = -1; }
      continue;
    }
    const long long cell = L.cell0 + __ldg(order + pos);
    const int b = (int)(cell / HW), u = (int)(cell % HW);
    const Cell cg = cell_geometry(L, u / L.Wb, u % L.Wb);
    const size_t o = ((size_t)b * HW + u) * D + ch;
    {   // pooled_c = N_c / (S_d + eps)
      float S[VEC], N[VEC];
      V<VEC>::ld(aux0 + o, S);
#pragma unroll
      for (int v = 0; v < VEC; ++v) N[v] = __ldg(aux1 + o + v) * (S[v] + L.eps);
      float gN[VEC], gS[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const float inv = 1.f / (S[v] + L.eps);
        const float gpc = __ldg(grad_in + o + v);
        gN[v] = gpc * inv;
        gS[v] = 0.f;
        gS[v] -= gpc * N[v] * inv * inv;
      }
      if (slot == 0) {
        V<VEC>::st(rows + c * D + ch, gN);
        V<VEC>::st(rows + (kBundle + c) * D + ch, gS);
      }
      if (lane == 0) {
        sm.kend[c] = march_end(L, cg.boundary);
        sm.kchk[c] = march_check(L, cg.boundary);
      }
    }
    if (lane == 0) {
      sm.cg[c] = cg;
      sm.bat[c] = b;
    }
  }
  __syncthreads();
  int kmax = 0;
  for (int c = 0; c < kBundle; ++c) kmax = max(kmax, sm.kend[c]);
  const int b0 = sm.bat[0];
  float* const o0 = out0 + (size_t)b0 * HW * D;
  float* const o1 = out1 + (size_t)b0 * HW * D;

  for (int k0 = 0; k0 < kmax; k0 += kChunk) {
    // ---- A1: thread = (waypoint kk = warp, cell c = lane)
    {
      const int kk = warp, c = lane, k = k0 + kk;
      float gx, gy;
      const bool live = k < sm.kend[c] && waypoint(L, sm.cg[c], k, sm.kchk[c], sm.cg[c].boundary, gx, gy);
      int2 xy = make_int2(kNoCorner, kNoCorner);
      if (live) {
        const BilXY q = bilinear_xy(gx, gy, L.Hb, L.Wb);
        xy = make_int2(q.x0, q.y0);
        sm.w[kk][c] = make_float4(q.w[0], q.w[1], q.w[2], q.w[3]);
      }
      sm.xy[kk][c] = xy;
      const bool boxed = live && sm.bat[c] == b0;
      const int bx = __reduce_min_sync(0xffffffffu, boxed ? xy.x : INT_MAX);
      const int by = __reduce_min_sync(0xffffffffu, boxed ? xy.y : INT_MAX);
      if (lane == 0) sm.box[kk] = make_int2(bx, by);
      // cells of each box pixel: bit c of who[kk][p] = corner (p % kBox - dx, p / kBox - dy) of cell c
      const int dx = boxed ? xy.x - bx : 0, dy = boxed ? xy.y - by : 0;
      bool direct = live && !boxed;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        direct |= boxed && corner_pixel(xy.x, xy.y, j, L.Hb, L.Wb) >= 0 &&
                  (dx + (j & 1) >= kBox || dy + (j >> 1) >= kBox);
      const unsigned dm = __ballot_sync(0xffffffffu, direct);
      if (lane == 0) sm.direct[kk] = dm;
#pragma unroll
      for (int p = 0; p < kBox * kBox; ++p) {
        const int px = p % kBox - dx, py = p / kBox - dy;
        const bool in = boxed && px >= 0 && px <= 1 && py >= 0 && py <= 1;
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == p) sm.who[kk][p] = m;
      }
    }
    __syncthreads();
    // ---- A2: thread = (waypoint, cell, float4); lanes of one cell adjacent, so a corner is one 64-byte line
#pragma unroll 4
    for (int i = threadIdx.x; i < kChunk * kBundle * LPW; i += kBundleThreads) {
      const int l = i % LPW, c = (i / LPW) % kBundle, kk = i / (LPW * kBundle);
      const int2 xy = sm.xy[kk][c];
      if (xy.x == kNoCorner) continue;
      const int b = sm.bat[c], chl = l * VEC;
      const float4 w4 = sm.w[kk][c];
      const float wj[4] = {w4.x, w4.y, w4.z, w4.w};
      int oj[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) oj[j] = corner_pixel(xy.x, xy.y, j, L.Hb, L.Wb);
      float v0[VEC], v1[VEC];
      {
        const float* pmap = map0 + (size_t)b * HW * D;
        const float* fmap = feat + (size_t)b * HW * D;
        float pg[VEC], f[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) { pg[v] = 0.f; f[v] = 0.f; }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (oj[j] >= 0) {
            float t[VEC], s[VEC];
            V<VEC>::ld(pmap + (size_t)oj[j] * D + chl, t);
            V<VEC>::ld(fmap + (size_t)oj[j] * D + chl, s);
#pragma unroll
            for (int v = 0; v < VEC; ++v) { pg[v] += t[v] * wj[j]; f[v] += s[v] * wj[j]; }
          }
        }
        const float* gN = rows + c * D + chl;
        const float* gS = rows + (kBundle + c) * D + chl;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          v0[v] = gN[v] * pg[v];                 // grad_feat
          v1[v] = gS[v] + gN[v] * f[v];          // grad_prob_map
        }
      }
      float* vs = vec + ((size_t)kk * kBundle + c) * D + chl;
      V<VEC>::st(vs, v0);
      V<VEC>::st(vs + (size_t)kChunk * kBundle * D, v1);
    }
    __syncthreads();
    // ---- corners the box does not cover, reduced straight to global memory (kept out of A2 so that its gathers
    //      are not ordered behind reductions)
    for (int i = threadIdx.x; i < kChunk * kBundle * LPW; i += kBundleThreads) {
      const int l = i % LPW, c = (i / LPW) % kBundle, kk = i / (LPW * kBundle);
      if (!((sm.direct[kk] >> c) & 1u)) continue;
      const int2 xy = sm.xy[kk][c], box = sm.box[kk];
      const int b = sm.bat[c], chl = l * VEC;
      const float4 w4 = sm.w[kk][c];
      const float wj[4] = {w4.x, w4.y, w4.z, w4.w};
      const float* vs = vec + ((size_t)kk * kBundle + c) * D + chl;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int o = corner_pixel(xy.x, xy.y, j, L.Hb, L.Wb);
        const int dx = xy.x + (j & 1) - box.x, dy = xy.y + (j >> 1) - box.y;
        if (o < 0 || (b == b0 && dx < kBox && dy < kBox)) continue;
        float t[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) t[v] = vs[v] * wj[j];
        V<VEC>::red(out0 + ((size_t)b * HW + o) * D + chl, t);
#pragma unroll
        for (int v = 0; v < VEC; ++v) t[v] = vs[(size_t)kChunk * kBundle * D + v] * wj[j];
        V<VEC>::red(out1 + ((size_t)b * HW + o) * D + chl, t);
      }
    }
    // ---- B: thread = (waypoint, box pixel, float4)
    for (int i = threadIdx.x; i < kChunk * kBox * kBox * LPW; i += kBundleThreads) {
      const int l = i % LPW, p = (i / LPW) % (kBox * kBox), kk = i / (LPW * kBox * kBox);
      unsigned m = sm.who[kk][p];
      if (!m) continue;
      const int2 box = sm.box[kk];
      const int px = box.x + p % kBox, py = box.y + p / kBox;
      if (px < 0 || px >= L.Wb || py < 0 || py >= L.Hb) continue;
      float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
      const float* vk = vec + (size_t)kk * kBundle * D + l * VEC;
      for (; m; m &= m - 1) {             // the pixel's cells in cell order
        const int c = __ffs(m) - 1;
        const int2 xy = sm.xy[kk][c];
        const int dx = px - xy.x, dy = py - xy.y;
        const float4 w4 = sm.w[kk][c];
        const float w = dy ? (dx ? w4.w : w4.z) : (dx ? w4.y : w4.x);
        const float4 v0 = *reinterpret_cast<const float4*>(vk + c * D);
        a0.x += v0.x * w; a0.y += v0.y * w; a0.z += v0.z * w; a0.w += v0.w * w;
        const float4 v1 = *reinterpret_cast<const float4*>(vk + (size_t)kChunk * kBundle * D + c * D);
        a1.x += v1.x * w; a1.y += v1.y * w; a1.z += v1.z * w; a1.w += v1.w * w;
      }
      const size_t o = (size_t)(py * L.Wb + px) * D + l * VEC;
      red_add_v4(o0 + o, a0);
      red_add_v4(o1 + o, a1);
    }
    __syncthreads();
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

// Phase 2 backward in bundles: cell order (key kernel + CUB's stable radix sort) and the bundle kernel.  The order's scratch (two keys and two
// indices per cell, the sort's temp storage) is stream-ordered from the library's pool.
int pool_bwd_bundled(const LrDims& L, const float* map0, const float* feat, const float* grad_in, float* out0, float* out1,
               const float* aux0, const float* aux1, cudaStream_t st, const char* who) {
  VIDAR_REQUIRE(L.ncells < INT_MAX, "%s: %lld cells, at most 2^31 - 1", who, L.ncells);
  const int n = (int)L.ncells, HW = L.Hb * L.Wb;
  const long long nbat = (L.cell0 + L.ncells - 1) / HW - L.cell0 / HW + 1;
  int bits = kAngleBits;
  while ((1LL << (bits - kAngleBits)) < nbat) ++bits;
  const size_t smem = bundle_smem_bytes(L.D);
  if (cudaFuncSetAttribute(latent_pool_bwd_bundle_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return set_error(VIDAR_E_CUDA, "%s: cannot opt in to %zu bytes of shared memory", who, smem);
  using Key = unsigned long long;
  size_t tmp = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, tmp, (const Key*)nullptr, (Key*)nullptr, (const int*)nullptr,
                                                  (int*)nullptr, n, 0, bits, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cell order: %s", who, cudaGetErrorString(e));
  const size_t off = ((sizeof(Key) + sizeof(int)) * 2 * (size_t)n + 255) & ~(size_t)255;
  cudaMemPool_t pool;
  e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, off + tmp, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  Key* k0 = reinterpret_cast<Key*>(s);
  Key* k1 = k0 + n;
  int* i0 = reinterpret_cast<int*>(k1 + n);
  int* i1 = i0 + n;
  latent_order_key_kernel<<<(n + 255) / 256, 256, 0, st>>>(L, k0, i0);
  e = cub::DeviceRadixSort::SortPairs(s + off, tmp, k0, k1, i0, i1, n, 0, bits, st);
  if (e == cudaSuccess)
    latent_pool_bwd_bundle_kernel<<<(unsigned)((n + kBundle - 1) / kBundle), kBundleThreads, smem, st>>>(
        L, i1, map0, feat, grad_in, out0, out1, aux0, aux1);
  const cudaError_t ef = cudaFreeAsync(s, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cell order: %s", who, cudaGetErrorString(e));
  if (ef != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(ef));
  return VIDAR_OK;
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

// aux: [3, bs, Hb, Wb, D] floats written by the forward (product of non-zero factors, number of
// zero factors, sum of sampled probabilities) and read by the backward instead of a second march.
static int prob_fwd(const LrDims& L, int vec, const float* occ, float* prob, float* aux, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  const dim3 grid(lr_blocks(L)), block(kCellsPerBlock * 32);
  if (vec == 4) latent_prob_fwd_kernel<4><<<grid, block, 0, st>>>(L, occ, prob, aux, aux + n);
  else latent_prob_fwd_kernel<1><<<grid, block, 0, st>>>(L, occ, prob, aux, aux + n);
  return check_launch("LatentRendering.prob_forward");
}

static int pool_fwd(const LrDims& L, int vec, int G, const float* prob, const float* feat, float* pooled,
                    float* aux, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  LR_DISPATCH_VG(latent_pool_fwd_kernel, L, prob, feat, pooled, aux + 2 * n);
  return check_launch("LatentRendering.pool_forward");
}

static int pool_bwd(const LrDims& L, int vec, int G, const float* prob, const float* feat, const float* pooled,
                    const float* aux, const float* grad_pooled, float* grad_prob_map, float* grad_feat,
                    cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  if (vec == 4 && G == 1) {
    const int rc = pool_bwd_bundled(L, prob, feat, grad_pooled, grad_feat, grad_prob_map, aux + 2 * n, pooled, st,
                                    "LatentRendering.pool_backward");
    if (rc) return rc;
  } else {
    LR_DISPATCH_VG(latent_pool_bwd_kernel, L, prob, feat, grad_pooled, grad_prob_map, grad_feat, aux + 2 * n, pooled);
  }
  return check_launch("LatentRendering.pool_backward");
}

static int prob_bwd(const LrDims& L, int vec, const float* occ, const float* aux, const float* grad_prob_total,
                    float* grad_occ, cudaStream_t st) {
  if (L.ncells == 0) return VIDAR_OK;
  const size_t n = (size_t)L.bs * L.Hb * L.Wb * L.D;
  const dim3 grid(lr_blocks(L)), block(kCellsPerBlock * 32);
  if (vec == 4) latent_prob_bwd_kernel<4><<<grid, block, 0, st>>>(L, occ, grad_prob_total, grad_occ, aux, aux + n);
  else latent_prob_bwd_kernel<1><<<grid, block, 0, st>>>(L, occ, grad_prob_total, grad_occ, aux, aux + n);
  return check_launch("LatentRendering.prob_backward");
}

// ---- entry points: one phase per call on a cell range, so the host can put a collective between
// the phases when the BEV cells are sharded over GPUs (SURVEY.md 8e).
extern "C" int vidar_latent_prob_forward(const float* occ, float* prob, float* aux, int bs, int D, int Hb,
                                         int Wb, int grid_num, float grid_step, int act, long long cell0,
                                         long long ncells, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, 1, Hb, Wb, grid_num, grid_step, 0.f, act, vec, "LatentRendering.prob_forward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(occ && prob && aux, "LatentRendering.prob_forward: null pointer argument");
  return prob_fwd(L, vec, occ, prob, aux, (cudaStream_t)stream);
}

extern "C" int vidar_latent_pool_forward(const float* prob, const float* feat, float* pooled, float* aux,
                                         int bs, int D, int G, int Hb, int Wb, int grid_num, float grid_step,
                                         float eps, long long cell0, long long ncells, void* stream) {
  LrDims L;
  int vec;
  int rc = check_lr(L, bs, D, G, Hb, Wb, grid_num, grid_step, eps, 1, vec, "LatentRendering.pool_forward", cell0, ncells);
  if (rc) return rc;
  VIDAR_REQUIRE(prob && feat && pooled && aux, "LatentRendering.pool_forward: null pointer argument");
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
  VIDAR_REQUIRE(prob && feat && pooled && aux && grad_pooled && grad_prob_map && grad_feat,
                "LatentRendering.pool_backward: null pointer argument");
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
  VIDAR_REQUIRE(occ && aux && grad_prob_total && grad_occ, "LatentRendering.prob_backward: null pointer argument");
  return prob_bwd(L, vec, occ, aux, grad_prob_total, grad_occ, (cudaStream_t)stream);
}
