// ViDAR head ray sampler, fused cross-entropy and arg-max decode for H100 (sm_90a).
//
// Reference (pure PyTorch, many launches and [R,513] intermediates):
//   projects/mmdet3d_plugin/bevformer/dense_heads/vidar_head_base.py
//     _get_grid_features :420-509   waypoints + trilinear F.grid_sample + -inf mask
//     loss               :586-592   F.cross_entropy(label 0) over the 513 logits of a ray
//     get_point_cloud_prediction :706-738   zeros -> -inf, argmax, waypoint length
// Per ray (origin o, GT point g, voxel units), SURVEY.md A.4:
//     u = (g-o)/|g-o| ; x_0 = g ; x_{k+1} = o + u * ((k+0.5)*step), k < num_way
//     n = 2*x/(W,H,Z) - 1 ; logit_k = trilinear(sigma, n_k)  (align_corners=False, zeros)
//                           or -inf when any |n_k| >= 1
// All coordinate arithmetic is done in fp32 with the reference's operation order (explicit
// _rn intrinsics, no FMA contraction) so the same voxel corners are picked.
//
// Mapping: one warp per ray, lanes over waypoints (lane l handles k = l, l+32, ...):
// neighbouring lanes sample neighbouring voxels, so the 8-corner gathers of a warp fall in
// a handful of lines of the 2.56 MB frame volume (L1/L2 resident).  The fused CE path keeps
// an online log-sum-exp per lane, merges lanes by shuffle, and writes 2 floats per ray
// instead of the reference's [R,513] logits + mask + transposed copy; its backward
// recomputes the logits and scatters softmax-minus-onehot straight into grad_sigma.
#include <math.h>

#include "common.cuh"

namespace vidar {
namespace {

struct RayDims {
  int R, F, Z, Y, X, num_way, with_gt;
  float step;
};

struct Sample {
  float ix, iy, iz;   // un-normalised grid_sample coordinates
  float length;       // |x - o|
  bool masked;        // any |n| >= 1  (logit = -inf)
};

struct RaySetup {
  float ox, oy, oz, gx, gy, gz, ux, uy, uz;
  int f;
  bool live;          // frame in [0, F): a ray of another frame (e.g. -1 for padding) is skipped, nothing is read
};

__device__ __forceinline__ RaySetup load_ray(const RayDims& D, const float* __restrict__ origin,
                                             const float* __restrict__ points,
                                             const int32_t* __restrict__ frame, int r) {
  RaySetup s;
  s.f = frame ? frame[r] : 0;
  s.live = s.f >= 0 && s.f < D.F;
  if (!s.live) return s;
  const float* o = origin + (size_t)s.f * 3;
  s.ox = o[0]; s.oy = o[1]; s.oz = o[2];
  s.gx = points[(size_t)r * 3]; s.gy = points[(size_t)r * 3 + 1]; s.gz = points[(size_t)r * 3 + 2];
  const float rx = __fsub_rn(s.gx, s.ox), ry = __fsub_rn(s.gy, s.oy), rz = __fsub_rn(s.gz, s.oz);
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry)), __fmul_rn(rz, rz)));
  s.ux = __fdiv_rn(rx, nrm); s.uy = __fdiv_rn(ry, nrm); s.uz = __fdiv_rn(rz, nrm);
  return s;
}

// sample k of the ray (k = 0 is the GT point when with_gt)
__device__ __forceinline__ Sample make_sample(const RayDims& D, const RaySetup& s, int k) {
  float x, y, z;
  if (D.with_gt && k == 0) {
    x = s.gx; y = s.gy; z = s.gz;
  } else {
    const float t = __fmul_rn((float)(k - D.with_gt) + 0.5f, D.step);
    x = __fadd_rn(s.ox, __fmul_rn(s.ux, t));
    y = __fadd_rn(s.oy, __fmul_rn(s.uy, t));
    z = __fadd_rn(s.oz, __fmul_rn(s.uz, t));
  }
  Sample q;
  const float dx = __fsub_rn(x, s.ox), dy = __fsub_rn(y, s.oy), dz = __fsub_rn(z, s.oz);
  q.length = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  const float nx = __fsub_rn(__fmul_rn(__fdiv_rn(x, (float)D.X), 2.f), 1.f);
  const float ny = __fsub_rn(__fmul_rn(__fdiv_rn(y, (float)D.Y), 2.f), 1.f);
  const float nz = __fsub_rn(__fmul_rn(__fdiv_rn(z, (float)D.Z), 2.f), 1.f);
  // `(grid <= -1) | (grid >= 1)`: NaN compares false -> not masked, like the reference
  q.masked = (nx <= -1.f) || (nx >= 1.f) || (ny <= -1.f) || (ny >= 1.f) || (nz <= -1.f) || (nz >= 1.f);
  // grid_sample un-normalisation, align_corners=False: ((n + 1) * size - 1) / 2 (x 0.5: same bits)
  q.ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(nx, 1.f), (float)D.X), 1.f), 0.5f);
  q.iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(ny, 1.f), (float)D.Y), 1.f), 0.5f);
  q.iz = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(nz, 1.f), (float)D.Z), 1.f), 0.5f);
  return q;
}

__device__ __forceinline__ bool gt_inside(const RayDims& D, const RaySetup& s) {
  const float nx = __fsub_rn(__fmul_rn(__fdiv_rn(s.gx, (float)D.X), 2.f), 1.f);
  const float ny = __fsub_rn(__fmul_rn(__fdiv_rn(s.gy, (float)D.Y), 2.f), 1.f);
  const float nz = __fsub_rn(__fmul_rn(__fdiv_rn(s.gz, (float)D.Z), 2.f), 1.f);
  return nx > -1.f && nx < 1.f && ny > -1.f && ny < 1.f && nz > -1.f && nz < 1.f;
}

// 8 corners: index (or -1 when out of bounds) and weight, in grid_sample's order
// (tnw, tne, tsw, tse, bnw, bne, bsw, bse) = x fastest, then y, then z.
struct Corners {
  int idx[8];
  float w[8];
};

__device__ __forceinline__ Corners corners(const RayDims& D, const Sample& q) {
  Corners c;
  const float fx = floorf(q.ix), fy = floorf(q.iy), fz = floorf(q.iz);
  const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
  const float wx1 = q.ix - fx, wy1 = q.iy - fy, wz1 = q.iz - fz;     // weight of the +1 corner
  const float wx0 = (fx + 1.f) - q.ix, wy0 = (fy + 1.f) - q.iy, wz0 = (fz + 1.f) - q.iz;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int xx = x0 + (j & 1), yy = y0 + ((j >> 1) & 1), zz = z0 + (j >> 2);
    const bool in = xx >= 0 && xx < D.X && yy >= 0 && yy < D.Y && zz >= 0 && zz < D.Z;
    c.idx[j] = in ? (zz * D.Y + yy) * D.X + xx : -1;
    c.w[j] = ((j & 1) ? wx1 : wx0) * ((j & 2) ? wy1 : wy0) * ((j & 4) ? wz1 : wz0);
  }
  return c;
}

__device__ __forceinline__ float trilinear(const float* __restrict__ vol, const Corners& c) {
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (c.idx[j] >= 0) acc += __ldg(vol + c.idx[j]) * c.w[j];
  return acc;
}

// NaN coordinates: floorf(NaN) -> int conversion is 0 on the GPU, weights NaN -> NaN logit
// (the reference propagates NaN too).

constexpr int kRaysPerBlock = 8;   // 8 warps

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The order of torch's max / argmax: a NaN above every number, the smaller index on ties (and among NaNs).
// A lane that holds no sample starts at (-inf, INT_MAX), so its first sample always replaces it.
__device__ __forceinline__ bool argmax_takes(float v, int k, float best, int best_k) {
  const bool vn = isnan(v), bn = isnan(best);
  if (vn != bn) return vn;
  return (vn || v == best) ? k < best_k : v > best;
}

// warp arg-max of (value, index) in that order, carrying the winner's length
__device__ __forceinline__ void warp_argmax(float& best, int& best_k, float& best_len) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int ok = __shfl_xor_sync(0xffffffffu, best_k, o);
    const float ol = __shfl_xor_sync(0xffffffffu, best_len, o);
    if (argmax_takes(ov, ok, best, best_k)) { best = ov; best_k = ok; best_len = ol; }
  }
}

// ---- materialising sampler (API parity with _get_grid_features) --------------------------
__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_sample_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                  const float* __restrict__ points, const int32_t* __restrict__ frame,
                  float* __restrict__ logits, float* __restrict__ length, float* __restrict__ valid) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  const float* vol = sigma + (size_t)s.f * D.Z * D.Y * D.X;
  const int K = D.num_way + D.with_gt;
  if (valid && lane == 0) valid[r] = (s.live && (!D.with_gt || gt_inside(D, s))) ? 1.f : 0.f;
  if (!s.live) {
    for (int k = lane; k < K; k += 32) {
      if (logits) logits[(size_t)r * K + k] = -INFINITY;
      if (length) length[(size_t)r * K + k] = 0.f;
    }
    return;
  }
  for (int k = lane; k < K; k += 32) {
    const Sample q = make_sample(D, s, k);
    float v = -INFINITY;
    if (!q.masked) v = trilinear(vol, corners(D, q));
    if (logits) logits[(size_t)r * K + k] = v;
    if (length) length[(size_t)r * K + k] = q.length;
  }
}

__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_sample_bwd_kernel(RayDims D, const float* __restrict__ origin, const float* __restrict__ points,
                      const int32_t* __restrict__ frame, const float* __restrict__ grad_logits,
                      float* __restrict__ grad_sigma) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live) return;
  float* gvol = grad_sigma + (size_t)s.f * D.Z * D.Y * D.X;
  const int K = D.num_way + D.with_gt;
  for (int k = lane; k < K; k += 32) {
    const float g = grad_logits[(size_t)r * K + k];
    if (g == 0.f) continue;
    const Sample q = make_sample(D, s, k);
    if (q.masked) continue;
    const Corners c = corners(D, q);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c.idx[j] >= 0) red_add_f32(gvol + c.idx[j], g * c.w[j]);
  }
}

// ---- fused cross-entropy (label 0) ---------------------------------------------------------
__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_ce_fwd_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                  const float* __restrict__ points, const int32_t* __restrict__ frame,
                  float* __restrict__ ce, float* __restrict__ lse_out, float* __restrict__ valid) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live || !gt_inside(D, s)) {   // the reference drops the ray (:464-467)
    if (lane == 0) { ce[r] = 0.f; lse_out[r] = 0.f; valid[r] = 0.f; }
    return;
  }
  const float* vol = sigma + (size_t)s.f * D.Z * D.Y * D.X;
  const int K = D.num_way + 1;
  float m = -INFINITY, acc = 0.f, logit0 = 0.f;
  for (int k = lane; k < K; k += 32) {
    const Sample q = make_sample(D, s, k);
    if (q.masked) continue;
    const float v = trilinear(vol, corners(D, q));
    if (k == 0) logit0 = v;
    if (v > m) { acc = acc * expf(m - v) + 1.f; m = v; }
    else acc += expf(v - m);
  }
  const float M = warp_max(m);
  const float S = warp_sum((m == -INFINITY) ? 0.f : acc * expf(m - M));
  const float lse = M + logf(S);
  logit0 = __shfl_sync(0xffffffffu, logit0, 0);
  if (lane == 0) { ce[r] = lse - logit0; lse_out[r] = lse; valid[r] = 1.f; }
}

__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_ce_bwd_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                  const float* __restrict__ points, const int32_t* __restrict__ frame,
                  const float* __restrict__ lse_in, const float* __restrict__ grad_ce,
                  float* __restrict__ grad_sigma) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const float g = grad_ce ? grad_ce[r] : 1.f;
  if (g == 0.f) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live || !gt_inside(D, s)) return;
  const size_t voff = (size_t)s.f * D.Z * D.Y * D.X;
  const float* vol = sigma + voff;
  float* gvol = grad_sigma + voff;
  const float lse = lse_in[r];
  const int K = D.num_way + 1;
  for (int k = lane; k < K; k += 32) {
    const Sample q = make_sample(D, s, k);
    if (q.masked) continue;
    const Corners c = corners(D, q);
    const float v = trilinear(vol, c);
    const float dl = g * (expf(v - lse) - (k == 0 ? 1.f : 0.f));   // softmax - onehot(0)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c.idx[j] >= 0) red_add_f32(gvol + c.idx[j], dl * c.w[j]);
  }
}

// ---- fused gumbel decode of the dense loss term --------------------------------------------
// ViDARHeadBase._custom_gumbel_softmax_distance (vidar_head_base.py:754-773) on the sampler's
// logits without the GT slot (`dense_feat_total[0][..., 1:]`, :631-636), per ray:
//   idx   = argmax_k (logit_k + gumbel_k)                 F.gumbel_softmax(hard=True), forward value; the
//                                                         reference takes the arg-max of softmax(logit + gumbel),
//                                                         which can round two distinct maxima to one value
//                                                         (DESIGN.md 4.4): this is the exact arg-max in fp32
//   pred  = length_idx                                    ((1 - s) + s == 1 exactly in fp32)
//   p     = sum_{length_k > pred} e^{logit_k} / sum_k e^{logit_k}
//   out   = (1 - p.detach() + p) * pred  = pred,          d out / d logit_j = pred * softmax_j * ([length_j > pred] - p)
// The [rays, 512] logits, softmax and one-hot tensors of the reference are never written; the
// noise is an input (drawn by the host exactly like F.gumbel_softmax draws it).
__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_gumbel_fwd_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                      const float* __restrict__ points, const int32_t* __restrict__ frame,
                      const float* __restrict__ noise, float* __restrict__ dist,
                      float* __restrict__ lse_out, float* __restrict__ p_out) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live || !gt_inside(D, s)) {
    if (lane == 0) { dist[r] = 0.f; lse_out[r] = 0.f; p_out[r] = 0.f; }
    return;
  }
  const float* vol = sigma + (size_t)s.f * D.Z * D.Y * D.X;
  const float* nz = noise + (size_t)r * D.num_way;
  float m = -INFINITY, acc = 0.f, best = -INFINITY, best_len = 0.f;
  int best_k = 0x7fffffff;
  for (int k = 1 + lane; k <= D.num_way; k += 32) {
    const Sample q = make_sample(D, s, k);
    const float v = q.masked ? -INFINITY : trilinear(vol, corners(D, q));
    const float y = v + __ldg(nz + k - 1);
    if (argmax_takes(y, k, best, best_k)) { best = y; best_k = k; best_len = q.length; }
    if (v > m) { acc = acc * expf(m - v) + 1.f; m = v; }
    else if (v > -INFINITY) acc += expf(v - m);
  }
  warp_argmax(best, best_k, best_len);
  const float M = warp_max(m);
  const float S = warp_sum((m == -INFINITY) ? 0.f : acc * expf(m - M));
  float nx = 0.f;
  for (int k = 1 + lane; k <= D.num_way; k += 32) {
    const Sample q = make_sample(D, s, k);
    if (q.masked || !(q.length > best_len)) continue;
    nx += expf(trilinear(vol, corners(D, q)) - M);
  }
  nx = warp_sum(nx);
  // every waypoint masked (the origin outside the volume): S = 0, the reference's softmax is NaN; here the
  // first waypoint's length, lse = -inf, p_next = 0, and the backward scatters nothing (DESIGN.md 4.4)
  if (lane == 0) { dist[r] = best_len; lse_out[r] = M + logf(S); p_out[r] = S > 0.f ? nx / S : 0.f; }
}

__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_gumbel_bwd_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                      const float* __restrict__ points, const int32_t* __restrict__ frame,
                      const float* __restrict__ dist, const float* __restrict__ lse_in,
                      const float* __restrict__ p_in, const float* __restrict__ grad_dist,
                      float* __restrict__ grad_sigma) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const float pred = dist[r];
  const float g = grad_dist[r] * pred;
  if (g == 0.f) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live || !gt_inside(D, s)) return;
  const size_t voff = (size_t)s.f * D.Z * D.Y * D.X;
  const float* vol = sigma + voff;
  float* gvol = grad_sigma + voff;
  const float lse = lse_in[r], p = p_in[r];
  for (int k = 1 + lane; k <= D.num_way; k += 32) {
    const Sample q = make_sample(D, s, k);
    if (q.masked) continue;
    const Corners c = corners(D, q);
    const float dl = g * expf(trilinear(vol, c) - lse) * ((q.length > pred ? 1.f : 0.f) - p);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c.idx[j] >= 0) red_add_f32(gvol + c.idx[j], dl * c.w[j]);
  }
}

// ---- inference decode: zeros -> -inf, first arg-max, its length ---------------------------
__global__ void __launch_bounds__(kRaysPerBlock * 32)
ray_argmax_kernel(RayDims D, const float* __restrict__ sigma, const float* __restrict__ origin,
                  const float* __restrict__ points, const int32_t* __restrict__ frame,
                  float* __restrict__ depth, float* __restrict__ index) {
  const int r = blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= D.R) return;
  const RaySetup s = load_ray(D, origin, points, frame, r);
  if (!s.live) {
    if (lane == 0) {
      depth[r] = 0.f;
      if (index) index[r] = 0.f;
    }
    return;
  }
  const float* vol = sigma + (size_t)s.f * D.Z * D.Y * D.X;
  float best = -INFINITY, best_len = 0.f;
  int best_k = 0x7fffffff;
  for (int k = lane; k < D.num_way; k += 32) {
    const Sample q = make_sample(D, s, k);
    float v = trilinear(vol, corners(D, q));     // no mask here: outside samples are exactly 0
    if (v == 0.f) v = -INFINITY;                  // masked_fill(sigma == 0, -inf)  (:728)
    if (argmax_takes(v, k, best, best_k)) { best = v; best_k = k; best_len = q.length; }
  }
  warp_argmax(best, best_k, best_len);
  if (lane == 0) {
    depth[r] = best_len;
    if (index) index[r] = (float)best_k;
  }
}

int check_dims(RayDims& D, int R, int F, int Z, int Y, int X, int num_way, float step, int with_gt,
               const char* who) {
  VIDAR_REQUIRE(R >= 0 && F > 0 && Z > 0 && Y > 0 && X > 0 && num_way > 0,
                "%s: bad sizes R=%d F=%d grid=%dx%dx%d num_way=%d", who, R, F, Z, Y, X, num_way);
  VIDAR_REQUIRE((long long)Z * Y * X < (1LL << 31), "%s: volume too large", who);
  D = RayDims{R, F, Z, Y, X, num_way, with_gt, step};
  return VIDAR_OK;
}

inline unsigned ray_blocks(int R) { return (unsigned)((R + kRaysPerBlock - 1) / kRaysPerBlock); }

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_ray_sample(const float* sigma, const float* origin, const float* points,
                                const int32_t* frame, float* logits, float* length, float* valid,
                                int R, int F, int Z, int Y, int X, int num_way, float step,
                                int with_gt, void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, with_gt ? 1 : 0, "ray_sample");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points, "ray_sample: null pointer argument");
  ray_sample_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, logits, length, valid);
  return check_launch("ray_sample");
}

extern "C" int vidar_ray_sample_backward(const float* origin, const float* points,
                                         const int32_t* frame, const float* grad_logits,
                                         float* grad_sigma, int R, int F, int Z, int Y, int X,
                                         int num_way, float step, int with_gt, void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, with_gt ? 1 : 0, "ray_sample_backward");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(origin && points && grad_logits && grad_sigma, "ray_sample_backward: null pointer argument");
  ray_sample_bwd_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, origin, points, frame, grad_logits, grad_sigma);
  return check_launch("ray_sample_backward");
}

extern "C" int vidar_ray_ce_forward(const float* sigma, const float* origin, const float* points,
                                    const int32_t* frame, float* ce, float* lse, float* valid,
                                    int R, int F, int Z, int Y, int X, int num_way, float step,
                                    void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, 1, "ray_ce_forward");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points && ce && lse && valid, "ray_ce_forward: null pointer argument");
  ray_ce_fwd_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, ce, lse, valid);
  return check_launch("ray_ce_forward");
}

extern "C" int vidar_ray_ce_backward(const float* sigma, const float* origin, const float* points,
                                     const int32_t* frame, const float* lse, const float* grad_ce,
                                     float* grad_sigma, int R, int F, int Z, int Y, int X,
                                     int num_way, float step, void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, 1, "ray_ce_backward");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points && lse && grad_sigma, "ray_ce_backward: null pointer argument");
  ray_ce_bwd_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, lse, grad_ce, grad_sigma);
  return check_launch("ray_ce_backward");
}

extern "C" int vidar_ray_argmax(const float* sigma, const float* origin, const float* points,
                                const int32_t* frame, float* depth, float* index, int R, int F,
                                int Z, int Y, int X, int num_way, float step, void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, 0, "ray_argmax");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points && depth, "ray_argmax: null pointer argument");
  ray_argmax_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, depth, index);
  return check_launch("ray_argmax");
}

extern "C" int vidar_ray_gumbel_forward(const float* sigma, const float* origin, const float* points,
                                        const int32_t* frame, const float* noise, float* dist, float* lse,
                                        float* p_next, int R, int F, int Z, int Y, int X, int num_way,
                                        float step, void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, 1, "ray_gumbel_forward");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points && noise && dist && lse && p_next, "ray_gumbel_forward: null pointer argument");
  ray_gumbel_fwd_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, noise, dist, lse, p_next);
  return check_launch("ray_gumbel_forward");
}

extern "C" int vidar_ray_gumbel_backward(const float* sigma, const float* origin, const float* points,
                                         const int32_t* frame, const float* dist, const float* lse,
                                         const float* p_next, const float* grad_dist, float* grad_sigma,
                                         int R, int F, int Z, int Y, int X, int num_way, float step,
                                         void* stream) {
  RayDims D;
  int rc = check_dims(D, R, F, Z, Y, X, num_way, step, 1, "ray_gumbel_backward");
  if (rc) return rc;
  if (R == 0) return VIDAR_OK;
  VIDAR_REQUIRE(sigma && origin && points && dist && lse && p_next && grad_dist && grad_sigma,
                "ray_gumbel_backward: null pointer argument");
  ray_gumbel_bwd_kernel<<<ray_blocks(R), kRaysPerBlock * 32, 0, (cudaStream_t)stream>>>(
      D, sigma, origin, points, frame, dist, lse, p_next, grad_dist, grad_sigma);
  return check_launch("ray_gumbel_backward");
}
