// BEV pillar -> camera projection of the BEV encoder (`point_sampling`) for H100 (sm_90a).
//
// Reference: projects/mmdet3d_plugin/bevformer/modules/encoder.py:94-156 -- PyTorch: the
// [D,B,cams,Q,4,4] lidar2img repeat (61 MB at 6 cams x 40000 pillars x 4 anchors), a batched
// matmul, divisions and five mask ops.  Here: one thread per (cam, b, q, d), fp32, no TF32:
//   p = lidar2img[b,cam] @ (x, y, z, 1),  (x,y,z) = ref * (range_max - range_min) + range_min
//   mask = p.z > eps ; uv = p.xy / max(p.z, eps) / (img_w, img_h)
//   mask &= 0 < u < 1 and 0 < v < 1
// Outputs directly in the layout the caller permutes to (:148-149):
//   reference_points_cam [cams, B, Q, D, 2],  bev_mask [cams, B, Q, D] (uint8 0/1).
#include "common.cuh"

namespace vidar {
namespace {

struct PsDims {
  int B, D, Q, cams;
  float r0[3], rs[3];   // range min, range size
  float img_h, img_w;
};

__global__ void __launch_bounds__(256)
point_sampling_kernel(PsDims P, const float* __restrict__ ref3d, const float* __restrict__ l2i,
                      float* __restrict__ ref_cam, unsigned char* __restrict__ mask) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over cams*B*Q*D, D fastest
  const long long total = (long long)P.cams * P.B * P.Q * P.D;
  if (idx >= total) return;
  const int d = (int)(idx % P.D);
  const int q = (int)((idx / P.D) % P.Q);
  const int b = (int)((idx / ((long long)P.D * P.Q)) % P.B);
  const int cam = (int)(idx / ((long long)P.D * P.Q * P.B));
  const float* r = ref3d + (((size_t)b * P.D + d) * P.Q + q) * 3;       // ref_3d [B, D, Q, 3]
  const float x = __fadd_rn(__fmul_rn(r[0], P.rs[0]), P.r0[0]);
  const float y = __fadd_rn(__fmul_rn(r[1], P.rs[1]), P.r0[1]);
  const float z = __fadd_rn(__fmul_rn(r[2], P.rs[2]), P.r0[2]);
  const float* m = l2i + ((size_t)b * P.cams + cam) * 16;
  // row . (x, y, z, 1): one fp32 FMA chain.  The reference's batched matmul sums in another order, so
  // only ~20% of coordinates are bit-identical to it; masks differ only within rounding of a border.
  const float px = fmaf(m[0], x, fmaf(m[1], y, fmaf(m[2], z, m[3])));
  const float py = fmaf(m[4], x, fmaf(m[5], y, fmaf(m[6], z, m[7])));
  const float pz = fmaf(m[8], x, fmaf(m[9], y, fmaf(m[10], z, m[11])));
  const float eps = 1e-5f;
  bool ok = pz > eps;
  const float den = fmaxf(pz, eps);
  const float u = __fdiv_rn(__fdiv_rn(px, den), P.img_w);
  const float v = __fdiv_rn(__fdiv_rn(py, den), P.img_h);
  ok = ok && (v > 0.f) && (v < 1.f) && (u < 1.f) && (u > 0.f);
  reinterpret_cast<float2*>(ref_cam)[idx] = make_float2(u, v);
  mask[idx] = ok ? 1 : 0;
}


// ---- visible-pillar lists of SpatialCrossAttention (spatial_cross_attention.py:136-140), on the device.
// The reference runs `nonzero()` per camera on the host-visible mask and pads to the longest list (a
// host sync per layer).  Here: one block per camera writes the ascending list of visible pillars of
// batch element 0 and its length; consumers launch over the upper bound Q and exit on j >= count.
__global__ void __launch_bounds__(1024)
sca_compact_kernel(const unsigned char* __restrict__ mask, int* __restrict__ idx, int* __restrict__ count,
                   int bs, int Q, int D) {
  const int cam = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ int warp_tot[32];
  __shared__ int base_s;
  if (tid == 0) base_s = 0;
  __syncthreads();
  const unsigned char* m = mask + (size_t)cam * bs * Q * D;       // batch element 0 of this camera
  for (int q0 = 0; q0 < Q; q0 += 1024) {
    const int q = q0 + tid;
    bool hit = false;
    if (q < Q) {
      for (int d = 0; d < D; ++d) hit = hit || (m[(size_t)q * D + d] != 0);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    const int before = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    int woff = 0, total = 0;
    // 32 warp totals: every thread sums the prefix it needs (cheap, no second barrier for a scan)
    for (int w = 0; w < 32; ++w) {
      const int t = warp_tot[w];
      if (w < warp) woff += t;
      total += t;
    }
    const int base = base_s;
    if (hit) idx[(size_t)cam * Q + base + woff + before] = q;
    __syncthreads();
    if (tid == 0) base_s = base + total;
    __syncthreads();
  }
  if (tid == 0) count[cam] = base_s;
}

// 1 / clamp(#cameras whose mask hits pillar (b, q), 1)   (spatial_cross_attention.py:168-171)
__global__ void __launch_bounds__(256)
sca_inv_count_kernel(const unsigned char* __restrict__ mask, float* __restrict__ inv, int cams, int bs, int Q, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;            // over bs * Q
  if (i >= bs * Q) return;
  const int b = i / Q, q = i % Q;
  int n = 0;
  for (int c = 0; c < cams; ++c) {
    const unsigned char* m = mask + (((size_t)c * bs + b) * Q + q) * D;
    bool hit = false;
    for (int d = 0; d < D; ++d) hit = hit || (m[d] != 0);
    n += hit ? 1 : 0;
  }
  inv[i] = __fdiv_rn(1.f, (float)max(n, 1));
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_point_sampling(const float* ref3d, const float* lidar2img, const float* pc_range_host,
                                    float* ref_cam, unsigned char* bev_mask, int B, int D, int Q, int cams,
                                    float img_h, float img_w, void* stream) {
  VIDAR_REQUIRE(ref3d && lidar2img && pc_range_host && ref_cam && bev_mask, "point_sampling: null pointer argument");
  VIDAR_REQUIRE(B > 0 && D > 0 && Q > 0 && cams > 0 && img_h > 0 && img_w > 0, "point_sampling: bad sizes");
  PsDims P;
  P.B = B; P.D = D; P.Q = Q; P.cams = cams;
  for (int i = 0; i < 3; ++i) {
    P.r0[i] = pc_range_host[i];
    P.rs[i] = pc_range_host[i + 3] - pc_range_host[i];
  }
  P.img_h = img_h; P.img_w = img_w;
  const long long total = (long long)cams * B * Q * D;
  const long long nb = (total + 255) / 256;
  VIDAR_REQUIRE(nb < 2147483647LL, "point_sampling: problem too large");
  point_sampling_kernel<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(P, ref3d, lidar2img, ref_cam, bev_mask);
  return check_launch("point_sampling");
}

extern "C" int vidar_sca_compact(const unsigned char* bev_mask, int32_t* idx, int32_t* count, float* inv_count,
                                 int cams, int bs, int Q, int D, void* stream) {
  VIDAR_REQUIRE(bev_mask && idx && count && inv_count, "sca_compact: null pointer argument");
  VIDAR_REQUIRE(cams > 0 && bs > 0 && Q > 0 && D > 0, "sca_compact: bad sizes cams=%d bs=%d Q=%d D=%d", cams, bs, Q, D);
  cudaStream_t st = (cudaStream_t)stream;
  sca_compact_kernel<<<(unsigned)cams, 1024, 0, st>>>(bev_mask, idx, count, bs, Q, D);
  int rc = check_launch("sca_compact");
  if (rc) return rc;
  sca_inv_count_kernel<<<(unsigned)(((long long)bs * Q + 255) / 256), 256, 0, st>>>(bev_mask, inv_count, cams, bs, Q, D);
  return check_launch("sca_compact(inv_count)");
}
