// Multi-scale deformable attention, forward + backward, for H100 (sm_90a).
//
// Replaces mmcv-full 1.4.0 `_ext.ms_deform_attn_{forward,backward}` as called from
// projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:118-124,150-160.
// Semantics (SURVEY.md A.1): pixel = loc * (W,H) - 0.5, bilinear with per-corner zero
// padding, a sample contributes only if -1 < pixel < size; out = sum_{l,p} w * bilerp.
//
// Mapping.  The op is a sparse gather: per (b, q, h) it reads L*P samples x 4 corners x C
// floats (one 128-byte line per corner for C = 32).  One warp owns 32 samples at a time:
//   * lane j decodes sample j once (coordinates, corner offsets, validity) -- the
//     reference re-derives this once per *channel* thread (32x redundant);
//   * the warp is then split into NG = 32/CV groups of CV lanes, a lane holding 4
//     consecutive channels (float4): every corner fetch is a 16-byte vector load and a
//     group of CV lanes covers one head vector, so a warp-level load instruction
//     touches NG lines instead of 1 (4x fewer LSU instructions than lane = channel);
//   * sample parameters travel from the decoding lane to its group by warp shuffle;
//   * backward reduces grad_loc / grad_attn over channels with a 4-value transposed
//     shuffle reduction (no shared memory, no __syncthreads -- the reference does a
//     smem write + 2 barriers + a serial 32-way sum per sample), and scatters
//     grad_value with 16-byte vector reductions (red.global.add.v4.f32).
// Work order: for L*P >= 32 a block is 8 consecutive queries of one (b, h) and
// neighbouring blocks are the other heads of the same queries, so the lines a block
// touches are neighbours in the image (L1/L2 locality).
#include <type_traits>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kWarpsPerBlock = 8;

struct MsdaParams {
  const float* value;
  const int64_t* shapes;
  const int64_t* lsi;
  const float* loc;
  const float* attn;
  int B, K, H, C, L, Q, P, LP;
  int ipw;            // items (b,q,h) per warp (vector kernels)
  int lp_shift;       // log2(LP) when ipw > 1
  int pix_stride;     // H*C floats between neighbouring pixels
  long long items;    // B*Q*H
  // fused sampling-location / softmax epilogue (EPI kernels): `loc` then holds the raw offsets
  // of the sampling_offsets Linear, `attn` the logits of the attention_weights Linear
  const float* ref;   // [B, Q, D, 2] projected Z-anchors (reference_points_cam), normalised
  int D;
  // Row-indirect mode (IDX kernels): a row of batch element n = b*ncl + cl is entry j of camera
  // (cam0 + cl)'s visible-pillar list; results go to / gradients come from the dense BEV slot grid.
  const int* idx;      // [cams, Qd] pillar of row j, or nullptr (row j is pillar j)
  const int* count;    // [cams] live rows per camera, or nullptr (all Q rows are live)
  const float* inv;    // [bs, Qd] output scale 1 / #cameras seeing the pillar, or nullptr
  int ncl, cam0, bs, Qd;   // cameras in this launch, first camera, batch size, pillars per batch element
  int S, s_lo, s_hi;   // the launch covers rows with (j / 64) % S in [s_lo, s_hi)   (rank sub-slices)
  // Queue-mean prologue (SEG kernels: TemporalSelfAttention, the future decoder): an item (b, q, h) holds G segments
  // of 2^seg_shift = L*P samples (LP = G*L*P).  Segment g samples value batch b*G + g, which lies g*Kv pixels past
  // the item's slab (K = G*Kv); `loc` / `attn` hold the raw offsets / logits, `ref` is [B*G, Q, L, 2], and the
  // output is the mean over g: the forward scales the weights, the backward grad_out, by qscale = 1/G.
  int G, seg_shift, Kv;
  float qscale;
};

// Decode one sample: pixel coordinates -> clamped base pixel, corner mask, fractions.
// meta = mask(4b) | dx << 4 | dyW << 5 ; mask == 0 <=> sample contributes nothing.
__device__ __forceinline__ void decode_sample(float lx, float ly, int Hl, int Wl, int start,
                                              int& base, int& meta, float& lh, float& lw,
                                              int scale = 1) {
  // mmcv: h_im = loc_h * spatial_h - 0.5 (no fused multiply-add there either)
  const float h_im = __fsub_rn(__fmul_rn(ly, (float)Hl), 0.5f);
  const float w_im = __fsub_rn(__fmul_rn(lx, (float)Wl), 0.5f);
  base = 0;
  meta = 0;
  lh = 0.f;
  lw = 0.f;
  if (h_im > -1.f && w_im > -1.f && h_im < (float)Hl && w_im < (float)Wl) {
    const float hf = floorf(h_im), wf = floorf(w_im);
    const int h_low = (int)hf, w_low = (int)wf;
    lh = h_im - hf;
    lw = w_im - wf;
    const bool h0 = h_low >= 0, w0 = w_low >= 0;
    const bool h1 = h_low + 1 <= Hl - 1, w1 = w_low + 1 <= Wl - 1;
    const int mask = (int)(h0 && w0) | ((int)(h0 && w1) << 1) | ((int)(h1 && w0) << 2) |
                     ((int)(h1 && w1) << 3);
    const int hl = max(h_low, 0), wl = max(w_low, 0);
    const int hh = min(h_low + 1, Hl - 1), wh = min(w_low + 1, Wl - 1);
    // scale = 1: pixel units (generic kernels); scale = H*C: float offsets (vector kernels)
    base = (start + hl * Wl + wl) * scale;
    meta = mask | ((wh - wl) << 4) | (((hh - hl) * Wl * scale) << 5);
  }
}

// Bilinear corner weights of a decoded sample, pre-multiplied by its attention weight aw.  Invalid corners get
// weight 0; their (clamped) address aliases a valid corner's pixel.
__device__ __forceinline__ void corner_weights(int meta, float lh, float lw, float aw, float& w1, float& w2,
                                               float& w3, float& w4) {
  const float hh = 1.f - lh, hw = 1.f - lw;
  w1 = (meta & 1) ? aw * (hh * hw) : 0.f;
  w2 = (meta & 2) ? aw * (hh * lw) : 0.f;
  w3 = (meta & 4) ? aw * (lh * hw) : 0.f;
  w4 = (meta & 8) ? aw * (lh * lw) : 0.f;
}

// Float offsets of a decoded sample's four corners inside its slab.  decode_sample's base and row step are in units
// of `unit` floats (1 when it scaled them to floats, the pixel stride when it left them in pixels); the column step
// is one pixel stride `pix`.
__device__ __forceinline__ uint4 corner_offsets(int base, int meta, unsigned unit, unsigned pix) {
  const unsigned o1 = (unsigned)base * unit;
  const unsigned o2 = o1 + ((meta & 16) ? pix : 0u);
  const unsigned o3 = o1 + (unsigned)(meta >> 5) * unit;
  return make_uint4(o1, o2, o3, o3 + (o2 - o1));
}

// Cache policy of the gather.  The fine pyramid levels have (almost) no reuse inside an SM -- a
// 24x24-pixel window per anchor and two samples in it -- while one head's coarse levels (15x25: 48 KB,
// 29x50: 186 KB) are re-read by every query: fine-level lines are loaded with L1::no_allocate so they
// do not evict the coarse slabs (kHintBit of a sample's meta word selects the policy).  msda_forward_kernel
// decides where the policy applies.
constexpr int kHintBit = 1 << 30;
// Per-head level slabs (H_l*W_l*C*4 bytes) larger than this stream, so at the SpatialCrossAttention shape everything
// but the 48 KB 15x25 level does (a sweep of the threshold at that shape chose it).
constexpr unsigned kStreamBytes = 100000u;
__device__ __forceinline__ float4 ldg4_na(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float4 ldg4_h(const float* p, bool na) { return na ? ldg4_na(p) : ldg4(p); }

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
// Explicitly rounded fp32 (fmaf / __fmul_rn): the order of operations is fixed, so results do not
// depend on the compiler's contraction choices.
__device__ __forceinline__ void f4_fma(float4& a, float s, const float4& v) {
  a.x = fmaf(s, v.x, a.x);
  a.y = fmaf(s, v.y, a.y);
  a.z = fmaf(s, v.z, a.z);
  a.w = fmaf(s, v.w, a.w);
}
__device__ __forceinline__ float f4_dot(const float4& a, const float4& b) {
  const float lo = fmaf(a.x, b.x, __fmul_rn(a.z, b.z));
  const float hi = fmaf(a.y, b.y, __fmul_rn(a.w, b.w));
  return __fadd_rn(lo, hi);
}
__device__ __forceinline__ float4 f4_scale(float s, const float4& v) {
  return make_float4(__fmul_rn(s, v.x), __fmul_rn(s, v.y), __fmul_rn(s, v.z), __fmul_rn(s, v.w));
}

// Forward: sum of the NG groups' float4 partial head vectors over the warp (every group ends with the total).
template <int CV>
__device__ __forceinline__ float4 group_sum(float4 acc) {
#pragma unroll
  for (int off = CV; off < 32; off <<= 1) {
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
    acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
    acc.w += __shfl_xor_sync(0xffffffffu, acc.w, off);
  }
  return acc;
}

// Backward: (d1..d4) are this lane's channel share of sum_c g*v_k for the four corners of its group's sample.  A
// transposed reduction over the CV lanes of the group takes 4 shuffles; afterwards lane class
// (cl & CV/2, cl & CV/4) = (0,0):d1 (0,1):d2 (1,0):d3 (1,1):d4.  Returns, in every lane, the four sums of the group
// whose first lane is `back`, for the lane that decoded that group's sample to keep.
template <int CV>
__device__ __forceinline__ float4 reduce_corners(float d1, float d2, float d3, float d4, int cl, int back) {
  const bool up1 = (cl & (CV / 2)) != 0;
  const float e0 = __shfl_xor_sync(0xffffffffu, up1 ? d1 : d3, CV / 2);
  const float e1 = __shfl_xor_sync(0xffffffffu, up1 ? d2 : d4, CV / 2);
  const float k0 = (up1 ? d3 : d1) + e0;    // lower half: d1   upper half: d3
  const float k1 = (up1 ? d4 : d2) + e1;    // lower half: d2   upper half: d4
  const bool up2 = (cl & (CV / 4)) != 0;
  const float eb = __shfl_xor_sync(0xffffffffu, up2 ? k0 : k1, CV / 4);
  float k = (up2 ? k1 : k0) + eb;
#pragma unroll
  for (int off = CV / 8; off >= 1; off >>= 1) k += __shfl_xor_sync(0xffffffffu, k, off);
  const float t1 = __shfl_sync(0xffffffffu, k, back);
  const float t2 = __shfl_sync(0xffffffffu, k, back + CV / 4);
  const float t3 = __shfl_sync(0xffffffffu, k, back + CV / 2);
  const float t4 = __shfl_sync(0xffffffffu, k, back + CV / 2 + CV / 4);
  return make_float4(t1, t2, t3, t4);
}

// Backward, in the lane that decoded the sample: its corner sums r (sum_c g*v_k) -> the gradients of its attention
// weight (ga) and of its location (gx, gy).  An out-of-image corner contributes v = 0 to every gradient (mmcv
// col2im_bilinear).
__device__ __forceinline__ void sample_grads(int meta, float lh, float lw, float aw, float fW, float fH,
                                             const float4& r, float& ga, float& gx, float& gy) {
  const float hh = 1.f - lh, hw = 1.f - lw;
  const float r1 = (meta & 1) ? r.x : 0.f, r2 = (meta & 2) ? r.y : 0.f;
  const float r3 = (meta & 4) ? r.z : 0.f, r4 = (meta & 8) ? r.w : 0.f;
  const bool ok = (meta & 15) != 0;
  ga = ok ? (hh * hw) * r1 + (hh * lw) * r2 + (lh * hw) * r3 + (lh * lw) * r4 : 0.f;
  gx = ok ? fW * aw * (hh * (r2 - r1) + lh * (r4 - r3)) : 0.f;
  gy = ok ? fH * aw * (hw * (r3 - r1) + lw * (r4 - r2)) : 0.f;
}


// EPI (MSDeformableAttention3D, spatial_cross_attention.py:339-371 folded into the kernel): lane s
// holds sample s = l*P + p of one (b,q,h); the attention weight is the softmax of the 32 logits
// (`attention_weights.softmax(-1)`, :342) and the location is
//   loc = offsets / (W_l, H_l) + reference_points_cam[b, q, p % D]      (:356-371)
// with the reference's operation order (a true division, then an add; no FMA contraction).
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
__device__ __forceinline__ float2 epi_loc(float2 off, float Wl, float Hl, float2 r) {
  return make_float2(__fadd_rn(__fdiv_rn(off.x, Wl), r.x), __fadd_rn(__fdiv_rn(off.y, Hl), r.y));
}
__device__ __forceinline__ void epi_decode(const MsdaParams& p, size_t refrow, int s, float Wl, float Hl,
                                           const float* loc0, const float* att0, float2& xy, float& aw) {
  const float logit = __ldg(att0 + s);
  const float e = expf(logit - warp_max(logit));
  aw = __fdiv_rn(e, warp_sum(e));
  const float2 off = __ldg(reinterpret_cast<const float2*>(loc0) + s);
  const int z = (s % p.P) % p.D;
  const float2 r = __ldg(reinterpret_cast<const float2*>(p.ref) + refrow + z);   // refrow: anchor 0 of this row
  xy = epi_loc(off, Wl, Hl, r);
}

// SEG (TemporalSelfAttention, temporal_self_attention.py:196-261; the future decoder, vidar_decoder.py:466-506): the
// softmax runs over aligned segments of 2^shift lanes, one (item, queue entry) each.  The butterfly goes from the
// widest offset down, like warp_max / warp_sum and torch's warp softmax.  Every lane of the warp calls it (lanes
// without a sample fill whole segments and pass a dummy logit).
__device__ __forceinline__ float seg_max(float v, int shift) {
  for (int o = (1 << shift) >> 1; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float seg_sum(float v, int shift) {
  for (int o = (1 << shift) >> 1; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float seg_softmax(float logit, int shift) {
  const float e = expf(logit - seg_max(logit, shift));
  return __fdiv_rn(e, seg_sum(e, shift));
}
// Sample sl (< G*L*P) of item (b, q, h), queue entry g = sl / (L*P) at level l: its location offsets / (W_l, H_l) +
// ref[b*G + g, q, l] (epi_loc's order), its level's size and the level's start inside the item's G-batch slab.
// `off` points at the sample's two raw offsets.
__device__ __forceinline__ void seg_decode(const MsdaParams& p, long long item, int sl, const float* off,
                                           float2& xy, int& start, int& Hl, int& Wl) {
  const int g = sl >> p.seg_shift;
  const int l = (sl & ((1 << p.seg_shift) - 1)) / p.P;
  Hl = (int)__ldg(p.shapes + 2 * l);
  Wl = (int)__ldg(p.shapes + 2 * l + 1);
  const unsigned bq = (unsigned)item / (unsigned)p.H;
  const unsigned b = bq / (unsigned)p.Q, q = bq - b * (unsigned)p.Q;
  const size_t refrow = (((size_t)b * p.G + g) * p.Q + q) * p.L + l;
  xy = epi_loc(__ldg(reinterpret_cast<const float2*>(off)), (float)Wl, (float)Hl,
               __ldg(reinterpret_cast<const float2*>(p.ref) + refrow));
  start = (int)__ldg(p.lsi + l) + g * p.Kv;
}

// Which (b,q,h) items does this warp own?  Returns false if none.
//  ipw == 1 : block = 8 consecutive queries of one (b,h); blocks ordered (b, h, qtile).
//  ipw  > 1 : ipw consecutive items in memory order (heads of the same query first).
// All divisions happen here, once per warp -- never inside the sample loop.
__device__ __forceinline__ bool warp_items(const MsdaParams& p, long long& item0) {
  const int warp = threadIdx.x >> 5;
  if (p.ipw == 1) {
    // blocks ordered (b, h, qtile): at any moment the whole chip works on ONE (b, h) slab, so
    // an SM's L1 holds a single head's coarse levels (15x25: 48 KB, 29x50: 186 KB) instead of
    // thrashing between eight.
    const unsigned blk = blockIdx.x;
    const unsigned nqt = (p.Q + kWarpsPerBlock - 1) / kWarpsPerBlock;
    const unsigned qt = blk % nqt;
    const unsigned t = blk / nqt;
    const unsigned h = t % p.H;
    const unsigned b = t / p.H;
    const int q = qt * kWarpsPerBlock + warp;
    if (q >= p.Q) return false;
    item0 = ((long long)b * p.Q + q) * p.H + h;
    return true;
  }
  item0 = ((long long)blockIdx.x * kWarpsPerBlock + warp) * p.ipw;
  return item0 < p.items;
}

// base pointer offset (floats) of item's (b, h) slab inside value / grad_value
__device__ __forceinline__ size_t slab_offset(const MsdaParams& p, long long item64) {
  const unsigned item = (unsigned)item64;            // items < 2^31 on the vector path
  const unsigned qh = (unsigned)p.Q * (unsigned)p.H;
  const unsigned b = item / qh;
  const unsigned h = item % (unsigned)p.H;
  return (size_t)b * p.K * p.pix_stride + (size_t)h * p.C;
}

// Where a row's per-query data lives.  Plain: everything is indexed by the item (rebatched layout).
// IDX: the row is (camera c, list entry j) -> pillar q; `dense` indexes per-(b, pillar, head) arrays
// (BEV slots, and -- in the fused-prologue kernels -- the offsets / logits computed once per pillar).
struct Row {
  long long dense;   // ((b*Qd + q)*H + h)
  size_t refrow;     // float2 index of the row's Z-anchor 0 in p.ref
  float inv;         // output scale
};
// Is list entry j of batch element n one of this launch's rows?  (below its camera's live count, in the launch's
// sub-slice.)  Signed indexing: with unsigned arithmetic here rows_key_kernel<false> spills at its 32 registers.
__device__ __forceinline__ bool row_live(const MsdaParams& p, int n, int j) {
  if (p.count && j >= __ldg(p.count + p.cam0 + n % p.ncl)) return false;
  if (p.S > 1) {
    const int sl = (j >> 6) % p.S;
    if (sl < p.s_lo || sl >= p.s_hi) return false;
  }
  return true;
}
// float2 index of Z-anchor 0 of camera c's row for pillar q of batch element b in reference_points_cam
// [cams, bs, Qd, D, 2]
__device__ __forceinline__ size_t anchor_row(const MsdaParams& p, size_t c, size_t b, size_t q) {
  return ((c * p.bs + b) * p.Qd + q) * p.D;
}
template <bool IDX>
__device__ __forceinline__ bool resolve_row(const MsdaParams& p, long long item0, Row& r) {
  if (!IDX) {
    r.dense = item0;
    r.refrow = (size_t)((unsigned)item0 / (unsigned)p.H) * p.D;      // ref [B, Q, D, 2]
    r.inv = 1.f;
    return true;
  }
  const unsigned item = (unsigned)item0;
  const unsigned h = item % (unsigned)p.H;
  const unsigned nj = item / (unsigned)p.H;
  const unsigned j = nj % (unsigned)p.Q, n = nj / (unsigned)p.Q;
  const unsigned cl = n % (unsigned)p.ncl, b = n / (unsigned)p.ncl;
  const unsigned c = (unsigned)p.cam0 + cl;
  if (!row_live(p, (int)n, (int)j)) return false;
  const unsigned q = p.idx ? (unsigned)__ldg(p.idx + (size_t)c * p.Qd + j) : j;
  const size_t bq = (size_t)b * p.Qd + q;
  r.dense = (long long)(bq * p.H + h);
  r.refrow = anchor_row(p, c, b, q);
  r.inv = p.inv ? __ldg(p.inv + bq) : 1.f;
  return true;
}

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

template <int CV>
__device__ __forceinline__ void store_item(const MsdaParams& p, float* __restrict__ out,
                                           long long item, float4 acc, int g, int cl) {
  acc = group_sum<CV>(acc);
  if (g == 0 && item < p.items)
    *reinterpret_cast<float4*>(out + (size_t)item * p.C + cl * 4) = acc;
}

// MULTI = several items per warp (L*P a power of two < 32, one 32-sample chunk).
// EPI = fused softmax / sampling-location epilogue (L*P == 32, !MULTI only).
// SEG = the queue-mean prologue (G*L*P <= 32 samples per item, MULTI or not): softmax per segment, locations from
// the raw offsets, the G value batches of an item in one slab, the output scaled by 1/G.
// 6 blocks (48 warps) per SM: the register cap (42) is what the tuned round-1 kernel used (40)
template <int CV, bool MULTI, bool EPI = false, bool IDX = false, bool SEG = false>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 6)
msda_forward_kernel(const MsdaParams p, float* __restrict__ out) {
  // The streaming hint (kStreamBytes, ldg4_na) applies to this kernel without IDX and nowhere else.  The backward
  // keeps plain loads: they share the LSU -> XBAR request path with the reductions, and a no-allocate miss cannot
  // merge with a neighbouring warp's pending miss.  The rows forward (IDX) keeps them too: its epilogue also sends
  // 245 MB of slot reductions through L2.
  constexpr bool NA = !IDX;
  constexpr int NG = 32 / CV;       // sample groups per warp
  constexpr int ITERS = 32 / NG;    // == CV
  const int lane = threadIdx.x & 31;
  const int g = lane / CV;          // group = which sample of the current NG
  const int cl = lane % CV;         // which float4 of the head vector
  long long item0;
  if (!warp_items(p, item0)) return;
  Row row;
  if (!resolve_row<IDX>(p, item0, row)) return;

  const int span = MULTI ? 32 : p.LP;                  // samples owned by this warp
  const int nchunks = MULTI ? 1 : (span + 31) >> 5;
  // fused prologue + IDX: offsets / logits exist once per pillar (dense); otherwise per row
  const long long prow = (EPI && IDX) ? row.dense : item0;
  const float* vb = p.value + slab_offset(p, item0) + cl * 4;   // moves with the item (MULTI)
  float* slot = IDX ? out + (size_t)row.dense * p.C + cl * 4 : out;   // IDX: this lane's share of the BEV slot
  const unsigned pix = (unsigned)p.pix_stride;

  float4 acc = f4_zero();
  for (int chunk = 0; chunk < nchunks; ++chunk) {
    // derived per chunk, not kept live through the sample loop (the IDX forwards spill at 40 registers otherwise)
    const float* loc0 = p.loc + (size_t)prow * p.LP * 2;
    const float* att0 = p.attn + (size_t)prow * p.LP;
    // ---- lane j decodes sample j of the chunk; weights are pre-multiplied by attention
    const int s = chunk * 32 + lane;
    int base = 0, meta = 0;
    float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
    const bool live = MULTI ? (item0 + (s >> p.lp_shift) < p.items) : (s < span);
    // SEG: the softmax is a segment-wide reduction, so every lane takes part
    const float sw = SEG ? seg_softmax(live ? __ldg(att0 + s) : 0.f, p.seg_shift) : 0.f;
    if (SEG && live) {
      int Hl, Wl, start;
      float2 xy;
      seg_decode(p, MULTI ? item0 + (s >> p.lp_shift) : item0, MULTI ? (s & (p.LP - 1)) : s, loc0 + 2 * s, xy, start,
                 Hl, Wl);
      float lh, lw;
      decode_sample(xy.x, xy.y, Hl, Wl, start, base, meta, lh, lw, p.pix_stride);
      if (NA && meta && (unsigned)(Hl * Wl) * (unsigned)p.C * 4u > kStreamBytes) meta |= kHintBit;
      // the mean over the queue, folded into the weights (exact when G is a power of two)
      corner_weights(meta, lh, lw, __fmul_rn(sw, p.qscale), w1, w2, w3, w4);
    } else if (!SEG && live) {
      const int sl = MULTI ? (s & (p.LP - 1)) : s;
      const int l = sl / p.P;
      const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
      float2 xy;
      float aw;
      if (EPI) {            // all 32 lanes are live here (L*P == 32)
        epi_decode(p, row.refrow, s, (float)Wl, (float)Hl, loc0, att0, xy, aw);
      } else {
        xy = __ldg(reinterpret_cast<const float2*>(loc0) + s);
        aw = __ldg(att0 + s);
      }
      float lh, lw;
      decode_sample(xy.x, xy.y, Hl, Wl, (int)__ldg(p.lsi + l), base, meta, lh, lw, p.pix_stride);
      if (NA && meta && (unsigned)(Hl * Wl) * (unsigned)p.C * 4u > kStreamBytes) meta |= kHintBit;
      corner_weights(meta, lh, lw, aw, w1, w2, w3, w4);
    }
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
      if (!MULTI && chunk * 32 + it * NG >= span) break;
      const int src = it * NG + g;
      const int sbase = __shfl_sync(0xffffffffu, base, src);
      const int smeta = __shfl_sync(0xffffffffu, meta, src);
      const float a1 = __shfl_sync(0xffffffffu, w1, src);
      const float a2 = __shfl_sync(0xffffffffu, w2, src);
      const float a3 = __shfl_sync(0xffffffffu, w3, src);
      const float a4 = __shfl_sync(0xffffffffu, w4, src);
      if (MULTI && it > 0 && ((it * NG) & (p.LP - 1)) == 0) {
        // item changes every LP/NG iterations: flush the finished one, move the slab pointer
        const int il = (it * NG) >> p.lp_shift;
        store_item<CV>(p, out, item0 + il - 1, acc, g, cl);
        acc = f4_zero();
        vb = p.value + slab_offset(p, item0 + il) + cl * 4;
      }
      const float* vbi = vb;
      asm volatile("" : "+l"(vbi));   // keep the slab base in a 64-bit register pair
      if (smeta & 15) {
        // four independent 16-byte loads, issued back to back (32-bit offsets, 64-bit base)
        const uint4 o = corner_offsets(sbase, smeta & ~kHintBit, 1u, pix);
        const bool na = NA && (smeta & kHintBit) != 0;   // warp-uniform when a level's points fill whole iterations
        const float4 v1 = ldg4_h(vbi + o.x, na);
        const float4 v2 = ldg4_h(vbi + o.y, na);
        const float4 v3 = ldg4_h(vbi + o.z, na);
        const float4 v4 = ldg4_h(vbi + o.w, na);
        f4_fma(acc, a1, v1);
        f4_fma(acc, a2, v2);
        f4_fma(acc, a3, v3);
        f4_fma(acc, a4, v4);
      }
    }
  }
  if (IDX) {
    // SpatialCrossAttention's scatter-add + count normalisation (spatial_cross_attention.py:164-171) as
    // the epilogue: the head vector goes straight into the BEV slot of its pillar.
    acc = group_sum<CV>(acc);
    if (g == 0) red_add_v4(slot, f4_scale(row.inv, acc));
    return;
  }
  store_item<CV>(p, out, MULTI ? item0 + p.ipw - 1 : item0, acc, g, cl);
}

// 4 blocks (32 warps) per SM = 64 registers, the round-1 operating point
template <int CV, bool MULTI, bool EPI = false, bool IDX = false, bool SEG = false>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 4)
msda_backward_kernel(const MsdaParams p, const float* __restrict__ grad_out,
                     float* __restrict__ grad_value, float* __restrict__ grad_loc,
                     float* __restrict__ grad_attn) {
  constexpr int NG = 32 / CV;
  constexpr int ITERS = 32 / NG;
  const int lane = threadIdx.x & 31;
  const int g = lane / CV;
  const int cl = lane % CV;
  long long item0;
  if (!warp_items(p, item0)) return;
  Row row;
  if (!resolve_row<IDX>(p, item0, row)) return;

  const int span = MULTI ? 32 : p.LP;
  const int nchunks = MULTI ? 1 : (span + 31) >> 5;
  const long long prow = (EPI && IDX) ? row.dense : item0;
  const float* loc0 = p.loc + (size_t)prow * p.LP * 2;
  const float* att0 = p.attn + (size_t)prow * p.LP;
  float* gloc0 = grad_loc + (size_t)prow * p.LP * 2;
  float* gatt0 = grad_attn + (size_t)prow * p.LP;
  const unsigned pix = (unsigned)p.pix_stride;
  size_t slab = slab_offset(p, item0) + cl * 4;
  float4 go = f4_zero();
  // IDX: grad_out is the gradient of the BEV slot grid; the row's share is slot[pillar] / count
  if (!MULTI) go = IDX ? f4_scale(row.inv, ldg4(grad_out + (size_t)row.dense * p.C + cl * 4))
                       : ldg4(grad_out + (size_t)item0 * p.C + cl * 4);
  if (SEG && !MULTI) go = f4_scale(p.qscale, go);   // through the mean over the queue

  for (int chunk = 0; chunk < nchunks; ++chunk) {
    const int s = chunk * 32 + lane;
    int base = 0, meta = 0;
    float lh = 0.f, lw = 0.f, aw = 0.f, fH = 0.f, fW = 0.f;
    float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
    const bool live = MULTI ? (item0 + (s >> p.lp_shift) < p.items) : (s < span);
    const float sw = SEG ? seg_softmax(live ? __ldg(att0 + s) : 0.f, p.seg_shift) : 0.f;
    if (live) {
      const int sl = MULTI ? (s & (p.LP - 1)) : s;
      int Hl, Wl, start;
      float2 xy;
      if (SEG) {
        seg_decode(p, MULTI ? item0 + (s >> p.lp_shift) : item0, sl, loc0 + 2 * s, xy, start, Hl, Wl);
        aw = sw;
      } else {
        const int l = sl / p.P;
        Hl = (int)__ldg(p.shapes + 2 * l);
        Wl = (int)__ldg(p.shapes + 2 * l + 1);
        if (EPI) {
          epi_decode(p, row.refrow, s, (float)Wl, (float)Hl, loc0, att0, xy, aw);
        } else {
          xy = __ldg(reinterpret_cast<const float2*>(loc0) + s);
          aw = __ldg(att0 + s);
        }
        start = (int)__ldg(p.lsi + l);
      }
      decode_sample(xy.x, xy.y, Hl, Wl, start, base, meta, lh, lw, p.pix_stride);
      fH = (float)Hl;
      fW = (float)Wl;
      corner_weights(meta, lh, lw, aw, w1, w2, w3, w4);
    }
    float4 r = f4_zero();   // this lane's sample: sum_c g*v_k
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
      if (!MULTI && chunk * 32 + it * NG >= span) break;
      const int src = it * NG + g;
      const int sbase = __shfl_sync(0xffffffffu, base, src);
      const int smeta = __shfl_sync(0xffffffffu, meta, src);
      const float a1 = __shfl_sync(0xffffffffu, w1, src);
      const float a2 = __shfl_sync(0xffffffffu, w2, src);
      const float a3 = __shfl_sync(0xffffffffu, w3, src);
      const float a4 = __shfl_sync(0xffffffffu, w4, src);
      if (MULTI && ((it * NG) & (p.LP - 1)) == 0) {
        const long long item = item0 + ((it * NG) >> p.lp_shift);
        if (item < p.items) {
          slab = slab_offset(p, item) + cl * 4;
          go = ldg4(grad_out + (size_t)item * p.C + cl * 4);
          if (SEG) go = f4_scale(p.qscale, go);
        } else {
          go = f4_zero();
        }
      }
      float d1 = 0.f, d2 = 0.f, d3 = 0.f, d4 = 0.f;
      if (smeta & 15) {
        const uint4 o = corner_offsets(sbase, smeta, 1u, pix);
        const float* vs = p.value + slab;
        float* gs = grad_value + slab;
        asm volatile("" : "+l"(vs), "+l"(gs));
        const float4 v1 = ldg4(vs + o.x);
        const float4 v2 = ldg4(vs + o.y);
        const float4 v3 = ldg4(vs + o.z);
        const float4 v4 = ldg4(vs + o.w);
        // grad_value: top_grad * attn * corner weight as 16-byte vector reductions.  An
        // out-of-image corner has weight 0 and aliases a valid pixel: its reduction adds 0.
        red_add_v4(gs + o.x, f4_scale(a1, go));
        red_add_v4(gs + o.y, f4_scale(a2, go));
        red_add_v4(gs + o.z, f4_scale(a3, go));
        red_add_v4(gs + o.w, f4_scale(a4, go));
        d1 = f4_dot(go, v1); d2 = f4_dot(go, v2); d3 = f4_dot(go, v3); d4 = f4_dot(go, v4);
      }
      // ---- reduce over the group, hand the four sums back to the lane that decoded the sample (lane it*NG + g')
      const float4 t = reduce_corners<CV>(d1, d2, d3, d4, cl, (lane & (NG - 1)) * CV);
      if ((lane / NG) == it) r = t;
    }
    // ---- every lane finishes its own sample; coalesced stores
    if (SEG) {
      // grad_off = grad_loc / (W,H); grad_logit = w * (grad_w - sum_j w_j grad_w_j) over the sample's segment, a
      // reduction every lane takes part in (without a sample: meta = 0 and aw = 0, so ga = 0)
      float ga, gx, gy;
      sample_grads(meta, lh, lw, aw, fW, fH, r, ga, gx, gy);
      const float dot = seg_sum(aw * ga, p.seg_shift);
      if (live) {
        gatt0[s] = aw * (ga - dot);
        reinterpret_cast<float2*>(gloc0)[s] = make_float2(__fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
      }
    } else if (live) {
      float ga, gx, gy;
      sample_grads(meta, lh, lw, aw, fW, fH, r, ga, gx, gy);
      if (EPI) {
        // through loc = off / (W,H) + ref and w = softmax(logits): grad_off = grad_loc / (W,H),
        // grad_logit = w * (grad_w - sum_j w_j grad_w_j)   (all 32 lanes take part in the sum)
        const float dot = warp_sum(aw * ga);
        if (IDX) {
          // offsets / logits are shared by every camera that sees the pillar: accumulate (caller zeroes)
          red_add_f32(gatt0 + s, aw * (ga - dot));
          red_add_v2(gloc0 + 2 * s, __fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
        } else {
          gatt0[s] = aw * (ga - dot);
          reinterpret_cast<float2*>(gloc0)[s] = make_float2(__fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
        }
      } else {
        gatt0[s] = ga;
        reinterpret_cast<float2*>(gloc0)[s] = make_float2(gx, gy);
      }
    }
  }
}

// ---- small L*P (temporal self-attention, future decoder: L*P = 4 or 8) -------------------
// When a 32-sample chunk holds at least NG whole items, give each group of CV lanes its OWN
// item: the group walks that item's L*P samples and finishes the head vector by itself, so the
// cross-group shuffle reduction + flush of the generic MULTI path (8 shuffles per item, i.e.
// 2 shuffles per sample at L*P = 4) disappears and every group stores 128 contiguous bytes.
template <int CV>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
msda_forward_small_kernel(const MsdaParams p, float* __restrict__ out) {
  constexpr int NG = 32 / CV;
  const int lane = threadIdx.x & 31;
  const int g = lane / CV, cl = lane % CV;
  long long item0;
  if (!warp_items(p, item0)) return;
  const float* loc0 = p.loc + (size_t)item0 * p.LP * 2;
  const float* att0 = p.attn + (size_t)item0 * p.LP;
  const unsigned pix = (unsigned)p.pix_stride;
  // lane j decodes sample j of the chunk (32 samples = ipw items)
  int base = 0, meta = 0;
  float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
  if (item0 + (lane >> p.lp_shift) < p.items) {
    const float2 xy = __ldg(reinterpret_cast<const float2*>(loc0) + lane);
    const float aw = __ldg(att0 + lane);
    const int l = (lane & (p.LP - 1)) / p.P;
    const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
    float lh, lw;
    decode_sample(xy.x, xy.y, Hl, Wl, (int)__ldg(p.lsi + l), base, meta, lh, lw, p.pix_stride);
    corner_weights(meta, lh, lw, aw, w1, w2, w3, w4);
  }
  const int rounds = p.ipw / NG;
  for (int r = 0; r < rounds; ++r) {
    const int il = r * NG + g;                       // this group's item in the chunk
    const long long item = item0 + il;
    const bool live = item < p.items;
    const float* vb = p.value + (live ? slab_offset(p, item) : 0) + cl * 4;
    asm volatile("" : "+l"(vb));
    float4 acc = f4_zero();
    for (int sidx = 0; sidx < p.LP; ++sidx) {
      const int src = (il << p.lp_shift) + sidx;
      const int sbase = __shfl_sync(0xffffffffu, base, src);
      const int smeta = __shfl_sync(0xffffffffu, meta, src);
      const float a1 = __shfl_sync(0xffffffffu, w1, src);
      const float a2 = __shfl_sync(0xffffffffu, w2, src);
      const float a3 = __shfl_sync(0xffffffffu, w3, src);
      const float a4 = __shfl_sync(0xffffffffu, w4, src);
      if (smeta & 15) {
        const uint4 o = corner_offsets(sbase, smeta, 1u, pix);
        const float4 v1 = ldg4(vb + o.x);
        const float4 v2 = ldg4(vb + o.y);
        const float4 v3 = ldg4(vb + o.z);
        const float4 v4 = ldg4(vb + o.w);
        f4_fma(acc, a1, v1);
        f4_fma(acc, a2, v2);
        f4_fma(acc, a3, v3);
        f4_fma(acc, a4, v4);
      }
    }
    if (live) *reinterpret_cast<float4*>(out + (size_t)item * p.C + cl * 4) = acc;
  }
}

template <int CV>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
msda_backward_small_kernel(const MsdaParams p, const float* __restrict__ grad_out,
                           float* __restrict__ grad_value, float* __restrict__ grad_loc,
                           float* __restrict__ grad_attn) {
  constexpr int NG = 32 / CV;
  const int lane = threadIdx.x & 31;
  const int g = lane / CV, cl = lane % CV;
  long long item0;
  if (!warp_items(p, item0)) return;
  const float* loc0 = p.loc + (size_t)item0 * p.LP * 2;
  const float* att0 = p.attn + (size_t)item0 * p.LP;
  const unsigned pix = (unsigned)p.pix_stride;
  int base = 0, meta = 0;
  float lh = 0.f, lw = 0.f, aw = 0.f, fH = 0.f, fW = 0.f;
  float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
  const bool mine = item0 + (lane >> p.lp_shift) < p.items;
  if (mine) {
    const float2 xy = __ldg(reinterpret_cast<const float2*>(loc0) + lane);
    aw = __ldg(att0 + lane);
    const int l = (lane & (p.LP - 1)) / p.P;
    const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
    decode_sample(xy.x, xy.y, Hl, Wl, (int)__ldg(p.lsi + l), base, meta, lh, lw, p.pix_stride);
    fH = (float)Hl;
    fW = (float)Wl;
    corner_weights(meta, lh, lw, aw, w1, w2, w3, w4);
  }
  float r1 = 0.f, r2 = 0.f, r3 = 0.f, r4 = 0.f;
  const int rounds = p.ipw / NG;
  const int my_il = lane >> p.lp_shift;              // item (in the chunk) of the sample this lane decoded
  for (int r = 0; r < rounds; ++r) {
    const int il = r * NG + g;
    const long long item = item0 + il;
    const bool live = item < p.items;
    const size_t slab = (live ? slab_offset(p, item) : 0) + cl * 4;
    const float4 go = live ? ldg4(grad_out + (size_t)item * p.C + cl * 4) : f4_zero();
    const float* vs = p.value + slab;
    float* gs = grad_value + slab;
    asm volatile("" : "+l"(vs), "+l"(gs));
    for (int sidx = 0; sidx < p.LP; ++sidx) {
      const int src = (il << p.lp_shift) + sidx;
      const int sbase = __shfl_sync(0xffffffffu, base, src);
      const int smeta = __shfl_sync(0xffffffffu, meta, src);
      const float a1 = __shfl_sync(0xffffffffu, w1, src);
      const float a2 = __shfl_sync(0xffffffffu, w2, src);
      const float a3 = __shfl_sync(0xffffffffu, w3, src);
      const float a4 = __shfl_sync(0xffffffffu, w4, src);
      float d1 = 0.f, d2 = 0.f, d3 = 0.f, d4 = 0.f;
      if (smeta & 15) {
        const uint4 o = corner_offsets(sbase, smeta, 1u, pix);
        const float4 v1 = ldg4(vs + o.x);
        const float4 v2 = ldg4(vs + o.y);
        const float4 v3 = ldg4(vs + o.z);
        const float4 v4 = ldg4(vs + o.w);
        red_add_v4(gs + o.x, f4_scale(a1, go));
        red_add_v4(gs + o.y, f4_scale(a2, go));
        red_add_v4(gs + o.z, f4_scale(a3, go));
        red_add_v4(gs + o.w, f4_scale(a4, go));
        d1 = f4_dot(go, v1); d2 = f4_dot(go, v2); d3 = f4_dot(go, v3); d4 = f4_dot(go, v4);
      }
      // reduce_corners written out: through the helper, nvcc contracts the first product of sample_grads' ga sum
      // on the other side in this kernel, which changes grad_attn in the last bits
      const bool up1 = (cl & (CV / 2)) != 0;
      const float e0 = __shfl_xor_sync(0xffffffffu, up1 ? d1 : d3, CV / 2);
      const float e1 = __shfl_xor_sync(0xffffffffu, up1 ? d2 : d4, CV / 2);
      const float k0 = (up1 ? d3 : d1) + e0;
      const float k1 = (up1 ? d4 : d2) + e1;
      const bool up2 = (cl & (CV / 4)) != 0;
      const float eb = __shfl_xor_sync(0xffffffffu, up2 ? k0 : k1, CV / 4);
      float k = (up2 ? k1 : k0) + eb;
#pragma unroll
      for (int off = CV / 8; off >= 1; off >>= 1) k += __shfl_xor_sync(0xffffffffu, k, off);
      // hand back to the decoding lane: its sample is processed by group (my_il % NG) in round my_il / NG
      const int back = (my_il & (NG - 1)) * CV;
      const float t1 = __shfl_sync(0xffffffffu, k, back);
      const float t2 = __shfl_sync(0xffffffffu, k, back + CV / 4);
      const float t3 = __shfl_sync(0xffffffffu, k, back + CV / 2);
      const float t4 = __shfl_sync(0xffffffffu, k, back + CV / 2 + CV / 4);
      if ((my_il / NG) == r && (lane & (p.LP - 1)) == sidx) { r1 = t1; r2 = t2; r3 = t3; r4 = t4; }
    }
  }
  if (mine) {
    float ga, gx, gy;
    sample_grads(meta, lh, lw, aw, fW, fH, make_float4(r1, r2, r3, r4), ga, gx, gy);
    grad_attn[(size_t)item0 * p.LP + lane] = ga;
    reinterpret_cast<float2*>(grad_loc)[(size_t)item0 * p.LP + lane] = make_float2(gx, gy);
  }
}

// ---- row-indirect backward at SpatialCrossAttention's shape (C = 32, L*P = 32, P = 8): tile aggregation --------
// The per-corner grad_value reductions of msda_backward_kernel (4 x 128-byte lines per sample) saturate the
// SM -> L2 request path.  Rows close together in the *image* hit the same pixels, so the rows of each batch element
// are first put in image order (a stable counting sort by a 16 x 16 cell of the row's mean sampling location), and
// one CTA then owns a tile of kTileRows ordered rows of one head.  Per pyramid level it gathers and computes the
// sampling-location / attention gradients as msda_backward_kernel does (same arithmetic), writes one record per
// pair of horizontally adjacent corners (left pixel, two weights, row) to shared memory, sorts the records by pixel
// and sums the runs with lane = channel, so a (pixel, head) line is reduced about once per tile instead of once per
// corner.
constexpr int kTileRows = 256;                               // rows per tile
constexpr int kTilePoints = 8;                               // points per level (P)
constexpr int kTileRecs = kTileRows * kTilePoints * 2;       // corner-pair records per level (top, bottom)
constexpr int kRecBits = 12;                                 // record index bits: log2(kTileRecs)
constexpr int kTileThreads = 512;                            // 16 warps, 16 rows each
constexpr int kTileItems = kTileRecs / kTileThreads;         // records per thread in the sort
constexpr int kTileSeg = kTileRecs / (kTileThreads / 8);     // sorted records summed by one 8-lane group
constexpr int kCells = 256;                                  // 16 x 16 image cells of the row order
constexpr int kOrderChunk = 1024;                            // rows per block of the row-order kernels
static_assert(kTileRecs == 1 << kRecBits, "record index width");

// floor(n / d) for n < 2^22 from rd = 1 / d rounded to fp32: n + 0.5 is exact, its quotient lies at least 0.5 / d from
// an integer, and the two fp32 roundings move it by less than (n + 0.5) / d * 2^-23 < 0.5 / d.
__device__ __forceinline__ unsigned div_small(unsigned n, float rd) {
  return (unsigned)__fmul_rn(__fadd_rn(__uint2float_rn(n), 0.5f), rd);
}

// Row order, pass 1: each live row's image cell (-1 = not a row of this launch) and the cell histogram of every
// chunk of kOrderChunk rows.  The cell is taken from the mean of head 0's sampling locations, or with the fused
// epilogue (EPI) from the mean of the pillar's reference_points_cam Z-anchors.
template <bool EPI>
__global__ void __launch_bounds__(kOrderChunk)
rows_key_kernel(const MsdaParams p, int* __restrict__ key, int* __restrict__ hist) {
  __shared__ int cnt[kCells];
  const int n = blockIdx.y, j = blockIdx.x * kOrderChunk + threadIdx.x;
  if (threadIdx.x < kCells) cnt[threadIdx.x] = 0;
  __syncthreads();
  if (j < p.Q) {
    int k = -1;
    if (row_live(p, n, j)) {
      const int c = p.cam0 + n % p.ncl, b = n / p.ncl;
      float sx = 0.f, sy = 0.f, s;
      if (EPI) {
        const size_t q = p.idx ? (size_t)__ldg(p.idx + (size_t)c * p.Qd + j) : (size_t)j;
        const float2* r = reinterpret_cast<const float2*>(p.ref) + anchor_row(p, c, b, q);
        for (int i = 0; i < p.D; ++i) {
          const float2 v = __ldg(r + i);
          sx += v.x;
          sy += v.y;
        }
        s = 16.f / (float)p.D;
      } else {
        const float4* l = reinterpret_cast<const float4*>(p.loc + ((size_t)n * p.Q + j) * p.H * p.LP * 2);
        for (int i = 0; i < p.LP / 2; ++i) {
          const float4 v = __ldg(l + i);
          sx += v.x + v.z;
          sy += v.y + v.w;
        }
        s = 16.f / (float)p.LP;
      }
      k = min(max((int)(sy * s), 0), 15) * 16 + min(max((int)(sx * s), 0), 15);
      atomicAdd(&cnt[k], 1);
    }
    key[(size_t)n * p.Q + j] = k;
  }
  __syncthreads();
  if (threadIdx.x < kCells) hist[((size_t)n * gridDim.x + blockIdx.x) * kCells + threadIdx.x] = cnt[threadIdx.x];
}

// pass 2, one block per batch element: hist becomes the first ordered position of each (chunk, cell), cell-major
__global__ void __launch_bounds__(kCells)
rows_scan_kernel(int* __restrict__ hist, int* __restrict__ nlive, int nch) {
  using Scan = cub::BlockScan<int, kCells>;
  __shared__ typename Scan::TempStorage tmp;
  int* h = hist + (size_t)blockIdx.x * nch * kCells + threadIdx.x;
  int run = 0;
  for (int ch = 0; ch < nch; ++ch) {
    const int v = h[(size_t)ch * kCells];
    h[(size_t)ch * kCells] = run;
    run += v;
  }
  int base, total;
  Scan(tmp).ExclusiveSum(run, base, total);
  for (int ch = 0; ch < nch; ++ch) h[(size_t)ch * kCells] += base;
  if (threadIdx.x == 0) nlive[blockIdx.x] = total;
}

// pass 3: perm[n][position] = j, stable (rows of a cell keep their list order)
__global__ void __launch_bounds__(kOrderChunk)
rows_scatter_kernel(const int* __restrict__ key, const int* __restrict__ hist, int* __restrict__ perm, int Q) {
  constexpr int W = kOrderChunk / 32;
  __shared__ int wc[W][kCells];   // rows of each cell in each warp, then their exclusive prefix over warps
  const int n = blockIdx.y, j = blockIdx.x * kOrderChunk + threadIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < W * kCells; i += kOrderChunk) (&wc[0][0])[i] = 0;
  __syncthreads();
  const int k = j < Q ? key[(size_t)n * Q + j] : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, k);
  const int rank = __popc(peers & ((1u << lane) - 1u));
  if (k >= 0 && rank == 0) wc[warp][k] = __popc(peers);
  __syncthreads();
  if (threadIdx.x < kCells) {
    int run = 0;
    for (int w = 0; w < W; ++w) {
      const int v = wc[w][threadIdx.x];
      wc[w][threadIdx.x] = run;
      run += v;
    }
  }
  __syncthreads();
  if (k >= 0) perm[(size_t)n * Q + hist[((size_t)n * gridDim.x + blockIdx.x) * kCells + k] + wc[warp][k] + rank] = j;
}

using TileSort = cub::BlockRadixSort<unsigned, kTileThreads, kTileItems, cub::NullType, 5, false>;
// The records and the sort's temp storage are static shared memory: their addresses are then constants rather than
// registers (the kernel runs at the 64-register limit of 2 x 512 threads per SM).
union __align__(16) TileKeys {
  unsigned key[kTileRecs + kTileRecs / kTileSeg];   // records; once sorted, one pad word per group segment
  typename TileSort::TempStorage sort;
};
struct TileSmem {                        // dynamic shared memory
  float w[2 * kTileRecs];                // attn * bilinear weight of record r's left (w[2r]) and right (w[2r+1]) corner
  float4 go[kTileRows * 8];              // row's grad_out head vector, scaled by 1 / #cameras
  int item[kTileRows];                   // row's item index (EPI: its pillar's (b, q, h) index), -1 past the last row
  size_t slab;                           // float offset of the (n, h) slab in value / grad_value
};
// EPI only, after TileSmem: the row's softmax statistics and its 32 attention gradients, which the logit gradient
// needs together after the last level.  137 KB in all: one CTA per SM.
struct TileSmemEpi {
  float ga[kTileRows * 32];
  float2 stat[kTileRows];                // max and sum of exp(logit - max) over the row's 32 logits
  int refrow[kTileRows];                 // float2 index of the row's Z-anchor 0 in reference_points_cam
};
template <bool EPI>
constexpr size_t tile_smem_bytes() { return sizeof(TileSmem) + (EPI ? sizeof(TileSmemEpi) : 0); }

// grid: (batch element n, head h, tile) with the tile fastest; perm / nlive from the row-order kernels.
// EPI: MSDeformableAttention3D's softmax and sampling-location prologue as in epi_decode, offset / logit gradients
// accumulated into the per-pillar rows as in msda_backward_kernel<.., EPI, IDX>.
template <bool EPI>
__global__ void __launch_bounds__(kTileThreads, EPI ? 1 : 2)
msda_backward_tile_kernel(const MsdaParams p, const int* __restrict__ perm, const int* __restrict__ nlive,
                          const float* __restrict__ grad_out, float* __restrict__ grad_value,
                          float* __restrict__ grad_loc, float* __restrict__ grad_attn) {
  constexpr int CV = 8, NG = 4, P = kTilePoints, NT = kTileThreads, RW = kTileRows / (NT / 32);   // RW rows per warp
  // 128-byte aligned: keeps the dynamic region at the offset this kernel was tuned and measured with
  extern __shared__ __align__(128) unsigned char tile_smem[];
  TileSmem& sm = *reinterpret_cast<TileSmem*>(tile_smem);
  TileSmemEpi& se = *reinterpret_cast<TileSmemEpi*>(tile_smem + sizeof(TileSmem));
  __shared__ TileKeys tk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane / CV, cl = lane % CV;
  const int ntiles = (p.Q + kTileRows - 1) / kTileRows;
  const int t = blockIdx.x % ntiles, nh = blockIdx.x / ntiles;
  const int h = nh % p.H, n = nh / p.H;
  const int nrows = min(kTileRows, __ldg(nlive + n) - t * kTileRows);
  if (nrows <= 0) return;
  const int b = n / p.ncl, c = p.cam0 + n % p.ncl;

  // this warp's RW rows of the tile (4 per step, 8 lanes x float4 per head vector)
  for (int i = 0; i < RW; i += 4) {
    const int r = warp * RW + i + g;
    float4 go = f4_zero();
    int j = 0;
    size_t q = 0, bq = 0;
    if (r < nrows) {
      j = __ldg(perm + (size_t)n * p.Q + t * kTileRows + r);
      q = p.idx ? (size_t)__ldg(p.idx + (size_t)c * p.Qd + j) : (size_t)j;
      bq = (size_t)b * p.Qd + q;
      go = f4_scale(p.inv ? __ldg(p.inv + bq) : 1.f, ldg4(grad_out + (bq * p.H + h) * p.C + cl * 4));
    }
    if (cl == 0) {
      sm.item[r] = r < nrows ? (int)(EPI ? bq * p.H + h : ((size_t)n * p.Q + j) * p.H + h) : -1;
      if (EPI) se.refrow[r] = (int)anchor_row(p, c, b, q);
    }
    sm.go[r * 8 + cl] = go;
  }
  if (threadIdx.x == 0) sm.slab = (size_t)n * p.K * p.pix_stride + (size_t)h * p.C;
  __syncwarp();
  if (EPI) {
    // softmax statistics of each row, lane = sample (the warp_max / warp_sum of epi_decode, so the weights are
    // bit-identical); rows past the last are at the warp's end
    for (int i = 0; i < RW; ++i) {
      const int item = sm.item[warp * RW + i];
      if (item < 0) break;
      const float logit = __ldg(p.attn + (size_t)item * p.LP + lane);
      const float m = warp_max(logit);
      const float sum = warp_sum(expf(logit - m));
      if (lane == 0) se.stat[warp * RW + i] = make_float2(m, sum);
    }
  }
  // the level loop reads the row items and the slab offset from shared memory: n, h and nrows need no registers there
  __syncthreads();

  const unsigned pix = (unsigned)p.pix_stride;
  for (int l = 0; l < p.L; ++l) {
    const size_t slab = sm.slab + cl * 4;
    const float* vs = p.value + slab;
    const int Hl = (int)__ldg(p.shapes + 2 * l), Wl = (int)__ldg(p.shapes + 2 * l + 1);
    const int start = (int)__ldg(p.lsi + l);
    const float fH = (float)Hl, fW = (float)Wl;
    // A record's pixel is a slot h * (Wl + 1) + x' of the level's rows padded by one column in front: x' = w + 1, and
    // x' = 0 holds only invalid corners.  Slots are below Hl * (Wl + 1) < 2 * K < 2^20, so the key fits 32 bits.
    const int pb = 32 - __clz(Hl * (Wl + 1));       // pixel bits of the level's sort key
    const unsigned none = (1u << pb) - 1;           // pixel field of an unused record: sorts last
    // ---- row phase: a chunk is 4 rows x this level's 8 points, lane j decodes point j % 8 of row j / 8
#pragma unroll 1
    for (int ck = 0; ck < RW / 4; ++ck) {
      const int r = warp * RW + ck * 4 + (lane >> 3);
      const int item = sm.item[r];
      const bool live = item >= 0;
      size_t si = 0;   // sample index (row's item * L*P + l*P + point)
      int base = 0, meta = 0;
      float lh = 0.f, lw = 0.f, aw = 0.f;
      float w1 = 0.f, w2 = 0.f, w3 = 0.f, w4 = 0.f;
      if (live) {
        si = (size_t)item * p.LP + l * P + (lane & 7);
        float2 xy = __ldg(reinterpret_cast<const float2*>(p.loc) + si);
        if (EPI) {
          // epi_decode: w = softmax(logits), loc = offsets / (W, H) + reference_points_cam[p % D]
          const float2 st = se.stat[r];
          aw = __fdiv_rn(expf(__ldg(p.attn + si) - st.x), st.y);
          const float2 rf = __ldg(reinterpret_cast<const float2*>(p.ref) + se.refrow[r] + (lane & 7) % p.D);
          xy = epi_loc(xy, fW, fH, rf);
        } else {
          aw = __ldg(p.attn + si);
        }
        decode_sample(xy.x, xy.y, Hl, Wl, start, base, meta, lh, lw);   // base, dy in pixels
        corner_weights(meta, lh, lw, aw, w1, w2, w3, w4);
      }
      float4 rs = f4_zero();
#pragma unroll
      for (int it = 0; it < CV; ++it) {
        const int src = it * NG + g;
        const int sbase = __shfl_sync(0xffffffffu, base, src);
        const int smeta = __shfl_sync(0xffffffffu, meta, src);
        const float4 go = sm.go[(warp * RW + ck * 4 + (it >> 1)) * 8 + cl];   // row of sample src
        float d1 = 0.f, d2 = 0.f, d3 = 0.f, d4 = 0.f;
        if (smeta & 15) {
          const uint4 o = corner_offsets(sbase, smeta, pix, pix);
          d1 = f4_dot(go, ldg4(vs + o.x));
          d2 = f4_dot(go, ldg4(vs + o.y));
          d3 = f4_dot(go, ldg4(vs + o.z));
          d4 = f4_dot(go, ldg4(vs + o.w));
        }
        // reduction and hand-back, as in msda_backward_kernel
        const float4 t = reduce_corners<CV>(d1, d2, d3, d4, cl, (lane & (NG - 1)) * CV);
        if ((lane / NG) == it) rs = t;
      }
      // this sample's 2 corner-pair records: record = (row in tile, point, half), half 0 = corners (1, 2) in row
      // h_low, 1 = corners (3, 4) in row h_low + 1; key = slot of the pair's left pixel (w_low) << kRecBits | record,
      // or `none` if neither corner is valid.  The clamped base is (max(h_low, 0), max(w_low, 0)); the mask tells
      // h_low = -1 (no corner in the top row) and w_low = -1 (no left corner, slot x' = 0).
      const unsigned rec = ((unsigned)(warp * RW + ck * 4) << 4) + lane * 2;
      const unsigned px = (unsigned)(base - start), hl = div_small(px, __frcp_rn(fW));
      const unsigned left = px + hl + ((meta & 5) ? 1u : 0u);
      uint2 kk;
      kk.x = (((meta & 3) ? left : none) << kRecBits) | rec;
      kk.y = (((meta & 12) ? left + ((meta & 3) ? (unsigned)Wl + 1u : 0u) : none) << kRecBits) | (rec + 1);
      *reinterpret_cast<uint2*>(&tk.key[rec]) = kk;
      *reinterpret_cast<float4*>(&sm.w[2 * rec]) = make_float4(w1, w2, w3, w4);
      if (live) {
        float ga, gx, gy;
        sample_grads(meta, lh, lw, aw, fW, fH, rs, ga, gx, gy);
        if (EPI) {
          // offsets are shared by every camera that sees the pillar: accumulate (caller zeroes); the logit
          // gradient waits for the row's other levels
          se.ga[r * 32 + l * P + (lane & 7)] = ga;
          red_add_v2(grad_loc + 2 * si, __fdiv_rn(gx, fW), __fdiv_rn(gy, fH));
        } else {
          grad_attn[si] = ga;
          reinterpret_cast<float2*>(grad_loc)[si] = make_float2(gx, gy);
        }
      }
    }
    __syncthreads();

    // ---- tile phase: sort the level's records by pixel (stable, so the summation order is fixed)
    unsigned keys[kTileItems];
#pragma unroll
    for (int i = 0; i < kTileItems; ++i) keys[i] = tk.key[i * NT + threadIdx.x];
    __syncthreads();   // the sort's temp storage aliases key[]
    TileSort(tk.sort).SortBlockedToStriped(keys, kRecBits, kRecBits + pb);
    __syncthreads();
    // sorted position R = i*NT + tid is stored at R + R / kTileSeg (the pad keeps the 4 groups of a warp on
    // different banks)
#pragma unroll
    for (int i = 0; i < kTileItems; ++i) {
      const int R = i * NT + threadIdx.x;
      tk.key[R + R / kTileSeg] = keys[i];
    }
    __syncthreads();

    // group G (8 lanes x float4 = one head vector) sums the records at sorted positions [G*kTileSeg, (G+1)*kTileSeg).
    // Slot s receives the left corners of pairs keyed s and the right corners of pairs keyed s - 1, which sort next
    // to each other: the group keeps accumulators for slots cur and cur + 1 and sends one 128-byte reduction per
    // touched pixel (a pixel whose records straddle two groups is reduced twice)
    float* gl = grad_value + slab + (size_t)start * pix;
    asm volatile("" : "+l"(gl));   // computed here, not kept live through the sort (64-register budget)
    const unsigned* ks = tk.key + (warp * NG + g) * (kTileSeg + 1);
    const unsigned W1 = (unsigned)Wl + 1u;
    const float rW1 = __frcp_rn(fW + 1.f);
    // slot s = h * W1 + x' is pixel h * Wl + x' - 1; slot x' = 0 only ever holds invalid corners (weight 0, and
    // perhaps an address outside the level) and is never reduced
    const auto flush = [&](unsigned s, const float4& a) {
      const unsigned hs = div_small(s, rW1);
      if (s != hs * W1) red_add_v4(gl + (s - hs - 1u) * pix, a);
    };
    // records are read 4 at a time so that their shared-memory loads overlap; unused records (pixel `none`, weight 0)
    // sort last and accumulate into slots that are never reduced
    unsigned cur = none;
    float4 a0 = f4_zero(), a1 = f4_zero();   // slots cur, cur + 1
    for (int i0 = 0; i0 < kTileSeg; i0 += 4) {
      unsigned kq[4];
      float2 wq[4];
      float4 gq[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) kq[u] = ks[i0 + u];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const unsigned rec = kq[u] & (kTileRecs - 1);
        wq[u] = reinterpret_cast<const float2*>(sm.w)[rec];
        gq[u] = sm.go[(rec >> 4) * 8 + cl];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const unsigned kp = kq[u] >> kRecBits;
        if (kp != cur) {
          // next slot: cur + 1 carries on; any other key ends both
          const bool next = kp == cur + 1u;
          if (cur != none) {
            flush(cur, a0);
            if (!next) flush(cur + 1u, a1);
          }
          a0 = next ? a1 : f4_zero();
          a1 = f4_zero();
          cur = kp;
        }
        f4_fma(a0, wq[u].x, gq[u]);
        f4_fma(a1, wq[u].y, gq[u]);
      }
      if (cur == none) break;
    }
    if (cur != none) {
      flush(cur, a0);
      flush(cur + 1u, a1);
    }
    __syncthreads();   // key[] / w[] are rewritten by the next level
  }
  if (EPI) {
    // grad_logit = w * (grad_w - sum_j w_j grad_w_j), lane = sample as in msda_backward_kernel
    for (int i = 0; i < RW; ++i) {
      const int r = warp * RW + i;
      const int item = sm.item[r];
      if (item < 0) break;
      const size_t si = (size_t)item * p.LP + lane;
      const float2 st = se.stat[r];
      const float aw = __fdiv_rn(expf(__ldg(p.attn + si) - st.x), st.y);
      const float ga = se.ga[r * 32 + lane];
      const float dot = warp_sum(aw * ga);
      red_add_f32(grad_attn + si, aw * (ga - dot));
    }
  }
}

// ---- generic fallback (any C): one thread per (item, channel); scalar atomics.
__global__ void msda_forward_generic_kernel(const MsdaParams p, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.items * p.C) return;
  const int c = (int)(idx % p.C);
  const long long item = idx / p.C;
  const int h = (int)(item % p.H);
  const int b = (int)(item / ((long long)p.Q * p.H));
  const size_t pix_stride = (size_t)p.H * p.C;
  const float* vb = p.value + ((size_t)b * p.K * p.H + h) * p.C + c;
  float acc = 0.f;
  for (int s = 0; s < p.LP; ++s) {
    const int l = s / p.P;
    const int Hl = (int)p.shapes[2 * l], Wl = (int)p.shapes[2 * l + 1];
    int base, meta;
    float lh, lw;
    decode_sample(p.loc[((size_t)item * p.LP + s) * 2], p.loc[((size_t)item * p.LP + s) * 2 + 1],
                  Hl, Wl, (int)p.lsi[l], base, meta, lh, lw);
    const int mask = meta & 15;
    if (!mask) continue;
    const float aw = p.attn[(size_t)item * p.LP + s];
    const size_t dx = (size_t)((meta >> 4) & 1) * pix_stride, dy = (size_t)(meta >> 5) * pix_stride;
    const float* p1 = vb + (size_t)base * pix_stride;
    const float v1 = (mask & 1) ? p1[0] : 0.f, v2 = (mask & 2) ? p1[dx] : 0.f;
    const float v3 = (mask & 4) ? p1[dy] : 0.f, v4 = (mask & 8) ? p1[dy + dx] : 0.f;
    const float hh = 1.f - lh, hw = 1.f - lw;
    acc += aw * (hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4);
  }
  out[idx] = acc;
}

__global__ void msda_backward_generic_kernel(const MsdaParams p, const float* __restrict__ grad_out,
                                             float* __restrict__ grad_value,
                                             float* __restrict__ grad_loc,
                                             float* __restrict__ grad_attn) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.items * p.C) return;
  const int c = (int)(idx % p.C);
  const long long item = idx / p.C;
  const int h = (int)(item % p.H);
  const int b = (int)(item / ((long long)p.Q * p.H));
  const size_t pix_stride = (size_t)p.H * p.C;
  const size_t voff = ((size_t)b * p.K * p.H + h) * p.C + c;
  const float go = grad_out[idx];
  for (int s = 0; s < p.LP; ++s) {
    const int l = s / p.P;
    const int Hl = (int)p.shapes[2 * l], Wl = (int)p.shapes[2 * l + 1];
    int base, meta;
    float lh, lw;
    const size_t si = (size_t)item * p.LP + s;
    decode_sample(p.loc[si * 2], p.loc[si * 2 + 1], Hl, Wl, (int)p.lsi[l], base, meta, lh, lw);
    const int mask = meta & 15;
    if (!mask) continue;
    const float aw = p.attn[si];
    const size_t dx = (size_t)((meta >> 4) & 1) * pix_stride, dy = (size_t)(meta >> 5) * pix_stride;
    const size_t o1 = voff + (size_t)base * pix_stride;
    const float v1 = (mask & 1) ? p.value[o1] : 0.f, v2 = (mask & 2) ? p.value[o1 + dx] : 0.f;
    const float v3 = (mask & 4) ? p.value[o1 + dy] : 0.f, v4 = (mask & 8) ? p.value[o1 + dy + dx] : 0.f;
    const float hh = 1.f - lh, hw = 1.f - lw;
    const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
    const float top = go * aw;
    if (mask & 1) red_add_f32(grad_value + o1, w1 * top);
    if (mask & 2) red_add_f32(grad_value + o1 + dx, w2 * top);
    if (mask & 4) red_add_f32(grad_value + o1 + dy, w3 * top);
    if (mask & 8) red_add_f32(grad_value + o1 + dy + dx, w4 * top);
    red_add_f32(grad_attn + si, go * (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4));
    red_add_f32(grad_loc + si * 2, (float)Wl * top * (hh * (v2 - v1) + lh * (v4 - v3)));
    red_add_f32(grad_loc + si * 2 + 1, (float)Hl * top * (hw * (v3 - v1) + lw * (v4 - v2)));
  }
}

int fill_params(MsdaParams& p, const float* value, const int64_t* shapes, const int64_t* lsi,
                const float* loc, const float* attn, int B, int K, int H, int C, int L, int Q,
                int P, int im2col_step, const char* who) {
  VIDAR_REQUIRE(value && shapes && lsi && loc && attn, "%s: null pointer argument", who);
  VIDAR_REQUIRE(B > 0 && K > 0 && H > 0 && C > 0 && L > 0 && Q > 0 && P > 0,
                "%s: all of B,K,H,C,L,Q,P must be positive (got %d,%d,%d,%d,%d,%d,%d)", who, B, K,
                H, C, L, Q, P);
  VIDAR_REQUIRE(im2col_step > 0, "%s: im2col_step must be positive", who);
  const int step = im2col_step < B ? im2col_step : B;
  // mmcv: AT_ASSERTM(batch % im2col_step_ == 0, "batch(%d) must divide im2col_step(%d)")
  VIDAR_REQUIRE(B % step == 0, "%s: batch(%d) must divide im2col_step(%d)", who, B, step);
  p.value = value;
  p.shapes = shapes;
  p.lsi = lsi;
  p.loc = loc;
  p.attn = attn;
  p.B = B; p.K = K; p.H = H; p.C = C; p.L = L; p.Q = Q; p.P = P;
  p.LP = L * P;
  p.items = (long long)B * Q * H;
  p.ipw = 1;
  p.lp_shift = 0;
  p.pix_stride = H * C;
  p.ref = nullptr;
  p.D = 1;
  p.idx = nullptr; p.count = nullptr; p.inv = nullptr;
  p.ncl = B; p.cam0 = 0; p.bs = 1; p.Qd = Q;
  p.S = 1; p.s_lo = 0; p.s_hi = 1;
  p.G = 1; p.seg_shift = 0; p.Kv = K; p.qscale = 1.f;
  return VIDAR_OK;
}

// vector kernels: C in {16,32,64}, 32-bit intra-batch offsets and item counts
inline bool vec_ok(const MsdaParams& p) {
  return (p.C == 16 || p.C == 32 || p.C == 64) && (long long)p.K * p.H * p.C < (1LL << 25) &&   /* offsets ride in meta bits 5..29 */
         p.items < (1LL << 31) && (long long)p.Q * p.H < (1LL << 31);
}

// items per warp for the vector kernels: pack several (b,q,h) into one 32-sample chunk
// when L*P is small (temporal self-attention: L*P = 4).
inline void set_ipw(MsdaParams& p, int CV) {
  const int NG = 32 / CV;
  p.ipw = (p.LP >= 2 && p.LP < 32 && 32 % p.LP == 0 && p.LP % NG == 0) ? 32 / p.LP : 1;
  p.lp_shift = 0;
  while ((1 << p.lp_shift) < p.LP) ++p.lp_shift;
}

inline long long num_blocks(const MsdaParams& p) {
  if (p.ipw == 1) {
    const long long nqt = (p.Q + kWarpsPerBlock - 1) / kWarpsPerBlock;
    return (long long)p.B * nqt * p.H;
  }
  const long long warps = (p.items + p.ipw - 1) / p.ipw;
  return (warps + kWarpsPerBlock - 1) / kWarpsPerBlock;
}

// The tile-aggregating rows backward: C = 32, 8 points on each of 4 levels (SpatialCrossAttention).
// A level's padded pixel slot (< 2K) and the record index share a 32-bit sort key.
inline bool tile_backward_ok(const MsdaParams& p) {
  return p.C == 32 && p.P == kTilePoints && p.LP == 32 && p.K < (1 << 19);
}
static_assert(20 + kRecBits <= 32, "sort key width at K < 2^19");

// Row order + tile kernel.  The order's scratch (two ints per row and a cell histogram per 1024 rows) is
// stream-ordered (cudaMallocFromPoolAsync / cudaFreeAsync): no host sync, and a CUDA graph captures it as
// allocation nodes, so the C signature needs no workspace argument.
template <bool EPI>
int launch_rows_backward_tiled(const MsdaParams& p, const float* grad_out, float* grad_value, float* grad_loc,
                               float* grad_attn, cudaStream_t st, const char* who) {
  const int nch = (p.Q + kOrderChunk - 1) / kOrderChunk;
  const long long ntiles = (p.Q + kTileRows - 1) / kTileRows;
  const long long nb = (long long)p.B * p.H * ntiles;
  VIDAR_REQUIRE(nb < 2147483647LL && p.B < 65536, "%s: problem too large", who);
  // row items and Z-anchor rows are 32-bit in the tile kernel
  VIDAR_REQUIRE(!EPI || ((long long)p.bs * p.Qd * p.H < (1LL << 31) &&
                         (long long)(p.cam0 + p.ncl) * p.bs * p.Qd * p.D < (1LL << 31)),
                "%s: problem too large", who);
  // the row order reads head 0's sampling locations as float4
  VIDAR_REQUIRE(EPI || ((uintptr_t)p.loc & 15u) == 0, "%s: sampling_loc must be 16-byte aligned", who);
  const size_t smem = tile_smem_bytes<EPI>();
  if (cudaFuncSetAttribute(msda_backward_tile_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return set_error(VIDAR_E_CUDA, "%s: cannot opt in to %zu bytes of shared memory", who, smem);
  cudaMemPool_t pool;
  cudaError_t e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  const size_t nkey = (size_t)p.B * p.Q, nhist = (size_t)p.B * nch * kCells;
  int* scratch = nullptr;
  e = cudaMallocFromPoolAsync((void**)&scratch, sizeof(int) * (2 * nkey + nhist + p.B), pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  int* key = scratch;
  int* perm = key + nkey;
  int* hist = perm + nkey;
  int* nlive = hist + nhist;
  rows_key_kernel<EPI><<<dim3(nch, p.B), kOrderChunk, 0, st>>>(p, key, hist);
  rows_scan_kernel<<<p.B, kCells, 0, st>>>(hist, nlive, nch);
  rows_scatter_kernel<<<dim3(nch, p.B), kOrderChunk, 0, st>>>(key, hist, perm, p.Q);
  msda_backward_tile_kernel<EPI><<<(unsigned)nb, kTileThreads, smem, st>>>(p, perm, nlive, grad_out, grad_value,
                                                                           grad_loc, grad_attn);
  e = cudaFreeAsync(scratch, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(e));
  return check_launch(who);
}

// Calls f(std::integral_constant<int, CV>{}) for head width C in {16, 32, 64}: CV = C / 4 lanes per head vector.
template <class F>
void with_cv(int C, const F& f) {
  if (C == 32) f(std::integral_constant<int, 8>{});
  else if (C == 16) f(std::integral_constant<int, 4>{});
  else f(std::integral_constant<int, 16>{});
}

// The forward of every entry point, once its arguments are checked.  The plain op (!EPI && !IDX) takes the generic
// kernel at head widths the vector kernels do not support (the fused epilogue and the row map require them), and
// packs several items into a warp when L*P is small (set_ipw): the small kernel once every lane group gets an item
// of its own, MULTI below that.  The row map (IDX) keeps fill_rows' one item per warp.  The queue-mean prologue
// (SEG) packs items like the plain op, below head dim 64, but always into msda_forward_kernel, MULTI or not.
template <bool EPI, bool IDX, bool SEG = false>
int msda_forward(MsdaParams& p, float* out, cudaStream_t st, const char* who) {
  VIDAR_REQUIRE(out, "%s: null output", who);
  if (!EPI && !IDX && !SEG && !vec_ok(p)) {
    const long long nb = (p.items * p.C + 255) / 256;
    VIDAR_REQUIRE(nb < 2147483647LL, "%s: problem too large", who);
    msda_forward_generic_kernel<<<(unsigned)nb, 256, 0, st>>>(p, out);
    return check_launch(who);
  }
  if (!IDX) set_ipw(p, p.C / 4);
  if (SEG && p.C == 64) p.ipw = 1;   // one item per warp: the MULTI forward spills at head dim 64
  const long long nb = num_blocks(p);
  VIDAR_REQUIRE(nb < 2147483647LL, "%s: problem too large", who);
  const dim3 grid((unsigned)nb), block(kWarpsPerBlock * 32);
  with_cv(p.C, [&](auto cv) {
    constexpr int CV = decltype(cv)::value;
    if constexpr (SEG) {
      if constexpr (CV < 16) {
        if (p.ipw > 1) {
          msda_forward_kernel<CV, true, false, false, true><<<grid, block, 0, st>>>(p, out);
          return;
        }
      }
      msda_forward_kernel<CV, false, false, false, true><<<grid, block, 0, st>>>(p, out);
    } else if constexpr (!EPI && !IDX) {
      if (p.ipw >= 32 / CV) msda_forward_small_kernel<CV><<<grid, block, 0, st>>>(p, out);
      else if (p.ipw > 1) msda_forward_kernel<CV, true><<<grid, block, 0, st>>>(p, out);
      else msda_forward_kernel<CV, false><<<grid, block, 0, st>>>(p, out);
    } else {
      msda_forward_kernel<CV, false, EPI, IDX><<<grid, block, 0, st>>>(p, out);
    }
  });
  return check_launch(who);
}

// The backward of every entry point, once its arguments are checked: the kernels the forward picks, or the tile
// kernel for the row map where tile_backward_ok.
template <bool EPI, bool IDX, bool SEG = false>
int msda_backward(MsdaParams& p, const float* grad_out, float* grad_value, float* grad_loc, float* grad_attn,
                  cudaStream_t st, const char* who) {
  VIDAR_REQUIRE(grad_out && grad_value && grad_loc && grad_attn, "%s: null gradient pointer", who);
  if (IDX && tile_backward_ok(p))
    return launch_rows_backward_tiled<EPI>(p, grad_out, grad_value, grad_loc, grad_attn, st, who);
  if (!EPI && !IDX && !SEG && !vec_ok(p)) {
    cudaError_t e = cudaMemsetAsync(grad_loc, 0, sizeof(float) * 2 * (size_t)p.items * p.LP, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(grad_attn, 0, sizeof(float) * (size_t)p.items * p.LP, st);
    if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: memset: %s", who, cudaGetErrorString(e));
    const long long nb = (p.items * p.C + 255) / 256;
    VIDAR_REQUIRE(nb < 2147483647LL, "%s: problem too large", who);
    msda_backward_generic_kernel<<<(unsigned)nb, 256, 0, st>>>(p, grad_out, grad_value, grad_loc, grad_attn);
    return check_launch(who);
  }
  if (!IDX) set_ipw(p, p.C / 4);
  if (SEG && p.C == 64) p.ipw = 1;   // one item per warp: the MULTI forward spills at head dim 64
  const long long nb = num_blocks(p);
  VIDAR_REQUIRE(nb < 2147483647LL, "%s: problem too large", who);
  const dim3 grid((unsigned)nb), block(kWarpsPerBlock * 32);
  with_cv(p.C, [&](auto cv) {
    constexpr int CV = decltype(cv)::value;
    if constexpr (SEG) {
      if constexpr (CV < 16) {
        if (p.ipw > 1) {
          msda_backward_kernel<CV, true, false, false, true><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc,
                                                                                     grad_attn);
          return;
        }
      }
      msda_backward_kernel<CV, false, false, false, true><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc,
                                                                                  grad_attn);
    } else if constexpr (!EPI && !IDX) {
      if (p.ipw >= 32 / CV)
        msda_backward_small_kernel<CV><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc, grad_attn);
      else if (p.ipw > 1)
        msda_backward_kernel<CV, true><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc, grad_attn);
      else
        msda_backward_kernel<CV, false><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc, grad_attn);
    } else {
      msda_backward_kernel<CV, false, EPI, IDX><<<grid, block, 0, st>>>(p, grad_out, grad_value, grad_loc, grad_attn);
    }
  });
  return check_launch(who);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_msda_forward(const float* value, const int64_t* spatial_shapes,
                                  const int64_t* level_start, const float* sampling_loc,
                                  const float* attn_weight, float* out, int B, int K, int H, int C,
                                  int L, int Q, int P, int im2col_step, void* stream) {
  const char* who = "ms_deform_attn_forward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, sampling_loc, attn_weight, B, K, H,
                       C, L, Q, P, im2col_step, who);
  if (rc) return rc;
  return msda_forward<false, false>(p, out, (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_backward(const float* value, const int64_t* spatial_shapes,
                                   const int64_t* level_start, const float* sampling_loc,
                                   const float* attn_weight, const float* grad_out,
                                   float* grad_value, float* grad_sampling_loc,
                                   float* grad_attn_weight, int B, int K, int H, int C, int L,
                                   int Q, int P, int im2col_step, void* stream) {
  const char* who = "ms_deform_attn_backward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, sampling_loc, attn_weight, B, K, H,
                       C, L, Q, P, im2col_step, who);
  if (rc) return rc;
  return msda_backward<false, false>(p, grad_out, grad_value, grad_sampling_loc, grad_attn_weight,
                                     (cudaStream_t)stream, who);
}

// ---- MSDeformableAttention3D with the softmax and the sampling-location arithmetic folded in
static int check_sca(MsdaParams& p, const float* ref, int D, const char* who) {
  VIDAR_REQUIRE(ref, "%s: null reference points", who);
  VIDAR_REQUIRE(D > 0 && p.P % D == 0, "%s: num_points (%d) must be a multiple of the number of Z anchors (%d)", who, p.P, D);
  VIDAR_REQUIRE(p.LP == 32, "%s: the fused epilogue needs num_levels * num_points == 32 (got %d)", who, p.LP);
  VIDAR_REQUIRE(vec_ok(p) && (p.C == 16 || p.C == 32 || p.C == 64), "%s: head dim must be 16, 32 or 64 (got %d)", who, p.C);
  p.ref = ref;
  p.D = D;
  return VIDAR_OK;
}

extern "C" int vidar_msda_sca_forward(const float* value, const int64_t* spatial_shapes,
                                      const int64_t* level_start, const float* ref_points,
                                      const float* offsets, const float* logits, float* out, int B,
                                      int K, int H, int C, int L, int Q, int P, int D, void* stream) {
  const char* who = "msda_sca_forward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, B, K, H, C, L, Q, P, B, who);
  if (rc) return rc;
  rc = check_sca(p, ref_points, D, who);
  if (rc) return rc;
  return msda_forward<true, false>(p, out, (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_sca_backward(const float* value, const int64_t* spatial_shapes,
                                       const int64_t* level_start, const float* ref_points,
                                       const float* offsets, const float* logits, const float* grad_out,
                                       float* grad_value, float* grad_offsets, float* grad_logits, int B,
                                       int K, int H, int C, int L, int Q, int P, int D, void* stream) {
  const char* who = "msda_sca_backward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, B, K, H, C, L, Q, P, B, who);
  if (rc) return rc;
  rc = check_sca(p, ref_points, D, who);
  if (rc) return rc;
  return msda_backward<true, false>(p, grad_out, grad_value, grad_offsets, grad_logits, (cudaStream_t)stream, who);
}

// ---- TemporalSelfAttention / the future decoder's deformable attention with the softmax, the sampling-location
// arithmetic and TSA's mean over the queue folded in: items are (b, q, h) of the output, each with G*L*P samples
static int check_tsa(MsdaParams& p, const float* ref, int G, const char* who) {
  VIDAR_REQUIRE(ref, "%s: null reference points", who);
  const int LP = p.LP;
  VIDAR_REQUIRE(LP <= 32 && (LP & (LP - 1)) == 0,
                "%s: the fused prologue needs num_levels * num_points in {1, 2, 4, 8, 16, 32} (got %d)", who, LP);
  VIDAR_REQUIRE(G > 0 && G <= 32 / LP, "%s: num_queue * num_levels * num_points must be at most 32 (got %d x %d)",
                who, G, LP);
  VIDAR_REQUIRE(p.C == 16 || p.C == 32 || p.C == 64, "%s: head dim must be 16, 32 or 64 (got %d)", who, p.C);
  // the G value batches of an item are one slab addressed with 32-bit offsets
  VIDAR_REQUIRE((long long)G * p.K * p.H * p.C < (1LL << 25), "%s: problem too large", who);
  p.Kv = p.K;
  p.K = G * p.K;
  VIDAR_REQUIRE(vec_ok(p), "%s: problem too large", who);
  p.G = G;
  p.seg_shift = 0;
  while ((1 << p.seg_shift) < LP) ++p.seg_shift;
  p.LP = G * LP;
  p.qscale = 1.f / (float)G;
  p.ref = ref;
  return VIDAR_OK;
}

extern "C" int vidar_msda_tsa_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                      const float* ref_points, const float* offsets, const float* logits, float* out,
                                      int B, int G, int K, int H, int C, int L, int Q, int P, void* stream) {
  const char* who = "msda_tsa_forward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, B, K, H, C, L, Q, P, B, who);
  if (rc) return rc;
  rc = check_tsa(p, ref_points, G, who);
  if (rc) return rc;
  return msda_forward<false, false, true>(p, out, (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_tsa_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                       const float* ref_points, const float* offsets, const float* logits,
                                       const float* grad_out, float* grad_value, float* grad_offsets,
                                       float* grad_logits, int B, int G, int K, int H, int C, int L, int Q, int P,
                                       void* stream) {
  const char* who = "msda_tsa_backward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, B, K, H, C, L, Q, P, B, who);
  if (rc) return rc;
  rc = check_tsa(p, ref_points, G, who);
  if (rc) return rc;
  return msda_backward<false, false, true>(p, grad_out, grad_value, grad_offsets, grad_logits, (cudaStream_t)stream,
                                           who);
}

// ---- row-indirect entry points: SpatialCrossAttention's rebatch / scatter-add fused into the op ------
// Rows are (camera, j) entries of per-camera visible-pillar lists (vidar_sca_compact); the forward adds
// each row's head vectors, scaled by 1/#cameras, straight into the BEV slot grid and the backward reads
// the slot gradient back through the same map (spatial_cross_attention.py:136-171 without the
// [cams, max_len, C] intermediates, the index_add_ and the host sync on max_len).
static int fill_rows(MsdaParams& p, const int32_t* idx, const int32_t* count, const float* inv, int bs, int ncl,
                     int cam0, int Qd, int S, int s_lo, int s_hi, const char* who) {
  VIDAR_REQUIRE(bs > 0 && ncl > 0 && cam0 >= 0 && Qd > 0, "%s: bad sizes bs=%d cameras=%d cam0=%d pillars=%d", who, bs, ncl, cam0, Qd);
  VIDAR_REQUIRE(p.B == bs * ncl, "%s: value batch (%d) must be bs * cameras (%d x %d)", who, p.B, bs, ncl);
  VIDAR_REQUIRE(p.Q <= Qd, "%s: rows per camera (%d) exceed the pillar count (%d)", who, p.Q, Qd);
  VIDAR_REQUIRE(idx || p.Q == Qd, "%s: without an index list every pillar is a row (rows %d != pillars %d)", who, p.Q, Qd);
  VIDAR_REQUIRE(S >= 1 && s_lo >= 0 && s_lo <= s_hi && s_hi <= S, "%s: bad sub-slice [%d, %d) of %d", who, s_lo, s_hi, S);
  VIDAR_REQUIRE(vec_ok(p), "%s: head dim must be 16, 32 or 64 (got %d)", who, p.C);
  p.idx = idx; p.count = count; p.inv = inv;
  p.bs = bs; p.ncl = ncl; p.cam0 = cam0; p.Qd = Qd;
  p.S = S; p.s_lo = s_lo; p.s_hi = s_hi;
  p.ipw = 1;
  p.lp_shift = 0;
  return VIDAR_OK;
}

extern "C" int vidar_msda_rows_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                       const float* sampling_loc, const float* attn_weight, const int32_t* idx,
                                       const int32_t* count, const float* inv_count, float* slots, int bs, int ncl,
                                       int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P, int S, int s_lo,
                                       int s_hi, void* stream) {
  const char* who = "msda_rows_forward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, sampling_loc, attn_weight, bs * ncl, K, H, C, L, Qrows, P,
                       bs * ncl, who);
  if (rc) return rc;
  rc = fill_rows(p, idx, count, inv_count, bs, ncl, cam0, Qd, S, s_lo, s_hi, who);
  if (rc) return rc;
  return msda_forward<false, true>(p, slots, (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_rows_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                        const float* sampling_loc, const float* attn_weight, const int32_t* idx,
                                        const int32_t* count, const float* inv_count, const float* grad_slots,
                                        float* grad_value, float* grad_sampling_loc, float* grad_attn_weight, int bs,
                                        int ncl, int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P, int S,
                                        int s_lo, int s_hi, void* stream) {
  const char* who = "msda_rows_backward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, sampling_loc, attn_weight, bs * ncl, K, H, C, L, Qrows, P,
                       bs * ncl, who);
  if (rc) return rc;
  rc = fill_rows(p, idx, count, inv_count, bs, ncl, cam0, Qd, S, s_lo, s_hi, who);
  if (rc) return rc;
  return msda_backward<false, true>(p, grad_slots, grad_value, grad_sampling_loc, grad_attn_weight,
                                    (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_sca_rows_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                           const float* ref_cam, const float* offsets, const float* logits,
                                           const int32_t* idx, const int32_t* count, const float* inv_count, float* slots,
                                           int bs, int ncl, int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P,
                                           int D, int S, int s_lo, int s_hi, void* stream) {
  const char* who = "msda_sca_rows_forward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, bs * ncl, K, H, C, L, Qrows, P, bs * ncl, who);
  if (rc) return rc;
  rc = check_sca(p, ref_cam, D, who);
  if (rc) return rc;
  rc = fill_rows(p, idx, count, inv_count, bs, ncl, cam0, Qd, S, s_lo, s_hi, who);
  if (rc) return rc;
  return msda_forward<true, true>(p, slots, (cudaStream_t)stream, who);
}

extern "C" int vidar_msda_sca_rows_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                            const float* ref_cam, const float* offsets, const float* logits,
                                            const int32_t* idx, const int32_t* count, const float* inv_count,
                                            const float* grad_slots, float* grad_value, float* grad_offsets,
                                            float* grad_logits, int bs, int ncl, int cam0, int K, int H, int C, int L,
                                            int Qrows, int Qd, int P, int D, int S, int s_lo, int s_hi, void* stream) {
  const char* who = "msda_sca_rows_backward";
  MsdaParams p;
  int rc = fill_params(p, value, spatial_shapes, level_start, offsets, logits, bs * ncl, K, H, C, L, Qrows, P, bs * ncl, who);
  if (rc) return rc;
  rc = check_sca(p, ref_cam, D, who);
  if (rc) return rc;
  rc = fill_rows(p, idx, count, inv_count, bs, ncl, cam0, Qd, S, s_lo, s_hi, who);
  if (rc) return rc;
  return msda_backward<true, true>(p, grad_slots, grad_value, grad_offsets, grad_logits, (cudaStream_t)stream, who);
}
