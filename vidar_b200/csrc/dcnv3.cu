// Deformable convolution v3 (InternImage's DCNv3 core op): one-level deformable sampling with per-group weights.
//
// input [N, H, W, G*Cg], offset [N, Ho, Wo, G*K*2] as (dx, dy) pairs, mask [N, Ho, Wo, G*K], output [N, Ho, Wo, G*Cg],
// all channel-last, K = kh*kw.  Kernel point p = i*kh + j, i < kw along x (outer), j < kh along y.  With
// s = offset_scale, cw = (dw*(kw-1)) >> 1 and ch = (dh*(kh-1)) >> 1, point p of (n, ho, wo, g) samples at
//   x = wo*sw - pw + cw + (i*dw - cw + dx) * s,   y = ho*sh - ph + ch + (j*dh - ch + dy) * s
// in pixels of the unpadded input.  It contributes only inside the open range -1 < y < H, -1 < x < W, as the
// bilinear form on the floor cell with corners outside the image reading 0:
//   out[n, ho, wo, g, c] = sum_p mask[n, ho, wo, g, p] * bilinear(input[n, :, :, g*Cg + c], y, x).
//
// An item is one (pixel, group); items are numbered (n, ho, wo, g), so item t's 2K offsets start at 2K t, its K
// weights at K t and its output at Cg t.  A lane group of L lanes (a power of two, L <= 32) owns one item and covers
// its Cg channels with 16-byte vectors (4 floats, or 8 fp16 / bf16 values) when Cg is a multiple of the vector width
// and the buffers are 16-byte aligned, one channel per lane otherwise.  The item's offsets and weights are read once
// per lane group: lane l loads point p0 + l of each run of L points and shuffles it to the others.
//
// Storage type T is float, __half or __nv_bfloat16 for input, offset, mask, output, grad_output, grad_offset and
// grad_mask; every value is converted to fp32 on load, all arithmetic is fp32 and each stored value is rounded once.
// grad_input is accumulated in fp32 (red.global.add) into a caller-zeroed buffer.
#include "channel_vec.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;

struct Dcnv3Geom {
  int H, W, Ho, Wo, G, Cg, kh, kw, sh, sw, ph, pw, dh, dw;
  float s;
};

// Where one kernel point of an item samples: the floor cell, fractional parts and which corners are in the image.
struct Tap {
  bool inside;
  int y0, x0;
  float ly, lx;
  bool v00, v01, v10, v11;
};

__device__ __forceinline__ Tap locate(const Dcnv3Geom& g, float y, float x) {
  Tap t;
  t.inside = y > -1.f && x > -1.f && y < (float)g.H && x < (float)g.W;
  const float yf = floorf(y), xf = floorf(x);
  t.y0 = (int)yf;
  t.x0 = (int)xf;
  t.ly = y - yf;
  t.lx = x - xf;
  t.v00 = t.inside && t.y0 >= 0 && t.x0 >= 0;
  t.v01 = t.inside && t.y0 >= 0 && t.x0 + 1 <= g.W - 1;
  t.v10 = t.inside && t.y0 + 1 <= g.H - 1 && t.x0 >= 0;
  t.v11 = t.inside && t.y0 + 1 <= g.H - 1 && t.x0 + 1 <= g.W - 1;
  return t;
}

// The lane group of this thread: its first lane's bit pattern as a shuffle mask.
__device__ __forceinline__ unsigned group_mask(int L) {
  const unsigned bits = L == 32 ? 0xffffffffu : ((1u << L) - 1u);
  return bits << ((threadIdx.x & 31) & ~(L - 1));
}

// Per-item constants: the item's image, the sample origin for i = j = 0 with offset 0, and its offset / weight rows.
struct Item {
  long long img;  // element offset of input[n, 0, 0, g*Cg]
  float bx, by;   // x (y) = bx + (i*dw + dx) * s
};

__device__ __forceinline__ Item item_of(const Dcnv3Geom& g, long long t) {
  const long long pix = t / g.G;
  const int grp = (int)(t - pix * g.G);
  const long long HWo = (long long)g.Ho * g.Wo;
  const long long n = pix / HWo;
  const int q = (int)(pix - n * HWo);
  const int ho = q / g.Wo, wo = q - ho * g.Wo;
  const int cw = (g.dw * (g.kw - 1)) >> 1, ch = (g.dh * (g.kh - 1)) >> 1;
  Item it;
  it.img = (n * g.H * g.W) * (long long)(g.G * g.Cg) + (long long)grp * g.Cg;
  it.bx = (float)(wo * g.sw - g.pw + cw) - (float)cw * g.s;
  it.by = (float)(ho * g.sh - g.ph + ch) - (float)ch * g.s;
  return it;
}

// Loads lane l's point p0 + l of item t (when p0 + l < K): dx, dy and the weight, as fp32.
template <typename T>
__device__ __forceinline__ void load_point(const T* __restrict__ offset, const T* __restrict__ mask, long long t, int K,
                                           int p, float& dx, float& dy, float& m) {
  dx = dy = m = 0.f;
  if (p < K) {
    const T* op = offset + (t * K + p) * 2;
    dx = to_f(__ldg(op));
    dy = to_f(__ldg(op + 1));
    m = to_f(__ldg(mask + t * K + p));
  }
}

// out[t, c] for the lane's channels c = sub*V + k*L*V.  Channel runs are the outer loop so that one accumulator
// suffices; with Cg <= L*V (every vector case up to Cg = 128 fp32 / 256 16-bit) there is one run.  The bound of one
// block per SM leaves ptxas the registers the unrolled point loop needs: under the plain bound it spilled 8-24 bytes.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) dcnv3_forward_kernel(const T* __restrict__ input, const T* __restrict__ offset,
                                                                 const T* __restrict__ mask, T* __restrict__ output,
                                                                 Dcnv3Geom g, long long items, int lg) {
  using Op = Vec<T, V>;
  const int L = 1 << lg;
  const long long t = ((long long)blockIdx.x * kThreads + threadIdx.x) >> lg;
  if (t >= items) return;  // the whole lane group leaves together
  const int sub = threadIdx.x & (L - 1);
  const unsigned gm = group_mask(L);
  const int K = g.kh * g.kw;
  const int C = g.G * g.Cg;
  const Item it = item_of(g, t);
  const T* img = input + it.img;
  for (int c0 = 0; c0 < g.Cg; c0 += L * V) {
    const int c = c0 + sub * V;
    typename Op::T acc = Op::zero();
    for (int p0 = 0; p0 < K; p0 += L) {
      float mdx, mdy, mm;
      load_point(offset, mask, t, K, p0 + sub, mdx, mdy, mm);
      const int np = K - p0 < L ? K - p0 : L;
      for (int q = 0; q < np; ++q) {
        const float dx = __shfl_sync(gm, mdx, q, L), dy = __shfl_sync(gm, mdy, q, L), m = __shfl_sync(gm, mm, q, L);
        const int p = p0 + q;
        const int i = p / g.kh, j = p - i * g.kh;
        const Tap s = locate(g, fmaf((float)(j * g.dh) + dy, g.s, it.by), fmaf((float)(i * g.dw) + dx, g.s, it.bx));
        if (!s.inside || c >= g.Cg) continue;
        const float w00 = (1.f - s.ly) * (1.f - s.lx), w01 = (1.f - s.ly) * s.lx, w10 = s.ly * (1.f - s.lx),
                    w11 = s.ly * s.lx;
        const T* p00 = img + ((long long)s.y0 * g.W + s.x0) * C + c;
        const T* p01 = p00 + C;
        const T* p10 = p00 + (long long)g.W * C;
        const T* p11 = p10 + C;
        typename Op::T v = Op::zero();
        if (s.v00) v = Op::fma(w00, Op::load(p00), v);
        if (s.v01) v = Op::fma(w01, Op::load(p01), v);
        if (s.v10) v = Op::fma(w10, Op::load(p10), v);
        if (s.v11) v = Op::fma(w11, Op::load(p11), v);
        acc = Op::fma(m, v, acc);
      }
    }
    if (c < g.Cg) Op::store(output + t * g.Cg + c, acc);
  }
}

// Backward from grad_output (layout of output):
//   grad_input [N, H, W, G*Cg] fp32, caller-zeroed  += m * corner weight * grad_out      (red.global.add)
//   grad_offset [N, Ho, Wo, G*K*2]                   = s * m * sum_c grad_out * d v_c / d(x, y)
//   grad_mask   [N, Ho, Wo, G*K]                     = sum_c grad_out * v_c
// d v / d(x, y) is the derivative of the bilinear form on the floor cell (one-sided on integer lines); a point outside
// the open range gets 0 for every gradient.  The channel sums are reduced across the lane group by shuffles and each
// (item, point) is written once, by lane p mod L.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) dcnv3_backward_kernel(
    const T* __restrict__ input, const T* __restrict__ offset, const T* __restrict__ mask,
    const T* __restrict__ grad_output, float* __restrict__ grad_input, T* __restrict__ grad_offset,
    T* __restrict__ grad_mask, Dcnv3Geom g, long long items, int lg) {
  using Op = Vec<T, V>;
  const int L = 1 << lg;
  const long long t = ((long long)blockIdx.x * kThreads + threadIdx.x) >> lg;
  if (t >= items) return;
  const int sub = threadIdx.x & (L - 1);
  const unsigned gm = group_mask(L);
  const int K = g.kh * g.kw;
  const int C = g.G * g.Cg;
  const Item it = item_of(g, t);
  const T* go = grad_output + t * g.Cg;
  for (int p0 = 0; p0 < K; p0 += L) {
    float mdx, mdy, mm;
    load_point(offset, mask, t, K, p0 + sub, mdx, mdy, mm);
    float own_x = 0.f, own_y = 0.f, own_m = 0.f;  // the sums of point p0 + sub
    const int np = K - p0 < L ? K - p0 : L;
    for (int q = 0; q < np; ++q) {
      const float dx = __shfl_sync(gm, mdx, q, L), dy = __shfl_sync(gm, mdy, q, L), m = __shfl_sync(gm, mm, q, L);
      const int p = p0 + q;
      const int i = p / g.kh, j = p - i * g.kh;
      const Tap s = locate(g, fmaf((float)(j * g.dh) + dy, g.s, it.by), fmaf((float)(i * g.dw) + dx, g.s, it.bx));
      if (!s.inside) continue;  // uniform over the lane group: every gradient of this point is 0
      const float hy = 1.f - s.ly, hx = 1.f - s.lx;
      const float w00 = hy * hx, w01 = hy * s.lx, w10 = s.ly * hx, w11 = s.ly * s.lx;
      const long long o00 = it.img + ((long long)s.y0 * g.W + s.x0) * C;
      const long long o01 = o00 + C, o10 = o00 + (long long)g.W * C, o11 = o10 + C;
      // v and d v / d(x, y) are the same four-corner combinations for every channel, so the channel sums are taken
      // per corner (d_ab = grad_out . x_ab) and combined once: four dot products instead of three vector forms.
      float sum_v = 0.f, sum_x = 0.f, sum_y = 0.f;
      for (int c = sub * V; c < g.Cg; c += L * V) {
        const typename Op::T gv = Op::load(go + c);
        const typename Op::T z = Op::zero();
        const typename Op::T x00 = s.v00 ? Op::load(input + o00 + c) : z;
        const typename Op::T x01 = s.v01 ? Op::load(input + o01 + c) : z;
        const typename Op::T x10 = s.v10 ? Op::load(input + o10 + c) : z;
        const typename Op::T x11 = s.v11 ? Op::load(input + o11 + c) : z;
        const float d00 = Op::dot(gv, x00), d01 = Op::dot(gv, x01), d10 = Op::dot(gv, x10), d11 = Op::dot(gv, x11);
        sum_v += fmaf(w11, d11, fmaf(w10, d10, fmaf(w01, d01, w00 * d00)));
        sum_x += fmaf(s.ly, d11 - d10, hy * (d01 - d00));
        sum_y += fmaf(s.lx, d11 - d01, hx * (d10 - d00));
        const typename Op::T gmv = Op::scale(m, gv);
        if (s.v00) Op::red(grad_input + o00 + c, Op::scale(w00, gmv));
        if (s.v01) Op::red(grad_input + o01 + c, Op::scale(w01, gmv));
        if (s.v10) Op::red(grad_input + o10 + c, Op::scale(w10, gmv));
        if (s.v11) Op::red(grad_input + o11 + c, Op::scale(w11, gmv));
      }
      for (int o = L >> 1; o > 0; o >>= 1) {
        sum_v += __shfl_xor_sync(gm, sum_v, o, L);
        sum_x += __shfl_xor_sync(gm, sum_x, o, L);
        sum_y += __shfl_xor_sync(gm, sum_y, o, L);
      }
      if (q == sub) {
        own_x = g.s * m * sum_x;
        own_y = g.s * m * sum_y;
        own_m = sum_v;
      }
    }
    if (sub < np) {
      const long long p = t * K + p0 + sub;
      store1(grad_offset + 2 * p, own_x);
      store1(grad_offset + 2 * p + 1, own_y);
      store1(grad_mask + p, own_m);
    }
  }
}

int validate(const char* who, int dtype, int N, int H, int W, int G, int Cg, int kh, int kw, int sh, int sw, int ph,
             int pw, int dh, int dw, int im2col_step, int& Ho, int& Wo) {
  VIDAR_REQUIRE(dtype == VIDAR_DTYPE_F32 || dtype == VIDAR_DTYPE_F16 || dtype == VIDAR_DTYPE_BF16,
                "%s: unsupported dtype %d", who, dtype);
  VIDAR_REQUIRE(N > 0 && H > 0 && W > 0 && G > 0 && Cg > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 &&
                    pw >= 0 && dh > 0 && dw > 0,
                "%s: bad sizes N=%d H=%d W=%d group=%d group_channels=%d kernel %dx%d stride %dx%d pad %dx%d "
                "dilation %dx%d",
                who, N, H, W, G, Cg, kh, kw, sh, sw, ph, pw, dh, dw);
  VIDAR_REQUIRE(im2col_step > 0, "%s: im2col_step must be positive", who);
  const int step = im2col_step < N ? im2col_step : N;
  VIDAR_REQUIRE(N % step == 0, "%s: batch(%d) must divide im2col_step(%d)", who, N, step);
  const long long ho = ((long long)H + 2LL * ph - ((long long)dh * (kh - 1) + 1)) / sh + 1;
  const long long wo = ((long long)W + 2LL * pw - ((long long)dw * (kw - 1) + 1)) / sw + 1;
  VIDAR_REQUIRE(ho > 0 && wo > 0 && ho < (1LL << 31) && wo < (1LL << 31), "%s: empty output (%lld x %lld)", who, ho,
                wo);
  VIDAR_REQUIRE((long long)G * Cg < (1LL << 31) && (long long)G * kh * kw * 2 < (1LL << 31),
                "%s: group * group_channels = %lld or group * K = %lld is too large", who, (long long)G * Cg,
                (long long)G * kh * kw);
  Ho = (int)ho;
  Wo = (int)wo;
  return VIDAR_OK;
}

// Lanes per item: enough 16-byte vectors (or channels) to cover Cg, as a power of two, at most a warp.
int lanes_log2(int Cg, int V) {
  const int need = (Cg + V - 1) / V;
  int lg = 0;
  while (lg < 5 && (1 << lg) < need) ++lg;
  return lg;
}

template <typename T>
int forward(const char* who, const void* input, const void* offset, const void* mask, void* output, const Dcnv3Geom& g,
            long long items, cudaStream_t st) {
  const T *x = (const T*)input, *o = (const T*)offset, *m = (const T*)mask;
  const bool vec = g.Cg % kVec<T> == 0 && aligned16(input) && aligned16(output);
  const int lg = lanes_log2(g.Cg, vec ? kVec<T> : 1);
  const long long blocks = ((items << lg) + kThreads - 1) / kThreads;
  VIDAR_REQUIRE(blocks < (1LL << 31), "%s: %lld items is too many", who, items);
  if (vec)
    dcnv3_forward_kernel<T, kVec<T>><<<(unsigned)blocks, kThreads, 0, st>>>(x, o, m, (T*)output, g, items, lg);
  else
    dcnv3_forward_kernel<T, 1><<<(unsigned)blocks, kThreads, 0, st>>>(x, o, m, (T*)output, g, items, lg);
  return check_launch(who);
}

template <typename T>
int backward(const char* who, const void* input, const void* offset, const void* mask, const void* grad_output,
             float* grad_input, void* grad_offset, void* grad_mask, const Dcnv3Geom& g, long long items,
             cudaStream_t st) {
  const T *x = (const T*)input, *o = (const T*)offset, *m = (const T*)mask, *gy = (const T*)grad_output;
  const bool vec = g.Cg % kVec<T> == 0 && aligned16(input) && aligned16(grad_output) && aligned16(grad_input);
  const int lg = lanes_log2(g.Cg, vec ? kVec<T> : 1);
  const long long blocks = ((items << lg) + kThreads - 1) / kThreads;
  VIDAR_REQUIRE(blocks < (1LL << 31), "%s: %lld items is too many", who, items);
  if (vec)
    dcnv3_backward_kernel<T, kVec<T>><<<(unsigned)blocks, kThreads, 0, st>>>(x, o, m, gy, grad_input, (T*)grad_offset,
                                                                            (T*)grad_mask, g, items, lg);
  else
    dcnv3_backward_kernel<T, 1><<<(unsigned)blocks, kThreads, 0, st>>>(x, o, m, gy, grad_input, (T*)grad_offset,
                                                                      (T*)grad_mask, g, items, lg);
  return check_launch(who);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_dcnv3_forward(const void* input, const void* offset, const void* mask, void* output, int dtype,
                                   int N, int H, int W, int group, int group_channels, int kernel_h, int kernel_w,
                                   int stride_h, int stride_w, int pad_h, int pad_w, int dilation_h, int dilation_w,
                                   float offset_scale, int im2col_step, void* stream) {
  const char* who = "dcnv3_forward";
  VIDAR_REQUIRE(input && offset && mask && output, "%s: null pointer argument", who);
  int Ho = 0, Wo = 0;
  const int rc = validate(who, dtype, N, H, W, group, group_channels, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                          pad_w, dilation_h, dilation_w, im2col_step, Ho, Wo);
  if (rc) return rc;
  const Dcnv3Geom g{H, W, Ho, Wo, group, group_channels, kernel_h, kernel_w, stride_h, stride_w,
                    pad_h, pad_w, dilation_h, dilation_w, offset_scale};
  const long long items = (long long)N * Ho * Wo * group;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == VIDAR_DTYPE_F32) return forward<float>(who, input, offset, mask, output, g, items, st);
  if (dtype == VIDAR_DTYPE_F16) return forward<__half>(who, input, offset, mask, output, g, items, st);
  return forward<__nv_bfloat16>(who, input, offset, mask, output, g, items, st);
}

extern "C" int vidar_dcnv3_backward(const void* input, const void* offset, const void* mask, const void* grad_output,
                                    float* grad_input, void* grad_offset, void* grad_mask, int dtype, int N, int H,
                                    int W, int group, int group_channels, int kernel_h, int kernel_w, int stride_h,
                                    int stride_w, int pad_h, int pad_w, int dilation_h, int dilation_w,
                                    float offset_scale, int im2col_step, void* stream) {
  const char* who = "dcnv3_backward";
  VIDAR_REQUIRE(input && offset && mask && grad_output && grad_input && grad_offset && grad_mask,
                "%s: null pointer argument", who);
  int Ho = 0, Wo = 0;
  const int rc = validate(who, dtype, N, H, W, group, group_channels, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                          pad_w, dilation_h, dilation_w, im2col_step, Ho, Wo);
  if (rc) return rc;
  const Dcnv3Geom g{H, W, Ho, Wo, group, group_channels, kernel_h, kernel_w, stride_h, stride_w,
                    pad_h, pad_w, dilation_h, dilation_w, offset_scale};
  const long long items = (long long)N * Ho * Wo * group;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == VIDAR_DTYPE_F32)
    return backward<float>(who, input, offset, mask, grad_output, grad_input, grad_offset, grad_mask, g, items, st);
  if (dtype == VIDAR_DTYPE_F16)
    return backward<__half>(who, input, offset, mask, grad_output, grad_input, grad_offset, grad_mask, g, items, st);
  return backward<__nv_bfloat16>(who, input, offset, mask, grad_output, grad_input, grad_offset, grad_mask, g, items,
                                 st);
}
