// Modulated deformable convolution (DCNv2, mmcv's ModulatedDeformConv2d) around an explicit column matrix.
//
// For output pixel (n, ho, wo) and kernel point k = i * kw + j the sample sits at
//   h = ho * sh - ph + i * dh + offset[n, 2k, ho, wo],   w = wo * sw - pw + j * dw + offset[n, 2k + 1, ho, wo]
// and reads the bilinear value v_c of x[n, c] from the floor cell (0 when h <= -1, h >= H, w <= -1 or w >= W; a corner
// outside the image adds 0).  Column row m = (n, ho, wo) holds mask[n, k, ho, wo] * v_c at k * C + c, so the
// convolution is cols [M, kh*kw*C] times the weight permuted to [Cout, kh, kw, C] -- a GEMM the host runs.
//
// x is channel-last (NHWC): every bilinear corner is one contiguous C-element line, and a column row is written as
// kh*kw full lines.  One warp per (row, kernel point); its lanes stride over the channels, one 16-byte vector at a
// time when C is a multiple of its width (4 floats, or 8 fp16 / bf16 values) and the buffers are 16-byte aligned,
// one channel at a time otherwise.
//
// Storage type T is float, __half or __nv_bfloat16 for x, offset, mask and the columns.  Every value is converted to
// fp32 on load; the bilinear weights, products and sums are fp32.  A 16-bit im2col rounds each column element once on
// its store.  col2im accumulates grad_x and writes grad_offset / grad_mask in fp32 whatever T is.
#include "channel_vec.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct DcnGeom {
  int C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0;
};

// Where item (local row m, kernel point k) samples: image n, modulation, and the bilinear cell.
struct Sample {
  long long n;
  float m;            // mask value
  bool inside;        // within the open range (-1, H) x (-1, W)
  int y0, x0;         // floor corner
  float lh, lw;       // fractional parts
  bool v00, v01, v10, v11;
};

template <typename T>
__device__ __forceinline__ Sample locate(const T* __restrict__ offset, const T* __restrict__ mask, const DcnGeom& g,
                                         long long m, int k) {
  const int K = g.kh * g.kw;
  const long long HW = (long long)g.Ho * g.Wo;
  Sample s;
  const long long nl = m / HW;
  const long long p = m - nl * HW;
  const int ho = (int)(p / g.Wo), wo = (int)(p - (long long)ho * g.Wo);
  const int i = k / g.kw, j = k - i * g.kw;
  s.n = g.n0 + nl;
  const T* op = offset + (s.n * 2 * K + 2 * k) * HW + p;
  const float h = (float)(ho * g.sh - g.ph + i * g.dh) + to_f(__ldg(op));
  const float w = (float)(wo * g.sw - g.pw + j * g.dw) + to_f(__ldg(op + HW));
  s.m = to_f(__ldg(mask + (s.n * K + k) * HW + p));
  s.inside = !(h <= -1.f || h >= (float)g.H || w <= -1.f || w >= (float)g.W);
  const float hf = floorf(h), wf = floorf(w);
  s.y0 = (int)hf;
  s.x0 = (int)wf;
  s.lh = h - hf;
  s.lw = w - wf;
  s.v00 = s.inside && s.y0 >= 0 && s.x0 >= 0;
  s.v01 = s.inside && s.y0 >= 0 && s.x0 + 1 <= g.W - 1;
  s.v10 = s.inside && s.y0 + 1 <= g.H - 1 && s.x0 >= 0;
  s.v11 = s.inside && s.y0 + 1 <= g.H - 1 && s.x0 + 1 <= g.W - 1;
  return s;
}

// cols [rows, K * C]: row m, kernel point k, channel c at (m * K + k) * C + c.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) dcn_im2col_kernel(const T* __restrict__ x, const T* __restrict__ offset,
                                                              const T* __restrict__ mask, T* __restrict__ cols,
                                                              DcnGeom g, long long items) {
  using Op = Vec<T, V>;
  const int lane = threadIdx.x & 31;
  const int K = g.kh * g.kw;
  const long long stride = (long long)gridDim.x * kWarps;
  for (long long it = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5); it < items; it += stride) {
    const long long m = it / K;
    const int k = (int)(it - m * K);
    const Sample s = locate(offset, mask, g, m, k);
    T* out = cols + it * g.C;
    const float w00 = (1.f - s.lh) * (1.f - s.lw), w01 = (1.f - s.lh) * s.lw, w10 = s.lh * (1.f - s.lw), w11 = s.lh * s.lw;
    const T* img = x + s.n * g.H * g.W * g.C;
    const T* p00 = img + ((long long)s.y0 * g.W + s.x0) * g.C;
    const T* p01 = p00 + g.C;
    const T* p10 = p00 + (long long)g.W * g.C;
    const T* p11 = p10 + g.C;
    for (int c = lane * V; c < g.C; c += 32 * V) {
      typename Op::T v = Op::zero();
      if (s.v00) v = Op::fma(w00, Op::load(p00 + c), v);
      if (s.v01) v = Op::fma(w01, Op::load(p01 + c), v);
      if (s.v10) v = Op::fma(w10, Op::load(p10 + c), v);
      if (s.v11) v = Op::fma(w11, Op::load(p11 + c), v);
      Op::store(out + c, Op::scale(s.m, v));
    }
  }
}

// Backward of the sampling from grad_cols (same layout as cols):
//   grad_x [N, H, W, C] (caller-zeroed)  += mask * corner weight * grad_col     (red.global.add)
//   grad_offset [N, 2K, Ho, Wo]           = mask * sum_c grad_col * d v_c / d(h, w)
//   grad_mask [N, K, Ho, Wo]              = sum_c grad_col * v_c
// The derivative is that of the bilinear form on the floor cell (one-sided on integer lines, 0 outside the open range).
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) dcn_col2im_kernel(const T* __restrict__ x, const T* __restrict__ offset,
                                                              const T* __restrict__ mask,
                                                              const T* __restrict__ grad_cols, float* __restrict__ grad_x,
                                                              float* __restrict__ grad_offset, float* __restrict__ grad_mask,
                                                              DcnGeom g, long long items) {
  using Op = Vec<T, V>;
  const int lane = threadIdx.x & 31;
  const int K = g.kh * g.kw;
  const long long HW = (long long)g.Ho * g.Wo;
  const long long stride = (long long)gridDim.x * kWarps;
  for (long long it = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5); it < items; it += stride) {
    const long long m = it / K;
    const int k = (int)(it - m * K);
    const Sample s = locate(offset, mask, g, m, k);
    const T* gc = grad_cols + it * g.C;
    const float hh = 1.f - s.lh, hw = 1.f - s.lw;
    const float w00 = hh * hw, w01 = hh * s.lw, w10 = s.lh * hw, w11 = s.lh * s.lw;
    const long long img = s.n * g.H * g.W * g.C;
    const long long o00 = img + ((long long)s.y0 * g.W + s.x0) * g.C;
    const long long o01 = o00 + g.C, o10 = o00 + (long long)g.W * g.C, o11 = o10 + g.C;
    float sum_v = 0.f, sum_h = 0.f, sum_w = 0.f;
    if (s.inside) {
      for (int c = lane * V; c < g.C; c += 32 * V) {
        const typename Op::T gv = Op::load(gc + c);
        const typename Op::T z = Op::zero();
        const typename Op::T x00 = s.v00 ? Op::load(x + o00 + c) : z;
        const typename Op::T x01 = s.v01 ? Op::load(x + o01 + c) : z;
        const typename Op::T x10 = s.v10 ? Op::load(x + o10 + c) : z;
        const typename Op::T x11 = s.v11 ? Op::load(x + o11 + c) : z;
        const typename Op::T v = Op::fma(w11, x11, Op::fma(w10, x10, Op::fma(w01, x01, Op::scale(w00, x00))));
        const typename Op::T dvh = Op::fma(s.lw, Op::sub(x11, x01), Op::scale(hw, Op::sub(x10, x00)));
        const typename Op::T dvw = Op::fma(s.lh, Op::sub(x11, x10), Op::scale(hh, Op::sub(x01, x00)));
        sum_v += Op::dot(gv, v);
        sum_h += Op::dot(gv, dvh);
        sum_w += Op::dot(gv, dvw);
        const typename Op::T gm = Op::scale(s.m, gv);
        if (s.v00) Op::red(grad_x + o00 + c, Op::scale(w00, gm));
        if (s.v01) Op::red(grad_x + o01 + c, Op::scale(w01, gm));
        if (s.v10) Op::red(grad_x + o10 + c, Op::scale(w10, gm));
        if (s.v11) Op::red(grad_x + o11 + c, Op::scale(w11, gm));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum_v += __shfl_xor_sync(0xffffffffu, sum_v, o);
      sum_h += __shfl_xor_sync(0xffffffffu, sum_h, o);
      sum_w += __shfl_xor_sync(0xffffffffu, sum_w, o);
    }
    if (lane == 0) {
      const long long p = m % HW;
      grad_offset[(s.n * 2 * K + 2 * k) * HW + p] = s.m * sum_h;
      grad_offset[(s.n * 2 * K + 2 * k + 1) * HW + p] = s.m * sum_w;
      grad_mask[(s.n * K + k) * HW + p] = sum_v;
    }
  }
}

int validate(const char* who, int N, int C, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
             int dh, int dw, int n0, int nb) {
  VIDAR_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0 && dh > 0 &&
                    dw > 0,
                "%s: bad sizes N=%d C=%d H=%d W=%d kernel %dx%d stride %dx%d padding %dx%d dilation %dx%d", who, N, C, H, W,
                kh, kw, sh, sw, ph, pw, dh, dw);
  const long long ho = ((long long)H + 2LL * ph - ((long long)dh * (kh - 1) + 1)) / sh + 1;
  const long long wo = ((long long)W + 2LL * pw - ((long long)dw * (kw - 1) + 1)) / sw + 1;
  VIDAR_REQUIRE(Ho > 0 && Wo > 0 && Ho == ho && Wo == wo, "%s: output size %dx%d does not match the convolution (%lldx%lld)",
                who, Ho, Wo, ho, wo);
  VIDAR_REQUIRE(n0 >= 0 && nb >= 0 && (long long)n0 + nb <= N, "%s: bad image range [%d, %d + %d) of %d", who, n0, n0, nb, N);
  VIDAR_REQUIRE((long long)kh * kw * C <= (1LL << 30), "%s: kh * kw * C = %lld is too large", who, (long long)kh * kw * C);
  return VIDAR_OK;
}

int grid_for(long long items) {
  const long long want = (items + kWarps - 1) / kWarps;
  const long long cap = (long long)num_sms() * 16;
  return (int)(want < cap ? want : cap);
}

// The vector kernel when C fills whole 16-byte vectors and the buffers are 16-byte aligned, else the scalar one.
template <typename T>
int im2col(const char* who, const void* x, const void* offset, const void* mask, void* cols, const DcnGeom& g,
           long long items, cudaStream_t st) {
  const T *xt = (const T*)x, *ot = (const T*)offset, *mt = (const T*)mask;
  if (g.C % kVec<T> == 0 && aligned16(x) && aligned16(cols))
    dcn_im2col_kernel<T, kVec<T>><<<grid_for(items), kThreads, 0, st>>>(xt, ot, mt, (T*)cols, g, items);
  else
    dcn_im2col_kernel<T, 1><<<grid_for(items), kThreads, 0, st>>>(xt, ot, mt, (T*)cols, g, items);
  return check_launch(who);
}

template <typename T>
int col2im(const char* who, const void* x, const void* offset, const void* mask, const void* grad_cols, float* grad_x,
           float* grad_offset, float* grad_mask, const DcnGeom& g, long long items, cudaStream_t st) {
  const T *xt = (const T*)x, *ot = (const T*)offset, *mt = (const T*)mask, *gt = (const T*)grad_cols;
  if (g.C % kVec<T> == 0 && aligned16(x) && aligned16(grad_cols) && aligned16(grad_x))
    dcn_col2im_kernel<T, kVec<T>><<<grid_for(items), kThreads, 0, st>>>(xt, ot, mt, gt, grad_x, grad_offset, grad_mask,
                                                                        g, items);
  else
    dcn_col2im_kernel<T, 1><<<grid_for(items), kThreads, 0, st>>>(xt, ot, mt, gt, grad_x, grad_offset, grad_mask, g,
                                                                  items);
  return check_launch(who);
}

int check_dtype(const char* who, int dtype) {
  VIDAR_REQUIRE(dtype == VIDAR_DTYPE_F16 || dtype == VIDAR_DTYPE_BF16, "%s: unsupported dtype %d", who, dtype);
  return VIDAR_OK;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_dcn_im2col(const float* x, const float* offset, const float* mask, float* cols, int N, int C, int H,
                                int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                                int n0, int nb, void* stream) {
  const char* who = "dcn_im2col";
  VIDAR_REQUIRE(x && offset && mask && cols, "%s: null pointer argument", who);
  int rc = validate(who, N, C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0, nb);
  if (rc) return rc;
  if (nb == 0) return VIDAR_OK;
  const DcnGeom g{C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0};
  return im2col<float>(who, x, offset, mask, cols, g, (long long)nb * Ho * Wo * kh * kw, (cudaStream_t)stream);
}

extern "C" int vidar_dcn_im2col_half(const void* x, const void* offset, const void* mask, void* cols, int dtype, int N,
                                     int C, int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw,
                                     int dh, int dw, int n0, int nb, void* stream) {
  const char* who = "dcn_im2col_half";
  VIDAR_REQUIRE(x && offset && mask && cols, "%s: null pointer argument", who);
  int rc = check_dtype(who, dtype);
  if (rc) return rc;
  rc = validate(who, N, C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0, nb);
  if (rc) return rc;
  if (nb == 0) return VIDAR_OK;
  const DcnGeom g{C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0};
  const long long items = (long long)nb * Ho * Wo * kh * kw;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == VIDAR_DTYPE_F16 ? im2col<__half>(who, x, offset, mask, cols, g, items, st)
                                  : im2col<__nv_bfloat16>(who, x, offset, mask, cols, g, items, st);
}

extern "C" int vidar_dcn_col2im(const float* x, const float* offset, const float* mask, const float* grad_cols,
                                float* grad_x, float* grad_offset, float* grad_mask, int N, int C, int H, int W, int Ho,
                                int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int n0, int nb,
                                void* stream) {
  const char* who = "dcn_col2im";
  VIDAR_REQUIRE(x && offset && mask && grad_cols && grad_x && grad_offset && grad_mask, "%s: null pointer argument", who);
  int rc = validate(who, N, C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0, nb);
  if (rc) return rc;
  if (nb == 0) return VIDAR_OK;
  const DcnGeom g{C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0};
  return col2im<float>(who, x, offset, mask, grad_cols, grad_x, grad_offset, grad_mask, g,
                       (long long)nb * Ho * Wo * kh * kw, (cudaStream_t)stream);
}

extern "C" int vidar_dcn_col2im_half(const void* x, const void* offset, const void* mask, const void* grad_cols,
                                     float* grad_x, float* grad_offset, float* grad_mask, int dtype, int N, int C, int H,
                                     int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh,
                                     int dw, int n0, int nb, void* stream) {
  const char* who = "dcn_col2im_half";
  VIDAR_REQUIRE(x && offset && mask && grad_cols && grad_x && grad_offset && grad_mask, "%s: null pointer argument", who);
  int rc = check_dtype(who, dtype);
  if (rc) return rc;
  rc = validate(who, N, C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0, nb);
  if (rc) return rc;
  if (nb == 0) return VIDAR_OK;
  const DcnGeom g{C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, n0};
  const long long items = (long long)nb * Ho * Wo * kh * kw;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == VIDAR_DTYPE_F16
             ? col2im<__half>(who, x, offset, mask, grad_cols, grad_x, grad_offset, grad_mask, g, items, st)
             : col2im<__nv_bfloat16>(who, x, offset, mask, grad_cols, grad_x, grad_offset, grad_mask, g, items, st);
}
