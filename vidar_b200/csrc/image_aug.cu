// The multi-view image pipelines of ViDAR's configs (datasets/pipelines/transform_3d.py, augmentation.py), from one
// frame's uint8 BGR images [N, H, W, 3] to the network's float32 [N, 3, Hp, Wp], bit for bit the reference's cv2 /
// PIL / numpy statements:
//   * PhotoMetricDistortionMultiViewImage -> CropResizeFlipImage (crop, then resize) or RandomCropResizeFlipImage
//     (resize, then crop) -> NormalizeMultiviewImage -> PadMultiViewImage, in two launches (vidar_image_aug_apply);
//   * PhotoMetricDistortionMultiViewImage (optional) -> NormalizeMultiviewImage -> PadMultiViewImage, in one launch
//     on the unclamped float32 photometric output (vidar_image_aug_normalize);
//   * the OpenScene configs' PhotoMetricDistortionMultiViewImage (optional) -> NormalizeMultiviewImage ->
//     RandomScaleImageMultiViewImage(scales=[2/3]) -> PadMultiViewImage, in one launch (vidar_image_aug_scale).
//
// Pass 1 (one block per cropped row and image): every source pixel of the row gets the photometric float32 math
// once -- brightness x + delta, contrast x * alpha (before the HSV round trip in mode 1, after it in mode 0),
// cv2's float BGR <-> HSV with its fused multiply-adds, saturation, hue with its wrap, the channel permutation --
// and numpy's wrapping cast to uint8 (truncation toward zero, low 8 bits), into shared memory; pixels of the crop
// box outside the image are 0, as PIL's crop fills them.  Then Pillow's horizontal bicubic pass (22-bit integer
// taps, accumulator from 1 << 21, >> 22, clamp) writes the uint8 intermediate [N, crop_h, mid_w, 3], or the
// staged row as is when Pillow skips that pass (out_w == crop_w).  Only the resized columns inside the window
// (below) are computed: mid_w of them, from column mid_x = max(win_x, 0) on.
// Pass 2 (one block per output row and image): Pillow's vertical pass (skipped when out_h == crop_h) for the
// resized rows inside the window, the window itself -- PIL's crop of the resized image, 0 outside it -- the
// left-right flip, the optional BGR -> RGB swap, mmcv's imnormalize (x - mean in float32, then the product with
// 1/std in double rounded to float32), the bottom / right padding and the HWC -> CHW transpose, one plane at a
// time so that a warp's stores are contiguous.  CropResizeFlipImage's window is the whole resized image.
//
// Every float operation is an explicit __f*_rn intrinsic, so nvcc cannot contract a product and a sum into an FMA
// that cv2 does not use; the ones cv2's vector code fuses are __fmaf_rn.  The taps are computed on the host in
// float64 by Pillow's rules (vidar_b200/image_aug.py) and read from global memory.
#include <float.h>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxImages = 64;        // per-image draws travel in the kernel arguments
constexpr int kMaxSide = 8192;

struct Photo {
  float delta, alpha, sat, hue;       // brightness delta, contrast factor, saturation factor, hue delta
  int flags;                          // bit 0 brightness, 1 contrast, 2 saturation, 3 hue, 4 contrast first (mode 1)
  int perm[3];                        // output channel c takes input channel perm[c]
};

struct Geom {
  int H, W, cx, cy, cw, ch, ow, oh, wx, wy, ww, wh, mx, mw, Hp, Wp, hk, vk, flip, to_rgb;
  float mean[3], pad[3];
  double stdinv[3];
};

struct Photos {
  Photo p[kMaxImages];
};

__device__ __forceinline__ unsigned char wrap_u8(float x) {
  return (unsigned char)(__float2int_rz(x) & 255);
}

// cv2.cvtColor(BGR2HSV) on float32 (its vector path): h in degrees, s, v.
__device__ __forceinline__ void bgr2hsv(float b, float g, float r, float& h, float& s, float& v) {
  v = fmaxf(fmaxf(r, g), b);
  const float diff = __fsub_rn(v, fminf(fminf(r, g), b));
  s = __fdiv_rn(diff, __fadd_rn(fabsf(v), FLT_EPSILON));
  const float d = __fdiv_rn(60.f, __fadd_rn(diff, FLT_EPSILON));
  if (v == r) {
    h = __fmaf_rn(__fsub_rn(g, b), d, 0.f);
    if (h < 0.f) h = __fmaf_rn(__fsub_rn(g, b), d, 360.f);
  } else if (v == g) {
    h = __fmaf_rn(__fsub_rn(b, r), d, 120.f);
  } else {
    h = __fmaf_rn(__fsub_rn(r, g), d, 240.f);
  }
}

// cv2.cvtColor(HSV2BGR) on float32 with h in degrees.
__device__ __forceinline__ void hsv2bgr(float h, float s, float v, float out[3]) {
  if (s == 0.f) {
    out[0] = out[1] = out[2] = v;
    return;
  }
  h = __fmul_rn(h, 6.f / 360.f);
  while (h < 0.f) h = __fadd_rn(h, 6.f);
  while (h >= 6.f) h = __fsub_rn(h, 6.f);
  int sector = __float2int_rd(h);
  h = __fsub_rn(h, (float)sector);
  if ((unsigned)sector >= 6u) {
    sector = 0;
    h = 0.f;
  }
  const float t0 = v, t1 = __fmul_rn(v, __fsub_rn(1.f, s)), t2 = __fmul_rn(v, __fmaf_rn(-s, h, 1.f)),
              t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, h), 1.f));
  // OpenCV's sector table {{1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}}: 2 bits per entry, 6 per sector
  constexpr unsigned long long kSectors = 13ull | 33ull << 6 | 19ull << 12 | 24ull << 18 | 52ull << 24 | 6ull << 30;
  const unsigned e = (unsigned)(kSectors >> (6 * sector));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const unsigned i = (e >> (2 * c)) & 3u;
    out[c] = i == 0 ? t0 : i == 1 ? t1 : i == 2 ? t2 : t3;
  }
}

// PhotoMetricDistortionMultiViewImage's float32 statements on one BGR pixel, channel permutation included.
__device__ __forceinline__ void photometric(const Photo& p, const unsigned char* in, float out[3]) {
  float x[3] = {(float)in[0], (float)in[1], (float)in[2]};
  if (p.flags & 1) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(x[c], p.delta);
  }
  if ((p.flags & 2) && (p.flags & 16)) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __fmul_rn(x[c], p.alpha);
  }
  float h, s, v;
  bgr2hsv(x[0], x[1], x[2], h, s, v);
  if (p.flags & 4) s = __fmul_rn(s, p.sat);
  if (p.flags & 8) {
    h = __fadd_rn(h, p.hue);
    if (h > 360.f) h = __fsub_rn(h, 360.f);
    if (h < 0.f) h = __fadd_rn(h, 360.f);
  }
  hsv2bgr(h, s, v, x);
  if ((p.flags & 2) && !(p.flags & 16)) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __fmul_rn(x[c], p.alpha);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = x[p.perm[c]];
}

// The photometric statements, then np.uint8.
__device__ __forceinline__ void distort(const Photo& p, const unsigned char* in, unsigned char* out) {
  float x[3];
  photometric(p, in, x);
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = wrap_u8(x[c]);
}

// mmcv's imnormalize of one pixel: the optional BGR -> RGB swap, x - mean in float32, times 1/std in double.
__device__ __forceinline__ void normalize(const Geom& g, const float px[3], float v[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float val = px[g.to_rgb ? 2 - c : c];
    v[c] = __double2float_rn(__dmul_rn((double)__fsub_rn(val, g.mean[c]), g.stdinv[c]));
  }
}

__device__ __forceinline__ unsigned char clip8(int acc) {
  return (unsigned char)min(max(acc >> 22, 0), 255);
}

// Pass 1: photometric + cast of one cropped source row into shared memory, then the horizontal taps.
template <bool PHOTO, bool HORIZ>
__global__ void __launch_bounds__(kThreads) image_aug_rows_kernel(const unsigned char* __restrict__ src,
                                                                  unsigned char* __restrict__ mid,
                                                                  const int* __restrict__ htaps, const Geom g,
                                                                  const Photos photos) {
  extern __shared__ unsigned char row[];                      // [cw, 3]
  const int y = blockIdx.x, n = blockIdx.y, sy = g.cy + y;
  const bool inside = sy >= 0 && sy < g.H;
  const unsigned char* in = src + ((long long)n * g.H + (inside ? sy : 0)) * g.W * 3;
  for (int x = threadIdx.x; x < g.cw; x += kThreads) {
    const int sx = g.cx + x;
    unsigned char* o = row + 3 * x;
    if (inside && sx >= 0 && sx < g.W) {
      const unsigned char* p = in + 3 * sx;
      if (PHOTO) {
        distort(photos.p[n], p, o);
      } else {
        o[0] = p[0];
        o[1] = p[1];
        o[2] = p[2];
      }
    } else {
      o[0] = o[1] = o[2] = 0;
    }
  }
  __syncthreads();
  unsigned char* out = mid + ((long long)n * g.ch + y) * g.mw * 3;
  for (int x = threadIdx.x; x < g.mw; x += kThreads) {
    const int rx = g.mx + x;
    if (HORIZ) {
      const int* t = htaps + (long long)rx * (2 + g.hk);
      const int x0 = __ldg(t), cnt = __ldg(t + 1);
      int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
      for (int k = 0; k < cnt; ++k) {
        const int w = __ldg(t + 2 + k);
        const unsigned char* p = row + 3 * (x0 + k);
        a0 += p[0] * w;
        a1 += p[1] * w;
        a2 += p[2] * w;
      }
      out[3 * x] = clip8(a0);
      out[3 * x + 1] = clip8(a1);
      out[3 * x + 2] = clip8(a2);
    } else {
      out[3 * x] = row[3 * rx];
      out[3 * x + 1] = row[3 * rx + 1];
      out[3 * x + 2] = row[3 * rx + 2];
    }
  }
}

// Pass 2: vertical taps, window, flip, channel order, normalisation and padding of one output row, written as CHW.
template <bool VERT>
__global__ void __launch_bounds__(kThreads) image_aug_cols_kernel(const unsigned char* __restrict__ mid,
                                                                  float* __restrict__ out,
                                                                  const int* __restrict__ vtaps, const Geom g) {
  const int y = blockIdx.x, n = blockIdx.y, ry = g.wy + y;
  const long long plane = (long long)g.Hp * g.Wp;
  float* o = out + (long long)n * 3 * plane + (long long)y * g.Wp;
  const bool row_in = y < g.wh;                               // inside the window
  const bool row_img = row_in && ry >= 0 && ry < g.oh;        // and inside the resized image
  int y0 = ry, cnt = 1;
  const int* t = nullptr;
  if (VERT && row_img) {
    t = vtaps + (long long)ry * (2 + g.vk);
    y0 = __ldg(t);
    cnt = __ldg(t + 1);
  }
  const unsigned char* base = mid + (long long)n * g.ch * g.mw * 3;
  for (int x = threadIdx.x; x < g.Wp; x += kThreads) {
    float v[3] = {g.pad[0], g.pad[1], g.pad[2]};
    if (row_in && x < g.ww) {
      const int rx = g.wx + (g.flip ? g.ww - 1 - x : x);
      float px[3] = {0.f, 0.f, 0.f};
      if (row_img && rx >= 0 && rx < g.ow) {
        const int xs = rx - g.mx;
        if (VERT) {
          int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
          for (int k = 0; k < cnt; ++k) {
            const int w = __ldg(t + 2 + k);
            const unsigned char* p = base + ((long long)(y0 + k) * g.mw + xs) * 3;
            a0 += p[0] * w;
            a1 += p[1] * w;
            a2 += p[2] * w;
          }
          px[0] = clip8(a0);
          px[1] = clip8(a1);
          px[2] = clip8(a2);
        } else {
          const unsigned char* p = base + ((long long)y0 * g.mw + xs) * 3;
          px[0] = p[0];
          px[1] = p[1];
          px[2] = p[2];
        }
      }
      normalize(g, px, v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane + x] = v[c];
  }
}

// The chain without a crop step: the photometric statements (when PHOTO) on the float32 pixels with no uint8 cast,
// normalisation and padding of one output row, written as CHW.
template <bool PHOTO>
__global__ void __launch_bounds__(kThreads) image_aug_normalize_kernel(const unsigned char* __restrict__ src,
                                                                       float* __restrict__ out, const Geom g,
                                                                       const Photos photos) {
  const int y = blockIdx.x, n = blockIdx.y;
  const long long plane = (long long)g.Hp * g.Wp;
  float* o = out + (long long)n * 3 * plane + (long long)y * g.Wp;
  const unsigned char* in = src + ((long long)n * g.H + min(y, g.H - 1)) * g.W * 3;
  for (int x = threadIdx.x; x < g.Wp; x += kThreads) {
    float v[3] = {g.pad[0], g.pad[1], g.pad[2]};
    if (y < g.H && x < g.W) {
      const unsigned char* p = in + 3 * x;
      float px[3];
      if (PHOTO) {
        photometric(photos.p[n], p, px);
      } else {
        px[0] = p[0];
        px[1] = p[1];
        px[2] = p[2];
      }
      normalize(g, px, v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane + x] = v[c];
  }
}

// The OpenScene chain (RandomScaleImageMultiViewImage after the normalisation): the photometric statements (when
// PHOTO) on float32, the normalisation, then mmcv.imresize -- cv2.resize INTER_LINEAR on float32 HWC -- by 2/3, then
// the padding, for one output row, written as CHW.  At a 3:2 ratio output pixel d reads source pixels floor(1.5 d)
// and the next one with weight 0.25 (d even) or 0.75 (d odd), never past the last one.  cv2 with IPP, as the
// package's wheel ships it, interpolates each of the two source rows along x first and then between them, each
// step a + t * (b - a) with one fused multiply-add; the source pixels are recomputed for each output pixel that
// reads them.
template <bool PHOTO>
__device__ __forceinline__ void scale_source(const Geom& g, const Photo& p, const unsigned char* px, float v[3]) {
  float x[3];
  if (PHOTO) {
    photometric(p, px, x);
  } else {
    x[0] = px[0];
    x[1] = px[1];
    x[2] = px[2];
  }
  normalize(g, x, v);
}

template <bool PHOTO>
__global__ void __launch_bounds__(kThreads) image_aug_scale_kernel(const unsigned char* __restrict__ src,
                                                                   float* __restrict__ out, const Geom g,
                                                                   const Photos photos) {
  const int y = blockIdx.x, n = blockIdx.y;
  const long long plane = (long long)g.Hp * g.Wp;
  float* o = out + (long long)n * 3 * plane + (long long)y * g.Wp;
  const bool row_in = y < g.oh;
  const int sy = (3 * y) >> 1;
  const float fy = (y & 1) ? 0.75f : 0.25f;
  const unsigned char* r0 = src + ((long long)n * g.H + (row_in ? sy : 0)) * g.W * 3;
  const unsigned char* r1 = r0 + (row_in ? (long long)g.W * 3 : 0);
  const Photo& p = photos.p[n];
  for (int x = threadIdx.x; x < g.Wp; x += kThreads) {
    float v[3] = {g.pad[0], g.pad[1], g.pad[2]};
    if (row_in && x < g.ow) {
      const int sx = (3 * x) >> 1;
      const float fx = (x & 1) ? 0.75f : 0.25f;
      float a0[3], a1[3], b0[3], b1[3];
      scale_source<PHOTO>(g, p, r0 + 3 * sx, a0);
      scale_source<PHOTO>(g, p, r0 + 3 * sx + 3, a1);
      scale_source<PHOTO>(g, p, r1 + 3 * sx, b0);
      scale_source<PHOTO>(g, p, r1 + 3 * sx + 3, b1);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float h0 = __fmaf_rn(fx, __fsub_rn(a1[c], a0[c]), a0[c]);
        const float h1 = __fmaf_rn(fx, __fsub_rn(b1[c], b0[c]), b0[c]);
        v[c] = __fmaf_rn(fy, __fsub_rn(h1, h0), h0);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane + x] = v[c];
  }
}

// photo_i / photo_f (host) -> the kernel-argument copy of the draws, after checking them.
int read_photos(const char* who, int N, const int32_t* photo_i, const float* photo_f, Photos& photos) {
  for (int n = 0; n < N; ++n) {
    const int32_t* pi = photo_i + 8 * n;
    const float* pf = photo_f + 4 * n;
    int flags = 0;
    for (int k = 0; k < 5; ++k) {
      VIDAR_REQUIRE(pi[k] == 0 || pi[k] == 1, "%s: image %d: photometric flag %d is %d (need 0 or 1)", who, n, k,
                    pi[k]);
      flags |= pi[k] << k;
    }
    const int a = pi[5], b = pi[6], c = pi[7];
    VIDAR_REQUIRE(a >= 0 && a < 3 && b >= 0 && b < 3 && c >= 0 && c < 3 && a != b && b != c && a != c,
                  "%s: image %d: (%d, %d, %d) is not a permutation of (0, 1, 2)", who, n, a, b, c);
    photos.p[n] = Photo{pf[0], pf[1], pf[2], pf[3], flags, {a, b, c}};
  }
  return VIDAR_OK;
}

void set_norm(Geom& g, const float* mean, const double* stdinv, const float* pad_val) {
  for (int c = 0; c < 3; ++c) {
    g.mean[c] = mean[c];
    g.stdinv[c] = stdinv[c];
    g.pad[c] = pad_val[c];
  }
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_image_aug_apply(const unsigned char* src, unsigned char* mid, float* out, int N, int H, int W,
                                     const int32_t* photo_i, const float* photo_f, int crop_x, int crop_y,
                                     int crop_w, int crop_h, int out_w, int out_h, int win_x, int win_y, int win_w,
                                     int win_h, const int32_t* htaps, int hk, const int32_t* vtaps, int vk, int flip,
                                     int to_rgb, const float* mean, const double* stdinv, const float* pad_val, int Hp,
                                     int Wp, void* stream) {
  const char* who = "image_aug_apply";
  VIDAR_REQUIRE(src && mid && out && mean && stdinv && pad_val, "%s: null pointer argument", who);
  VIDAR_REQUIRE(N >= 1 && N <= kMaxImages, "%s: %d images per call (need 1..%d)", who, N, kMaxImages);
  VIDAR_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide && crop_w >= 1 && crop_h >= 1 &&
                    crop_w <= kMaxSide && crop_h <= kMaxSide && out_w >= 1 && out_h >= 1 && out_w <= kMaxSide &&
                    out_h <= kMaxSide && win_w >= 1 && win_h >= 1 && win_w <= kMaxSide && win_h <= kMaxSide &&
                    Hp >= win_h && Wp >= win_w && Hp <= kMaxSide && Wp <= kMaxSide,
                "%s: bad sizes (image %d x %d, crop %d x %d, out %d x %d, window %d x %d, padded %d x %d; sides in "
                "[1, %d], padded at least the window)", who, H, W, crop_h, crop_w, out_h, out_w, win_h, win_w, Hp, Wp,
                kMaxSide);
  VIDAR_REQUIRE(crop_x > -kMaxSide && crop_y > -kMaxSide && crop_x < kMaxSide && crop_y < kMaxSide,
                "%s: crop origin (%d, %d) out of range", who, crop_x, crop_y);
  const int mid_x = max(win_x, 0), mid_w = min(win_x + win_w, out_w) - mid_x;
  VIDAR_REQUIRE(win_x > -kMaxSide && win_y > -kMaxSide && mid_w >= 1 && win_y < out_h && win_y + win_h > 0,
                "%s: window (%d, %d) + (%d x %d) does not overlap the resized %d x %d image", who, win_x, win_y,
                win_w, win_h, out_w, out_h);
  VIDAR_REQUIRE((out_w == crop_w) == (htaps == nullptr) && (out_h == crop_h) == (vtaps == nullptr),
                "%s: tap tables must be given exactly for the axes whose size changes", who);
  VIDAR_REQUIRE((!htaps || hk >= 1) && (!vtaps || vk >= 1), "%s: bad tap counts (%d, %d)", who, hk, vk);
  VIDAR_REQUIRE((flip == 0 || flip == 1) && (to_rgb == 0 || to_rgb == 1), "%s: flip and to_rgb must be 0 or 1", who);
  VIDAR_REQUIRE((photo_i == nullptr) == (photo_f == nullptr), "%s: photo_i and photo_f go together", who);
  Photos photos{};
  if (photo_i) {
    const int rc = read_photos(who, N, photo_i, photo_f, photos);
    if (rc != VIDAR_OK) return rc;
  }
  Geom g{};
  g.H = H; g.W = W; g.cx = crop_x; g.cy = crop_y; g.cw = crop_w; g.ch = crop_h; g.ow = out_w; g.oh = out_h;
  g.wx = win_x; g.wy = win_y; g.ww = win_w; g.wh = win_h; g.mx = mid_x; g.mw = mid_w;
  g.Hp = Hp; g.Wp = Wp; g.hk = hk; g.vk = vk; g.flip = flip; g.to_rgb = to_rgb;
  set_norm(g, mean, stdinv, pad_val);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)crop_w * 3;
  const dim3 g1((unsigned)crop_h, (unsigned)N), g2((unsigned)Hp, (unsigned)N);
  const int* ht = (const int*)htaps;
  if (photo_i && htaps) image_aug_rows_kernel<true, true><<<g1, kThreads, smem, st>>>(src, mid, ht, g, photos);
  else if (photo_i) image_aug_rows_kernel<true, false><<<g1, kThreads, smem, st>>>(src, mid, ht, g, photos);
  else if (htaps) image_aug_rows_kernel<false, true><<<g1, kThreads, smem, st>>>(src, mid, ht, g, photos);
  else image_aug_rows_kernel<false, false><<<g1, kThreads, smem, st>>>(src, mid, ht, g, photos);
  int rc = check_launch(who);
  if (rc != VIDAR_OK) return rc;
  if (vtaps) image_aug_cols_kernel<true><<<g2, kThreads, 0, st>>>(mid, out, (const int*)vtaps, g);
  else image_aug_cols_kernel<false><<<g2, kThreads, 0, st>>>(mid, out, nullptr, g);
  return check_launch(who);
}

extern "C" int vidar_image_aug_normalize(const unsigned char* src, float* out, int N, int H, int W,
                                         const int32_t* photo_i, const float* photo_f, int to_rgb, const float* mean,
                                         const double* stdinv, const float* pad_val, int Hp, int Wp, void* stream) {
  const char* who = "image_aug_normalize";
  VIDAR_REQUIRE(src && out && mean && stdinv && pad_val, "%s: null pointer argument", who);
  VIDAR_REQUIRE(N >= 1 && N <= kMaxImages, "%s: %d images per call (need 1..%d)", who, N, kMaxImages);
  VIDAR_REQUIRE(H >= 1 && W >= 1 && Hp >= H && Wp >= W && Hp <= kMaxSide && Wp <= kMaxSide,
                "%s: bad sizes (image %d x %d, padded %d x %d; sides in [1, %d], padded at least the image)", who, H,
                W, Hp, Wp, kMaxSide);
  VIDAR_REQUIRE(to_rgb == 0 || to_rgb == 1, "%s: to_rgb must be 0 or 1", who);
  VIDAR_REQUIRE((photo_i == nullptr) == (photo_f == nullptr), "%s: photo_i and photo_f go together", who);
  Photos photos{};
  if (photo_i) {
    const int rc = read_photos(who, N, photo_i, photo_f, photos);
    if (rc != VIDAR_OK) return rc;
  }
  Geom g{};
  g.H = H; g.W = W; g.Hp = Hp; g.Wp = Wp; g.to_rgb = to_rgb;
  set_norm(g, mean, stdinv, pad_val);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)Hp, (unsigned)N);
  if (photo_i) image_aug_normalize_kernel<true><<<grid, kThreads, 0, st>>>(src, out, g, photos);
  else image_aug_normalize_kernel<false><<<grid, kThreads, 0, st>>>(src, out, g, photos);
  return check_launch(who);
}

extern "C" int vidar_image_aug_scale(const unsigned char* src, float* out, int N, int H, int W,
                                     const int32_t* photo_i, const float* photo_f, int to_rgb, const float* mean,
                                     const double* stdinv, const float* pad_val, int out_h, int out_w, int Hp, int Wp,
                                     void* stream) {
  const char* who = "image_aug_scale";
  VIDAR_REQUIRE(src && out && mean && stdinv && pad_val, "%s: null pointer argument", who);
  VIDAR_REQUIRE(N >= 1 && N <= kMaxImages, "%s: %d images per call (need 1..%d)", who, N, kMaxImages);
  VIDAR_REQUIRE(H >= 3 && W >= 3 && H <= kMaxSide && W <= kMaxSide && 2 * H == 3 * out_h && 2 * W == 3 * out_w,
                "%s: image %d x %d to %d x %d: only a scale of 2/3 on sides divisible by 3 is supported", who, H, W,
                out_h, out_w);
  VIDAR_REQUIRE(Hp >= out_h && Wp >= out_w && Hp <= kMaxSide && Wp <= kMaxSide,
                "%s: padded size %d x %d must hold the %d x %d image and be at most %d", who, Hp, Wp, out_h, out_w,
                kMaxSide);
  VIDAR_REQUIRE(to_rgb == 0 || to_rgb == 1, "%s: to_rgb must be 0 or 1", who);
  VIDAR_REQUIRE((photo_i == nullptr) == (photo_f == nullptr), "%s: photo_i and photo_f go together", who);
  Photos photos{};
  if (photo_i) {
    const int rc = read_photos(who, N, photo_i, photo_f, photos);
    if (rc != VIDAR_OK) return rc;
  }
  Geom g{};
  g.H = H; g.W = W; g.oh = out_h; g.ow = out_w; g.Hp = Hp; g.Wp = Wp; g.to_rgb = to_rgb;
  set_norm(g, mean, stdinv, pad_val);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)Hp, (unsigned)N);
  if (photo_i) image_aug_scale_kernel<true><<<grid, kThreads, 0, st>>>(src, out, g, photos);
  else image_aug_scale_kernel<false><<<grid, kThreads, 0, st>>>(src, out, g, photos);
  return check_launch(who);
}
