// GridMask (models/utils/grid_mask.py GridMask.forward): out = x * mask, or x * mask + offset * (1 - mask), with the
// mask evaluated in registers instead of being built on the host, rotated by PIL and uploaded.
//
// The reference draws a stripe period d, a stripe length l, starts st_h / st_w and an angle r, writes the stripes
// into a (hh, ww) = (int(1.5 h), int(1.5 w)) mask of ones, rotates it with PIL's `Image.rotate(r)` (nearest, no
// expand, fill 0) and crops the centre (h, w) window at ((hh - h) // 2, (ww - w) // 2).  Pillow's nearest affine
// transform is a 16.16 fixed-point map from output to input pixel; with its coefficients a0..a5 (host code below)
//   xin = (a2 + Y*a1 + X*a0) >> 16,  yin = (a5 + Y*a4 + X*a3) >> 16     (arithmetic shift: floor)
// for the output pixel (Y, X) of the mask frame.  (xin, yin) outside the mask reads 0; inside it reads 0 on a
// stripe and 1 elsewhere, where row yin is on a stripe when use_h, yin >= st_h, (yin - st_h) / d < hh / d and
// (yin - st_h) % d < l (columns likewise with use_w, st_w, ww).  mode 1 inverts the mask.
//
// x / out are contiguous [N, C, h, w]; offset (optional) is one [h, w] plane.  A thread owns V consecutive pixels of
// a plane: it evaluates their mask once and applies it to the same pixels of a run of planes (blockIdx.y, stepping
// by gridDim.y), with 16-byte vectors (4 floats, 8 fp16 / bf16) when h*w is a multiple of V and every buffer is
// 16-byte aligned, one pixel per thread otherwise.  Values are converted to fp32 on load and rounded once on store.
// The mask is 0 or 1, so x * mask and offset * (1 - mask) are exact and their sum rounds once, as the reference's
// separate storage-dtype products and sum do; non-finite inputs propagate the same way (inf * 0 = NaN).
#include <math.h>
#include <stdlib.h>

#include "channel_vec.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr int kPlanesPerThread = 6;   // planes a thread applies its mask to (grid.y = planes / 6, rounded up)
constexpr int kMaxSide = 8192;        // h, w <= 8192: Pillow's 32-bit fixed-point coordinates cannot overflow

struct GridGeom {
  long long a0, a1, a2, a3, a4, a5;   // Pillow's 16.16 affine map, mask-frame output pixel -> input pixel
  int w, hh, ww, oy, ox;              // image width, mask frame, crop origin in the mask frame
  int d, l, st_h, st_w, nh, nw;       // stripe period, length, starts, stripe counts hh / d and ww / d
  int use_h, use_w, mode;
};

// The mask value (0 or 1) of flat pixel p = y * w + x of the image (p < 8192^2: 32-bit division).
__device__ __forceinline__ float mask_at(const GridGeom& g, int p) {
  const long long Y = p / g.w + g.oy, X = p % g.w + g.ox;
  const long long xin = (g.a2 + Y * g.a1 + X * g.a0) >> 16;
  const long long yin = (g.a5 + Y * g.a4 + X * g.a3) >> 16;
  bool one = false;                                                            // PIL's fill outside the mask
  if (xin >= 0 && xin < g.ww && yin >= 0 && yin < g.hh) {
    const int r = (int)yin - g.st_h, c = (int)xin - g.st_w;
    const bool row = g.use_h && r >= 0 && r / g.d < g.nh && r % g.d < g.l;
    const bool col = g.use_w && c >= 0 && c / g.d < g.nw && c % g.d < g.l;
    one = !(row || col);
  }
  return one != (g.mode == 1) ? 1.f : 0.f;
}

template <typename T, int V, bool OFFSET>
__global__ void __launch_bounds__(kThreads) grid_mask_kernel(const T* __restrict__ x, const T* __restrict__ offset,
                                                             T* __restrict__ out, const GridGeom g, long long hw,
                                                             long long planes) {
  using VT = Vec<T, V>;
  const long long p0 = ((long long)blockIdx.x * kThreads + threadIdx.x) * V;
  if (p0 >= hw) return;
  typename VT::T m, keep;                                                       // mask, and offset * (1 - mask)
#pragma unroll
  for (int i = 0; i < V; ++i) lane(m, i) = mask_at(g, (int)p0 + i);
  if (OFFSET) {
    keep = VT::load(offset + p0);
#pragma unroll
    for (int i = 0; i < V; ++i) lane(keep, i) = __fmul_rn(lane(keep, i), 1.f - lane(m, i));
  }
#pragma unroll kPlanesPerThread
  for (long long n = blockIdx.y; n < planes; n += gridDim.y) {
    const long long at = n * hw + p0;
    typename VT::T v = VT::load(x + at);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float y = __fmul_rn(lane(v, i), lane(m, i));
      lane(v, i) = OFFSET ? __fadd_rn(y, lane(keep, i)) : y;
    }
    VT::store(out + at, v);
  }
}

// round(v, 15) of Python: the value printed with 15 decimals (correctly rounded) and read back.
double round15(double v) {
  char buf[64];
  snprintf(buf, sizeof buf, "%.15f", v);
  return strtod(buf, nullptr);
}

long long fix16(double v) { return (long long)floor(v * 65536.0 + 0.5); }

// a*x + b*y with both products rounded before the sum, as Python evaluates it (never contracted into an fma).
double dot2(double a, double x, double b, double y) {
  volatile double p = a * x, q = b * y;
  return p + q;
}

// Pillow's `Image.rotate(r)` of a (hh, ww) image as the fixed-point map of its nearest affine transform: the inverse
// rotation about (ww / 2, hh / 2) with entries rounded to 15 decimals, in fp64 in Pillow's order of operations, then
// converted to 16.16 with the half-pixel centre folded into the translation.  Angles 0 and 180 (and 90 / 270 of a
// square) take Pillow's copy / transpose shortcuts, which this map reproduces pixel for pixel.
void pillow_rotation(int r, int hh, int ww, GridGeom& g) {
  const double angle = -((double)(((r % 360) + 360) % 360) * (M_PI / 180.0));
  const double m0 = round15(cos(angle)), m1 = round15(sin(angle)), m3 = round15(-sin(angle)), m4 = round15(cos(angle));
  const double cx = ww / 2.0, cy = hh / 2.0;
  const double m2 = (dot2(m0, -cx, m1, -cy) + 0.0) + cx;
  const double m5 = (dot2(m3, -cx, m4, -cy) + 0.0) + cy;
  g.a0 = fix16(m0);
  g.a1 = fix16(m1);
  g.a3 = fix16(m3);
  g.a4 = fix16(m4);
  g.a2 = fix16(m2 + m0 * 0.5 + m1 * 0.5);
  g.a5 = fix16(m5 + m3 * 0.5 + m4 * 0.5);
}

template <typename T>
int apply(const char* who, const void* x, const void* offset, void* out, const GridGeom& g, long long hw,
          long long planes, cudaStream_t st) {
  const bool vec = hw % kVec<T> == 0 && aligned16(x) && aligned16(out) && (!offset || aligned16(offset));
  const int V = vec ? kVec<T> : 1;
  const long long blocks = (hw / V + kThreads - 1) / kThreads;
  VIDAR_REQUIRE(blocks < (1LL << 31), "%s: %lld pixels per plane is too many", who, hw);
  long long gy = (planes + kPlanesPerThread - 1) / kPlanesPerThread;
  gy = gy < 65535 ? gy : 65535;
  const dim3 grid((unsigned)blocks, (unsigned)gy);
  const T *xi = (const T*)x, *oi = (const T*)offset;
  T* o = (T*)out;
  if (vec && offset) grid_mask_kernel<T, kVec<T>, true><<<grid, kThreads, 0, st>>>(xi, oi, o, g, hw, planes);
  else if (vec) grid_mask_kernel<T, kVec<T>, false><<<grid, kThreads, 0, st>>>(xi, oi, o, g, hw, planes);
  else if (offset) grid_mask_kernel<T, 1, true><<<grid, kThreads, 0, st>>>(xi, oi, o, g, hw, planes);
  else grid_mask_kernel<T, 1, false><<<grid, kThreads, 0, st>>>(xi, oi, o, g, hw, planes);
  return check_launch(who);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_grid_mask_apply(const void* x, const void* offset, void* out, int dtype, int N, int C, int h,
                                     int w, int d, int l, int st_h, int st_w, int r, int use_h, int use_w, int mode,
                                     void* stream) {
  const char* who = "grid_mask_apply";
  VIDAR_REQUIRE(x && out, "%s: null pointer argument", who);
  VIDAR_REQUIRE(dtype == VIDAR_DTYPE_F32 || dtype == VIDAR_DTYPE_F16 || dtype == VIDAR_DTYPE_BF16,
                "%s: unsupported dtype %d", who, dtype);
  VIDAR_REQUIRE(N >= 0 && C >= 0 && h > 0 && w > 0 && h <= kMaxSide && w <= kMaxSide,
                "%s: bad sizes (N %d, C %d, h %d, w %d; h and w must be in [1, %d])", who, N, C, h, w, kMaxSide);
  VIDAR_REQUIRE(d >= 2 && l >= 0 && l <= d && st_h >= 0 && st_h < d && st_w >= 0 && st_w < d,
                "%s: bad draw (d %d, l %d, st_h %d, st_w %d; need d >= 2, 0 <= l <= d, 0 <= st_h, st_w < d)", who, d,
                l, st_h, st_w);
  VIDAR_REQUIRE((use_h == 0 || use_h == 1) && (use_w == 0 || use_w == 1) && (mode == 0 || mode == 1),
                "%s: use_h, use_w and mode must be 0 or 1 (got %d, %d, %d)", who, use_h, use_w, mode);
  const size_t esize = dtype == VIDAR_DTYPE_F32 ? 4 : 2;
  VIDAR_REQUIRE((uintptr_t)x % esize == 0 && (uintptr_t)out % esize == 0 && (uintptr_t)offset % esize == 0,
                "%s: x, offset and out must be aligned to their %zu-byte elements", who, esize);
  const long long planes = (long long)N * C, hw = (long long)h * w;
  if (planes == 0) return VIDAR_OK;
  GridGeom g{};
  g.w = w;
  g.hh = h + h / 2;                                       // int(1.5 * h)
  g.ww = w + w / 2;
  g.oy = (g.hh - h) / 2;
  g.ox = (g.ww - w) / 2;
  g.d = d;
  g.l = l;
  g.st_h = st_h;
  g.st_w = st_w;
  g.nh = g.hh / d;
  g.nw = g.ww / d;
  g.use_h = use_h;
  g.use_w = use_w;
  g.mode = mode;
  pillow_rotation(r, g.hh, g.ww, g);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == VIDAR_DTYPE_F32) return apply<float>(who, x, offset, out, g, hw, planes, st);
  if (dtype == VIDAR_DTYPE_F16) return apply<__half>(who, x, offset, out, g, hw, planes, st);
  return apply<__nv_bfloat16>(who, x, offset, out, g, hw, planes, st);
}
