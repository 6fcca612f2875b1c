// Channel vectors of a channel-last feature map, shared by the deformable sampling kernels (dcn.cu, dcnv3.cu) and,
// as vectors of consecutive pixels of one plane, by the GridMask kernel (grid_mask.cu).
//
// Storage type T is float, __half or __nv_bfloat16.  Every value is converted to fp32 on load (`to_f`) and rounded
// once on a 16-bit store (`store1`).  Vec<T, V> handles V consecutive channels as fp32 values in registers:
//   Vec<float, 4>  one 16-byte float4, red into fp32 with one red.global.add.v4.f32
//   Vec<T, 1>      one channel of any storage type, red.global.add.f32
//   Vec<T, 8>      eight 16-bit channels in one 16-byte load / store, two float4 in registers, two v4 reds
// kVec<T> is the 16-byte width of T.  The vector forms need 16-byte aligned addresses.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace vidar {

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ void store1(float* p, float v) { *p = v; }
__device__ __forceinline__ void store1(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void store1(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// V channels of storage type T as fp32 values: load / store convert, red adds into an fp32 buffer.
template <typename T, int V> struct Vec;
template <> struct Vec<float, 4> {
  using T = float4;
  static __device__ __forceinline__ T load(const float* p) { return ldg4(p); }
  static __device__ __forceinline__ void store(float* p, T v) { *reinterpret_cast<float4*>(p) = v; }
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ T fma(float a, T x, T y) {
    return make_float4(fmaf(a, x.x, y.x), fmaf(a, x.y, y.y), fmaf(a, x.z, y.z), fmaf(a, x.w, y.w));
  }
  static __device__ __forceinline__ T scale(float a, T x) { return make_float4(a * x.x, a * x.y, a * x.z, a * x.w); }
  static __device__ __forceinline__ T sub(T a, T b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
  static __device__ __forceinline__ float dot(T a, T b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
  static __device__ __forceinline__ void red(float* p, T v) { red_add_v4(p, v); }
};
template <typename S> struct Vec<S, 1> {
  using T = float;
  static __device__ __forceinline__ T load(const S* p) { return to_f(__ldg(p)); }
  static __device__ __forceinline__ void store(S* p, T v) { store1(p, v); }
  static __device__ __forceinline__ T zero() { return 0.f; }
  static __device__ __forceinline__ T fma(float a, T x, T y) { return fmaf(a, x, y); }
  static __device__ __forceinline__ T scale(float a, T x) { return a * x; }
  static __device__ __forceinline__ T sub(T a, T b) { return a - b; }
  static __device__ __forceinline__ float dot(T a, T b) { return a * b; }
  static __device__ __forceinline__ void red(float* p, T v) { red_add_f32(p, v); }
};

// Eight 16-bit channels: one 16-byte load / store (a uint4 holding four half2 / bfloat162 pairs), two fp32 float4s
// in registers, two red.global.add.v4.f32 into the fp32 gradient.
struct F8 {
  float4 a, b;
};
template <typename S> struct Pair;
template <> struct Pair<__half> {
  static __device__ __forceinline__ float2 unpack(unsigned u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }
  static __device__ __forceinline__ unsigned pack(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<unsigned*>(&h);
  }
};
template <> struct Pair<__nv_bfloat16> {
  static __device__ __forceinline__ float2 unpack(unsigned u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  }
  static __device__ __forceinline__ unsigned pack(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<unsigned*>(&h);
  }
};
template <typename S> struct Vec<S, 8> {
  using T = F8;
  using V4 = Vec<float, 4>;
  static __device__ __forceinline__ T load(const S* p) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    const float2 q0 = Pair<S>::unpack(u.x), q1 = Pair<S>::unpack(u.y), q2 = Pair<S>::unpack(u.z), q3 = Pair<S>::unpack(u.w);
    return {make_float4(q0.x, q0.y, q1.x, q1.y), make_float4(q2.x, q2.y, q3.x, q3.y)};
  }
  static __device__ __forceinline__ void store(S* p, T v) {
    *reinterpret_cast<uint4*>(p) = make_uint4(Pair<S>::pack(v.a.x, v.a.y), Pair<S>::pack(v.a.z, v.a.w),
                                              Pair<S>::pack(v.b.x, v.b.y), Pair<S>::pack(v.b.z, v.b.w));
  }
  static __device__ __forceinline__ T zero() { return {V4::zero(), V4::zero()}; }
  static __device__ __forceinline__ T fma(float a, T x, T y) { return {V4::fma(a, x.a, y.a), V4::fma(a, x.b, y.b)}; }
  static __device__ __forceinline__ T scale(float a, T x) { return {V4::scale(a, x.a), V4::scale(a, x.b)}; }
  static __device__ __forceinline__ T sub(T a, T b) { return {V4::sub(a.a, b.a), V4::sub(a.b, b.b)}; }
  static __device__ __forceinline__ float dot(T a, T b) { return V4::dot(a.a, b.a) + V4::dot(a.b, b.b); }
  static __device__ __forceinline__ void red(float* p, T v) {
    red_add_v4(p, v.a);
    red_add_v4(p + 4, v.b);
  }
};

// Element i of a register vector of Vec<T, V> (float, float4 or F8); i is a compile-time constant once the caller's
// loop over the V elements is unrolled, so the vector stays in registers.
__device__ __forceinline__ float& lane(float& v, int) { return v; }
__device__ __forceinline__ float& lane(float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }
__device__ __forceinline__ float& lane(F8& v, int i) { return i < 4 ? lane(v.a, i) : lane(v.b, i - 4); }

// The vector width of storage type T: 16 bytes.
template <typename T> constexpr int kVec = 16 / sizeof(T);

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace vidar
