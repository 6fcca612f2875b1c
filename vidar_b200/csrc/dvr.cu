// Voxel ray-casters (dvr / dvxlr / dvxlr_v2) for H100 (sm_90a).
//
// Reference: third_lib/dvr/dvr.cu (init :14-63, render_forward :65-317, render :385-627),
// third_lib/dvxlr/dvxlr.cu (render :160-457, get_grad_sigma :63-112),
// third_lib/dvxlr/dvxlr_v2.cu (indicator / ray_pred :408-423, second scatter :62-64).
//
// What is kept bit-for-bit: the Amanatides-Woo traversal in fp64 with the reference's
// operation order (float->int truncation of the origin, the -1:+1 / 0:+1 first-boundary
// rule, strict-< tie order X<Y, X<Z, Y<Z else Z, the rounded "path" voxel of
// render_forward/dvxlr, the consecutive-duplicate merge of dvxlr, termination rules),
// so every branch decision of the one-thread walk (serial_ray) equals the reference's.  The
// warp-per-ray kernel computes crossing times as fma(i, tDelta, tMax0) instead of by
// repeated addition and the rounded path voxel as round(fma(last, d, v0)): a decision can
// differ from the reference's only when two crossing times (or a path coordinate and a .5
// tie) agree to ~1e-13 relative.  Every step is therefore checked for such a near-tie (1e-9
// relative) and a ray that has one -- lattice-aligned origins / end points, e.g. a half-integer
// origin puts EVERY crossing on a round() tie -- is handed to the serial code; for all other
// rays the decisions are identical and pred/gt agree to 1e-12 relative
// (tests/test_dvr_gpu.py::test_warp_per_ray_voxel_mismatch_rate).
//
// What is redesigned: the reference keeps five MAX_D-long fp64/int3 arrays per thread
// (52-75 KB of local memory per ray, dvr.cu:176-179,490-494,594) and walks them three
// times.  Here a ray is a register-only stream:
//     T_i = exp(-csd_i),  Delta_i = d_{i+1} - d_i
//     pred      = sum_i (T_{i-1} - T_i) d_i + T_last d_last          (same order as ref)
//     dpred/dsigma_j = -dt_j * (S_0 - R_j),   R_j = sum_{k<j} T_k Delta_k,  S_0 = R_last
// (SURVEY.md A.2; identical to the D_i recursion at dvr.cu:595-608).  The gradient needs
// S_0 before the first emission, so gradient kernels walk the ray twice (pass 1: pred,
// S_0; pass 2: emit) instead of storing the path.  Gradients are accumulated with
// red.global.add.f32 (the reference's `+=` at dvr.cu:622 is a data race).
// Launch (launch_rays): one ray per warp (render_warp_kernel, 4 rays per block) when a ray's
// crossing records fit its shared-memory budget (warp_ray_config); otherwise, and always for
// the lists of dvxlr.render / render_v2, one ray per thread (render_thread_kernel) in 64-thread
// blocks (30k rays -> 469 blocks over 132 SMs; the reference's 1024-thread blocks give 30).
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace vidar {
namespace {

enum Variant { V_DVR_FWD = 0, V_DVR_RENDER = 1, V_DVXLR = 2 };

template <int V> struct Traits;
template <> struct Traits<V_DVR_FWD>    { static constexpr bool kRounded = true;  static constexpr bool kMerge = false; static constexpr int kNegBoundary = -1; };
template <> struct Traits<V_DVR_RENDER> { static constexpr bool kRounded = false; static constexpr bool kMerge = false; static constexpr int kNegBoundary = 0; };
template <> struct Traits<V_DVXLR>      { static constexpr bool kRounded = true;  static constexpr bool kMerge = true;  static constexpr int kNegBoundary = -1; };

// What a ray-caster call computes per ray; `mode` is the call's run-time option.
//   M_FWD: pred, gt (`mode` = train phase)          M_LOSS_GRAD: dvr.render (`mode` = loss type)
//   M_FUSED_BWD: fused backward of DifferentiableVoxelRendering[V2] (external grad_pred / grad_ray_pred)
//   M_LISTS: pred, gt and the per-ray lists of dvxlr.render / render_v2
enum Mode { M_FWD = 0, M_LOSS_GRAD = 1, M_FUSED_BWD = 2, M_LISTS = 3 };

// The buffers of a call besides sigma / pred / gt / grad_sigma; what a mode does not use is nullptr.
struct RayExtra {
  int max_d;                   // M_FUSED_BWD, M_LISTS: list length (the MAX_D cap)
  const float* grad_pred;      // M_FUSED_BWD: [N, M]
  const float* grad_ray_pred;  // M_FUSED_BWD, v2: [N, M, max_d]
  float* grad_sigma_regul;     // M_FUSED_BWD, v2: like sigma
  float* dd_dsigma;            // M_LISTS: [N, M, max_d] or nullptr
  float* indices;              // M_LISTS: [N, M, max_d, 3] or nullptr
  float* ray_pred;             // M_LISTS, v2: [N, M, max_d]
  float* indicator;            // M_LISTS, v2: [N, M, max_d]
  const float* sigma_regul;    // M_LISTS, v2: like sigma
};

struct Grid {
  int N, M, T, To, Z, Y, X;
};

struct Ray {
  double xo, yo, zo, dx, dy, dz, gt_d;
  int vx0, vy0, vz0;
  int n, ts;
  bool ok;
};

__device__ __forceinline__ Ray load_ray(const Grid& G, const float* __restrict__ origin,
                                        const float* __restrict__ points,
                                        const float* __restrict__ tindex, int n, int c) {
  Ray r;
  r.ok = false;
  r.n = n;
  const float tf = tindex[(size_t)n * G.M + c];
  if (tf < 0.f) return r;                      // padded ray (dvr.cu:100)
  const int t = (int)tf;                       // float used as an index: truncation
  if (t >= G.To) return r;                     // reference: out-of-bounds read
  if (G.T != 1 && t >= G.T) return r;          // reference: device assert (dvr.cu:93)
  r.ts = (G.T == 1) ? 0 : t;
  const float* o = origin + ((size_t)n * G.To + t) * 3;   // origin indexed by t, not ts (:109)
  const float* e = points + ((size_t)n * G.M + c) * 3;
  r.xo = o[0]; r.yo = o[1]; r.zo = o[2];
  const double xe = e[0], ye = e[1], ze = e[2];
  r.vx0 = (int)r.xo; r.vy0 = (int)r.yo; r.vz0 = (int)r.zo;
  const double rx = xe - r.xo, ry = ye - r.yo, rz = ze - r.zo;
  r.gt_d = sqrt(rx * rx + ry * ry + rz * rz);
  r.dx = rx / r.gt_d; r.dy = ry / r.gt_d; r.dz = rz / r.gt_d;
  r.ok = true;
  return r;
}

// The traversal loop shared by every kernel.  `visit(px,py,pz,_d,last_d)` is called for
// each step taken while inside the grid, in order.
template <int V, typename Visitor>
__device__ __forceinline__ void walk(const Grid& G, const Ray& r, Visitor& visit) {
  using TR = Traits<V>;
  int vx = r.vx0, vy = r.vy0, vz = r.vz0;
  double path_vx = (double)vx, path_vy = (double)vy, path_vz = (double)vz;
  const int stepX = (r.dx >= 0) ? 1 : -1;
  const int stepY = (r.dy >= 0) ? 1 : -1;
  const int stepZ = (r.dz >= 0) ? 1 : -1;
  const double nbx = vx + (stepX < 0 ? TR::kNegBoundary : 1);
  const double nby = vy + (stepY < 0 ? TR::kNegBoundary : 1);
  const double nbz = vz + (stepZ < 0 ? TR::kNegBoundary : 1);
  double tMaxX = (r.dx != 0) ? (nbx - r.xo) / r.dx : DBL_MAX;
  double tMaxY = (r.dy != 0) ? (nby - r.yo) / r.dy : DBL_MAX;
  double tMaxZ = (r.dz != 0) ? (nbz - r.zo) / r.dz : DBL_MAX;
  const double tDeltaX = (r.dx != 0) ? stepX / r.dx : DBL_MAX;
  const double tDeltaY = (r.dy != 0) ? stepY / r.dy : DBL_MAX;
  const double tDeltaZ = (r.dz != 0) ? stepZ / r.dz : DBL_MAX;
  double last_d = 0.0;
  bool was_inside = false;
  // Safety net only: the reference loops forever on NaN directions that never enter
  // the grid; every finite ray leaves within this many steps.
  long long guard = 4LL * ((long long)G.X + G.Y + G.Z) + 64 +
                    (long long)(fabs(r.xo) + fabs(r.yo) + fabs(r.zo)) * 2;
  if (!(guard < (1LL << 24))) guard = 1LL << 24;
  while (guard-- > 0) {
    const bool inside = (0 <= vx && vx < G.X) && (0 <= vy && vy < G.Y) && (0 <= vz && vz < G.Z);
    int px = vx, py = vy, pz = vz;
    if (inside) {
      was_inside = true;
      if (TR::kRounded) {
        px = (int)round(path_vx); px = px < G.X ? px : G.X - 1; px = px >= 0 ? px : 0;
        py = (int)round(path_vy); py = py < G.Y ? py : G.Y - 1; py = py >= 0 ? py : 0;
        pz = (int)round(path_vz); pz = pz < G.Z ? pz : G.Z - 1; pz = pz >= 0 ? pz : 0;
      }
    } else if (was_inside) {
      break;
    } else if (last_d > r.gt_d) {
      break;
    }
    double _d;
    if (tMaxX < tMaxY) {
      if (tMaxX < tMaxZ) { _d = tMaxX; vx += stepX; tMaxX += tDeltaX; }
      else               { _d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
    } else {
      if (tMaxY < tMaxZ) { _d = tMaxY; vy += stepY; tMaxY += tDeltaY; }
      else               { _d = tMaxZ; vz += stepZ; tMaxZ += tDeltaZ; }
    }
    if (TR::kRounded) {
      const double adv = fmax(0.0, _d - last_d);
      path_vx += adv * r.dx;
      path_vy += adv * r.dy;
      path_vz += adv * r.dz;
    }
    if (inside) visit(px, py, pz, _d, last_d);
    last_d = _d;
  }
}

// A committed segment: voxel, sigma there, length dt, exit distance d, index i.
// Segmenter turns visits into segments, applying dvxlr's duplicate merge
// (dvxlr.cu:366-373): a visit to the voxel of the pending segment extends it.
template <bool MERGE, typename Sink>
struct Segmenter {
  const float* __restrict__ sig;  // sigma + (n*T + ts)*Z*Y*X
  int Y, X;
  Sink& sink;
  bool has = false;
  int px = 0, py = 0, pz = 0;
  double psigma = 0, pdt = 0, pd = 0;
  __device__ __forceinline__ Segmenter(const float* s, int Y_, int X_, Sink& k) : sig(s), Y(Y_), X(X_), sink(k) {}
  __device__ __forceinline__ void operator()(int x, int y, int z, double _d, double last_d) {
    if (MERGE) {
      if (has && x == px && y == py && z == pz) {
        const double start = last_d - pdt;       // last_d -= dt[count]
        pdt = fmax(0.0, _d - start);
        pd = _d;
        return;
      }
      if (has) sink.commit(px, py, pz, psigma, pdt, pd);
      has = true;
      px = x; py = y; pz = z;
      psigma = (double)__ldg(sig + ((size_t)z * Y + y) * X + x);
      pdt = fmax(0.0, _d - last_d);
      pd = _d;
    } else {
      const double s = (double)__ldg(sig + ((size_t)z * Y + y) * X + x);
      sink.commit(x, y, z, s, fmax(0.0, _d - last_d), _d);
    }
  }
  __device__ __forceinline__ void finish() {
    if (MERGE && has) sink.commit(px, py, pz, psigma, pdt, pd);
  }
};

// The transmittance recursion over a ray's segments, shared by both passes: step() hands
// segment i (exit distance d) to `emit` as (i, R_i), R_i = sum_{k<i} T_k Delta_k, then
// advances T_prev to T_i = exp(-csd_i).  After the last segment R = S_0.
struct Transmittance {
  int count = 0;
  double csd = 0.0, T_prev = 1.0, d_last = 0.0, R = 0.0;
  template <typename Emit>
  __device__ __forceinline__ void step(double sigma, double dt, double d, Emit&& emit) {
    if (count > 0) R += T_prev * (d - d_last);
    emit(count, R);
    const double sd = sigma * dt;
    csd = (count == 0) ? sd : csd + sd;
    T_prev = exp(-csd);
    d_last = d;
    ++count;
  }
};

// Pass 1: expected distance, in the reference's summation order, plus S_0.
struct Composite : Transmittance {
  double exp_d = 0.0;
  __device__ __forceinline__ void commit(int, int, int, double sigma, double dt, double d) {
    const double T_before = (count == 0) ? 1.0 : T_prev;   // p_0 = 1 - T_0
    step(sigma, dt, d, [](int, double) {});
    exp_d += (T_before - T_prev) * d;
  }
  // pred = sum p_i d_i + p_out * max_d   (dvr.cu:286-298)
  __device__ __forceinline__ double pred() const { return exp_d + T_prev * d_last; }
};

// Pass 2 sinks.  Each emits, for segment i, something of dd_i = -dt_i (S0 - R_i).
struct ScatterSink : Transmittance {  // atomically add coef * dd_i into grad_sigma
  float* __restrict__ gsig;   // grad_sigma + frame offset
  const float* __restrict__ grp;  // grad_ray_pred row for this ray (v2) or nullptr
  float* __restrict__ gsreg;  // grad_sigma_regul + frame offset (v2) or nullptr
  int Y, X, max_d;
  double S0, coef;
  bool nan_to_zero;
  __device__ __forceinline__ void commit(int x, int y, int z, double sigma, double dt, double d) {
    step(sigma, dt, d, [&](int i, double R) {
      if (i >= max_d) return;
      const size_t vo = ((size_t)z * Y + y) * X + x;
      // float(dd) * float(coef) like `gradpred[..., None] * dd_dsigma` on fp32 tensors
      float g = (float)(-dt * (S0 - R)) * (float)coef;
      if (nan_to_zero && isnan(g)) g = 0.f;
      if (g != 0.f) red_add_f32(gsig + vo, g);
      if (grp) {
        const float gr = grp[i];
        if (gr != 0.f) red_add_f32(gsreg + vo, gr);
      }
    });
  }
};

struct RenderGradSink : Transmittance {  // dvr.render: grad_sigma += dl_dd * dd_i in fp64 then fp32 atomics
  float* __restrict__ gsig;
  int Y, X;
  double S0, dl_dd;
  __device__ __forceinline__ void commit(int x, int y, int z, double sigma, double dt, double d) {
    step(sigma, dt, d, [&](int, double R) {
      const float g = (float)(dl_dd * (-dt * (S0 - R)));
      if (g != 0.f) red_add_f32(gsig + ((size_t)z * Y + y) * X + x, g);
    });
  }
};

struct ListSink : Transmittance {  // dvxlr.render: write the per-ray lists
  float* __restrict__ dd;       // [max_d]
  float* __restrict__ idx;      // [max_d,3]
  float* __restrict__ ray_pred; // [max_d] or nullptr
  float* __restrict__ indicator;
  const float* __restrict__ sreg;  // sigma_regul + frame offset
  int Y, X, max_d;
  double S0, gt_raw;
  bool reached = false;
  __device__ __forceinline__ void commit(int x, int y, int z, double sigma, double dt, double d) {
    step(sigma, dt, d, [&](int i, double R) {
      if (i >= max_d) return;
      if (dd) {
        dd[i] = (float)(-dt * (S0 - R));
        idx[i * 3 + 0] = (float)z;
        idx[i * 3 + 1] = (float)y;
        idx[i * 3 + 2] = (float)x;
      }
      if (ray_pred) {
        float ind = 0.f;
        if (!reached && d >= gt_raw) { ind = 1.f; reached = true; }
        indicator[i] = ind;
        ray_pred[i] = __ldg(sreg + ((size_t)z * Y + y) * X + x);
      }
    });
  }
};

constexpr int kRayBlock = 64;

__global__ void init_kernel(Grid G, const float* __restrict__ points,
                            const float* __restrict__ tindex, float* __restrict__ occ) {
  const int n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= G.M) return;
  const float tf = tindex[(size_t)n * G.M + c];
  if (tf < 0.f) return;
  const int t = (int)tf;
  if (G.T != 1 && t >= G.T) return;
  const int ts = (G.T == 1) ? 0 : t;
  const float* e = points + ((size_t)n * G.M + c) * 3;
  const int vx = (int)e[0], vy = (int)e[1], vz = (int)e[2];
  if (0 <= vx && vx < G.X && 0 <= vy && vy < G.Y && 0 <= vz && vz < G.Z)
    occ[((((size_t)n * G.T + ts) * G.Z + vz) * G.Y + vy) * G.X + vx] = 1.f;
}

// Walks the ray and hands its segments (merged for dvxlr) to `sink`.
template <int V, typename Sink>
__device__ __forceinline__ void walk_segments(const Grid& G, const Ray& r, const float* sig, Sink& sink) {
  Segmenter<Traits<V>::kMerge, Sink> seg(sig, G.Y, G.X, sink);
  walk<V>(G, r, seg);
  seg.finish();
}

// One ray by one thread, bit-faithful: the body of render_thread_kernel and the fallback of
// render_warp_kernel.  Pass 1 gives pred and S_0; the gradient and list modes walk the ray again.
template <int V, int MODE>
__device__ void serial_ray(const Grid& G, const Ray& r, const float* __restrict__ sigma,
                           float* __restrict__ pred_dist, float* __restrict__ gt_dist,
                           float* __restrict__ grad_sigma, int n, int c, int mode, const RayExtra& ex) {
  const size_t vol = (size_t)G.Z * G.Y * G.X;
  const size_t foff = ((size_t)n * G.T + r.ts) * vol;
  const float* sg = sigma + foff;
  Composite comp;
  walk_segments<V>(G, r, sg, comp);
  if (comp.count == 0) return;
  const double exp_d = comp.pred();
  const size_t ray = (size_t)n * G.M + c;
  if constexpr (MODE == M_FUSED_BWD) {
    const bool v2 = ex.grad_ray_pred != nullptr;
    ScatterSink sink{{}, grad_sigma + foff, v2 ? ex.grad_ray_pred + ray * ex.max_d : nullptr,
                     v2 ? ex.grad_sigma_regul + foff : nullptr, G.Y, G.X, ex.max_d, comp.R,
                     (double)ex.grad_pred[ray], !v2};
    walk_segments<V>(G, r, sg, sink);
  } else {
    double gt = r.gt_d;
    if (MODE == M_LOSS_GRAD || Traits<V>::kMerge || mode == 1) gt = fmin(gt, comp.d_last);
    pred_dist[ray] = (float)exp_d;
    gt_dist[ray] = (float)gt;
    if constexpr (MODE == M_LOSS_GRAD) {   // dvr.cu:576-625
      double dl_dd = 1.0;
      if (mode == 0) dl_dd = (exp_d >= gt) ? 1 : -1;
      else if (mode == 1) dl_dd = (exp_d - gt);
      else if (mode == 2) dl_dd = (exp_d >= gt) ? (1.0 / gt) : -(1.0 / gt);
      RenderGradSink sink{{}, grad_sigma + foff, G.Y, G.X, comp.R, dl_dd};
      walk_segments<V>(G, r, sg, sink);
    } else if constexpr (MODE == M_LISTS) {
      const size_t row = ray * ex.max_d;
      ListSink sink{{}, ex.dd_dsigma ? ex.dd_dsigma + row : nullptr, ex.indices ? ex.indices + row * 3 : nullptr,
                    ex.ray_pred ? ex.ray_pred + row : nullptr, ex.indicator ? ex.indicator + row : nullptr,
                    ex.sigma_regul ? ex.sigma_regul + foff : nullptr, G.Y, G.X, ex.max_d, comp.R, r.gt_d};
      walk_segments<V>(G, r, sg, sink);
    }
  }
}

// One ray per thread: the lists (M_LISTS) always, every other mode when the warp kernel's
// records do not fit in shared memory (launch_rays).
template <int V, int MODE>
__global__ void __launch_bounds__(kRayBlock)
render_thread_kernel(Grid G, const float* __restrict__ sigma, const float* __restrict__ origin,
                     const float* __restrict__ points, const float* __restrict__ tindex,
                     float* __restrict__ pred_dist, float* __restrict__ gt_dist,
                     float* __restrict__ grad_sigma, int mode, RayExtra ex) {
  const int n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= G.M) return;
  const Ray r = load_ray(G, origin, points, tindex, n, c);
  if (r.ok) serial_ray<V, MODE>(G, r, sigma, pred_dist, gt_dist, grad_sigma, n, c, mode, ex);
}

// ------------------------------------------------------------------------------------------
// One ray per WARP (dvr.render_forward / dvr.render).  The serial march above leaves the chip
// at 9 % of its warp slots (30k threads of dependent fp64 work).  Here the 32 lanes of a warp
// share one ray:
//   phase 1  the ray's parameter range [0, t_exit] is cut into 32 slices; lane j finds, in
//            closed form, how many X/Y/Z boundary crossings precede its slice
//            (count_a(T) = ceil((T - tMax0_a) / tDelta_a)), runs the reference's DDA (same
//            strict-< tie order) over the crossings of its slice only, and writes
//            (crossing time, voxel) records to shared memory in global order;
//   phase 2  lanes take the records 32 at a time: sigma gather, warp scan of sigma*delta,
//            T = exp(-csd), pred += (T_prev - T) t, scan of T_prev (t - t_prev) -> U;
//   phase 3  (dvr.render) grad_sigma[voxel] += dL/dd * -delta (S0 - U)  by red.global.add.
// One exp per step instead of one per step per pass, 32x the threads, and the per-ray critical
// path drops from ~500 dependent steps to ~8 + three scans.  Crossing times come from
// tMax0 + i*tDelta (fused) instead of the reference's repeated addition: identical branch
// decisions except within ~1e-13 of an exact tie, where the two orders differ by a
// zero-length segment.  Rays whose origin is outside the grid (the reference's
// "march until you enter or pass the end point" logic) or whose crossing count exceeds the
// shared-memory budget take the serial code on lane 0.
constexpr int kWarpRaysPerBlock = 4;

// relative distance below which two crossing times / a path coordinate and a .5 tie count as a near-tie
// (render_warp_kernel): such rays take the serial traversal, whose decisions are the reference's
constexpr double kTieEps = 1e-9;

template <typename T>
__device__ __forceinline__ T warp_incl_scan(T v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// crossings of one axis strictly before parameter T, capped at `hi` (crossings until the ray
// leaves the grid along that axis)
__device__ __forceinline__ int crossings_before(double T, double tMax0, double tDelta, bool moves, int hi) {
  if (!moves || !(T > tMax0)) return 0;
  const double q = ceil((T - tMax0) / tDelta);
  return q >= (double)hi ? hi : (int)q;
}

// Merge variants (dvxlr): a run of consecutive records with the same (rounded) voxel is ONE segment --
// length from the crossing before the run to the run's last crossing (dvxlr.cu:366-373) -- closed by
// the run's last record.  run_head returns the head record of the run that lane's record belongs to
// (a warp max-scan of the head flags) and carries it across chunks in `carry_head`.  It touches no
// shared memory: with the record loads moved in here as well, the compiler lays out the whole warp
// kernel differently (one more stack slot in render_warp_kernel<V_DVXLR, M_FWD>).
__device__ __forceinline__ int run_head(bool head, int k, int lane, int& carry_head) {
  int hs = head ? k : -1;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, hs, o);
    if (lane >= o) hs = max(hs, u);
  }
  hs = max(hs, carry_head);
  carry_head = __shfl_sync(0xffffffffu, hs, 31);
  return hs;
}

// Every mode but M_LISTS; mode: M_LOSS_GRAD ? loss_type : train_phase.  Merge variants: a run's segment is
// carried by its last record (run_head); list ordinals (the MAX_D cap, grad_ray_pred slots) come from an
// add-scan of the tail flags.
template <int V, int MODE>
__global__ void __launch_bounds__(kWarpRaysPerBlock * 32)
render_warp_kernel(Grid G, const float* __restrict__ sigma, const float* __restrict__ origin,
                   const float* __restrict__ points, const float* __restrict__ tindex,
                   float* __restrict__ pred_dist, float* __restrict__ gt_dist,
                   float* __restrict__ grad_sigma, int mode, int cap, RayExtra ex) {
  using TR = Traits<V>;
  constexpr bool GRAD = MODE != M_FWD;
  constexpr bool MERGE = TR::kMerge;
  extern __shared__ double smem_d[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.y;
  const int c = blockIdx.x * kWarpRaysPerBlock + warp;
  if (c >= G.M) return;
  // per-warp records: ts[cap] crossing time, us[cap] prefix U, vx[cap] voxel index (-1 = outside)
  double* ts = smem_d + (size_t)warp * cap * 2;
  double* us = ts + cap;
  int* vxs = reinterpret_cast<int*>(smem_d + (size_t)kWarpRaysPerBlock * cap * 2) + (size_t)warp * cap;

  const Ray r = load_ray(G, origin, points, tindex, n, c);
  if (!r.ok) return;
  const int N3[3] = {G.X, G.Y, G.Z};
  const int v0[3] = {r.vx0, r.vy0, r.vz0};
  const double dir[3] = {r.dx, r.dy, r.dz};
  const double org[3] = {r.xo, r.yo, r.zo};
  int stp[3], hi[3];
  double tMax0[3], tDelta[3];
  bool moves[3];
  bool eligible = true;
  long long bound = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    eligible = eligible && v0[a] >= 0 && v0[a] < N3[a] && (dir[a] == dir[a]);
    stp[a] = (dir[a] >= 0) ? 1 : -1;
    moves[a] = dir[a] != 0;
    const double nb = v0[a] + (stp[a] < 0 ? TR::kNegBoundary : 1);
    tMax0[a] = moves[a] ? (nb - org[a]) / dir[a] : DBL_MAX;
    tDelta[a] = moves[a] ? stp[a] / dir[a] : DBL_MAX;
    hi[a] = stp[a] > 0 ? N3[a] - v0[a] : v0[a] + 1;     // crossings until the voxel index leaves [0, N)
    if (moves[a]) bound += hi[a];
  }
  eligible = eligible && bound > 0 && bound <= cap && isfinite(r.gt_d) && r.gt_d > 0;
  if (!eligible) {
    if (lane == 0) serial_ray<V, MODE>(G, r, sigma, pred_dist, gt_dist, grad_sigma, n, c, mode, ex);
    return;
  }
  // ---- phase 1: slices of the parameter range
  double t_exit = DBL_MAX;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (moves[a]) t_exit = fmin(t_exit, fma((double)(hi[a] - 1), tDelta[a], tMax0[a]));
  const double w = t_exit * (1.0 / 32.0);
  const double T_lo = (double)lane * w;
  // the last slice ends just past the exit crossing (t == t_exit must be included; crossings of
  // the other axes after it would be steps outside the grid)
  const double T_hi = (lane == 31) ? t_exit + t_exit * 1e-11 + 1e-300 : (double)(lane + 1) * w;
  int ia[3], rem[3], nsteps = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ia[a] = crossings_before(T_lo, tMax0[a], tDelta[a], moves[a], hi[a]);
    rem[a] = crossings_before(T_hi, tMax0[a], tDelta[a], moves[a], hi[a]) - ia[a];
    nsteps += rem[a];
  }
  // exclusive scan of the per-lane step counts -> where this lane writes
  const int incl = warp_incl_scan(nsteps, lane);
  const int N = __shfl_sync(0xffffffffu, incl, 31);
  const int off = incl - nsteps;
  // Near-tie detection.  Crossing times here are fma(i, tDelta, tMax0); the reference adds tDelta i
  // times, so the two agree to ~1e-13 relative but not bit for bit.  That only matters where a branch
  // decision hangs on the last bits: two axes crossing at (almost) the same parameter, or -- rounded-path
  // variants -- a path coordinate (almost) exactly on a .5 round() tie (e.g. half-integer origins: every
  // crossing).  Such rays are walked by the bit-faithful serial code instead.
  bool tie = false;
  {
    int v[3], gi[3];
    double tm[3], last = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      v[a] = v0[a] + stp[a] * ia[a];
      gi[a] = ia[a];
      tm[a] = moves[a] ? fma((double)ia[a], tDelta[a], tMax0[a]) : DBL_MAX;
      if (ia[a] > 0) last = fmax(last, fma((double)(ia[a] - 1), tDelta[a], tMax0[a]));
    }
    for (int sidx = 0; sidx < nsteps; ++sidx) {
      const double tx = rem[0] > 0 ? tm[0] : DBL_MAX;
      const double ty = rem[1] > 0 ? tm[1] : DBL_MAX;
      const double tz = rem[2] > 0 ? tm[2] : DBL_MAX;
      // the reference's choice: X if tx < ty and tx < tz; Y if !(tx < ty) and ty < tz; else Z
      const int ax = (tx < ty) ? ((tx < tz) ? 0 : 2) : ((ty < tz) ? 1 : 2);
      const double tcur = ax == 0 ? tx : (ax == 1 ? ty : tz);
      // pending crossings of the other axes (unmasked: the neighbouring slice's first crossing counts);
      // two 0-th crossings are exact in both formulations and need no flag
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (a != ax && moves[a] && gi[a] < hi[a] && (gi[a] > 0 || gi[ax] > 0) &&
            fabs(tm[a] - tcur) <= kTieEps * fabs(tcur))
          tie = true;
      }
      const bool inside = v[0] >= 0 && v[0] < G.X && v[1] >= 0 && v[1] < G.Y && v[2] >= 0 && v[2] < G.Z;
      int idx = -1;
      if (inside) {
        int px = v[0], py = v[1], pz = v[2];
        if (TR::kRounded) {   // nearest voxel to v0 + last * dir  (dvr.cu:200-212, 255-257)
          const double cx = fma(last, r.dx, (double)r.vx0), cy = fma(last, r.dy, (double)r.vy0),
                       cz = fma(last, r.dz, (double)r.vz0);
          if (last > 0.0) {
            tie = tie || fabs(fabs(cx - floor(cx)) - 0.5) <= kTieEps * fmax(1.0, fabs(cx)) ||
                  fabs(fabs(cy - floor(cy)) - 0.5) <= kTieEps * fmax(1.0, fabs(cy)) ||
                  fabs(fabs(cz - floor(cz)) - 0.5) <= kTieEps * fmax(1.0, fabs(cz));
          }
          px = (int)round(cx); px = px < G.X ? px : G.X - 1; px = px >= 0 ? px : 0;
          py = (int)round(cy); py = py < G.Y ? py : G.Y - 1; py = py >= 0 ? py : 0;
          pz = (int)round(cz); pz = pz < G.Z ? pz : G.Z - 1; pz = pz >= 0 ? pz : 0;
        }
        idx = (pz * G.Y + py) * G.X + px;
      }
      ts[off + sidx] = tcur;
      vxs[off + sidx] = idx;
      if (ax == 0) { v[0] += stp[0]; tm[0] += tDelta[0]; --rem[0]; ++gi[0]; }
      else if (ax == 1) { v[1] += stp[1]; tm[1] += tDelta[1]; --rem[1]; ++gi[1]; }
      else { v[2] += stp[2]; tm[2] += tDelta[2]; --rem[2]; ++gi[2]; }
      last = fmax(last, tcur);
    }
  }
  if (__any_sync(0xffffffffu, tie)) {
    if (lane == 0) serial_ray<V, MODE>(G, r, sigma, pred_dist, gt_dist, grad_sigma, n, c, mode, ex);
    return;
  }
  __syncwarp();
  // ---- phase 2: compositing over the records, 32 steps at a time
  const size_t vol = (size_t)G.Z * G.Y * G.X;
  const size_t foff = ((size_t)n * G.T + r.ts) * vol;
  const float* sg = sigma + foff;
  double carry_csd = 0.0, carry_U = 0.0, T_carry = 1.0, pred_part = 0.0, d_last = 0.0;
  int carry_head = 0;                                   // MERGE: record index of the current run's head
  for (int base = 0; base < N; base += 32) {
    const int k = base + lane;
    const bool valid = k < N;
    const int idx = valid ? vxs[k] : -1;
    const bool ins = idx >= 0;
    const double tk = valid ? ts[k] : 0.0;
    bool tail = ins;                                     // does this record close a segment?
    double t0 = (valid && k > 0) ? ts[k - 1] : 0.0;      // parameter at which its segment starts
    int hs = k;
    if (MERGE) {
      const bool head = ins && (k == 0 || vxs[k - 1] != idx);
      tail = ins && (k == N - 1 || vxs[k + 1] != idx);
      hs = run_head(head, k, lane, carry_head);
      t0 = (hs > 0) ? ts[hs - 1] : 0.0;
    }
    const double dt = tail ? fmax(0.0, tk - t0) : 0.0;
    const double sd = tail ? (double)__ldg(sg + idx) * dt : 0.0;
    const double csd = warp_incl_scan(sd, lane) + carry_csd;
    const double T = exp(-csd);
    double Tp = __shfl_up_sync(0xffffffffu, T, 1);
    if (lane == 0) Tp = T_carry;
    if (tail) {
      pred_part += (Tp - T) * tk;
      d_last = fmax(d_last, tk);
    }
    const double term = (tail && hs > 0) ? Tp * (tk - t0) : 0.0;      // T_prev (d_i - d_{i-1}), first segment: 0
    const double U = warp_incl_scan(term, lane) + carry_U;
    if (GRAD && valid) us[k] = U;
    carry_csd = __shfl_sync(0xffffffffu, csd, 31);
    carry_U = __shfl_sync(0xffffffffu, U, 31);
    T_carry = __shfl_sync(0xffffffffu, T, 31);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    pred_part += __shfl_xor_sync(0xffffffffu, pred_part, o);
    d_last = fmax(d_last, __shfl_xor_sync(0xffffffffu, d_last, o));
  }
  const double exp_d = pred_part + T_carry * d_last;    // + p_out * max_d
  double gt = r.gt_d;
  if (MODE == M_LOSS_GRAD || MERGE || mode == 1) gt = fmin(gt, d_last);
  if (MODE != M_FUSED_BWD && lane == 0) {
    pred_dist[(size_t)n * G.M + c] = (float)exp_d;
    gt_dist[(size_t)n * G.M + c] = (float)gt;
  }
  if (!GRAD) return;
  // ---- phase 3: gradient emission, one record per lane
  const size_t ray = (size_t)n * G.M + c;
  double coef = 1.0;
  if (MODE == M_LOSS_GRAD) {
    if (mode == 0) coef = (exp_d >= gt) ? 1 : -1;
    else if (mode == 1) coef = (exp_d - gt);
    else if (mode == 2) coef = (exp_d >= gt) ? (1.0 / gt) : -(1.0 / gt);
  }
  const float coef_f = (MODE == M_FUSED_BWD) ? __ldg(ex.grad_pred + ray) : 0.f;
  const float* grp = (MODE == M_FUSED_BWD && ex.grad_ray_pred) ? ex.grad_ray_pred + ray * ex.max_d : nullptr;
  float* gs = grad_sigma + foff;
  float* gsr = grp ? ex.grad_sigma_regul + foff : nullptr;
  const double S0 = carry_U;
  __syncwarp();
  carry_head = 0;
  int carry_ord = 0;                                     // segments closed before this chunk
  for (int base = 0; base < N; base += 32) {
    const int k = base + lane;
    const bool valid = k < N;
    const int idx = valid ? vxs[k] : -1;
    const bool ins = idx >= 0;
    bool tail = ins;
    double t0 = (valid && k > 0) ? ts[k - 1] : 0.0;
    if (MERGE) {
      const bool head = ins && (k == 0 || vxs[k - 1] != idx);
      tail = ins && (k == N - 1 || vxs[k + 1] != idx);
      const int hs = run_head(head, k, lane, carry_head);
      t0 = (hs > 0) ? ts[hs - 1] : 0.0;
    }
    int ord = 0;                                         // list slot of this segment (MAX_D cap, v2 slots)
    if (MODE == M_FUSED_BWD) {
      const unsigned tb = __ballot_sync(0xffffffffu, tail);
      ord = carry_ord + __popc(tb & ((1u << lane) - 1u));
      carry_ord += __popc(tb);
    }
    if (!tail) continue;
    const double dt = fmax(0.0, ts[k] - t0);
    if (MODE == M_LOSS_GRAD) {
      const float g = (float)(coef * (-dt * (S0 - us[k])));
      if (g != 0.f) red_add_f32(gs + idx, g);
    } else if (ord < ex.max_d) {
      // float(dd) * float(grad) like `gradpred[..., None] * dd_dsigma` on fp32 tensors (e2e_predictor_utils.py:106)
      float g = (float)(-dt * (S0 - us[k])) * coef_f;
      if (!grp && isnan(g)) g = 0.f;                     // v1: nan_to_num (:107-108)
      if (g != 0.f) red_add_f32(gs + idx, g);
      if (grp) {
        const float gr = __ldg(grp + ord);
        if (gr != 0.f) red_add_f32(gsr + idx, gr);
      }
    }
  }
}

// dvxlr.get_grad_sigma[_v2]: one warp per ray, lanes stride over the list so reads are
// coalesced.  Exact zeros are skipped: the reference adds the zero padding of all
// 1026 slots to voxel (0,0,0) (dvxlr.cu:101-110), which changes nothing but serialises
// ~25M atomics on one address.
__global__ void __launch_bounds__(256)
list_scatter_kernel(Grid G, const float* __restrict__ em, const float* __restrict__ indices,
                    const float* __restrict__ tindex, const float* __restrict__ indicator,
                    const float* __restrict__ grad_ray_pred, float* __restrict__ grad_sigma,
                    float* __restrict__ grad_sigma_regul, int max_d) {
  const int n = blockIdx.y;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= G.M) return;
  const float tf = tindex[(size_t)n * G.M + c];
  if (tf < 0.f) return;
  const int t = (int)tf;
  if (G.T != 1 && t >= G.T) return;
  const int ts = (G.T == 1) ? 0 : t;
  const size_t vol = (size_t)G.Z * G.Y * G.X;
  const size_t foff = ((size_t)n * G.T + ts) * vol;
  const size_t ray = (size_t)n * G.M + c;
  const float* e = em + ray * max_d;
  const float* id = indices + ray * max_d * 3;
  for (int i = lane; i < max_d; i += 32) {
    const float v = e[i];
    const bool reg = indicator && indicator[ray * max_d + i] >= 0.f;
    if (v == 0.f && !reg) continue;
    const int z = (int)id[i * 3], y = (int)id[i * 3 + 1], x = (int)id[i * 3 + 2];
    if (z < 0 || z >= G.Z || y < 0 || y >= G.Y || x < 0 || x >= G.X) continue;
    const size_t vo = foff + ((size_t)z * G.Y + y) * G.X + x;
    if (v != 0.f) red_add_f32(grad_sigma + vo, v);
    if (reg) {
      const float gr = grad_ray_pred[ray * max_d + i];
      if (gr != 0.f) red_add_f32(grad_sigma_regul + vo, gr);
    }
  }
}

int check_grid(Grid& G, int N, int M, int T, int To, int Z, int Y, int X, const char* who) {
  VIDAR_REQUIRE(N > 0 && M >= 0 && T > 0 && To > 0 && Z > 0 && Y > 0 && X > 0,
                "%s: bad sizes N=%d M=%d T=%d To=%d grid=%dx%dx%d", who, N, M, T, To, Z, Y, X);
  VIDAR_REQUIRE(N <= 65535, "%s: batch %d exceeds gridDim.y", who, N);
  G = Grid{N, M, T, To, Z, Y, X};
  return VIDAR_OK;
}

// shared-memory budget of the warp-per-ray kernels: 20 bytes per crossing record, cap =
// X+Y+Z+8 records per ray.  Returns false when it does not fit (fall back to thread-per-ray).
template <typename K>
bool warp_ray_config(const Grid& G, K kernel, int& cap, size_t& smem) {
  cap = ((G.X + G.Y + G.Z + 8 + 31) / 32) * 32;
  smem = (size_t)kWarpRaysPerBlock * cap * (2 * sizeof(double) + sizeof(int));
  if (smem > 200 * 1024) return false;
  if (smem > 48 * 1024) {
    // The opt-in is per (kernel, device) and cheap: set it on every launch that needs it.  (A cached
    // flag keyed only on the kernel's *type* is shared by instantiations with the same signature and
    // is wrong on a second device.)
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
  }
  return true;
}

inline dim3 ray_grid(const Grid& G, int per_block) {
  return dim3((unsigned)((G.M + per_block - 1) / per_block), (unsigned)G.N);
}

// One ray per warp when the records fit (never for the lists), else one ray per thread.
template <int V, int MODE>
void launch_rays(const Grid& G, const float* sigma, const float* origin, const float* points,
                 const float* tindex, float* pred_dist, float* gt_dist, float* grad_sigma, int mode,
                 const RayExtra& ex, cudaStream_t stream) {
  if constexpr (MODE != M_LISTS) {
    int cap;
    size_t smem;
    if (warp_ray_config(G, render_warp_kernel<V, MODE>, cap, smem)) {
      render_warp_kernel<V, MODE><<<ray_grid(G, kWarpRaysPerBlock), kWarpRaysPerBlock * 32, smem, stream>>>(
          G, sigma, origin, points, tindex, pred_dist, gt_dist, grad_sigma, mode, cap, ex);
      return;
    }
  }
  render_thread_kernel<V, MODE><<<ray_grid(G, kRayBlock), kRayBlock, 0, stream>>>(
      G, sigma, origin, points, tindex, pred_dist, gt_dist, grad_sigma, mode, ex);
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_dvr_init(const float* points, const float* tindex, float* occupancy, int N,
                              int M, int T, int Z, int Y, int X, void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, T, Z, Y, X, "dvr.init");
  if (rc) return rc;
  VIDAR_REQUIRE(points && tindex && occupancy, "dvr.init: null pointer argument");
  if (M == 0) return VIDAR_OK;
  init_kernel<<<ray_grid(G, 256), 256, 0, (cudaStream_t)stream>>>(G, points, tindex, occupancy);
  return check_launch("dvr.init");
}

extern "C" int vidar_dvr_render_forward(const float* sigma, const float* origin,
                                        const float* points, const float* tindex,
                                        float* pred_dist, float* gt_dist, int N, int M, int T,
                                        int To, int Z, int Y, int X, int train_phase,
                                        void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, To, Z, Y, X, "dvr.render_forward");
  if (rc) return rc;
  VIDAR_REQUIRE(sigma && origin && points && tindex && pred_dist && gt_dist,
                "dvr.render_forward: null pointer argument");
  VIDAR_REQUIRE(train_phase == 0 || train_phase == 1, "UNKNOWN PHASE NAME: %d", train_phase);
  if (M == 0) return VIDAR_OK;
  launch_rays<V_DVR_FWD, M_FWD>(G, sigma, origin, points, tindex, pred_dist, gt_dist, nullptr, train_phase,
                                RayExtra{}, (cudaStream_t)stream);
  return check_launch("dvr.render_forward");
}

extern "C" int vidar_dvr_render(const float* sigma, const float* origin, const float* points,
                                const float* tindex, float* pred_dist, float* gt_dist,
                                float* grad_sigma, int N, int M, int T, int To, int Z, int Y,
                                int X, int loss_type, void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, To, Z, Y, X, "dvr.render");
  if (rc) return rc;
  VIDAR_REQUIRE(sigma && origin && points && tindex && pred_dist && gt_dist && grad_sigma,
                "dvr.render: null pointer argument");
  VIDAR_REQUIRE(loss_type >= 0 && loss_type <= 2, "UNKNOWN LOSS TYPE: %d", loss_type);
  if (M == 0) return VIDAR_OK;
  launch_rays<V_DVR_RENDER, M_LOSS_GRAD>(G, sigma, origin, points, tindex, pred_dist, gt_dist, grad_sigma,
                                        loss_type, RayExtra{}, (cudaStream_t)stream);
  return check_launch("dvr.render");
}

extern "C" int vidar_dvxlr_forward(const float* sigma, const float* origin, const float* points,
                                   const float* tindex, float* pred_dist, float* gt_dist, int N,
                                   int M, int T, int To, int Z, int Y, int X, void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, To, Z, Y, X, "dvxlr.forward");
  if (rc) return rc;
  VIDAR_REQUIRE(sigma && origin && points && tindex && pred_dist && gt_dist,
                "dvxlr.forward: null pointer argument");
  if (M == 0) return VIDAR_OK;
  launch_rays<V_DVXLR, M_FWD>(G, sigma, origin, points, tindex, pred_dist, gt_dist, nullptr, 1, RayExtra{},
                              (cudaStream_t)stream);
  return check_launch("dvxlr.forward");
}

extern "C" int vidar_dvxlr_render(const float* sigma, const float* origin, const float* points,
                                  const float* tindex, const float* sigma_regul,
                                  float* pred_dist, float* gt_dist, float* dd_dsigma,
                                  float* indices, float* ray_pred, float* indicator, int N, int M,
                                  int T, int To, int Z, int Y, int X, int max_d, void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, To, Z, Y, X, "dvxlr.render");
  if (rc) return rc;
  VIDAR_REQUIRE(sigma && origin && points && tindex && pred_dist && gt_dist,
                "dvxlr.render: null pointer argument");
  VIDAR_REQUIRE((dd_dsigma == nullptr) == (indices == nullptr),
                "dvxlr.render: dd_dsigma and indices go together");
  VIDAR_REQUIRE(max_d > 0, "dvxlr.render: max_d must be positive");
  const bool v2 = sigma_regul || ray_pred || indicator;
  VIDAR_REQUIRE(!v2 || (sigma_regul && ray_pred && indicator),
                "dvxlr.render_v2: sigma_regul, ray_pred and indicator must all be given");
  if (M == 0) return VIDAR_OK;
  launch_rays<V_DVXLR, M_LISTS>(G, sigma, origin, points, tindex, pred_dist, gt_dist, nullptr, 1,
                                RayExtra{max_d, nullptr, nullptr, nullptr, dd_dsigma, indices, ray_pred,
                                         indicator, sigma_regul},
                                (cudaStream_t)stream);
  return check_launch("dvxlr.render");
}

extern "C" int vidar_dvxlr_get_grad_sigma(const float* elementwise_mult, const float* indices,
                                          const float* tindex, const float* indicator,
                                          const float* grad_ray_pred, float* grad_sigma,
                                          float* grad_sigma_regul, int N, int M, int T, int Z,
                                          int Y, int X, int max_d, void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, T, Z, Y, X, "dvxlr.get_grad_sigma");
  if (rc) return rc;
  VIDAR_REQUIRE(elementwise_mult && indices && tindex && grad_sigma,
                "dvxlr.get_grad_sigma: null pointer argument");
  const bool v2 = indicator || grad_ray_pred || grad_sigma_regul;
  VIDAR_REQUIRE(!v2 || (indicator && grad_ray_pred && grad_sigma_regul),
                "dvxlr.get_grad_sigma_v2: indicator, grad_ray_pred and grad_sigma_regul must all be given");
  VIDAR_REQUIRE(max_d > 0, "dvxlr.get_grad_sigma: max_d must be positive");
  if (M == 0) return VIDAR_OK;
  list_scatter_kernel<<<ray_grid(G, 8), 256, 0, (cudaStream_t)stream>>>(
      G, elementwise_mult, indices, tindex, indicator, grad_ray_pred, grad_sigma, grad_sigma_regul,
      max_d);
  return check_launch("dvxlr.get_grad_sigma");
}

extern "C" int vidar_dvxlr_backward_fused(const float* sigma, const float* origin,
                                          const float* points, const float* tindex,
                                          const float* grad_pred, const float* grad_ray_pred,
                                          float* grad_sigma, float* grad_sigma_regul, int N,
                                          int M, int T, int To, int Z, int Y, int X, int max_d,
                                          void* stream) {
  Grid G;
  int rc = check_grid(G, N, M, T, To, Z, Y, X, "dvxlr.backward_fused");
  if (rc) return rc;
  VIDAR_REQUIRE(sigma && origin && points && tindex && grad_pred && grad_sigma,
                "dvxlr.backward_fused: null pointer argument");
  VIDAR_REQUIRE((grad_ray_pred == nullptr) == (grad_sigma_regul == nullptr),
                "dvxlr.backward_fused: grad_ray_pred and grad_sigma_regul go together");
  VIDAR_REQUIRE(max_d > 0, "dvxlr.backward_fused: max_d must be positive");
  if (M == 0) return VIDAR_OK;
  launch_rays<V_DVXLR, M_FUSED_BWD>(G, sigma, origin, points, tindex, nullptr, nullptr, grad_sigma, 1,
                                    RayExtra{max_d, grad_pred, grad_ray_pred, grad_sigma_regul},
                                    (cudaStream_t)stream);
  return check_launch("dvxlr.backward_fused");
}
