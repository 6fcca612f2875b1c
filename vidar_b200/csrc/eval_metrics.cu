// ViDAR's evaluation metrics, H100 (sm_90a): Chamfer distance inside the point-cloud range and the
// L1 / AbsRel ray-depth errors of every (sample, frame) of a batch in a fixed number of launches.
//
// Reference: bevformer/detectors/vidar.py:452-497 (per-pair loop), utils/e2e_predictor_utils.py:146-183
// (compute_chamfer_distance_inner) and utils/eval_utils.py:17-225 (clamp, _clamp, spherical_projection,
// compute_ray_errors).  Every fp32 statement the reference evaluates is evaluated here in its order with
// explicit __f*_rn intrinsics (nvcc would contract `a + b * c` to an FMA); arctan2 is evaluated in fp64 and
// rounded to fp32.  Sums are fp64, in a fixed order: per-block tree, then the blocks of a segment in order.
//
// Layout (S = 3N segments, N = samples x frames, n = b * F + f):
//   queries    [pred xyz (Pp) | gt xyz (Pg) | gt spherical (Pg)]   segments 0..N-1 | N..2N-1 | 2N..3N-1
//   candidates [gt xyz (Pg) | pred xyz (Pp) | pred spherical (Pp)]
// so one segmented NN launch (knn.cu) serves both Chamfer directions and the spherical search.
//
// vidar_eval_decode_clouds builds those clouds on the device from the head's decoded rays
// (dense_heads/vidar_head_base.py:698-745 get_point_cloud_prediction, :363-389 get_rendered_pcds): row r of sample b
// joins cloud n = b * F + t when tindex == t, gt_dist > 0 and (within_grid) its metre point is inside pc_range.  A
// stable counting sort keyed by (b, t) (counting_sort.cuh) keeps the rows of a cloud in their original order, which
// decides NN ties as the boolean masks of the reference do.  Every other row goes, as NaN, into one trailing segment
// N that every search and sum masks out; its row of the metric table is dropped by the caller.
#include "common.cuh"
#include "counting_sort.cuh"

namespace vidar {
namespace {

constexpr int kEvalThreads = 256;

struct Range6 {
  float v[6];
};

// eval_utils.PC_RANGE and inside_volume's 0.02 m slack; numpy compares a float32 array against a Python
// float in float32, so the bounds are the float32 roundings of the double expressions.
__constant__ float kRange[6] = {-70.f, -70.f, -4.5f, 70.f, 70.f, 4.5f};
__constant__ float kSlack[6] = {(float)(-70.0 - 0.02), (float)(-70.0 - 0.02), (float)(-4.5 - 0.02),
                             (float)(70.0 + 0.02), (float)(70.0 + 0.02), (float)(4.5 + 0.02)};
constexpr float kMaxValue = 1e8f;

__device__ __forceinline__ float norm3(float x, float y, float z) {      // sqrt(x*x + y*y + z*z), numpy order
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

__device__ __forceinline__ float atan2_f64(float y, float x) { return (float)atan2((double)y, (double)x); }

__device__ __forceinline__ bool inside_slack(const float p[3]) {
  return kSlack[0] <= p[0] && p[0] <= kSlack[3] && kSlack[1] <= p[1] && p[1] <= kSlack[4] && kSlack[2] <= p[2] &&
         p[2] <= kSlack[5];
}

__device__ __forceinline__ bool inside_range(const float p[3]) {
  return kRange[0] <= p[0] && p[0] <= kRange[3] && kRange[1] <= p[1] && p[1] <= kRange[4] && kRange[2] <= p[2] &&
         p[2] <= kRange[5];
}

// np.isclose(d, 0.0): |d| <= 1e-8, compared in float64
__device__ __forceinline__ bool near_zero(float d) { return (double)fabsf(d) <= 1e-8; }

// Next plane in ascending distance after the ones in `done` (ties: lower plane index; NaN distances are never
// accepted by the callers, so they are skipped).  Returns -1 when none is left.
__device__ __forceinline__ int next_plane(const float t[6], unsigned done, float& tk) {
  int best = -1;
#pragma unroll
  for (int k = 0; k < 6; ++k)
    if (!(done >> k & 1u) && !isnan(t[k]) && (best < 0 || t[k] < tk)) { best = k; tk = t[k]; }
  return best;
}

enum { kClampOk = 0, kClampDegenerate = 1, kClampNoTouch = 2 };

// eval_utils.clamp for one point p against origin o: points inside PC_RANGE stay; every other point goes
// through _clamp (:81-174).  On return p is the clamped point and no its ray origin.
__device__ int clamp_point(float p[3], const float o[3], bool origin_inside, float no[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) no[a] = o[a];
  if (inside_range(p)) return kClampOk;
  const float e0 = __fsub_rn(p[0], o[0]), e1 = __fsub_rn(p[1], o[1]), e2 = __fsub_rn(p[2], o[2]);
  if (e0 == 0.f && e1 == 0.f && e2 == 0.f) return kClampDegenerate;
  const float l = norm3(e0, e1, e2);
  const float d[3] = {__fdiv_rn(e0, l), __fdiv_rn(e1, l), __fdiv_rn(e2, l)};
  bool hit = true;
  if (!origin_inside) {
    hit = false;
    float t[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const int a = k >> 1;
      const float bound = (k & 1) ? kRange[3 + a] : kRange[a];
      t[k] = near_zero(d[a]) ? kMaxValue : __fdiv_rn(__fsub_rn(bound, o[a]), d[a]);
    }
    unsigned done = 0;
    for (int r = 0; r < 6; ++r) {
      float tk = 0.f;
      const int k = next_plane(t, done, tk);
      if (k < 0) break;
      done |= 1u << k;
      if (__fadd_rn(tk, 1e-4f) >= 0.f) {
        float x[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) x[a] = __fadd_rn(o[a], __fmul_rn(tk, d[a]));
        if (inside_slack(x)) {
          hit = true;
#pragma unroll
          for (int a = 0; a < 3; ++a) no[a] = x[a];
          if (tk > l) {
#pragma unroll
            for (int a = 0; a < 3; ++a) p[a] = x[a];
          }
          break;
        }
      }
    }
  }
  if (!hit) {
#pragma unroll
    for (int a = 0; a < 3; ++a) no[a] = p[a] = INFINITY;
    return kClampOk;
  }
  if (inside_slack(p)) return kClampOk;
  float t[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const int a = k >> 1;
    const float bound = (k & 1) ? kRange[3 + a] : kRange[a];
    t[k] = near_zero(d[a]) ? kMaxValue : __fdiv_rn(__fsub_rn(bound, p[a]), -d[a]);
  }
  unsigned done = 0;
  for (int r = 0; r < 6; ++r) {
    float tk = 0.f;
    const int k = next_plane(t, done, tk);
    if (k < 0) break;
    done |= 1u << k;
    if (__fadd_rn(tk, 1e-4f) >= 0.f) {
      float x[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) x[a] = __fadd_rn(p[a], __fmul_rn(tk, -d[a]));
      if (inside_slack(x)) {
#pragma unroll
        for (int a = 0; a < 3; ++a) p[a] = x[a];
        return kClampOk;
      }
    }
  }
  return kClampNoTouch;
}

// One thread per input point (and per offset entry): fills the query / candidate buffers, masks and offsets.
__global__ void eval_prologue_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                     const float* __restrict__ origin, const int64_t* __restrict__ pred_off,
                                     const int64_t* __restrict__ gt_off, Range6 pc, float* __restrict__ qbuf,
                                     float* __restrict__ cbuf, unsigned char* __restrict__ q_mask,
                                     unsigned char* __restrict__ c_mask, int64_t* __restrict__ q_off,
                                     int64_t* __restrict__ c_off, int N, long long Pp, long long Pg) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t <= 3LL * N) {
    const int r = (int)(t / N), k = (int)(t % N);
    const int64_t pe = (r == 3) ? Pp : pred_off[k], ge = (r == 3) ? Pg : gt_off[k];
    // segment starts per region; t == 3N writes the end of the last region
    const int rr = (r == 3) ? 2 : r;
    q_off[t] = rr == 0 ? pe : rr == 1 ? Pp + ge : Pp + Pg + ge;
    c_off[t] = rr == 0 ? ge : rr == 1 ? Pg + pe : Pg + Pp + pe;
  }
  if (t >= Pp + Pg) return;
  const bool is_pred = t < Pp;
  const int64_t p = is_pred ? t : t - Pp;
  const int n = find_segment(is_pred ? pred_off : gt_off, N, p);
  const float* src = (is_pred ? pred : gt) + p * 3;
  const float x = src[0], y = src[1], z = src[2];
  const float v[3] = {x, y, z};
  // get_inside_mask (e2e_predictor_utils.py:146-160): torch compares in float32, bounds inclusive
  const bool inside = pc.v[0] <= x && x <= pc.v[3] && pc.v[1] <= y && y <= pc.v[4] && pc.v[2] <= z && z <= pc.v[5];
  // spherical_projection (eval_utils.py:177-182) of point - origin
  const float rx = __fsub_rn(x, origin[n * 3 + 0]), ry = __fsub_rn(y, origin[n * 3 + 1]),
              rz = __fsub_rn(z, origin[n * 3 + 2]);
  const float dist = norm3(rx, ry, rz);
  const float sph[3] = {atan2_f64(rx, ry), atan2_f64(rz, ry), 1.f};
  const bool far = dist > 1e-2f;
  // pred: query of the forward term, candidate of the backward term and of the spherical search;
  // gt:   candidate of the forward term, query of the backward term and of the spherical search
  const int64_t xyz_q = is_pred ? p : Pp + p;
  const int64_t xyz_c = is_pred ? Pg + p : p;
  float* sph_dst = is_pred ? cbuf + (Pg + Pp + p) * 3 : qbuf + (Pp + Pg + p) * 3;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    qbuf[xyz_q * 3 + a] = v[a];
    cbuf[xyz_c * 3 + a] = v[a];
    sph_dst[a] = sph[a];
  }
  q_mask[xyz_q] = inside;
  c_mask[xyz_c] = inside;
  if (is_pred) c_mask[Pg + Pp + p] = far;
  else q_mask[Pp + Pg + p] = far;
}

// Per (block, segment) partials: [a, b, c, flags].  Forward / backward Chamfer segments: a = sum of squared NN
// distances of the kept queries, b = their count.  Ray segments (one thread per gt point): a = sum l1,
// b = sum absrel, c = kept gt points (`count`), flags = VIDAR_EVAL_* of the failures the reference raises.
__global__ void __launch_bounds__(kEvalThreads)
eval_partials_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ origin,
                     const int64_t* __restrict__ pred_off, const int64_t* __restrict__ gt_off,
                     const int64_t* __restrict__ q_off, const unsigned char* __restrict__ q_mask,
                     const float* __restrict__ dists, const int64_t* __restrict__ idx, double* __restrict__ partials,
                     float* __restrict__ rays, int N) {
  __shared__ double red[kEvalThreads / 32];
  const int s = blockIdx.y, region = s / N, n = s % N;
  const int64_t q0 = q_off[s];
  const long long Lq = q_off[s + 1] - q0;
  if ((long long)blockIdx.x * kEvalThreads >= Lq) return;
  const long long i = (long long)blockIdx.x * kEvalThreads + threadIdx.x;
  const bool live = i < Lq && q_mask[q0 + i];
  double a = 0.0, b = 0.0, c = 0.0;
  unsigned flags = 0;
  if (region < 2) {
    if (live) { a = (double)dists[q0 + i]; b = 1.0; }
  } else if (i < Lq) {
    const int64_t g = gt_off[n] + i;
    float* ray = rays ? rays + g * 9 : nullptr;
    if (ray)
      for (int k = 0; k < 9; ++k) ray[k] = NAN;
    if (live) {
      c = 1.0;
      const int64_t j = idx[q0 + i];
      if (j < 0) {
        flags |= VIDAR_EVAL_NO_PRED;
      } else {
        const float o[3] = {origin[n * 3 + 0], origin[n * 3 + 1], origin[n * 3 + 2]};
        const float* pp = pred + (pred_off[n] + j) * 3;
        const float d_hat = norm3(__fsub_rn(pp[0], o[0]), __fsub_rn(pp[1], o[1]), __fsub_rn(pp[2], o[2]));
        float gp[3], ip[3], v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { gp[k] = gt[g * 3 + k]; v[k] = __fsub_rn(gp[k], o[k]); }
        const float vn = norm3(v[0], v[1], v[2]);
#pragma unroll
        for (int k = 0; k < 3; ++k) ip[k] = __fadd_rn(o[k], __fmul_rn(d_hat, __fdiv_rn(v[k], vn)));
        if (ray)
          for (int k = 0; k < 3; ++k) ray[k] = ip[k];
        const bool origin_inside = inside_slack(o);
        float go[3], io[3];
        const int rg = clamp_point(gp, o, origin_inside, go);
        const int ri = clamp_point(ip, o, origin_inside, io);
        if (rg == kClampDegenerate) flags |= VIDAR_EVAL_GT_DEGENERATE;
        if (rg == kClampNoTouch) flags |= VIDAR_EVAL_GT_OUTSIDE;
        if (ri == kClampDegenerate) flags |= VIDAR_EVAL_INTERP_DEGENERATE;
        if (ri == kClampNoTouch) flags |= VIDAR_EVAL_INTERP_OUTSIDE;
        if (ray)
          for (int k = 0; k < 3; ++k) { ray[3 + k] = gp[k]; ray[6 + k] = ip[k]; }
        const bool invalid = (isinf(gp[0]) && isinf(gp[1]) && isinf(gp[2])) ||
                             (isnan(gp[0]) && isnan(gp[1]) && isnan(gp[2]));
        if (!invalid && !flags) {
          const float dc = norm3(__fsub_rn(gp[0], go[0]), __fsub_rn(gp[1], go[1]), __fsub_rn(gp[2], go[2]));
          if (dc > 0.01f) {
            const float l1 = norm3(__fsub_rn(gp[0], ip[0]), __fsub_rn(gp[1], ip[1]), __fsub_rn(gp[2], ip[2]));
            a = (double)l1;
            b = (double)__fdiv_rn(l1, dc);
          }
        }
      }
    }
  }
  a = block_sum<kEvalThreads>(a, red);
  b = block_sum<kEvalThreads>(b, red);
  c = block_sum<kEvalThreads>(c, red);
  flags = __reduce_or_sync(0xffffffffu, flags);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = (double)flags;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned f = 0;
    for (int w = 0; w < kEvalThreads / 32; ++w) f |= (unsigned)red[w];
    double* dst = partials + ((size_t)s * gridDim.x + blockIdx.x) * 4;
    dst[0] = a; dst[1] = b; dst[2] = c; dst[3] = (double)f;
  }
}

// One thread per (sample, frame): the blocks of its three segments, in block order.
__global__ void eval_finish_kernel(const int64_t* __restrict__ q_off, const double* __restrict__ partials,
                                   double* __restrict__ out, int N, int nbx) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double acc[3][3] = {};
  unsigned flags = 0;
  for (int r = 0; r < 3; ++r) {
    const int s = r * N + n;
    const long long Lq = q_off[s + 1] - q_off[s];
    int nb = (int)((Lq + kEvalThreads - 1) / kEvalThreads);
    if (nb > nbx) nb = nbx;      // only a fully masked segment (decode_clouds' trailing one) is longer than max_len
    for (int bx = 0; bx < nb; ++bx) {
      const double* p = partials + ((size_t)s * nbx + bx) * 4;
      acc[r][0] += p[0]; acc[r][1] += p[1]; acc[r][2] += p[2];
      flags |= (unsigned)p[3];
    }
  }
  double* o = out + (size_t)n * VIDAR_EVAL_FIELDS;
  o[0] = acc[2][0]; o[1] = acc[2][1]; o[2] = acc[2][2];     // sum l1, sum absrel, count
  o[3] = acc[0][0]; o[4] = acc[0][1];                       // sum forward d, pred points inside
  o[5] = acc[1][0]; o[6] = acc[1][1];                       // sum backward d, gt points inside
  o[7] = (double)flags;
}

// ------------------------------------------------------------------ decoded rays -> per-(sample, frame) clouds
struct DecodeDims {
  int bs, M, F, nchunk, within;
  float scale;      // (pc_range[3] - pc_range[0]) / bev_w, as torch rounds the Python float
  float pc[6];
};

// Frame t of row i of sample b when the row joins cloud b * F + t, else -1; gt_dist (metres) of a joining row.
// gt_dist = sqrt(sum (g_vox - o_vox)^2) * scale (ray_head.decode_ray_depth, then `gt_dist * scale`).
__device__ __forceinline__ int decode_frame(const DecodeDims& D, const float* __restrict__ rays,
                                            const float* __restrict__ points, const float* __restrict__ tindex,
                                            const float* __restrict__ origin_vox, int b, int i, float& gt_dist) {
  const size_t k = (size_t)b * D.M + i;
  const float t = tindex[k];
  if (!(t >= 0.f && t < (float)D.F && t == floorf(t))) return -1;
  const int f = (int)t;
  const float* o = origin_vox + ((size_t)b * D.F + f) * 3;
  const float* g = rays + k * 3;
  gt_dist = __fmul_rn(norm3(__fsub_rn(g[0], o[0]), __fsub_rn(g[1], o[1]), __fsub_rn(g[2], o[2])), D.scale);
  if (!(gt_dist > 0.f)) return -1;
  if (D.within) {     // get_inside_mask on the metre point, float32 bounds, inclusive
    const float* p = points + k * 3;
    if (!(D.pc[0] <= p[0] && p[0] <= D.pc[3] && D.pc[1] <= p[1] && p[1] <= D.pc[4] && D.pc[2] <= p[2] &&
          p[2] <= D.pc[5]))
      return -1;
  }
  return f;
}

// grid (nchunk, bs): per-(cloud, chunk) row counts
__global__ void __launch_bounds__(kSortChunk)
decode_count_kernel(DecodeDims D, const float* __restrict__ rays, const float* __restrict__ points,
                    const float* __restrict__ tindex, const float* __restrict__ origin_vox, int* __restrict__ counts) {
  extern __shared__ int hist[];       // [32][F]
  const int b = blockIdx.y, c = blockIdx.x, i = c * kSortChunk + threadIdx.x;
  float gd = 0.f;
  const int f = i < D.M ? decode_frame(D, rays, points, tindex, origin_vox, b, i, gd) : -1;
  sort_count(f, D.F, b, c, D.nchunk, hist, counts);
}

// One block: cloud offsets off[0..N] (cloud n = slot b * F + t), then off[N + 1] = bs * M closes the trailing segment.
__global__ void decode_offsets_kernel(DecodeDims D, int* __restrict__ counts, int64_t* __restrict__ off) {
  const int N = D.bs * D.F;
  sort_offsets(N, D.nchunk, counts, off);
  if (threadIdx.x == 0) off[N + 1] = (int64_t)D.bs * D.M;
}

// grid as the count kernel: every joining row to its place in its cloud, both points rendered from the metre
// origin o and point p with get_rendered_pcds' statements, o + ((p - o) / sqrt(sum (p - o)^2)) * dist, for
// dist = depth * scale (pred) and gt_dist (gt).  Rows [off[N], bs * M) of both clouds are NaN.
__global__ void __launch_bounds__(kSortChunk)
decode_scatter_kernel(DecodeDims D, const float* __restrict__ depth, const float* __restrict__ rays,
                      const float* __restrict__ points, const float* __restrict__ tindex,
                      const float* __restrict__ origin_vox, const float* __restrict__ origin,
                      const int* __restrict__ counts, const int64_t* __restrict__ off, float* __restrict__ pred,
                      float* __restrict__ gt) {
  extern __shared__ int hist[];
  const int b = blockIdx.y, c = blockIdx.x, i = c * kSortChunk + threadIdx.x;
  float gd = 0.f;
  const int f = i < D.M ? decode_frame(D, rays, points, tindex, origin_vox, b, i, gd) : -1;
  const int pos = sort_rank(f, D.F, hist);
  const int64_t r = (int64_t)b * D.M + i;
  if (i < D.M && r >= off[D.bs * D.F]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) pred[r * 3 + a] = gt[r * 3 + a] = NAN;
  }
  if (f < 0) return;
  const int n = b * D.F + f;
  const int64_t dst = off[n] + counts[(size_t)n * D.nchunk + c] + pos;
  const float* o = origin + (size_t)n * 3;
  const float* p = points + r * 3;
  const float v[3] = {__fsub_rn(p[0], o[0]), __fsub_rn(p[1], o[1]), __fsub_rn(p[2], o[2])};
  const float len = norm3(v[0], v[1], v[2]);
  const float pd = __fmul_rn(depth[r], D.scale);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float u = __fdiv_rn(v[a], len);
    pred[dst * 3 + a] = __fadd_rn(o[a], __fmul_rn(u, pd));
    gt[dst * 3 + a] = __fadd_rn(o[a], __fmul_rn(u, gd));
  }
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_eval_decode_clouds(const float* depth, const float* rays, const float* points,
                                        const float* tindex, const float* origin_vox, const float* origin,
                                        const float* pc_range_host, float scale, int within_grid, float* pred,
                                        float* gt, int64_t* off, int bs, int M, int F, void* stream) {
  const char* who = "eval_decode_clouds";
  VIDAR_REQUIRE(bs > 0 && M >= 0 && F > 0 && F <= 64, "%s: bad sizes bs=%d M=%d F=%d (F <= 64)", who, bs, M, F);
  VIDAR_REQUIRE(bs <= 65535 && (long long)bs * F + 1 <= 65535 / 3, "%s: %lld clouds, at most %d", who,
                (long long)bs * F, 65535 / 3 - 1);
  VIDAR_REQUIRE((long long)bs * M < (1LL << 31), "%s: %lld rows, at most 2^31 - 1", who, (long long)bs * M);
  VIDAR_REQUIRE(off && (M == 0 || (depth && rays && points && tindex && origin_vox && origin && pred && gt)),
                "%s: null pointer argument", who);
  VIDAR_REQUIRE(!within_grid || pc_range_host, "%s: within_grid needs pc_range", who);
  DecodeDims D{};
  D.bs = bs; D.M = M; D.F = F; D.within = within_grid ? 1 : 0; D.scale = scale;
  D.nchunk = (M + kSortChunk - 1) / kSortChunk;
  if (within_grid)
    for (int k = 0; k < 6; ++k) D.pc[k] = pc_range_host[k];
  cudaStream_t st = (cudaStream_t)stream;
  const int N = bs * F;
  const size_t bytes = sizeof(int) * ((size_t)N * D.nchunk + 1);
  cudaMemPool_t pool;
  cudaError_t e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  int* counts = nullptr;
  e = cudaMallocFromPoolAsync((void**)&counts, bytes, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  const dim3 grid(D.nchunk, bs);
  const size_t smem = sizeof(int) * 32 * F;
  int rc = VIDAR_OK;
  if (M > 0) {
    decode_count_kernel<<<grid, kSortChunk, smem, st>>>(D, rays, points, tindex, origin_vox, counts);
    rc = check_launch("eval_decode_clouds(count)");
  }
  if (!rc) {
    decode_offsets_kernel<<<1, 256, 0, st>>>(D, counts, off);
    rc = check_launch("eval_decode_clouds(offsets)");
  }
  if (!rc && M > 0) {
    decode_scatter_kernel<<<grid, kSortChunk, smem, st>>>(D, depth, rays, points, tindex, origin_vox, origin, counts,
                                                          off, pred, gt);
    rc = check_launch("eval_decode_clouds(scatter)");
  }
  e = cudaFreeAsync(counts, st);
  if (rc) return rc;
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(e));
  return VIDAR_OK;
}

extern "C" int vidar_eval_prologue(const float* pred, const float* gt, const float* origin, const int64_t* pred_off,
                                   const int64_t* gt_off, const float* pc_range_host, float* qbuf, float* cbuf,
                                   unsigned char* q_mask, unsigned char* c_mask, int64_t* q_off, int64_t* c_off,
                                   int N, long long Pp, long long Pg, void* stream) {
  VIDAR_REQUIRE(origin && pred_off && gt_off && pc_range_host && q_off && c_off,
                "eval_prologue: null pointer argument");
  VIDAR_REQUIRE(N > 0 && N <= 65535 / 3 && Pp >= 0 && Pg >= 0 && Pp < (1LL << 31) && Pg < (1LL << 31),
                "eval_prologue: bad sizes N=%d Pp=%lld Pg=%lld", N, Pp, Pg);
  VIDAR_REQUIRE((Pp == 0 || pred) && (Pg == 0 || gt), "eval_prologue: null point buffer");
  VIDAR_REQUIRE((Pp + Pg == 0) || (qbuf && cbuf && q_mask && c_mask), "eval_prologue: null output buffer");
  Range6 pc;
  for (int k = 0; k < 6; ++k) pc.v[k] = pc_range_host[k];
  const long long total = (Pp + Pg > 3LL * N + 1) ? Pp + Pg : 3LL * N + 1;
  eval_prologue_kernel<<<(unsigned)((total + kEvalThreads - 1) / kEvalThreads), kEvalThreads, 0,
                         (cudaStream_t)stream>>>(pred, gt, origin, pred_off, gt_off, pc, qbuf, cbuf, q_mask, c_mask,
                                                 q_off, c_off, N, Pp, Pg);
  return check_launch("eval_prologue");
}

extern "C" int vidar_eval_metrics(const float* pred, const float* gt, const float* origin, const int64_t* pred_off,
                                  const int64_t* gt_off, const int64_t* q_off, const unsigned char* q_mask,
                                  const float* dists, const int64_t* idx, double* partials, double* out,
                                  float* rays, int N, int max_len, void* stream) {
  VIDAR_REQUIRE(origin && pred_off && gt_off && q_off && partials && out, "eval_metrics: null pointer argument");
  VIDAR_REQUIRE(N > 0 && N <= 65535 / 3 && max_len >= 0, "eval_metrics: bad sizes N=%d max_len=%d", N, max_len);
  cudaStream_t st = (cudaStream_t)stream;
  const int nbx = (max_len + kEvalThreads - 1) / kEvalThreads;
  if (nbx > 0) {
    VIDAR_REQUIRE(pred && gt && q_mask && dists && idx, "eval_metrics: null point / search buffer");
    eval_partials_kernel<<<dim3(nbx, 3 * N), kEvalThreads, 0, st>>>(pred, gt, origin, pred_off, gt_off, q_off,
                                                                     q_mask, dists, idx, partials, rays, N);
    int rc = check_launch("eval_metrics(partials)");
    if (rc) return rc;
  }
  eval_finish_kernel<<<(N + 127) / 128, 128, 0, st>>>(q_off, partials, out, N, nbx);
  return check_launch("eval_metrics(finish)");
}
