// The point half of a ViDAR pre-training sample (vidar_b200/point_pipeline.py, include/vidar_b200.h §xi): the
// multi-sweep merge of CustomLoadPointsFromMultiSweeps, the first-occurrence voxel sampler of
// CustomVoxelBasedPointSampler (mmdet3d's _points_to_voxel_reverse_kernel with max_points = 1) and union2one's ego
// mask / queue-index column, for every frame of a queue in one fixed sequence of launches.
//
// Index spaces (all global over the call, frame-major):
//   g  over the uploaded segments' raw points, segment after segment.  A segment is a raw [n, cols] float32 array
//      (cols 5: nuScenes' x, y, z, intensity, time; cols 6: nuPlan's x, y, z, intensity, ring, lidar_info),
//      optionally filtered (remove-close, then an optional ego box, float32 comparisons on the raw x / y) and
//      optionally moved into the key frame's LiDAR coordinates (f32(f32(dot64(p, R[i])) + t64[i])).
//   m  over the merged points: the survivors of g in g's order (an exclusive scan of the keep flags), so each frame's
//      merged cloud is its key frame followed by its sweeps, as the reference concatenates them.
//   k  over shuffled slots: frame f's slot k reads merged point cur_off_f + perm[k] (numpy's draws, made on the host).
// A voxel frame keeps slot k when k is the smallest slot of its voxel (atomicMin into the frame's grid), and writes
// it to row out_off_f + (number of kept slots before k) when that rank is below max_voxels: the voxels in the order
// numba first meets them.  A frame without the sampler keeps every slot in merged order.  Kept points inside the
// union2one ego box become NaN rows; every row not written stays NaN.  A row is (x, y, z, intensity, queue index)
// with 5 columns, (x, y, z, intensity, column 4, queue index) with 6: union2one overwrites the last column.  With 6
// columns, column 4 is the segment's time (LoadPointsFromMultiSweeps sets it: 0 for the key frame, ts - sweep_ts for a
// sweep; the sampler's time_dim reads it) or, without the multi-sweep step, the raw column 4.
#include <cub/device/device_scan.cuh>
#include <math.h>

#include "common.cuh"

namespace vidar {
namespace {

constexpr int kThreads = 256;
constexpr long long kMaxCellsPerFrame = 1LL << 24;   // voxel grid cap: 64 MB of uint32 per frame
constexpr int kSegD = 17;

// seg_i [S, 5] int64: raw row offset, n, g offset, filter (0 none, 1 close, 2 close + ego box), flags (bit 0: the
//   sweep transform; bit 1: column 4 := the segment's time, 6 columns only)
// seg_d [S, 17] double: R row-major (9), t (3), ego box (x_lo, y_lo, x_hi, y_hi; float32 values), time (float32 value)
// frame_i [F, 10] int64: cur_off (m and k), n_cur, out_off, cap = rows of the frame, queue index, voxel (0 / 1),
//   grid_off, perm_off, g_off, g_n
// frame_f [F, 6] float: lo (3), voxel size (3);  frame_g [F, 3] int64: grid dims (x, y, z)
struct Tables {
  const float* raw;
  const int64_t* seg_i;
  const double* seg_d;
  const int64_t* frame_i;
  const float* frame_f;
  const int64_t* frame_g;
  const int32_t* perm;
  int S, F, cols;
};

__device__ __forceinline__ int find_seg(const Tables& t, long long g) {
  int lo = 0, hi = t.S - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.seg_i[mid * 5 + 2] <= g) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ int find_frame(const Tables& t, long long k) {
  int lo = 0, hi = t.F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.frame_i[mid * 10 + 0] <= k) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) pp_init_kernel(unsigned* grid, long long cells, float* out, long long outn,
                                                           int* keep, long long rows) {
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < cells || i < outn; i += stride) {
    if (i < cells) grid[i] = 0xffffffffu;
    if (i < outn) out[i] = __int_as_float(0x7fc00000);
    if (i < rows) keep[i] = 0;
  }
}

// remove-close (|x| < 1 and |y| < 1) then, with filter 2, the ego box: CustomLoadPointsFromMultiSweeps._remove_close
__global__ void __launch_bounds__(kThreads) pp_filter_kernel(const Tables t, long long n, int* flag) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n) return;
  const int s = find_seg(t, g);
  const int64_t* si = t.seg_i + s * 5;
  const float* p = t.raw + (si[0] + (g - si[2])) * t.cols;
  const float x = p[0], y = p[1];
  int keep = 1;
  if (si[3] >= 1) {
    keep = !(fabsf(x) < 1.f && fabsf(y) < 1.f);
    if (keep && si[3] == 2) {
      const double* b = t.seg_d + s * kSegD + 12;
      keep = !((float)b[0] <= x && (float)b[2] >= x && (float)b[1] <= y && (float)b[3] >= y);
    }
  }
  flag[g] = keep;
}

// The sweep transform `pts[:, :3] @ R.T` in float64 rounded to float32 on assignment, then `+= t` in float64 rounded
// again; the products and sums are explicit so that nothing is contracted into an fma.
__global__ void __launch_bounds__(kThreads) pp_merge_kernel(const Tables t, long long n, const int* flag,
                                                            const int* pos, float4* merged, float* merged4,
                                                            long long n_cur) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n || !flag[g]) return;
  const long long m = pos[g];
  if (m >= n_cur) return;
  const int s = find_seg(t, g);
  const int64_t* si = t.seg_i + s * 5;
  const float* p = t.raw + (si[0] + (g - si[2])) * t.cols;
  float4 q = make_float4(p[0], p[1], p[2], p[3]);
  if (t.cols == 6) merged4[m] = (si[4] & 2) ? (float)t.seg_d[s * kSegD + 16] : p[4];
  if (si[4] & 1) {
    const double* d = t.seg_d + s * kSegD;
    const double x = q.x, y = q.y, z = q.z;
    float r[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double dot = __dadd_rn(__dadd_rn(__dmul_rn(x, d[3 * i]), __dmul_rn(y, d[3 * i + 1])), __dmul_rn(z, d[3 * i + 2]));
      r[i] = __double2float_rn(__dadd_rn((double)__double2float_rn(dot), d[9 + i]));
    }
    q.x = r[0];
    q.y = r[1];
    q.z = r[2];
  }
  merged[m] = q;
}

// Voxel coordinate of q in frame f, numba's float32 statements: floor(f32(f32(p - lo) / vs)), -1 when outside the
// grid (a non-finite coordinate counts as outside).
__device__ __forceinline__ long long voxel_of(const Tables& t, int f, float4 q) {
  const float* ff = t.frame_f + f * 6;
  const int64_t* gd = t.frame_g + f * 3;
  const float v[3] = {q.x, q.y, q.z};
  long long c[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float cf = floorf(__fdiv_rn(__fsub_rn(v[j], ff[j]), ff[3 + j]));
    if (!(cf >= 0.f && cf < (float)gd[j])) return -1;
    c[j] = (long long)cf;
  }
  return (c[2] * gd[1] + c[1]) * gd[0] + c[0];
}

__device__ __forceinline__ long long merged_index(const Tables& t, const int64_t* fi, long long kl) {
  return fi[0] + (fi[5] ? (long long)t.perm[fi[7] + kl] : kl);
}

__global__ void __launch_bounds__(kThreads) pp_voxel_kernel(const Tables t, long long n_cur, const float4* merged,
                                                            unsigned* grid, long long* vox) {
  const long long k = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (k >= n_cur) return;
  const int f = find_frame(t, k);
  const int64_t* fi = t.frame_i + f * 10;
  if (!fi[5]) return;
  const long long kl = k - fi[0];
  const long long cell = voxel_of(t, f, merged[merged_index(t, fi, kl)]);
  vox[k] = cell < 0 ? -1 : fi[6] + cell;
  if (cell >= 0) atomicMin(grid + fi[6] + cell, (unsigned)kl);
}

__global__ void __launch_bounds__(kThreads) pp_winner_kernel(const Tables t, long long n_cur, const unsigned* grid,
                                                             const long long* vox, int* win) {
  const long long k = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (k >= n_cur) return;
  const int f = find_frame(t, k);
  const int64_t* fi = t.frame_i + f * 10;
  if (!fi[5]) {
    win[k] = 1;
    return;
  }
  const long long v = vox[k];
  win[k] = v >= 0 && grid[v] == (unsigned)(k - fi[0]);
}

// Writes the kept slots.  With counts, thread f < F also writes frame f's merged points (from the merge's scan) and
// kept slots (from the sampler's scan), so a caller can compare them with the host's counts.
__global__ void __launch_bounds__(kThreads) pp_emit_kernel(const Tables t, long long n_cur, const float4* merged,
                                                           const float* merged4, const int* win, const int* rank, const int* flag,
                                                           const int* pos, float ego0, float ego1, float ego2,
                                                           float ego3, int use_ego, float* out, int* keep,
                                                           int* counts) {
  const long long k = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (counts && k < t.F) {
    const int64_t* fi = t.frame_i + k * 10;
    const long long a = fi[0], b = fi[0] + fi[1], ga = fi[8], gb = fi[8] + fi[9];
    counts[2 * k] = fi[9] ? (int)(pos[gb - 1] + flag[gb - 1] - pos[ga]) : 0;
    const long long kept = fi[1] ? rank[b - 1] + win[b - 1] - rank[a] : 0;
    counts[2 * k + 1] = (int)(kept < fi[3] ? kept : fi[3]);
  }
  if (k >= n_cur || !win[k]) return;
  const int f = find_frame(t, k);
  const int64_t* fi = t.frame_i + f * 10;
  const long long r = rank[k] - rank[fi[0]];
  if (r >= fi[3]) return;
  const long long m = merged_index(t, fi, k - fi[0]);
  const float4 q = merged[m];
  const long long row = fi[2] + r;
  if (use_ego && ego0 <= q.x && ego2 >= q.x && ego1 <= q.y && ego3 >= q.y) return;
  float* o = out + row * t.cols;
  o[0] = q.x;
  o[1] = q.y;
  o[2] = q.z;
  o[3] = q.w;
  if (t.cols == 6) o[4] = merged4[m];
  o[t.cols - 1] = (float)fi[4];
  keep[row] = 1;
}

__global__ void __launch_bounds__(kThreads) pp_compact_kernel(const float* out, const int* keep, const int* cpos,
                                                              long long rows, int cols, float* outc, int64_t* count) {
  const long long r = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (r >= rows) return;
  if (r == rows - 1) *count = (int64_t)cpos[r] + keep[r];
  if (!keep[r]) return;
  const float* a = out + r * cols;
  float* b = outc + (long long)cpos[r] * cols;
  for (int j = 0; j < cols; ++j) b[j] = a[j];
}

inline unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_point_pipeline_gather(const float* raw, const int64_t* seg_i, const double* seg_d, int S,
                                           const int64_t* frame_i, const float* frame_f, const int64_t* frame_g, int F,
                                           const int32_t* perm, long long n_g, long long n_cur, long long cells,
                                           const float* ego, float* out, long long rows, int32_t* counts,
                                           float* out_compact, int64_t* count, int cols, void* stream) {
  const char* who = "point_pipeline_gather";
  VIDAR_REQUIRE(S >= 1 && F >= 1 && n_g >= 0 && n_cur >= 0 && n_cur <= n_g && rows >= 0 && cells >= 0,
                "%s: bad sizes (S %d, F %d, points %lld, merged %lld, rows %lld, cells %lld)", who, S, F, n_g, n_cur,
                rows, cells);
  VIDAR_REQUIRE(cols == 5 || cols == 6, "%s: rows of 5 or 6 columns (got %d)", who, cols);
  VIDAR_REQUIRE(n_g < INT_MAX && rows < INT_MAX && rows * cols < (1LL << 40) && cells <= kMaxCellsPerFrame * F,
                "%s: %lld points, %lld rows or %lld voxel cells is too many", who, n_g, rows, cells);
  VIDAR_REQUIRE(seg_i && seg_d && frame_i && frame_f && frame_g && (raw || n_g == 0) && (out || rows == 0) &&
                    (perm || n_cur == 0) && ((!out_compact) == (!count) || (rows == 0 && count)),
                "%s: null pointer argument", who);
  VIDAR_REQUIRE(((uintptr_t)seg_i | (uintptr_t)seg_d | (uintptr_t)frame_i | (uintptr_t)frame_g) % 8 == 0 &&
                    ((uintptr_t)raw | (uintptr_t)frame_f | (uintptr_t)out | (uintptr_t)perm) % 4 == 0,
                "%s: misaligned table", who);
  cudaStream_t st = (cudaStream_t)stream;
  if (count && rows == 0 && cudaMemsetAsync(count, 0, sizeof(int64_t), st) != cudaSuccess)
    return set_error(VIDAR_E_CUDA, "%s: cudaMemsetAsync failed", who);
  const Tables t{raw, seg_i, seg_d, frame_i, frame_f, frame_g, perm, S, F, cols};
  const long long n_scan = n_g > rows ? n_g : rows;
  size_t tmp = 0;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const int*)nullptr, (int*)nullptr, (int)(n_scan + 1), st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scan: %s", who, cudaGetErrorString(e));
  const size_t b_flag = align256(sizeof(int) * (n_g + 1)), b_merged = align256(sizeof(float4) * (n_cur + 1));
  const size_t b_merged4 = cols == 6 ? align256(sizeof(float) * (n_cur + 1)) : 0;
  const size_t b_vox = align256(sizeof(long long) * (n_cur + 1)), b_win = align256(sizeof(int) * (n_cur + 1));
  const size_t b_grid = align256(sizeof(unsigned) * (cells + 1)), b_rows = align256(sizeof(int) * (rows + 1));
  const size_t total = 2 * b_flag + b_merged + b_merged4 + b_vox + 2 * b_win + b_grid + 2 * b_rows + align256(tmp);
  cudaMemPool_t pool;
  e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, total, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  unsigned char* c = s;
  int* flag = (int*)c;
  c += b_flag;
  int* pos = (int*)c;
  c += b_flag;
  float4* merged = (float4*)c;
  c += b_merged;
  float* merged4 = b_merged4 ? (float*)c : nullptr;
  c += b_merged4;
  long long* vox = (long long*)c;
  c += b_vox;
  int* win = (int*)c;
  c += b_win;
  int* rank = (int*)c;
  c += b_win;
  unsigned* grid = (unsigned*)c;
  c += b_grid;
  int* keep = (int*)c;
  c += b_rows;
  int* cpos = (int*)c;
  c += b_rows;
  void* scan_tmp = c;

  int rc = VIDAR_OK;
  const long long outn = rows * cols, init_n = cells > outn ? cells : outn;
  const float e0 = ego ? ego[0] : 0.f, e1 = ego ? ego[1] : 0.f, e2 = ego ? ego[2] : 0.f, e3 = ego ? ego[3] : 0.f;
  do {
    unsigned ib = blocks_for(init_n);
    ib = ib < 4096 ? (ib ? ib : 1) : 4096;
    pp_init_kernel<<<ib, kThreads, 0, st>>>(grid, cells, out, outn, keep, rows);
    if ((rc = check_launch(who)) != VIDAR_OK) break;
    if (n_g > 0) {
      pp_filter_kernel<<<blocks_for(n_g), kThreads, 0, st>>>(t, n_g, flag);
      if ((rc = check_launch(who)) != VIDAR_OK) break;
      e = cub::DeviceScan::ExclusiveSum(scan_tmp, tmp, flag, pos, (int)n_g, st);
      if (e != cudaSuccess) {
        rc = set_error(VIDAR_E_CUDA, "%s: scan: %s", who, cudaGetErrorString(e));
        break;
      }
      pp_merge_kernel<<<blocks_for(n_g), kThreads, 0, st>>>(t, n_g, flag, pos, merged, merged4, n_cur);
      if ((rc = check_launch(who)) != VIDAR_OK) break;
    }
    if (n_cur > 0) {
      pp_voxel_kernel<<<blocks_for(n_cur), kThreads, 0, st>>>(t, n_cur, merged, grid, vox);
      if ((rc = check_launch(who)) != VIDAR_OK) break;
      pp_winner_kernel<<<blocks_for(n_cur), kThreads, 0, st>>>(t, n_cur, grid, vox, win);
      if ((rc = check_launch(who)) != VIDAR_OK) break;
      e = cub::DeviceScan::ExclusiveSum(scan_tmp, tmp, win, rank, (int)n_cur, st);
      if (e != cudaSuccess) {
        rc = set_error(VIDAR_E_CUDA, "%s: scan: %s", who, cudaGetErrorString(e));
        break;
      }
    }
    const long long emit_n = n_cur > F ? n_cur : F;
    pp_emit_kernel<<<blocks_for(emit_n), kThreads, 0, st>>>(t, n_cur, merged, merged4, win, rank, flag, pos, e0, e1, e2, e3,
                                                             ego != nullptr, out, keep, counts);
    if ((rc = check_launch(who)) != VIDAR_OK) break;
    if (out_compact && rows > 0) {
      e = cub::DeviceScan::ExclusiveSum(scan_tmp, tmp, keep, cpos, (int)rows, st);
      if (e != cudaSuccess) {
        rc = set_error(VIDAR_E_CUDA, "%s: scan: %s", who, cudaGetErrorString(e));
        break;
      }
      pp_compact_kernel<<<blocks_for(rows), kThreads, 0, st>>>(out, keep, cpos, rows, cols, out_compact, count);
      if ((rc = check_launch(who)) != VIDAR_OK) break;
    }
  } while (0);
  const cudaError_t ef = cudaFreeAsync(s, st);
  if (rc != VIDAR_OK) return rc;
  if (ef != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(ef));
  return VIDAR_OK;
}
