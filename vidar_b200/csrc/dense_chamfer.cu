// The dense loss term of the ViDAR head ('loss.dense_voxel'), H100 (sm_90a): the Chamfer distance between the
// gumbel-decoded dense rays and the GT cloud of every (sample, frame) pair of a batch, forward and backward, in a
// fixed number of launches and without a host sync.  Also the GT alignment of ViDARHeadV1, which reuses the same
// stable counting sort.
//
// Reference: dense_heads/vidar_head_base.py:594-659 (per-pair loop over boolean masks), get_rendered_pcds
// :344-389, mmdet3d chamfer_distance (criterion 'l2', reduction 'mean').  Per pair n:
//   pred = {((o + unit(p - o) * d) - o) * 0.1 : rays n*R0 .. (n+1)*R0-1 with d > 0
//           [and p inside pc_range when eval_within_grid]}
//   gt   = {(g - o) * 0.1 : rows of the pair's (gt sample, frame) slot, 0 < x < W-1, 0 < y < H-1, 0 < z < Z-1}
//   loss[group] = sum_{n in group} w_n * (mean_pred min_gt |.|^2 + mean_gt min_pred |.|^2) / 2 / norm[group],
//          pairs without gt skipped; gt but no pred gives NaN like the per-pair path.
// Pairs come from a device pair table.  ViDARRayHead: pair n = b * F + f, one group, norm = sum(loss_weight) * bs;
// ViDARHeadV1: one group per head frame, pairs of zero weight left out.
// fp32 statements in the reference's order with explicit _rn intrinsics (no FMA contraction).
//
// Layout (P pairs; Pp = P * R0 dense rays; G = gt points kept; Pq = Pp + Sg * M buffer rows):
//   qbuf [pred (Pp) | gt (G) | unused]   segments 0..P-1: pred queries (masked, not compacted), P..2P-1: gt queries
//   cbuf [gt (G) | pred (Pp) | unused]   the candidates of the same segments
// so one call of the segmented NN search (knn.cu) serves both directions.  The gt rows of a sample arrive in any
// frame order; they are compacted per (gt sample, frame) slot by a stable counting sort (chunk histograms, a scan,
// a scatter that ranks inside a chunk with warp matches), so the original order inside a pair decides NN ties, as
// in the per-pair path.  Pairs are in slot order, and slots without a pair count no rows, so the pairs' gt
// segments are contiguous.
//
// Launches: forward 7 (histogram + pred points, offsets, scatter, NN search 2, partial sums, finish), backward 1,
// whatever the pair count.  Sums are fp64 in a fixed order (per-block tree, blocks of a segment in order, pairs in
// order), so two calls give the same bits; the backward scatters into grad_dist with red.global.add.f32 like the
// per-pair path's knn backward.
#include "common.cuh"
#include "counting_sort.cuh"

namespace vidar {
namespace {

constexpr int kChunk = kSortChunk;    // gt rows per block of the counting sort, one per thread (32 warps)
constexpr int kSumThreads = 256;
constexpr int kMaxFrames = 64;
constexpr int kMaxJobs = 256;         // (head frame, slot) jobs of the GT alignment

// ------------------------------------------------------------------ dense Chamfer
struct DenseDims {
  int P, Sg, Fg, R0, M, W, H, Z, within, nchunk, groups;
  long long Pp, Pq;
  float pc[6];
};

// the device pair table, pairs in increasing slot order
struct PairTable {
  const int32_t* slots;               // [Sg * Fg] pair of each (gt sample, frame) slot, -1 = none
  const int32_t* tab;                 // [P, 3] slot, origin row, group
  const float* w;                     // [P]
  const float* norm;                  // [groups]
  __device__ int slot_pair(int slot) const { return slots[slot]; }
  __device__ int slot(int n) const { return tab[n * 3]; }
  __device__ int origin_row(int n) const { return tab[n * 3 + 1]; }
  __device__ float weight(int n) const { return w[n]; }
  __device__ int group(int n) const { return tab[n * 3 + 2]; }
  __device__ float norm_of(int g) const { return norm[g]; }
};

// frame of gt row i of gt sample s, or -1 when the row belongs to no pair (padding, other frames, outside the box)
__device__ __forceinline__ int gt_frame(const DenseDims& D, const PairTable& Pr, const float* __restrict__ gt,
                                        const float* __restrict__ tindex, int s, int i) {
  const size_t k = (size_t)s * D.M + i;
  const float t = tindex[k];
  const float x = gt[k * 3], y = gt[k * 3 + 1], z = gt[k * 3 + 2];
  const bool box = x < (float)(D.W - 1) && x > 0.f && y < (float)(D.H - 1) && y > 0.f && z < (float)(D.Z - 1) &&
                   z > 0.f;
  const int f = (box && t >= 0.f && t < (float)D.Fg && t == floorf(t)) ? (int)t : -1;
  return (f >= 0 && Pr.slot_pair(s * D.Fg + f) >= 0) ? f : -1;
}

// unit(p - o): r / sqrt((r_x^2 + r_y^2) + r_z^2)
__device__ __forceinline__ void ray_unit(const float* p, const float* o, float u[3]) {
  const float r[3] = {__fsub_rn(p[0], o[0]), __fsub_rn(p[1], o[1]), __fsub_rn(p[2], o[2])};
  const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], r[0]), __fmul_rn(r[1], r[1])), __fmul_rn(r[2], r[2])));
#pragma unroll
  for (int a = 0; a < 3; ++a) u[a] = __fdiv_rn(r[a], n);
}

// grid (Sg * nchunk + pred blocks).  gt chunks: per-(slot, chunk) counts of kept rows.  Pred blocks: the pred
// points of every ray into qbuf (row k = ray k) and their query mask.
__global__ void __launch_bounds__(kChunk)
dense_count_kernel(DenseDims D, PairTable Pr, const float* __restrict__ dist, const float* __restrict__ points,
                   const float* __restrict__ origin, const float* __restrict__ gt, const float* __restrict__ tindex,
                   int* __restrict__ counts, float* __restrict__ qbuf, unsigned char* __restrict__ q_mask) {
  extern __shared__ int hist[];       // [32][Fg]
  const int ng = D.Sg * D.nchunk;
  if ((int)blockIdx.x < ng) {
    const int s = blockIdx.x / D.nchunk, c = blockIdx.x % D.nchunk, i = c * kChunk + threadIdx.x;
    const int f = i < D.M ? gt_frame(D, Pr, gt, tindex, s, i) : -1;
    sort_count(f, D.Fg, s, c, D.nchunk, hist, counts);
    return;
  }
  const long long k = (long long)(blockIdx.x - ng) * kChunk + threadIdx.x;
  if (k >= D.Pp) return;
  const float* o = origin + (size_t)Pr.origin_row((int)(k / D.R0)) * 3;
  const float p[3] = {points[k * 3], points[k * 3 + 1], points[k * 3 + 2]};
  const float d = dist[k];
  bool keep = d > 0.f;
  if (D.within)   // get_inside_mask on the voxel-unit ray end points against the metre range, as the reference does
    keep = keep && D.pc[0] <= p[0] && p[0] <= D.pc[3] && D.pc[1] <= p[1] && p[1] <= D.pc[4] && D.pc[2] <= p[2] &&
           p[2] <= D.pc[5];
  float u[3];
  ray_unit(p, o, u);
#pragma unroll
  for (int a = 0; a < 3; ++a) qbuf[k * 3 + a] = __fmul_rn(__fsub_rn(__fadd_rn(o[a], __fmul_rn(u[a], d)), o[a]), 0.1f);
  q_mask[k] = keep;
}

// One block: chunk counts -> slot offsets soff[0..Sg*Fg] of the compacted gt rows, then the segment offsets of
// both searches.  c_off[0..P] = gt pair offsets; c_off[P] = G.
__global__ void dense_offsets_kernel(DenseDims D, PairTable Pr, int* __restrict__ counts, int64_t* __restrict__ soff,
                                     int64_t* __restrict__ q_off, int64_t* __restrict__ c_off) {
  const int S = D.Sg * D.Fg;
  sort_offsets(S, D.nchunk, counts, soff);
  const int64_t G = soff[S];
  for (int n = threadIdx.x; n <= D.P; n += blockDim.x) {
    const int64_t g0 = n < D.P ? soff[Pr.slot(n)] : G;
    q_off[n] = (int64_t)n * D.R0;
    q_off[D.P + n] = D.Pp + g0;
    c_off[n] = g0;
    if (n > 0) c_off[D.P + n] = G + (int64_t)n * D.R0;
  }
}

// grid as the count kernel.  gt chunks: stable scatter of the kept rows, scaled, into both buffers; rows of
// qbuf past Pp + G are masked.  Pred blocks: the pred points into cbuf behind the gt rows.
__global__ void __launch_bounds__(kChunk)
dense_scatter_kernel(DenseDims D, PairTable Pr, const float* __restrict__ origin, const float* __restrict__ gt,
                     const float* __restrict__ tindex, const int* __restrict__ counts,
                     const int64_t* __restrict__ soff, float* __restrict__ qbuf, float* __restrict__ cbuf,
                     unsigned char* __restrict__ q_mask, unsigned char* __restrict__ c_mask) {
  extern __shared__ int hist[];       // [32][Fg]
  const int64_t G = soff[D.Sg * D.Fg];
  const int ng = D.Sg * D.nchunk;
  if ((int)blockIdx.x < ng) {
    const int s = blockIdx.x / D.nchunk, c = blockIdx.x % D.nchunk, i = c * kChunk + threadIdx.x;
    const int f = i < D.M ? gt_frame(D, Pr, gt, tindex, s, i) : -1;
    const int pos = sort_rank(f, D.Fg, hist);
    if (i < D.M) {
      const int64_t row = (int64_t)s * D.M + i;
      if (row >= G) q_mask[D.Pp + row] = 0;
    }
    if (f < 0) return;
    const int slot = s * D.Fg + f;
    const int64_t dst = soff[slot] + counts[(size_t)slot * D.nchunk + c] + pos;
    const size_t k = (size_t)s * D.M + i;
    const float* o = origin + (size_t)Pr.origin_row(Pr.slot_pair(slot)) * 3;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float v = __fmul_rn(__fsub_rn(gt[k * 3 + a], o[a]), 0.1f);
      cbuf[dst * 3 + a] = v;
      qbuf[(D.Pp + dst) * 3 + a] = v;
    }
    c_mask[dst] = 1;
    q_mask[D.Pp + dst] = 1;
    return;
  }
  const long long k = (long long)(blockIdx.x - ng) * kChunk + threadIdx.x;
  if (k >= D.Pp) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) cbuf[(G + k) * 3 + a] = qbuf[k * 3 + a];
  c_mask[G + k] = q_mask[k];
}

// Per (block, segment): [sum of squared NN distances, count] of the kept queries.  A kept query without a nearest
// neighbour (no candidate, or a NaN point that is nearer to nothing) adds NaN, as the per-pair mean does.
__global__ void __launch_bounds__(kSumThreads)
dense_partials_kernel(const int64_t* __restrict__ q_off, const unsigned char* __restrict__ q_mask,
                      const float* __restrict__ dists, const int64_t* __restrict__ idx, double* __restrict__ partials) {
  __shared__ double red[kSumThreads / 32];
  const int s = blockIdx.y;
  const int64_t q0 = q_off[s];
  const long long Lq = q_off[s + 1] - q0;
  if ((long long)blockIdx.x * kSumThreads >= Lq) return;
  const long long i = (long long)blockIdx.x * kSumThreads + threadIdx.x;
  const bool live = i < Lq && q_mask[q0 + i];
  const double d = live ? (idx[q0 + i] < 0 ? (double)NAN : (double)dists[q0 + i]) : 0.0;
  const double a = block_sum<kSumThreads>(d, red);
  const double n = block_sum<kSumThreads>(live ? 1.0 : 0.0, red);
  if (threadIdx.x == 0) {
    double* dst = partials + ((size_t)s * gridDim.x + blockIdx.x) * 2;
    dst[0] = a;
    dst[1] = n;
  }
}

// One block: pairs [P, 4] = (sum pred->gt, pred count, sum gt->pred, gt count), then each group's loss, pairs in
// order.
__global__ void dense_finish_kernel(DenseDims D, PairTable Pr, const int64_t* __restrict__ q_off,
                                    const double* __restrict__ partials, double* __restrict__ pairs,
                                    float* __restrict__ loss, int nbx) {
  const int S = D.P;
  for (int n = threadIdx.x; n < S; n += blockDim.x) {
    for (int r = 0; r < 2; ++r) {
      const int s = r * S + n;
      const long long Lq = q_off[s + 1] - q_off[s];
      const int nb = (int)((Lq + kSumThreads - 1) / kSumThreads);
      double a = 0.0, c = 0.0;
      for (int bx = 0; bx < nb; ++bx) {
        a += partials[((size_t)s * nbx + bx) * 2];
        c += partials[((size_t)s * nbx + bx) * 2 + 1];
      }
      pairs[n * 4 + 2 * r] = a;
      pairs[n * 4 + 2 * r + 1] = c;
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < D.groups; g += blockDim.x) {
    double acc = 0.0;
    for (int n = 0; n < S; ++n) {
      const double* p = pairs + n * 4;
      if (Pr.group(n) == g && p[3] > 0) acc += (double)Pr.weight(n) * ((p[0] / p[1] + p[2] / p[3]) / 2.0);
    }
    loss[g] = (float)(acc / (double)Pr.norm_of(g));
  }
}

// One thread per query row of either direction.  d loss / d pred point of a pair with gt, chained through
// pred = ((o + u * d) - o) * 0.1:  d/dd = 0.1 * u . d/dpred.
//   pred query i (ray k):  c_n * 2 (p_i - g_nn)      c_n = grad_loss[group] * w_n / (2 norm) / (pred count)
//   gt query j:            -c_n * 2 (g_j - p_nn)     c_n = grad_loss[group] * w_n / (2 norm) / (gt count), onto p_nn's ray
__global__ void __launch_bounds__(kSumThreads)
dense_backward_kernel(DenseDims D, PairTable Pr, const float* __restrict__ points, const float* __restrict__ origin,
                      const float* __restrict__ qbuf, const float* __restrict__ cbuf,
                      const unsigned char* __restrict__ q_mask, const int64_t* __restrict__ q_off,
                      const int64_t* __restrict__ c_off, const int64_t* __restrict__ idx,
                      const double* __restrict__ pairs, const float* __restrict__ grad_loss,
                      float* __restrict__ grad_dist) {
  const int S = D.P;
  const long long t = (long long)blockIdx.x * kSumThreads + threadIdx.x;
  if (t >= D.Pp + c_off[S] || !q_mask[t]) return;
  const int64_t j = idx[t];
  if (j < 0) return;
  const bool pred_query = t < D.Pp;
  const int n = pred_query ? (int)(t / D.R0) : find_segment(q_off + S, S, t);
  const double* pr = pairs + n * 4;
  if (!(pr[3] > 0)) return;
  const float coef = (float)((double)grad_loss[Pr.group(n)] * Pr.weight(n) / (2.0 * Pr.norm_of(Pr.group(n))) /
                             (pred_query ? pr[1] : pr[3]));
  const int64_t cand = c_off[pred_query ? n : S + n] + j;
  const long long ray = pred_query ? t : (long long)n * D.R0 + j;
  const float* o = origin + (size_t)Pr.origin_row(n) * 3;
  const float p[3] = {points[ray * 3], points[ray * 3 + 1], points[ray * 3 + 2]};
  float u[3];
  ray_unit(p, o, u);
  float g = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float diff = 2.0f * coef * (qbuf[t * 3 + a] - cbuf[cand * 3 + a]);
    g += u[a] * (0.1f * (pred_query ? diff : -diff));
  }
  red_add_f32(grad_dist + ray, g);
}

int dense_dims(DenseDims& D, int P, int groups, int Sg, int Fg, int R0, int M, const char* who) {
  VIDAR_REQUIRE(P > 0 && groups > 0 && Sg > 0 && Fg > 0 && Fg <= kMaxFrames && R0 > 0 && M >= 0,
                "%s: bad sizes pairs=%d groups=%d samples=%d frames=%d R0=%d M=%d (frames <= %d)", who, P, groups,
                Sg, Fg, R0, M, kMaxFrames);
  VIDAR_REQUIRE(2LL * P <= 65535, "%s: %d pairs, at most 32767", who, P);
  VIDAR_REQUIRE((long long)Sg * Fg <= (1LL << 20), "%s: %lld (sample, frame) slots, at most 2^20", who,
                (long long)Sg * Fg);
  const long long Pp = (long long)P * R0, Pq = Pp + (long long)Sg * M;
  VIDAR_REQUIRE(Pq < (1LL << 31), "%s: %lld rows, at most 2^31 - 1", who, Pq);
  D = DenseDims{};
  D.P = P; D.groups = groups; D.Sg = Sg; D.Fg = Fg; D.R0 = R0; D.M = M;
  D.nchunk = (M + kChunk - 1) / kChunk;
  D.Pp = Pp; D.Pq = Pq;
  return VIDAR_OK;
}

int dense_forward(const DenseDims& D, const PairTable& Pr, const float* dist, const float* points, const float* origin,
                  const float* gt, const float* gt_tindex, float* qbuf, float* cbuf, unsigned char* q_mask,
                  unsigned char* c_mask, int64_t* q_off, int64_t* c_off, int64_t* idx, double* pairs, float* loss,
                  void* stream, const char* who) {
  cudaStream_t st = (cudaStream_t)stream;
  const int P = D.P, S = D.Sg * D.Fg, max_len = D.R0 > D.M ? D.R0 : D.M;
  const int nbx = (max_len + kSumThreads - 1) / kSumThreads;
  // stream-ordered scratch: chunk counts, slot offsets, the search's keys and distances, the partial sums
  const size_t n_counts = (size_t)S * D.nchunk, n_part = (size_t)2 * P * nbx * 2;
  const size_t o_soff = (sizeof(int) * n_counts + 255) & ~(size_t)255;
  const size_t o_keys = o_soff + ((sizeof(int64_t) * (S + 1) + 255) & ~(size_t)255);
  const size_t o_dists = o_keys + ((sizeof(unsigned long long) * D.Pq + 255) & ~(size_t)255);
  const size_t o_part = o_dists + ((sizeof(float) * D.Pq + 255) & ~(size_t)255);
  const size_t bytes = o_part + sizeof(double) * n_part;
  cudaMemPool_t pool;
  cudaError_t e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, bytes, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  int* counts = reinterpret_cast<int*>(s);
  int64_t* soff = reinterpret_cast<int64_t*>(s + o_soff);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(s + o_keys);
  float* dists = reinterpret_cast<float*>(s + o_dists);
  double* partials = reinterpret_cast<double*>(s + o_part);

  const unsigned grid = (unsigned)((long long)D.Sg * D.nchunk + (D.Pp + kChunk - 1) / kChunk);
  const size_t smem = sizeof(int) * 32 * D.Fg;
  dense_count_kernel<<<grid, kChunk, smem, st>>>(D, Pr, dist, points, origin, gt, gt_tindex, counts, qbuf, q_mask);
  int rc = check_launch("dense_chamfer(count)");
  if (!rc) {
    dense_offsets_kernel<<<1, 256, 0, st>>>(D, Pr, counts, soff, q_off, c_off);
    rc = check_launch("dense_chamfer(offsets)");
  }
  if (!rc) {
    dense_scatter_kernel<<<grid, kChunk, smem, st>>>(D, Pr, origin, gt, gt_tindex, counts, soff, qbuf, cbuf, q_mask,
                                                     c_mask);
    rc = check_launch("dense_chamfer(scatter)");
  }
  if (!rc)
    rc = vidar_nn_segments_forward(qbuf, cbuf, q_off, c_off, q_mask, c_mask, dists, idx, keys, 2 * P, D.Pq, max_len,
                                   max_len, stream);
  if (!rc) {
    dense_partials_kernel<<<dim3(nbx, 2 * P), kSumThreads, 0, st>>>(q_off, q_mask, dists, idx, partials);
    rc = check_launch("dense_chamfer(partials)");
  }
  if (!rc) {
    dense_finish_kernel<<<1, 256, 0, st>>>(D, Pr, q_off, partials, pairs, loss, nbx);
    rc = check_launch("dense_chamfer(finish)");
  }
  e = cudaFreeAsync(s, st);
  if (rc) return rc;
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(e));
  return VIDAR_OK;
}

int dense_backward(const DenseDims& D, const PairTable& Pr, const float* points, const float* origin, const float* qbuf,
                   const float* cbuf, const unsigned char* q_mask, const int64_t* q_off, const int64_t* c_off,
                   const int64_t* idx, const double* pairs, const float* grad_loss, float* grad_dist, void* stream,
                   const char* who) {
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(grad_dist, 0, sizeof(float) * (size_t)D.Pp, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: memset: %s", who, cudaGetErrorString(e));
  dense_backward_kernel<<<(unsigned)((D.Pq + kSumThreads - 1) / kSumThreads), kSumThreads, 0, st>>>(
      D, Pr, points, origin, qbuf, cbuf, q_mask, q_off, c_off, idx, pairs, grad_loss, grad_dist);
  return check_launch(who);
}

// ------------------------------------------------------------------ GT alignment (ViDARHeadV1)
// Segment s = i * bs + b (head frame i, sample b), key v = the slot whose source frame is the row's frame.
struct AlignDims {
  int bs, M, Cg, H, V, nchunk, with_points;
  float off[3], scale[3], cells[3];   // voxel = ((x - off) * scale) * cells, per axis
  int src[kMaxJobs];                  // [H, V] source frame of each (head frame, slot), -1 = none
};

__device__ __forceinline__ int align_key(const AlignDims& A, const float* __restrict__ gt, int s, int r) {
  if (r >= A.M) return -1;
  const float f = gt[((size_t)(s % A.bs) * A.M + r) * A.Cg + A.Cg - 1];
  const int* src = A.src + (s / A.bs) * A.V;
  for (int v = 0; v < A.V; ++v)
    if (src[v] >= 0 && f == (float)src[v]) return v;
  return -1;
}

__global__ void __launch_bounds__(kChunk)
align_count_kernel(AlignDims A, const float* __restrict__ gt, int* __restrict__ counts) {
  extern __shared__ int hist[];       // [32][V]
  const int s = blockIdx.y, c = blockIdx.x;
  sort_count(align_key(A, gt, s, c * kChunk + threadIdx.x), A.V, s, c, A.nchunk, hist, counts);
}

__global__ void align_offsets_kernel(AlignDims A, int* __restrict__ counts, int64_t* __restrict__ off) {
  sort_offsets(A.H * A.bs * A.V, A.nchunk, counts, off);
}

// Rows of a segment: its slots in order, the rows of a slot in their original order, then padding (NaN, tindex -1).
// x' = [x y z 1] @ T, summed left to right.
__global__ void __launch_bounds__(kChunk)
align_scatter_kernel(AlignDims A, const float* __restrict__ gt, const float* __restrict__ mats,
                     const int* __restrict__ counts, const int64_t* __restrict__ off, float* __restrict__ rays,
                     float* __restrict__ tindex, float* __restrict__ points) {
  extern __shared__ int hist[];
  const int s = blockIdx.y, c = blockIdx.x, r = c * kChunk + threadIdx.x;
  const int v = align_key(A, gt, s, r);
  const int pos = sort_rank(v, A.V, hist);
  const int64_t base = off[(size_t)s * A.V];
  const int64_t kept = off[(size_t)(s + 1) * A.V] - base;
  if (r < A.M && r >= kept) {
    const size_t d = (size_t)s * A.M + r;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      rays[d * 3 + a] = NAN;
      if (A.with_points) points[d * 3 + a] = NAN;
    }
    tindex[d] = -1.f;
  }
  if (v < 0) return;
  const int i = s / A.bs, b = s % A.bs, slot = s * A.V + v;
  const size_t d = (size_t)s * A.M + (off[slot] - base) + counts[(size_t)slot * A.nchunk + c] + pos;
  const float* T = mats + ((size_t)(i * A.V + v) * A.bs + b) * 16;
  const float* p = gt + ((size_t)b * A.M + r) * A.Cg;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[0], T[a]), __fmul_rn(p[1], T[4 + a])),
                                        __fmul_rn(p[2], T[8 + a])), T[12 + a]);
    rays[d * 3 + a] = __fmul_rn(__fmul_rn(__fsub_rn(x, A.off[a]), A.scale[a]), A.cells[a]);
    if (A.with_points) points[d * 3 + a] = x;
  }
  tindex[d] = (float)v;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_dense_chamfer_groups_forward(const float* dist, const float* points, const float* origin,
                                                  const float* gt, const float* gt_tindex, const int32_t* slot_pair,
                                                  const int32_t* pair_table, const float* pair_weight,
                                                  const float* group_norm, const float* pc_range_host, float* qbuf,
                                                  float* cbuf, unsigned char* q_mask, unsigned char* c_mask,
                                                  int64_t* q_off, int64_t* c_off, int64_t* idx, double* pairs,
                                                  float* loss, int P, int groups, int R0, int Sg, int Fg, int M,
                                                  int W, int H, int Z, int within_grid, void* stream) {
  const char* who = "dense_chamfer_groups_forward";
  DenseDims D;
  int rc = dense_dims(D, P, groups, Sg, Fg, R0, M, who);
  if (rc) return rc;
  VIDAR_REQUIRE(W > 0 && H > 0 && Z > 0, "%s: bad grid %dx%dx%d", who, W, H, Z);
  VIDAR_REQUIRE(pc_range_host, "%s: null pc_range", who);
  D.W = W; D.H = H; D.Z = Z; D.within = within_grid ? 1 : 0;
  for (int k = 0; k < 6; ++k) D.pc[k] = pc_range_host[k];
  VIDAR_REQUIRE(dist && points && origin && slot_pair && pair_table && pair_weight && group_norm && qbuf && cbuf &&
                q_mask && c_mask && q_off && c_off && idx && pairs && loss, "%s: null pointer argument", who);
  VIDAR_REQUIRE(M == 0 || (gt && gt_tindex), "%s: null gt buffer", who);
  const PairTable Pr{slot_pair, pair_table, pair_weight, group_norm};
  return dense_forward(D, Pr, dist, points, origin, gt, gt_tindex, qbuf, cbuf, q_mask, c_mask, q_off, c_off, idx,
                       pairs, loss, stream, who);
}

extern "C" int vidar_dense_chamfer_groups_backward(const float* points, const float* origin, const float* qbuf,
                                                   const float* cbuf, const unsigned char* q_mask,
                                                   const int64_t* q_off, const int64_t* c_off, const int64_t* idx,
                                                   const double* pairs, const int32_t* pair_table,
                                                   const float* pair_weight, const float* group_norm,
                                                   const float* grad_loss, float* grad_dist, int P, int groups,
                                                   int R0, int Sg, int Fg, int M, void* stream) {
  const char* who = "dense_chamfer_groups_backward";
  DenseDims D;
  int rc = dense_dims(D, P, groups, Sg, Fg, R0, M, who);
  if (rc) return rc;
  VIDAR_REQUIRE(points && origin && qbuf && cbuf && q_mask && q_off && c_off && idx && pairs && pair_table &&
                pair_weight && group_norm && grad_loss && grad_dist, "%s: null pointer argument", who);
  const PairTable Pr{nullptr, pair_table, pair_weight, group_norm};
  return dense_backward(D, Pr, points, origin, qbuf, cbuf, q_mask, q_off, c_off, idx, pairs, grad_loss, grad_dist,
                        stream, who);
}

extern "C" int vidar_head_align_gt(const float* gt, const float* mats, const int32_t* jobs_host,
                                   const float* voxel_host, float* rays, float* tindex, float* points, int bs, int M,
                                   int Cg, int H, int V, void* stream) {
  const char* who = "head_align_gt";
  VIDAR_REQUIRE(bs > 0 && M >= 0 && Cg >= 4 && H > 0 && V > 0 && V <= kMaxFrames && H * V <= kMaxJobs,
                "%s: bad sizes bs=%d M=%d Cg=%d H=%d V=%d (Cg >= 4, V <= %d, H*V <= %d)", who, bs, M, Cg, H, V,
                kMaxFrames, kMaxJobs);
  VIDAR_REQUIRE((long long)H * bs <= 65535, "%s: %d (head frame, sample) segments, at most 65535", who, H * bs);
  VIDAR_REQUIRE((long long)H * bs * M * 3 < (1LL << 31), "%s: %lld output rows, too many", who,
                (long long)H * bs * M);
  VIDAR_REQUIRE(jobs_host && voxel_host, "%s: null host table", who);
  VIDAR_REQUIRE(rays && tindex && (M == 0 || (gt && mats)), "%s: null pointer argument", who);
  if (M == 0) return VIDAR_OK;
  AlignDims A{};
  A.bs = bs; A.M = M; A.Cg = Cg; A.H = H; A.V = V;
  A.nchunk = (M + kChunk - 1) / kChunk;
  A.with_points = points ? 1 : 0;
  for (int a = 0; a < 3; ++a) {
    A.off[a] = voxel_host[a];
    A.scale[a] = voxel_host[3 + a];
    A.cells[a] = voxel_host[6 + a];
  }
  for (int j = 0; j < H * V; ++j) A.src[j] = jobs_host[j];
  cudaStream_t st = (cudaStream_t)stream;
  const int S = H * bs * V;
  const size_t o_off = (sizeof(int) * (size_t)S * A.nchunk + 255) & ~(size_t)255;
  const size_t bytes = o_off + sizeof(int64_t) * (S + 1);
  cudaMemPool_t pool;
  cudaError_t e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: scratch memory pool: %s", who, cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, bytes, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaMallocFromPoolAsync: %s", who, cudaGetErrorString(e));
  int* counts = reinterpret_cast<int*>(s);
  int64_t* off = reinterpret_cast<int64_t*>(s + o_off);
  const dim3 grid(A.nchunk, H * bs);
  const size_t smem = sizeof(int) * 32 * V;
  align_count_kernel<<<grid, kChunk, smem, st>>>(A, gt, counts);
  int rc = check_launch("head_align_gt(count)");
  if (!rc) {
    align_offsets_kernel<<<1, 256, 0, st>>>(A, counts, off);
    rc = check_launch("head_align_gt(offsets)");
  }
  if (!rc) {
    align_scatter_kernel<<<grid, kChunk, smem, st>>>(A, gt, mats, counts, off, rays, tindex, points);
    rc = check_launch("head_align_gt(scatter)");
  }
  e = cudaFreeAsync(s, st);
  if (rc) return rc;
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "%s: cudaFreeAsync: %s", who, cudaGetErrorString(e));
  return VIDAR_OK;
}
