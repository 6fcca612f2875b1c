// The dense loss term of the ViDAR head ('loss.dense_voxel'), H100 (sm_90a): the Chamfer distance between the
// gumbel-decoded dense rays and the GT cloud of every (sample, frame) pair of a batch, forward and backward, in a
// fixed number of launches and without a host sync.
//
// Reference: dense_heads/vidar_head_base.py:594-659 (per-pair loop over boolean masks), get_rendered_pcds
// :344-389, mmdet3d chamfer_distance (criterion 'l2', reduction 'mean').  Per pair n = b * F + f:
//   pred = {((o + unit(p - o) * d) - o) * 0.1 : rays f*R0 .. (f+1)*R0-1 of sample b with d > 0
//           [and p inside pc_range when eval_within_grid]}
//   gt   = {(g - o) * 0.1 : gt_tindex == f, 0 < x < W-1, 0 < y < H-1, 0 < z < Z-1}     o = origin[b, f]
//   loss = sum_n w_f * (mean_pred min_gt |.|^2 + mean_gt min_pred |.|^2) / 2 / (sum(w) * bs), pairs without gt
//          skipped; gt but no pred gives NaN like the per-pair path.
// fp32 statements in the reference's order with explicit _rn intrinsics (no FMA contraction).
//
// Layout (S = bs * F pairs; Pp = S * R0 dense rays; G = gt points kept; Pq = Pp + bs * M buffer rows):
//   qbuf [pred (Pp) | gt (G) | unused]   segments 0..S-1: pred queries (masked, not compacted), S..2S-1: gt queries
//   cbuf [gt (G) | pred (Pp) | unused]   the candidates of the same segments
// so one call of the segmented NN search (knn.cu) serves both directions.  The gt rows of a sample arrive in any
// frame order; they are compacted per pair by a stable counting sort (chunk histograms, a scan, a scatter that
// ranks inside a chunk with warp matches), so the original order inside a pair decides NN ties, as in the
// per-pair path.
//
// Launches: forward 7 (histogram + pred points, offsets, scatter, NN search 2, partial sums, finish), backward 1,
// whatever bs and F.  Sums are fp64 in a fixed order (per-block tree, blocks of a segment in order, pairs in
// order), so two calls give the same bits; the backward scatters into grad_dist with red.global.add.f32 like the
// per-pair path's knn backward.
#include "common.cuh"

namespace vidar {
namespace {

constexpr int kChunk = 1024;          // gt rows per block of the counting sort, one per thread (32 warps)
constexpr int kSumThreads = 256;
constexpr int kMaxFrames = 64;

struct DenseDims {
  int bs, F, R0, To, M, W, H, Z, within, nchunk;
  long long Pp, Pq;
  float pc[6];
  float w[kMaxFrames];                // per-frame loss weight
  float norm;                         // sum(loss_weight) * bs
};

// frame of gt row i of sample b, or -1 when the row belongs to no pair (padding, other frames, outside the box)
__device__ __forceinline__ int gt_frame(const DenseDims& D, const float* __restrict__ gt,
                                        const float* __restrict__ tindex, int b, int i) {
  const size_t k = (size_t)b * D.M + i;
  const float t = tindex[k];
  const float x = gt[k * 3], y = gt[k * 3 + 1], z = gt[k * 3 + 2];
  const bool box = x < (float)(D.W - 1) && x > 0.f && y < (float)(D.H - 1) && y > 0.f && z < (float)(D.Z - 1) &&
                   z > 0.f;
  return (box && t >= 0.f && t < (float)D.F && t == floorf(t)) ? (int)t : -1;
}

// unit(p - o): r / sqrt((r_x^2 + r_y^2) + r_z^2)
__device__ __forceinline__ void ray_unit(const float* p, const float* o, float u[3]) {
  const float r[3] = {__fsub_rn(p[0], o[0]), __fsub_rn(p[1], o[1]), __fsub_rn(p[2], o[2])};
  const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], r[0]), __fmul_rn(r[1], r[1])), __fmul_rn(r[2], r[2])));
#pragma unroll
  for (int a = 0; a < 3; ++a) u[a] = __fdiv_rn(r[a], n);
}

// Per warp and frame, the number of lanes holding that frame, written by the lowest such lane into
// hist[warp * F + f]; returns the lane's rank among them.  hist must be zeroed before.
__device__ __forceinline__ int warp_frame_rank(int f, int F, int* hist) {
  const unsigned peers = __match_any_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31;
  if (f >= 0 && lane == __ffs(peers) - 1) hist[(threadIdx.x >> 5) * F + f] = __popc(peers);
  return __popc(peers & ((1u << lane) - 1u));
}

// grid (nchunk + pred blocks, bs).  gt chunks: per-(pair, chunk) counts of kept rows.  Pred blocks: the pred
// points of every ray into qbuf (rows b*F*R0 + r) and their query mask.
__global__ void __launch_bounds__(kChunk)
dense_count_kernel(DenseDims D, const float* __restrict__ dist, const float* __restrict__ points,
                   const float* __restrict__ origin, const float* __restrict__ gt, const float* __restrict__ tindex,
                   int* __restrict__ counts, float* __restrict__ qbuf, unsigned char* __restrict__ q_mask) {
  extern __shared__ int hist[];       // [32][F]
  const int b = blockIdx.y;
  if ((int)blockIdx.x < D.nchunk) {
    const int c = blockIdx.x, i = c * kChunk + threadIdx.x;
    for (int e = threadIdx.x; e < 32 * D.F; e += kChunk) hist[e] = 0;
    __syncthreads();
    const int f = i < D.M ? gt_frame(D, gt, tindex, b, i) : -1;
    warp_frame_rank(f, D.F, hist);
    __syncthreads();
    for (int g = threadIdx.x; g < D.F; g += kChunk) {
      int n = 0;
      for (int w = 0; w < 32; ++w) n += hist[w * D.F + g];
      counts[((size_t)b * D.F + g) * D.nchunk + c] = n;
    }
    return;
  }
  const long long r = (long long)(blockIdx.x - D.nchunk) * kChunk + threadIdx.x;
  if (r >= (long long)D.F * D.R0) return;
  const int f = (int)(r / D.R0);
  const size_t k = (size_t)b * D.F * D.R0 + r;
  const float* o = origin + ((size_t)b * D.To + f) * 3;
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

// One block: chunk counts -> exclusive chunk offsets inside each pair, pair offsets of the compacted gt rows, and
// the segment offsets of both searches.  c_off[0..S] = gt pair offsets; c_off[S] = G.
__global__ void dense_offsets_kernel(DenseDims D, int* __restrict__ counts, int64_t* __restrict__ q_off,
                                     int64_t* __restrict__ c_off) {
  const int S = D.bs * D.F;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    int acc = 0;
    for (int c = 0; c < D.nchunk; ++c) {
      const int v = counts[(size_t)s * D.nchunk + c];
      counts[(size_t)s * D.nchunk + c] = acc;
      acc += v;
    }
    c_off[s + 1] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    c_off[0] = 0;
    for (int s = 0; s < S; ++s) { acc += c_off[s + 1]; c_off[s + 1] = acc; }
  }
  __syncthreads();
  const int64_t G = c_off[S];
  for (int s = threadIdx.x; s <= S; s += blockDim.x) {
    q_off[s] = (int64_t)s * D.R0;
    q_off[S + s] = D.Pp + c_off[s];
    if (s > 0) c_off[S + s] = G + (int64_t)s * D.R0;
  }
}

// grid (nchunk + pred blocks, bs).  gt chunks: stable scatter of the kept rows, scaled, into both buffers; rows of
// qbuf past Pp + G are masked.  Pred blocks: the pred points into cbuf behind the gt rows.
__global__ void __launch_bounds__(kChunk)
dense_scatter_kernel(DenseDims D, const float* __restrict__ origin, const float* __restrict__ gt,
                     const float* __restrict__ tindex, const int* __restrict__ counts,
                     const int64_t* __restrict__ c_off, float* __restrict__ qbuf, float* __restrict__ cbuf,
                     unsigned char* __restrict__ q_mask, unsigned char* __restrict__ c_mask) {
  extern __shared__ int hist[];       // [32][F]
  const int b = blockIdx.y;
  const int S = D.bs * D.F;
  const int64_t G = c_off[S];
  if ((int)blockIdx.x < D.nchunk) {
    const int c = blockIdx.x, i = c * kChunk + threadIdx.x;
    for (int e = threadIdx.x; e < 32 * D.F; e += kChunk) hist[e] = 0;
    __syncthreads();
    const int f = i < D.M ? gt_frame(D, gt, tindex, b, i) : -1;
    const int rank = warp_frame_rank(f, D.F, hist);
    __syncthreads();
    if (i < D.M) {
      const int64_t slot = (int64_t)b * D.M + i;
      if (slot >= G) q_mask[D.Pp + slot] = 0;
    }
    if (f < 0) return;
    const int n = b * D.F + f;
    int pos = rank;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pos += hist[w * D.F + f];
    const int64_t dst = c_off[n] + counts[(size_t)n * D.nchunk + c] + pos;
    const size_t k = (size_t)b * D.M + i;
    const float* o = origin + ((size_t)b * D.To + f) * 3;
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
  const long long r = (long long)(blockIdx.x - D.nchunk) * kChunk + threadIdx.x;
  if (r >= (long long)D.F * D.R0) return;
  const size_t k = (size_t)b * D.F * D.R0 + r;
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

// One block: pairs [S, 4] = (sum pred->gt, pred count, sum gt->pred, gt count), then the loss, pairs in order.
__global__ void dense_finish_kernel(DenseDims D, const int64_t* __restrict__ q_off,
                                    const double* __restrict__ partials, double* __restrict__ pairs,
                                    float* __restrict__ loss, int nbx) {
  const int S = D.bs * D.F;
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
  if (threadIdx.x == 0) {
    double acc = 0.0;
    for (int n = 0; n < S; ++n) {
      const double* p = pairs + n * 4;
      if (p[3] > 0) acc += (double)D.w[n % D.F] * ((p[0] / p[1] + p[2] / p[3]) / 2.0);
    }
    loss[0] = (float)(acc / (double)D.norm);
  }
}

// One thread per query row of either direction.  d loss / d pred point of a pair with gt, chained through
// pred = ((o + u * d) - o) * 0.1:  d/dd = 0.1 * u . d/dpred.
//   pred query i (ray k):  c_f * 2 (p_i - g_nn)      c_f = grad_loss * w_f / (2 norm) / (pred count)
//   gt query j:            -c_b * 2 (g_j - p_nn)     c_b = grad_loss * w_f / (2 norm) / (gt count), onto p_nn's ray
__global__ void __launch_bounds__(kSumThreads)
dense_backward_kernel(DenseDims D, const float* __restrict__ points, const float* __restrict__ origin,
                      const float* __restrict__ qbuf, const float* __restrict__ cbuf,
                      const unsigned char* __restrict__ q_mask, const int64_t* __restrict__ q_off,
                      const int64_t* __restrict__ c_off, const int64_t* __restrict__ idx,
                      const double* __restrict__ pairs, const float* __restrict__ grad_loss,
                      float* __restrict__ grad_dist) {
  const int S = D.bs * D.F;
  const long long t = (long long)blockIdx.x * kSumThreads + threadIdx.x;
  if (t >= D.Pp + c_off[S] || !q_mask[t]) return;
  const int64_t j = idx[t];
  if (j < 0) return;
  const bool pred_query = t < D.Pp;
  const int n = pred_query ? (int)(t / D.R0) : find_segment(q_off + S, S, t);
  const double* pr = pairs + n * 4;
  if (!(pr[3] > 0)) return;
  const float coef = (float)((double)grad_loss[0] * D.w[n % D.F] / (2.0 * D.norm) / (pred_query ? pr[1] : pr[3]));
  const int64_t cand = c_off[pred_query ? n : S + n] + j;
  const long long ray = pred_query ? t : (long long)n * D.R0 + j;
  const float* o = origin + ((size_t)(n / D.F) * D.To + n % D.F) * 3;
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

int dense_dims(DenseDims& D, const float* weights_host, float weight_sum, int bs, int F, int R0, int To, int M,
               const char* who) {
  VIDAR_REQUIRE(bs > 0 && F > 0 && F <= kMaxFrames && R0 > 0 && To >= F && M >= 0,
                "%s: bad sizes bs=%d F=%d R0=%d To=%d M=%d (F <= %d)", who, bs, F, R0, To, M, kMaxFrames);
  VIDAR_REQUIRE(2LL * bs * F <= 65535, "%s: %d pairs, at most 32767", who, bs * F);
  const long long Pp = (long long)bs * F * R0, Pq = Pp + (long long)bs * M;
  VIDAR_REQUIRE(Pq < (1LL << 31), "%s: %lld rows, at most 2^31 - 1", who, Pq);
  VIDAR_REQUIRE(weights_host, "%s: null loss weights", who);
  D = DenseDims{};
  D.bs = bs; D.F = F; D.R0 = R0; D.To = To; D.M = M;
  D.nchunk = (M + kChunk - 1) / kChunk;
  D.Pp = Pp; D.Pq = Pq;
  for (int f = 0; f < F; ++f) D.w[f] = weights_host[f];
  D.norm = weight_sum * (float)bs;
  return VIDAR_OK;
}

}  // namespace
}  // namespace vidar

using namespace vidar;

extern "C" int vidar_dense_chamfer_forward(const float* dist, const float* points, const float* origin,
                                           const float* gt, const float* gt_tindex, const float* weights_host,
                                           const float* pc_range_host, float weight_sum, float* qbuf, float* cbuf,
                                           unsigned char* q_mask, unsigned char* c_mask, int64_t* q_off,
                                           int64_t* c_off, int64_t* idx, double* pairs, float* loss, int bs, int F,
                                           int R0, int To, int M, int W, int H, int Z, int within_grid,
                                           void* stream) {
  DenseDims D;
  int rc = dense_dims(D, weights_host, weight_sum, bs, F, R0, To, M, "dense_chamfer_forward");
  if (rc) return rc;
  VIDAR_REQUIRE(W > 0 && H > 0 && Z > 0, "dense_chamfer_forward: bad grid %dx%dx%d", W, H, Z);
  VIDAR_REQUIRE(pc_range_host, "dense_chamfer_forward: null pc_range");
  D.W = W; D.H = H; D.Z = Z; D.within = within_grid ? 1 : 0;
  for (int k = 0; k < 6; ++k) D.pc[k] = pc_range_host[k];
  VIDAR_REQUIRE(dist && points && origin && qbuf && cbuf && q_mask && c_mask && q_off && c_off && idx && pairs && loss,
                "dense_chamfer_forward: null pointer argument");
  VIDAR_REQUIRE(M == 0 || (gt && gt_tindex), "dense_chamfer_forward: null gt buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = bs * F, max_len = R0 > M ? R0 : M;
  const int nbx = (max_len + kSumThreads - 1) / kSumThreads;
  // stream-ordered scratch: chunk counts, the search's keys and distances, the partial sums
  const size_t n_counts = (size_t)S * D.nchunk, n_part = (size_t)2 * S * nbx * 2;
  const size_t o_keys = (sizeof(int) * n_counts + 255) & ~(size_t)255;
  const size_t o_dists = o_keys + ((sizeof(unsigned long long) * D.Pq + 255) & ~(size_t)255);
  const size_t o_part = o_dists + ((sizeof(float) * D.Pq + 255) & ~(size_t)255);
  const size_t bytes = o_part + sizeof(double) * n_part;
  cudaMemPool_t pool;
  cudaError_t e = scratch_pool(&pool);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "dense_chamfer_forward: scratch memory pool: %s", cudaGetErrorString(e));
  unsigned char* s = nullptr;
  e = cudaMallocFromPoolAsync((void**)&s, bytes, pool, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "dense_chamfer_forward: cudaMallocFromPoolAsync: %s", cudaGetErrorString(e));
  int* counts = reinterpret_cast<int*>(s);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(s + o_keys);
  float* dists = reinterpret_cast<float*>(s + o_dists);
  double* partials = reinterpret_cast<double*>(s + o_part);

  const dim3 grid(D.nchunk + (unsigned)(((long long)F * R0 + kChunk - 1) / kChunk), bs);
  const size_t smem = sizeof(int) * 32 * F;
  dense_count_kernel<<<grid, kChunk, smem, st>>>(D, dist, points, origin, gt, gt_tindex, counts, qbuf, q_mask);
  rc = check_launch("dense_chamfer(count)");
  if (!rc) {
    dense_offsets_kernel<<<1, 256, 0, st>>>(D, counts, q_off, c_off);
    rc = check_launch("dense_chamfer(offsets)");
  }
  if (!rc) {
    dense_scatter_kernel<<<grid, kChunk, smem, st>>>(D, origin, gt, gt_tindex, counts, c_off, qbuf, cbuf, q_mask, c_mask);
    rc = check_launch("dense_chamfer(scatter)");
  }
  if (!rc)
    rc = vidar_nn_segments_forward(qbuf, cbuf, q_off, c_off, q_mask, c_mask, dists, idx, keys, 2 * S, D.Pq, max_len,
                                   max_len, stream);
  if (!rc) {
    dense_partials_kernel<<<dim3(nbx, 2 * S), kSumThreads, 0, st>>>(q_off, q_mask, dists, idx, partials);
    rc = check_launch("dense_chamfer(partials)");
  }
  if (!rc) {
    dense_finish_kernel<<<1, 256, 0, st>>>(D, q_off, partials, pairs, loss, nbx);
    rc = check_launch("dense_chamfer(finish)");
  }
  e = cudaFreeAsync(s, st);
  if (rc) return rc;
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "dense_chamfer_forward: cudaFreeAsync: %s", cudaGetErrorString(e));
  return VIDAR_OK;
}

extern "C" int vidar_dense_chamfer_backward(const float* points, const float* origin, const float* qbuf,
                                            const float* cbuf, const unsigned char* q_mask, const int64_t* q_off,
                                            const int64_t* c_off, const int64_t* idx, const double* pairs,
                                            const float* weights_host, float weight_sum, const float* grad_loss,
                                            float* grad_dist, int bs, int F, int R0, int To, int M, void* stream) {
  DenseDims D;
  int rc = dense_dims(D, weights_host, weight_sum, bs, F, R0, To, M, "dense_chamfer_backward");
  if (rc) return rc;
  VIDAR_REQUIRE(points && origin && qbuf && cbuf && q_mask && q_off && c_off && idx && pairs && grad_loss && grad_dist,
                "dense_chamfer_backward: null pointer argument");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(grad_dist, 0, sizeof(float) * (size_t)D.Pp, st);
  if (e != cudaSuccess) return set_error(VIDAR_E_CUDA, "dense_chamfer_backward: memset: %s", cudaGetErrorString(e));
  dense_backward_kernel<<<(unsigned)((D.Pq + kSumThreads - 1) / kSumThreads), kSumThreads, 0, st>>>(
      D, points, origin, qbuf, cbuf, q_mask, q_off, c_off, idx, pairs, grad_loss, grad_dist);
  return check_launch("dense_chamfer_backward");
}
