/*
 * vidar_b200.h -- C ABI of libvidar_b200.so: the H100 (sm_90a) kernels that sit
 * under ViDAR's two hot-path operator boundaries.
 *
 *   (i)  multi-scale deformable attention   (mmcv `_ext.ms_deform_attn_{forward,backward}`,
 *        bound at projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:10-12,
 *        called at :42-48, :74-84, :118-124, :150-160)
 *   (ii) the voxel ray-caster family        (third_lib/dvr/dvr.cpp:65-69, third_lib/dvxlr/dvxlr.cpp:61-65,
 *        third_lib/dvxlr/dvxlr_v2.cpp:67-70) and the in-model renderers built on the same
 *        volume (latent_rendering.py:79-162, vidar_head_base.py:420-509,586-592,662-752).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to a dense, contiguous, 16-byte aligned buffer
 *     unless the parameter name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     no entry point synchronises the device or allocates memory;
 *   - return value 0 = success, non-zero = VIDAR_E_* ; vidar_last_error() gives the
 *     message of the last failure on the calling thread (the Python layer turns it
 *     into RuntimeError/ValueError, the reference raises through TORCH_CHECK);
 *   - all floating-point I/O is fp32 (the reference casts to fp32 with
 *     custom_fwd(cast_inputs=torch.float32), multi_scale_deformable_attn_function.py:93;
 *     the ray-casters are dispatched on float tensors, dvr.cu:367).
 *
 * No torch types appear here: the library links only against libcudart.
 */
#ifndef VIDAR_B200_H_
#define VIDAR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  VIDAR_OK = 0,
  VIDAR_E_INVALID = 1,   /* bad argument (shape, null pointer, unknown enum) */
  VIDAR_E_CUDA = 2,      /* a CUDA runtime call or launch failed */
  VIDAR_E_UNSUPPORTED = 3
};

/* Message of the last error raised on this thread ("" if none). */
const char* vidar_last_error(void);
/* Library / build identification, e.g. "vidar_b200 0.1 sm_90a". */
const char* vidar_version(void);
/* Number of kernels this library has launched since load (all threads).  bench.py
 * reports the delta across the timed region as `gpu_launches`. */
int64_t vidar_launch_count(void);

/* ------------------------------------------------------------------------------------
 * (i) Multi-scale deformable attention
 * ---------------------------------------------------------------------------------- */

/* Replaces ext_module.ms_deform_attn_forward
 *   (multi_scale_deformable_attn_function.py:118-124).
 *   value            [B, K, H, C]        K = sum_l Hl*Wl
 *   spatial_shapes   [L, 2] int64 (h, w) (device)
 *   level_start      [L]    int64        (device)
 *   sampling_loc     [B, Q, H, L, P, 2]  (x, y) normalised to [0,1]
 *   attn_weight      [B, Q, H, L, P]
 *   out              [B, Q, H*C]         fully overwritten
 * im2col_step is validated like mmcv (B % min(B, im2col_step) == 0) and otherwise unused. */
int vidar_msda_forward(const float* value, const int64_t* spatial_shapes,
                       const int64_t* level_start, const float* sampling_loc,
                       const float* attn_weight, float* out,
                       int B, int K, int H, int C, int L, int Q, int P,
                       int im2col_step, void* stream);

/* Replaces ext_module.ms_deform_attn_backward
 *   (multi_scale_deformable_attn_function.py:150-160).
 *   grad_out          [B, Q, H*C]
 *   grad_value        [B, K, H, C]        accumulated with atomics: caller zeroes it
 *                                         (torch.zeros_like, :146)
 *   grad_sampling_loc [B, Q, H, L, P, 2]  fully overwritten
 *   grad_attn_weight  [B, Q, H, L, P]     fully overwritten                              */
int vidar_msda_backward(const float* value, const int64_t* spatial_shapes,
                        const int64_t* level_start, const float* sampling_loc,
                        const float* attn_weight, const float* grad_out,
                        float* grad_value, float* grad_sampling_loc,
                        float* grad_attn_weight,
                        int B, int K, int H, int C, int L, int Q, int P,
                        int im2col_step, void* stream);

/* MSDeformableAttention3D's sampling with its elementwise prologue folded in
 *   (spatial_cross_attention.py:339-371 + the two calls above):
 *     attn = softmax_{L*P}(logits)                       (:339-342)
 *     loc  = offsets / (W_l, H_l) + ref_points[b, q, p % D]   (:356-371, point p = j*D + z)
 *   ref_points  [B, Q, D, 2]        projected Z-anchors (reference_points_cam), normalised
 *   offsets     [B, Q, H, L, P, 2]  raw output of the sampling_offsets Linear (pixels of level l)
 *   logits      [B, Q, H, L*P]      raw output of the attention_weights Linear
 * Requires L*P == 32 and head dim 16/32/64 (the shipped SCA configuration: 4 levels x 8 points).
 * Backward: grad_value accumulated (caller zeroes), grad_offsets / grad_logits overwritten; the
 * reference points carry no gradient (they come from the camera geometry). */
int vidar_msda_sca_forward(const float* value, const int64_t* spatial_shapes,
                           const int64_t* level_start, const float* ref_points,
                           const float* offsets, const float* logits, float* out,
                           int B, int K, int H, int C, int L, int Q, int P, int D, void* stream);
int vidar_msda_sca_backward(const float* value, const int64_t* spatial_shapes,
                            const int64_t* level_start, const float* ref_points,
                            const float* offsets, const float* logits, const float* grad_out,
                            float* grad_value, float* grad_offsets, float* grad_logits,
                            int B, int K, int H, int C, int L, int Q, int P, int D, void* stream);

/* TemporalSelfAttention (temporal_self_attention.py:196-261) and the future decoder's deformable attention
 *   (vidar_decoder.py:466-506) with their elementwise prologue and TSA's queue mean folded in.  G queue entries
 *   per sample (TSA: num_bev_queue = 2; the decoder: 1):
 *     attn = softmax_{L*P}(logits[b, q, h, g])
 *     loc  = offsets[b, q, h, g, l, p] / (W_l, H_l) + ref_points[b*G + g, q, l]   (a true division, then an add)
 *     out[b, q, h] = 1/G * sum_g  msda(value[b*G + g], loc, attn)[q, h]
 *   value       [B*G, K, H, C]       queue entry g of sample b is value batch b*G + g
 *   ref_points  [B*G, Q, L, 2]       normalised 2-D reference points, per level
 *   offsets     [B, Q, H, G, L, P, 2]  raw output of the sampling_offsets Linear (pixels of level l)
 *   logits      [B, Q, H, G, L*P]    raw output of the attention_weights Linear
 *   out         [B, Q, H*C]          fully overwritten; the [B*G, Q, H*C] per-entry output never exists
 * Requires L*P in {1, 2, 4, 8, 16, 32}, G*L*P <= 32 and head dim 16/32/64.
 * Backward: grad_value [B*G, K, H, C] accumulated (caller zeroes), grad_offsets / grad_logits overwritten; the
 * reference points carry no gradient. */
int vidar_msda_tsa_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                           const float* ref_points, const float* offsets, const float* logits, float* out,
                           int B, int G, int K, int H, int C, int L, int Q, int P, void* stream);
int vidar_msda_tsa_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                            const float* ref_points, const float* offsets, const float* logits,
                            const float* grad_out, float* grad_value, float* grad_offsets, float* grad_logits,
                            int B, int G, int K, int H, int C, int L, int Q, int P, void* stream);

/* Row-indirect variants: SpatialCrossAttention's rebatch / scatter-add (spatial_cross_attention.py:135-172)
 * folded into the op (SURVEY.md 8f-1).  A row is entry j of camera c's visible-pillar list:
 *   idx        [cams, Qd] int32   pillar of row j (ascending; entries >= count[c] unused), NULL: row j = pillar j
 *   count      [cams]     int32   live rows per camera, on the DEVICE (no host sync), NULL: all Qrows rows live
 *   inv_count  [bs, Qd]           1 / clamp(#cameras seeing the pillar, 1)  (:168-171), NULL: 1
 *   value      [bs*ncl, K, H, C]  the launch's cameras cam0 .. cam0+ncl-1, batch-major (n = b*ncl + camera)
 *   slots      [bs, Qd, H*C]      caller-zeroed; every live row adds inv_count * (its head vectors) to the slot
 *                                 of its pillar with red.global.add.v4.f32 (the reference's `slots[j, idx] += ...`
 *                                 followed by `slots / count`)
 * The launch covers rows j with (j / 64) % S in [s_lo, s_hi): interleaved sub-slices of a camera's list, the
 * unit of work when cameras are sharded over ranks (SURVEY.md 8e); S = 1, [0, 1) = every row.
 * `rows`: sampling locations / weights given per row, [bs*ncl, Qrows, H, L, P(, 2)] -- the plain op's inputs.
 * `sca_rows`: the fused MSDeformableAttention3D prologue of vidar_msda_sca_*, with
 *   ref_cam [cams, bs, Qd, D, 2] (reference_points_cam as point_sampling lays it out) and offsets / logits
 *   DENSE per pillar, [bs, Qd, H, L, P, 2] / [bs, Qd, H, L*P]: they are Linear(query) rows, equal for every
 *   camera that sees the pillar, so they are computed once per pillar and read through idx.
 * Backward: grad_slots [bs, Qd, H*C] is read through the same map; grad_value accumulated (caller zeroes);
 *   rows:     grad_sampling_loc / grad_attn_weight written for the rows of this launch (caller zeroes the rest);
 *   sca_rows: grad_offsets / grad_logits ACCUMULATED over cameras with red.global.add (caller zeroes).
 *   At C = 32 with 4 levels x 8 points both backwards first put the rows in image order, with stream-ordered
 *   scratch (8 B per row) from a memory pool of the library; `rows` then needs sampling_loc 16-byte aligned. */
int vidar_sca_compact(const unsigned char* bev_mask, int32_t* idx, int32_t* count, float* inv_count,
                      int cams, int bs, int Q, int D, void* stream);
int vidar_msda_rows_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                            const float* sampling_loc, const float* attn_weight, const int32_t* idx,
                            const int32_t* count, const float* inv_count, float* slots, int bs, int ncl,
                            int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P, int S, int s_lo,
                            int s_hi, void* stream);
int vidar_msda_rows_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                             const float* sampling_loc, const float* attn_weight, const int32_t* idx,
                             const int32_t* count, const float* inv_count, const float* grad_slots,
                             float* grad_value, float* grad_sampling_loc, float* grad_attn_weight, int bs,
                             int ncl, int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P, int S,
                             int s_lo, int s_hi, void* stream);
int vidar_msda_sca_rows_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                const float* ref_cam, const float* offsets, const float* logits,
                                const int32_t* idx, const int32_t* count, const float* inv_count, float* slots,
                                int bs, int ncl, int cam0, int K, int H, int C, int L, int Qrows, int Qd, int P,
                                int D, int S, int s_lo, int s_hi, void* stream);
int vidar_msda_sca_rows_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                 const float* ref_cam, const float* offsets, const float* logits,
                                 const int32_t* idx, const int32_t* count, const float* inv_count,
                                 const float* grad_slots, float* grad_value, float* grad_offsets,
                                 float* grad_logits, int bs, int ncl, int cam0, int K, int H, int C, int L,
                                 int Qrows, int Qd, int P, int D, int S, int s_lo, int s_hi, void* stream);

/* (i-c) The Linear layer in front of the sampling (SURVEY.md 8f-4): value_proj of MSDeformableAttention3D
 * (spatial_cross_attention.py:333) over the flattened camera features (modules/transformer.py:159-179),
 * y [M, N] = x [M, K] w[N, K]^T + bias[N], fp32 in / out.  wgmma tensor cores with a 3xTF32 split (fp32
 * accuracy, ~1e-6 relative: a plain TF32 GEMM would miss the 1e-4 parity bar), operands by TMA, accumulators in
 * registers.  K % 32 == 0, N % 128 == 0; bias may be NULL.  w_split: 2*N*K floats of caller-owned scratch. */
int vidar_linear_tf32x3(const float* x, const float* w, const float* bias, float* y, float* w_split,
                        int M, int N, int K, void* stream);

/* ------------------------------------------------------------------------------------
 * (ii-a) dvr / dvxlr / dvxlr_v2 voxel ray-casters
 *   sigma   [N, T, Z, Y, X]   (reference names the dims H, L, W)
 *   origin  [N, T, 3]         voxel units (x, y, z)
 *   points  [N, M, 3]         voxel units (x, y, z), NaN for padded rays
 *   tindex  [N, M]            FLOAT frame index, < 0 = padded ray (skipped)
 *   T  = sigma frames, To = origin frames (origin is indexed by t, sigma by
 *        ts = (T == 1) ? 0 : t, dvr.cu:97,109)
 * ---------------------------------------------------------------------------------- */

/* dvr.init / dvxlr.init (dvr.cu:14-63,705-738; dvxlr.cu:12-61,528-561).
 *   occupancy [N, T, Z, Y, X]  caller zeroes it; set to 1 at every ray end point. */
int vidar_dvr_init(const float* points, const float* tindex, float* occupancy,
                   int N, int M, int T, int Z, int Y, int X, void* stream);

/* dvr.render_forward (dvr.cu:65-317,327-383).  train_phase: 0 = "test", 1 = "train".
 *   pred_dist, gt_dist [N, M]  caller fills with -1 (dvr.cu:354-355); rays that never
 *   enter the grid keep it. */
int vidar_dvr_render_forward(const float* sigma, const float* origin, const float* points,
                             const float* tindex, float* pred_dist, float* gt_dist,
                             int N, int M, int T, int To, int Z, int Y, int X,
                             int train_phase, void* stream);

/* dvr.render (dvr.cu:385-627,639-694): forward + loss gradient in one call.
 *   loss_type: 0 = "l1" (also "bce", dvr.cu:667-668), 1 = "l2", 2 = "absrel".
 *   grad_sigma [N, T, Z, Y, X]  caller zeroes it; accumulated atomically (the
 *   reference's `+=` at dvr.cu:622 is a documented race; this is the race-free sum). */
int vidar_dvr_render(const float* sigma, const float* origin, const float* points,
                     const float* tindex, float* pred_dist, float* gt_dist,
                     float* grad_sigma, int N, int M, int T, int To, int Z, int Y, int X,
                     int loss_type, void* stream);

/* dvxlr.render (dvxlr.cu:160-517) and dvxlr_v2.render_v2 (dvxlr_v2.cu:119-493).
 *   max_d                  third dim of the list outputs (reference: 1026, dvxlr.cu:10)
 *   dd_dsigma [N, M, max_d]      caller zeroes            (dvxlr.cu:492)
 *   indices   [N, M, max_d, 3]   caller zeroes; (z, y, x) stored as float (dvxlr.cu:450-452)
 *   (dd_dsigma and indices may both be NULL: the lists are then not written -- used by
 *    the fused autograd path, which never needs them)
 *   v2 only (pass NULL for v1):
 *   sigma_regul [N, T, Z, Y, X]
 *   ray_pred  [N, M, max_d]      caller zeroes            (dvxlr_v2.cu:467)
 *   indicator [N, M, max_d]      caller fills with -1     (dvxlr_v2.cu:468)               */
int vidar_dvxlr_render(const float* sigma, const float* origin, const float* points,
                       const float* tindex, const float* sigma_regul,
                       float* pred_dist, float* gt_dist, float* dd_dsigma, float* indices,
                       float* ray_pred, float* indicator,
                       int N, int M, int T, int To, int Z, int Y, int X, int max_d,
                       void* stream);

/* Forward half of DifferentiableVoxelRendering without the lists: pred_dist / gt_dist
 * only (both caller-filled with -1), same traversal as dvxlr.render. */
int vidar_dvxlr_forward(const float* sigma, const float* origin, const float* points,
                        const float* tindex, float* pred_dist, float* gt_dist,
                        int N, int M, int T, int To, int Z, int Y, int X, void* stream);

/* dvxlr.get_grad_sigma (dvxlr.cu:63-156) and dvxlr_v2.get_grad_sigma_v2 (dvxlr_v2.cu:12-115).
 *   elementwise_mult [N, M, max_d]; indices [N, M, max_d, 3]
 *   grad_sigma [N, T, Z, Y, X] caller zeroes.
 *   v2 only (NULL for v1): indicator, grad_ray_pred [N, M, max_d]; grad_sigma_regul like
 *   grad_sigma, caller zeroes. */
int vidar_dvxlr_get_grad_sigma(const float* elementwise_mult, const float* indices,
                               const float* tindex, const float* indicator,
                               const float* grad_ray_pred, float* grad_sigma,
                               float* grad_sigma_regul,
                               int N, int M, int T, int Z, int Y, int X, int max_d,
                               void* stream);

/* Fused backward of DifferentiableVoxelRendering[V2] (e2e_predictor_utils.py:91-143):
 * re-walks every ray and scatters grad_pred[n,m] * d pred/d sigma straight into
 * grad_sigma -- the [N,M,1026(,3)] lists are never materialised.  Same result as
 * dvxlr.render + `gradpred[...,None]*dd_dsigma` (NaN -> 0, :104-108) + get_grad_sigma.
 *   grad_pred [N, M];  grad_sigma caller-zeroed.
 *   v2 only (NULL otherwise): grad_ray_pred [N, M, max_d] -> grad_sigma_regul. */
int vidar_dvxlr_backward_fused(const float* sigma, const float* origin, const float* points,
                               const float* tindex, const float* grad_pred,
                               const float* grad_ray_pred, float* grad_sigma,
                               float* grad_sigma_regul,
                               int N, int M, int T, int To, int Z, int Y, int X, int max_d,
                               void* stream);

/* ------------------------------------------------------------------------------------
 * (ii-b) ViDAR head: ray sampler, fused cross-entropy, arg-max decode
 *   (projects/mmdet3d_plugin/bevformer/dense_heads/vidar_head_base.py:420-509, 586-592, 706-738)
 *   sigma  [F, Z, Y, X]  the F frame volumes of one batch element
 *   origin [F, 3], points [R, 3] (voxel units), frame [R] int32 frame of each ray (NULL = 0)
 *   A ray whose frame is outside [0, F) (e.g. -1 for a padded row) is invalid: valid 0, ce / lse / dist / depth 0,
 *   logits -inf, no gradient; only its frame entry is read.
 *   Per ray: sample 0 = the GT point (with_gt), then num_way waypoints at
 *   o + u*(k+0.5)*step; K = num_way + with_gt samples; logit = trilinear grid_sample
 *   (align_corners=False, zeros) or -inf where any normalised coordinate leaves (-1,1).
 * ---------------------------------------------------------------------------------- */

/* Materialising sampler = the per-(batch,frame) body of _get_grid_features (:433-500).
 *   logits [R, K] (NULL = skip), length [R, K] |x-o| (NULL = skip),
 *   valid [R] 1/0: GT point strictly inside the volume (:464) (NULL = skip). */
int vidar_ray_sample(const float* sigma, const float* origin, const float* points,
                     const int32_t* frame, float* logits, float* length, float* valid,
                     int R, int F, int Z, int Y, int X, int num_way, float step, int with_gt,
                     void* stream);

/* Its backward: grad_sigma [F,Z,Y,X] (caller-zeroed) += trilinear scatter of grad_logits. */
int vidar_ray_sample_backward(const float* origin, const float* points, const int32_t* frame,
                              const float* grad_logits, float* grad_sigma,
                              int R, int F, int Z, int Y, int X, int num_way, float step,
                              int with_gt, void* stream);

/* Fused sampler + F.cross_entropy(label 0) (:586-588): ce[r] = logsumexp(logits) - logit_0.
 *   ce, lse, valid [R]; rays whose GT point is outside get ce = 0, valid = 0. */
int vidar_ray_ce_forward(const float* sigma, const float* origin, const float* points,
                         const int32_t* frame, float* ce, float* lse, float* valid,
                         int R, int F, int Z, int Y, int X, int num_way, float step,
                         void* stream);

/* Backward of the fused CE: grad_sigma (caller-zeroed) += sum_r grad_ce[r] * d ce[r]/d sigma.
 *   lse from the forward; grad_ce NULL = all ones. */
int vidar_ray_ce_backward(const float* sigma, const float* origin, const float* points,
                          const int32_t* frame, const float* lse, const float* grad_ce,
                          float* grad_sigma, int R, int F, int Z, int Y, int X, int num_way,
                          float step, void* stream);

/* Inference decode (:706-732): exact zeros -> -inf, first arg-max over the num_way
 * waypoints; depth [R] = its |x-o| (voxel units), index [R] (float, NULL = skip). */
int vidar_ray_argmax(const float* sigma, const float* origin, const float* points,
                     const int32_t* frame, float* depth, float* index,
                     int R, int F, int Z, int Y, int X, int num_way, float step, void* stream);

/* Fused gumbel decode of the dense loss term: ViDARHeadBase._custom_gumbel_softmax_distance
 * (vidar_head_base.py:754-773) applied to the sampler's logits without the GT slot (:631-636).
 *   noise [R, num_way]  Gumbel(0,1) noise, drawn by the host like F.gumbel_softmax draws it
 *   dist  [R]           length of the sampled waypoint (0 for rays whose end point is outside)
 *   lse, p_next [R]     saved for the backward (log-sum-exp of the logits, softmax mass beyond dist)
 * Backward: grad_sigma (caller-zeroed) += grad_dist[r] * dist[r] * softmax_k * ([len_k > dist[r]] - p_next[r]). */
int vidar_ray_gumbel_forward(const float* sigma, const float* origin, const float* points,
                             const int32_t* frame, const float* noise, float* dist, float* lse,
                             float* p_next, int R, int F, int Z, int Y, int X, int num_way,
                             float step, void* stream);
int vidar_ray_gumbel_backward(const float* sigma, const float* origin, const float* points,
                              const int32_t* frame, const float* dist, const float* lse,
                              const float* p_next, const float* grad_dist, float* grad_sigma,
                              int R, int F, int Z, int Y, int X, int num_way, float step,
                              void* stream);

/* ------------------------------------------------------------------------------------
 * (ii-c) LatentRendering core
 *   (projects/mmdet3d_plugin/bevformer/modules/ray_operations/latent_rendering.py:98-161:
 *   everything between the three Linear layers).  act: 0 = 'exp' (1-exp(-relu x)), 1 = 'sigmoid'.
 *   CHANNEL-LAST maps, as the Linear layers emit them:
 *   occ    [bs, Hb, Wb, D]     output of unsup_raymarching_head (:94), D = pred_height
 *   feat   [bs, Hb, Wb, D*G]   output of lora_a (:134); channel = d*G + j
 *   prob   [bs, Hb, Wb, D]     out: occ_path_prob (:127-128)
 *   pooled [bs, Hb*Wb, D*G]    out: ray-pooled feature that feeds lora_b (:148-153)
 *   grid_num waypoints of step grid_step / (min(Hb,Wb)//2) (:101-104); eps (:80,147).
 *   Supported: D a power of two <= 32, G in {1, 2, 4, 8, 16} (the reference default
 *   pred_height=1, reduction=16, embed_dims=256 is D=1, G=16).
 *   aux    [3, bs, Hb, Wb, D]  filled by the forward (product of the non-zero transmittance
 *          factors, count of zero factors, sum of sampled probabilities) and read by the backward,
 *          so that it does not march the rays again to recompute them.
 *
 * One phase per call, on a range [cell0, cell0+ncells) of the bs*Hb*Wb BEV cells (row-major):
 * when the cells are sharded over GPUs the host places a collective on the small maps between
 * the phases (vidar_b200/modules/latent_rendering.py).  Forward: prob_forward, then
 * pool_forward on the complete prob map.  Backward: pool_backward adds the gradient that
 * reaches the prob map through the ray pooling to grad_prob_map; prob_backward reads
 * grad_prob_total = that sum plus grad_prob [bs,Hb,Wb,D], the gradient reaching `prob` from
 * outside the core (the final product, :158-160).  grad_pooled is [bs,Hb*Wb,D*G].
 * aux and pooled (the forward's outputs) must not be NULL.
 * A range with cell0 < 0, ncells < 0 or cell0 + ncells > bs*Hb*Wb is rejected.
 * Outputs are indexed by GLOBAL cell.  The scatter targets grad_prob_map, grad_feat and
 * grad_occ (shaped like prob, feat and occ) are full maps that this range's contributions are
 * added to: the caller zeroes them, or starts grad_prob_map as a copy of grad_prob so that it
 * ends as grad_prob_total.
 * ---------------------------------------------------------------------------------- */
int vidar_latent_prob_forward(const float* occ, float* prob, float* aux, int bs, int D, int Hb,
                              int Wb, int grid_num, float grid_step, int act,
                              long long cell0, long long ncells, void* stream);
int vidar_latent_pool_forward(const float* prob, const float* feat, float* pooled, float* aux,
                              int bs, int D, int G, int Hb, int Wb, int grid_num,
                              float grid_step, float eps,
                              long long cell0, long long ncells, void* stream);
int vidar_latent_pool_backward(const float* prob, const float* feat, const float* pooled,
                               const float* aux, const float* grad_pooled,
                               float* grad_prob_map, float* grad_feat,
                               int bs, int D, int G, int Hb, int Wb, int grid_num,
                               float grid_step, float eps,
                               long long cell0, long long ncells, void* stream);
int vidar_latent_prob_backward(const float* occ, const float* aux, const float* grad_prob_total,
                               float* grad_occ, int bs, int D, int Hb, int Wb, int grid_num,
                               float grid_step, int act, long long cell0, long long ncells,
                               void* stream);

/* LatentRendering's projections around the ray-marching core, fused (one kernel per direction
 * on each side; replaces 3 + 6 skinny cuBLAS GEMMs and the elementwise kernels between them):
 *   latent_rendering.py:94   occ  = unsup_raymarching_head(embed)   (single Linear, num_pred_fcs == 0)
 *   latent_rendering.py:134  feat = lora_a(embed)
 *   latent_rendering.py:153-155  out = lora_b(pooled).view(.., D, E/D) * prob.view(.., D, 1)
 * rows = bs*Hb*Wb (or any contiguous row range of it: pass offset pointers); E = embed_dims
 * (128 or 256), D = pred_height, A = embed_dims / reduction; D + A <= 32.
 * Weights in nn.Linear layout [out, in].  Backward entry points ADD into grad_w and grad_b
 * (caller zero-fills) and overwrite the per-row gradients. */
int vidar_latent_proj_in_forward(const float* embed, const float* w_occ, const float* b_occ,
                                 const float* w_feat, const float* b_feat, float* occ, float* feat,
                                 long long rows, int E, int D, int A, void* stream);
int vidar_latent_proj_in_backward(const float* embed, const float* w_occ, const float* w_feat,
                                  const float* grad_occ, const float* grad_feat, float* grad_embed,
                                  float* grad_w_occ, float* grad_b_occ, float* grad_w_feat,
                                  float* grad_b_feat, long long rows, int E, int D, int A,
                                  void* stream);
int vidar_latent_proj_out_forward(const float* pooled, const float* prob, const float* w,
                                  const float* b, float* out, long long rows, int E, int D, int A,
                                  void* stream);
int vidar_latent_proj_out_backward(const float* grad_out, const float* pooled, const float* prob,
                                   const float* w, const float* b, float* grad_pooled,
                                   float* grad_prob, float* grad_w, float* grad_b,
                                   long long rows, int E, int D, int A, void* stream);

/* ------------------------------------------------------------------------------------
 * (i-b) BEV pillar -> camera projection, BEVFormerEncoder.point_sampling
 *   (projects/mmdet3d_plugin/bevformer/modules/encoder.py:94-156)
 *   ref3d [B, D, Q, 3] normalised pillar points; lidar2img [B, cams, 4, 4];
 *   pc_range_host: 6 floats in HOST memory (x0,y0,z0,x1,y1,z1); img_h/img_w = img_shape
 *   out: ref_cam [cams, B, Q, D, 2], bev_mask [cams, B, Q, D] (uint8 0/1).
 * ---------------------------------------------------------------------------------- */
int vidar_point_sampling(const float* ref3d, const float* lidar2img, const float* pc_range_host,
                         float* ref_cam, unsigned char* bev_mask, int B, int D, int Q, int cams,
                         float img_h, float img_w, void* stream);

/* ------------------------------------------------------------------------------------
 * (iii) nearest neighbour (K = 1) for the Chamfer distance -- SURVEY.md 8(f) item 2
 *   (third_lib/chamfer_dist/chamferdist/chamferdist/knn.cu:21-260, knn_cpu.cpp:7-106,
 *   chamfer.py:20-133; used by bevformer/utils/e2e_predictor_utils.py:163-183)
 *   p1 [N, P1, D], p2 [N, P2, D] (D = 2, 3 or 4); lengths1/2 [N] int64 (NULL = full)
 *   dists [N, P1] squared distance to the nearest p2 point, idx [N, P1] int64; zero padded
 *   beyond lengths1.  scratch: N*P1 uint64 (fully overwritten).
 * ---------------------------------------------------------------------------------- */
int vidar_nn_forward(const float* p1, const float* p2, const int64_t* lengths1,
                     const int64_t* lengths2, float* dists, int64_t* idx,
                     unsigned long long* scratch, int N, int P1, int P2, int D, void* stream);

/* knn_points_backward (knn_cpu.cpp:64-106): grad_p1 [N,P1,D] and grad_p2 [N,P2,D], both
 * caller-zeroed. */
int vidar_nn_backward(const float* p1, const float* p2, const int64_t* lengths1,
                      const int64_t* lengths2, const int64_t* idx, const float* grad_dists,
                      float* grad_p1, float* grad_p2, int N, int P1, int P2, int D, void* stream);

/* Segmented, masked NN (D = 3): segment s pairs the queries [q_off[s], q_off[s+1]) of q [Pq, 3] with the
 * candidates [c_off[s], c_off[s+1]) of c [Pc, 3]; q_off / c_off [S+1] int64 on the device.  q_mask / c_mask
 * (uint8, NULL = all kept): a zero entry is neither query nor candidate.  Per query: dists [Pq] the squared
 * distance to the nearest kept candidate of its segment (ties: smallest index), idx [Pq] its index within the
 * candidate segment, or VIDAR_NN_MASKED (masked query) / VIDAR_NN_EMPTY (no kept candidate at a finite
 * distance), with dists 0.  max_q / max_c: host-known upper bounds of the segment lengths (size the grid).
 * scratch: Pq uint64 (fully overwritten). */
#define VIDAR_NN_MASKED (-1)
#define VIDAR_NN_EMPTY (-2)
int vidar_nn_segments_forward(const float* q, const float* c, const int64_t* q_off, const int64_t* c_off,
                              const unsigned char* q_mask, const unsigned char* c_mask, float* dists,
                              int64_t* idx, unsigned long long* scratch, int S, long long Pq, int max_q,
                              int max_c, void* stream);

/* ------------------------------------------------------------------------------------
 * (iv) ViDAR's evaluation metrics -- Chamfer distance inside the point-cloud range and L1 / AbsRel ray errors
 *   (bevformer/detectors/vidar.py:452-497, utils/e2e_predictor_utils.py:146-183, utils/eval_utils.py:17-225)
 *   N = samples x frames clouds, n = b * F + f.  pred [Pp, 3], gt [Pg, 3] flat fp32, cloud n at rows
 *   [pred_off[n], pred_off[n+1]) / [gt_off[n], gt_off[n+1]) (int64 [N+1], device); origin [N, 3].
 * ---------------------------------------------------------------------------------- */

/* Fills the 3N-segment search layout:
 *   qbuf [Pp + 2Pg, 3] = pred xyz | gt xyz | gt spherical,  q_mask [Pp + 2Pg]
 *   cbuf [Pg + 2Pp, 3] = gt xyz | pred xyz | pred spherical, c_mask [Pg + 2Pp]
 *   q_off, c_off [3N+1]: segment n = forward Chamfer, N+n = backward Chamfer, 2N+n = spherical search.
 * xyz masks: inside pc_range_host (6 floats, HOST memory, inclusive); spherical points (atan2(x, y),
 * atan2(z, y), 1) of point - origin, masked where |point - origin| <= 1e-2. */
int vidar_eval_prologue(const float* pred, const float* gt, const float* origin, const int64_t* pred_off,
                        const int64_t* gt_off, const float* pc_range_host, float* qbuf, float* cbuf,
                        unsigned char* q_mask, unsigned char* c_mask, int64_t* q_off, int64_t* c_off,
                        int N, long long Pp, long long Pg, void* stream);

/* Ray errors and the deterministic per-cloud reduction over the NN results of the 3N segments
 * (vidar_nn_segments_forward on the prologue's layout; dists / idx [Pp + 2Pg]).
 *   partials: 3N * ceil(max_len / 256) * 4 doubles of scratch, max_len >= every cloud's size (a cloud whose points
 *       are all masked, like the trailing segment of vidar_eval_decode_clouds, may be longer: it adds nothing)
 *   out [N, VIDAR_EVAL_FIELDS] fp64: sum l1, sum absrel, count (gt points kept), sum forward d, pred points
 *       inside, sum backward d, gt points inside, flags (VIDAR_EVAL_* bits)
 *   rays [Pg, 9] (NULL = skip): interpolated point, clamped gt, clamped interpolated point (NaN for masked gt) */
#define VIDAR_EVAL_FIELDS 8
#define VIDAR_EVAL_GT_DEGENERATE 1       /* a gt ray outside PC_RANGE ends at its origin (RuntimeError) */
#define VIDAR_EVAL_GT_OUTSIDE 2          /* a clamped gt ray never touches the volume (AssertionError) */
#define VIDAR_EVAL_INTERP_DEGENERATE 4   /* the same two failures of an interpolated point */
#define VIDAR_EVAL_INTERP_OUTSIDE 8
#define VIDAR_EVAL_NO_PRED 16            /* gt points kept but no pred point kept */
int vidar_eval_metrics(const float* pred, const float* gt, const float* origin, const int64_t* pred_off,
                       const int64_t* gt_off, const int64_t* q_off, const unsigned char* q_mask,
                       const float* dists, const int64_t* idx, double* partials, double* out, float* rays,
                       int N, int max_len, void* stream);

/* The head's decoded rays -> the pred and gt clouds of every (sample, frame), in place of get_point_cloud_prediction's
 * per-(sample, frame) boolean masks (dense_heads/vidar_head_base.py:698-745, get_rendered_pcds :363-389).
 *   depth [bs, M]        arg-max depth of every row (voxel units; vidar_ray_argmax)
 *   rays [bs, M, 3]      GT points in voxel units;  points [bs, M, 3] the same points in metres
 *   tindex [bs, M]       float frame of each row; -1 or any value outside [0, F) = in no cloud
 *   origin_vox, origin   [bs, F, 3] in voxel units / metres;  scale = (pc_range[3] - pc_range[0]) / bev_w
 *   pc_range_host        6 floats (HOST), read when within_grid
 * Row i of sample b joins cloud n = b * F + t when tindex == t, gt_dist = |rays - origin_vox| * scale > 0 and (within_grid)
 * its metre point is inside pc_range.  Outputs:
 *   pred, gt [bs * M, 3] metres: origin + unit(point - origin) * dist with dist = depth * scale / gt_dist, the rows of a
 *            cloud in their original order
 *   off [bs * F + 2] int64: cloud n at rows [off[n], off[n+1]); segment bs * F, rows [off[bs*F], bs * M), holds the
 *            other rows as NaN, so vidar_eval_prologue masks all of them.  Pred and gt share the offsets.
 * Feed the N + 1 = bs * F + 1 segments to vidar_eval_prologue / _metrics with Pp = Pg = bs * M, max_len = M, and drop
 * the last row of the table.  3 launches (1 when M = 0), scratch from the library's memory pool, no host sync. */
int vidar_eval_decode_clouds(const float* depth, const float* rays, const float* points, const float* tindex,
                             const float* origin_vox, const float* origin, const float* pc_range_host, float scale,
                             int within_grid, float* pred, float* gt, int64_t* off, int bs, int M, int F,
                             void* stream);

/* ------------------------------------------------------------------------------------
 * (v) The head's dense loss term 'loss.dense_voxel' (dense_heads/vidar_head_base.py:594-659, get_rendered_pcds
 *   :344-389): Chamfer distance between the decoded dense rays and the GT cloud of P (gt sample, frame) pairs
 *   named by a pair table, one loss per group, in a fixed number of launches and without a host sync.
 *   ViDARRayHead: P = bs*F pairs n = b*F + f, Sg = bs, Fg = F, one group; ViDARHeadV1: a group per head frame.
 *   dist [P*R0], points [P*R0, 3]  decoded ray lengths and ray end points (voxel units), rays of pair n at
 *                                  n*R0 .. (n+1)*R0-1;  origin [No, 3] (voxel units)
 *   gt [Sg, M, 3], gt_tindex [Sg, M]  Sg gt samples, float frame 0..Fg-1, -1 = padding, any order; NULL when M = 0
 *   slot_pair [Sg*Fg] int32 (device): the pair of each (gt sample, frame) slot, -1 = none
 *   pair_table [P, 3] int32 (device): slot, origin row, group; pairs in increasing slot order
 *   pair_weight [P], group_norm [groups] (device)
 *   pc_range_host: 6 floats (HOST), used when within_grid (the reference's get_inside_mask on the voxel-unit end
 *   points).  W, H, Z: the grid size (gt box 0 < x < W-1, ...).
 *   Pred cloud of n: rays with dist > 0, point (o + unit(p - o) * dist - o) * 0.1 with o its origin row; gt cloud
 *   of n: rows of its slot's frame strictly inside the box, (g - o) * 0.1, in row order (it decides NN ties).
 * Forward outputs (Pq = P*R0 + Sg*M; all but loss are also inputs of the backward):
 *   qbuf, cbuf [Pq, 3]; q_mask, c_mask [Pq]; q_off, c_off [2P+1] int64; idx [Pq] int64: the search layout
 *   (segments 0..P-1 pred -> gt, P..2P-1 gt -> pred) and each query's nearest neighbour
 *   pairs [P, 4] fp64: sum pred->gt squared distances, pred points, sum gt->pred, gt points
 *   loss [groups]: loss[g] = sum_{n in g} w_n * (mean pred->gt + mean gt->pred) / 2 / group_norm[g] over pairs
 *   with gt points; NaN when a pair has gt points but no pred point.  Fixed-order fp64 sums: the same bits on
 *   every call.
 * Scratch from the library's memory pool.  Backward: grad_dist [P*R0] fully overwritten (0 for rays outside the
 * pred cloud), grad_loss [groups] the upstream gradient (device). */
int vidar_dense_chamfer_groups_forward(const float* dist, const float* points, const float* origin, const float* gt,
                                       const float* gt_tindex, const int32_t* slot_pair, const int32_t* pair_table,
                                       const float* pair_weight, const float* group_norm, const float* pc_range_host,
                                       float* qbuf, float* cbuf, unsigned char* q_mask, unsigned char* c_mask,
                                       int64_t* q_off, int64_t* c_off, int64_t* idx, double* pairs, float* loss,
                                       int P, int groups, int R0, int Sg, int Fg, int M, int W, int H, int Z,
                                       int within_grid, void* stream);
int vidar_dense_chamfer_groups_backward(const float* points, const float* origin, const float* qbuf,
                                        const float* cbuf, const unsigned char* q_mask, const int64_t* q_off,
                                        const int64_t* c_off, const int64_t* idx, const double* pairs,
                                        const int32_t* pair_table, const float* pair_weight,
                                        const float* group_norm, const float* grad_loss, float* grad_dist, int P,
                                        int groups, int R0, int Sg, int Fg, int M, void* stream);

/* ------------------------------------------------------------------------------------
 * (vi) ViDARHeadV1._get_reference_gt_points (dense_heads/vidar_head_v1.py:94-148) for every head frame at once:
 *   gt [bs, M, Cg]       GT rows (metres), NaN-padded, the frame in the last column
 *   mats [H*V, bs, 4, 4] src -> tgt transform of each (head frame i, slot v) job and sample; x' = [x y z 1] @ T
 *   jobs_host [H*V] int32 (HOST): source frame of job (i, v), -1 = none
 *   voxel_host [9] (HOST): off[3], scale[3], cells[3]; ray = ((x' - off) * scale) * cells
 * Outputs, segment s = i * bs + b:  rays [H*bs, M, 3] voxel units, tindex [H*bs, M] (v, -1 = padding),
 * points [H*bs, M, 3] metres (NULL = skip).  Rows of a segment are slot-major, the source rows of a slot in their
 * order, then padding (NaN).  3 launches, no host sync. */
int vidar_head_align_gt(const float* gt, const float* mats, const int32_t* jobs_host, const float* voxel_host,
                        float* rays, float* tindex, float* points, int bs, int M, int Cg, int H, int V,
                        void* stream);

/* ------------------------------------------------------------------------------------
 * (vii) Modulated deformable convolution (DCNv2): mmcv's modulated_deform_conv2d, the deformable 3x3 convs of the
 *   image backbone (ResNet-101 dcn=dict(type='DCNv2', ...), stage_with_dcn=(False, False, True, True)), groups = 1,
 *   deform_groups = 1.  The host runs the contraction as a GEMM over an explicit column matrix.
 *   x       [N, H, W, C]        input, channel-last
 *   offset  [N, 2*kh*kw, Ho, Wo] (dy, dx) of kernel point k = i*kw + j at channels 2k, 2k+1
 *   mask    [N, kh*kw, Ho, Wo]  modulation (after the sigmoid)
 *   Ho, Wo must equal the convolution's output size for the stride (sh, sw), padding (ph, pw), dilation (dh, dw).
 *   A call covers the images [n0, n0 + nb); column row m = (n - n0) * Ho * Wo + ho * Wo + wo.
 * Sample of (n, ho, wo, k): h = ho*sh - ph + i*dh + dy, w = wo*sw - pw + j*dw + dx; v_c = bilinear value of x[n, :, :, c]
 * on the floor cell, 0 when h <= -1, h >= H, w <= -1 or w >= W, corners outside the image add 0.
 *   cols [nb*Ho*Wo, kh*kw*C]  fully overwritten: mask * v_c at k*C + c (so y = cols @ weight.permute(0,2,3,1)^T) */
int vidar_dcn_im2col(const float* x, const float* offset, const float* mask, float* cols, int N, int C, int H, int W,
                     int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int n0, int nb,
                     void* stream);
/* Backward of the sampling, from grad_cols [nb*Ho*Wo, kh*kw*C] (the gradient of cols):
 *   grad_x      [N, H, W, C]         caller-zeroed, accumulated (mask * corner weight * grad_col)
 *   grad_offset [N, 2*kh*kw, Ho, Wo] written for images [n0, n0 + nb): mask * sum_c grad_col * d v_c / d(h, w)
 *   grad_mask   [N, kh*kw, Ho, Wo]   written for images [n0, n0 + nb): sum_c grad_col * v_c
 * d v / d(h, w) is the derivative of the bilinear form on the floor cell (one-sided on integer lines, 0 outside the
 * open range).  Both calls take 16-byte vector paths when C % 4 == 0 and the buffers are 16-byte aligned. */
int vidar_dcn_col2im(const float* x, const float* offset, const float* mask, const float* grad_cols, float* grad_x,
                     float* grad_offset, float* grad_mask, int N, int C, int H, int W, int Ho, int Wo, int kh, int kw,
                     int sh, int sw, int ph, int pw, int dh, int dw, int n0, int nb, void* stream);

/* The same two calls with x, offset, mask and cols / grad_cols in 16 bits: `dtype` is VIDAR_DTYPE_F16 (IEEE half)
 * or VIDAR_DTYPE_BF16 (bfloat16); any other value returns VIDAR_E_INVALID ("unsupported dtype").  Every value is
 * converted to fp32 on load, so a sample lands where the fp32 op puts it for the same (rounded) offsets; bilinear
 * weights, products and sums are fp32.  im2col rounds each column element once, to `dtype`.  col2im accumulates
 * grad_x and writes grad_offset / grad_mask in fp32 (same layouts as above).  The vector paths (8 channels per
 * 16-byte load) run when C % 8 == 0 and the buffers are 16-byte aligned. */
#define VIDAR_DTYPE_F16 1
#define VIDAR_DTYPE_BF16 2
int vidar_dcn_im2col_half(const void* x, const void* offset, const void* mask, void* cols, int dtype, int N, int C,
                          int H, int W, int Ho, int Wo, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                          int n0, int nb, void* stream);
int vidar_dcn_col2im_half(const void* x, const void* offset, const void* mask, const void* grad_cols, float* grad_x,
                          float* grad_offset, float* grad_mask, int dtype, int N, int C, int H, int W, int Ho, int Wo,
                          int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int n0, int nb,
                          void* stream);

/* ------------------------------------------------------------------------------------
 * (viii) Deformable convolution v3 (InternImage's DCNv3 core op, ops_dcnv3 `dcnv3_forward` / `dcnv3_backward`).
 *   `dtype` VIDAR_DTYPE_F32, _F16 or _BF16 is the storage type of every buffer but grad_input; anything else returns
 *   VIDAR_E_INVALID ("unsupported dtype").  All arithmetic is fp32, each stored value is rounded once.
 *   input   [N, H, W, group*group_channels]      channel-last
 *   offset  [N, Ho, Wo, group*K*2]              (dx, dy) of kernel point p = i*kernel_h + j (i < kernel_w along x)
 *   mask    [N, Ho, Wo, group*K]                weights (softmaxed by the caller), K = kernel_h*kernel_w
 *   output  [N, Ho, Wo, group*group_channels]   fully overwritten
 *   Ho = (H + 2*pad_h - (dilation_h*(kernel_h-1)+1)) / stride_h + 1, Wo likewise; both must be positive.
 * Sample of (n, ho, wo, g, p), s = offset_scale, cw = (dilation_w*(kernel_w-1)) >> 1, ch likewise:
 *   x = wo*stride_w - pad_w + cw + (i*dilation_w - cw + dx)*s,  y = ho*stride_h - pad_h + ch + (j*dilation_h - ch + dy)*s;
 *   it adds mask * bilinear value (floor cell, corners outside the image read 0) when -1 < y < H and -1 < x < W.
 * im2col_step > 0 and N % min(N, im2col_step) == 0 (the reference's rule); it does not change the computation.
 * One launch each, on `stream`, no host sync.  Vector paths when group_channels is a multiple of 4 (fp32) / 8 (16-bit)
 * and input, output / grad_output, grad_input are 16-byte aligned. */
enum { VIDAR_DTYPE_F32 = 0 };  /* next to VIDAR_DTYPE_F16 = 1 and VIDAR_DTYPE_BF16 = 2 of the DCNv2 calls */
int vidar_dcnv3_forward(const void* input, const void* offset, const void* mask, void* output, int dtype, int N, int H,
                        int W, int group, int group_channels, int kernel_h, int kernel_w, int stride_h, int stride_w,
                        int pad_h, int pad_w, int dilation_h, int dilation_w, float offset_scale, int im2col_step,
                        void* stream);
/* Backward from grad_output [N, Ho, Wo, group*group_channels] (dtype):
 *   grad_input  [N, H, W, group*group_channels] fp32, caller-zeroed, accumulated (mask * corner weight * grad_out)
 *   grad_offset [N, Ho, Wo, group*K*2] (dtype)  written: offset_scale * mask * sum_c grad_out * d v_c / d(x, y)
 *   grad_mask   [N, Ho, Wo, group*K] (dtype)    written: sum_c grad_out * v_c
 * d v / d(x, y) is the derivative of the bilinear form on the floor cell (one-sided on integer lines); a point
 * outside the open range, one exactly on -1 included, gets 0 for every gradient. */
int vidar_dcnv3_backward(const void* input, const void* offset, const void* mask, const void* grad_output,
                         float* grad_input, void* grad_offset, void* grad_mask, int dtype, int N, int H, int W,
                         int group, int group_channels, int kernel_h, int kernel_w, int stride_h, int stride_w,
                         int pad_h, int pad_w, int dilation_h, int dilation_w, float offset_scale, int im2col_step,
                         void* stream);

/* ------------------------------------------------------------------------------------
 * (ix) GridMask (models/utils/grid_mask.py GridMask.forward) from its numpy draws, in one launch.
 *   x, out  [N, C, h, w] contiguous, `dtype` VIDAR_DTYPE_F32, _F16 or _BF16 (anything else returns VIDAR_E_INVALID)
 *   offset  [h, w] (dtype) or NULL
 *   out = x * mask                       (offset NULL)
 *   out = x * mask + offset * (1 - mask) (offset given)
 * in `dtype`: every product is exact (mask is 0 or 1) and the sum rounds once, as the reference's statements do.
 * mask [h, w] is the reference's: stripes of period d and length l from st_h / st_w (rows when use_h, columns when
 * use_w) on an (int(1.5 h), int(1.5 w)) frame of ones, rotated by PIL's Image.rotate(r) (nearest, fill 0), centre
 * crop, inverted when mode == 1; it is evaluated per pixel in registers, never stored.
 * Needs 1 <= h, w <= 8192, d >= 2, 0 <= l <= d, 0 <= st_h, st_w < d; use_h, use_w and mode 0 or 1; buffers
 * aligned to their elements.  16-byte vectors when h*w is a multiple of 4 (fp32) / 8 (16-bit) and x, offset and out
 * are 16-byte aligned.  out may not overlap x or offset.  N*C == 0 is a no-op.  One launch on `stream`, no scratch,
 * no host sync.  The backward (d out / d x = mask) is the same call on grad_out with offset NULL. */
int vidar_grid_mask_apply(const void* x, const void* offset, void* out, int dtype, int N, int C, int h, int w, int d,
                          int l, int st_h, int st_w, int r, int use_h, int use_w, int mode, void* stream);

/* ------------------------------------------------------------------------------------
 * (x) The multi-view image pipelines of the pre-training and fine-tuning configs (datasets/pipelines/transform_3d.py
 * PhotoMetricDistortionMultiViewImage, NormalizeMultiviewImage, PadMultiViewImage; augmentation.py
 * CropResizeFlipImage, RandomCropResizeFlipImage) from one frame's uint8 images, bit for bit the reference's cv2 /
 * PIL / numpy statements.
 *
 * vidar_image_aug_apply: photometric distortion with numpy's wrapping uint8 cast, crop / resize / window / flip,
 * normalisation and padding, in two launches on `stream`.
 *   src      [N, H, W, 3] uint8 BGR (device), 1 <= N <= 64
 *   mid      [N, crop_h, mid_w, 3] uint8 (device): the intermediate between the two passes, the only scratch;
 *            mid_w = min(win_x + win_w, out_w) - max(win_x, 0), the resized columns inside the window
 *   out      [N, 3, Hp, Wp] float32 (device), every element written
 *   photo_i  host int32 [N, 8] (brightness, contrast, saturation, hue gates, mode 1, perm[3]) and
 *   photo_f  host float [N, 4] (brightness delta, contrast factor, saturation factor, hue delta): one image's
 *            photometric draws each (both NULL: no photometric step); copied into the kernel arguments
 *   crop box (crop_x, crop_y, crop_x + crop_w, crop_y + crop_h) of the image, zero outside it; then Pillow's
 *   bicubic resize to (out_w, out_h); then the window (win_x, win_y, win_x + win_w, win_y + win_h) of the resized
 *   image, zero outside it (CropResizeFlipImage: (0, 0, out_w, out_h); RandomCropResizeFlipImage crops the whole
 *   image, and the window is its crop); with flip, the left-right flip of the window
 *   htaps    [out_w, 2 + hk] int32 (device): per resized column (xmin, count, count weights in 2^-22, zero-padded
 *            to hk); given exactly when out_w != crop_w.  vtaps [out_h, 2 + vk] likewise for rows.  Only the
 *            entries of resized columns / rows inside the window are read.
 *   to_rgb swaps channels 0 and 2; then out = f32(double(x - mean[c]) * stdinv[c]) with mean host float[3] and
 *   stdinv host double[3]; pixels at y >= win_h or x >= win_w are pad_val[c] (host float[3]).
 * Needs every side in [1, 8192], win_h <= Hp, win_w <= Wp, a window that overlaps the resized image, gates 0 or 1,
 * perm a permutation of (0, 1, 2).  No host sync.
 *
 * vidar_image_aug_normalize: the chain without a crop step, in one launch on `stream` with no scratch: the
 * photometric statements on float32 (no uint8 cast, unclamped) when photo_i / photo_f are given, then the same
 * normalisation and padding to [N, 3, Hp, Wp] (pixels at y >= H or x >= W are pad_val[c]).  Needs 1 <= N <= 64,
 * H <= Hp <= 8192, W <= Wp <= 8192.  No host sync. */
int vidar_image_aug_apply(const unsigned char* src, unsigned char* mid, float* out, int N, int H, int W,
                          const int32_t* photo_i, const float* photo_f, int crop_x, int crop_y, int crop_w,
                          int crop_h, int out_w, int out_h, int win_x, int win_y, int win_w, int win_h,
                          const int32_t* htaps, int hk, const int32_t* vtaps, int vk, int flip, int to_rgb,
                          const float* mean, const double* stdinv, const float* pad_val, int Hp, int Wp, void* stream);
int vidar_image_aug_normalize(const unsigned char* src, float* out, int N, int H, int W, const int32_t* photo_i,
                              const float* photo_f, int to_rgb, const float* mean, const double* stdinv,
                              const float* pad_val, int Hp, int Wp, void* stream);
/* vidar_image_aug_scale: the OpenScene configs' chain in one launch on `stream` with no scratch: the photometric
 * statements on float32 (unclamped) when photo_i / photo_f are given, the same normalisation, then
 * RandomScaleImageMultiViewImage's mmcv.imresize by 2/3 (cv2.resize INTER_LINEAR on float32, as cv2 with IPP
 * computes it: along x within each source row, then between the rows, each a + t * (b - a) with one fused
 * multiply-add) to out_h x out_w, then padding to [N, 3, Hp, Wp] (pixels at y >= out_h or x >= out_w are
 * pad_val[c]).  Needs 1 <= N <= 64, 2 * H == 3 * out_h, 2 * W == 3 * out_w, out_h <= Hp <= 8192,
 * out_w <= Wp <= 8192.  No host sync. */
int vidar_image_aug_scale(const unsigned char* src, float* out, int N, int H, int W, const int32_t* photo_i,
                          const float* photo_f, int to_rgb, const float* mean, const double* stdinv,
                          const float* pad_val, int out_h, int out_w, int Hp, int Wp, void* stream);

/* ------------------------------------------------------------------------------------
 * (xi) The point half of a pre-training sample (datasets/pipelines/loading.py CustomLoadPointsFromMultiSweeps,
 * CustomVoxelBasedPointSampler over mmdet3d 0.17.1's VoxelBasedPointSampler; nuscenes_vidar_dataset_v1.py union2one's
 * point statements) for every frame of a queue, in a fixed number of launches on `stream`.
 *   raw      float32 raw points, rows of `cols` = 5 (nuScenes) or 6 (nuPlan) (device); seg_i [S, 5] int64 and seg_d
 *            [S, 17] double (device): per segment raw row offset, n, offset in the call's point space, filter (0 none,
 *            1 remove-close, 2 also the ego box), flags (bit 0 the sweep transform, bit 1 column 4 := time, 6 columns
 *            only); R row-major, t, ego box (x_lo, y_lo, x_hi, y_hi), time.  Segments are frame-major
 *            and the call's point space is their concatenation (n_g points).
 *   frame_i  [F, 10] int64 (device): merged offset, merged count, output row offset, output rows, queue index,
 *            voxel sampler (0 / 1), grid offset, perm offset, point-space offset, point-space count;
 *            frame_f [F, 6] float (voxel lo, voxel size), frame_g [F, 3] int64 (grid dims) (device)
 *   perm     int32 (device): per voxel frame its shuffled order of the merged points (numpy's draws)
 *   n_cur    merged points over all frames (the host's count), cells = voxel grid cells over all frames
 *   ego      host float[4] (x_lo, y_lo, x_hi, y_hi) of union2one's mask, or NULL for no mask
 *   out      [rows, cols] float32 (device): each frame's kept points (x, y, z, intensity, queue index; with 6 columns
 *            x, y, z, intensity, column 4 -- the segment's time with flag bit 1, else the raw value --, queue index)
 *            in the reference's order within its rows; masked and unused rows are NaN
 *   counts   optional int32 [F, 2] (device): per frame the merged points and the kept points the device found
 *   out_compact / count: optional float32 [rows, cols] and int64 [1] (device): the non-NaN rows in order and their number
 * Needs every n below 2^31.  No host sync. */
int vidar_point_pipeline_gather(const float* raw, const int64_t* seg_i, const double* seg_d, int S,
                                const int64_t* frame_i, const float* frame_f, const int64_t* frame_g, int F,
                                const int32_t* perm, long long n_g, long long n_cur, long long cells, const float* ego,
                                float* out, long long rows, int32_t* counts, float* out_compact, int64_t* count,
                                int cols, void* stream);

/* ------------------------------------------------------------------------------------
 * (xii) Baseline JPEG decoding of a queue's camera images (the pre-training loader's cv2.imread(name,
 * IMREAD_UNCHANGED)), bit for bit libjpeg-turbo's default decode, in three launches on `stream` whatever n is.
 *   blob     device, 16-byte aligned, the layout vidar_b200/jpeg.py `pack` writes: int32 image headers [n, 64],
 *            derived Huffman tables [n, 6, 804], quantisation tables [n, 3, 64] (natural order), first block of each
 *            (image, component) [3n + 1], first pixel of each image [n + 1], subsequences [nsub, 5] (start bit, end
 *            bit, first subsequence of its restart interval, the interval's first and end block), then every image's
 *            entropy-coded bytes with stuffing and restart markers removed
 *   blocks   8x8 blocks over all images and components; samples = 64 * blocks; pixels = sum of H * W
 *   out      uint8 [pixels, 3] (device): each image's [H, W, 3] BGR at 3 * its first pixel
 * Needs 1 <= n <= 4096, blocks * 64, samples and pixels below 2^31.  Scratch (per-subsequence states, coefficients,
 * component planes) comes from the library's stream-ordered pool.  Corrupt entropy data gives unspecified pixels but
 * no access outside the blob, the scratch or out.  No host sync. */
int vidar_jpeg_decode(const void* blob, int n, int nsub, long long blocks, long long samples, long long pixels,
                      unsigned char* out, void* stream);

/* ------------------------------------------------------------------------------------
 * (xiii) The gradient bucket of the data-parallel step (vidar_b200/grad_bucket.py): n gradients in and out of one
 * flat fp32 bucket, for ONE all-reduce of every trainable parameter's gradient.  The table is in HOST memory:
 *   ptr_host    [n] device address of gradient i (fp32, contiguous, 4-byte aligned); pack: 0 = no gradient (packs
 *               as zeros); unpack: must be non-zero where numel_host[i] > 0
 *   numel_host  [n] its elements (0 allowed);  offset_host [n] its first element in the bucket (any value with
 *               offset + numel <= bucket_numel)
 *   scale_host  [n] pack only: bucket[offset_i + j] = grad_i[j] * scale_i, one fp32 multiply
 * unpack writes grad_i[j] = bucket[offset_i + j].  One launch per 1024 tensors on `stream`, no scratch, no host sync. */
int vidar_grad_bucket_pack(const int64_t* ptr_host, const int64_t* numel_host, const int64_t* offset_host,
                           const float* scale_host, int n, float* bucket, long long bucket_numel, void* stream);
int vidar_grad_bucket_unpack(const float* bucket, long long bucket_numel, const int64_t* ptr_host,
                             const int64_t* numel_host, const int64_t* offset_host, int n, void* stream);

/* ------------------------------------------------------------------------------------
 * (xiv) The optimizer step of the pre-training configs (vidar_b200/optim.py): clip every gradient to a total 2-norm
 * (torch.nn.utils.clip_grad_norm_) and step AdamW (torch.optim.AdamW's single-tensor update) over n parameters.  The
 * table is in HOST memory:
 *   param_host   [n] device address of parameter i (fp32, contiguous, 4-byte aligned; non-zero where numel > 0)
 *   grad_host    [n] device address of its gradient, same layout; 0 = no gradient: parameter i is skipped (no decay,
 *                no state change) and left out of the norm
 *   numel_host   [n] elements of parameter i (0 allowed)
 *   scalar_host  [n, 7] fp32 per parameter: 1 - lr*wd, -lr/bc1, 1/sqrt(bc2) (from its own step count), and
 *                1 - beta1, beta2, 1 - beta2, eps
 *   exp_avg, exp_avg_sq  flat fp32 state [state_numel] in table order: parameter i owns the numel_host[i] elements
 *                after those of parameters 0 .. i-1 (sum of numel_host <= state_numel)
 *   clip         non-zero: every gradient is multiplied by clamp(max_norm / (norm + 1e-6), max=1) first, norm being
 *                the 2-norm of every gradient (summed in fp64, in a fixed order), which is stored to grad_norm
 *                (device fp32 scalar); 0: no clipping, max_norm and grad_norm unused
 * Launches: one norm kernel (clip only) and one update kernel per run of at most 896 parameters that share beta1,
 * beta2 and eps -- two for the pre-training model.  Bitwise deterministic; no host sync; the norm partials come from
 * the library's stream-ordered pool. */
int vidar_adamw_step(const int64_t* param_host, const int64_t* grad_host, const int64_t* numel_host,
                     const float* scalar_host, int n, float* exp_avg, float* exp_avg_sq, long long state_numel,
                     int clip, float max_norm, float* grad_norm, void* stream);

/* ------------------------------------------------------------------------------------
 * (xv) TemporalSelfAttention's value with ego motion (modules/transformer.py:137-150, modules/encoder.py:225-229,
 * vidar_b200/ego_motion.py): the previous BEV rotated by the frame's yaw change, stacked with the query.
 *   prev, query  [bs, Q, C] fp32;  rows [bs, Q] int32: output cell q copies source cell rows[b, q] of sample b's
 *                previous BEV where rows[b, q] lies in [0, Q), zeros otherwise (any value is safe);  C a multiple
 *                of 4
 *   forward   value [bs * 2, Q, C]: value[2b] = the rotated previous BEV, value[2b + 1] = query[b]
 *   backward  grad_prev[b, s] = the sum of grad_value[2b, q] over the q with rows[b, q] = s, in ascending q (a stable
 *             radix sort of the map; no float atomics, bitwise deterministic); grad_query[b] = grad_value[2b + 1]
 * One launch forward; backward one memset, two small kernels, a radix sort and one gather, its scratch from the
 * library's stream-ordered pool.  No host sync. */
int vidar_bev_rotate_stack_forward(const float* prev, const float* query, const int32_t* rows, float* value, int bs,
                                   int Q, int C, void* stream);
int vidar_bev_rotate_stack_backward(const float* grad_value, const int32_t* rows, float* grad_prev, float* grad_query,
                                    int bs, int Q, int C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VIDAR_B200_H_ */
