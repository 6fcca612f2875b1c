"""Loss / decoding half of the ViDAR head on the CUDA ray kernels.

Mirror of the parts of `ViDARHeadBase` that sit on the hot path -- the future-BEV transformer the
reference class also owns is out of scope (SURVEY.md 2) -- with the reference's method names,
arguments, returned keys and arithmetic
(projects/mmdet3d_plugin/bevformer/dense_heads/vidar_head_base.py):

  _process_gt_points               :219-276   GT point lists -> padded voxel-unit rays + tindex
  loss                             :510-660   'regularization.loss' (CE over 513 ray samples),
                                              'dist.loss', 'loss.dense_voxel' (gumbel decode + Chamfer)
  get_point_cloud_prediction       :662-752   arg-max decode -> predicted / GT point clouds
  get_rendered_pcds                :344-389
  _custom_gumbel_softmax_distance  :754-773
  evaluate / evaluate_device       detectors/vidar.py:439-497 (forward_test's decode + metric loop), batched

What runs where: the CE term never materialises the [levels, rays, 513] logits
(`ray_head.ce_regularization_loss`, one fused kernel per frame set); the dense term's gumbel decode
is fused with the sampler as well (`ray_head.gumbel_distance`), and its Chamfer distance over every
(sample, frame) pair is one batched op (`ray_head.dense_chamfer_loss`: segmented nearest-neighbour search in
place of mmdet3d's O(N*M) distance matrix, `chamfer_distance` with criterion 'l2', reduction 'mean': the mean
squared NN distance each way).  With CE + dense (use_dist_loss=False) `loss` runs forward and backward without
a host sync.  `ViDARRayHeadV1` is the same for ViDARHeadV1 (vidar_head_v1.py): every head frame's GT
alignment and loss in one batched pass.  The distance term samples through `ray_head.get_grid_features` (CUDA
sampler) and then follows the reference's torch statements; decoding is `ray_head.decode_ray_depth`.
`evaluate` decodes, renders and scores every (sample, frame) in one pass without a host sync before its final
copy (`ray_head.ray_argmax` over every row, `ray_head.decode_clouds`, `evaluate.metrics_flat`).
CUDA only, like everything else in this package.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import bev_geometry, chamfer, ray_head
from . import evaluate as eval_metrics


def get_inside_mask(points, point_cloud_range):
    """bevformer/utils/e2e_predictor_utils.py:146-160."""
    r = point_cloud_range
    return ((r[0] <= points[..., 0]) & (points[..., 0] <= r[3]) & (r[1] <= points[..., 1]) & (points[..., 1] <= r[4])
            & (r[2] <= points[..., 2]) & (points[..., 2] <= r[5]))


def chamfer_l2_mean(src, dst):
    """mmdet3d.models.losses.chamfer_distance(src, dst) with its defaults (criterion 'l2',
    reduction 'mean', unit weights) -> (loss_src, loss_dst): mean squared distance to the nearest
    neighbour in the other cloud.  src [1,N,3], dst [1,M,3]."""
    a = chamfer.knn_points(src, dst)
    b = chamfer.knn_points(dst, src)
    return a.dists[..., 0].mean(), b.dists[..., 0].mean()


class ViDARRayHead:
    """The ray-supervision logic of ViDARHeadBase (not an nn.Module: it owns no parameters)."""

    def __init__(self, ray_grid_num=1026, ray_grid_step=1.0, use_ce_loss=True, use_dist_loss=False,
                 use_dense_loss=True, dense_loss_weight=1.0, loss_weight=None, eval_within_grid=False):
        self.ray_grid_num = ray_grid_num
        self.ray_grid_step = ray_grid_step
        self.use_ce_loss = use_ce_loss
        self.use_dist_loss = use_dist_loss
        self.use_dense_loss = use_dense_loss
        assert self.use_ce_loss or self.use_dist_loss or self.use_dense_loss
        self.dense_loss_weight = dense_loss_weight
        self.loss_weight = np.array(loss_weight)
        assert self.loss_weight.shape[-1] == 1
        self.eval_within_grid = eval_within_grid
        self.fuse_dense_decode = True     # False: dense term through the materialising sampler + torch statements
        self.fuse_dense_chamfer = True    # False: the reference's per-pair Chamfer loop (boolean masks, host syncs)

    # ------------------------------------------------------------------ ground truth (:219-276)
    def _process_gt_points(self, bev_preds, gt_points, batched_origin_points, valid_frames, start_idx,
                           pred_frame_num, bev_h, bev_w, pc_range):
        valid_frame_num, inter_num, bs, token_num, num_height_pred = bev_preds.shape
        frames = [i for i in range(start_idx, pred_frame_num) if i in valid_frames]
        # The reference selects every frame's points with a boolean mask (a host sync per (batch, frame)),
        # concatenates them in frame order and NaN-pads to the longest sample (:239-262).  Same rays, same
        # order, no sync: a stable sort by the frame's position in `frames`; points of other frames become
        # padding (NaN coordinates, tindex -1) at the tail instead of being dropped -- every consumer skips
        # padded rays, so only the padded length differs (it is the input length, known on the host).
        max_pts = max(int(p.shape[0]) for p in gt_points[:bs])
        pts = bev_preds.new_full((bs, max_pts, 3), float("nan"))
        tindex = bev_preds.new_full((bs, max_pts), -1.0)
        for b in range(bs):
            cur = gt_points[b]
            f = cur[:, -1]
            key = torch.full_like(f, float(len(frames)))
            for r, i in enumerate(frames):
                key = torch.where(f == i, torch.full_like(f, float(r)), key)
            order = torch.argsort(key, stable=True)
            keep = (key[order] < len(frames))
            srt = cur[order]
            pts[b, : cur.shape[0]] = torch.where(keep[:, None], srt[:, :3].to(pts.dtype), float("nan"))
            tindex[b, : cur.shape[0]] = torch.where(keep, srt[:, -1].to(pts.dtype) - start_idx, -1.0)
        if batched_origin_points is None:
            batched_origin_points = torch.zeros((bs, len(valid_frames), 3), dtype=bev_preds.dtype, device=bev_preds.device)
        origin_grids = bev_geometry.coords_to_voxel_grids(batched_origin_points, bev_h=bev_h, bev_w=bev_w,
                                                          pillar_num=num_height_pred, pc_range=pc_range)
        gt_grids = bev_geometry.coords_to_voxel_grids(pts, bev_h=bev_h, bev_w=bev_w, pillar_num=num_height_pred,
                                                      pc_range=pc_range)
        tindex = torch.clamp(tindex, max=valid_frame_num - 1)
        return origin_grids, batched_origin_points, gt_grids, pts, tindex

    # ------------------------------------------------------------------ decode helpers
    def get_rendered_pcds(self, origin, points, tindex, gt_dist, pred_dist, pc_range):
        """:344-389 -> pcds[b][t] = origin_t + unit(points - origin_t) * pred_dist for rays of frame t with gt_dist > 0."""
        bs, num_frames, _ = origin.shape
        pcds = []
        for b in range(bs):
            cur = []
            for t in range(num_frames):
                mask = torch.logical_and(tindex[b] == t, gt_dist[b] > 0.)
                if self.eval_within_grid:
                    mask = torch.logical_and(mask, get_inside_mask(points[b], pc_range))
                p = points[b][mask]
                r = p - origin[b, t].view(1, 3)
                r_norm = r / torch.sqrt((r ** 2).sum(1, keepdims=True))
                cur.append(origin[b, t].view(1, 3) + r_norm * pred_dist[b][mask].view(-1, 1))
            pcds.append(cur)
        return pcds

    def _custom_gumbel_softmax_distance(self, grid_embed, grid_length, gumbels=None):
        """:754-773: sample one waypoint per ray by Gumbel-max, return its length with the gradient of
        `length * P(a waypoint beyond it)` (straight-through on the probability).
        `gumbels`: optional pre-drawn Gumbel(0,1) noise of grid_embed's shape (tests pin the reference's
        CPU draw this way); None draws with the statement F.gumbel_softmax uses, so the generator is
        consumed exactly like in the reference.  The hard one-hot of F.gumbel_softmax is
        `y_hard - y_soft.detach() + y_soft`, whose picked entry is exactly 1.0f and whose other entries are
        exactly 0 in fp32, so `(hard * length).sum(-1)` equals the gather below bit for bit."""
        if gumbels is None:
            gumbels = -torch.empty_like(grid_embed, memory_format=torch.legacy_contiguous_format).exponential_().log()
        pick = (grid_embed + gumbels).softmax(-1).max(-1, keepdim=True)[1]
        sampled = grid_length.gather(-1, pick).squeeze(-1).detach()
        weight = torch.exp(grid_embed - grid_embed.max(-1, keepdim=True)[0])
        beyond = (weight * (grid_length > sampled.unsqueeze(-1)).float()).sum(-1) / weight.sum(-1)
        return (1 - beyond.detach() + beyond) * sampled

    @staticmethod
    def _dense_grid(bev_h, bev_w, Z, device):
        """The dense term's ray end points of one sample (vidar_head_base.py:611-619), [R0, 3] voxel units."""
        interval = 4
        g = bev_geometry.get_bev_grids_3d(bev_h // interval, bev_w // interval, Z // interval, bs=1, device=device)
        g[..., 0] = g[..., 0] * bev_w
        g[..., 1] = g[..., 1] * bev_h
        g[..., 2] = g[..., 2] * Z
        return g.view(-1, 3).contiguous()

    @staticmethod
    def _sigma_volume(level, bs, frames, heights, bev_h, bev_w):
        """[frames, bs, bev_h*bev_w, heights] -> [bs, frames, heights, bev_h, bev_w] (:557-563)."""
        return level.permute(1, 0, 3, 2).contiguous().view(bs, frames, heights, bev_h, bev_w)

    # ------------------------------------------------------------------ loss (:510-660)
    def loss(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, pred_frame_num,
             img_metas=None, batched_origin_points=None, loss_weight=None, gumbels=None):
        """`gumbels`: optional dict {'dist': noise, 'dense': noise} forwarded to the gumbel decode."""
        valid_frames = pred_dict["valid_frames"]
        sigma = pred_dict["next_bev_preds"][:, -1:].float()     # last intermediate output only (:540); force_fp32
        valid_frame_num, inter_num, bs, token_num, num_height_pred = sigma.shape
        (origin_grids, batched_origin_points, gt_grids, batched_gt_points, gt_tindex) = self._process_gt_points(
            sigma, gt_points, batched_origin_points, valid_frames, start_idx, pred_frame_num, tgt_bev_h, tgt_bev_w,
            tgt_pc_range)
        inter_sigma = [self._sigma_volume(sigma[:, i], bs, valid_frame_num, num_height_pred, tgt_bev_h, tgt_bev_w)
                       for i in range(inter_num)]
        step = self.ray_grid_step
        loss_weight = self.loss_weight if loss_weight is None else loss_weight
        gumbels = gumbels or {}
        loss_dict = dict()
        if self.use_dist_loss:
            r_mask, r_feat, r_w, r_len = ray_head.get_grid_features(origin_grids, gt_grids, gt_tindex, inter_sigma,
                                                                    loss_weight, step, self.ray_grid_num)
            r_pred = self._custom_gumbel_softmax_distance(r_feat + r_mask, r_len[None], gumbels.get("dist"))
            scale = (tgt_pc_range[3] - tgt_pc_range[0]) / tgt_bev_w
            dist_loss = torch.abs(r_pred - r_len[None, :, 0]) * scale
            loss_dict["dist.loss"] = (dist_loss * r_w).sum() / torch.clamp(r_w.sum(), min=1)
        if self.use_ce_loss:
            loss_dict["regularization.loss"] = ray_head.ce_regularization_loss(
                origin_grids, gt_grids, gt_tindex, inter_sigma, loss_weight, step, self.ray_grid_num)
        if self.use_dense_loss:
            tgt = inter_sigma[-1]
            grid = self._dense_grid(tgt_bev_h, tgt_bev_w, num_height_pred, sigma.device)
            R0 = grid.shape[0]
            voxel_grids = grid.repeat(bs * valid_frame_num, 1).view(bs, -1, 3)
            voxel_tindex = (torch.arange(valid_frame_num, dtype=gt_tindex.dtype, device=sigma.device)
                            .repeat_interleave(R0).repeat(bs, 1))
            if self.fuse_dense_decode:
                # sampler + gumbel decode in one kernel over the bs * F volumes (ray volume b * F + f): the
                # [bs, rays, ray_grid_num] logits / softmax / one-hot tensors are never written.  The noise is drawn
                # with the statement F.gumbel_softmax uses, on the shape its logits would have.
                noise = gumbels.get("dense")
                if noise is None:
                    noise = -torch.empty((bs, voxel_grids.shape[1], self.ray_grid_num), dtype=torch.float32,
                                         device=sigma.device).exponential_().log()
                frame = torch.arange(bs * valid_frame_num, dtype=torch.int32, device=sigma.device).repeat_interleave(R0)
                dense_dist = ray_head.gumbel_distance(
                    tgt.view(bs * valid_frame_num, num_height_pred, tgt_bev_h, tgt_bev_w),
                    origin_grids[:, :valid_frame_num].reshape(bs * valid_frame_num, 3).float(),
                    voxel_grids.view(-1, 3), frame, self.ray_grid_num, step,
                    noise.reshape(-1, self.ray_grid_num)).view(bs, -1)
            else:
                _, d_feat, _, d_len = ray_head.get_grid_features(
                    origin_grids, voxel_grids, voxel_tindex, [tgt], np.array([[1]] * valid_frame_num), step,
                    self.ray_grid_num, return_as_batch=True)
                d_feat = d_feat[0][..., 1:].contiguous()
                d_len = d_len[..., 1:].contiguous()
                dense_dist = self._custom_gumbel_softmax_distance(d_feat, d_len, gumbels.get("dense"))
            if self.fuse_dense_chamfer:
                # every (sample, frame) pair in one op: no boolean masks, no host sync
                dense = ray_head.dense_chamfer_loss(
                    dense_dist.contiguous(), voxel_grids.contiguous(), origin_grids.float().contiguous(),
                    gt_grids.float().contiguous(), gt_tindex.float().contiguous(),
                    (tgt_bev_w, tgt_bev_h, num_height_pred), [loss_weight[f, 0] for f in range(valid_frame_num)],
                    float(loss_weight.sum()), self.eval_within_grid, tgt_pc_range)
            else:
                voxel_pcd = self.get_rendered_pcds(origin_grids, voxel_grids, voxel_tindex, dense_dist, dense_dist,
                                                   tgt_pc_range)
                dense = 0
                for b in range(bs):
                    for f in range(valid_frame_num):
                        pred = voxel_pcd[b][f].view(1, -1, 3)
                        gt = gt_grids[b][gt_tindex[b] == f].view(1, -1, 3)
                        m = ((gt[..., 0] < tgt_bev_w - 1) & (gt[..., 0] > 0) & (gt[..., 1] < tgt_bev_h - 1)
                             & (gt[..., 1] > 0) & (gt[..., 2] < num_height_pred - 1) & (gt[..., 2] > 0))
                        gt = gt.squeeze(0)[m.squeeze(0)][None]
                        pred = (pred - origin_grids[b, f:f + 1]) * 0.1
                        gt = (gt - origin_grids[b, f:f + 1]) * 0.1
                        if gt.shape[1] == 0:
                            continue
                        loss_src, loss_tgt = chamfer_l2_mean(pred, gt)
                        dense = dense + ((loss_src + loss_tgt) / 2.) * loss_weight[f, 0]
                dense = dense / (loss_weight.sum() * bs)
            loss_dict["loss.dense_voxel"] = dense * self.dense_loss_weight
        return loss_dict

    # ------------------------------------------------------------------ decode (:662-752)
    def get_point_cloud_prediction(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range,
                                   img_metas=None, batched_origin_points=None):
        bev_preds = pred_dict["next_bev_preds"].float()
        valid_frames = pred_dict["valid_frames"]
        pred_frame_num, inter_num, bs, token_num, num_height_pred = bev_preds.shape
        (origin_grids, batched_origin_points, gt_grids, batched_gt_points, gt_tindex) = self._process_gt_points(
            bev_preds, gt_points, batched_origin_points, valid_frames, start_idx, pred_frame_num, tgt_bev_h, tgt_bev_w,
            tgt_pc_range)
        sigma = self._sigma_volume(bev_preds[:, -1], bs, pred_frame_num, num_height_pred, tgt_bev_h, tgt_bev_w)
        pred_dist = torch.zeros_like(gt_grids[..., 0])
        gt_dist = torch.zeros_like(pred_dist)
        for b in range(bs):
            pred_dist[b], gt_dist[b] = ray_head.decode_ray_depth(sigma[b], origin_grids[b], gt_grids[b], gt_tindex[b],
                                                                 self.ray_grid_step, self.ray_grid_num)
        scale = (tgt_pc_range[3] - tgt_pc_range[0]) / tgt_bev_w
        pred_dist, gt_dist = pred_dist * scale, gt_dist * scale
        pred_pcds = self.get_rendered_pcds(batched_origin_points, batched_gt_points, gt_tindex, gt_dist, pred_dist, tgt_pc_range)
        gt_pcds = self.get_rendered_pcds(batched_origin_points, batched_gt_points, gt_tindex, gt_dist, gt_dist, tgt_pc_range)
        return dict(pred_pcds=pred_pcds, gt_pcds=gt_pcds, origin=batched_origin_points)

    # ------------------------------------------------------------------ evaluation (vidar.py:439-497)
    def evaluate(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas=None,
                 batched_origin_points=None):
        """forward_test's decode and metric loop (vidar.py:439-497) in one batched device pass: the same arguments as
        get_point_cloud_prediction -> the per-sample ret_dict {f"frame.{t + start_idx}": {count, chamfer_distance,
        l1_error, absrel_error}}, equal to evaluate.frame_metrics(get_point_cloud_prediction(...)), with its
        exceptions.  One host copy at the end."""
        out, bs, F = self._evaluate_table(pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range,
                                          img_metas, batched_origin_points)
        return eval_metrics.frame_metrics_host(out, bs, F, start_idx)

    def evaluate_device(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas=None,
                        batched_origin_points=None):
        """Device part of `evaluate`: the [bs * F, 8] float64 table of evaluate.frame_metrics_device (row b * F + t),
        no host sync."""
        return self._evaluate_table(pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                                    batched_origin_points)[0]

    def _evaluate_table(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                        batched_origin_points):
        """get_point_cloud_prediction without its per-(sample, frame) loops: every row of the batch is decoded by one
        arg-max launch over the [bs * Fp] volumes, the clouds are built in place (ray_head.decode_clouds) and scored
        as bs * F clouds plus the trailing segment of the rows in no cloud, whose table row is dropped."""
        bev_preds = pred_dict["next_bev_preds"].float()
        valid_frames = pred_dict["valid_frames"]
        Fp, inter_num, bs, token_num, Z = bev_preds.shape
        (origin_grids, origin, gt_grids, points, gt_tindex) = self._process_gt_points(
            bev_preds, gt_points, batched_origin_points, valid_frames, start_idx, Fp, tgt_bev_h, tgt_bev_w, tgt_pc_range)
        F = origin.shape[1]
        if F < Fp:
            raise RuntimeError("origin must hold one row per frame of sigma")
        dev = bev_preds.device
        M = gt_grids.shape[1]
        sigma = self._sigma_volume(bev_preds[:, -1], bs, Fp, Z, tgt_bev_h, tgt_bev_w).view(bs * Fp, Z, tgt_bev_h,
                                                                                            tgt_bev_w)
        t = gt_tindex.float()
        keep = (t >= 0) & (t < Fp) & (t == t.floor())       # the rows decode_ray_depth decodes
        base = torch.arange(bs, dtype=torch.int32, device=dev)[:, None] * Fp
        frame = torch.where(keep, t.clamp(0, Fp - 1).to(torch.int32) + base, -1).view(-1).contiguous()
        rays = gt_grids.float().contiguous()
        origin_vox = origin_grids.float().contiguous()
        depth, _ = ray_head.ray_argmax(sigma, origin_vox[:, :Fp].reshape(bs * Fp, 3), rays.view(bs * M, 3), frame,
                                       self.ray_grid_num, self.ray_grid_step)
        scale = (tgt_pc_range[3] - tgt_pc_range[0]) / tgt_bev_w
        origin = origin.float().contiguous()
        pred, gt, off = ray_head.decode_clouds(depth.view(bs, M), rays, points.float().contiguous(),
                                               torch.where(keep, t, -1.0).contiguous(), origin_vox, origin, scale,
                                               self.eval_within_grid, tgt_pc_range)
        N = bs * F
        origins = torch.cat([origin.view(N, 3), origin.new_zeros(1, 3)])
        out = eval_metrics.metrics_flat(pred, gt, origins, off, off, M, tgt_pc_range)["out"]
        return out[:N], bs, F


class ViDARRayHeadV1(ViDARRayHead):
    """The loss / decode half of ViDARHeadV1 (dense_heads/vidar_head_v1.py): the head predicts
    `1 + pred_history_frame_num + pred_future_frame_num` head frames, each supervised by the GT of its own source
    frames moved into the target frames' coordinates.

    `loss` with CE + dense (use_dist_loss=False) runs every head frame in one batched pass, in a fixed number of
    library launches and without a host sync: the GT alignment of every (head frame, slot) job is one op
    (`ray_head.align_gt`), the CE term one `ray_ce` over [head frames * bs * frames] volumes, the dense term one
    gumbel decode and one grouped Chamfer op (`ray_head.dense_chamfer_group_loss`, a group per head frame) over the
    (head frame, sample, frame) pairs of non-zero weight only.  The reference computes the auxiliary head frames'
    zero-weight frames and multiplies them by zero; those pairs never reach the sampler or the nearest-neighbour
    search here.  Default Gumbel noise is drawn for the weighted pairs only, so the generator is consumed
    differently from the reference (pass `gumbels` to pin the noise).

    fuse_head_frames = False (or use_dist_loss) selects the reference's per-head-frame loop over
    `ViDARRayHead.loss` with a torch restatement of the alignment (boolean masks, host syncs); tests compare the
    two."""

    def __init__(self, history_queue_length, pred_history_frame_num=0, pred_future_frame_num=0,
                 per_frame_loss_weight=(1.0,), **kwargs):
        super().__init__(**kwargs)
        self.history_queue_length = history_queue_length
        self.pred_history_frame_num = pred_history_frame_num
        self.pred_future_frame_num = pred_future_frame_num
        self.pred_frame_num = 1 + pred_history_frame_num + pred_future_frame_num
        self.per_frame_loss_weight = per_frame_loss_weight
        if len(per_frame_loss_weight) != self.pred_frame_num:
            raise ValueError(f"per_frame_loss_weight needs {self.pred_frame_num} entries, got "
                             f"{len(per_frame_loss_weight)}")
        self.fuse_head_frames = True

    # ------------------------------------------------------------------ GT alignment (:94-148)
    @staticmethod
    def _transforms(img_metas, src_frames, tgt_frames):
        """total_cur2ref[src] @ total_ref2cur[tgt] per job and sample -> CPU float32 [jobs, bs, 4, 4], the
        reference's fp32 CPU matmul."""
        a = torch.from_numpy(np.array([[m["total_cur2ref_lidar_transform"][s] for m in img_metas]
                                       for s in src_frames])).float()
        b = torch.from_numpy(np.array([[m["total_ref2cur_lidar_transform"][t] for m in img_metas]
                                       for t in tgt_frames])).float()
        return torch.matmul(a, b)

    @staticmethod
    def _pack_gt(gt_points, device):
        """Ragged GT list -> [bs, Mmax, Cg] NaN-padded (shapes are host-known: no sync)."""
        return torch.nn.utils.rnn.pad_sequence([p.float() for p in gt_points], batch_first=True,
                                               padding_value=float("nan")).to(device).contiguous()

    @staticmethod
    def _voxel_table(bev_h, bev_w, pillar_num, pc_range):
        """bev_geometry.coords_to_voxel_grids as ((x - lo) * scale) * cells with torch's CUDA arithmetic for a
        tensor divided by a host scalar (a multiply by its fp32 reciprocal)."""
        r = pc_range
        span = [r[3] - r[0], r[4] - r[1], r[5] - r[2]]
        return ([np.float32(r[0]), np.float32(r[1]), np.float32(r[2])]
                + [np.float32(1.0) / np.float32(s) for s in span] + [np.float32(bev_w), np.float32(bev_h),
                                                                     np.float32(pillar_num)])

    def _get_reference_gt_points(self, gt_points, src_frame_idx_list, tgt_frame_idx_list, img_metas):
        """:94-148 -> (batched_gt_points: per sample [n_b, 4] rows (x, y, z, slot), slot-major,
        batched_origin_points [bs, slots, 3]).  One alignment op; the per-sample row counts come back to the
        host once (the list's shapes), instead of a boolean mask per (slot, sample)."""
        dev = gt_points[0].device
        mats = self._transforms(img_metas, src_frame_idx_list, tgt_frame_idx_list)
        _, tindex, pts = ray_head.align_gt(self._pack_gt(gt_points, dev), mats.to(dev), [list(src_frame_idx_list)],
                                           [0.0] * 3 + [1.0] * 3 + [0.0] * 3, with_points=True)
        counts = (tindex >= 0).sum(1).tolist()
        rows = [torch.cat([pts[b, :n], tindex[b, :n, None]], 1) for b, n in enumerate(counts)]
        return rows, mats[:, :, 3, :3].permute(1, 0, 2).contiguous().to(dev)

    def _align_torch(self, gt_points, src_frame_idx_list, tgt_frame_idx_list, img_metas):
        """The reference's statements (boolean mask per slot and sample), the transform written out in the
        alignment kernel's order: x' = ((x T0 + y T1) + z T2) + T3.  The reference of the tests."""
        dev = gt_points[0].device
        mats = self._transforms(img_metas, src_frame_idx_list, tgt_frame_idx_list).to(dev)
        per_b = [[] for _ in gt_points]
        for v, src in enumerate(src_frame_idx_list):
            for b, p in enumerate(gt_points):
                q = p[p[:, -1] == src].float()
                T = mats[v, b]
                xyz = [((q[:, 0] * T[0, a] + q[:, 1] * T[1, a]) + q[:, 2] * T[2, a]) + T[3, a] for a in range(3)]
                per_b[b].append(torch.stack(xyz + [torch.full_like(q[:, 0], float(v))], 1))
        return [torch.cat(r, 0) for r in per_b], mats[:, :, 3, :3].permute(1, 0, 2).contiguous()

    # ------------------------------------------------------------------ loss (:150-219)
    def _frame_plan(self, pred_dict):
        valid_frames = np.array(pred_dict["valid_frames"])
        start_frames = valid_frames + self.history_queue_length - self.pred_history_frame_num
        tgt_frames = valid_frames + self.history_queue_length
        if not pred_dict.get("full_prev_bev_exists", True):
            frame_idx_for_loss = [self.pred_history_frame_num] * self.pred_frame_num
        else:
            frame_idx_for_loss = list(range(self.pred_frame_num))
        return start_frames, tgt_frames, frame_idx_for_loss

    def _head_frame_weight(self, i):
        if i != self.pred_history_frame_num:     # auxiliary head frames supervise their first frame only
            return np.array([[1]] + [[0]] * (len(self.loss_weight) - 1))
        return self.loss_weight

    def loss(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, pred_frame_num,
             img_metas=None, batched_origin_points=None, gumbels=None):
        """ViDARHeadV1.loss: keys 'frame.{idx}.{k}.loss'.  `gumbels`: optional list, one entry per loss index,
        of the `gumbels` dict ViDARRayHead.loss takes for that head frame ({'dense': [bs, frames*R0, K]}); noise of
        zero-weight pairs is not read."""
        if not self.fuse_head_frames or self.use_dist_loss:
            return self._loss_per_head_frame(pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range,
                                             img_metas, gumbels)
        bev_preds = pred_dict["next_bev_preds"]
        V, _, Hf, bs, token_num, Z = bev_preds.shape
        if Hf != self.pred_frame_num or len(gt_points) != bs:
            raise ValueError(f"next_bev_preds [frames, inter, {self.pred_frame_num}, bs, tokens, Z] and bs GT "
                             f"lists expected, got {tuple(bev_preds.shape)} and {len(gt_points)} lists")
        dev = bev_preds.device
        start_frames, tgt_frames, frame_idx_for_loss = self._frame_plan(pred_dict)
        scale = np.zeros(Hf)
        for idx, i in enumerate(frame_idx_for_loss):
            if idx == i:
                scale[i] = self.per_frame_loss_weight[i]
        active = [i for i in range(Hf) if scale[i] != 0]
        # slot v of a head frame is the base loss's frame t = v - start_idx when v is one of its frames
        frames = [f for f in range(start_idx, len(self.loss_weight) - 1) if f < V]
        slot_t = np.full(V, -1)
        for f in frames:
            slot_t[f] = f - start_idx
        # host tables: per (head frame, sample, slot) the CE frame and weight; the weighted dense pairs
        S = Hf * bs
        ray_frame = np.full(S * V, -1)
        ray_w = np.zeros(S * V)
        pairs, pair_w, norms = [], [], np.ones(Hf)      # a head frame without pairs keeps norm 1 and loss 0
        for i in active:
            lw = self._head_frame_weight(i)
            norms[i] = np.float32(float(lw.sum())) * np.float32(bs)
            for b in range(bs):
                s = i * bs + b
                for v in range(V):
                    t = slot_t[v]
                    if t >= 0 and lw[t, 0] != 0:
                        ray_frame[s * V + v] = s * V + t
                        ray_w[s * V + v] = lw[t, 0]
                for t in range(V):
                    if lw[t, 0] != 0:
                        pairs.append((s, t, s * V + t, i))
                        pair_w.append(lw[t, 0])
        jobs = np.full((Hf, V), -1)
        src = np.zeros((Hf, V), dtype=np.int64)
        for i in range(Hf):
            src[i] = start_frames + i if i in active else tgt_frames
            if i in active:
                jobs[i] = src[i]
        mats = self._transforms(img_metas, src.ravel(), np.tile(tgt_frames, Hf))           # [Hf*V, bs, 4, 4]
        nm = mats.numel()
        host = np.concatenate([mats.numpy().ravel(), ray_frame, ray_w, slot_t]).astype(np.float32)
        table = ray_head._pinned_upload(host, np.float32, dev)
        mats_d = table[:nm].view(Hf * V, bs, 4, 4)
        ray_frame_d = table[nm:nm + S * V]
        ray_w_d = table[nm + S * V:nm + 2 * S * V]
        slot_t_d = table[nm + 2 * S * V:]

        # 1. GT of every (head frame, sample), slot-major, in voxel units
        rays, tv, _ = ray_head.align_gt(self._pack_gt(gt_points, dev), mats_d, jobs,
                                        self._voxel_table(tgt_bev_h, tgt_bev_w, Z, tgt_pc_range))
        key = (torch.arange(S, device=dev)[:, None] * V + tv.clamp(min=0).long())
        live = tv >= 0
        frame = torch.where(live, ray_frame_d[key], -1.0).to(torch.int32).view(-1).contiguous()
        w_ray = torch.where(live, ray_w_d[key], 0.0).view(Hf, -1)
        gt_t = torch.where(live, slot_t_d[tv.clamp(min=0).long()], -1.0).contiguous()
        origin = mats_d[:, :, 3, :3].view(Hf, V, bs, 3).permute(0, 2, 1, 3).reshape(S * V, 3)
        origin = bev_geometry.coords_to_voxel_grids(origin, bev_h=tgt_bev_h, bev_w=tgt_bev_w, pillar_num=Z,
                                                    pc_range=tgt_pc_range).contiguous()
        # [frames, inter, Hf, bs, tokens, Z] -> volumes [(i * bs + b) * V + v, Z, Y, X] of the last output
        sigma = (bev_preds[:, -1].float().permute(1, 2, 0, 4, 3).contiguous()
                 .view(S * V, Z, tgt_bev_h, tgt_bev_w))
        step, K = self.ray_grid_step, self.ray_grid_num
        terms = {}
        if self.use_ce_loss:
            ce, valid = ray_head.ray_ce(sigma, origin, rays.view(-1, 3), frame, K, step)
            w = w_ray * valid.view(Hf, -1)
            terms["regularization.loss"] = (ce.view(Hf, -1) * w).sum(1) / torch.clamp(w.sum(1), min=1)
        if self.use_dense_loss:
            dense = sigma.new_zeros(Hf)
            if pairs:
                tab = np.array(pairs, dtype=np.int64)
                P = len(pairs)
                grid = self._dense_grid(tgt_bev_h, tgt_bev_w, Z, dev)
                R0 = grid.shape[0]
                comp = torch.from_numpy(tab[:, 2].astype(np.int32)).pin_memory().to(dev, non_blocking=True)
                noise = self._pair_noise(gumbels, frame_idx_for_loss, tab, bs, R0, dev)
                dist = ray_head.gumbel_distance(sigma, origin, grid.repeat(P, 1),
                                                comp[:, None].expand(P, R0).reshape(-1).contiguous(), K, step, noise)
                dense = ray_head.dense_chamfer_group_loss(
                    dist, grid.repeat(P, 1), origin, rays, gt_t, (tgt_bev_w, tgt_bev_h, Z), tab, pair_w, norms,
                    self.eval_within_grid, tgt_pc_range)
            terms["loss.dense_voxel"] = dense * self.dense_loss_weight
        loss_dict = dict()
        for idx, i in enumerate(frame_idx_for_loss):
            for k, v in terms.items():
                loss_dict[f"frame.{idx}.{k}.loss"] = v[i] * (self.per_frame_loss_weight[i] * (idx == i))
        return loss_dict

    def _pair_noise(self, gumbels, frame_idx_for_loss, tab, bs, R0, device):
        """Gumbel noise [P*R0, K] of the weighted pairs: slices of the per-head-frame noise when given, else drawn
        with the statement F.gumbel_softmax uses."""
        P, K = tab.shape[0], self.ray_grid_num
        if gumbels is None:
            return -torch.empty((P * R0, K), dtype=torch.float32, device=device).exponential_().log()
        loss_idx = {i: idx for idx, i in enumerate(frame_idx_for_loss) if idx == i}
        parts = []
        for s, t, _, i in tab:
            parts.append(gumbels[loss_idx[int(i)]]["dense"][int(s) - int(i) * bs, t * R0:(t + 1) * R0])
        return torch.cat(parts, 0).float().contiguous()

    def _loss_per_head_frame(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                             gumbels):
        """The reference's loop (:167-219): one ViDARRayHead.loss per head frame."""
        bev_preds = pred_dict["next_bev_preds"]
        start_frames, tgt_frames, frame_idx_for_loss = self._frame_plan(pred_dict)
        loss_dict = dict()
        for idx, i in enumerate(frame_idx_for_loss):
            cur_bev_preds = bev_preds[:, :, i, ...].contiguous()
            src_frames = start_frames + i
            cur_gt_points, cur_origin_points = self._align_torch(gt_points, src_frames, tgt_frames, img_metas)
            cur_loss_dict = ViDARRayHead.loss(
                self, dict(next_bev_preds=cur_bev_preds, valid_frames=np.arange(0, len(src_frames))), cur_gt_points,
                start_idx=start_idx, tgt_bev_h=tgt_bev_h, tgt_bev_w=tgt_bev_w, tgt_pc_range=tgt_pc_range,
                pred_frame_num=len(self.loss_weight) - 1, img_metas=img_metas,
                batched_origin_points=cur_origin_points, loss_weight=self._head_frame_weight(i),
                gumbels=gumbels[idx] if gumbels is not None else None)
            cur_frame_loss_weight = self.per_frame_loss_weight[i] * (idx == i)
            for k, v in cur_loss_dict.items():
                loss_dict[f"frame.{idx}.{k}.loss"] = v * cur_frame_loss_weight
        return loss_dict

    # ------------------------------------------------------------------ decode (:221-252)
    def get_point_cloud_prediction(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range,
                                   img_metas=None, batched_origin_points=None):
        """The current head frame's prediction, decoded against its own frames' GT (src == tgt)."""
        cur = dict(pred_dict)
        cur["next_bev_preds"] = pred_dict["next_bev_preds"][:, :, self.pred_history_frame_num, ...].contiguous()
        valid_frames = np.array(pred_dict["valid_frames"])
        frames = valid_frames + self.history_queue_length
        valid_gt_points, cur_origin_points = self._get_reference_gt_points(gt_points, frames, frames, img_metas)
        return ViDARRayHead.get_point_cloud_prediction(self, cur, valid_gt_points, start_idx, tgt_bev_h, tgt_bev_w,
                                                       tgt_pc_range, img_metas=img_metas,
                                                       batched_origin_points=cur_origin_points)

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas=None,
                 batched_origin_points=None):
        """ViDARRayHead.evaluate of the current head frame (`pred_history_frame_num`), equal to
        evaluate.frame_metrics(get_point_cloud_prediction(...)); the GT alignment is one align_gt op."""
        out, bs, F = self._evaluate_table(pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range,
                                          img_metas, batched_origin_points)
        return eval_metrics.frame_metrics_host(out, bs, F, start_idx)

    def evaluate_device(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas=None,
                        batched_origin_points=None):
        """Device part of `evaluate`: [bs * F, 8] float64 (row b * F + t), no host sync."""
        return self._evaluate_table(pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                                    batched_origin_points)[0]

    def _evaluate_table(self, pred_dict, gt_points, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                        batched_origin_points):
        """get_point_cloud_prediction's alignment (src == tgt frames) without the host row counts of
        _get_reference_gt_points: every sample keeps its M aligned rows, padding rows with frame -1, which
        _process_gt_points treats as rows of no frame."""
        cur = dict(pred_dict)
        cur["next_bev_preds"] = pred_dict["next_bev_preds"][:, :, self.pred_history_frame_num, ...].contiguous()
        frames = np.array(pred_dict["valid_frames"]) + self.history_queue_length
        dev = gt_points[0].device
        mats = self._transforms(img_metas, frames, frames)
        mats_d = ray_head._pinned_upload(mats.numpy(), np.float32, dev)
        _, tindex, pts = ray_head.align_gt(self._pack_gt(gt_points, dev), mats_d, [list(frames)],
                                           [0.0] * 3 + [1.0] * 3 + [0.0] * 3, with_points=True)
        rows = [torch.cat([pts[b], tindex[b, :, None]], 1) for b in range(len(gt_points))]
        origin = mats_d[:, :, 3, :3].permute(1, 0, 2).contiguous()
        return ViDARRayHead._evaluate_table(self, cur, rows, start_idx, tgt_bev_h, tgt_bev_w, tgt_pc_range, img_metas,
                                            origin)
