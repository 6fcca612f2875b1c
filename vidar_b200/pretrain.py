"""BASELINE.json configs[3]: one ViDAR-RN101 pre-training step on synthetic data, built around the
hot-path modules of this package, with the intra-sample sharding of SURVEY.md 8e.

This is a HARNESS, not a port of the detector: it composes the reference's step
(projects/mmdet3d_plugin/bevformer/detectors/vidar.py:239-387) from
  * a random-init ResNet-101 (strides 8/16/32; stage 1 frozen, BN in eval mode as in
    vidar_1_8_nusc_3future.py:88-95).  `dcn=True` (`build(device, dcn=True)`) is the reference's caffe-style backbone
    with a DCNv2 (vidar_b200/dcn.py) as conv2 of every block in stages 3-4; the default dcn=False runs torchvision's
    plain convolutions there.  Then a 4-level FPN (cfg :96-106);
  * the BEV encoder: 6 x [TemporalSelfAttention, LN, SpatialCrossAttention, LN, (LatentRendering in
    layer 2), FFN 256-512-256, LN]  (modules/encoder.py:159-253, encoder_v2.py:52-209, cfg :141-190);
  * the future decoder: 3 x [PredictionMSDeformableAttention (self), LN, PredictionMSDeformableAttention
    (cross to the previous BEV), LN, FFN, LN], rolled out for 3 future frames
    (modules/vidar_decoder.py:25-280, dense_heads/vidar_head_base.py:125-173);
  * the per-layer freespace head and the ray losses of ViDARHeadV1 (dense_heads/vidar_head_v1.py:45-92,
    150-219) through `vidar_b200.head.ViDARRayHead.loss`.
History frames run under no_grad like `obtain_history_bev` (bevformer.py:158-236); `CONFIGS` holds the training
regimes of the four nuScenes pre-training configs (the last history frame's encoder with gradient, a random drop
of the history, one sampled supervised future frame, the head's frames), for `build(device, config=name)`.

Sharding over a process group (one sample on all ranks -- the reference has replica DDP only):
  * cameras: each camera's image goes through backbone + FPN on ONE rank; a camera whose
    SpatialCrossAttention units are split over two ranks (vidar_b200.sca.unit_plan) has its features
    broadcast inside its 2-rank group (31.6 MB), gradients reduced back to the owner;
  * SpatialCrossAttention: camera-sharded sampling, reduce-scatter of the partial BEV slots, output_proj on
    the rank's rows, ONE all-gather of the BEV grid per layer (modules/deform_attn.py);
  * LatentRendering: BEV rows / cells sharded (modules/latent_rendering.py);
  * everything else (TSA, FFN, norms, decoder, head, loss) is replicated: every rank computes the same
    values and the same gradients, so only parameters that saw sharded data (backbone, FPN, embeddings of
    the camera features, SCA projections) need their gradients summed -- ONE bucketed all-reduce per step
    (`sharding.allreduce_partial_grads`), the counterpart of the reference's DDP all-reduce
    (apis/mmdet_train.py:72-81).
Data-parallel replicas of that (`build(..., grid=sharding.make_grid(S))`): world / S replicas, each sharding its own
sample over S ranks; `train_step(..., grid=grid)` averages every trainable gradient over the replicas in ONE
bucketed all-reduce over the world (`sharding.allreduce_grid_grads`).
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import bev_geometry, ego_motion as ego, optim, sca, sharding, synthetic
from . import evaluate as eval_metrics
from . import modules as _modules  # noqa: F401  (registers the attention classes)
from . import image_aug
from . import point_pipeline as point_aug
from .grid_mask import GridMask
from .head import ViDARRayHead
from .modules.deform_attn import _linear
from .registry import build_attention
from .sample_loader import SampleLoader, run_image_transforms, run_point_transforms  # noqa: F401

PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
EGO_MASK = (-0.8, -1.5, 0.8, 2.5)                    # the dataset's ego_mask (config :348)
EMBED, BEV_H, BEV_W, HEIGHTS = 256, 200, 200, 16


# ------------------------------------------------------------------------------------------------
# image side
# ------------------------------------------------------------------------------------------------
class ImageBackbone(nn.Module):
    """ResNet-101 C3..C5 (strides 8, 16, 32).  frozen_stages=1 and norm_eval=True (cfg :92-94).

    dcn=True is the reference's backbone (cfg :88-95): style='caffe' -- the stride of the first block of layer2..4 sits
    on its 1x1 conv1, not on the 3x3 conv2 -- and conv2 of every block of layer3 and layer4 (23 + 3 = 26 layers) is a
    DCNv2, `vidar_b200.dcn.ModulatedDeformConv2dPack(planes, planes, 3, padding=1, bias=False)` (stage_with_dcn=(False,
    False, True, True), fallback_on_stride=False).  dcn=False keeps torchvision's pytorch-style plain convolutions."""

    def __init__(self, dcn=False):
        super().__init__()
        import torchvision
        r = torchvision.models.resnet101(weights=None)
        if dcn:
            from .dcn import ModulatedDeformConv2dPack
            for li, layer in enumerate((r.layer2, r.layer3, r.layer4)):
                first = layer[0]
                first.conv1.stride, first.conv2.stride = (2, 2), (1, 1)
                if li > 0:
                    for blk in layer:
                        width = blk.conv2.in_channels
                        blk.conv2 = ModulatedDeformConv2dPack(width, width, 3, stride=1, padding=1, bias=False)
        self.dcn = dcn
        self.stem = nn.Sequential(r.conv1, r.bn1, r.relu, r.maxpool)
        self.layer1, self.layer2, self.layer3, self.layer4 = r.layer1, r.layer2, r.layer3, r.layer4
        for m in (self.stem, self.layer1):
            for p in m.parameters():
                p.requires_grad_(False)

    def train(self, mode=True):
        super().train(mode)
        for m in self.modules():                      # norm_eval
            if isinstance(m, nn.BatchNorm2d):
                m.eval()
        return self

    def forward(self, x):
        with torch.no_grad():
            x = self.layer1(self.stem(x))
        c3 = self.layer2(x)
        c4 = self.layer3(c3)
        c5 = self.layer4(c4)
        return c3, c4, c5


class FPN(nn.Module):
    """mmdet FPN(in=[512,1024,2048], out=256, start_level=0, add_extra_convs='on_output', num_outs=4,
    relu_before_extra_convs=True)  (cfg :96-106)."""

    def __init__(self, in_channels=(512, 1024, 2048), out_channels=EMBED):
        super().__init__()
        self.lateral = nn.ModuleList([nn.Conv2d(c, out_channels, 1) for c in in_channels])
        self.out = nn.ModuleList([nn.Conv2d(out_channels, out_channels, 3, padding=1) for _ in in_channels])
        self.extra = nn.Conv2d(out_channels, out_channels, 3, stride=2, padding=1)

    def forward(self, feats):
        lat = [l(f) for l, f in zip(self.lateral, feats)]
        for i in range(len(lat) - 1, 0, -1):
            lat[i - 1] = lat[i - 1] + F.interpolate(lat[i], size=lat[i - 1].shape[-2:], mode="nearest")
        outs = [o(x) for o, x in zip(self.out, lat)]
        outs.append(self.extra(F.relu(outs[-1])))
        return outs


class _ShareCameraFeatures(torch.autograd.Function):
    """Features of a camera whose SCA units are split over two ranks: broadcast from the rank that ran the
    backbone (`src`: its global rank); the co-owner's gradient is reduced back (all-reduce inside the 2-rank group)."""

    @staticmethod
    def forward(ctx, feat, src, group):
        import torch.distributed as dist
        ctx.group = group
        out = feat.contiguous().clone()
        dist.broadcast(out, src=src, group=group)
        return out

    @staticmethod
    def backward(ctx, g):
        import torch.distributed as dist
        g = g.contiguous().clone()
        dist.all_reduce(g, group=ctx.group)
        return g, None, None


# ------------------------------------------------------------------------------------------------
# BEV side
# ------------------------------------------------------------------------------------------------
class FFN(nn.Module):
    """mmcv FFN(embed 256, feedforward 512, 2 fcs, ReLU, dropout 0.1, residual)  (cfg :163-170)."""

    def __init__(self, dims=EMBED, hidden=2 * EMBED, drop=0.1):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(dims, hidden), nn.Linear(hidden, dims)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return x + self.drop(_linear(self.fc2, self.drop(F.relu(_linear(self.fc1, x)))))


class LearnedPositionalEncoding(nn.Module):
    def __init__(self, rows, cols, num_feats=EMBED // 2):
        super().__init__()
        self.row_embed, self.col_embed = nn.Embedding(rows, num_feats), nn.Embedding(cols, num_feats)

    def forward(self, bs):
        h, w = self.row_embed.num_embeddings, self.col_embed.num_embeddings
        x = self.col_embed.weight[None].expand(h, -1, -1)
        y = self.row_embed.weight[:, None].expand(-1, w, -1)
        return torch.cat([x, y], -1).view(1, h * w, -1).expand(bs, -1, -1)      # [bs, Q, C]


class EncoderLayer(nn.Module):
    """BEVFormerLayerV2 (encoder_v2.py:52-209): self_attn, norm, cross_attn, norm, [latent_render], ffn, norm."""

    def __init__(self, latent_render, bev_hw, grid_step=0.5, num_cams=6):
        super().__init__()
        self.bev_hw = bev_hw
        self.self_attn = build_attention(dict(type="TemporalSelfAttention", embed_dims=EMBED, num_levels=1))
        self.cross_attn = build_attention(dict(
            type="SpatialCrossAttention", pc_range=PC_RANGE, embed_dims=EMBED, num_cams=num_cams,
            deformable_attention=dict(type="MSDeformableAttention3D", embed_dims=EMBED, num_points=8, num_levels=4)))
        self.norms = nn.ModuleList([nn.LayerNorm(EMBED) for _ in range(3)])
        self.ffn = FFN()
        self.latent_render = build_attention(dict(
            type="LatentRendering", embed_dims=EMBED, num_pred_fcs=0, pred_height=HEIGHTS, grid_num=256,
            grid_step=grid_step, reduction=16, act="sigmoid")) if latent_render else None

    def forward(self, query, feats, bev_pos, ref_2d, prev_bev, shapes, lsi, ref_cam, bev_mask, bev_shapes, bev_lsi):
        query = self.self_attn(query, prev_bev, prev_bev, None, query_pos=bev_pos, reference_points=ref_2d,
                               spatial_shapes=bev_shapes, level_start_index=bev_lsi)
        query = self.norms[0](query)
        query = self.cross_attn(query, feats, feats, None, reference_points_cam=ref_cam, bev_mask=bev_mask,
                                spatial_shapes=shapes, level_start_index=lsi)
        query = self.norms[1](query)
        if self.latent_render is not None:
            bs, n, c = query.shape
            query = self.latent_render(query.view(bs, self.bev_hw[0], self.bev_hw[1], c)).view(bs, n, c)
        return self.norms[2](self.ffn(query))

    def forward_rows(self, x_full, feats, bev_pos, ref_2d, prev_bev, shapes, lsi, ref_cam, bev_mask, bev_shapes, bev_lsi,
                     group, last):
        """The same layer with the BEV rows sharded over `group` (SURVEY.md 8e: TSA / FFN / norms on the rank's rows,
        value replicated; bs = 1).  `x_full` [1, Q, C] is the replicated layer input; every row-wise stage runs on
        this rank's block only; the full grid is assembled twice: after the first norm (SpatialCrossAttention needs
        every pillar's offsets for its cameras) and at the end (the next layer's TSA samples the whole BEV).  Both
        all-gathers feed sharded consumers, so their backward is a reduce-scatter of partial gradients -- except the
        last layer's, whose consumers (decoder, head) are replicated."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        bs, Q, C = x_full.shape
        lo, hi = sharding.row_range(Q, rank, world)
        q = self.self_attn(x_full[:, lo:hi], prev_bev, prev_bev, None, query_pos=bev_pos[:, lo:hi],
                           reference_points=ref_2d[:, lo:hi], spatial_shapes=bev_shapes, level_start_index=bev_lsi,
                           row_range=(lo, hi))
        q = self.norms[0](q)                                                       # [1, rows, C]
        q_full = sharding.all_gather_rows(q[0], Q, group, grad="sum")[None]
        q = self.cross_attn(q_full, feats, feats, q, reference_points_cam=ref_cam, bev_mask=bev_mask,
                            spatial_shapes=shapes, level_start_index=lsi, rows_out=True, summed_query_grad=True)
        q = self.norms[1](q)                                                       # [rows, C]
        if self.latent_render is not None:
            q = self.latent_render.forward_rows(q, bs, self.bev_hw[0], self.bev_hw[1])
        q = self.norms[2](self.ffn(q))
        return sharding.all_gather_rows(q, Q, group, grad="slice" if last else "sum")[None]


class DecoderLayer(nn.Module):
    """PredictionTransformerLayer (vidar_decoder.py:104-280) without latent rendering (the shipped
    pre-train configs delete it from every decoder layer, SURVEY.md 3.3)."""

    def __init__(self):
        super().__init__()
        self.self_attn = build_attention(dict(type="PredictionMSDeformableAttention", embed_dims=EMBED, num_levels=1))
        self.cross_attn = build_attention(dict(type="PredictionMSDeformableAttention", embed_dims=EMBED, num_levels=1))
        self.norms = nn.ModuleList([nn.LayerNorm(EMBED) for _ in range(3)])
        self.ffn = FFN()

    def forward(self, query, prev_feats, bev_pos, tgt_points, ref_points, bev_shapes, bev_lsi):
        query = self.self_attn(query, None, None, None, query_pos=bev_pos, reference_points=tgt_points,
                               spatial_shapes=bev_shapes, level_start_index=bev_lsi)
        query = self.norms[0](query)
        query = self.cross_attn(query, prev_feats, prev_feats, None, query_pos=bev_pos, reference_points=ref_points,
                                spatial_shapes=bev_shapes, level_start_index=bev_lsi)
        query = self.norms[1](query)
        return self.norms[2](self.ffn(query))

    def forward_rows(self, x_full, prev_feats, bev_pos, tgt_points, ref_points, bev_shapes, bev_lsi, group):
        """The same layer on this rank's block of BEV rows (bs = 1): both attentions sample replicated values (the full
        query grid / the previous BEV) for the rank's rows, norms and FFN are row-wise, ONE all-gather returns the grid
        (backward: reduce-scatter -- `prev_feats` and `bev_pos` must come through `sharding.sum_grad`, replicated
        consumers of the result through `sharding.replicated_view`)."""
        import torch.distributed as dist
        Q = x_full.shape[1]
        lo, hi = sharding.row_range(Q, dist.get_rank(group), dist.get_world_size(group))
        pos = bev_pos[:, lo:hi]
        q = self.self_attn(x_full[:, lo:hi], None, x_full, None, query_pos=pos, reference_points=tgt_points[:, lo:hi],
                           spatial_shapes=bev_shapes, level_start_index=bev_lsi)
        q = self.norms[0](q)
        q = self.cross_attn(q, prev_feats, prev_feats, None, query_pos=pos, reference_points=ref_points[:, lo:hi],
                            spatial_shapes=bev_shapes, level_start_index=bev_lsi)
        q = self.norms[2](self.ffn(self.norms[1](q)))
        return sharding.all_gather_rows(q[0], Q, group, grad="sum")[None]


def run_decoder(layers, query, prev, bev_pos, ref, bev_shapes, bev_lsi, group=None, ref_points=None):
    """The future-BEV decoder stack -> (outputs of every layer stacked [inter, bs, Q, C] for the head, last output for
    the next future frame).  `ref` is the self-attention's reference points (tgt_points), `ref_points` the
    cross-attention's in the previous frame (default: `ref`).  `group`: row-sharded layers
    (`DecoderLayer.forward_rows`); the stacked outputs are then (like the returned last output) views for replicated
    consumers (`sharding.replicated_view`)."""
    inter = []
    ref_points = ref if ref_points is None else ref_points
    if group is None:
        for layer in layers:
            query = layer(query, prev, bev_pos, ref, ref_points, bev_shapes, bev_lsi)
            inter.append(query)
        return torch.stack(inter), inter[-1]
    query, prev, bev_pos = (sharding.sum_grad(t, group) for t in (query, prev, bev_pos))
    for layer in layers:
        query = layer.forward_rows(query, prev, bev_pos, ref, ref_points, bev_shapes, bev_lsi, group)
        inter.append(sharding.replicated_view(query, group))
    # the caller's use of the last output (next frame's `prev`, which passes through sum_grad again) is replicated too
    return torch.stack(inter), inter[-1]


class SyntheticViDAR(nn.Module):
    """The pre-training graph of ViDAR-RN101 (3 history frames, 3 future frames, 5 predicted head frames).

    `backbone_autocast` = torch.float16 or torch.bfloat16 runs the backbone and FPN of `extract_feat` under
    torch.autocast("cuda", dtype) and casts the FPN outputs to fp32 before the camera and level embeddings: what the
    reference's `auto_fp16` on `extract_feat` and the `force_fp32` ops after it amount to in its fp16 mode.  The
    default None runs everything in fp32.  The setting holds no state (the state_dict does not change).

    `grid_mask=True` adds the image augmentation of every ViDAR config (use_grid_mask=True with vidar.py:45-53's
    `GridMask(use_h=True, use_w=True, rotate=1, offset=False, ratio=0.5, mode=1, prob=0.7)`, `vidar_b200.grid_mask`):
    in training mode the current frame's images are masked before the backbone (vidar.py:139-140).  The history
    frames go through it in eval mode, as `obtain_history_bev` runs them: one prob-gate draw, no mask.  The draws come
    from numpy's global generator, so under a process group every rank must seed numpy with the same value -- as the
    reference's training script does (mmdet's init_random_seed broadcasts rank 0's seed, set_random_seed seeds numpy
    on every rank) -- and every rank draws once per call, also a rank whose backbone runs no camera; then each rank
    masks its own cameras with the same mask.  The default False leaves the graph as it was.

    `image_pipeline=True` runs the pre-training config's image transforms (vidar_1_8_nusc_3future.py:303-314,
    `vidar_b200.image_aug.config_pipeline`, held in `self.image_transforms`) on every history and current frame, in
    the dataset's order (oldest first; the first frame draws the crop / resize / flip and the later ones reuse it
    through `aug_param`): forward_train then takes uint8 BGR frames img [1, T, cams, H, W, 3] with `cam2img` and
    `lidar2cam` [1, cams, 4, 4] instead of lidar2img (`synthetic_sample(..., raw_images=True)`), and each frame's
    `img_metas` (lidar2img, img_shape = the padded shape) come from its transforms.  The host draws of all frames
    come first, as the dataloader makes them before the step; then each frame's images go through
    `apply_multiview` before the backbone (and GridMask, when on).  bs must be 1 (samples_per_gpu=1).  Under a
    process group every rank draws for all cameras -- numpy and `random` seeded alike on every rank -- and processes
    only its backbone cameras.  The default False leaves the graph as it was.

    `point_pipeline=True` builds gt_points from raw LiDAR frames on the device (`vidar_b200.point_pipeline`):
    forward_train / forward_test then take `point_infos`, one results dict per GT frame in queue order (the current
    frame, then the future ones; `synthetic_sample(..., raw_points=True)`), and ignore their gt_points argument.
    Training runs the train pipeline's point transforms (vidar_1_8_nusc_3future.py:279-305) on every GT frame first,
    in queue order, the test path LoadPointsFromFile only (:319-324); then `gather_gt_points` with the dataset's
    ego mask makes the padded [1, R, 5] gt_points with no host sync.  The default False leaves the graph as it was.

    Training regime (the options that tell the nuScenes pre-training configs apart; `CONFIGS` holds each config's
    values, and the defaults are the graph above):
      * `backward_history_frames` (0 or 1, the configs' backwarded_prev_frame_num): the last history frame's encoder
        runs with gradient in training, its backbone and FPN under no_grad (bevformer.py:191-215);
      * `drop_prev_rate` / `drop_prev_end_idx` (random_drop_prev_*, vidar.py:268-281; the start index is 1): with
        probability `drop_prev_rate` a drop index k = randint(1, end) cuts the frozen history chain -- frame i < k's BEV
        is discarded (bevformer.py:184-185), so those frames are not computed at all;
      * `supervise_all_future=False`: one future frame, drawn by np.random.choice, is supervised; the other roll-outs
        run under no_grad (vidar.py:333-357);
      * `head_history_frames` / `head_future_frames` / `per_frame_loss_weight`: the head's predicted frames per BEV
        feature (ViDARHeadV1's pred_history_frame_num / pred_future_frame_num / per_frame_loss_weight); the
        defaults are `history_frames`, 1 and (0.1, 0.1, 0.1, 1.0, 1.0);
      * `frame_loss_weight` (the head's loss_weight, e.g. ((1,), (0,))): when given, the loss weighs frames as
        ViDARHeadV1.loss does -- the current head frame by these weights, every other head frame on the current
        frame only, each head frame's losses times its `per_frame_loss_weight`.  None keeps the harness's weighting;
      * `latent_grid_step`: LatentRendering's grid_step;
      * `future_frames=0`: no decoder is built (the reference deletes it, vidar.py:109-115); the head keeps
        max(decoder_layers, 1) prediction layers and supervises the current frame;
      * `point_voxel_size`: the point pipeline's voxel sampler size in metres;
      * `reference_draws`: forward_train draws from numpy's global generator as the reference's does, before any
        other draw of the step: A1's rand() (random_drop_image_rate is 0 in every config, so it only consumes the
        draw), A2's rand() and randint, then the supervised future frame.  None (the default) draws only when a
        drop rate or `supervise_all_future=False` needs it.  Under a process group every rank of a shard group must
        seed numpy alike (as for GridMask) so that they draw the same drop index and future frame.

    `openscene=True` selects the OpenScene configs' pipelines (vidar_OpenScene_*_3future.py:274-312) wherever
    `image_pipeline` / `point_pipeline` are on: the nuPlan .pcd point loaders with sweeps_num=0 and the voxel sampler
    at 1 m (`point_pipeline.config_openscene_train_pipeline`; `point_voxel_size` is not read), gt_points of 6 columns,
    and photometric distortion, normalisation, the rescale by 2/3 and padding on the images
    (`image_aug.config_openscene_pipeline`): no crop, each frame's `lidar2img` is the dataset's scaled by 2/3 (the
    in-step pipeline forms it as cam2img @ lidar2cam, as `NuPlanViDARDatasetTemplate.get_data_info` does).  The test
    chains (`test_image_transforms`, `point_transforms[1]`) are the OpenScene test pipeline's.  It holds no state.

    `ego_motion=True` aligns the graph to a moving ego vehicle as the nuScenes configs do (rotate_prev_bev, use_shift,
    use_can_bus; `vidar_b200.ego_motion`).  Each image frame's metas then carry union2one's pose fields
    (`ego_motion.queue_metas`: a `SampleLoader` sample has them, the tensor path takes them as `pose_metas`), and:
      * the encoder embeds the frame's own can_bus, drops the previous BEV where prev_bev_exists is False, shifts the
        first half of TSA's hybrid reference points by the ego translation and rotates the previous BEV by the yaw
        change, straight into TSA's value (`ego_motion.rotate_stack`);
      * TSA's value follows BEVFormerEncoder / CustomBEVFormerEncoder (encoder.py:210-243): [aligned previous BEV,
        the initial query] from the first layer on, restacked with the LatentRendering layer's output after it
        (without a previous BEV the value is the layer input twice, as TSA builds it);
      * each future roll-out's cross-attention samples the previous frame at the target grid moved into its
        coordinates (`_align_bev_coordnates`), and `future_can_bus_mlp` is the head's Linear(4, 128), ReLU,
        Linear(128, 256), ReLU, LayerNorm over future_can_bus[k][:, (0, 1, 2, 17)].
    The default False keeps the graph, the state_dict and the draws as they were: the can_bus is the one passed in
    (zeros by default) for every frame, nothing is shifted or rotated, and TSA's value is [previous BEV or layer
    input, layer input] at every layer.  The row-sharded encoder does not support it."""

    def __init__(self, num_cams=6, encoder_layers=6, decoder_layers=3, future_frames=3, history_frames=3,
                 latent_layer=2, bev_hw=(BEV_H, BEV_W), ray_grid_num=512, dcn=False, backbone_autocast=None,
                 grid_mask=False, image_pipeline=False, point_pipeline=False, backward_history_frames=0,
                 drop_prev_rate=0.0, drop_prev_end_idx=None, supervise_all_future=True, head_history_frames=None,
                 head_future_frames=1, per_frame_loss_weight=None, frame_loss_weight=None, latent_grid_step=0.5,
                 point_voxel_size=1.0, reference_draws=None, ego_motion=False, openscene=False):
        super().__init__()
        self.openscene = bool(openscene)
        self.ego_motion = bool(ego_motion)
        if backward_history_frames not in (0, 1):
            raise ValueError(f"backward_history_frames must be 0 or 1 (got {backward_history_frames})")
        if future_frames < 0 or decoder_layers < 0 or (future_frames > 0 and decoder_layers == 0):
            raise ValueError(f"future_frames={future_frames} needs decoder_layers >= 1 (got {decoder_layers})")
        if not 0.0 <= drop_prev_rate <= 1.0:
            raise ValueError(f"drop_prev_rate must lie in [0, 1] (got {drop_prev_rate})")
        self.backward_history_frames = backward_history_frames
        self.drop_prev_rate, self.drop_prev_start_idx, self.drop_prev_end_idx = drop_prev_rate, 1, drop_prev_end_idx
        self.supervise_all_future = supervise_all_future
        self.reference_draws = (bool(reference_draws) if reference_draws is not None
                                else drop_prev_rate > 0 or not supervise_all_future)
        if not self.reference_draws and (drop_prev_rate > 0 or not supervise_all_future):
            raise ValueError("drop_prev_rate > 0 and supervise_all_future=False draw from numpy: reference_draws=False "
                             "cannot hold them")
        self.head_history_frames = history_frames if head_history_frames is None else head_history_frames
        self.head_future_frames = head_future_frames
        if not point_pipeline:
            self.point_transforms = None
        elif openscene:
            self.point_transforms = (point_aug.config_openscene_train_pipeline(PC_RANGE),
                                     point_aug.config_openscene_test_pipeline())
        else:
            self.point_transforms = (point_aug.config_train_pipeline(PC_RANGE, (point_voxel_size,) * 3),
                                     point_aug.config_test_pipeline())
        self.image_transforms = ((image_aug.config_openscene_pipeline() if openscene else image_aug.config_pipeline())
                                 if image_pipeline else None)
        self.test_image_transforms = (image_aug.config_openscene_test_pipeline() if openscene
                                      else image_aug.config_test_pipeline())
        if backbone_autocast not in (None, torch.float16, torch.bfloat16):
            raise ValueError(f"backbone_autocast must be None, torch.float16 or torch.bfloat16 (got {backbone_autocast})")
        self.backbone_autocast = backbone_autocast
        self.grid_mask = GridMask(True, True, rotate=1, offset=False, ratio=0.5, mode=1, prob=0.7) if grid_mask else None
        self.num_cams, self.future_frames, self.history_frames = num_cams, future_frames, history_frames
        self.bev_h, self.bev_w = bev_hw
        BEV_H, BEV_W = bev_hw          # noqa: N806  (shadows the module defaults below)
        self.backbone, self.neck = ImageBackbone(dcn=dcn), FPN()
        self.bev_embedding = nn.Embedding(BEV_H * BEV_W, EMBED)
        self.positional_encoding = LearnedPositionalEncoding(BEV_H, BEV_W)
        self.cams_embeds = nn.Parameter(torch.randn(num_cams, EMBED) * 0.02)
        self.level_embeds = nn.Parameter(torch.randn(4, EMBED) * 0.02)
        self.can_bus_mlp = nn.Sequential(nn.Linear(18, EMBED // 2), nn.ReLU(inplace=True), nn.Linear(EMBED // 2, EMBED),
                                         nn.ReLU(inplace=True), nn.LayerNorm(EMBED))
        self.encoder = nn.ModuleList([EncoderLayer(i == latent_layer, bev_hw, latent_grid_step, num_cams)
                                      for i in range(encoder_layers)])
        # future head (ViDARHeadV1); with no future frame the reference deletes the decoder and its embeddings
        self.future_bev_embedding = self.future_positional_encoding = None
        self.prev_frame_embedding = self.future_can_bus_mlp = None
        if future_frames > 0:
            self.future_bev_embedding = nn.Embedding(BEV_H * BEV_W, EMBED)
            self.future_positional_encoding = LearnedPositionalEncoding(BEV_H, BEV_W)
            self.prev_frame_embedding = nn.Parameter(torch.randn(1, EMBED))
            self.future_can_bus_mlp = nn.Sequential(nn.Linear(len(ego.CAN_BUS_DIMS) if self.ego_motion else 18, EMBED // 2),
                                                    nn.ReLU(inplace=True),
                                                    nn.Linear(EMBED // 2, EMBED), nn.ReLU(inplace=True),
                                                    nn.LayerNorm(EMBED))
        self.decoder = nn.ModuleList([DecoderLayer() for _ in range(decoder_layers if future_frames > 0 else 0)])
        # head frames per BEV feature: 3 history + current + 1 future by default (cfg :31-33)
        self.pred_frame_num = 1 + self.head_history_frames + head_future_frames
        self.bev_pred_head = nn.ModuleList([nn.Linear(EMBED, self.pred_frame_num * HEIGHTS)
                                            for _ in range(max(decoder_layers, 1))])
        self.frame_loss_weight = None if frame_loss_weight is None else np.array(frame_loss_weight, np.float64)
        if self.frame_loss_weight is not None and self.frame_loss_weight.shape != (future_frames + 2, 1):
            raise ValueError(f"frame_loss_weight: one [w] per frame 0 .. future_frames and a last ignored one "
                             f"({future_frames + 2} rows), got {frame_loss_weight}")
        self.ray_head = ViDARRayHead(ray_grid_num=ray_grid_num, ray_grid_step=1.0, use_ce_loss=True, use_dist_loss=False,
                                     use_dense_loss=True, loss_weight=[[1.0]] * (1 + future_frames))
        if per_frame_loss_weight is None:
            self.per_frame_loss_weight = (0.1, 0.1, 0.1, 1.0, 1.0)
        else:
            self.per_frame_loss_weight = tuple(float(w) for w in per_frame_loss_weight)
            if len(self.per_frame_loss_weight) != self.pred_frame_num:
                raise ValueError(f"per_frame_loss_weight: {self.pred_frame_num} head frames, got {per_frame_loss_weight}")
        self.timings = None
        self.set_process_group(None)

    # ---- sharding ------------------------------------------------------------------------------
    def set_process_group(self, group, row_sharded=False):
        """Shard one sample over `group`: cameras (backbone, SpatialCrossAttention), cells (LatentRendering).
        `row_sharded=True` additionally runs every row-wise stage of the encoder (TSA, norms, FFN) on the rank's
        block of BEV rows (`EncoderLayer.forward_rows`; bs = 1, rows divisible by the group size).

        Stores the layout the graph reads: `shard_size` / `shard_rank` (1 / 0 without a group), this rank's backbone
        and SpatialCrossAttention cameras (`my_backbone_cams`, `my_sca_cams`: all of them on one rank), and the
        groups and owners of the cameras shared by two ranks (`cam_groups`, `cam_src`: empty on one rank).
        `__init__` sets the layout of no group."""
        import torch.distributed as dist
        if row_sharded and self.ego_motion:
            raise ValueError("set_process_group: the row-sharded encoder does not support ego_motion=True")
        world = dist.get_world_size(group) if group is not None else 1
        rank = dist.get_rank(group) if group is not None else 0
        self.process_group, self.shard_size, self.shard_rank = group, world, rank
        self.row_sharded = bool(row_sharded) and world > 1
        owner = {c: r[0] for c, r in sca.camera_ranks(world, self.num_cams).items()}
        self.my_backbone_cams = [c for c, o in owner.items() if o == rank]
        self.my_sca_cams = sca.plan_cameras(sca.unit_plan(world, rank, self.num_cams))
        self.cam_groups = sca.camera_groups(world, self.num_cams, rank, group) if world > 1 else {}
        # the broadcast of a shared camera's features names its owner by global rank (`group` may be a sub-group)
        self.cam_src = {c: dist.get_global_rank(group, o) for c, o in owner.items()} if world > 1 else {}
        for layer in self.encoder:
            layer.cross_attn.set_process_group(group if world > 1 else None)
            if layer.latent_render is not None:
                layer.latent_render.process_group = group if world > 1 else None
        if world > 1:      # parameters that only see this rank's cameras
            for m in (self.backbone, self.neck):
                sharding.mark_partial(m)
            self.cams_embeds.vidar_partial_grad = True
            self.level_embeds.vidar_partial_grad = True
        for layer in self.encoder:      # row-wise stages see only this rank's rows: partial parameter gradients
            for m in (layer.self_attn, layer.norms, layer.ffn):
                for p_ in m.parameters():
                    p_.vidar_partial_grad = self.row_sharded
        for p_ in self.decoder.parameters():
            p_.vidar_partial_grad = self.row_sharded
        return self

    def _mark(self, name):
        if self.timings is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.timings.append((name, e))

    def backbone_cams(self):
        """The cameras whose images this rank's backbone runs (all of them without a process group)."""
        return list(self.my_backbone_cams)

    # ---- image features of one frame -> [cams, K, bs, C] (only this rank's SCA cameras are filled) ----
    def extract_feat(self, img, draw=None, cams_only=False):
        """img [bs, cams, 3, H, W] -> (feat_flatten [cams, K, bs, C], spatial_shapes, level_start_index).  `draw`: a
        GridMask draw (`self.grid_mask.sample`) applied to the images before the backbone.  `cams_only`: img holds
        this rank's backbone cameras only, float32 [len(backbone_cams()), 3, H, W] (bs 1; a `SampleLoader` frame or
        the output of the image pipeline), and goes to the backbone as it is."""
        mine = self.my_backbone_cams
        if cams_only and (img.dim() != 4 or img.shape[0] != len(mine)):
            raise ValueError(f"extract_feat: a frame of this rank's {len(mine)} backbone cameras is "
                             f"[{len(mine)}, 3, H, W] (got {tuple(img.shape)})")
        bs = 1 if cams_only else img.shape[0]
        per_cam = {}
        if mine:
            x = img if cams_only else img[:, mine].reshape(bs * len(mine), *img.shape[2:])
            if draw is not None:
                x = self.grid_mask.masked(x, draw)
            if self.backbone_autocast is None:
                outs = self.neck(self.backbone(x))
            else:
                with torch.autocast("cuda", dtype=self.backbone_autocast):
                    outs = self.neck(self.backbone(x))
                outs = [f.float() for f in outs]
            for i, c in enumerate(mine):
                lv = []
                for lvl, f in enumerate(outs):
                    f = f.view(bs, len(mine), *f.shape[1:])[:, i]                       # [bs, C, h, w]
                    f = f.flatten(2).permute(2, 0, 1)                                    # [hw, bs, C]
                    lv.append(f + self.cams_embeds[c][None, None] + self.level_embeds[lvl][None, None])   # transformer.py:166-172
                per_cam[c] = torch.cat(lv, 0)                                            # [K, bs, C]
            shapes = [tuple(f.shape[-2:]) for f in outs]
        else:
            h, w = img.shape[-2:]
            shapes = [(math.ceil(h / s), math.ceil(w / s)) for s in (8, 16, 32, 64)]
        K = sum(h * w for h, w in shapes)
        feats = img.new_zeros((self.num_cams, K, bs, EMBED))
        pieces = []
        for c in range(self.num_cams):
            f = per_cam.get(c)
            if c in self.cam_groups:                                                      # shared camera
                if f is None:
                    f = img.new_zeros((K, bs, EMBED)).requires_grad_(torch.is_grad_enabled())
                f = _ShareCameraFeatures.apply(f, self.cam_src[c], self.cam_groups[c])
            pieces.append(f if f is not None and c in self.my_sca_cams else feats[c])
        feats = torch.stack(pieces, 0)
        spatial_shapes = torch.tensor(shapes, dtype=torch.int64, device=img.device)
        lsi = torch.cat([spatial_shapes.new_zeros(1), (spatial_shapes[:, 0] * spatial_shapes[:, 1]).cumsum(0)[:-1]])
        return feats, spatial_shapes, lsi

    def _bev_grid(self, bs, device, pillars=False):
        """The BEV grid's constants, built on every call -> (ref_3d [bs, 4, Q, 3], the encoder's pillar points, or
        None without `pillars`; ref_2d [bs, Q, 1, 2]; bev_shapes [[bev_h, bev_w]]; bev_lsi [0])."""
        H, W = self.bev_h, self.bev_w          # noqa: N806
        ref_3d = (bev_geometry.get_reference_points(H, W, PC_RANGE[5] - PC_RANGE[2], 4, dim="3d", bs=bs, device=device)
                  if pillars else None)
        ref_2d = bev_geometry.get_reference_points(H, W, dim="2d", bs=bs, device=device)
        return ref_3d, ref_2d, torch.tensor([[H, W]], device=device), torch.tensor([0], device=device)

    # ---- BEV encoder (transformer.py:102-193 + encoder.py:159-253) ----
    def encode(self, feats, spatial_shapes, lsi, img_metas, can_bus, prev_bev):
        """One frame's BEV.  With `ego_motion` (transformer.py:114-157, encoder.py:196-243), `can_bus` is not read:
        the frame's own comes from img_metas, a scene start drops `prev_bev`, and a previous BEV is aligned -- the
        first half of TSA's hybrid reference points shifted by the ego translation, TSA's value [rotated previous
        BEV, initial query], restacked after the LatentRendering layer.  The host values (can_bus, shift) are
        uploaded pinned, without blocking."""
        bs = feats.shape[2]
        dev = feats.device
        Q = self.bev_h * self.bev_w
        shift = None
        if self.ego_motion:
            ego.require_metas(img_metas)
            if not img_metas[0]["prev_bev_exists"]:                              # bevformer.py:177, vidar.py:280
                prev_bev = None
            host = np.concatenate([np.array([m["can_bus"] for m in img_metas], np.float64),
                                   ego.bev_shift(img_metas, self.bev_h, self.bev_w)], 1)
            host = ego.upload(host, dev, self.bev_embedding.weight.dtype)        # [bs, 18 + 2]: can_bus, shift x / y
            can_bus, shift = host[:, :18], host[:, 18:]
        bev_pos = self.positional_encoding(bs)
        query = self.bev_embedding.weight[None].expand(bs, -1, -1) + self.can_bus_mlp(can_bus)[:, None]
        ref_3d, ref_2d, bev_shapes, bev_lsi = self._bev_grid(bs, dev, pillars=True)
        ref_cam, bev_mask = bev_geometry.point_sampling(ref_3d, PC_RANGE, img_metas)
        first, value = ref_2d, None
        if shift is not None and prev_bev is not None:
            first = ref_2d + shift[:, None, None, :]
            rows = ego.rotation_rows([m["can_bus"][-1] for m in img_metas], self.bev_h, self.bev_w, dev)
            value = ego.rotate_stack(prev_bev, query, rows)                      # [bs * 2, Q, C]
        hybrid = torch.stack([first, ref_2d], 1).reshape(bs * 2, Q, 1, 2)
        if self.row_sharded:
            if bs != 1 or Q % self.shard_size != 0:
                raise RuntimeError(f"row-sharded encoder: needs bs == 1 and BEV rows ({Q}) divisible by the group size "
                                   f"({self.shard_size})")
            # replicated tensors consumed by sharded stages: their gradients are per-rank partial sums
            query = sharding.sum_grad(query, self.process_group)
            bev_pos = sharding.sum_grad(bev_pos, self.process_group)
        for i, layer in enumerate(self.encoder):
            pv = value if value is not None else torch.stack(
                [prev_bev if prev_bev is not None else query, query], 1).reshape(bs * 2, Q, EMBED)
            if self.row_sharded:
                query = layer.forward_rows(query, feats, bev_pos, hybrid, pv, spatial_shapes, lsi, ref_cam, bev_mask,
                                           bev_shapes, bev_lsi, self.process_group, last=i == len(self.encoder) - 1)
            else:
                query = layer(query, feats, bev_pos, hybrid, pv, spatial_shapes, lsi, ref_cam, bev_mask, bev_shapes, bev_lsi)
            if value is not None and layer.latent_render is not None:            # encoder.py:238-243
                value = torch.stack([value.view(bs, 2, Q, EMBED)[:, 0], query], 1).reshape(bs * 2, Q, EMBED)
        return query

    # ---- future decoder (vidar_head_base.py:125-173) ----
    def decode_future(self, prev_bev_input, future_can_bus, ref_points=None):
        """One future roll-out.  With `ego_motion`: `future_can_bus` [bs, 4] is the target frame's future_can_bus at
        the head's can_bus_dims and `ref_points` [bs, Q, 1, 2] the target grid in the previous frame
        (`ego_motion.future_grids`), the cross-attention's reference points; the self-attention keeps the target
        grid."""
        if not len(self.decoder):
            raise RuntimeError("decode_future: the model was built with future_frames=0 and has no future decoder")
        bs = prev_bev_input.shape[0]
        bev_pos = self.future_positional_encoding(bs)
        query = self.future_bev_embedding.weight[None] + self.future_can_bus_mlp(future_can_bus)[:, None]
        prev = (prev_bev_input + self.prev_frame_embedding[None, :, None, :]).view(bs, -1, EMBED)
        _, ref, bev_shapes, bev_lsi = self._bev_grid(bs, prev_bev_input.device)      # ref: identity ego motion
        if self.row_sharded and (bs != 1 or query.shape[1] % self.shard_size != 0):
            raise RuntimeError("row-sharded decoder: needs bs == 1 and BEV rows divisible by the group size")
        # -> ([inter, bs, Q, C] for the head, the last layer's output for the next future frame)
        return run_decoder(self.decoder, query, prev, bev_pos, ref, bev_shapes, bev_lsi,
                           self.process_group if self.row_sharded else None, ref_points=ref_points)

    def forward_head(self, next_bev_feats):
        """vidar_head_v1.py:64-92: [frames, inter, bs, Q, C] -> [frames, inter, pred_frame, bs, Q, heights]."""
        hist = self.head_history_frames
        preds = []
        for lvl in range(next_bev_feats.shape[1]):
            p = self.bev_pred_head[lvl](next_bev_feats[:, lvl])
            p = p.view(*p.shape[:-1], HEIGHTS, self.pred_frame_num)
            base = p[..., hist][..., None]
            p = torch.cat([p[..., :hist] + base, base, p[..., hist + 1:] + base], -1)
            preds.append(p.permute(0, 4, 1, 2, 3).contiguous())
        return torch.stack(preds, 1)

    # ---- history BEV, current BEV, future roll-outs, head (vidar.py:239-387 and :392-437) ----
    def frame_transforms(self, img, cam2img, lidar2cam):
        """The host half of the image pipeline for every frame of img uint8 [1, T, cams, H, W, 3], in the dataset's
        order -> [results] per frame (`apply_multiview` input and img_metas)."""
        if img.dim() != 6 or img.shape[0] != 1 or img.dtype != torch.uint8 or img.shape[-1] != 3:
            raise ValueError(f"image_pipeline: img must be uint8 [1, T, cams, H, W, 3] (bs 1, samples_per_gpu=1; got "
                             f"{img.dtype} {tuple(img.shape)})")
        if cam2img is None or lidar2cam is None:
            raise ValueError("image_pipeline: forward needs cam2img and lidar2cam")
        frames = []
        for t in range(img.shape[1]):
            f = dict(img=list(img[0, t]), cam2img=[np.array(m, np.float64) for m in cam2img[0]],
                     lidar2cam=[np.array(m, np.float64) for m in lidar2cam[0]])
            if self.openscene:                                  # get_data_info's lidar2img: no crop step forms it
                f["lidar2img"] = [c @ l for c, l in zip(f["cam2img"], f["lidar2cam"])]
            frames.append(f)
        return run_image_transforms(self.image_transforms, frames)

    def _frames(self, img, lidar2img, cam2img, lidar2cam, img_metas, pose_metas, future_frames, feature_cache):
        """A sample's image frames in any of its three forms (see `_next_bev_preds`) -> (frame, cams_only, metas, hw):
        frame(t) is frame t's `extract_feat` input and `cams_only` its form, metas[t] the frame's img_metas with
        `pose_metas` merged, hw the padded image size.  The image pipeline's host draws are made here, for every frame
        in the dataset's order; its device half runs when frame(t) is called, just before that frame's backbone, so
        that only one frame's float images are held at a time."""
        loaded = img_metas is not None
        if feature_cache is not None and (not loaded or any("filename" not in m[0] for m in img_metas)):
            raise ValueError("_next_bev_preds: feature_cache needs a test-mode SampleLoader sample (img_metas with "
                             "each frame's filename)")
        if loaded:
            if len(img_metas) != len(img):
                raise ValueError(f"_next_bev_preds: {len(img)} loaded frames, {len(img_metas)} img_metas")
            frame, metas, hw = img.__getitem__, img_metas, tuple(img[-1].shape[-2:])
        elif self.image_transforms is not None:
            results = self.frame_transforms(img, cam2img, lidar2cam)
            metas = [[dict(lidar2img=np.stack(r["lidar2img"]), img_shape=r["img_shape"])] for r in results]
            hw = results[-1]["img_aug"].pad_hw
            mine = self.my_backbone_cams

            def frame(t):                             # this rank's cameras, as a SampleLoader frame holds them
                if not mine:
                    return img.new_empty((0, 3, *results[t]["img_aug"].pad_hw), dtype=torch.float32)
                return image_aug.apply_multiview(img[0, t, mine], results[t], mine)
        else:
            def frame(t):
                return img[:, t]
            metas = [[dict(lidar2img=np.asarray(lidar2img[b]), img_shape=[(img.shape[-2], img.shape[-1], 3)])
                      for b in range(img.shape[0])]] * img.shape[1]
            hw = img.shape[-2:]
        T, bs = len(metas), len(metas[0])
        if pose_metas is not None:
            if len(pose_metas) != T or bs != 1:
                raise ValueError(f"_next_bev_preds: pose_metas needs bs 1 and one dict per image frame ({T} frames, "
                                 f"bs {bs}, got {len(pose_metas)})")
            metas = [[dict(m[0], **p)] for m, p in zip(metas, pose_metas)]
        if self.ego_motion:
            for m in metas:
                ego.require_metas(m)
            ego.require_metas(metas[T - 1], future_frames)
        return frame, loaded or self.image_transforms is not None, metas, hw

    def _next_bev_preds(self, img, lidar2img, can_bus, future_frames, cam2img=None, lidar2cam=None, train=False,
                        drop_prev_index=-1, supervised=None, img_metas=None, feature_cache=None, pose_metas=None):
        """img [bs, T, cams, 3, H, W] -> next_bev_preds [1 + len(supervised), inter, pred_frame, bs, Q, 16]: the
        history BEV of the first T - 1 frames, the current frame's BEV as ref_bev, `future_frames` roll-outs with a
        queue of length 1 -- those not in `supervised` (default: all) under no_grad --, then the head over the current
        and the supervised frames.  With the image pipeline, img is uint8 [1, T, cams, H, W, 3] and the camera
        matrices come from cam2img / lidar2cam.

        The history as `obtain_history_bev` (bevformer.py:158-236): with `train`, the last
        `backward_history_frames` frames are backwarded -- backbone under no_grad, encoder with gradient --, the
        others frozen under no_grad; frozen frame i < `drop_prev_index` is not computed, as its BEV would be
        discarded.  Each of the two parts makes its eval-mode GridMask draw (one prob gate per extract_feat call of
        the reference), also when the drop skips every frozen frame.

        `img_metas` (a `SampleLoader` sample): img is then a list over the T frames of the pipelined images of this
        rank's backbone cameras, float32 [len(backbone_cams()), 3, H, W], and img_metas the frames' metas.

        `feature_cache` (a dict, with a test-mode `SampleLoader` sample, whose metas carry each frame's `filename`): a
        frame whose camera files were a frame of the previous call's sample takes that frame's stored extract_feat
        output (feats, spatial_shapes, level_start_index) instead of running the backbone again; on return the dict
        holds this sample's frames only.  A frame masked by a GridMask draw is always computed and never stored.  The
        GridMask draws are made as without the cache.

        `pose_metas` (with `ego_motion`, for the tensor path): one dict per image frame, `ego_motion.queue_metas`' (bs
        1), merged into each frame's metas; a `SampleLoader` sample's img_metas carry them already."""
        frame, cams_only, metas, hw = self._frames(img, lidar2img, cam2img, lidar2cam, img_metas, pose_metas,
                                                   future_frames, feature_cache)
        T, bs = len(metas), len(metas[0])
        dev = img[0].device
        can_bus = torch.zeros(bs, 18, device=dev) if can_bus is None else can_bus
        backwarded = min(self.backward_history_frames, T - 1) if train else 0
        frozen = T - 1 - backwarded
        fresh = None if feature_cache is None else {}

        def features(t, draw=None):
            if fresh is None or draw is not None:
                return self.extract_feat(frame(t), draw, cams_only=cams_only)
            key = tuple(metas[t][0]["filename"])
            out = feature_cache.get(key)
            if out is None:
                out = self.extract_feat(frame(t), cams_only=cams_only)
            fresh[key] = out
            return out

        prev_bev = None
        if self.grid_mask is not None and frozen > 0:                                # the history's eval-mode call
            self.grid_mask.sample(*hw, training=False)
        with torch.no_grad():                                                        # _obtain_frozen_history_bev
            for t in range(min(max(drop_prev_index, 0), frozen), frozen):
                feats, shapes, lsi = features(t)
                self._mark(f"hist{t}.backbone")
                prev_bev = self.encode(feats, shapes, lsi, metas[t], can_bus, prev_bev)
                self._mark(f"hist{t}.encoder")
        if backwarded and self.grid_mask is not None:                                # _obtain_backwarded_history_bev
            self.grid_mask.sample(*hw, training=False)
        for t in range(frozen, T - 1):
            with torch.no_grad():
                feats, shapes, lsi = features(t)
            self._mark(f"hist{t}.backbone")
            prev_bev = self.encode(feats, shapes, lsi, metas[t], can_bus, prev_bev)
            self._mark(f"hist{t}.encoder")
        draw = self.grid_mask.sample(*hw) if self.grid_mask is not None else None
        feats, shapes, lsi = features(T - 1, draw)
        if fresh is not None:                                                        # only this sample's frames
            feature_cache.clear()
            feature_cache.update(fresh)
        self._mark("cur.backbone")
        ref_bev = self.encode(feats, shapes, lsi, metas[T - 1], can_bus, prev_bev)
        self._mark("cur.encoder")
        inter_num = len(self.bev_pred_head)
        next_bev_feats = [ref_bev.unsqueeze(0).repeat(inter_num, 1, 1, 1)]
        prev_bev_input = ref_bev.unsqueeze(1)
        future_inputs = [(can_bus, None)] * future_frames
        if self.ego_motion and future_frames:                                        # vidar.py:319-363
            future_inputs = ego.future_inputs(metas[T - 1], future_frames, self.bev_h, self.bev_w, PC_RANGE, dev,
                                              self.bev_embedding.weight.dtype)
        for k in range(1, future_frames + 1):
            if supervised is None or k in supervised:
                pred_feat, last = self.decode_future(prev_bev_input, *future_inputs[k - 1])
                next_bev_feats.append(pred_feat)
            else:
                with torch.no_grad():
                    _, last = self.decode_future(prev_bev_input, *future_inputs[k - 1])
            prev_bev_input = last.unsqueeze(1)                                         # queue length 1 (vidar.py:359-360)
        self._mark("future_decoder")
        next_bev_feats = torch.stack(next_bev_feats, 0)
        return self.forward_head(next_bev_feats)                                        # [F, inter, pred_frame, bs, Q, 16]

    def host_draws(self, num_frames):
        """forward_train's own draws from numpy's global generator, in its order (vidar.py:262-281, :333-338) ->
        (drop_prev_index, supervised future frames or None for all).  No draw without `reference_draws`."""
        if not self.reference_draws:
            return -1, None
        np.random.rand()                                  # A1: random_drop_image_rate is 0.0 in every config
        drop_prev_index = -1
        if np.random.rand() < self.drop_prev_rate:        # A2
            end = self.drop_prev_end_idx if self.drop_prev_end_idx is not None else num_frames
            drop_prev_index = int(np.random.randint(self.drop_prev_start_idx, end))
        supervised = None
        if self.future_frames > 0 and not self.supervise_all_future:
            supervised = [int(np.random.choice(np.arange(1, self.future_frames + 1), 1)[0])]
        return drop_prev_index, supervised

    def gt_points_of(self, point_infos, training):
        """The point half of the sample with the point pipeline: every GT frame's transforms in queue order (numpy's
        draws), then one device pass -> gt_points [1, R, 5] (NaN rows belong to no frame)."""
        if not point_infos:
            raise ValueError("point_pipeline: forward needs point_infos (synthetic_sample(..., raw_points=True))")
        return self.gather_points(run_point_transforms(self.point_transforms[0 if training else 1], point_infos))

    def gather_points(self, point_frames, ego_mask=EGO_MASK):
        """The device half of gt_points_of: the transformed GT frames' results -> gt_points [1, R, 5] (6 columns with
        `openscene`), on the current stream.  `ego_mask`: union2one's ego box."""
        return point_aug.gather_gt_points(point_frames, ego_mask, self.bev_embedding.weight.device)

    # ---- one training forward (vidar.py:239-387) -> dict of losses ----
    def forward_train(self, img, lidar2img, gt_points, can_bus=None, cam2img=None, lidar2cam=None, point_infos=None,
                      draws=None, img_metas=None, pose_metas=None):
        """img [bs, T, cams, 3, H, W] (T-1 history frames + current), lidar2img: host array [bs, cams, 4, 4]
        (it lives in `img_metas` in the reference), gt_points: list over batch of [M, 4] (x, y, z metric,
        frame index 0 = current .. future_frames).  With the image pipeline: img uint8 [1, T, cams, H, W, 3] and
        host cam2img / lidar2cam [1, cams, 4, 4]; lidar2img is not read.  With the point pipeline gt_points is built
        from point_infos.  `draws`: `host_draws`'s (drop_prev_index, supervised future frames) to use instead of
        drawing them.

        A `SampleLoader` sample instead: `img_metas` given, img the list of the T frames' pipelined images of this
        rank's backbone cameras and gt_points its device [1, R, 5]; the transforms ran in the loader, so neither
        pipeline runs here and lidar2img, cam2img, lidar2cam and point_infos are not read.  `pose_metas`: see
        `_next_bev_preds` (ego_motion)."""
        loaded = img_metas is not None
        num_frames = len(img) if loaded else img.shape[1]
        drop_prev_index, supervised = self.host_draws(num_frames) if draws is None else draws
        if self.point_transforms is not None and not loaded:
            gt_points = self.gt_points_of(point_infos, True)
        next_bev_preds = self._next_bev_preds(img, lidar2img, can_bus, self.future_frames, cam2img, lidar2cam,
                                              train=self.training, drop_prev_index=drop_prev_index,
                                              supervised=supervised, img_metas=img_metas, pose_metas=pose_metas)
        valid_frames = [0] + (list(range(1, 1 + self.future_frames)) if supervised is None else list(supervised))
        fw = self.frame_loss_weight
        losses = {}
        for i in range(self.pred_frame_num):                                            # vidar_head_v1.py:179-218
            pred_dict = dict(next_bev_preds=next_bev_preds[:, :, i], valid_frames=valid_frames)
            if fw is None:
                lw = np.array([[self.per_frame_loss_weight[i]]] * len(valid_frames))
                scale = None
            else:           # the current head frame by the frame weights, the others on the current frame only
                lw = fw if i == self.head_history_frames else np.array([[1.0]] + [[0.0]] * (len(fw) - 1))
                scale = self.per_frame_loss_weight[i]
            ld = self.ray_head.loss(pred_dict, gt_points, 0, self.bev_h, self.bev_w, PC_RANGE, pred_frame_num=1 + self.future_frames,
                                    loss_weight=lw)
            for k, v in ld.items():
                losses[f"frame.{i}.{k}"] = v if scale is None else v * scale
        self._mark("head+loss")
        return losses

    # ---- inference (vidar.py:389-502) ----
    @torch.no_grad()
    def predict_future(self, img, lidar2img, future_frames, can_bus=None, img_metas=None, feature_cache=None,
                       pose_metas=None):
        """forward_test's prediction (vidar.py:392-437): the same inputs as forward_train, `future_frames` roll-outs
        (the reference's test_future_frame_num) -> pred_dict {next_bev_preds [1 + future_frames, inter, pred_frame,
        bs, Q, 16], valid_frames [0 .. future_frames]}.  `feature_cache`, `pose_metas`: see `_next_bev_preds`."""
        next_bev_preds = self._next_bev_preds(img, lidar2img, can_bus, future_frames, img_metas=img_metas,
                                              feature_cache=feature_cache, pose_metas=pose_metas)
        return dict(next_bev_preds=next_bev_preds, valid_frames=list(range(1 + future_frames)))

    def forward_test(self, img, lidar2img, gt_points, future_frames=6, can_bus=None, point_infos=None,
                     img_metas=None, pose_metas=None):
        """vidar.py:389-502 without submission writing and visualisation -> [ret_dict], ret_dict =
        {f"frame.{t}": {count, chamfer_distance, l1_error, absrel_error}} for the current frame (t = 0) and every
        future frame, scored on the current head frame (`head_history_frames`) by ray_head.evaluate (one batched device
        pass).  gt_points as forward_train's, frames 0 .. future_frames; the origin is zero in every frame.  Under a
        process group every rank computes the same result.  With the point pipeline gt_points is built from
        point_infos by the test pipeline.  `img_metas`: a `SampleLoader` sample, as in forward_train; its frames and
        gt_points went through the loader's train transforms, which this path then scores as they are."""
        if self.point_transforms is not None and img_metas is None:
            gt_points = self.gt_points_of(point_infos, False)
        pred_dict = self.predict_future(img, lidar2img, future_frames, can_bus, img_metas=img_metas,
                                        pose_metas=pose_metas)
        with torch.no_grad():
            ret = self.ray_head.evaluate(self._current_head_frame(pred_dict), gt_points, 0, self.bev_h, self.bev_w,
                                         PC_RANGE)
        return [ret]

    def _current_head_frame(self, pred_dict):
        """`predict_future`'s pred_dict with the current head frame (`head_history_frames`) only, the frame that
        forward_test and `evaluate` score."""
        return dict(pred_dict, next_bev_preds=pred_dict["next_bev_preds"][:, :, self.head_history_frames])


# ------------------------------------------------------------------------------------------------
# synthetic sample + step
# ------------------------------------------------------------------------------------------------
def synthetic_sample(device, frames=4, cams=6, img_hw=None, rays_per_frame=10000, future_frames=3, seed=0,
                     bev_hw=(BEV_H, BEV_W), raw_images=False, raw_points=False, points_per_frame=35000, files=False,
                     poses=False, scene_change=None, openscene=False):
    """6 x 3 x 928 x 1600 N(0,1) frames, a nuScenes-like rig, LiDAR-like future point clouds (SURVEY.md 8d cfg4).
    `raw_images=True` (for `SyntheticViDAR(image_pipeline=True)`): seeded uniform uint8 BGR frames
    [1, frames, cams, 900, 1600, 3] (img_hw defaults to the camera size) and the rig's host `cam2img` / `lidar2cam`
    [1, cams, 4, 4] float64 as well.
    `raw_points=True` (for `SyntheticViDAR(point_pipeline=True)`): `point_infos`, the results dicts of the
    1 + future_frames GT frames, each a LiDAR-like key frame and 2 sweeps of `points_per_frame` points with their
    own poses and timestamps (`synthetic.lidar_cloud`, `synthetic.sweep_pose`), written as .bin files to a
    temporary directory that is removed when the process exits.
    `files=True` (for `SampleLoader`): instead of a sample, the queue's results dicts as a dataset's get_data_info
    hands them to its pipeline, one per queue frame, oldest first: the `frames` image frames (the history and the
    current one) with `img_filename`, `cam2img` and `lidar2cam`, the current and the future frames with the point
    infos of `raw_points`.  Each camera image is a baseline 4:2:0 JPEG written by cv2.imwrite at quality
    `JPEG_QUALITY` (img_hw defaults to 900 x 1600), to a temporary directory removed at exit.  `device` is not used.
    `poses=True` (for `SyntheticViDAR(ego_motion=True)`): the queue frames follow a seeded drive (`synthetic.drive`,
    `scene_change` = the first frame of a second scene): with `files`, every queue frame carries its pose fields;
    otherwise the sample holds `pose_metas`, `ego_motion.queue_metas` of the frames + future_frames drive.
    `openscene=True` (with `files`, for the OpenScene presets): an OpenScene rig instead -- 8 cameras of 1920 x 1080
    (`synthetic.nuplan_camera_rig_split`; `cams` and `img_hw` are not read), every image frame also carrying the
    dataset's `lidar2img` = cam2img @ lidar2cam and a `sample_idx`, and each GT frame a binary .pcd with nuPlan's six
    fields and sweeps=[], as NuPlanViDARDatasetTemplate.get_data_info hands them on."""
    if openscene and not files:
        raise ValueError("synthetic_sample: openscene=True needs files=True")
    if files:
        return synthetic_queue(frames, cams, img_hw or (900, 1600), future_frames, points_per_frame, seed,
                               poses=poses, scene_change=scene_change, openscene=openscene)
    g = torch.Generator(device=device).manual_seed(seed)
    extra = {}
    if raw_images:
        img_hw = img_hw or (900, 1600)
        img = torch.randint(0, 256, (1, frames, cams, img_hw[0], img_hw[1], 3), device=device, generator=g,
                            dtype=torch.uint8)
        cam2img, lidar2cam = synthetic.camera_rig_split(cams)
        extra = dict(cam2img=cam2img[None], lidar2cam=lidar2cam[None])
    else:
        img_hw = img_hw or synthetic.IMG_HW
        img = torch.randn(1, frames, cams, 3, img_hw[0], img_hw[1], device=device, generator=g)
    lidar2img = synthetic.camera_rig(cams).numpy()[None]                     # host side, like img_metas
    pts = []
    _, origin, points, tindex = synthetic.dvr_inputs_lidar(M=rays_per_frame * (1 + future_frames), T=1 + future_frames, seed=seed,
                                                           grid=(HEIGHTS, bev_hw[0], bev_hw[1]))
    # voxel units -> metres (inverse of coords_to_voxel_grids)
    p = points[0]
    xyz = np.stack([p[:, 0] / bev_hw[1] * (PC_RANGE[3] - PC_RANGE[0]) + PC_RANGE[0],
                    p[:, 1] / bev_hw[0] * (PC_RANGE[4] - PC_RANGE[1]) + PC_RANGE[1],
                    p[:, 2] / HEIGHTS * (PC_RANGE[5] - PC_RANGE[2]) + PC_RANGE[2]], -1)
    pts.append(torch.from_numpy(np.concatenate([xyz, tindex[0][:, None]], -1).astype(np.float32)).to(device))
    if raw_points:
        extra["point_infos"] = synthetic_point_infos(1 + future_frames, points_per_frame, seed)
    if poses:
        drive = synthetic.drive(frames + future_frames, seed, scene_change)
        extra["pose_metas"] = ego.queue_metas([dict(p, img_filename=()) for p in drive[:frames]] + drive[frames:])
    return dict(img=img, lidar2img=lidar2img, gt_points=pts, **extra)


JPEG_QUALITY = 90


def _temp_dir(prefix):
    """A new temporary directory, removed when the process exits."""
    import atexit
    import shutil
    import tempfile
    root = tempfile.mkdtemp(prefix=prefix)
    atexit.register(shutil.rmtree, root, True)
    return root


def synthetic_queue(frames, cams, img_hw, future_frames, points_per_frame, seed=0, first_gt=None, poses=False,
                    scene_change=None, openscene=False):
    """`synthetic_sample(..., files=True)`: image frames 0 .. frames - 1, point frames first_gt (default frames - 1)
    .. frames - 1 + future_frames, every frame with the same rig.  `poses`: frame t also carries the pose fields of
    drive frame t (`synthetic.drive(..., scene_change)`); the default leaves the queue as without them.
    `openscene`: the OpenScene rig of `synthetic_sample`."""
    first_gt = frames - 1 if first_gt is None else first_gt
    import cv2
    root = _temp_dir("vidar_cameras_")
    rng = np.random.default_rng(seed + 1000003)
    if openscene:
        cams, img_hw = 8, synthetic.NUPLAN_IMG_HW
        cam2img, lidar2cam = synthetic.nuplan_camera_rig_split()
    else:
        cam2img, lidar2cam = synthetic.camera_rig_split(cams)
    params = [cv2.IMWRITE_JPEG_QUALITY, JPEG_QUALITY, cv2.IMWRITE_JPEG_PROGRESSIVE, 0,
              cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
    queue = []
    for t in range(frames):
        names = []
        for c in range(cams):
            name = os.path.join(root, f"{t}.cam{c}.jpg")
            if not cv2.imwrite(name, synthetic.camera_image(rng, img_hw), params):
                raise RuntimeError(f"synthetic_sample: cv2.imwrite could not write {name}")
            names.append(name)
        queue.append(dict(img_filename=names, cam2img=[m.copy() for m in cam2img],
                          lidar2cam=[m.copy() for m in lidar2cam]))
        if openscene:
            queue[-1].update(lidar2img=[c @ l for c, l in zip(cam2img, lidar2cam)], sample_idx=f"s{seed}f{t}")
    for k, info in enumerate(synthetic_point_infos(frames - first_gt + future_frames, points_per_frame, seed,
                                                   pcd=openscene)):
        if first_gt + k < frames:
            queue[first_gt + k].update(info)
        else:
            queue.append(info)
    if poses:
        for f, p in zip(queue, synthetic.drive(len(queue), seed, scene_change)):
            f.update(p)
    return queue


def synthetic_scene(num_samples, frames, future_frames, cams=6, img_hw=(900, 1600), points_per_frame=35000, seed=0,
                    poses=False, openscene=False):
    """One scene's files, written once (`synthetic_queue`), as the sliding-window queues a test dataset builds from
    consecutive keyframes (no load_frame_interval): sample i's image frames are the scene's frames i .. i + frames - 1
    (the history and the current frame), its GT frames i + frames - 1 .. i + frames - 1 + future_frames.  Each image
    frame carries `img_filename`, `cam2img`, `lidar2cam` and the test pipeline's `lidar2img` = cam2img @ lidar2cam
    (float64), so the queues serve the test-mode and the train-mode `SampleLoader` alike.  Neighbouring samples share
    frames - 1 image frames' files.  `poses`: every frame carries its pose fields of one drive over the scene
    (`synthetic.drive`).  `openscene`: the OpenScene rig of `synthetic_sample`, each image frame with its
    `sample_idx`.  -> [queue] of num_samples queues."""
    if num_samples < 1 or frames < 1 or future_frames < 0:
        raise ValueError(f"synthetic_scene: num_samples, frames >= 1 and future_frames >= 0 "
                         f"(got {num_samples}, {frames}, {future_frames})")
    total = num_samples + frames - 1
    scene = synthetic_queue(total, cams, img_hw, future_frames, points_per_frame, seed, first_gt=frames - 1,
                            poses=poses, openscene=openscene)
    pose = ego.POSE_KEYS if poses else ()
    tags = ("sample_idx",) if openscene else ()
    images = [dict(img_filename=list(f["img_filename"]), cam2img=f["cam2img"], lidar2cam=f["lidar2cam"],
                   lidar2img=[c @ l for c, l in zip(f["cam2img"], f["lidar2cam"])], **{k: f[k] for k in pose + tags})
              for f in scene[:total]]
    gts = [{k: f[k] for k in ("pts_filename", "timestamp", "sweeps") + pose} for f in scene if "pts_filename" in f]
    queues = []
    for i in range(num_samples):
        queue = [dict(images[t]) for t in range(i, i + frames)]
        queue[-1].update(gts[i])
        queues.append(queue + [dict(g) for g in gts[i + 1:i + 1 + future_frames]])
    return queues


def synthetic_point_infos(frames, n, seed=0, sweeps=2, pcd=False):
    """Results dicts (pts_filename, timestamp, sweeps) of `frames` LiDAR frames, files in a temporary directory.
    `pcd`: nuPlan key frames instead, binary .pcd files of six fields (`synthetic.write_pcd`) with sweeps=[]."""
    root = _temp_dir("vidar_points_")
    rng = np.random.default_rng(seed)
    infos = []
    for f in range(frames):
        ts = 1533151603547590 + 500000 * f
        if pcd:
            key = os.path.join(root, f"{f}.pcd")
            synthetic.write_pcd(key, synthetic.nuplan_cloud(rng, n))
            infos.append(dict(pts_filename=key, timestamp=ts / 1e6, sweeps=[]))
            continue
        key = os.path.join(root, f"{f}.bin")
        synthetic.lidar_cloud(rng, n).tofile(key)
        sw = []
        for j in range(sweeps):
            path = os.path.join(root, f"{f}.sweep{j}.bin")
            synthetic.lidar_cloud(rng, n).tofile(path)
            R, t = synthetic.sweep_pose(rng, j + 1)
            sw.append(dict(data_path=path, timestamp=ts - 50000 * (j + 1), sensor2lidar_rotation=R,
                           sensor2lidar_translation=t))
        infos.append(dict(pts_filename=key, timestamp=ts / 1e6, sweeps=sw))
    return infos


def train_step(model, optimizer, sample, group=None, record=False, scaler=None, grid=None):
    """forward_train + backward + gradient sync of the sharded parameters + clip(35) + AdamW step
    (config :379-388); with an `optim.AdamW` (`config_optimizer`) the clip is the one inside its step.  With a `torch.amp.GradScaler` (for a float16 `backbone_autocast`) the loss is scaled before
    the backward and the gradients unscaled before the clip; the scaler skips a step whose gradients are not finite.
    `grid` (`sharding.make_grid`, the model built with `build(..., grid=grid)`): `sample` is this replica's sample
    and the sync is the grid's one bucketed all-reduce (`sharding.allreduce_grid_grads`): every rank ends with the
    replica mean of the gradients.  `sample` may be a `SampleLoader` sample (its frames decoded and pipelined, its
    gt_points on the device).  -> (loss value tensor -- this replica's --, [(stage, ms)] when `record`)."""
    if grid is not None and group is not None:
        raise ValueError("train_step: pass group= or grid=, not both")
    model.timings = [] if record else None
    if record:
        model._mark("start")
    optimizer.zero_grad(set_to_none=True)
    losses = model.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"], can_bus=sample.get("can_bus"),
                                 cam2img=sample.get("cam2img"), lidar2cam=sample.get("lidar2cam"),
                                 point_infos=sample.get("point_infos"), img_metas=sample.get("img_metas"),
                                 pose_metas=sample.get("pose_metas"))
    loss = sum(losses.values())
    (loss if scaler is None else scaler.scale(loss)).backward()
    model._mark("backward")
    if grid is not None:
        sharding.allreduce_grid_grads(model, grid)
        model._mark("grad_sync")
    elif group is not None:
        sharding.allreduce_partial_grads(model, group)
        model._mark("grad_sync")
    if scaler is not None:
        scaler.unscale_(optimizer)
    if not isinstance(optimizer, optim.AdamW):            # optim.AdamW clips inside its step
        torch.nn.utils.clip_grad_norm_([p for p in model.parameters() if p.requires_grad], 35.0)
    if scaler is None:
        optimizer.step()
    else:
        scaler.step(optimizer)
        scaler.update()
    model._mark("optimizer")
    stages = None
    if record:
        torch.cuda.synchronize()
        ev = model.timings
        stages = [(ev[i + 1][0], ev[i][1].elapsed_time(ev[i + 1][1])) for i in range(len(ev) - 1)]
    model.timings = None
    return loss.detach(), stages


# The training regimes of the four nuScenes pre-training configs (projects/configs/vidar_pretrain/nusc_*), as
# SyntheticViDAR arguments: `build(device, config=name)`.  Sizes, the backbone (dcn) and the pipelines are not part of
# a preset; arguments passed to `build` override the preset's.
_HEAD_5 = dict(head_history_frames=3, head_future_frames=1, per_frame_loss_weight=(0.2, 0.4, 0.6, 1.0, 1.2))
_ONE_FUTURE = dict(history_frames=3, future_frames=0, decoder_layers=1, backward_history_frames=1, drop_prev_rate=0.1,
                   drop_prev_end_idx=3, frame_loss_weight=((1.0,), (0.0,)), point_voxel_size=0.5, reference_draws=True,
                   **_HEAD_5)
# The four OpenScene (nuPlan) training configs (projects/configs/vidar_pretrain/OpenScene/vidar_OpenScene_{train,mini}_
# {1_8,full}_3future.py) share one graph; only their dataset split and load_frame_interval (8 for 1_8, 1 for full)
# differ, and neither is part of the step.  num_cams=8; queue_length 4 = history_frames 3 + the current frame.
# future_queue_length_train = 3 is the number of future GT frames the dataset appends after the current one (its
# future_length): frames 0 .. 3, exactly the 1 + future_frames the model predicts and supervises (frame_loss_weight's
# fifth row belongs to no frame).  The nuScenes 3-future configs set future_queue_length_train = 4 with
# future_pred_frame_num_train = 3: the dataset appends a fourth future frame that no roll-out predicts, so those
# presets also take future_frames=3 with 1 + 3 GT frames.  The submit config is test-time only (queue_length 5, six
# roll-outs, ego_mask (0, 0, 0, 0)): `evaluate(..., future_frames=6, ego_mask=(0, 0, 0, 0), submission_path=...)`.
_OPENSCENE = dict(num_cams=8, history_frames=3, future_frames=3, decoder_layers=3, head_history_frames=0,
                  head_future_frames=0, per_frame_loss_weight=(1.0,), frame_loss_weight=((1.0,),) * 4 + ((0.0,),),
                  supervise_all_future=True, latent_grid_step=0.5, reference_draws=True, openscene=True)
OPENSCENE_CONFIGS = ("vidar_OpenScene_train_1_8_3future", "vidar_OpenScene_mini_1_8_3future",
                     "vidar_OpenScene_train_full_3future", "vidar_OpenScene_mini_full_3future")
CONFIGS = {
    "vidar_1_8_nusc_3future": dict(history_frames=3, future_frames=3, decoder_layers=3,
                                   frame_loss_weight=((1.0,),) * 4 + ((0.0,),), latent_grid_step=0.5,
                                   reference_draws=True, **_HEAD_5),
    "vidar_full_nusc_1future": dict(_ONE_FUTURE, latent_grid_step=0.5),
    "vidar_1_8_nusc_1future": dict(_ONE_FUTURE, latent_grid_step=1.0),
    "mem_efficient_vidar_1_8_nusc_3future": dict(history_frames=3, future_frames=3, decoder_layers=3,
                                                 supervise_all_future=False, head_history_frames=0,
                                                 head_future_frames=0, per_frame_loss_weight=(1.0,),
                                                 frame_loss_weight=((1.0,),) * 4 + ((0.0,),), latent_grid_step=1.0,
                                                 reference_draws=True),
    **{name: dict(_OPENSCENE) for name in OPENSCENE_CONFIGS},
}


def build(device, group=None, lr=2e-4, seed=0, row_sharded=False, grid=None, config=None, **model_kwargs):
    """-> (SyntheticViDAR in training mode with dropout off, AdamW).  `config`: a name in `CONFIGS`, whose training
    regime `model_kwargs` then override; None builds the default graph.  `group`: one sample sharded over it.  `grid`
    (`sharding.make_grid(S)`): data-parallel replicas of the sharded model -- the model shards over the grid's shard
    group of S ranks, and `train_step(..., grid=grid)` averages the gradients over the world / S replicas.  Every rank
    passes the same `seed` (the replicas start from the same parameters).

    Each replica trains on its own sample, and the host draws of a step (forward_train's drop index and supervised
    future frame under a preset, GridMask, the image and the point pipeline:
    numpy's global generator, and `random` for the image pipeline) must agree inside a shard group and differ across
    replicas.  Seed per replica, for example with base the run's seed:
        np.random.seed(base + grid.replica); random.seed(base + grid.replica)
        sample = synthetic_sample(device, seed=base + grid.replica, ...)
    The row-sharded encoder is not supported under a grid."""
    if grid is not None:
        if group is not None:
            raise ValueError("build: pass group= or grid=, not both")
        if row_sharded:
            raise ValueError("build: the row-sharded encoder is not supported under a grid")
        group = grid.group
    if config is not None:
        if config not in CONFIGS:
            raise ValueError(f"build: unknown config {config!r}; one of {sorted(CONFIGS)}")
        model_kwargs = dict(CONFIGS[config], **model_kwargs)
    torch.manual_seed(seed)
    model = SyntheticViDAR(**model_kwargs).to(device)
    model.set_process_group(group, row_sharded=row_sharded)
    model.train()
    for m in model.modules():                      # dropout off: replicated parts must stay identical over ranks
        if isinstance(m, nn.Dropout):
            m.p = 0.0
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=lr, weight_decay=0.01)
    return model, opt


def config_optimizer(model, lr=2e-4):
    """The configs' optimizer (vidar_1_8_nusc_3future.py:379-388, built by mmcv's DefaultOptimizerConstructor and
    OptimizerHook): AdamW, weight decay 0.01, one group per parameter with the backbone at lr_mult 0.1 (the config's
    `img_backbone` is this model's `backbone`), the gradients clipped to a total 2-norm of 35 -- as one
    `optim.AdamW` step.  `build()` keeps torch's single-group AdamW; pass this to `train_step` instead."""
    return optim.AdamW(optim.paramwise_groups(model, lr, 0.01, {"backbone": dict(lr_mult=0.1)}), lr=lr,
                       weight_decay=0.01, max_grad_norm=35)


# ------------------------------------------------------------------------------------------------
# evaluation from files (the configs' `evaluation = dict(pipeline=test_pipeline)`, tools/test.py)
# ------------------------------------------------------------------------------------------------
def evaluate(model, samples, future_frames=6, num_workers=0, prefetch=1, seed=0, grid=None, ego_mask=EGO_MASK,
             submission_path=None):
    """The dataset's evaluation over `samples` (queues of results dicts in dataset order, e.g. `synthetic_scene`'s):
    the test-mode `SampleLoader`, the prediction of `forward_test` per sample, then `evaluate.summarize` -> the
    summary {f"frame.{t}": {count, chamfer_distance, l1_error, absrel_error}}, equal to
    summarize([model.forward_test(...)[0] for each sample]) in dataset order (the reference's single_gpu_test /
    multi_gpu_test, then dataset.evaluate).  The model must be built with point_pipeline=True.

      * Each sample's metric table comes from the head's `evaluate_device` and stays on the device; the tables reach
        the host once, at the end (`summarize_tables`).
      * Feature reuse: consecutive samples of a scene share all image frames but the newest, and the test chain makes
        no draw, so a frame's backbone + FPN output is the same in every sample that holds it.  A frame whose camera
        files were in the previous sample takes that sample's features instead of running the backbone again
        (`predict_future(..., feature_cache=...)`); across a scene boundary the files differ and the frame is
        computed.  The cache lives for this call and holds one sample's frames.  GridMask's draws are made as without
        it, so numpy's generator advances alike.
      * `grid` (`sharding.make_grid`, the model built with it): replica r evaluates the contiguous block
        `sharding.shard_range(N, r, R)` of the samples (contiguous, so the reuse keeps working); every rank of its
        shard group walks the same block, so they hit and miss the cache together.  One all-gather of the tables over
        the world, then every rank builds the same summary, and raises the same exception for the first failing
        (sample, frame).

    A queue with fewer than 1 + future_frames GT frames is rejected before any work.

    The test chain is the model's (`test_image_transforms` and `point_transforms[1]`: the OpenScene test pipeline for
    a model built with openscene=True).  `ego_mask`: the dataset's union2one ego box (the submit config's is
    (0, 0, 0, 0)).  `submission_path` (the submit config's `_submission`, vidar.py:491-519): each sample's predicted
    points of every future frame t > 0 also go to `<submission_path>/<sample_idx>_<t>.txt`, one '%f' depth (the
    norm of the predicted point) per line, where `sample_idx` is the current image frame's; the depths of a sample's
    frames reach the host in one copy.  Every rank of a grid writes its replica's samples when its shard rank is 0."""
    samples = list(samples)
    for i, queue in enumerate(samples):
        gt = sum("pts_filename" in f for f in queue)
        if gt < 1 + future_frames:
            raise ValueError(f"evaluate: sample {i} has {gt} GT frames; future_frames={future_frames} needs "
                             f"{1 + future_frames} (the current frame and every future one)")
    replica, replicas = (grid.replica, grid.replicas) if grid is not None else (0, 1)
    lo, hi = sharding.shard_range(len(samples), replica, replicas)
    names = None
    if submission_path is not None:
        names = []
        for i, queue in enumerate(samples[lo:hi]):
            current = [f for f in queue if "img_filename" in f][-1]
            if "sample_idx" not in current:
                raise ValueError(f"evaluate: submission_path needs each sample's current image frame's sample_idx "
                                 f"(sample {lo + i} has none)")
            names.append(str(current["sample_idx"]))
        os.makedirs(submission_path, exist_ok=True)
    write = names is not None and (grid is None or grid.shard_rank == 0)
    loader = SampleLoader(model, samples[lo:hi], num_workers=num_workers, prefetch=prefetch, seed=seed, rank=replica,
                          test_mode=True, ego_mask=ego_mask)
    dev = model.bev_embedding.weight.device
    frames = 1 + future_frames
    tables, cache = [], {}
    with torch.no_grad():
        for sample in loader:
            pred = model.predict_future(sample["img"], None, future_frames, img_metas=sample["img_metas"],
                                        feature_cache=cache)
            tables.append(model.ray_head.evaluate_device(model._current_head_frame(pred), sample["gt_points"], 0,
                                                         model.bev_h, model.bev_w, PC_RANGE))
            if write:
                save_predictions(model, pred, sample["gt_points"], submission_path, names[sample["index"]])
            del pred, sample                       # freed before the next sample's device half
    cache.clear()
    table = torch.cat(tables) if tables else torch.zeros((0, eval_metrics.FIELDS), dtype=torch.float64, device=dev)
    return summarize_tables(table, len(samples), frames, grid)


def save_predictions(model, pred, gt_points, path, sample_idx):
    """The reference's `_save_prediction` for one sample (vidar.py:491-519): the head's decoded prediction
    (`get_point_cloud_prediction` of the current head frame), then per future frame t > 0 the file
    `<path>/<sample_idx>_<t>.txt` with sqrt(sum(pred_pcd ** 2, 1)) -- one '%f' per line.  The depths of all frames are
    computed on the device and copied to the host once."""
    decode = model.ray_head.get_point_cloud_prediction(model._current_head_frame(pred), gt_points, 0, model.bev_h,
                                                       model.bev_w, PC_RANGE)
    pcds = decode["pred_pcds"][0][1:]
    if not pcds:
        return
    depth = torch.cat([torch.sqrt((p ** 2).sum(1)) for p in pcds]).cpu().numpy()
    start = 0
    for t, p in enumerate(pcds, 1):
        with open(os.path.join(path, f"{sample_idx}_{t}.txt"), "w") as fh:
            fh.writelines("%f\n" % d for d in depth[start:start + p.shape[0]])
        start += p.shape[0]


def summarize_tables(table, num_samples, frames, grid=None):
    """The host end of `evaluate`: `table` [(hi - lo) * frames, 8] float64 (evaluate.FIELDS; row (i - lo) * frames +
    t for sample i, frame t) holds this replica's block [lo, hi) = sharding.shard_range(num_samples, replica, R) of
    the samples.  With a `grid` of more than one rank, the blocks are padded to the longest and all-gathered over
    `grid.world_group` (each replica's block is taken from its shard rank 0).  One host copy; then the first failing
    (sample, frame) in (sample, frame) order raises the exception forward_test raises for it, on every rank, and
    otherwise -> evaluate.summarize of the per-sample ret_dicts (the same sums, in dataset order)."""
    replica, replicas, shard = (grid.replica, grid.replicas, grid.shard_size) if grid is not None else (0, 1, 1)
    blocks = [sharding.shard_range(num_samples, r, replicas) for r in range(replicas)]
    lo, hi = blocks[replica]
    if tuple(table.shape) != ((hi - lo) * frames, eval_metrics.FIELDS):
        raise ValueError(f"summarize_tables: samples [{lo}, {hi}) x {frames} frames need a "
                         f"[{(hi - lo) * frames}, {eval_metrics.FIELDS}] table (got {tuple(table.shape)})")
    if replicas * shard > 1:
        import torch.distributed as dist
        longest = max(b - a for a, b in blocks) * frames
        padded = table.new_zeros((longest, eval_metrics.FIELDS))
        padded[:table.shape[0]] = table
        parts = [torch.empty_like(padded) for _ in range(replicas * shard)]
        dist.all_gather(parts, padded, group=grid.world_group)
        table = torch.cat([parts[r * shard][:(b - a) * frames] for r, (a, b) in enumerate(blocks)])
    host = table.cpu().numpy()
    for i in range(num_samples):
        for t in range(frames):
            eval_metrics.raise_for_flags(host[i * frames + t, 7], f"sample {i}, frame {t}")
    if num_samples == 0:
        return {}
    # one ret_dict summed over the samples in dataset order: the per-sample dicts' sums, as summarize forms them
    return eval_metrics.summarize([eval_metrics.frame_metrics_host(host, num_samples, frames)])
