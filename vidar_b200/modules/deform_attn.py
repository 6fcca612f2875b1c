"""Deformable-attention modules of the BEV encoder / future decoder, host side.

Same registry names, constructor kwargs, parameter names (`sampling_offsets`,
`attention_weights`, `value_proj`, `output_proj`), forward kwargs and numerics as the reference
classes, so the reference's config dicts build them and released checkpoints load:

  MSDeformableAttention3D          spatial_cross_attention.py:177-398
  SpatialCrossAttention            spatial_cross_attention.py:30-174
  TemporalSelfAttention            temporal_self_attention.py:25-271
  PredictionMSDeformableAttention  vidar_decoder.py:289-516
  CustomMSDeformableAttention      decoder.py:132-345   (detection decoder, fine-tuning only)
(paths under projects/mmdet3d_plugin/bevformer/modules/ of the reference).

Every sampling step runs the CUDA op in vidar_b200/csrc/msda.cu: `msda_apply` =
MultiScaleDeformableAttnFunction_fp32.apply around the reference's statements, or by default (`fuse_epilogue`) a
Function that takes the raw offsets / logits and runs the softmax and the sampling-location arithmetic (and
TemporalSelfAttention's queue mean) inside the kernel.  There is no PyTorch fallback branch (the
reference falls back to `multi_scale_deformable_attn_pytorch` on CPU tensors,
spatial_cross_attention.py:392-394): CPU tensors raise.
"""
import math
import warnings

import torch
import torch.nn as nn

from .. import linear as _tc
from ..msda import MSDeformAttn3DFusedFunction, MSDeformAttnQueueFusedFunction, MultiScaleDeformableAttnFunction_fp32
from ..registry import ATTENTION, BaseModule, build_attention, constant_init, xavier_init

msda_apply = MultiScaleDeformableAttnFunction_fp32.apply
msda3d_fused_apply = MSDeformAttn3DFusedFunction.apply
msda_queue_fused_apply = MSDeformAttnQueueFusedFunction.apply


TC_LINEAR = True      # Linear layers of these modules on the tensor cores (3xTF32, vidar_b200/linear.py) when the shape allows


def _linear(layer, x):
    """`layer(x)` for an nn.Linear: the wgmma 3xTF32 kernel (fp32-accurate) for fp32 CUDA inputs whose in / out
    features are multiples of 128 -- value_proj over 6 x 30825 rows is the one large GEMM on the path
    (spatial_cross_attention.py:333) -- otherwise the module itself (cuBLAS)."""
    if TC_LINEAR and layer.bias is not None and _tc.supported(layer.in_features, layer.out_features, x) and x.numel() > 0:
        return _tc.linear_tf32x3(x, layer.weight, layer.bias)
    return layer(x)


def _check_heads(embed_dims, num_heads):
    if embed_dims % num_heads != 0:
        raise ValueError(f"embed_dims must be divisible by num_heads, but got {embed_dims} and {num_heads}")
    d = embed_dims // num_heads
    if not (isinstance(d, int) and d > 0 and (d & (d - 1)) == 0):
        warnings.warn("You'd better set embed_dims in MultiScaleDeformAttention to make the dimension of "
                      "each attention head a power of 2 which is more efficient in our CUDA implementation.")


def _ring_offsets(num_heads, num_groups, num_points):
    """Initial bias of `sampling_offsets`: head h looks along direction 2*pi*h/num_heads
    (normalised to the unit square), point i at radius i+1 -> flat [heads*groups*points*2]
    (spatial_cross_attention.py:255-266, temporal_self_attention.py:108-119)."""
    theta = torch.arange(num_heads, dtype=torch.float32) * (2.0 * math.pi / num_heads)
    d = torch.stack([theta.cos(), theta.sin()], -1)
    d = d / d.abs().max(-1, keepdim=True)[0]
    radius = torch.arange(1, num_points + 1, dtype=torch.float32)
    g = d.view(num_heads, 1, 1, 2) * radius.view(1, 1, num_points, 1)
    return g.expand(num_heads, num_groups, num_points, 2).reshape(-1).clone()


def _queue_fusable(module, value, reference_points, offsets, logits, num_queue):
    """Does TemporalSelfAttention / PredictionMSDeformableAttention take the fused op?  fp32 CUDA tensors outside
    autocast, 2-D reference points and a shape the kernel takes; otherwise (CPU tensors, 4-D box reference points,
    autocast) the reference's statements run around the plain op."""
    if not (module.fuse_epilogue and value.is_cuda and reference_points.shape[-1] == 2
            and not torch.is_autocast_enabled()):
        return False
    if any(t.dtype != torch.float32 for t in (value, reference_points, offsets, logits)):
        return False
    BG, num_value, H, C = value.shape
    if tuple(reference_points.shape) != (BG, offsets.shape[1], module.num_levels, 2):
        return False
    return MSDeformAttnQueueFusedFunction.supported(module.num_levels, module.num_points, num_queue, C, num_value, H)


def _check_num_value(module, spatial_shapes, num_value):
    """The reference's `assert sum(H_l * W_l) == num_value`.  With the fused path enabled and the shapes on the GPU it
    is a device-side assert, so the step never waits for the GPU."""
    if module.fuse_epilogue and spatial_shapes.is_cuda:
        torch._assert_async((spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum() == num_value)
    else:
        assert (spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum() == num_value


def _wh(spatial_shapes):
    """[L,2] (h,w) -> (w,h) normaliser for pixel offsets."""
    return torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)


@ATTENTION.register_module()
class MSDeformableAttention3D(BaseModule):
    """Deformable attention whose reference points are the projections of a BEV pillar's
    Z-anchors into one camera (spatial_cross_attention.py:177-398).  No output projection and
    no residual here -- SpatialCrossAttention owns both."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=8, im2col_step=64,
                 dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__(init_cfg)
        _check_heads(embed_dims, num_heads)
        self.norm_cfg = norm_cfg
        self.batch_first = batch_first
        self.output_proj = None
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.fuse_epilogue = True      # False: materialise sampling_locations / attention_weights like the reference
        self.init_weights()

    def init_weights(self):
        constant_init(self.sampling_offsets, 0.)
        self.sampling_offsets.bias.data = _ring_offsets(self.num_heads, self.num_levels, self.num_points)
        constant_init(self.attention_weights, val=0., bias=0.)
        xavier_init(self.value_proj, distribution="uniform", bias=0.)
        self._is_init = True

    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, **kwargs):
        if value is None:
            value = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, num_query, _ = query.shape
        num_value = value.shape[1]
        assert (spatial_shapes[:, 0] * spatial_shapes[:, 1]).sum() == num_value
        H, L, P = self.num_heads, self.num_levels, self.num_points

        value = _linear(self.value_proj, value)
        if key_padding_mask is not None:
            value = value.masked_fill(key_padding_mask[..., None], 0.0)
        value = value.view(bs, num_value, H, -1)
        offsets = self.sampling_offsets(query).view(bs, num_query, H, L, P, 2)
        logits = self.attention_weights(query).view(bs, num_query, H, L * P)

        if reference_points.shape[-1] != 2:
            raise ValueError(f"Last dim of reference_points must be 2, but get {reference_points.shape[-1]} instead.")
        # point p = j * D + z samples around Z-anchor z  (:356-371)
        D = reference_points.shape[2]
        assert P % D == 0
        if (self.fuse_epilogue and value.is_cuda and value.dtype == torch.float32 and not torch.is_autocast_enabled()
                and MSDeformAttn3DFusedFunction.supported(L, P, value.shape[-1], D)):
            # softmax and the sampling-location arithmetic run inside the kernel (no loc / weights tensors)
            output = msda3d_fused_apply(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
            return output if self.batch_first else output.permute(1, 0, 2)
        weights = logits.softmax(-1).view(bs, num_query, H, L, P)
        offsets = offsets / _wh(spatial_shapes)[None, None, None, :, None, :]
        loc = offsets.view(bs, num_query, H, L, P // D, D, 2) + reference_points[:, :, None, None, None, :, :]
        loc = loc.view(bs, num_query, H, L, P, 2)

        output = msda_apply(value, spatial_shapes, level_start_index, loc, weights, self.im2col_step)
        if not self.batch_first:
            output = output.permute(1, 0, 2)
        return output


def _visible_lists(bev_mask):
    """Per-camera lists of visible pillars (batch element 0, spatial_cross_attention.py:136-140) as
    (idx [cams, max_len] ascending pillar indices padded with invisible ones, live [cams, max_len]
    bool, max_len) for the REBATCH path below (the reference's own data flow): one batched stable sort
    instead of six `nonzero()` calls, and -- like the reference -- one host sync for max_len.  The
    default (fused) path of SpatialCrossAttention needs neither the padding nor the sync."""
    hit = bev_mask[:, 0].sum(-1) > 0                                     # [cams, Q]
    counts = hit.sum(-1)
    max_len = int(counts.max())
    order = torch.argsort((~hit).to(torch.uint8), dim=1, stable=True)    # visible first, ascending
    idx = order[:, :max_len].contiguous()
    live = torch.arange(max_len, device=bev_mask.device)[None, :] < counts[:, None]
    return idx, live, max_len


@ATTENTION.register_module()
class SpatialCrossAttention(BaseModule):
    """BEV query -> 6 camera feature pyramids (spatial_cross_attention.py:30-174): each camera
    attends only with the BEV pillars it sees, results are averaged over the cameras that
    see a pillar, projected, and added to the residual.

    Default data flow (`fuse_rebatch`, SURVEY.md 8f-1): device-side visible lists, the sampling
    offsets / attention logits computed once per pillar, and ONE kernel per direction that samples
    every (camera, visible pillar) row and reduces it straight into the BEV slots
    (vidar_b200/sca.py) -- no host sync, no [cams, max_len, C] buffers, no index_add_.
    `process_group` (see `set_process_group`): the cameras are sharded over its ranks (SURVEY.md
    8e); each rank projects and samples only its cameras, the partial slot grids are
    reduce-scattered into row blocks, `output_proj` runs on the rank's rows and ONE all-gather
    returns the replicated BEV grid."""

    def __init__(self, embed_dims=256, num_cams=6, pc_range=None, dropout=0.1, init_cfg=None,
                 batch_first=False,
                 deformable_attention=dict(type="MSDeformableAttention3D", embed_dims=256, num_levels=4),
                 **kwargs):
        super().__init__(init_cfg)
        self.init_cfg = init_cfg
        self.dropout = nn.Dropout(dropout)
        self.pc_range = pc_range
        self.fp16_enabled = False
        self.deformable_attention = build_attention(deformable_attention)
        self.embed_dims = embed_dims
        self.num_cams = num_cams
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.batch_first = batch_first
        self.fuse_rebatch = True       # False: the reference's rebatch / index_add_ data flow
        self.process_group = None
        self.init_weight()

    def init_weight(self):
        xavier_init(self.output_proj, distribution="uniform", bias=0.)

    def set_process_group(self, group):
        """Shard the cameras over `group` (None: single GPU).  `value_proj` then sees only this rank's
        cameras, `output_proj` only its rows and the offsets / logits Linears only the gradient of this
        rank's cameras: their parameter gradients are per-rank partial sums, tagged for
        `sharding.allreduce_partial_grads` (one bucketed all-reduce per step)."""
        self.process_group = group
        partial = group is not None
        da = self.deformable_attention
        for m in (self.output_proj, getattr(da, "value_proj", None), getattr(da, "sampling_offsets", None),
                  getattr(da, "attention_weights", None)):
            if m is not None:
                for p_ in m.parameters():
                    p_.vidar_partial_grad = partial
        return self

    def _world(self):
        g = self.process_group
        if g is None:
            return 1, 0
        import torch.distributed as dist
        if not dist.is_initialized():
            return 1, 0
        return dist.get_world_size(g), dist.get_rank(g)

    def _fusable(self, query, value, reference_points_cam):
        da = self.deformable_attention
        if not (self.fuse_rebatch and isinstance(da, MSDeformableAttention3D) and da.batch_first):
            return False
        if not (query.is_cuda and query.dtype == torch.float32 and value.dtype == torch.float32
                and not torch.is_autocast_enabled()):
            return False
        D = reference_points_cam.size(3)
        return MSDeformAttn3DFusedFunction.supported(da.num_levels, da.num_points, da.embed_dims // da.num_heads, D)

    def forward(self, query, key, value, residual=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, reference_points_cam=None,
                bev_mask=None, level_start_index=None, flag="encoder", rows_out=False, summed_query_grad=False,
                **kwargs):
        """Sharded extras (not in the reference): `rows_out=True` returns only this rank's block of BEV rows
        (`sharding.row_range` of the bs*Q flattened rows; `residual` must then hold those rows) and skips the
        all-gather -- for row-wise consumers (LayerNorm, FFN, `LatentRendering.forward_rows`);
        `summed_query_grad=True` says the caller already sums the query's per-rank partial gradient (it came out of
        `sharding.all_gather_rows(..., grad="sum")`), so no all-reduce is added here."""
        if key is None:
            key = query
        if value is None:
            value = key
        world, _ = self._world()
        if rows_out and (world == 1 or residual is None):
            raise RuntimeError("rows_out needs a process group with more than one rank and the residual rows")
        inp_residual = query if residual is None else residual
        if query_pos is not None:
            query = query + query_pos
        if world > 1 and not summed_query_grad:
            # every rank samples only its cameras: the gradient that reaches the (replicated) query through
            # offsets / logits is a per-rank partial sum -> one all-reduce of the 41 MB BEV-query gradient
            from .. import sharding
            query = sharding.sum_grad(query, self.process_group)
        if self._fusable(query, value, reference_points_cam):
            slots = self._slots_fused(query, value, reference_points_cam, bev_mask, spatial_shapes, level_start_index)
        else:
            if self._world()[0] > 1:
                raise RuntimeError("camera sharding needs the fused SpatialCrossAttention path "
                                   "(MSDeformableAttention3D with num_levels * num_points == 32, fp32, CUDA)")
            slots = self._slots_rebatch(query, key, value, reference_points_cam, bev_mask, spatial_shapes, level_start_index)
        if world > 1:
            from .. import sharding
            bs, Q, C = slots.shape
            rows = sharding.reduce_scatter_rows(slots.reshape(bs * Q, C), self.process_group)     # this rank's pillars
            rows = self.dropout(_linear(self.output_proj, rows))
            if rows_out:
                return rows + inp_residual.reshape(-1, C)
            full = sharding.all_gather_rows(rows, bs * Q, self.process_group).view(bs, Q, C)       # the BEV grid
            return full + inp_residual          # the residual stays replicated (its gradient is the full one)
        return self.dropout(_linear(self.output_proj, slots)) + inp_residual

    # ---- default: rows sampled and reduced into the slots by one kernel (no rebatch tensors)
    def _slots_fused(self, query, value, reference_points_cam, bev_mask, spatial_shapes, level_start_index):
        from .. import sca
        da = self.deformable_attention
        bs, Q, C = query.shape
        cams, K = value.shape[0], value.shape[1]
        H, L, P = da.num_heads, da.num_levels, da.num_points
        idx, count, inv = sca.compact_visible(bev_mask)
        world, rank = self._world()
        # Linear(query) rows are the same for every camera that sees the pillar: once per pillar
        offsets = _linear(da.sampling_offsets, query).view(bs, Q, H, L, P, 2)
        logits = _linear(da.attention_weights, query).view(bs, Q, H, L * P)
        plan = sca.unit_plan(world, rank, cams)
        values = []
        for cam0, ncl, _, _, _ in plan:
            v = value[cam0:cam0 + ncl].permute(2, 0, 1, 3).reshape(bs * ncl, K, C)      # [bs*ncl, K, C], batch-major
            values.append(_linear(da.value_proj, v).view(bs * ncl, K, H, C // H))
        return sca.SCARowsFunction.apply(plan, bs, spatial_shapes, level_start_index, reference_points_cam,
                                         offsets, logits, idx, count, inv, *values)

    # ---- the reference's data flow (:135-172) on the CUDA op: any deformable_attention module
    def _slots_rebatch(self, query, key, value, reference_points_cam, bev_mask, spatial_shapes, level_start_index):
        bs, num_query, C = query.shape
        cams, D = self.num_cams, reference_points_cam.size(3)
        # visible-pillar lists per camera, taken from batch element 0 like the reference (:136-140)
        idx, live, max_len = _visible_lists(bev_mask)

        # rebatch (:143-152): padded rows are zeros
        q_re = query[:, idx] * live[None, :, :, None].to(query.dtype)        # [bs, cams, max_len, C]
        cam_ix = torch.arange(cams, device=query.device)[:, None]
        r_re = reference_points_cam[cam_ix, :, idx]                          # [cams, max_len, bs, D, 2]
        r_re = r_re.permute(2, 0, 1, 3, 4) * live[None, :, :, None, None].to(r_re.dtype)

        l = key.shape[1]
        key = key.permute(2, 0, 1, 3).reshape(bs * cams, l, self.embed_dims)
        value = value.permute(2, 0, 1, 3).reshape(bs * cams, l, self.embed_dims)
        out = self.deformable_attention(
            query=q_re.reshape(bs * cams, max_len, self.embed_dims), key=key, value=value,
            reference_points=r_re.reshape(bs * cams, max_len, D, 2), spatial_shapes=spatial_shapes,
            level_start_index=level_start_index).view(bs, cams, max_len, self.embed_dims)

        # scatter-add back (:164-166); padded rows carry zeros so their target index is irrelevant
        out = out * live[None, :, :, None].to(out.dtype)
        slots = torch.zeros_like(query)
        slots.index_add_(1, idx.reshape(-1), out.reshape(bs, cams * max_len, self.embed_dims))

        count = (bev_mask.sum(-1) > 0).permute(1, 2, 0).sum(-1)              # [bs, Q] cameras seeing it
        return slots / torch.clamp(count, min=1.0)[..., None]


@ATTENTION.register_module()
class TemporalSelfAttention(BaseModule):
    """BEV self-attention over [previous BEV, current BEV] (temporal_self_attention.py:25-271):
    offsets/weights are predicted from concat(prev, cur), each queue element is sampled
    separately (batch = bs * num_bev_queue) and the two results are averaged."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, num_bev_queue=2,
                 im2col_step=64, dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__(init_cfg)
        _check_heads(embed_dims, num_heads)
        self.norm_cfg = norm_cfg
        self.dropout = nn.Dropout(dropout)
        self.batch_first = batch_first
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.num_bev_queue = num_bev_queue
        self.sampling_offsets = nn.Linear(embed_dims * num_bev_queue,
                                          num_bev_queue * num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims * num_bev_queue,
                                           num_bev_queue * num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.fuse_epilogue = True      # False: materialise sampling_locations / attention_weights like the reference
        self.init_weights()

    def init_weights(self):
        constant_init(self.sampling_offsets, 0.)
        self.sampling_offsets.bias.data = _ring_offsets(
            self.num_heads, self.num_levels * self.num_bev_queue, self.num_points)
        constant_init(self.attention_weights, val=0., bias=0.)
        xavier_init(self.value_proj, distribution="uniform", bias=0.)
        xavier_init(self.output_proj, distribution="uniform", bias=0.)
        self._is_init = True

    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, flag="decoder", row_range=None, **kwargs):
        """`row_range=(lo, hi)` (not in the reference; SURVEY.md 8e "TSA shards by query rows with the value
        replicated"): `query`, `identity`, `query_pos` and `reference_points` hold only BEV rows lo..hi-1, `value`
        is the full [bs*2, num_value, C] stack; the result is those rows of the full call."""
        if row_range is not None and (value is None or not self.batch_first):
            raise RuntimeError("row_range needs batch_first=True and an explicit full `value` stack")
        if value is None:
            assert self.batch_first
            bs, len_bev, c = query.shape
            value = torch.stack([query, query], 1).reshape(bs * 2, len_bev, c)
        if identity is None:
            identity = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, num_query, embed_dims = query.shape
        num_value = value.shape[1]
        _check_num_value(self, spatial_shapes, num_value)
        assert self.num_bev_queue == 2
        H, L, P, Qn = self.num_heads, self.num_levels, self.num_points, self.num_bev_queue

        prev_rows = value[:bs] if row_range is None else value[:bs, row_range[0]:row_range[1]]
        if prev_rows.shape[1] != num_query:
            raise RuntimeError(f"{num_query} query rows but {prev_rows.shape[1]} rows of the previous BEV (row_range={row_range})")
        query = torch.cat([prev_rows, query], -1)
        value = _linear(self.value_proj, value)
        if key_padding_mask is not None:
            value = value.masked_fill(key_padding_mask[..., None], 0.0)
        value = value.reshape(bs * Qn, num_value, H, -1)

        offsets = self.sampling_offsets(query).view(bs, num_query, H, Qn, L, P, 2)
        logits = self.attention_weights(query).view(bs, num_query, H, Qn, L * P)
        if _queue_fusable(self, value, reference_points, offsets, logits, Qn):
            # softmax, sampling locations and the mean over the queue run inside the kernel
            output = msda_queue_fused_apply(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        else:
            output = self._sample(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        output = _linear(self.output_proj, output)
        if not self.batch_first:
            output = output.permute(1, 0, 2)
        return self.dropout(output) + identity

    def _sample(self, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        """The reference's statements around the plain op (temporal_self_attention.py:196-261) -> [bs, nq, C]."""
        bs, num_query, H, Qn, L, P, _ = offsets.shape
        weights = logits.softmax(-1).view(bs, num_query, H, Qn, L, P)
        # queue axis next to batch: [bs*Qn, num_query, H, L, P(,2)]
        weights = weights.permute(0, 3, 1, 2, 4, 5).reshape(bs * Qn, num_query, H, L, P).contiguous()
        offsets = offsets.permute(0, 3, 1, 2, 4, 5, 6).reshape(bs * Qn, num_query, H, L, P, 2)

        if reference_points.shape[-1] == 2:
            loc = reference_points[:, :, None, :, None, :] + offsets / _wh(spatial_shapes)[None, None, None, :, None, :]
        elif reference_points.shape[-1] == 4:
            loc = (reference_points[:, :, None, :, None, :2]
                   + offsets / P * reference_points[:, :, None, :, None, 2:] * 0.5)
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} instead.")

        output = msda_apply(value, spatial_shapes, level_start_index, loc, weights, self.im2col_step)
        # mean over the queue (:255-261): [bs*Qn, nq, C] -> [bs, nq, C]
        return output.view(bs, Qn, num_query, -1).mean(1)


@ATTENTION.register_module()
class PredictionMSDeformableAttention(BaseModule):
    """Deformable attention of the future-BEV decoder (vidar_decoder.py:289-516): self-attention
    on the query BEV or cross-attention to the stacked history BEVs (one 'level' per frame)."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64,
                 dropout=0.1, batch_first=True, norm_cfg=None, init_cfg=None):
        super().__init__(init_cfg)
        _check_heads(embed_dims, num_heads)
        self.norm_cfg = norm_cfg
        self.dropout = nn.Dropout(dropout)
        self.batch_first = batch_first
        self.fp16_enabled = False
        self.im2col_step = im2col_step
        self.embed_dims = embed_dims
        self.num_levels = num_levels
        self.num_heads = num_heads
        self.num_points = num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.fuse_epilogue = True      # False: materialise sampling_locations / attention_weights like the reference
        self.init_weights()

    def init_weights(self):
        constant_init(self.sampling_offsets, 0.)
        self.sampling_offsets.bias.data = _ring_offsets(self.num_heads, self.num_levels, self.num_points)
        constant_init(self.attention_weights, val=0., bias=0.)
        xavier_init(self.value_proj, distribution="uniform", bias=0.)
        xavier_init(self.output_proj, distribution="uniform", bias=0.)
        self._is_init = True

    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, flag="decoder", **kwargs):
        if value is None:
            value = query
        if identity is None:
            identity = query
        if query_pos is not None:
            query = query + query_pos
        bs, num_query, _ = query.shape
        num_value = value.shape[1]
        _check_num_value(self, spatial_shapes, num_value)
        H, L, P = self.num_heads, self.num_levels, self.num_points

        value = _linear(self.value_proj, value)
        if key_padding_mask is not None:
            value = value.masked_fill(key_padding_mask[..., None], 0.0)
        value = value.view(bs, num_value, H, -1)
        offsets = self.sampling_offsets(query).view(bs, num_query, H, L, P, 2)
        logits = self.attention_weights(query).view(bs, num_query, H, L * P)
        if _queue_fusable(self, value, reference_points, offsets, logits, 1):
            # softmax and the sampling-location arithmetic run inside the kernel
            output = msda_queue_fused_apply(value, spatial_shapes, level_start_index, reference_points,
                                            offsets.view(bs, num_query, H, 1, L, P, 2),
                                            logits.view(bs, num_query, H, 1, L * P))
        else:
            output = self._sample(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        output = _linear(self.output_proj, output)
        if not self.batch_first:
            output = output.permute(1, 0, 2)
        return self.dropout(output) + identity

    def _sample(self, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        """The reference's statements around the plain op (vidar_decoder.py:466-506) -> [bs, nq, C]."""
        bs, num_query, H, L, P, _ = offsets.shape
        weights = logits.softmax(-1).view(bs, num_query, H, L, P)
        if reference_points.shape[-1] == 2:
            loc = reference_points[:, :, None, :, None, :] + offsets / _wh(spatial_shapes)[None, None, None, :, None, :]
        elif reference_points.shape[-1] == 4:
            loc = (reference_points[:, :, None, :, None, :2]
                   + offsets / P * reference_points[:, :, None, :, None, 2:] * 0.5)
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} instead.")
        return msda_apply(value, spatial_shapes, level_start_index, loc, weights, self.im2col_step)


@ATTENTION.register_module()
class CustomMSDeformableAttention(PredictionMSDeformableAttention):
    """Deformable attention of the detection decoder (decoder.py:132-345): 900 object queries on
    the single 200x200 BEV level.  Same parameters and arithmetic as the prediction variant; the
    difference is the sequence-first default layout -- query `[num_query, bs, C]`, value
    `[num_key, bs, C]` are permuted to batch-first before the projections (decoder.py:279-282) and
    the output is permuted back (:340-343).  `identity` stays in the caller's layout."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64,
                 dropout=0.1, batch_first=False, norm_cfg=None, init_cfg=None):
        super().__init__(embed_dims, num_heads, num_levels, num_points, im2col_step, dropout,
                         batch_first, norm_cfg, init_cfg)

    def forward(self, query, key=None, value=None, identity=None, query_pos=None,
                key_padding_mask=None, reference_points=None, spatial_shapes=None,
                level_start_index=None, flag="decoder", **kwargs):
        if value is None:
            value = query
        if identity is None:
            identity = query
        if query_pos is not None:
            query = query + query_pos
            query_pos = None
        if not self.batch_first:
            query = query.permute(1, 0, 2)
            value = value.permute(1, 0, 2)
        # the parent adds `dropout(out) + identity` after permuting the output back
        return super().forward(query, key, value, identity, query_pos, key_padding_mask, reference_points,
                               spatial_shapes, level_start_index, flag, **kwargs)
