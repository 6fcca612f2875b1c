"""SpatialCrossAttention's data movement, fused into the deformable-attention op.

The reference (spatial_cross_attention.py:135-172) finds each camera's visible pillars with
`nonzero()` (a host sync), copies queries / reference points into `[bs, cams, max_len, .]` buffers,
runs MSDeformableAttention3D on the padded rows, then loops over (batch, camera) adding the rows
back into `slots` and divides by the number of cameras that see a pillar.  Here:

  * `compact_visible`   one kernel builds the per-camera ascending pillar lists, their lengths and
                        1 / #cameras on the device -- no host sync, no max_len;
  * `SCARowsFunction`   MSDeformableAttention3D's sampling on those rows with offsets / logits read
                        through the list (they are Linear(query) rows, identical for every camera that
                        sees the pillar, so they are computed ONCE per pillar instead of once per
                        (camera, pillar)), the softmax / sampling-location prologue in the kernel and the
                        scatter-add + count normalisation as the epilogue: head vectors are reduced
                        straight into the BEV slot grid (`red.global.add.v4.f32`);
  * `MSDARowsFunction`  the same row map around the plain op (sampling locations / weights given per
                        row) -- the cfg2 benchmark shape;
  * `unit_plan`         which (camera, row sub-slice) units a rank owns when the cameras are sharded
                        over a process group (SURVEY.md 8e), balanced whatever the list lengths are.

Kernels: vidar_b200/csrc/msda.cu (IDX instantiations), csrc/sca_glue.cu (compaction).
"""
import math

import torch
from torch.autograd.function import Function, once_differentiable

from . import _lib

SLICE_ROWS = 64     # granularity of the interleaved row sub-slices (msda.cu: (j / 64) % S)


def compact_visible(bev_mask):
    """bev_mask [cams, bs, Q, D] (bool / uint8, CUDA) ->
         idx   [cams, Q] int32  ascending pillar indices seen by the camera in batch element 0
                                (spatial_cross_attention.py:136-140), entries >= count undefined
         count [cams]    int32  list lengths (stays on the device)
         inv   [bs, Q]   f32    1 / clamp(#cameras whose mask hits the pillar, 1)   (:168-171)"""
    if bev_mask.dim() != 4:
        raise RuntimeError(f"bev_mask must be [num_cams, bs, num_query, D], got {tuple(bev_mask.shape)}")
    m = bev_mask.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    elif m.dtype != torch.uint8:
        m = (m != 0).view(torch.uint8)
    _lib.require_cuda(bev_mask=m)
    cams, bs, Q, D = m.shape
    idx = torch.empty((cams, Q), dtype=torch.int32, device=m.device)
    count = torch.empty((cams,), dtype=torch.int32, device=m.device)
    inv = torch.empty((bs, Q), dtype=torch.float32, device=m.device)
    with torch.cuda.device(m.device):
        _lib.check(_lib.lib().vidar_sca_compact(_lib.ptr(m), _lib.ptr(idx), _lib.ptr(count), _lib.ptr(inv),
                                                cams, bs, Q, D, _lib.stream_ptr(m.device)))
    return idx, count, inv


def unit_plan(world, rank, cams):
    """Launch groups of `rank` when `cams` cameras are sharded over `world` ranks:
    [(cam0, ncl, S, s_lo, s_hi), ...] -- cameras cam0 .. cam0+ncl-1, rows with (j // 64) % S in
    [s_lo, s_hi).  A camera is cut into S = world / gcd(cams, world) interleaved sub-slices so that
    cams * S units divide evenly; a rank owns consecutive units, i.e. at most two partial cameras.
    Interleaving (not contiguous ranges) keeps the shares equal for any visible-list length."""
    if world <= 1:
        return [(0, cams, 1, 0, 1)]
    S = world // math.gcd(cams, world)
    per = cams * S // world
    lo, hi = rank * per, (rank + 1) * per
    groups = []
    u = lo
    while u < hi:
        cam, s = divmod(u, S)
        e = min(hi, (cam + 1) * S)
        groups.append([cam, 1, S, s, s + (e - u)])
        u = e
    # merge whole consecutive cameras into one launch
    merged = []
    for g in groups:
        if merged and g[3] == 0 and g[4] == S and merged[-1][3] == 0 and merged[-1][4] == S \
                and merged[-1][0] + merged[-1][1] == g[0]:
            merged[-1][1] += 1
        else:
            merged.append(g)
    return [tuple(g) for g in merged]


def plan_cameras(plan):
    """Cameras touched by a plan, ascending."""
    return sorted({c for cam0, ncl, _, _, _ in plan for c in range(cam0, cam0 + ncl)})


def _check_common(values, plan, idx, count, inv):
    if len(values) != len(plan):
        raise RuntimeError(f"{len(plan)} launch groups but {len(values)} value tensors")
    for t, name in ((idx, "idx"), (count, "count")):
        if t is not None and (t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous()):
            raise RuntimeError(f"{name} must be a contiguous CUDA int32 tensor")
    if inv is not None and (inv.dtype != torch.float32 or not inv.is_cuda or not inv.is_contiguous()):
        raise RuntimeError("inv_count must be a contiguous CUDA float32 tensor")


class SCARowsFunction(Function):
    """apply(plan, bs, spatial_shapes, level_start_index, ref_cam [cams,bs,Q,D,2],
             offsets [bs,Q,H,L,P,2], logits [bs,Q,H,L*P], idx, count, inv, *values) -> slots [bs,Q,H*C]

    values[g]: [bs*ncl_g, K, H, C] projected image features of launch group g (batch-major:
    n = b*ncl + camera).  The returned slots hold this rank's share of
    sum_cameras MSDeformableAttention3D(...) / #cameras, i.e. SpatialCrossAttention's `slots` before
    `output_proj` (spatial_cross_attention.py:164-171); with a one-group plan over all cameras it is
    the whole thing.  Gradients: offsets, logits (dense, summed over cameras) and every value."""

    @staticmethod
    def forward(ctx, plan, bs, spatial_shapes, level_start_index, ref_cam, offsets, logits, idx, count, inv, *values):
        values = [_lib.aligned(v.float().contiguous()) for v in values]
        ref_cam = _lib.aligned(ref_cam.float().contiguous())
        offsets = _lib.aligned(offsets.float().contiguous())
        logits = _lib.aligned(logits.float().contiguous())
        spatial_shapes = spatial_shapes.contiguous()
        level_start_index = level_start_index.contiguous()
        _check_common(values, plan, idx, count, inv)
        _lib.require_cuda(ref_cam=ref_cam, offsets=offsets, logits=logits, spatial_shapes=spatial_shapes,
                          level_start_index=level_start_index, **{f"value{i}": v for i, v in enumerate(values)})
        if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
            raise RuntimeError("spatial_shapes / level_start_index must be int64 tensors")
        if ref_cam.dim() != 5 or ref_cam.shape[1] != bs or ref_cam.shape[-1] != 2:
            raise RuntimeError(f"reference_points_cam must be [num_cams, bs, num_query, D, 2], got {tuple(ref_cam.shape)}")
        cams, _, Qd, D, _ = ref_cam.shape
        L = spatial_shapes.shape[0]
        _, K, H, C = values[0].shape
        if offsets.numel() % (bs * Qd * H * L * 2):
            raise RuntimeError("offsets must be [bs, num_query, num_heads, num_levels, num_points, 2]")
        P = offsets.numel() // (bs * Qd * H * L * 2)
        if logits.numel() != bs * Qd * H * L * P:
            raise RuntimeError("logits must be [bs, num_query, num_heads, num_levels * num_points]")
        if idx is not None and tuple(idx.shape) != (cams, Qd):
            raise RuntimeError(f"idx must be [num_cams, num_query] = {(cams, Qd)}, got {tuple(idx.shape)}")
        slots = torch.zeros((bs, Qd, H * C), dtype=torch.float32, device=offsets.device)
        L_ = _lib.lib()
        with torch.cuda.device(offsets.device):
            st = _lib.stream_ptr(offsets.device)
            for (cam0, ncl, S, lo, hi), v in zip(plan, values):
                if tuple(v.shape) != (bs * ncl, K, H, C):
                    raise RuntimeError(f"value of cameras {cam0}..{cam0 + ncl - 1} must be {(bs * ncl, K, H, C)}, got {tuple(v.shape)}")
                _lib.check(L_.vidar_msda_sca_rows_forward(
                    _lib.ptr(v), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref_cam), _lib.ptr(offsets),
                    _lib.ptr(logits), _lib.ptr(idx), _lib.ptr(count), _lib.ptr(inv), _lib.ptr(slots), bs, ncl, cam0, K, H, C,
                    L, Qd, Qd, P, D, S, lo, hi, st))
        ctx.save_for_backward(spatial_shapes, level_start_index, ref_cam, offsets, logits, idx, count, inv, *values)
        ctx.meta = (plan, bs, K, H, C, L, Qd, P, D)
        return slots

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_slots):
        spatial_shapes, level_start_index, ref_cam, offsets, logits, idx, count, inv, *values = ctx.saved_tensors
        plan, bs, K, H, C, L, Qd, P, D = ctx.meta
        g = _lib.aligned(grad_slots.float().contiguous())
        grad_offsets = torch.zeros_like(offsets)
        grad_logits = torch.zeros_like(logits)
        gvs = []
        L_ = _lib.lib()
        with torch.cuda.device(offsets.device):
            st = _lib.stream_ptr(offsets.device)
            for (cam0, ncl, S, lo, hi), v in zip(plan, values):
                gv = torch.zeros_like(v)
                _lib.check(L_.vidar_msda_sca_rows_backward(
                    _lib.ptr(v), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref_cam), _lib.ptr(offsets),
                    _lib.ptr(logits), _lib.ptr(idx), _lib.ptr(count), _lib.ptr(inv), _lib.ptr(g), _lib.ptr(gv),
                    _lib.ptr(grad_offsets), _lib.ptr(grad_logits), bs, ncl, cam0, K, H, C, L, Qd, Qd, P, D, S, lo, hi, st))
                gvs.append(gv)
        return (None, None, None, None, None, grad_offsets, grad_logits, None, None, None, *gvs)


class MSDARowsFunction(Function):
    """The plain op behind the same row map: apply(plan, bs, num_pillars, spatial_shapes,
    level_start_index, idx | None, count | None, inv | None, *[value_g, loc_g, attn_g ...]) -> slots.

    value_g [bs*ncl, K, H, C], loc_g [bs*ncl, rows, H, L, P, 2], attn_g [bs*ncl, rows, H, L, P]:
    `ms_deform_attn_forward` on the rows of launch group g with its output rows added into
    slots[b, idx[cam, j]] (scaled by inv) instead of being written to a [bs*ncl, rows, H*C] tensor;
    backward reads the slot gradient back through the map.  idx None: row j is pillar j."""

    @staticmethod
    def forward(ctx, plan, bs, Qd, spatial_shapes, level_start_index, idx, count, inv, *tensors):
        if len(tensors) != 3 * len(plan):
            raise RuntimeError("expected (value, sampling_locations, attention_weights) per launch group")
        tensors = [_lib.aligned(t.float().contiguous()) for t in tensors]
        values, locs, attns = tensors[0::3], tensors[1::3], tensors[2::3]
        _check_common(values, plan, idx, count, inv)
        spatial_shapes = spatial_shapes.contiguous()
        level_start_index = level_start_index.contiguous()
        _lib.require_cuda(spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                          **{f"tensor{i}": t for i, t in enumerate(tensors)})
        if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
            raise RuntimeError("spatial_shapes / level_start_index must be int64 tensors")
        _, K, H, C = values[0].shape
        L, P = locs[0].shape[3], locs[0].shape[4]
        slots = torch.zeros((bs, Qd, H * C), dtype=torch.float32, device=values[0].device)
        L_ = _lib.lib()
        with torch.cuda.device(slots.device):
            st = _lib.stream_ptr(slots.device)
            for (cam0, ncl, S, lo, hi), v, loc, aw in zip(plan, values, locs, attns):
                rows = loc.shape[1]
                if tuple(v.shape) != (bs * ncl, K, H, C) or tuple(loc.shape) != (bs * ncl, rows, H, L, P, 2) \
                        or tuple(aw.shape) != (bs * ncl, rows, H, L, P):
                    raise RuntimeError("value / sampling_locations / attention_weights shapes do not match the launch group")
                _lib.check(L_.vidar_msda_rows_forward(
                    _lib.ptr(v), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(loc), _lib.ptr(aw),
                    _lib.ptr(idx), _lib.ptr(count), _lib.ptr(inv), _lib.ptr(slots), bs, ncl, cam0, K, H, C, L, rows, Qd, P,
                    S, lo, hi, st))
        ctx.save_for_backward(spatial_shapes, level_start_index, idx, count, inv, *tensors)
        ctx.meta = (plan, bs, Qd, K, H, C, L, P)
        return slots

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_slots):
        spatial_shapes, level_start_index, idx, count, inv, *tensors = ctx.saved_tensors
        plan, bs, Qd, K, H, C, L, P = ctx.meta
        values, locs, attns = tensors[0::3], tensors[1::3], tensors[2::3]
        g = _lib.aligned(grad_slots.float().contiguous())
        grads = []
        L_ = _lib.lib()
        with torch.cuda.device(g.device):
            st = _lib.stream_ptr(g.device)
            for (cam0, ncl, S, lo, hi), v, loc, aw in zip(plan, values, locs, attns):
                gv = torch.zeros_like(v)
                # rows outside this launch's share (dead rows, other ranks' sub-slices) receive no gradient
                partial = count is not None or S > 1
                gl = torch.zeros_like(loc) if partial else torch.empty_like(loc)
                ga = torch.zeros_like(aw) if partial else torch.empty_like(aw)
                _lib.check(L_.vidar_msda_rows_backward(
                    _lib.ptr(v), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(loc), _lib.ptr(aw),
                    _lib.ptr(idx), _lib.ptr(count), _lib.ptr(inv), _lib.ptr(g), _lib.ptr(gv), _lib.ptr(gl), _lib.ptr(ga),
                    bs, ncl, cam0, K, H, C, L, loc.shape[1], Qd, P, S, lo, hi, st))
                grads += [gv, gl, ga]
        return (None, None, None, None, None, None, None, None, *grads)


def camera_ranks(world, cams):
    """{camera: [ranks that own units of it]} under `unit_plan`."""
    owners = {c: [] for c in range(cams)}
    for r in range(world):
        for c in plan_cameras(unit_plan(world, r, cams)):
            owners[c].append(r)
    return owners


def camera_groups(world, cams, rank, group=None):
    """Process groups of the cameras whose units are split over several ranks: the partial `grad_value`
    of such a camera is summed inside its group (its image features live on every rank of the group).
    EVERY rank must call this (new_group is collective).  `world` / `rank`: size of and rank in the shard group
    `group` (None: the whole world).  The camera groups of every shard group are made on every rank, in one order,
    from global ranks (`sharding.shard_layouts`).  -> {camera: group} for this rank's shared cameras."""
    import torch.distributed as dist

    from .sharding import shard_layouts
    layouts, mine = shard_layouts(group, world)
    shared = [(c, members) for c, members in camera_ranks(world, cams).items() if len(members) > 1]
    groups = {}
    for ranks in layouts:
        for c, members in shared:
            g = dist.new_group([ranks[m] for m in members])
            if ranks == mine and rank in members:
                groups[c] = g
    return groups
