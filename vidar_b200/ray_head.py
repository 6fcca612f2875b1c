"""ViDAR head ray operations on the GPU kernels of vidar_b200/csrc/ray_head.cu.

Host-side mirror of the ray part of
projects/mmdet3d_plugin/bevformer/dense_heads/vidar_head_base.py:

  get_grid_features(...)      == ViDARHeadBase._get_grid_features (:420-509): same arguments
                                 (plus ray_grid_num, an attribute of the head), same four
                                 returned tensors, same ray order and dropping rule;
  ce_regularization_loss(...) == the `use_ce_loss` branch of ViDARHeadBase.loss (:586-592),
                                 computed by the FUSED sampler+cross-entropy kernels: the
                                 [lvl, R, 513] logits are never materialised;
  decode_ray_depth(...)       == the per-(batch, frame) body of get_point_cloud_prediction
                                 (:706-738): arg-max waypoint -> distance;
  dense_chamfer_loss(...)     == the Chamfer loop of the `use_dense_loss` branch of ViDARHeadBase.loss
                                 (:638-659) over every (sample, frame) pair in one batched op, no host
                                 sync: dense_chamfer_group_loss with pair n = b*F + f and one group;
  dense_chamfer_group_loss(...) == the same Chamfer term over a pair table (csrc/dense_chamfer.cu), one
                                 loss per group (ViDARHeadV1: a group per head frame);
  align_gt(...)               == ViDARHeadV1._get_reference_gt_points (vidar_head_v1.py:94-148) for every
                                 (head frame, target frame) job in one op;
  decode_clouds(...)          == get_point_cloud_prediction's rendering of the decoded rays (:698-745,
                                 get_rendered_pcds :363-389) for every (sample, frame) at once, as flat
                                 clouds with device offsets (csrc/eval_metrics.cu), no host sync.

Low-level autograd ops: `ray_sample` (logits/lengths, differentiable w.r.t. sigma) and `ray_ce`.
All tensors must be CUDA; there is no PyTorch fallback.
"""
import ctypes as C
import functools

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib


def _prep(sigma, origin, points, frame):
    _lib.require_cuda(sigma=sigma, origin=origin, points=points, frame=frame)
    if sigma.dim() != 4 or origin.dim() != 2 or points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("expected sigma [F,Z,Y,X], origin [F,3], points [R,3]")
    if sigma.dtype != torch.float32 or origin.dtype != torch.float32 or points.dtype != torch.float32:
        raise RuntimeError("sigma / origin / points must be float32")
    F, Z, Y, X = sigma.shape
    if origin.shape[0] != F:
        raise RuntimeError("origin must hold one row per frame of sigma")
    if frame is not None and (frame.dtype != torch.int32 or frame.shape != (points.shape[0],)):
        raise RuntimeError("frame must be int32 [R]")
    return points.shape[0], F, Z, Y, X


def _call(fn, device, *args):
    with torch.cuda.device(device):
        _lib.check(fn(*args, _lib.stream_ptr(device)))


class _RaySample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sigma, origin, points, frame, num_way, step, with_gt):
        sigma = sigma.contiguous()
        R, F, Z, Y, X = _prep(sigma, origin, points, frame)
        K = num_way + int(with_gt)
        logits = torch.empty((R, K), dtype=torch.float32, device=sigma.device)
        length = torch.empty((R, K), dtype=torch.float32, device=sigma.device)
        valid = torch.empty((R,), dtype=torch.float32, device=sigma.device)
        if R:
            _call(_lib.lib().vidar_ray_sample, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
                  _lib.ptr(points), _lib.ptr(frame), _lib.ptr(logits), _lib.ptr(length),
                  _lib.ptr(valid), R, F, Z, Y, X, int(num_way), float(step), int(with_gt))
        ctx.save_for_backward(origin, points, frame)
        ctx.meta = (tuple(sigma.shape), int(num_way), float(step), int(with_gt))
        ctx.mark_non_differentiable(length, valid)
        return logits, length, valid

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_logits, _gl, _gv):
        origin, points, frame = ctx.saved_tensors
        shape, num_way, step, with_gt = ctx.meta
        F, Z, Y, X = shape
        grad_sigma = torch.zeros(shape, dtype=torch.float32, device=grad_logits.device)
        R = points.shape[0]
        if R:
            # -inf logits receive NaN/0 gradients from log-softmax; masked samples are skipped
            g = torch.nan_to_num(grad_logits.float(), nan=0.0, posinf=0.0, neginf=0.0).contiguous()
            _call(_lib.lib().vidar_ray_sample_backward, g.device, _lib.ptr(origin), _lib.ptr(points),
                  _lib.ptr(frame), _lib.ptr(g), _lib.ptr(grad_sigma), R, F, Z, Y, X, num_way, step, with_gt)
        return grad_sigma, None, None, None, None, None, None


def ray_sample(sigma, origin, points, frame, num_way, step, with_gt=True):
    """-> (logits [R,K], length [R,K], valid [R]); K = num_way + with_gt; differentiable in sigma."""
    return _RaySample.apply(sigma, origin.contiguous(), points.contiguous(), frame, num_way, step, with_gt)


class _RayCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sigma, origin, points, frame, num_way, step):
        sigma = sigma.contiguous()
        R, F, Z, Y, X = _prep(sigma, origin, points, frame)
        ce = torch.zeros((R,), dtype=torch.float32, device=sigma.device)
        lse = torch.zeros((R,), dtype=torch.float32, device=sigma.device)
        valid = torch.zeros((R,), dtype=torch.float32, device=sigma.device)
        if R:
            _call(_lib.lib().vidar_ray_ce_forward, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
                  _lib.ptr(points), _lib.ptr(frame), _lib.ptr(ce), _lib.ptr(lse), _lib.ptr(valid),
                  R, F, Z, Y, X, int(num_way), float(step))
        ctx.save_for_backward(sigma, origin, points, frame, lse)
        ctx.meta = (int(num_way), float(step))
        ctx.mark_non_differentiable(valid)
        return ce, valid

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_ce, _gv):
        sigma, origin, points, frame, lse = ctx.saved_tensors
        num_way, step = ctx.meta
        F, Z, Y, X = sigma.shape
        grad_sigma = torch.zeros_like(sigma)
        R = points.shape[0]
        if R:
            g = grad_ce.float().contiguous()
            _call(_lib.lib().vidar_ray_ce_backward, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
                  _lib.ptr(points), _lib.ptr(frame), _lib.ptr(lse), _lib.ptr(g), _lib.ptr(grad_sigma),
                  R, F, Z, Y, X, num_way, step)
        return grad_sigma, None, None, None, None, None


def ray_ce(sigma, origin, points, frame, num_way, step):
    """Fused sampler + cross-entropy(label 0) -> (ce [R], valid [R])."""
    return _RayCE.apply(sigma, origin.contiguous(), points.contiguous(), frame, num_way, step)


class _RayGumbel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sigma, origin, points, frame, noise, num_way, step):
        sigma = sigma.contiguous()
        R, F, Z, Y, X = _prep(sigma, origin, points, frame)
        noise = noise.float().contiguous()
        if tuple(noise.shape) != (R, int(num_way)):
            raise RuntimeError(f"noise must be [rays, num_way] = {(R, int(num_way))}, got {tuple(noise.shape)}")
        out = torch.zeros((3, R), dtype=torch.float32, device=sigma.device)      # dist, lse, p_next
        if R:
            _call(_lib.lib().vidar_ray_gumbel_forward, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
                  _lib.ptr(points), _lib.ptr(frame), _lib.ptr(noise), _lib.ptr(out[0]), _lib.ptr(out[1]),
                  _lib.ptr(out[2]), R, F, Z, Y, X, int(num_way), float(step))
        ctx.save_for_backward(sigma, origin, points, frame, out)
        ctx.meta = (int(num_way), float(step))
        return out[0].clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_dist):
        sigma, origin, points, frame, out = ctx.saved_tensors
        num_way, step = ctx.meta
        F, Z, Y, X = sigma.shape
        grad_sigma = torch.zeros_like(sigma)
        R = points.shape[0]
        if R:
            g = grad_dist.float().contiguous()
            _call(_lib.lib().vidar_ray_gumbel_backward, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
                  _lib.ptr(points), _lib.ptr(frame), _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(out[2]),
                  _lib.ptr(g), _lib.ptr(grad_sigma), R, F, Z, Y, X, num_way, step)
        return grad_sigma, None, None, None, None, None, None


def gumbel_distance(sigma, origin, points, frame, num_way, step, noise):
    """Fused sampler + `_custom_gumbel_softmax_distance` (vidar_head_base.py:754-773) over the
    num_way waypoints of every ray (no GT slot): sigma [F,Z,Y,X], origin [F,3], points [R,3],
    frame int32 [R], noise [R,num_way] Gumbel(0,1) -> dist [R], differentiable in sigma."""
    return _RayGumbel.apply(sigma, origin.contiguous(), points.contiguous(), frame, noise, num_way, step)


def ray_argmax(sigma, origin, points, frame, num_way, step):
    """-> (depth [R] voxel units, index [R] float) of the arg-max waypoint."""
    sigma = sigma.contiguous()
    origin, points = origin.contiguous(), points.contiguous()
    R, F, Z, Y, X = _prep(sigma, origin, points, frame)
    depth = torch.zeros((R,), dtype=torch.float32, device=sigma.device)
    index = torch.zeros((R,), dtype=torch.float32, device=sigma.device)
    if R:
        _call(_lib.lib().vidar_ray_argmax, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
              _lib.ptr(points), _lib.ptr(frame), _lib.ptr(depth), _lib.ptr(index),
              R, F, Z, Y, X, int(num_way), float(step))
    return depth, index


def _host_weights(loss_weights, device):
    """[frame, level] loss weights as a device tensor, by a pinned non-blocking copy (no host sync)."""
    host = torch.from_numpy(np.ascontiguousarray(loss_weights, dtype=np.float32)).pin_memory()
    return host.to(device, non_blocking=True)


def _ray_frames(gt_tindex, num_frames):
    """int32 frame of every ray: its tindex when that is a frame in [0, num_frames), else -1 (skipped by the
    kernels).  No compaction, so no host sync."""
    t = gt_tindex
    keep = (t >= 0) & (t < num_frames) & (t == t.floor())     # `cur_tindex == frame_idx`
    return torch.where(keep, t, -1.0).to(torch.int32).contiguous()


def _frame_sorted_rays(gt_grids, gt_tindex, num_frames):
    """Rays of one batch element grouped by frame (frame-major, original order inside a frame,
    like the reference's double loop) -> (points [R,3], frame int32 [R])."""
    t = gt_tindex
    keep = (t >= 0) & (t < num_frames) & (t == t.floor())     # `cur_tindex == frame_idx`
    idx = keep.nonzero().squeeze(-1)
    order = torch.argsort(t[idx], stable=True)
    idx = idx[order]
    return gt_grids[idx].contiguous(), t[idx].to(torch.int32).contiguous()


def get_grid_features(batched_origin_grids, batched_gt_grids, batched_gt_tindex, intermediate_sigma,
                      loss_weights, ray_grid_step, ray_grid_num, return_as_batch=False):
    """ViDARHeadBase._get_grid_features (:420-509).  intermediate_sigma: list (one per
    intermediate level) of [bs, F, Z, Y, X]; loss_weights indexable as [frame, level].
    Returns (r_mask_total [R,K] 0/-inf, r_feat_total [lvl,R,K], r_loss_weight_total [lvl,R],
    r_grid_length [R,K]) with invalid-GT rays dropped."""
    bs, F = intermediate_sigma[0].shape[:2]
    lw = torch.as_tensor(loss_weights, dtype=torch.float32, device=batched_gt_grids.device)
    masks, feats, weights, lengths = [], [], [], []
    for b in range(bs):
        pts, frame = _frame_sorted_rays(batched_gt_grids[b], batched_gt_tindex[b], F)
        origin = batched_origin_grids[b, :F].contiguous().float()
        lvl_feats, keep, length = [], None, None
        for sig in intermediate_sigma:
            logits, length, valid = ray_sample(sig[b], origin, pts, frame, ray_grid_num, ray_grid_step, True)
            keep = valid > 0
            lvl_feats.append(logits[keep])
        feats.append(torch.stack(lvl_feats, 0))
        length = length[keep]
        lengths.append(length)
        masks.append(torch.isinf(feats[-1][0]) & (feats[-1][0] < 0))
        weights.append(lw[frame[keep].long()].t().contiguous())           # [lvl, R]
    r_mask = torch.cat(masks, 0)
    r_mask_total = torch.zeros_like(r_mask, dtype=torch.float32).masked_fill(r_mask, float("-inf"))
    r_feat_total = torch.cat(feats, 1)
    r_loss_weight_total = torch.cat(weights, 1)
    r_grid_length = torch.cat(lengths, 0)
    if return_as_batch:
        n_lvl = len(intermediate_sigma)
        r_mask_total = r_mask_total.view(bs, -1, *r_mask_total.shape[1:])
        r_feat_total = r_feat_total.view(n_lvl, bs, -1, *r_feat_total.shape[2:])
        r_loss_weight_total = r_loss_weight_total.view(n_lvl, bs, -1, *r_loss_weight_total.shape[2:])
        r_grid_length = r_grid_length.view(bs, -1, *r_grid_length.shape[1:])
    return r_mask_total, r_feat_total, r_loss_weight_total, r_grid_length


def ce_regularization_loss(batched_origin_grids, batched_gt_grids, batched_gt_tindex, intermediate_sigma,
                           loss_weights, ray_grid_step, ray_grid_num):
    """`regularization.loss` of ViDARHeadBase.loss (:586-592) without materialising the logits:
    sum(ce * w) / clamp(sum(w), min=1) over intermediate levels and valid rays."""
    bs, F = intermediate_sigma[0].shape[:2]
    lw = _host_weights(loss_weights, batched_gt_grids.device)
    num = batched_gt_grids.new_zeros(())
    den = batched_gt_grids.new_zeros(())
    for b in range(bs):
        # every row, rays of no predicted frame (padding, frame -1) contribute valid = 0
        pts = batched_gt_grids[b].float().contiguous()
        frame = _ray_frames(batched_gt_tindex[b], F)
        origin = batched_origin_grids[b, :F].contiguous().float()
        for lvl, sig in enumerate(intermediate_sigma):
            ce, valid = ray_ce(sig[b], origin, pts, frame, ray_grid_num, ray_grid_step)
            w = lw[frame.clamp(min=0).long(), lvl] * valid
            num = num + (ce * w).sum()
            den = den + w.sum()
    return num / torch.clamp(den, min=1)


def decode_ray_depth(sigma, origin_grids, gt_grids, gt_tindex, ray_grid_step, ray_grid_num):
    """Per batch element: sigma [F,Z,Y,X], origin_grids [F,3], gt_grids [M,3], gt_tindex [M] ->
    (pred_dist [M], gt_dist [M]) in voxel units, zeros for rays of no frame
    (get_point_cloud_prediction :700-734)."""
    F = sigma.shape[0]
    t = gt_tindex
    keep = (t >= 0) & (t < F) & (t == t.floor())
    idx = keep.nonzero().squeeze(-1)
    frame = t[idx].to(torch.int32).contiguous()
    pts = gt_grids[idx].contiguous()
    depth, _ = ray_argmax(sigma, origin_grids[:F].contiguous().float(), pts, frame, ray_grid_num, ray_grid_step)
    pred = gt_grids.new_zeros(gt_grids.shape[0])
    gt = gt_grids.new_zeros(gt_grids.shape[0])
    pred[idx] = depth
    gt[idx] = torch.sqrt(((pts - origin_grids[frame.long()]) ** 2).sum(-1))
    return pred, gt


def dense_chamfer_loss(dist, points, origin, gt, gt_tindex, grid, frame_weights, weight_sum, eval_within_grid=False,
                       pc_range=None, return_pairs=False):
    """`loss.dense_voxel` before its `dense_loss_weight` (vidar_head_base.py:594-659), every (sample, frame) pair
    at once, differentiable in `dist`.

    dist [bs, F*R0] decoded lengths (`gumbel_distance`), points [bs, F*R0, 3] frame-major ray end points, origin
    [bs, >=F, 3], gt [bs, M, 3] and gt_tindex [bs, M] (float, -1 = padding, any order), all voxel units on one CUDA
    device; grid = (W, H, Z); frame_weights: F host floats (loss_weight[f, 0]); weight_sum: loss_weight.sum(), the
    loss divides by weight_sum * bs; pc_range: metres, used by eval_within_grid like get_rendered_pcds.
    Returns the 0-dim loss (and, with return_pairs, [bs*F, 4] float64 per pair n = b*F + f: sum pred->gt squared
    distances, pred points, sum gt->pred, gt points)."""
    frame_weights = [float(v) for v in frame_weights]
    F = len(frame_weights)
    if dist.dim() != 2 or F == 0 or dist.shape[1] % F:
        raise RuntimeError(f"dist must be [bs, F*R0] with F = {F} frame weights, got {tuple(dist.shape)}")
    bs, FR = dist.shape
    M = gt.shape[1] if gt.dim() == 3 else -1
    if (tuple(points.shape) != (bs, FR, 3) or origin.dim() != 3 or origin.shape[0] != bs or origin.shape[1] < F
            or origin.shape[2] != 3 or tuple(gt.shape) != (bs, M, 3) or tuple(gt_tindex.shape) != (bs, M)):
        raise RuntimeError("expected points [bs, F*R0, 3], origin [bs, >=F, 3], gt [bs, M, 3], gt_tindex [bs, M]")
    for name, t in (("dist", dist), ("points", points), ("origin", origin), ("gt", gt), ("gt_tindex", gt_tindex)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32")
    if eval_within_grid and pc_range is None:
        raise RuntimeError("eval_within_grid needs pc_range")
    _lib.require_cuda(dist=dist, points=points, origin=origin, gt=gt, gt_tindex=gt_tindex)
    norm = float(np.float32(weight_sum) * np.float32(bs))        # the fp32 product weight_sum * bs
    loss, pairs = _chamfer_groups(dist.view(-1), points.view(-1, 3), origin.view(-1, 3), gt, gt_tindex, grid,
                                  _frame_tables(bs, F, origin.shape[1], tuple(frame_weights), norm), bs * F, 1, F,
                                  eval_within_grid, pc_range)
    return (loss.view(()), pairs) if return_pairs else loss.view(())


@functools.lru_cache(maxsize=64)
def _frame_tables(bs, F, To, frame_weights, norm):
    """dense_chamfer_loss's host tables, built once per shape and weights (the loss is host-bound at small bs):
    pair n = b*F + f of sample b's frame f, origin row b*To + f, weight frame_weights[f], one group."""
    b, f = np.divmod(np.arange(bs * F), F)
    return _host_tables(np.stack([b, f, b * To + f, np.zeros_like(b)], 1), np.tile(np.float32(frame_weights), bs),
                        np.float32([norm]), bs, F)


def _host_tables(tab, w, norms, Sg, Fg):
    """The pair tables as one int32 host array: pair of each (gt sample, frame) slot [Sg*Fg] (-1 = none), (slot,
    origin row, group) of each pair [P, 3], then the float32 bits of the pair weights [P] and group norms."""
    slot = tab[:, 0] * Fg + tab[:, 1]
    slot_pair = np.full(Sg * Fg, -1, dtype=np.int64)
    slot_pair[slot] = np.arange(tab.shape[0])
    ints = np.concatenate([slot_pair, np.stack([slot, tab[:, 2], tab[:, 3]], 1).ravel()]).astype(np.int32)
    return np.concatenate([ints, np.concatenate([w, norms]).astype(np.float32).view(np.int32)])


def _chamfer_groups(dist, points, origin, gt, gt_tindex, grid, host, P, groups, Fg, eval_within_grid, pc_range):
    """Checked arguments of dense_chamfer_group_loss -> (loss [groups], pairs [P, 4]); the host tables reach the
    device in one pinned non-blocking copy."""
    Sg, M = gt.shape[:2]
    table = _pinned_upload(host, np.int32, dist.device)
    n = Sg * Fg + 3 * P
    tables = (table[: Sg * Fg], table[Sg * Fg:n], table[n:n + P].view(torch.float32), table[n + P:].view(torch.float32))
    return _DenseChamferGroups.apply(dist, points, origin, gt, gt_tindex, tables,
                                     (P, groups, dist.shape[0] // P, Sg, Fg, M), grid, eval_within_grid,
                                     pc_range if pc_range is not None else [0.0] * 6)


def _pinned_upload(host, dtype, device):
    """Host array -> device tensor by one pinned non-blocking copy (no host sync)."""
    t = torch.from_numpy(np.ascontiguousarray(host, dtype=dtype)).pin_memory()
    return t.to(device, non_blocking=True)


class _DenseChamferGroups(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dist, points, origin, gt, gt_tindex, tables, dims, grid, within_grid, pc_range):
        slot_pair, pair_tab, pair_w, group_norm = tables
        P, groups, R0, Sg, Fg, M = dims
        dev = dist.device
        W, H, Z = (int(v) for v in grid)
        Pq = P * R0 + Sg * M
        qbuf = torch.empty((Pq, 3), dtype=torch.float32, device=dev)
        cbuf = torch.empty((Pq, 3), dtype=torch.float32, device=dev)
        q_mask = torch.empty(Pq, dtype=torch.uint8, device=dev)
        c_mask = torch.empty(Pq, dtype=torch.uint8, device=dev)
        seg_off = torch.empty((2, 2 * P + 1), dtype=torch.int64, device=dev)
        idx = torch.empty(Pq, dtype=torch.int64, device=dev)
        pairs = torch.empty((P, 4), dtype=torch.float64, device=dev)
        loss = torch.empty(groups, dtype=torch.float32, device=dev)
        rng = (C.c_float * 6)(*[float(v) for v in pc_range])
        Pt = _lib.ptr
        _call(_lib.lib().vidar_dense_chamfer_groups_forward, dev, Pt(dist), Pt(points), Pt(origin), Pt(gt),
              Pt(gt_tindex), Pt(slot_pair), Pt(pair_tab), Pt(pair_w), Pt(group_norm), C.cast(rng, C.c_void_p),
              Pt(qbuf), Pt(cbuf), Pt(q_mask), Pt(c_mask), Pt(seg_off[0]), Pt(seg_off[1]), Pt(idx), Pt(pairs),
              Pt(loss), P, groups, R0, Sg, Fg, M, W, H, Z, int(bool(within_grid)))
        ctx.save_for_backward(points, origin, qbuf, cbuf, q_mask, seg_off, idx, pairs, pair_tab, pair_w, group_norm)
        ctx.dims = dims
        ctx.mark_non_differentiable(pairs)
        return loss, pairs

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss, _gp):
        points, origin, qbuf, cbuf, q_mask, seg_off, idx, pairs, pair_tab, pair_w, group_norm = ctx.saved_tensors
        P, groups, R0, Sg, Fg, M = ctx.dims
        g = grad_loss.float().contiguous()
        grad_dist = torch.empty(P * R0, dtype=torch.float32, device=qbuf.device)
        Pt = _lib.ptr
        _call(_lib.lib().vidar_dense_chamfer_groups_backward, qbuf.device, Pt(points), Pt(origin), Pt(qbuf),
              Pt(cbuf), Pt(q_mask), Pt(seg_off[0]), Pt(seg_off[1]), Pt(idx), Pt(pairs), Pt(pair_tab), Pt(pair_w),
              Pt(group_norm), Pt(g), Pt(grad_dist), P, groups, R0, Sg, Fg, M)
        return grad_dist, None, None, None, None, None, None, None, None, None


def dense_chamfer_group_loss(dist, points, origin, gt, gt_tindex, grid, pairs, pair_weights, group_norms,
                             eval_within_grid=False, pc_range=None, return_pairs=False):
    """`dense_chamfer_loss` over a pair table, one loss per group, differentiable in `dist`.

    dist [P*R0] decoded lengths, points [P*R0, 3] ray end points (rays of pair n at n*R0 ..), origin [No, 3],
    gt [Sg, M, 3] and gt_tindex [Sg, M] (float frame in [0, Fg), -1 = padding, any order), voxel units on one CUDA
    device; grid = (W, H, Z).  Host tables: pairs [P, 4] ints (gt sample, gt frame, origin row, group), in increasing
    (gt sample, gt frame) order; pair_weights [P]; group_norms [groups].
    loss[g] = sum over the pairs n of group g of w_n * (mean pred->gt + mean gt->pred) / 2 / group_norms[g].
    Returns loss [groups] (and, with return_pairs, the [P, 4] float64 per-pair sums of dense_chamfer_loss)."""
    tab = np.asarray(pairs, dtype=np.int64).reshape(-1, 4)
    w = np.asarray(pair_weights, dtype=np.float32).reshape(-1)
    norms = np.asarray(group_norms, dtype=np.float32).reshape(-1)
    P, groups = tab.shape[0], norms.shape[0]
    if P == 0 or w.shape[0] != P or groups == 0:
        raise RuntimeError(f"need P > 0 pairs [P, 4] with P weights and > 0 group norms, got {tab.shape}, "
                           f"{w.shape}, {norms.shape}")
    if dist.dim() != 1 or dist.shape[0] % P:
        raise RuntimeError(f"dist must be [P*R0] with P = {P} pairs, got {tuple(dist.shape)}")
    R0 = dist.shape[0] // P
    if gt.dim() != 3 or gt.shape[2] != 3 or tuple(gt_tindex.shape) != tuple(gt.shape[:2]):
        raise RuntimeError("expected gt [Sg, M, 3] and gt_tindex [Sg, M]")
    Sg, M = gt.shape[:2]
    if tuple(points.shape) != (P * R0, 3) or origin.dim() != 2 or origin.shape[1] != 3:
        raise RuntimeError("expected points [P*R0, 3] and origin [No, 3]")
    for name, t in (("dist", dist), ("points", points), ("origin", origin), ("gt", gt), ("gt_tindex", gt_tindex)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32")
    Fg = int(tab[:, 1].max()) + 1
    slot = tab[:, 0] * Fg + tab[:, 1]
    if ((tab[:, 0] < 0) | (tab[:, 0] >= Sg) | (tab[:, 1] < 0)).any() or (np.diff(slot) <= 0).any():
        raise RuntimeError("pairs must name distinct (gt sample, frame) slots in increasing order")
    if ((tab[:, 2] < 0) | (tab[:, 2] >= origin.shape[0]) | (tab[:, 3] < 0) | (tab[:, 3] >= groups)).any():
        raise RuntimeError("pair origin row or group out of range")
    if eval_within_grid and pc_range is None:
        raise RuntimeError("eval_within_grid needs pc_range")
    _lib.require_cuda(dist=dist, points=points, origin=origin, gt=gt, gt_tindex=gt_tindex)
    loss, pair_sums = _chamfer_groups(dist, points, origin, gt, gt_tindex, grid, _host_tables(tab, w, norms, Sg, Fg),
                                      P, groups, Fg, eval_within_grid, pc_range)
    return (loss, pair_sums) if return_pairs else loss


def align_gt(gt, mats, jobs, voxel, with_points=False):
    """GT alignment of ViDARHeadV1 for every head frame (vidar_head_v1.py:94-148), csrc/dense_chamfer.cu.

    gt [bs, M, Cg] float32 GT rows in metres, NaN-padded, the frame in the last column; mats [H*V, bs, 4, 4]
    float32 (device) src -> tgt transform per (head frame, slot) job; jobs: host ints [H, V], the source frame of
    each job, -1 = none; voxel: host (offset[3], scale[3], cells[3]), ray = ((x' - offset) * scale) * cells.
    Returns rays [H*bs, M, 3] voxel units, tindex [H*bs, M] (slot, -1 = padding) and, with_points, the aligned
    points [H*bs, M, 3] in metres: per (head frame, sample) the slots in order, the rows of a slot in their order,
    then padding."""
    jobs = np.asarray(jobs, dtype=np.int64)
    if jobs.ndim != 2:
        raise RuntimeError(f"jobs must be [head frames, slots], got shape {jobs.shape}")
    H, V = jobs.shape
    if gt.dim() != 3 or gt.shape[2] < 4 or gt.dtype != torch.float32:
        raise RuntimeError("gt must be float32 [bs, M, Cg >= 4]")
    bs, M, Cg = gt.shape
    if tuple(mats.shape) != (H * V, bs, 4, 4) or mats.dtype != torch.float32:
        raise RuntimeError(f"mats must be float32 {(H * V, bs, 4, 4)}, got {tuple(mats.shape)}")
    voxel = np.asarray(voxel, dtype=np.float32).reshape(-1)
    if voxel.shape != (9,):
        raise RuntimeError("voxel must hold 9 floats: offset[3], scale[3], cells[3]")
    _lib.require_cuda(gt=gt, mats=mats)
    dev = gt.device
    rays = torch.empty((H * bs, M, 3), dtype=torch.float32, device=dev)
    tindex = torch.empty((H * bs, M), dtype=torch.float32, device=dev)
    points = torch.empty((H * bs, M, 3), dtype=torch.float32, device=dev) if with_points else None
    j = (C.c_int32 * (H * V))(*[int(v) for v in jobs.ravel()])
    vx = (C.c_float * 9)(*[float(v) for v in voxel])
    _call(_lib.lib().vidar_head_align_gt, dev, _lib.ptr(gt), _lib.ptr(mats), C.cast(j, C.c_void_p),
          C.cast(vx, C.c_void_p), _lib.ptr(rays), _lib.ptr(tindex), _lib.ptr(points), bs, M, Cg, H, V)
    return rays, tindex, points


def decode_clouds(depth, rays, points, tindex, origin_vox, origin, scale, within_grid=False, pc_range=None):
    """The pred and gt clouds of every (sample, frame) from the decoded rays, csrc/eval_metrics.cu.

    depth [bs, M] arg-max depth (voxel units), rays [bs, M, 3] GT points in voxel units and points [bs, M, 3] in metres,
    tindex [bs, M] float frame (-1 or outside [0, F) = in no cloud), origin_vox / origin [bs, F, 3] voxel units /
    metres, all float32 on one CUDA device; scale = (pc_range[3] - pc_range[0]) / bev_w; pc_range: metres, used by
    within_grid like get_rendered_pcds.  Returns pred, gt [bs * M, 3] and off [bs * F + 2] int64: cloud n = b * F + t
    at rows [off[n], off[n+1]), then one segment of every other row (NaN points, masked by the metrics)."""
    if rays.dim() != 3 or rays.shape[2] != 3:
        raise RuntimeError(f"rays must be [bs, M, 3], got {tuple(rays.shape)}")
    bs, M = rays.shape[:2]
    F = origin.shape[1] if origin.dim() == 3 else -1
    if (tuple(depth.shape) != (bs, M) or tuple(points.shape) != (bs, M, 3) or tuple(tindex.shape) != (bs, M)
            or tuple(origin.shape) != (bs, F, 3) or tuple(origin_vox.shape) != (bs, F, 3)):
        raise RuntimeError("expected depth [bs, M], points [bs, M, 3], tindex [bs, M], origin / origin_vox [bs, F, 3]")
    for name, t in (("depth", depth), ("rays", rays), ("points", points), ("tindex", tindex),
                    ("origin_vox", origin_vox), ("origin", origin)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32")
    if within_grid and pc_range is None:
        raise RuntimeError("eval_within_grid needs pc_range")
    _lib.require_cuda(depth=depth, rays=rays, points=points, tindex=tindex, origin_vox=origin_vox, origin=origin)
    dev = rays.device
    pred = torch.empty((bs * M, 3), dtype=torch.float32, device=dev)
    gt = torch.empty((bs * M, 3), dtype=torch.float32, device=dev)
    off = torch.empty(bs * F + 2, dtype=torch.int64, device=dev)
    rng = (C.c_float * 6)(*[float(v) for v in (pc_range if pc_range is not None else [0.0] * 6)])
    P = _lib.ptr
    _call(_lib.lib().vidar_eval_decode_clouds, dev, P(depth), P(rays), P(points), P(tindex), P(origin_vox), P(origin),
          C.cast(rng, C.c_void_p), float(scale), int(bool(within_grid)), P(pred), P(gt), P(off), bs, M, F)
    return pred, gt, off
