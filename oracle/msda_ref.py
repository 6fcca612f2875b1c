"""CPU oracle for multi-scale deformable attention.  TEST INFRASTRUCTURE ONLY.

The arithmetic of this path lives in a dependency that is NOT vendored in the reference:
mmcv-full==1.4.0 (README.md:103 of the reference), `_ext.ms_deform_attn_{forward,backward}`
and its any-device twin `mmcv.ops.multi_scale_deform_attn.multi_scale_deformable_attn_pytorch`
(imported at projects/mmdet3d_plugin/bevformer/modules/spatial_cross_attention.py:8 and used on
non-CUDA tensors at :393-394).  This file restates the published algorithm (Deformable-DETR,
Zhu et al. 2020, as implemented by mmcv): per level, bilinear `grid_sample(padding='zeros',
align_corners=False)` of the value map at `2*loc-1`, weighted by the attention weights and
summed over levels x points.

Two independent statements are given:
  * `msda_grid_sample`  -- the grid_sample formulation (what the reference's CPU path runs);
    autograd provides its backward;
  * `msda_explicit`     -- the per-corner formulation the CUDA kernels follow
    (SURVEY.md A.1: pixel = loc*size - 0.5, four individually zero-padded corners,
    analytic gradients), in numpy float64.
On top of `msda_grid_sample`, `msda_rows` / `msda_sca_rows` state SpatialCrossAttention's row map (per-camera
visible-pillar lists scattered into the BEV slots), the operation of the vidar_msda_rows_* / vidar_msda_sca_rows_*
entry points.
Pinning: tests/test_oracle_msda.py checks both against each other and against the
same-lineage implementation shipped in `transformers`
(`transformers.models.deformable_detr.modeling_deformable_detr`), which is present in this
image; the reference itself holds no golden vectors for this op (SURVEY.md 8c).
"""
import numpy as np
import torch
import torch.nn.functional as F


def msda_grid_sample(value, spatial_shapes, sampling_locations, attention_weights):
    """value [B,K,H,C]; spatial_shapes [L,2] (h,w); sampling_locations [B,Q,H,L,P,2] (x,y in
    [0,1]); attention_weights [B,Q,H,L,P] -> [B,Q,H*C].  Differentiable torch ops only."""
    B, K, H, C = value.shape
    _, Q, _, L, P, _ = sampling_locations.shape
    shapes = [(int(h), int(w)) for h, w in torch.as_tensor(spatial_shapes).tolist()]
    assert sum(h * w for h, w in shapes) == K
    out = value.new_zeros(B * H, C, Q)
    start = 0
    # [B,Q,H,L,P] -> [B*H, Q, L, P]
    w_all = attention_weights.permute(0, 2, 1, 3, 4).reshape(B * H, Q, L, P)
    for lvl, (h, w) in enumerate(shapes):
        # value of this level as an image batch [B*H, C, h, w]
        v = value[:, start:start + h * w].permute(0, 2, 3, 1).reshape(B * H, C, h, w)
        start += h * w
        # grid [B*H, Q, P, 2] in [-1, 1]
        g = sampling_locations[:, :, :, lvl].permute(0, 2, 1, 3, 4).reshape(B * H, Q, P, 2)
        s = F.grid_sample(v, 2.0 * g - 1.0, mode="bilinear", padding_mode="zeros",
                          align_corners=False)            # [B*H, C, Q, P]
        out = out + (s * w_all[:, None, :, lvl, :]).sum(-1)
    return out.reshape(B, H * C, Q).transpose(1, 2).contiguous()


def msda_grid_sample_backward(value, spatial_shapes, sampling_locations, attention_weights,
                              grad_output, dtype=torch.float64):
    """(grad_value, grad_loc, grad_attn) of msda_grid_sample by autograd, in `dtype`."""
    v = value.detach().to(dtype).requires_grad_(True)
    loc = sampling_locations.detach().to(dtype).requires_grad_(True)
    aw = attention_weights.detach().to(dtype).requires_grad_(True)
    out = msda_grid_sample(v, spatial_shapes, loc, aw)
    out.backward(grad_output.to(dtype))
    return v.grad, loc.grad, aw.grad


def _rows_into_slots(slots, group, bs, rows_out, idx, count, inv):
    """Add the live rows of one launch group into slots [bs, Qd, H*C].  rows_out [bs*ncl, rows, H*C]: row j of
    batch element n = b*ncl + camera.  Rows that are not live (j >= count[cam], or (j // 64) % S outside
    [s_lo, s_hi)) add nothing; the others go to pillar idx[cam, j] (j without a list), scaled by inv[b, q]."""
    cam0, ncl, S, lo, hi = group
    dev = rows_out.device
    rows = rows_out.shape[1]
    j = torch.arange(rows, device=dev)
    n = torch.arange(bs * ncl, device=dev)
    b, cam = n // ncl, cam0 + n % ncl
    live = (((j // 64) % S >= lo) & ((j // 64) % S < hi)).expand(bs * ncl, rows)
    if count is not None:
        live = live & (j[None] < count.to(dev).long()[cam][:, None])
    q = idx.to(dev)[cam][:, :rows].long() if idx is not None else j.expand(bs * ncl, rows)
    bb = b[:, None].expand(bs * ncl, rows)
    out = rows_out[live]
    if inv is not None:
        out = out * inv.to(device=dev, dtype=out.dtype)[bb[live], q[live]][:, None]
    return slots.index_put((bb[live], q[live]), out, accumulate=True)


def msda_rows(plan, bs, Qd, spatial_shapes, idx, count, inv, groups):
    """The row map of `MSDARowsFunction` (SpatialCrossAttention's rebatch + scatter-add around the op) in
    differentiable torch: autograd gives every gradient, on any device and dtype.
    plan [(cam0, ncl, S, s_lo, s_hi)]; groups [(value [bs*ncl, K, H, C], loc [bs*ncl, rows, H, L, P, 2],
    attn [bs*ncl, rows, H, L, P])] per launch group; idx [cams, Qd] | None; count [cams] | None;
    inv [bs, Qd] | None  ->  slots [bs, Qd, H*C]."""
    H, C = groups[0][0].shape[2:]
    slots = groups[0][0].new_zeros(bs, Qd, H * C)
    for group, (v, loc, aw) in zip(plan, groups):
        slots = _rows_into_slots(slots, group, bs, msda_grid_sample(v, spatial_shapes, loc, aw), idx, count, inv)
    return slots


def sca_locations(spatial_shapes, offsets, ref):
    """MSDeformableAttention3D's sampling locations in its own fp32 statements (spatial_cross_attention.py:356-371):
    offsets [..., H, L, P, 2] / (W_l, H_l) + ref [..., D, 2] at Z-anchor p % D.  Returned in offsets' dtype with
    d(loc)/d(offsets) = 1 / (W_l, H_l), but with the fp32 value, which the fused kernels reproduce bit for bit."""
    shapes = torch.as_tensor(spatial_shapes).to(offsets.device)
    L, P, D = offsets.shape[-3], offsets.shape[-2], ref.shape[-2]
    lead = offsets.shape[:-4]
    H = offsets.shape[-4]
    wh32 = torch.stack([shapes[:, 1], shapes[:, 0]], -1).float()
    o32 = offsets.detach().float()
    r32 = ref.detach().float().reshape(*lead, 1, 1, 1, D, 2)
    loc32 = ((o32 / wh32.view(L, 1, 2)).view(*lead, H, L, P // D, D, 2) + r32).view(*lead, H, L, P, 2)
    wh = wh32.to(offsets.dtype).view(L, 1, 2)
    return loc32.to(offsets.dtype) + (offsets - offsets.detach()) / wh


def msda_sca_rows(plan, bs, spatial_shapes, idx, count, inv, ref_cam, offsets, logits, values):
    """The fused row map of `SCARowsFunction`: offsets [bs, Qd, H, L, P, 2] and logits [bs, Qd, H, L*P] are dense
    per pillar and gathered through idx for every (camera, row); ref_cam [cams, bs, Qd, D, 2].  Locations from
    `sca_locations`, softmax and sampling in the inputs' dtype.  values[g] [bs*ncl, K, H, C] -> slots [bs, Qd, H*C];
    autograd gives the per-pillar offset / logit gradients summed over cameras."""
    _, Qd, H, L, P, _ = offsets.shape
    C = values[0].shape[-1]
    slots = offsets.new_zeros(bs, Qd, H * C)
    for (cam0, ncl, S, lo, hi), v in zip(plan, values):
        n = torch.arange(bs * ncl, device=offsets.device)
        b, cam = n // ncl, cam0 + n % ncl
        q = idx.to(offsets.device)[cam].long() if idx is not None else torch.arange(Qd, device=offsets.device).expand(bs * ncl, Qd)
        q = q.clamp(0, Qd - 1)            # list entries past count are undefined; those rows are masked below
        bb = b[:, None].expand_as(q)
        loc = sca_locations(spatial_shapes, offsets[bb, q], ref_cam.to(offsets.device)[cam[:, None], bb, q])
        w = logits[bb, q].softmax(-1).view(bs * ncl, Qd, H, L, P)
        slots = _rows_into_slots(slots, (cam0, ncl, S, lo, hi), bs, msda_grid_sample(v, spatial_shapes, loc, w),
                                 idx, count, inv)
    return slots


def msda_explicit(value, spatial_shapes, level_start_index, sampling_locations,
                  attention_weights, grad_output=None):
    """Per-corner statement in numpy float64.  Returns out, or (out, gv, gloc, gattn) when
    grad_output is given.  Python loops over (level, point) only; vectorised over b,q,h."""
    value = np.asarray(value, np.float64)
    loc = np.asarray(sampling_locations, np.float64)
    aw = np.asarray(attention_weights, np.float64)
    shapes = np.asarray(spatial_shapes).astype(np.int64)
    lsi = np.asarray(level_start_index).astype(np.int64)
    B, K, H, C = value.shape
    _, Q, _, L, P, _ = loc.shape
    out = np.zeros((B, Q, H, C))
    if grad_output is not None:
        go = np.asarray(grad_output, np.float64).reshape(B, Q, H, C)
        gv = np.zeros_like(value)
        gloc = np.zeros_like(loc)
        gaw = np.zeros_like(aw)
    bi = np.arange(B)[:, None, None]
    hi = np.arange(H)[None, None, :]
    for l in range(L):
        Hl, Wl = int(shapes[l, 0]), int(shapes[l, 1])
        for p in range(P):
            x = loc[:, :, :, l, p, 0] * Wl - 0.5
            y = loc[:, :, :, l, p, 1] * Hl - 0.5
            ok = (y > -1) & (x > -1) & (y < Hl) & (x < Wl)
            xs = np.where(ok, x, 0.0)
            ys = np.where(ok, y, 0.0)
            x0 = np.floor(xs).astype(np.int64)
            y0 = np.floor(ys).astype(np.int64)
            lw = xs - x0
            lh = ys - y0
            hw, hh = 1 - lw, 1 - lh
            corners = []
            for (yy, xx, wgt) in ((y0, x0, hh * hw), (y0, x0 + 1, hh * lw),
                                  (y0 + 1, x0, lh * hw), (y0 + 1, x0 + 1, lh * lw)):
                m = ok & (yy >= 0) & (yy <= Hl - 1) & (xx >= 0) & (xx <= Wl - 1)
                idx = lsi[l] + np.clip(yy, 0, Hl - 1) * Wl + np.clip(xx, 0, Wl - 1)
                v = value[bi, idx, hi] * m[..., None]          # [B,Q,H,C]
                corners.append((idx, m, wgt, v))
            a = aw[:, :, :, l, p]
            val = sum(wgt[..., None] * v for (_, _, wgt, v) in corners)
            out += a[..., None] * val
            if grad_output is not None:
                v1, v2, v3, v4 = (c[3] for c in corners)
                top = go * a[..., None]
                for (idx, m, wgt, _) in corners:
                    contrib = (wgt * m)[..., None] * top
                    np.add.at(gv, (np.broadcast_to(bi, idx.shape), idx,
                                   np.broadcast_to(hi, idx.shape)), contrib)
                g_w = (hh[..., None] * (v2 - v1) + lh[..., None] * (v4 - v3))
                g_h = (hw[..., None] * (v3 - v1) + lw[..., None] * (v4 - v2))
                gloc[:, :, :, l, p, 0] = Wl * (g_w * top).sum(-1) * ok
                gloc[:, :, :, l, p, 1] = Hl * (g_h * top).sum(-1) * ok
                gaw[:, :, :, l, p] = (go * val).sum(-1) * ok
    out = out.reshape(B, Q, H * C)
    if grad_output is None:
        return out
    return out, gv, gloc, gaw
