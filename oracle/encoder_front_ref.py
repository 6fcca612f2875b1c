"""Host oracles of the BEV encoder's front end and error bounds of LatentRendering's fused projections.

Camera projection (`point_sampling`, modules/encoder.py:94-156).  The reference builds the world point
    (x, y, z) = ref * (range_max - range_min) + range_min,
multiplies it, as (x, y, z, 1), by each sample's 4 x 4 lidar2img in fp32 with TF32 off, keeps the points
with p.z > eps (eps = 1e-5), divides p.xy by max(p.z, eps), then u by the image width and v by the image
height, and keeps the points with 0 < v < 1 and 0 < u < 1.  Here:

  * `point_sampling_fp64`   those statements in fp64 on the fp32 inputs, with the decision margins
                            p.z - eps, u, 1 - u, v and 1 - v and a bound on each margin's fp32 error;
  * `point_sampling_fp32`   the statement order of csrc/sca_glue.cu's `point_sampling_kernel` in numpy
                            float32, one numpy op per CUDA intrinsic (every one is correctly rounded, so
                            the kernel must match it bit for bit);
  * `fmaf`                  a correctly rounded fp32 fused multiply-add: the fp64 product of two fp32
                            values is exact, TwoSum gives the exact sum as s + err, and the one case where
                            rounding s to fp32 would round twice (s exactly halfway between two fp32
                            values, err != 0) is moved off the midpoint toward err first;
  * `visible_lists`         SpatialCrossAttention's per-camera lists `mask[c, 0].sum(-1).nonzero()` and the
                            1 / clamp(#cameras, 1) normaliser (spatial_cross_attention.py:136-140, 168-171).

Projection bounds (csrc/latent_proj.cu).  u = 2^-24 is fp32's unit roundoff and g(n) = n u / (1 - n u).
Every inequality is elementwise, on fp32 inputs, with abs quantities computed on |inputs| in fp64:

  * proj_in_fwd    occ | feat = b + sum_k x w, an fma chain of E terms from the bias:
                       g(E) (|b| + sum_k |x| |w|)
  * grad_embed     sum_n g w over N1 = D + A terms:                   g(N1) sum_n |g| |w|
  * proj_out_fwd   out = (bb + sum_i p wb) * prob, A fmas and one product:
                       g(A + 1) (|bb| + sum_i |p| |wb|) |prob|
  * grad_pooled    sum_e (grad_out * prob) wb over E terms, one rounding of the product:
                       g(E + 1) sum_e |grad_out| |prob| |wb|
  * grad_prob      sum over the E / D channels of height d of grad_out * lin, lin = bb + sum_i p wb rounded
                   by A fmas; each lane dots 4 channels (1 product, 3 fmas) and log2(E / 4D) shuffle adds
                   join the lanes of a group:
                       g(A + 4 + log2(E / 4D)) sum_e |grad_out| (|bb| + sum_i |p| |wb|)
  * weight / bias gradients   each block sums its rows_per_block rows in registers, the grid's partial
                   sums are added into the output with red.add in any order, on top of what the buffer held:
                       g(rows_per_block + grid + 1) (|acc| + sum_rows |g| |x|)    (x = 1 for a bias,
                   and |g| carries one more rounding, g(1), where it is grad_out * prob)
The bounds are first order; tests multiply them by SAFETY = 2.
"""
import math
from fractions import Fraction

import numpy as np
import torch

EPS = float(np.float32(1e-5))       # the reference's eps as its fp32 comparison sees it
U32 = 2.0 ** -24


def gamma(n):
    return n * U32 / (1.0 - n * U32)


# ------------------------------------------------------------------------------ camera projection

def fmaf(a, b, c):
    """Correctly rounded fp32 a * b + c on float32 arrays (normal-range results)."""
    a, b, c = (np.asarray(t, np.float32).astype(np.float64) for t in (a, b, c))
    p = a * b                                    # exact: 24 + 24 significant bits
    s = p + c
    bp = s - c                                   # TwoSum
    err = (p - bp) + (c - (s - bp))
    bits = np.ascontiguousarray(s).view(np.uint64)
    low = bits & np.uint64((1 << 29) - 1)        # fp64 bits below fp32's last mantissa bit
    mid = (low == np.uint64(1 << 28)) & (err != 0)
    s = np.where(mid, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def fraction_round_f32(x):
    """Round an exact Fraction to the nearest fp32, ties to even (an independent check of `fmaf`)."""
    f = np.float32(float(x))
    best = None
    for cand in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(cand)) - x)
        even = (np.array(cand, np.float32).view(np.uint32) & 1) == 0
        key = (d, not even)
        if best is None or key < best[0]:
            best = (key, cand)
    return np.float32(best[1])


def _l2i(lidar2img):
    return np.asarray(lidar2img, np.float32)                   # [bs, cams, 4, 4]


def point_sampling_fp32(ref3d, lidar2img, pc_range, img_hw):
    """`point_sampling_kernel` statement by statement.  ref3d [bs, D, Q, 3] -> (ref_cam [cams, bs, Q, D, 2]
    float32, mask [cams, bs, Q, D] bool)."""
    f32 = np.float32
    pc = np.asarray(pc_range, f32)
    rs = [f32(pc[i + 3] - pc[i]) for i in range(3)]
    ref = np.asarray(ref3d, f32).transpose(0, 2, 1, 3)          # [bs, Q, D, 3]
    x, y, z = (f32(ref[..., i] * rs[i]) + pc[i] for i in range(3))
    m = _l2i(lidar2img).transpose(1, 0, 2, 3)[:, :, None, None]  # [cams, bs, 1, 1, 4, 4]
    row = lambda k: fmaf(m[..., k, 0], x, fmaf(m[..., k, 1], y, fmaf(m[..., k, 2], z, m[..., k, 3])))
    px, py, pz = row(0), row(1), row(2)
    eps = f32(1e-5)
    den = np.maximum(pz, eps)
    u = (px / den) / f32(img_hw[1])
    v = (py / den) / f32(img_hw[0])
    mask = (pz > eps) & (v > 0) & (v < 1) & (u < 1) & (u > 0)
    return np.stack((u, v), -1).astype(f32), mask


def point_sampling_fp64(ref3d, lidar2img, pc_range, img_hw):
    """The reference's statements in fp64 on the fp32 inputs.  Returns a dict with `ref_cam`
    [cams, bs, Q, D, 2], `mask` [cams, bs, Q, D], the margins `pz_eps` (p.z - eps) and `uv_margin`
    (min of u, 1 - u, v, 1 - v), and `pz_bound` / `uv_bound`: first-order bounds on how far an fp32
    evaluation of the same statements (any order of the 4-term dot product, fma or not) can move each
    margin.  A point whose margin is below its bound may legitimately be decided either way."""
    H, W = float(img_hw[0]), float(img_hw[1])
    pc = np.asarray(pc_range, np.float32).astype(np.float64)
    ref = np.asarray(ref3d, np.float32).astype(np.float64).transpose(0, 2, 1, 3)     # [bs, Q, D, 3]
    xyz = [ref[..., i] * (pc[i + 3] - pc[i]) + pc[i] for i in range(3)]
    # fp32 world point: one rounding in the range size, two in r * size + min
    xyz_err = [3 * U32 * (np.abs(ref[..., i] * (pc[i + 3] - pc[i])) + abs(pc[i])) for i in range(3)]
    m = _l2i(lidar2img).astype(np.float64).transpose(1, 0, 2, 3)[:, :, None, None]
    p, perr = [], []
    for k in range(3):
        val = m[..., k, 3] + sum(m[..., k, i] * xyz[i] for i in range(3))
        mag = np.abs(m[..., k, 3]) + sum(np.abs(m[..., k, i] * xyz[i]) for i in range(3))
        p.append(val)
        perr.append(gamma(4) * mag + sum(np.abs(m[..., k, i]) * xyz_err[i] for i in range(3)))
    px, py, pz = p
    den = np.maximum(pz, EPS)
    u, v = px / den / W, py / den / H
    mask = (pz > EPS) & (v > 0) & (v < 1) & (u < 1) & (u > 0)
    # u = fl(fl(px / den) / W): perturbations of px and pz, then two correctly rounded divisions
    absden = np.abs(den)
    uerr = (perr[0] + np.abs(u) * W * perr[2]) / (absden * W) + gamma(2) * np.abs(u)
    verr = (perr[1] + np.abs(v) * H * perr[2]) / (absden * H) + gamma(2) * np.abs(v)
    uv_margin = np.minimum(np.minimum(u, 1 - u), np.minimum(v, 1 - v))
    return dict(ref_cam=np.stack((u, v), -1), mask=mask, pz_eps=pz - EPS, pz_bound=perr[2],
                uv_margin=uv_margin, uv_bound=np.maximum(uerr, verr), u_bound=uerr, v_bound=verr)


def ambiguous(o, safety=2.0):
    """Points whose fp64 decision is within `safety` x its rounding bound of flipping."""
    near_z = np.abs(o["pz_eps"]) <= safety * o["pz_bound"]
    near_edge = (o["pz_eps"] > 0) & (np.abs(o["uv_margin"]) <= safety * o["uv_bound"])
    return near_z | near_edge


def visible_lists(mask):
    """mask [cams, bs, Q, D] -> (list of per-camera ascending pillar indices of batch element 0,
    counts [cams] int, inv [bs, Q] float32 = 1 / clamp(#cameras that see the pillar, 1))."""
    mask = np.asarray(mask, bool)
    hit = mask.sum(-1) > 0                                       # [cams, bs, Q]
    idx = [np.nonzero(hit[c, 0])[0] for c in range(mask.shape[0])]
    counts = np.array([len(i) for i in idx], np.int64)
    n = np.maximum(hit.sum(0), 1).astype(np.float32)             # [bs, Q]
    return idx, counts, (np.float32(1) / n).astype(np.float32)


# ------------------------------------------------------------------------------ projection bounds
# Inputs are torch tensors (any device); pass them in fp64.  Launch geometry of csrc/latent_proj.cu:
# rows per block tile and blocks per SM of each kernel's `grid_for`.
PROJ_TILE_ROWS = {"proj_in_fwd": 64, "proj_in_bwd": 32, "proj_out_fwd": 32, "proj_out_bwd": 32}
PROJ_PER_SM = {"proj_in_fwd": 2, "proj_in_bwd": 2, "proj_out_fwd": 4, "proj_out_bwd": 2}


def proj_launch(kernel, rows, sms):
    """(grid, rows one round of the grid covers, rows the busiest block sums) of a kernel's launch."""
    tile = PROJ_TILE_ROWS[kernel]
    tiles = -(-rows // tile)
    grid = max(1, min(tiles, sms * PROJ_PER_SM[kernel]))
    return grid, grid * tile, -(-tiles // grid) * tile


def _expand_prob(q, E):
    D = q.shape[-1]
    return q.repeat_interleave(E // D, dim=-1)


def bound_proj_in_fwd(x, w, b):
    return gamma(x.shape[-1]) * (b.abs() + x.abs() @ w.abs().t())


def bound_grad_embed(g, w):
    return gamma(g.shape[-1]) * (g.abs() @ w.abs())


def bound_weight_grad(g, x, rows_per_block, grid, acc=None, g_rounded=False):
    """grad_W [n, k] += sum_rows g[:, n] x[:, k]."""
    s = g.abs().t() @ x.abs()
    n = rows_per_block + grid + 1 + (1 if g_rounded else 0)
    return gamma(n) * (s + (acc.abs() if acc is not None else 0))


def bound_bias_grad(g, rows_per_block, grid, acc=None, g_rounded=False):
    n = rows_per_block + grid + 1 + (1 if g_rounded else 0)
    return gamma(n) * (g.abs().sum(0) + (acc.abs() if acc is not None else 0))


def bound_proj_out_fwd(p, q, wb, bb):
    E = wb.shape[0]
    return gamma(p.shape[-1] + 1) * (bb.abs() + p.abs() @ wb.abs().t()) * _expand_prob(q.abs(), E)


def bound_grad_pooled(go, q, wb):
    E = wb.shape[0]
    return gamma(E + 1) * ((go.abs() * _expand_prob(q.abs(), E)) @ wb.abs())


def bound_grad_prob(go, p, wb, bb, D):
    E, A = wb.shape
    per = E // D
    lin = bb.abs() + p.abs() @ wb.abs().t()
    n = A + 4 + int(math.log2(max(per // 4, 1)))
    return gamma(n) * (go.abs() * lin).view(-1, D, per).sum(-1)


def proj_bounds(d, sms, acc=None):
    """Bounds of every quantity `proj_reference` returns, for fp64 inputs `d` (its keyword arguments),
    on a card with `sms` SMs; `acc` maps weight / bias gradient names to what their buffers held."""
    acc = acc or {}
    rows, E = d["x"].shape
    D = d["w_occ"].shape[0]
    grid_in, _, rpb_in = proj_launch("proj_in_bwd", rows, sms)
    grid_out, _, rpb_out = proj_launch("proj_out_bwd", rows, sms)
    gl = d["g_out"] * _expand_prob(d["prob"].abs(), E)
    return dict(
        occ=bound_proj_in_fwd(d["x"], d["w_occ"], d["b_occ"]), feat=bound_proj_in_fwd(d["x"], d["w_feat"], d["b_feat"]),
        out=bound_proj_out_fwd(d["pooled"], d["prob"], d["w_b"], d["b_b"]),
        grad_embed=bound_grad_embed(torch.cat((d["g_occ"], d["g_feat"]), 1), torch.cat((d["w_occ"], d["w_feat"]), 0)),
        grad_w_occ=bound_weight_grad(d["g_occ"], d["x"], rpb_in, grid_in, acc.get("grad_w_occ")),
        grad_b_occ=bound_bias_grad(d["g_occ"], rpb_in, grid_in, acc.get("grad_b_occ")),
        grad_w_feat=bound_weight_grad(d["g_feat"], d["x"], rpb_in, grid_in, acc.get("grad_w_feat")),
        grad_b_feat=bound_bias_grad(d["g_feat"], rpb_in, grid_in, acc.get("grad_b_feat")),
        grad_pooled=bound_grad_pooled(d["g_out"], d["prob"], d["w_b"]),
        grad_prob=bound_grad_prob(d["g_out"], d["pooled"], d["w_b"], d["b_b"], D),
        grad_w_b=bound_weight_grad(gl, d["pooled"], rpb_out, grid_out, acc.get("grad_w_b"), g_rounded=True),
        grad_b_b=bound_bias_grad(gl, rpb_out, grid_out, acc.get("grad_b_b"), g_rounded=True))


def proj_reference(x, w_occ, b_occ, w_feat, b_feat, w_b, b_b, pooled, prob, g_occ, g_feat, g_out):
    """fp64 values of everything the four kernels compute (inputs in fp64)."""
    E, D = x.shape[-1], w_occ.shape[0]
    lin = pooled @ w_b.t() + b_b
    qe = _expand_prob(prob, E)
    gl = g_out * qe
    return dict(occ=x @ w_occ.t() + b_occ, feat=x @ w_feat.t() + b_feat, out=lin * qe,
                grad_embed=g_occ @ w_occ + g_feat @ w_feat,
                grad_w_occ=g_occ.t() @ x, grad_b_occ=g_occ.sum(0), grad_w_feat=g_feat.t() @ x,
                grad_b_feat=g_feat.sum(0), grad_pooled=gl @ w_b,
                grad_prob=(g_out * lin).view(-1, D, E // D).sum(-1), grad_w_b=gl.t() @ pooled,
                grad_b_b=gl.sum(0))
