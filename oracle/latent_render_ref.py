"""CPU oracle for the LatentRendering core.  TEST INFRASTRUCTURE.

Restates projects/mmdet3d_plugin/bevformer/modules/ray_operations/latent_rendering.py:98-161
(SURVEY.md A.3) with torch ops on channel-last maps: phase 1 = transmittance product to the
cell, phase 2 = probability-weighted pooling of the lora_a feature along the ray.  Pinned by
tests/golden/latent_rendering.npz, produced by running the reference LatentRendering class in
this container (tools/make_golden_latent.py).  `latent_core_fp64` is the same operator with
the kernels' fp32 geometry and fp64 arithmetic, pinned by tests/test_oracle_latent.py."""
import numpy as np
import torch
import torch.nn.functional as F


def _cells(Hb, Wb, dtype, device="cpu"):
    ys = torch.linspace(0.5, Hb - 0.5, Hb, dtype=dtype, device=device) / Hb
    xs = torch.linspace(0.5, Wb - 0.5, Wb, dtype=dtype, device=device) / Wb
    cy, cx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([cx.reshape(-1), cy.reshape(-1)], -1)          # [HW, 2] (x, y)


def sqrt_rn(v):
    """Correctly rounded square root in v's dtype, like the kernels' __fsqrt_rn.  torch's CPU fp32 sqrt
    can be an ulp off; the fp64 root of an fp32 value always rounds to the correctly rounded fp32 root."""
    return torch.sqrt(v.double()).to(v.dtype)


def geometry(Hb, Wb, grid_num, grid_step, dtype=torch.float32, device="cpu", cells=None, sqrt=torch.sqrt):
    """The rays of every cell (or of `cells`, a slice of the Hb*Wb cell indices), in `dtype`:
    grid [n, grid_num+1, 2] (grid_sample coordinates of the waypoints, then of the cell itself),
    m1 [n, grid_num+1] phase-1 mask |g_k| < |g_cell|, m2 [n, grid_num] phase-2 mask
    |g_k| < min(1/|r_x|, 1/|r_y|).  Both masks are bool."""
    c = _cells(Hb, Wb, dtype, device)                                  # [HW,2]
    if cells is not None:
        c = c[cells]
    r = c - 0.5
    rn = torch.nan_to_num(r / sqrt((r ** 2).sum(-1, keepdim=True)))
    t = torch.from_numpy(np.arange(grid_num) + 0.5).to(dtype).to(device) * (grid_step / (min(Hb, Wb) // 2))
    way = 0.5 + rn[:, None, :] * t[None, :, None]                     # [HW,G,2]
    grid = torch.cat([way, c[:, None, :]], 1) * 2 - 1                 # [HW,G+1,2]
    length = sqrt((grid ** 2).sum(-1))                                # [HW,G+1]
    m1 = length < length[:, -1:]                                      # [HW,G+1]
    bound = torch.minimum(1 / rn[:, 0].abs(), 1 / rn[:, 1].abs())     # [HW]
    m2 = length[:, :-1] < bound[:, None]                              # [HW,G]
    return grid, m1, m2


def _activate(x, act):
    return torch.sigmoid(x) if act == "sigmoid" else 1 - torch.exp(-F.relu(x))


def latent_core(occ, feat, grid_num, grid_step, eps=1e-3, act="sigmoid", cells=None, prob_map=None):
    """occ [bs,Hb,Wb,D], feat [bs,Hb,Wb,D*G] -> prob [bs,Hb,Wb,D], pooled [bs,Hb*Wb,D*G].
    `cells` (a slice of the Hb*Wb cell indices) + `prob_map` restrict the work to a subset of
    cells for CPU timing samples (bench.py): outputs then cover only those cells."""
    bs, Hb, Wb, D = occ.shape
    Ca = feat.shape[-1]
    grid, m1, m2 = geometry(Hb, Wb, grid_num, grid_step, occ.dtype, occ.device, cells)
    g_b = grid[None].expand(bs, -1, -1, -1)
    x = F.grid_sample(occ.permute(0, 3, 1, 2), g_b, align_corners=False)     # [bs,D,HW,G+1]
    a = _activate(x, act)
    m = m1.to(occ.dtype)
    trans = torch.prod(1 - a * m[None, None], -1)                     # [bs,D,HW]
    prob = (trans * a[..., -1]).permute(0, 2, 1)
    if cells is None:
        prob = prob.reshape(bs, Hb, Wb, D)
        prob_map = prob
    # phase 2
    gw = g_b[:, :, :-1]
    fs = F.grid_sample(feat.permute(0, 3, 1, 2), gw, align_corners=False)    # [bs,Ca,HW,G]
    ps = F.grid_sample(prob_map.permute(0, 3, 1, 2), gw, align_corners=False)    # [bs,D,HW,G]
    ps = ps * m2.to(occ.dtype)[None, None]
    pi = ps / (ps.sum(-1, keepdim=True) + eps)
    n_cells = grid.shape[0]
    pooled = (fs.view(bs, D, Ca // D, n_cells, grid_num) * pi[:, :, None]).sum(-1)   # [bs,D,g,HW]
    pooled = pooled.reshape(bs, Ca, n_cells).permute(0, 2, 1)
    return prob, pooled


def latent_core_fp64(occ, feat, grid_num, grid_step, eps=1e-3, act="sigmoid"):
    """latent_core with the geometry in fp32 and everything else in fp64.

    The waypoints and both masks come from `geometry` in fp32 with correctly rounded square
    roots: the IEEE statements the CUDA kernels evaluate, so a mask can only differ from the
    kernel's where the kernel's march bounds are wrong.  Sampling, activation, product, pooling
    and normalisation run in fp64 on occ / feat; bilinear sampling with zero padding is
    continuous in position, so fp32 waypoints move the values by O(fp32 ulp) only.  Returns fp64
    prob [bs,Hb,Wb,D], pooled [bs,Hb*Wb,D*G], differentiable w.r.t. occ and feat (the grid is a
    constant)."""
    bs, Hb, Wb, D = occ.shape
    Ca = feat.shape[-1]
    grid, m1, m2 = geometry(Hb, Wb, grid_num, grid_step, sqrt=sqrt_rn)
    occ, feat = occ.double(), feat.double()
    g_b = grid.double()[None].expand(bs, -1, -1, -1)
    a = _activate(F.grid_sample(occ.permute(0, 3, 1, 2), g_b, align_corners=False), act)    # [bs,D,HW,G+1]
    trans = torch.prod(1 - a * m1.double()[None, None], -1)           # [bs,D,HW]
    prob = (trans * a[..., -1]).permute(0, 2, 1).reshape(bs, Hb, Wb, D)
    gw = g_b[:, :, :-1]
    fs = F.grid_sample(feat.permute(0, 3, 1, 2), gw, align_corners=False)    # [bs,Ca,HW,G]
    ps = F.grid_sample(prob.permute(0, 3, 1, 2), gw, align_corners=False) * m2.double()[None, None]
    pi = ps / (ps.sum(-1, keepdim=True) + eps)
    pooled = (fs.view(bs, D, Ca // D, Hb * Wb, grid_num) * pi[:, :, None]).sum(-1)   # [bs,D,g,HW]
    return prob, pooled.reshape(bs, Ca, Hb * Wb).permute(0, 2, 1)
