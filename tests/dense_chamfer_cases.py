"""Seeded cases of the head's dense Chamfer term (tools/make_golden_dense_chamfer.py and the tests).

Every case is what ViDARHeadBase.loss is called with (GT point lists in metres, origins, the grid) plus the
decoded ray lengths `dist` [bs, F*R0] that the gumbel decode would return, supplied directly so that the loss
and its gradient in dist can be compared."""
import numpy as np
import torch

from tests import head_cases as hc

FRAMES = 2
LOSS_W = [[0.7], [1.3]]
# 1 m voxels over power-of-two extents (metres -> voxels is exact); dense ray ends at voxel 2, 6, 10, 14
GRID = dict(bev_h=16, bev_w=16, z=8, pc_range=[-8.0, -8.0, -4.0, 8.0, 8.0, 4.0])
NAMES = ("head", "gt_outside", "faces", "dist_zero", "within_grid", "bs2_ragged", "ties")


def rays_per_frame(c):
    return (c["bev_h"] // 4) * (c["bev_w"] // 4) * (c["z"] // 4)


def _points(g, n, lo, hi, frames):
    xyz = torch.tensor(lo) + (torch.tensor(hi) - torch.tensor(lo)) * torch.rand(n, 3, generator=g)
    t = torch.randint(0, frames + 1, (n, 1), generator=g).float()          # frame `frames` is not predicted
    return torch.cat([xyz, torch.rand(n, 1, generator=g), t], 1)


def case(name):
    """-> dict(bev_h, bev_w, z, pc_range, bs, preds, gt_points, origin, dist, within)."""
    g = torch.Generator().manual_seed(NAMES.index(name) + 100)
    if name == "head":
        h = hc.case()
        c = dict(bev_h=hc.BEV_H, bev_w=hc.BEV_W, z=hc.Z, pc_range=hc.PC_RANGE, bs=hc.BS,
                 preds=h["pred_dict"]["next_bev_preds"], gt_points=h["gt_points"], origin=h["origin"], within=False)
    else:
        c = dict(GRID, within=name == "within_grid")
        r = c["pc_range"]
        lo, hi = [r[0] - 1.0, r[1] - 1.0, r[2] - 0.5], [r[3] + 1.0, r[4] + 1.0, r[5] + 0.5]
        sizes = {"bs2_ragged": (400, 12)}.get(name, (150,))
        c["bs"] = len(sizes)
        c["gt_points"] = [_points(g, n, lo, hi, FRAMES) for n in sizes]
        c["origin"] = 0.6 * torch.randn(c["bs"], FRAMES, 3, generator=g)
        if name == "gt_outside":        # frame 1: every GT point beyond the box (x > W - 1 in voxel units)
            p = c["gt_points"][0]
            p[p[:, 4] == 1, 0] = r[3] - 0.5 + 2.0 * torch.rand(int((p[:, 4] == 1).sum()), generator=g)
        if name == "faces":             # x exactly on the faces x = 0 and x = W - 1 (excluded), y / z inside
            p = c["gt_points"][0]
            p[:20, 0] = r[0]
            p[20:40, 0] = r[0] + (c["bev_w"] - 1)
            p[:40, 4] = torch.arange(40).float() % FRAMES
            p[:40, 1:3] = p[:40, 1:3].clamp(min=torch.tensor(r[1:3]) + 1.5, max=torch.tensor(r[4:6]) - 1.5)
        if name == "ties":              # origin on a ray centre: collinear rays, equal lengths -> duplicate pred points
            c["origin"] = torch.tensor([[[2.0, -2.0, -2.0], [2.0, -2.0, -2.0]]])     # voxel (10, 6, 2)
            p = c["gt_points"][0]
            c["gt_points"][0] = torch.cat([p, p[:30], p[10:20]])                    # duplicate GT points
        c["preds"] = torch.randn(FRAMES, 1, c["bs"], c["bev_h"] * c["bev_w"], c["z"], generator=g)
    R = rays_per_frame(c) * FRAMES
    dist = 0.5 + 8.0 * torch.rand(c["bs"], R, generator=g)
    if name == "dist_zero":
        dist[torch.rand(c["bs"], R, generator=g) < 0.3] = 0.0
    if name == "ties":
        dist[:] = 3.0
        dist[0, 6::rays_per_frame(c)] = 0.0           # the ray ending at the origin itself (direction 0 / 0)
    c["dist"] = dist
    return c


def call_kw(c):
    return dict(start_idx=0, tgt_bev_h=c["bev_h"], tgt_bev_w=c["bev_w"], tgt_pc_range=c["pc_range"])
