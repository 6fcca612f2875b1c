"""fp64 oracle of the head's dense Chamfer term.  TEST INFRASTRUCTURE.

Restates the `use_dense_loss` branch of ViDARHeadBase.loss after the gumbel decode (vidar_head_base.py:638-659,
get_rendered_pcds :344-389, mmdet3d chamfer_distance with criterion 'l2', reduction 'mean') per (sample, frame)
pair.  Which points enter a cloud and which neighbour is nearest are decided on the fp32 values the reference
computes (first index on ties, like torch.min); the loss is then evaluated in fp64 from a float64 leaf `dist`,
and its gradient comes from fp64 autograd.  Pinned by tests/golden/dense_chamfer.npz, made by running the
reference's own loss (tools/make_golden_dense_chamfer.py)."""
import numpy as np
import torch

f32 = np.float32


def _unit(p, o):
    r = p - o
    return r / np.sqrt((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2])[:, None]


def _nearest(q, c):
    """Index of the nearest c row of every q row, squared distance summed in x, y, z order in fp32."""
    d = (q[:, None, 0] - c[None, :, 0]) ** 2
    d = d + (q[:, None, 1] - c[None, :, 1]) ** 2
    d = d + (q[:, None, 2] - c[None, :, 2]) ** 2
    return np.argmin(d, axis=1)


def dense_chamfer(dist, points, origin, gt, gt_tindex, grid, frame_weights, weight_sum, eval_within_grid=False,
                  pc_range=None):
    """Arguments as vidar_b200.ray_head.dense_chamfer_loss, as numpy arrays (float32, or float64 whose values are
    then used as they are) -> (loss float, grad_dist float64 [bs, F*R0])."""
    arrays = [np.asarray(a) for a in (dist, points, origin, gt, gt_tindex)]
    dist64, points64, origin64, gt64, _ = (a.astype(np.float64) for a in arrays)
    dist, points, origin, gt, gt_tindex = (a.astype(f32) for a in arrays)
    W, H, Z = grid
    F = len(frame_weights)
    bs, FR = dist.shape
    R0 = FR // F
    leaf = torch.tensor(dist64, requires_grad=True)
    total = torch.zeros((), dtype=torch.float64)
    for b in range(bs):
        for f in range(F):
            o = origin[b, f]
            p, d = points[b, f * R0:(f + 1) * R0], dist[b, f * R0:(f + 1) * R0]
            keep = d > 0
            if eval_within_grid:
                lo, hi = np.asarray(pc_range[:3], f32), np.asarray(pc_range[3:], f32)
                keep &= ((lo <= p) & (p <= hi)).all(-1)
            g = gt[b]
            sel = ((gt_tindex[b] == f) & (g[:, 0] < W - 1) & (g[:, 0] > 0) & (g[:, 1] < H - 1) & (g[:, 1] > 0)
                   & (g[:, 2] < Z - 1) & (g[:, 2] > 0))
            g = g[sel]
            if len(g) == 0:
                continue
            rows = np.nonzero(keep)[0]
            if len(rows) == 0:
                total = total + float("nan")
                continue
            pred32 = ((o + _unit(p[rows], o) * d[rows, None]) - o) * f32(0.1)
            gt32 = (g - o) * f32(0.1)
            i_pg, i_gp = _nearest(pred32, gt32), _nearest(gt32, pred32)
            o64 = torch.from_numpy(origin64[b, f])
            u64 = torch.from_numpy(_unit(points64[b, f * R0 + rows], origin64[b, f]))
            pred = ((o64 + u64 * leaf[b, f * R0 + rows][:, None]) - o64) * 0.1
            gtc = (torch.from_numpy(gt64[b][sel]) - o64) * 0.1
            src = ((pred - gtc[i_pg]) ** 2).sum(-1).mean()
            dst = ((gtc - pred[i_gp]) ** 2).sum(-1).mean()
            total = total + (src + dst) / 2 * float(frame_weights[f])
    loss = total / (float(weight_sum) * bs)
    if loss.requires_grad:
        loss.backward()
        grad = leaf.grad.numpy()
    else:
        grad = np.zeros(dist.shape)
    return float(loss.detach()), grad
