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


def _nearest(q, c, block=1024):
    """Index of the nearest c row of every q row (the first on ties) and that squared distance, summed in x, y, z
    order in fp32; queries in blocks of `block` rows, so memory stays at block * len(c)."""
    idx = np.zeros(len(q), np.int64)
    dmin = np.zeros(len(q), f32)
    for s in range(0, len(q), block):
        a = q[s:s + block]
        d = (a[:, None, 0] - c[None, :, 0]) ** 2
        d = d + (a[:, None, 1] - c[None, :, 1]) ** 2
        d = d + (a[:, None, 2] - c[None, :, 2]) ** 2
        j = np.argmin(d, axis=1)
        idx[s:s + block] = j
        dmin[s:s + block] = d[np.arange(len(a)), j]
    return idx, dmin


def dense_chamfer(dist, points, origin, gt, gt_tindex, grid, frame_weights, weight_sum, eval_within_grid=False,
                  pc_range=None, return_pairs=False):
    """Arguments as vidar_b200.ray_head.dense_chamfer_loss, as numpy arrays (float32, or float64 whose values are
    then used as they are) -> (loss float, grad_dist float64 [bs, F*R0]) and, with return_pairs, the per-pair sums
    of dense_chamfer_groups."""
    F = len(frame_weights)
    bs, FR = np.asarray(dist).shape
    To = np.asarray(origin).shape[1]
    b, f = np.divmod(np.arange(bs * F), F)
    pairs = np.stack([b, f, b * To + f, np.zeros_like(b)], 1)
    loss, grad, sums = dense_chamfer_groups(
        np.asarray(dist).reshape(-1), np.asarray(points).reshape(-1, 3), np.asarray(origin).reshape(-1, 3), gt,
        gt_tindex, grid, pairs, [frame_weights[k] for k in f], [1.0], eval_within_grid, pc_range,
        norm_fn=lambda _: float(weight_sum) * bs)
    return (float(loss[0]), grad.reshape(bs, FR)) + ((sums,) if return_pairs else ())


def dense_chamfer_groups(dist, points, origin, gt, gt_tindex, grid, pairs, pair_weights, group_norms,
                         eval_within_grid=False, pc_range=None, norm_fn=None):
    """Arguments as vidar_b200.ray_head.dense_chamfer_group_loss, as numpy arrays -> (loss float [groups], the
    fp64 gradient of loss.sum() in dist [P*R0], pair sums [P, 4] float64: sum over kept pred points of the fp32
    squared distance to the nearest gt point, their count, the same from gt to pred; a sum over points without a
    nearest point is NaN)."""
    arrays = [np.asarray(a) for a in (dist, points, origin, gt, gt_tindex)]
    dist64, points64, origin64, gt64, _ = (a.astype(np.float64) for a in arrays)
    dist, points, origin, gt, gt_tindex = (a.astype(f32) for a in arrays)
    W, H, Z = grid
    pairs = np.asarray(pairs, np.int64).reshape(-1, 4)
    P = len(pairs)
    R0 = len(dist) // P
    groups = len(group_norms)
    leaf = torch.tensor(dist64, requires_grad=True)
    total = [torch.zeros((), dtype=torch.float64) for _ in range(groups)]
    sums = np.zeros((P, 4))
    for n, (s, f, orow, grp) in enumerate(pairs):
        o = origin[orow]
        rays = slice(n * R0, (n + 1) * R0)
        p, d = points[rays], dist[rays]
        keep = d > 0
        if eval_within_grid:
            lo, hi = np.asarray(pc_range[:3], f32), np.asarray(pc_range[3:], f32)
            keep &= ((lo <= p) & (p <= hi)).all(-1)
        g = gt[s]
        sel = ((gt_tindex[s] == f) & (g[:, 0] < W - 1) & (g[:, 0] > 0) & (g[:, 1] < H - 1) & (g[:, 1] > 0)
               & (g[:, 2] < Z - 1) & (g[:, 2] > 0))
        g = g[sel]
        rows = np.nonzero(keep)[0]
        sums[n, 1], sums[n, 3] = len(rows), len(g)
        if len(g) == 0:
            sums[n, 0] = np.nan if len(rows) else 0.0
            continue
        if len(rows) == 0:
            sums[n, 2] = np.nan
            total[grp] = total[grp] + float("nan")
            continue
        pred32 = ((o + _unit(p[rows], o) * d[rows, None]) - o) * f32(0.1)
        gt32 = (g - o) * f32(0.1)
        (i_pg, d_pg), (i_gp, d_gp) = _nearest(pred32, gt32), _nearest(gt32, pred32)
        sums[n, 0], sums[n, 2] = d_pg.astype(np.float64).sum(), d_gp.astype(np.float64).sum()
        o64 = torch.from_numpy(origin64[orow])
        u64 = torch.from_numpy(_unit(points64[n * R0 + rows], origin64[orow]))
        pred = ((o64 + u64 * leaf[n * R0 + rows][:, None]) - o64) * 0.1
        gtc = (torch.from_numpy(gt64[s][sel]) - o64) * 0.1
        src = ((pred - gtc[i_pg]) ** 2).sum(-1).mean()
        dst = ((gtc - pred[i_gp]) ** 2).sum(-1).mean()
        total[grp] = total[grp] + (src + dst) / 2 * float(pair_weights[n])
    norm = norm_fn or (lambda g: float(group_norms[g]))
    loss = torch.stack([total[g] / norm(g) for g in range(groups)])
    if loss.requires_grad:
        loss.sum().backward()
    grad = leaf.grad.numpy() if leaf.grad is not None else np.zeros(dist.shape)
    return loss.detach().numpy(), grad, sums
