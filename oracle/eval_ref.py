"""CPU oracle for ViDAR's evaluation metrics.  TEST INFRASTRUCTURE.

Vectorised numpy restatement of utils/eval_utils.py:17-225 (clamp / _clamp without the per-ray loop,
spherical_projection, compute_ray_errors), utils/e2e_predictor_utils.py:146-183
(compute_chamfer_distance_inner) and the per-pair loop of detectors/vidar.py:452-497.  float32 throughout, as
the reference evaluates it; arctan2 is evaluated in fp64 and rounded to fp32 (the one statement whose last bit
depends on the math library); error sums are fp64.  NN searches use knn_ref.nn.  Pinned by tests/golden/eval.npz,
made by running the reference's own eval_utils.py (tools/make_golden_eval.py)."""
import numpy as np

from . import knn_ref

f32 = np.float32
PC_RANGE = [-70.0, -70.0, -4.5, 70.0, 70.0, 4.5]
MAX_VALUE = f32(1e8)
# numpy compares float32 arrays with Python floats in float32 (NEP 50)
_LO = np.array(PC_RANGE[:3], f32)
_HI = np.array(PC_RANGE[3:], f32)
_SLO = np.array([v - 0.02 for v in PC_RANGE[:3]], f32)
_SHI = np.array([v + 0.02 for v in PC_RANGE[3:]], f32)


def atan2_f32(y, x):
    return np.arctan2(np.asarray(y, np.float64), np.asarray(x, np.float64)).astype(f32)


def _norm(v):
    return np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])


def spherical_projection(pcd):
    pcd = np.asarray(pcd, f32)
    return atan2_f32(pcd[:, 0], pcd[:, 1]), atan2_f32(pcd[:, 2], pcd[:, 1]), _norm(pcd)


def inside_volume(p):
    return ((_SLO <= p) & (p <= _SHI)).all(-1)


def _visit_planes(t, start, step, active, record):
    """Visit the 6 planes of every ray in ascending distance (ties: lower plane index) and stop at the first one
    with t + 1e-4 >= 0 whose intersection start + t * step lies inside the volume; record(mask, t, x)."""
    order = np.argsort(t, axis=0, kind="stable")
    cols = np.arange(t.shape[1])
    done = ~active
    for r in range(6):
        tk = t[order[r], cols]
        x = start + tk[:, None] * step
        acc = ~done & (tk + f32(1e-4) >= 0) & inside_volume(x)
        record(acc, tk, x)
        done |= acc
    return done


def _plane_distances(start, d, sign):
    t = np.empty((6, len(d)), f32)
    for k in range(6):
        a = k // 2
        bound = (_HI if k & 1 else _LO)[a]
        with np.errstate(invalid="ignore", divide="ignore"):
            t[k] = np.where(np.abs(d[:, a]).astype(np.float64) <= 1e-8, MAX_VALUE,
                            (bound - start[:, a]) / (d[:, a] if sign > 0 else -d[:, a]))
    return t


def _clamp(points, origin):
    """_clamp (:81-174) for all rays at once -> (new_origin, points); raises like the reference."""
    points = points.copy()
    e = points - origin
    if (e == 0).all(1).any():
        raise RuntimeError("Origin and the end point should not be identical")
    with np.errstate(invalid="ignore", divide="ignore"):
        l = _norm(e)
        d = e / l[:, None]
    new_origin = np.broadcast_to(origin, points.shape).copy()
    hit = np.ones(len(points), bool)
    if not inside_volume(origin[0]):
        hit[:] = False
        org = np.broadcast_to(origin, points.shape)

        def rec(acc, tk, x):
            new_origin[acc] = x[acc]
            far = acc & (tk > l)
            points[far] = x[far]
            hit[acc] = True
        with np.errstate(invalid="ignore", over="ignore"):
            _visit_planes(_plane_distances(org, d, +1), org, d, np.ones(len(points), bool), rec)
    points[~hit] = np.inf
    new_origin[~hit] = np.inf
    need = hit & ~inside_volume(points)
    if need.any():
        t = _plane_distances(points, d, -1)

        def rec2(acc, tk, x):
            points[acc] = x[acc]
        with np.errstate(invalid="ignore", over="ignore"):
            done = _visit_planes(t, points.copy(), -d, need, rec2)
        if not done.all():
            raise AssertionError("a clamped ray does not touch the volume")
    return new_origin, points


def clamp(pcd, origin):
    """clamp(..., return_invalid_mask=True) (:39-78) -> (origins, points, invalid)."""
    pcd = np.array(pcd, f32)
    origin = np.asarray(origin, f32).reshape(1, 3)
    inner = ((_LO <= pcd) & (pcd <= _HI)).all(1)
    origins = np.zeros_like(pcd) + origin
    if (~inner).any():
        o, p = _clamp(pcd[~inner], origin)
        pcd[~inner] = p
        origins[~inner] = o
    invalid = np.isinf(pcd).all(1) | np.isnan(pcd).all(1)
    return origins, pcd, invalid


def compute_ray_errors(pred_pcd, gt_pcd, origin, return_intermediates=False):
    """eval_utils.compute_ray_errors -> (l1, absrel) as fp64 (sums in fp64), optionally with the
    intermediates: kept masks, NN index into the kept pred points, interpolated and clamped points."""
    pred_pcd, gt_pcd = np.asarray(pred_pcd, f32), np.asarray(gt_pcd, f32)
    origin = np.asarray(origin, f32).reshape(3)
    th_h, ph_h, d_h = spherical_projection(pred_pcd - origin[None])
    th, ph, d = spherical_projection(gt_pcd - origin[None])
    mask_hat, mask = d_h > f32(1e-2), d > f32(1e-2)
    count = int(mask.sum())
    if count and not mask_hat.any():
        raise ValueError("gt points are kept but no pred point is")
    ps = np.stack([th_h[mask_hat], ph_h[mask_hat], np.ones(int(mask_hat.sum()), f32)], 1)
    gs = np.stack([th[mask], ph[mask], np.ones(count, f32)], 1)
    if count:
        _, idx = knn_ref.nn(gs[None], ps[None])
        idx = idx[0]
    else:
        idx = np.zeros(0, np.int64)
    gt = gt_pcd[mask]
    v = gt - origin[None]
    unit = v / np.sqrt((v * v).sum(1, keepdims=True))
    interp = origin[None] + d_h[mask_hat][idx][:, None] * unit
    go, gc, invalid = clamp(gt, origin)
    _, ic, _ = clamp(interp, origin)
    keep = ~invalid
    dc = _norm(gc[keep] - go[keep])
    valid = dc > f32(0.01)
    l1 = _norm(gc[keep][valid] - ic[keep][valid])
    absrel = l1 / dc[valid]
    with np.errstate(invalid="ignore", divide="ignore"):
        res = (np.float64(l1.astype(np.float64).sum()) / count, np.float64(absrel.astype(np.float64).sum()) / count)
    if not return_intermediates:
        return res
    return res, dict(mask_hat=mask_hat, mask=mask, idx=idx, interp=interp, clamped_gt=gc, clamped_interp=ic,
                     invalid=invalid, count=count)


def get_inside_mask(points, pc_range):
    p = np.asarray(points, f32)
    lo, hi = np.array(pc_range[:3], f32), np.array(pc_range[3:], f32)
    return ((lo <= p) & (p <= hi)).all(-1)


def compute_chamfer_distance_inner(pred_pcd, gt_pcd, pc_range):
    """0.0 if either side has no inside point, else (sum fwd / n_pred + sum bwd / n_gt) / 2 (fp64 sums of the
    fp32 squared NN distances)."""
    pred, gt = np.asarray(pred_pcd, f32), np.asarray(gt_pcd, f32)
    p, g = pred[get_inside_mask(pred, pc_range)], gt[get_inside_mask(gt, pc_range)]
    if len(p) == 0 or len(g) == 0:
        return 0.0
    fd, _ = knn_ref.nn(p[None], g[None])
    bd, _ = knn_ref.nn(g[None], p[None])
    return float((fd.astype(np.float64).sum() / len(p) + bd.astype(np.float64).sum() / len(g)) / 2.0)


def decode_clouds(depth, rays, points, tindex, origin_vox, origin, scale, within_grid=False, pc_range=None):
    """ray_head.decode_clouds (the arg-max decode's clouds of every (sample, frame), eval_metrics.cu) in fp32
    statements of the kernel's order: gt_dist = norm3(ray - origin_vox) * scale, a row joins cloud b * F + t when
    its tindex t is a frame in [0, F), gt_dist > 0 and (within_grid) its metre point is inside pc_range; a cloud
    holds its rows in their original order, both points o + ((p - o) / norm3(p - o)) * dist with dist = depth *
    scale (pred) and gt_dist (gt); rows past the last cloud are NaN.  norm3(v) = sqrt((x*x + y*y) + z*z).
    -> pred, gt [bs * M, 3], off [bs * F + 2] int64."""
    depth, rays, points, tindex = (np.asarray(a, f32) for a in (depth, rays, points, tindex))
    origin_vox, origin = np.asarray(origin_vox, f32), np.asarray(origin, f32)
    scale = f32(scale)
    bs, M = depth.shape
    F = origin.shape[1]
    pred = np.full((bs * M, 3), np.nan, f32)
    gt = np.full((bs * M, 3), np.nan, f32)
    off = np.zeros(bs * F + 2, np.int64)
    n3 = lambda v: np.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])
    row = 0
    for b in range(bs):
        t = tindex[b]
        with np.errstate(invalid="ignore"):
            frame = (t >= 0) & (t < f32(F)) & (t == np.floor(t))
        f = np.where(frame, t, 0).astype(np.int64)
        gd = n3(rays[b] - origin_vox[b, f]) * scale
        keep = frame & (gd > 0)
        if within_grid:
            keep &= get_inside_mask(points[b], pc_range)
        for fr in range(F):
            sel = np.nonzero(keep & (f == fr))[0]
            o = origin[b, fr]
            v = points[b, sel] - o
            u = v / n3(v)[:, None]
            pred[row:row + len(sel)] = o + u * (depth[b, sel] * scale)[:, None]
            gt[row:row + len(sel)] = o + u * gd[sel][:, None]
            row += len(sel)
            off[b * F + fr + 1] = row
    off[bs * F + 1] = bs * M
    return pred, gt, off


def frame_metrics(pred_pcds, gt_pcds, origin, pc_range, start_idx=0):
    """vidar.py:452-497's per-pair loop on the oracle functions."""
    origin = np.asarray(origin, f32)
    ret = {}
    for f in range(len(pred_pcds[0])):
        d = dict(count=0, chamfer_distance=0.0, l1_error=0.0, absrel_error=0.0)
        for b in range(len(pred_pcds)):
            d["chamfer_distance"] += compute_chamfer_distance_inner(pred_pcds[b][f], gt_pcds[b][f], pc_range)
            l1, absrel = compute_ray_errors(pred_pcds[b][f], gt_pcds[b][f], origin[b, f])
            d["l1_error"] += float(l1)
            d["absrel_error"] += float(absrel)
            d["count"] += 1
        ret[f"frame.{f + start_idx}"] = d
    return ret
