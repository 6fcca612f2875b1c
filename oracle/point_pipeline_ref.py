"""numpy restatement of a pre-training sample's point half given its draws: the multi-sweep merge
(loading.py:115-223), mmdet3d 0.17.1's first-occurrence voxel sampler with max_points = 1 and union2one's ego mask /
queue-index column (nuscenes_vidar_dataset_v1.py:22-36, 57-70, 199-200).  It reads the plans that
vidar_b200.point_pipeline's transforms record (segments, the composed shuffle order, the VoxelGenerator
parameters) and is the reference of the GPU tests; the golden (tools/make_golden_point_pipeline.py) checks it
against the reference's own statements.

Parity notes, each one a statement of the reference restated here:
  * the sweep transform is `pts[:, :3] @ R.T` in float64, rounded to float32 on assignment, then `+= t` in float64
    and rounded again; the dot is summed (x R[i,0] + y R[i,1]) + z R[i,2] with every product rounded;
  * the filters compare float32 coordinates with float32 bounds (numpy's casting of a Python float against a
    float32 array; torch's likewise in union2one);
  * the voxel coordinate is floor(f32(f32(p - lo) / vs)) with float32 lo / vs, inside when 0 <= c < grid, with
    grid = round(f32(hi - lo) / vs)."""
import numpy as np

F32 = np.float32


def keep_mask(raw, filt):
    """CustomLoadPointsFromMultiSweeps._remove_close: not (|x| < 1 and |y| < 1), then outside the ego box."""
    if filt is None:
        return np.ones(raw.shape[0], bool)
    x, y = raw[:, 0], raw[:, 1]
    keep = ~((np.abs(x) < F32(1.0)) & (np.abs(y) < F32(1.0)))
    if len(filt):
        b = [F32(v) for v in filt]
        keep &= ~((b[0] <= x) & (b[2] >= x) & (b[1] <= y) & (b[3] >= y))
    return keep


def sweep_transform(pts, R, t):
    """f32(f32(dot64(p, R[i])) + t[i]) for the three coordinates of float32 pts [n, >= 3]."""
    out = pts.copy()
    x, y, z = (pts[:, j].astype(np.float64) for j in range(3))
    for i in range(3):
        dot = (x * R[i, 0] + y * R[i, 1]) + z * R[i, 2]
        out[:, i] = (dot.astype(F32).astype(np.float64) + t[i]).astype(F32)
    return out


def merged(plan):
    """The frame's current points [M, 5] float32 in the reference's concatenation order (all of them for a frame
    without the sampler)."""
    segs = plan.current() if plan.perm is not None else plan.segments
    parts = []
    for s in segs:
        p = s.raw[keep_mask(s.raw, s.filt)]
        parts.append(sweep_transform(p, s.R, s.t) if s.R is not None else p.copy())
    return np.concatenate(parts, 0) if parts else np.zeros((0, 5), F32)


def first_voxels(pts, lo, vs, grid, max_voxels):
    """Indices into pts (in pts' order) of the points that first meet their voxel, at most max_voxels of them:
    _points_to_voxel_reverse_kernel with max_points = 1."""
    lo, vs = np.asarray(lo, F32), np.asarray(vs, F32)
    c = np.floor((pts[:, :3] - lo) / vs)
    inside = np.all((c >= 0) & (c < np.asarray(grid)), 1)
    idx = np.nonzero(inside)[0]
    ci = c[idx].astype(np.int64)
    cell = (ci[:, 2] * grid[1] + ci[:, 1]) * grid[0] + ci[:, 0]
    _, first = np.unique(cell, return_index=True)
    return idx[np.sort(first)][:max_voxels]


def frame_points(plan):
    """The frame's sampled points [n, 5] (its `results['points']` after the pipeline)."""
    pts = merged(plan)
    if plan.perm is None:
        return pts
    cur = pts[plan.perm]
    return cur[first_voxels(cur, plan.lo, plan.voxel_size, plan.grid, plan.max_voxels)]


def ego_keep(pts, ego_mask):
    """union2one's _mask_points: keep the points outside the box (float32 comparisons)."""
    if ego_mask is None:
        return np.ones(pts.shape[0], bool)
    b = [F32(v) for v in ego_mask]
    x, y = pts[:, 0], pts[:, 1]
    return ~((b[0] <= x) & (b[2] >= x) & (b[1] <= y) & (b[3] >= y))


def gather(plans, ego_mask, padded=False):
    """gt_points of the frames' plans in queue order: [sum M, 5] float32, or with `padded` the device's padded form
    [R, 5] (each frame's sampled rows in order, masked and unused rows NaN)."""
    out = []
    for i, plan in enumerate(plans):
        pts = frame_points(plan)
        keep = ego_keep(pts, ego_mask)
        pts = pts.copy()
        pts[:, -1] = i
        if padded:
            n_cur = plan.perm.shape[0] if plan.perm is not None else pts.shape[0]
            cap = min(n_cur, plan.max_voxels) if plan.perm is not None else n_cur
            rows = np.full((cap, 5), np.nan, F32)
            rows[np.nonzero(keep)[0]] = pts[keep]
            out.append(rows)
        else:
            out.append(pts[keep])
    return np.concatenate(out, 0) if out else np.zeros((0, 5), F32)


def counts(plans):
    """Per frame (merged points, sampled points) -> int [F, 2]."""
    res = []
    for plan in plans:
        m = merged(plan).shape[0]
        res.append((m, frame_points(plan).shape[0]))
    return np.array(res, np.int64).reshape(-1, 2)
