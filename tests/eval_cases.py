"""Seeded inputs for ViDAR's evaluation metrics (tools/make_golden_eval.py stores them in tests/golden/eval.npz).

LiDAR-like clouds: 32 beams from -30 to +10 degrees elevation, ranges 2-70 m; pred = gt moved along and across
the rays with points dropped.  The frames cover every branch of the reference's metric code:
  0-2  plain frames, some points beyond +-70 m and above 4.5 m (clamping), a few within 1e-2 m of the origin
  3    axis-aligned rays far outside the volume (the isclose branch of _clamp)
  4    origin outside the volume (the first loop of _clamp; rays that miss become invalid)
  5    repeated directions: pred points duplicated and scaled by 2 along the same ray (spherical ties)
  6    no point inside the model's point-cloud range (the 0.0 Chamfer branch)
"""
import numpy as np

PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
F32 = np.float32


def lidar(rng, n, origin, rmin=2.0, rmax=70.0):
    elev = np.deg2rad(rng.integers(0, 32, n) * (40.0 / 31.0) - 30.0)
    az = rng.uniform(-np.pi, np.pi, n)
    r = rng.uniform(rmin, rmax, n)
    d = np.stack([np.cos(elev) * np.cos(az), np.cos(elev) * np.sin(az), np.sin(elev)], 1)
    return (origin[None].astype(np.float64) + r[:, None] * d).astype(F32)


def perturb(rng, gt, origin, drop=0.1):
    v = gt.astype(np.float64) - origin
    r = np.linalg.norm(v, axis=1, keepdims=True)
    u = v / np.maximum(r, 1e-9)
    r2 = r * rng.uniform(0.85, 1.15, r.shape) + rng.normal(0, 0.3, r.shape)
    side = rng.normal(0, 0.01, v.shape)
    p = origin + np.abs(r2) * (u + side)
    keep = rng.random(len(p)) > drop
    return p[keep].astype(F32)


def frame(rng, n, origin, far=0.05, near=3):
    origin = np.asarray(origin, F32)
    gt = lidar(rng, n, origin)
    k = int(far * n)
    gt[:k] = lidar(rng, k, origin, 70.0, 100.0)           # beyond +-70 m / above 4.5 m
    pred = perturb(rng, gt, origin.astype(np.float64))
    gt[k:k + near] = origin + rng.uniform(-4e-3, 4e-3, (near, 3)).astype(F32)
    pred[:near] = origin + rng.uniform(-4e-3, 4e-3, (near, 3)).astype(F32)
    return pred, gt, origin


def cases(n=1500, seed=0):
    """-> list of (pred [P,3], gt [G,3], origin [3]) float32 triples, one per frame."""
    rng = np.random.default_rng(seed)
    out = [frame(rng, n, [0.5, -1.25, 1.75]), frame(rng, n + 137, [3.0, 2.5, 1.5]), frame(rng, n - 211, [-10.0, 20.0, 1.0])]
    # 3: axis-aligned rays from an origin on the grid, far outside the volume
    pred, gt, o = frame(rng, n, [0.0, 0.0, 1.0])
    ax = []
    for a in range(3):
        for s in (-1.0, 1.0):
            for r in (80.0, 120.0) if a < 2 else (6.0, 9.0):
                p = o.astype(np.float64).copy()
                p[a] += s * r
                ax.append(p)
    ax = np.array(ax, F32)
    gt = np.concatenate([ax, gt])
    pred = np.concatenate([(o + (ax - o) * F32(0.5)).astype(F32), pred])
    out.append((pred, gt, o))
    # 4: origin outside the volume; some rays enter it, some miss
    o4 = np.array([85.0, 10.0, 1.5], F32)
    gt = lidar(rng, n, o4, 2.0, 160.0)
    out.append((perturb(rng, gt, o4.astype(np.float64)), gt, o4))
    # 5: repeated directions -- grid-exact offsets so 2 * v is exact and arctan2 sees the same ratios
    o5 = np.array([1.0, -2.0, 0.5], F32)
    v = (rng.integers(-2048, 2048, (n, 3)) / 64.0).astype(F32)
    v[:, 2] /= 8
    gt = (o5 + v).astype(F32)
    base = (o5 + v[::3] * F32(0.75)).astype(F32)
    pred = np.concatenate([base, base, (o5 + v[::3] * F32(1.5)).astype(F32), (o5 + v[1::3]).astype(F32)])
    out.append((pred, gt, o5))
    # 6: nothing inside PC_RANGE (everything above z = 3 m)
    o6 = np.array([0.0, 0.0, 1.0], F32)
    gt = lidar(rng, n // 4, o6, 5.0, 40.0)
    gt[:, 2] = np.abs(gt[:, 2]) + F32(3.5)
    pred = perturb(rng, gt, o6.astype(np.float64))
    pred[:, 2] = np.abs(pred[:, 2]) + F32(3.5)
    out.append((pred, gt, o6))
    return out
