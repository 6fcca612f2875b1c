"""The point half of a pre-training sample: `vidar_b200.point_pipeline` (host draws on index vectors, then one
device pass) against the reference's host statements, per frame and per sample.

A sample runs the train pipeline 10 times (4 previous frames and the current one, then the current one again and
4 future frames); union2one keeps 8 of the runs' points.  Each frame is a LiDAR-like key frame and 2 sweeps of
35 000 points (`synthetic.lidar_cloud`).  File reads are replaced by preloaded arrays on both sides.

Reported: host wall clock to a synchronised gt_points (ours: draws + pack + upload + device pass; the reference:
the multi-sweep statements, mmdet3d's two 2-D shuffles, the voxel sampler, union2one's mask and concatenation,
and the upload of the result), device time of the pass by CUDA events, and bytes uploaded.  The reference's
statements are restated in `reference_frame` (its voxeliser as the oracle's vectorised first-occurrence, which
returns numba's points); the shuffles, which dominate, are the reference's own calls.

    python tools/bench_point_pipeline.py [--points 35000] [--out /tmp/bench_point_pipeline.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import point_pipeline_ref  # noqa: E402
from tools.gpu_timing import card, event_ms, host_ms  # noqa: E402
from vidar_b200 import point_pipeline as pp  # noqa: E402
from vidar_b200 import pretrain, synthetic  # noqa: E402

EGO = (-0.8, -1.5, 0.8, 2.5)
RUNS, KEPT = 10, 8


def reference_frame(key, sweeps, ts, sampler):
    """The reference's host statements for one frame (loading.py:129-165, 216-223, mmdet3d's
    VoxelBasedPointSampler.__call__) -> sampled float32 [n, 5]."""
    points = key.copy()
    points[:, 4] = 0
    parts = [points]
    for raw, R, t, sts in sweeps:
        p = np.copy(raw)
        x, y = p[:, 0], p[:, 1]
        p = p[np.logical_not(np.logical_and(np.abs(x) < 1.0, np.abs(y) < 1.0))]
        ego = np.logical_and(np.logical_and(EGO[0] <= p[:, 0], EGO[2] >= p[:, 0]),
                             np.logical_and(EGO[1] <= p[:, 1], EGO[3] >= p[:, 1]))
        p = p[np.logical_not(ego)]
        p[:, :3] = p[:, :3] @ R.T
        p[:, :3] += t
        p[:, 4] = ts - sts
        parts.append(p)
    pts = np.concatenate(parts, 0)
    pts[:, 4] = 0
    flag = pts[:, 4] == 0
    cur = pts[flag]
    prev = pts[~flag]
    if prev.shape[0] == 0:
        prev = cur
    np.random.shuffle(cur)
    np.random.shuffle(prev)
    return cur[point_pipeline_ref.first_voxels(cur, sampler.lo, sampler.voxel_size, sampler.grid, sampler.max_voxels)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=35000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_pipeline needs a CUDA device")
    dev = torch.device("cuda", 0)
    infos = pretrain.synthetic_point_infos(KEPT, args.points, seed=0)
    files = {}
    for info in infos:
        for path in [info["pts_filename"]] + [s["data_path"] for s in info["sweeps"]]:
            files[path] = np.fromfile(path, np.float32)
    pp.read_points = files.__getitem__                    # preloaded arrays instead of file reads
    steps = pp.config_train_pipeline()
    sampler = steps[2]

    def ours(frames, gather=True):
        res = []
        for info in frames:
            r = dict(info)
            for s in steps:
                r = s(r)
            res.append(r)
        return pp.gather_gt_points(res[:KEPT] if gather else res, EGO, dev) if gather else res

    def reference(frames):
        out = []
        for i, info in enumerate(frames):
            key = files[info["pts_filename"]].reshape(-1, 5)
            sw = [(files[s["data_path"]].reshape(-1, 5), s["sensor2lidar_rotation"], s["sensor2lidar_translation"],
                   s["timestamp"] / 1e6) for s in info["sweeps"]]
            p = reference_frame(key, sw, info["timestamp"], sampler)
            if i < KEPT:
                x, y = p[:, 0], p[:, 1]
                p = p[~((EGO[0] <= x) & (EGO[2] >= x) & (EGO[1] <= y) & (EGO[3] >= y))].copy()
                p[:, -1] = i
                out.append(p)
        return torch.from_numpy(np.concatenate(out, 0)).to(dev)

    sample = infos[:KEPT] + infos[KEPT - 4:KEPT - 2]        # 10 runs, 8 kept
    one = infos[:1]
    np.random.seed(0)
    a = ours(one)
    np.random.seed(0)
    b = reference(one)
    torch.cuda.synchronize()
    same = torch.equal(a[0][~torch.isnan(a[0, :, 0])], b)
    res = dict(card=card(), points_per_cloud=args.points, same_as_reference_one_frame=bool(same))
    res["frame_host_ms"] = host_ms({"ours": lambda: ours(one), "reference": lambda: reference(one)}, args.steps, 1)
    res["sample_host_ms"] = host_ms({"ours": lambda: ours(sample), "reference": lambda: reference(sample)},
                                    args.steps, 1)
    recorded = ours(infos[:KEPT], gather=False)
    res["device_pass_ms_8_frames"] = event_ms(lambda: pp.gather_gt_points(recorded, EGO, dev), 20, 3)
    raw, perm = pp.upload_bytes(recorded)
    ref_bytes = sum(point_pipeline_ref.gather([pp.frame_plan(r) for r in recorded], EGO).nbytes for _ in [0])
    res["upload_bytes"] = dict(ours_raw=raw, ours_int32_orders=perm, ours_total=raw + perm, reference_float32=ref_bytes)
    res["host_shuffle_ms_per_frame"] = dict(
        index_vectors=host_ms(lambda: [np.random.shuffle(np.arange(3 * args.points, dtype=np.int32)) for _ in (0, 1)],
                              args.steps, 1),
        rows_2d=host_ms(lambda: [np.random.shuffle(np.zeros((3 * args.points, 5), np.float32)) for _ in (0, 1)],
                        args.steps, 1))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
