"""Write tests/golden/point_pipeline.npz: the reference's own point statements on small LiDAR-like queues.

Each case seeds numpy, runs the reference's transforms (mmdet3d's LoadPointsFromFile, the reference's
CustomLoadPointsFromMultiSweeps and CustomVoxelBasedPointSampler, through tools/ref_shim.install_point_pipelines)
on every frame of its queue in the dataset's order -- the previous frames, the current frame's draw-only run whose
points union2one drops, then the current and future frames -- and then the reference's union2one on the result.
It stores the inputs (key frames and sweeps on a 1/64 m lattice, plus float32 edge points), numpy's state after
every transform call and the gt_points.

    python tools/make_golden_point_pipeline.py [--out tests/golden/point_pipeline.npz]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import ref_shim  # noqa: E402
from vidar_b200 import synthetic  # noqa: E402

PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
EGO = [-0.8, -1.5, 0.8, 2.5]
SWEEPS = dict(sweeps_num=2, use_dim=[0, 1, 2, 3, 4], pad_empty_sweeps=True, remove_close=True, ego_mask=EGO,
              hard_sweeps_timestamp=0, random_select=False)
SAMPLER = dict(cur_sweep_cfg=dict(max_num_points=1, point_cloud_range=PC_RANGE, voxel_size=[1.0, 1.0, 1.0],
                                  max_voxels=50000), time_dim=4)
N = 1500


def edge_points():
    """float32 points at +-51.2f, at the 1-ulp neighbours of voxel faces and of the ego / remove-close bounds."""
    f = np.float32

    def around(v):
        v = f(v)
        return [np.nextafter(v, f(-np.inf)), v, np.nextafter(v, f(np.inf))]

    pts = []
    for i, x in enumerate(around(-51.2) + around(51.2) + around(-51.2 + 1) + around(f(-51.2) + f(50)) + around(50.8)):
        pts.append((x, f(-20 + 3 * i), f(-4.5 + i % 8)))
    for i, y in enumerate(around(-51.2) + around(51.2) + around(f(-51.2) + f(77))):
        pts.append((f(-10 + 3 * i), y, f(-4.5 + i % 8)))
    for i, z in enumerate(around(-5.0) + around(3.0) + around(f(-5.0) + f(2))):
        pts.append((f(-30 + 3 * i), f(30.25), z))
    for i, x in enumerate(around(-0.8) + around(0.8)):                     # ego box x faces, y inside
        pts.append((x, f(2.0), f(-4.5 + i % 8)))
    for i, y in enumerate(around(-1.5) + around(2.5)):                     # ego box y faces, x inside
        pts.append((f(0.5), y, f(-4.5 + i % 8)))
    for i, x in enumerate(around(-1.0) + around(1.0)):                     # remove-close x bound
        pts.append((x, f(0.5), f(-4.5 + i % 8)))
    for i, y in enumerate(around(-1.0) + around(1.0)):                     # remove-close y bound, x outside the box
        pts.append((f(0.9), y, f(-4.5 + i % 8)))
    p = np.array(pts, f)
    return np.concatenate([p, np.full((len(p), 1), f(7)), np.zeros((len(p), 1), f)], 1)


def case_list():
    far = dict(sweeps=1, n=400, far=True)             # every point outside the range: no survivors
    return [
        dict(name="config", seed=1, frames=[dict(sweeps=3)], current=0),
        dict(name="pad_empty", seed=2, frames=[dict(sweeps=0)], current=0),
        dict(name="fewer_sweeps", seed=3, frames=[dict(sweeps=1)], current=0),
        dict(name="random_select", seed=4, frames=[dict(sweeps=5)], current=0, sweeps=dict(random_select=True)),
        dict(name="hard_none", seed=5, frames=[dict(sweeps=3)], current=0, sweeps=dict(hard_sweeps_timestamp=None)),
        dict(name="hard_nonzero", seed=6, frames=[dict(sweeps=2, n=300)], current=0,
             sweeps=dict(hard_sweeps_timestamp=0.5)),
        dict(name="max_voxels", seed=7, frames=[dict(sweeps=2)], current=0,
             sampler=dict(max_voxels=150)),
        dict(name="edges", seed=8, frames=[dict(sweeps=0, n=300, edges=True)], current=0),
        dict(name="queue3", seed=9, frames=[dict(sweeps=2, n=700), far, dict(sweeps=3, n=700)], current=1),
    ]


def make_inputs(case):
    rng = np.random.default_rng(case["seed"])
    arrays, frames = {}, []
    for f, fr in enumerate(case["frames"]):
        n = fr.get("n", N)
        key = synthetic.lidar_cloud(rng, n)
        if fr.get("far"):
            key[:, 0] = np.abs(key[:, 0]) + np.float32(60)
        if fr.get("edges"):
            key = np.concatenate([key, edge_points()], 0)
        ts = 1533151603547590 + 500000 * f
        arrays[f"{case['name']}.{f}.key"] = key
        poses, sts = [], []
        for j in range(fr["sweeps"]):
            sw = synthetic.lidar_cloud(rng, n)
            if fr.get("far"):
                sw[:, 0] = np.abs(sw[:, 0]) + np.float32(60)
            R, t = synthetic.sweep_pose(rng, j + 1)
            arrays[f"{case['name']}.{f}.sweep{j}"] = sw
            poses.append(np.concatenate([R.reshape(9), t]))
            sts.append(ts - 50000 * (j + 1) + (7 if j == 2 else 0))
        arrays[f"{case['name']}.{f}.pose"] = np.array(poses, np.float64).reshape(-1, 12)
        arrays[f"{case['name']}.{f}.sweep_ts"] = np.array(sts, np.int64)
        arrays[f"{case['name']}.{f}.ts"] = np.int64(ts)
    return arrays


def frame_info(arrays, name, f, root):
    """The dataset's results dict of frame f (files written under root)."""
    def put(key):
        path = os.path.join(root, key + ".bin")
        if not os.path.exists(path):
            arrays[key].tofile(path)
        return path
    pose, sts = arrays[f"{name}.{f}.pose"], arrays[f"{name}.{f}.sweep_ts"]
    sweeps = [dict(data_path=put(f"{name}.{f}.sweep{j}"), timestamp=int(sts[j]),
                   sensor2lidar_rotation=pose[j, :9].reshape(3, 3).copy(), sensor2lidar_translation=pose[j, 9:].copy())
              for j in range(len(sts))]
    return dict(pts_filename=put(f"{name}.{f}.key"), timestamp=int(arrays[f"{name}.{f}.ts"]) / 1e6, sweeps=sweeps,
                pts_mask_fields=[], pts_seg_fields=[])


def run_order(case):
    """(frame, gathered) in the dataset's order: previous frames, the current frame's draw-only run, then the
    current and future frames."""
    p = case["current"]
    n = len(case["frames"])
    return [(f, True) for f in range(p)] + [(p, False)] + [(f, True) for f in range(p, n)]


def state_row():
    st = np.random.get_state()
    return np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "tests", "golden", "point_pipeline.npz"))
    args = ap.parse_args()
    ref = ref_shim.install_point_pipelines()
    DC = ref["DataContainer"]
    out, metas = {}, []
    with tempfile.TemporaryDirectory() as root:
        for case in case_list():
            name = case["name"]
            arrays = make_inputs(case)
            out.update(arrays)
            sweeps = dict(SWEEPS, **case.get("sweeps", {}))
            sampler = dict(SAMPLER, cur_sweep_cfg=dict(SAMPLER["cur_sweep_cfg"], **case.get("sampler", {})))
            steps = [ref["LoadPointsFromFile"](coord_type="LIDAR", load_dim=5, use_dim=5),
                     ref["CustomLoadPointsFromMultiSweeps"](**sweeps), ref["CustomVoxelBasedPointSampler"](**sampler)]
            np.random.seed(case["seed"])
            states, gauss, prev, fut = [], [], [], []
            p = case["current"]
            for f, gathered in run_order(case):
                results = frame_info(arrays, name, f, root)
                for s in steps:
                    results = s(results)
                    k, g = state_row()
                    states.append(k)
                    gauss.append(g)
                meta = dict(scene_token="scene", ego2global_translation=[0.0, 0.0, 0.0],
                            ego2global_rotation=[1.0, 0.0, 0.0, 0.0], lidar2ego_translation=[0.0, 0.0, 0.0],
                            lidar2ego_rotation=[1.0, 0.0, 0.0, 0.0], can_bus=np.zeros(18))
                item = dict(points=DC(results["points"].tensor), img_metas=DC(meta), img=DC(torch.zeros(1)))
                (prev if (not gathered or f < p) else fut).append(item)
            gt = ref["union2one"](prev, fut, EGO)["gt_points"].data.numpy()
            out[f"{name}.gt"] = gt
            out[f"{name}.states"] = np.stack(states)
            out[f"{name}.gauss"] = np.array(gauss)
            metas.append(dict(case, sweeps_kwargs=sweeps, sampler_kwargs=sampler, ego_mask=EGO))
            print(f"{name}: gt_points {gt.shape}, {len(states)} states")
    out["cases"] = np.array(json.dumps(metas))
    np.savez_compressed(args.out, **out)
    print(f"wrote {args.out} ({os.path.getsize(args.out) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
