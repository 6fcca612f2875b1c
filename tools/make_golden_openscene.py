"""Write tests/golden/openscene.npz: the reference's own OpenScene input statements on small inputs.

  * `PointCloud.parse(bytes).to_pcd_bin2().T` (datasets/pipelines/nuplan_loading.py) on binary .pcd files with
    nuPlan's six fields and trailing bytes, and the exception class it raises on malformed headers and streams;
  * the OpenScene configs' point transforms -- LoadNuPlanPointsFromFile, LoadNuPlanPointsFromMultiSweeps and the
    voxel sampler -- on each GT frame of a queue, numpy's state after every call, then NuPlanViDARDatasetV1's
    union2one: gt_points;
  * RandomScaleImageMultiViewImage([2/3]) with mmcv.imresize as cv2 computes it here: the resized float32 images,
    lidar2img, img_shape, ori_shape and numpy's state.
All through tools/ref_shim.py.

    python tools/make_golden_openscene.py [--out tests/golden/openscene.npz]
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
SWEEPS = dict(sweeps_num=0, use_dim=[0, 1, 2, 3, 4, 5], file_client_args=dict(backend="disk"), pad_empty_sweeps=True,
              remove_close=True, ego_mask=EGO, hard_sweeps_timestamp=0, random_select=False)
SAMPLER = dict(cur_sweep_cfg=dict(max_num_points=1, point_cloud_range=PC_RANGE, voxel_size=[1.0, 1.0, 1.0],
                                  max_voxels=50000), time_dim=4)
GOOD = ("# .PCD v0.7\nVERSION 0.7\nFIELDS x y z intensity ring lidar_info\nSIZE 4 4 4 4 2 1\nTYPE F F F F U U\n"
        "COUNT 1 1 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
BAD_HEADERS = {
    "count2": GOOD.replace("COUNT 1 1 1 1 1 1", "COUNT 1 1 1 1 1 2"),
    "ascii": GOOD.replace("DATA binary", "DATA ascii"),
    "sizes": GOOD.replace("SIZE 4 4 4 4 2 1", "SIZE 4 4 4 4 2"),
    "no_points": GOOD.replace("POINTS {n}\n", ""),
}


def state_row():
    st = np.random.get_state()
    return np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4])


def pcd_cases(rng, root, out, meta):
    ref = ref_shim.install_nuplan_pipelines()
    PointCloud = ref["PointCloud"]
    for name, n, garbage in (("pcd_small", 5, 0), ("pcd_garbage", 700, 33)):
        path = os.path.join(root, name + ".pcd")
        synthetic.write_pcd(path, synthetic.nuplan_cloud(rng, n), garbage)
        data = open(path, "rb").read()
        out[f"{name}.bytes"] = np.frombuffer(data, np.uint8)
        out[f"{name}.points"] = PointCloud.parse(data).to_pcd_bin2().T
    cloud = synthetic.nuplan_cloud(rng, 4)
    body = synthetic.write_pcd(os.path.join(root, "body.pcd"), cloud) or open(os.path.join(root, "body.pcd"), "rb").read()
    body = body[body.index(b"DATA binary\n") + len(b"DATA binary\n"):]
    for name, head in dict(BAD_HEADERS, truncated=GOOD).items():
        data = head.format(n=4).encode() + (body[:-20] if name == "truncated" else body)
        try:
            PointCloud.parse(data)
            err = None
        except Exception as e:          # noqa: BLE001  (the class is the golden)
            err = type(e).__name__
        out[f"bad_{name}.bytes"] = np.frombuffer(data, np.uint8)
        meta["errors"][name] = err
    return ref


def point_case(ref, rng, root, out, meta):
    DC = ref["DataContainer"]
    steps = [ref["LoadNuPlanPointsFromFile"](coord_type="LIDAR"), ref["LoadNuPlanPointsFromMultiSweeps"](**SWEEPS),
             ref["CustomVoxelBasedPointSampler"](**SAMPLER)]
    infos = []
    for f in range(3):
        path = os.path.join(root, f"queue.{f}.pcd")
        cloud = synthetic.nuplan_cloud(rng, 900)
        cloud[:5, :2] = [[0.5, 0.5], [0.2, 2.0], [-0.8, -1.5], [0.8, 2.5], [0.0, 0.0]]     # close / ego box edges
        synthetic.write_pcd(path, cloud, 8)
        out[f"queue.{f}.bytes"] = np.fromfile(path, np.uint8)
        infos.append(dict(pts_filename=path, timestamp=(1533151603547590 + 500000 * f) / 1e6, sweeps=[],
                          pts_mask_fields=[], pts_seg_fields=[]))
    np.random.seed(11)
    states, gauss, items, after = [], [], [], []
    for f, info in enumerate(infos):
        results = dict(info)
        for s in steps:
            results = s(results)
            k, g = state_row()
            states.append(k)
            gauss.append(g)
            if s is steps[1]:
                after.append(results["points"].tensor.numpy().copy())
        meta_f = dict(scene_token="scene", ego2global_translation=[0.0, 0.0, 0.0],
                      ego2global_rotation=[1.0, 0.0, 0.0, 0.0], lidar2ego_translation=[0.0, 0.0, 0.0],
                      lidar2ego_rotation=[1.0, 0.0, 0.0, 0.0], can_bus=np.zeros(18))
        items.append(dict(points=DC(results["points"].tensor), img_metas=DC(meta_f), img=DC(torch.zeros(1))))
    gt = ref["nuplan_union2one"](items[:1], items, EGO)["gt_points"].data.numpy()
    for f, a in enumerate(after):
        out[f"queue.{f}.sweeps_out"] = a
    out["queue.gt"] = gt
    out["queue.states"] = np.stack(states)
    out["queue.gauss"] = np.array(gauss)
    meta["queue"] = dict(frames=3, seed=11, sweeps_kwargs=SWEEPS, sampler_kwargs=SAMPLER, ego_mask=EGO)


def scale_case(rng, out, meta):
    RandomScale = ref_shim.install_scale_pipeline()
    imgs = [(rng.standard_normal((96, 150, 3)) * 60).astype(np.float32) for _ in range(2)]
    l2i = [rng.standard_normal((4, 4)) for _ in range(2)]
    np.random.seed(5)
    res = RandomScale(scales=[2 / 3])(dict(img=list(imgs), lidar2img=list(l2i)))
    k, g = state_row()
    for i in range(2):
        out[f"scale.img{i}"] = imgs[i]
        out[f"scale.lidar2img_in{i}"] = l2i[i]
        out[f"scale.out{i}"] = res["img"][i]
        out[f"scale.lidar2img{i}"] = res["lidar2img"][i]
    out["scale.state"], out["scale.gauss"] = k, g
    meta["scale"] = dict(seed=5, img_shape=[list(s) for s in res["img_shape"]],
                         ori_shape=[list(s) for s in res["ori_shape"]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "tests", "golden", "openscene.npz"))
    args = ap.parse_args()
    rng = np.random.default_rng(2024)
    out, meta = {}, dict(errors={})
    with tempfile.TemporaryDirectory() as root:
        ref = pcd_cases(rng, root, out, meta)
        point_case(ref, rng, root, out, meta)
    scale_case(rng, out, meta)
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(args.out, **out)
    print(meta["errors"], out["queue.gt"].shape)
    print(f"wrote {args.out} ({os.path.getsize(args.out) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
