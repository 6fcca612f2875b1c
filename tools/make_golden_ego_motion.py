"""Write tests/golden/ego_motion.npz: the reference's own ego-motion statements on seeded synthetic drives.

Per case (a `synthetic.drive` of history + current + future frames, one case with a scene change in the history), it
runs, through tools/ref_shim.py:
  * NuScenesDataset.get_data_info's can_bus fill on every frame (datasets/nuscenes_dataset.py), then
    NuScenesViDARDatasetV1.union2one (datasets/nuscenes_vidar_dataset_v1.py) on the queue, with the current frame's
    results dict made once for each queue as _prepare_data_info makes it (not one dict shared by both);
  * PerceptionTransformer.get_bev_features' shift statements (modules/transformer.py, delta_global .. shift) on every
    image frame's metas, at 200 x 200 and 50 x 50;
  * ViDAR._get_history_ref_to_previous_transform and _align_bev_coordnates (detectors/vidar.py) over the future
    frames with a queue of one previous frame, as forward_train updates ref_to_history, at 50 x 50.
pyquaternion and the nuScenes devkit are not installed: `vidar_b200.ego_motion`'s restated Quaternion,
transform_matrix and quaternion_yaw stand in for them.

    python tools/make_golden_ego_motion.py [--out tests/golden/ego_motion.npz]
"""
import argparse
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import ref_shim  # noqa: E402
from vidar_b200 import ego_motion, synthetic  # noqa: E402

PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
CASES = [dict(seed=0, frames=4, future=3, scene_change=None),
         dict(seed=1, frames=4, future=6, scene_change=None),
         dict(seed=2, frames=4, future=3, scene_change=2)]
META_KEYS = ("can_bus", "prev_bev_exists", "lidar2global_rotation", "ref_lidar_to_cur_lidar")
CUR_KEYS = ("future_can_bus", "future2ref_lidar_transform", "ref2future_lidar_transform",
            "total_cur2ref_lidar_transform", "total_ref2cur_lidar_transform")


def _helpers():
    return dict(np=np, torch=torch, copy=__import__("copy"), Quaternion=ego_motion.Quaternion,
                transform_matrix=ego_motion.transform_matrix, quaternion_yaw=ego_motion.quaternion_yaw)


def get_data_info():
    ns = _helpers()
    return ref_shim._load_methods(os.path.join(ref_shim.REF_DATASETS, "nuscenes_dataset.py"), "CustomNuScenesDataset",
                                  ("get_data_info",), ns)["get_data_info"]


def union2one():
    ns = dict(_helpers(), DC=ref_shim.install_point_pipelines()["DataContainer"])
    return ref_shim._load_methods(os.path.join(ref_shim.REF_DATASETS, "nuscenes_vidar_dataset_v1.py"),
                                  "NuScenesViDARDatasetV1", ("union2one",), ns)["union2one"]


def shift_statements():
    """get_bev_features' statements from `delta_global = ...` to `shift = ...`, as one function of (img_metas, bs,
    bev_h, bev_w) -> shift [bs, 2]."""
    path = os.path.join(ref_shim.REF_BEVFORMER, "modules", "transformer.py")
    src = open(path).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "get_bev_features")
    lines = src.splitlines()[fn.lineno - 1:fn.end_lineno]
    start = next(i for i, line in enumerate(lines) if "delta_global = " in line)
    end = next(i for i, line in enumerate(lines) if line.strip().startswith("shift = bev_queries.new_tensor"))
    body = textwrap.dedent("\n".join(lines[start:end + 1]))

    def run(img_metas, bs, bev_h, bev_w):
        ns = dict(np=np, kwargs=dict(img_metas=img_metas), bs=bs, grid_length=[0.512, 0.512], bev_h=bev_h,
                  bev_w=bev_w, self=types.SimpleNamespace(use_shift=True), bev_queries=torch.zeros(1))
        exec(compile(body, path, "exec"), ns)
        return ns["shift"].numpy()
    return run


def align_methods(bev_h, bev_w):
    stub = ref_shim.load_functions(os.path.join("utils", "e2e_predictor_utils.py"),
                                   ("get_bev_grids", "bev_grids_to_coordinates", "bev_coords_to_grids"))
    get_bev_grids = stub.pop("get_bev_grids")
    stub["get_bev_grids"] = lambda H, W, bs=1, device="cpu", **kw: get_bev_grids(H, W, bs, device="cpu", **kw)
    ns = dict(np=np, torch=torch, e2e_predictor_utils=types.SimpleNamespace(**stub))
    m = ref_shim._load_methods(os.path.join(ref_shim.REF_BEVFORMER, "detectors", "vidar.py"), "ViDAR",
                               ("_get_history_ref_to_previous_transform", "_align_bev_coordnates"), ns)
    owner = types.SimpleNamespace(bev_h=bev_h, bev_w=bev_w, point_cloud_range=PC_RANGE)
    return (lambda *a: m["_get_history_ref_to_previous_transform"](owner, *a),
            lambda *a: m["_align_bev_coordnates"](owner, *a))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "ego_motion.npz"))
    args = ap.parse_args()
    info_fn, union, shift_fn = get_data_info(), union2one(), shift_statements()
    DC = ref_shim.install_point_pipelines()["DataContainer"]
    out = {}
    for c, case in enumerate(CASES):
        T, F = case["frames"], case["future"]
        drive = synthetic.drive(T + F, case["seed"], case["scene_change"])
        for t, p in enumerate(drive):
            for k in ("ego2global_translation", "ego2global_rotation", "lidar2ego_translation", "lidar2ego_rotation",
                      "can_bus"):
                out[f"c{c}.in{t}.{k}"] = np.asarray(p[k], np.float64)
            out[f"c{c}.in{t}.scene"] = np.int64(p["scene_token"].endswith("-1"))
        queue = []
        for t, p in [*enumerate(drive[:T]), *enumerate(drive[T - 1:], T - 1)]:     # the current frame twice
            info = dict(token=f"t{t}", lidar_path="", sweeps=[], prev="", next="", frame_idx=t, timestamp=t * 5e5,
                        **{k: (np.array(v, np.float64) if k == "can_bus" else v) for k, v in p.items()})
            ds = types.SimpleNamespace(data_infos=[info], modality=dict(use_camera=False), test_mode=True,
                                       include_test=False)
            d = info_fn(ds, 0)
            d["lidar2ego_translation"], d["lidar2ego_rotation"] = p["lidar2ego_translation"], p["lidar2ego_rotation"]
            queue.append(dict(img_metas=DC(d), img=DC(torch.zeros(1)), points=DC(torch.zeros((1, 5)))))
        ds = types.SimpleNamespace(ego_mask=None, future_length=F)
        # _prepare_data_info (nuscenes_vidar_dataset_template.py:107-142) makes the current frame's results dict
        # twice: once for the previous queue, once as the future queue's first entry
        res = union(ds, queue[:T], queue[T:])
        metas = res["img_metas"].data
        for t in range(T):
            for k in META_KEYS:
                out[f"c{c}.m{t}.{k}"] = np.asarray(metas[t][k])
            for hw in (200, 50):
                out[f"c{c}.m{t}.shift{hw}"] = shift_fn([metas[t]], 1, hw, hw)
        for k in CUR_KEYS:
            out[f"c{c}.cur.{k}"] = np.asarray(metas[T - 1][k])
        history, align = align_methods(50, 50)
        ref_bev = torch.zeros(1, 1, 1)
        r2h = history(ref_bev, 1, [[metas[T - 1]]])
        for k in range(1, F + 1):
            tgt, ref_grids, ref2future = align(k, r2h, [metas[T - 1]])
            out[f"c{c}.tgt{k}"], out[f"c{c}.ref{k}"] = tgt.numpy(), ref_grids.numpy()
            r2h = torch.cat([r2h, ref2future.unsqueeze(1)], 1)[:, 1:].contiguous()
    np.savez_compressed(args.out, **out)
    print(f"wrote {args.out}: {len(out)} arrays")


if __name__ == "__main__":
    main()
