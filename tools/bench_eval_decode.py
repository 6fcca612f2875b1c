"""Time ViDARRayHeadV1's evaluation at the test shape: `evaluate` (one batched device pass) against
`frame_metrics(get_point_cloud_prediction(...))` (per-(sample, frame) decode and boolean masks), alternating in one
process.

    python tools/bench_eval_decode.py [--steps 20] [--warmup 3] [--gt 30000]

Shape: bs 1, 7 frames (current + 6 future), 200 x 200 x 16 sigma of the current head frame, ray_grid_num 512,
`--gt` GT points per frame, seeded rigid frame transforms in img_metas.  Both paths end in host numbers, so each call
is timed with a host clock around the synchronised call (median of --steps, the paths alternating, both warmed up).
Per path: vidar_b200 kernel launches and host syncs per call (counted by tools/gpu_timing.py's count_syncs), and
the largest relative difference of the four metrics between the paths.  The card's name, power limit and SM
clock are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gpu_timing import card, count_syncs, host_ms  # noqa: E402
from vidar_b200 import _lib, evaluate  # noqa: E402
from vidar_b200.head import ViDARRayHeadV1  # noqa: E402

F, H, W, Z, NUM_WAY, INTER = 7, 200, 200, 16, 512, 3
HISTORY_QUEUE_LENGTH, PRED_HISTORY = 4, 3
HEAD_FRAMES = PRED_HISTORY + 2
PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
METRICS = ("chamfer_distance", "l1_error", "absrel_error", "count")


def _rigid(rng):
    ang = np.radians([2.0, 2.0, 6.0]) * rng.uniform(-1, 1, 3)
    c, s = np.cos(ang), np.sin(ang)
    rx = np.array([[1, 0, 0], [0, c[0], -s[0]], [0, s[0], c[0]]])
    ry = np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]])
    rz = np.array([[c[2], -s[2], 0], [s[2], c[2], 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = (rz @ ry @ rx).T
    T[3, :3] = np.array([3.0, 3.0, 0.3]) * rng.uniform(-1, 1, 3)
    return T


def inputs(gt_per_frame, seed=0):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    preds = torch.randn(F, INTER, HEAD_FRAMES, 1, H * W, Z, generator=g).to(dev)
    n = gt_per_frame * F
    lo, hi = torch.tensor(PC_RANGE[:3]), torch.tensor(PC_RANGE[3:])
    xyz = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    t = (torch.randint(0, F, (n, 1), generator=g) + HISTORY_QUEUE_LENGTH).float()       # target frames 4 .. 10
    gt = [torch.cat([xyz, torch.rand(n, 1, generator=g), t], 1).to(dev)]
    cur2ref = np.stack([_rigid(rng) for _ in range(HISTORY_QUEUE_LENGTH + F)])
    metas = [dict(total_cur2ref_lidar_transform=cur2ref, total_ref2cur_lidar_transform=np.linalg.inv(cur2ref))]
    pd = dict(next_bev_preds=preds, valid_frames=list(range(F)))
    kw = dict(start_idx=0, tgt_bev_h=H, tgt_bev_w=W, tgt_pc_range=PC_RANGE, img_metas=metas)
    return pd, gt, kw


def fused(head, pd, gt, kw):
    return head.evaluate(pd, gt, **kw)


def unfused(head, pd, gt, kw):
    dec = head.get_point_cloud_prediction(pd, gt, **kw)
    return evaluate.frame_metrics(dec["pred_pcds"], dec["gt_pcds"], dec["origin"], kw["tgt_pc_range"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gt", type=int, default=30000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_decode needs a CUDA device")
    head = ViDARRayHeadV1(HISTORY_QUEUE_LENGTH, pred_history_frame_num=PRED_HISTORY, pred_future_frame_num=1,
                          per_frame_loss_weight=(0.1,) * HEAD_FRAMES, ray_grid_num=NUM_WAY,
                          loss_weight=np.ones((F, 1)))
    pd, gt, kw = inputs(a.gt)
    paths = {"evaluate": lambda: fused(head, pd, gt, kw),
             "frame_metrics(get_point_cloud_prediction)": lambda: unfused(head, pd, gt, kw)}
    name = card()
    res, outs = {}, {}
    with torch.no_grad():
        ms = host_ms(paths, a.steps, a.warmup)                  # the two paths alternating
        for k, fn in paths.items():
            n0 = _lib.launch_count()
            outs[k] = fn()
            torch.cuda.synchronize()
            res[k] = dict(launches=_lib.launch_count() - n0)
            res[k]["host_syncs"], res[k]["sync_sites"] = count_syncs(fn)
            res[k]["median_ms"] = round(ms[k], 3)
    fo, uo = (outs[k] for k in paths)
    rel = 0.0
    for f in uo:
        for m in METRICS:
            x, y = float(fo[f][m]), float(uo[f][m])
            if not (np.isnan(x) and np.isnan(y)):
                rel = max(rel, abs(x - y) / max(abs(y), 1e-30))
    points = {f: int(v["count"]) for f, v in fo.items()}
    print(json.dumps(dict(tool="bench_eval_decode", card=name, bs=1, frames=F, sigma=[H, W, Z], ray_grid_num=NUM_WAY,
                          gt_per_frame=a.gt, steps=a.steps, paths=res, max_rel_diff_of_metrics=rel, counts=points,
                          speedup=round(res[list(paths)[1]]["median_ms"] / res["evaluate"]["median_ms"], 2))),
          flush=True)


if __name__ == "__main__":
    main()
