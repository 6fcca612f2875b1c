"""Time ViDARRayHeadV1.loss forward + backward at the pre-training head shape, batched over every head frame
(`fuse_head_frames = True`, the default) and through the per-head-frame loop over ViDARRayHead.loss, alternating in
one process.

    python tools/bench_head_v1_loss.py [--steps 20] [--warmup 3] [--gt 10000 30000]

Shape: bs 1, 5 head frames (3 history, current, 1 future; history_queue_length 4), 4 target frames, 200 x 200 x 16
sigma, ray_grid_num 512, 10 000 dense rays per frame (the 50 x 50 x 4 dense grid), CE + dense (use_dist_loss=False),
the shipped per-frame and frame loss weights; `--gt` GT points per source frame (9 source frames), random rigid
frame transforms.  Both paths get the same inputs and the same pre-drawn Gumbel noise, so their outputs are
compared at the timed size.  Per path: median time of loss + backward by CUDA events, vidar_b200 kernel launches per
call, and host syncs per call counted in a separate pass (tools/gpu_timing.py's count_syncs).  The card's name,
power limit and SM clocks are read in the same run.  Prints one JSON line per GT size."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gpu_timing import card, count_syncs, event_ms  # noqa: E402
from vidar_b200 import _lib  # noqa: E402
from vidar_b200.head import ViDARRayHeadV1  # noqa: E402

V, HF, H, W, Z, NUM_WAY, HQL, N_SRC = 4, 5, 200, 200, 16, 512, 4, 9
PC_RANGE = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
LOSS_W = [[1], [1], [1], [1], [0]]
HEAD_KW = dict(history_queue_length=HQL, pred_history_frame_num=3, pred_future_frame_num=1,
               per_frame_loss_weight=(0.2, 0.4, 0.6, 1.0, 1.2), ray_grid_num=NUM_WAY, use_dist_loss=False,
               loss_weight=LOSS_W)


def rigid(g):
    a = np.radians(6.0) * (2 * torch.rand(1, generator=g).item() - 1)
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a), np.sin(a)], [-np.sin(a), np.cos(a)]]
    T[3, :3] = np.array([3.0, 3.0, 0.3]) * (2 * torch.rand(3, generator=g).numpy() - 1)
    return T


def inputs(gt_per_frame, seed=0):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(seed)
    preds = torch.randn(V, 1, HF, 1, H * W, Z, generator=g).to(dev)
    n = gt_per_frame * N_SRC
    lo, hi = torch.tensor(PC_RANGE[:3]), torch.tensor(PC_RANGE[3:])
    xyz = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    t = torch.randint(0, N_SRC, (n, 1), generator=g).float()
    gt = [torch.cat([xyz, torch.rand(n, 1, generator=g), t], 1).to(dev)]
    cur2ref = np.stack([rigid(g) for _ in range(N_SRC)])
    metas = [dict(total_cur2ref_lidar_transform=cur2ref, total_ref2cur_lidar_transform=np.linalg.inv(cur2ref))]
    R = (H // 4) * (W // 4) * (Z // 4) * V
    noise = [{"dense": (-torch.empty(1, R, NUM_WAY).exponential_(generator=g).log()).to(dev)} for _ in range(HF)]
    kw = dict(start_idx=0, tgt_bev_h=H, tgt_bev_w=W, tgt_pc_range=PC_RANGE, pred_frame_num=None, img_metas=metas,
              gumbels=noise)
    return preds, gt, kw


def call(head, preds, gt, kw):
    p = preds.clone().requires_grad_(True)
    out = head.loss(dict(next_bev_preds=p, valid_frames=list(range(V))), gt, **kw)
    sum(out.values()).backward()
    return out, p.grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gt", type=int, nargs="+", default=[10000, 30000])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_head_v1_loss needs a CUDA device")
    heads = {}
    for fused in (True, False):
        h = ViDARRayHeadV1(**HEAD_KW)
        h.fuse_head_frames = fused
        heads["batched" if fused else "per_head_frame"] = h
    name = card()
    for n_gt in a.gt:
        preds, gt, kw = inputs(n_gt)
        calls = {k: (lambda h=h: call(h, preds, gt, kw)) for k, h in heads.items()}
        ms = event_ms(calls, a.steps, a.warmup)                 # the two paths alternating
        res, outs = {}, {}
        for k, fn in calls.items():
            n0 = _lib.launch_count()
            outs[k] = fn()
            torch.cuda.synchronize()
            res[k] = dict(launches=_lib.launch_count() - n0)
            res[k]["syncs"], res[k]["sync_sites"] = count_syncs(fn)
            res[k]["median_ms"] = round(ms[k], 3)
        (ob, gb), (op, gp) = outs["batched"], outs["per_head_frame"]
        ob, op = ({k: float(v.detach()) for k, v in o.items()} for o in (ob, op))
        cmp = {k: dict(batched=ob[k], per_head_frame=op[k], rel_diff=abs(ob[k] - op[k]) / max(abs(op[k]), 1e-30))
               for k in ob}
        cmp["grad_max_abs_diff_over_max"] = float((gb - gp).abs().max() / gp.abs().max())
        print(json.dumps(dict(tool="bench_head_v1_loss", card=name, bs=1, head_frames=HF, frames=V, sigma=[H, W, Z],
                              ray_grid_num=NUM_WAY, dense_rays_per_frame=(H // 4) * (W // 4) * (Z // 4),
                              gt_per_frame=n_gt, steps=a.steps, paths=res, compare=cmp)), flush=True)


if __name__ == "__main__":
    main()
