"""Ego motion's cost on the H100.

  (a) TSA's value with the previous BEV rotated, at 200 x 200 x 256 (bs 1): `ego_motion.rotate_stack` (one kernel
      forward; sort + gather backward) against the reference's statements (permute, torchvision `rotate` about
      [100, 100], permute, stack; autograd through them backward).  CUDA events around the device work, L2 flushed
      before each call, median of 20.  The row map (`ego_motion.rotation_rows`) is timed apart: it is built once per
      frame.  Achieved bytes/s count the algorithm's traffic -- forward: read prev and query, write the [2, Q, C]
      value; backward: read the [2, Q, C] gradient, write both gradients -- against the 3.35 TB/s H100 SXM data
      sheet figure.
  (b) the full-size `vidar_1_8_nusc_3future` step from files (dcn, GridMask, both pipelines, `SampleLoader` with
      prefetch 1), with and without ego_motion, in alternating rounds; host syncs per step from
      tools/gpu_timing.py's count_syncs.
The card's name, power limit and SM clock are read in the same run.

    python tools/bench_ego_motion.py [--steps 4] [--warmup 2] [--rounds 2] [--out /tmp/bench_ego_motion.json]
"""
import argparse
import json
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gpu_timing import card, count_syncs, event_ms, window_ms  # noqa: E402
from vidar_b200 import ego_motion as ego, pretrain  # noqa: E402

PEAK_BW = 3.35e12
CONFIG = "vidar_1_8_nusc_3future"


def reference_value(prev, query, angle, H, W):
    from torchvision.transforms.functional import rotate
    tmp = rotate(prev[0].reshape(H, W, -1).permute(2, 0, 1), angle, center=[100, 100])
    return torch.stack([tmp.permute(1, 2, 0).reshape(H * W, -1)[None], query], 1).reshape(2, H * W, -1)


def kernel_part(dev, iters=20):
    H = W = 200
    C, Q, angle = 256, 200 * 200, 1.9
    g = torch.Generator(device=dev).manual_seed(0)
    prev = torch.randn(1, Q, C, device=dev, generator=g, requires_grad=True)
    query = torch.randn(1, Q, C, device=dev, generator=g, requires_grad=True)
    grad = torch.randn(2, Q, C, device=dev, generator=g)
    rows = ego.rotation_rows([angle], H, W, dev)
    fwd_bytes = 4 * (2 * Q * C + 2 * Q * C)
    bwd_bytes = 4 * (2 * Q * C + 2 * Q * C)
    with torch.no_grad():
        fwd = event_ms(dict(kernel=lambda: ego.rotate_stack(prev, query, rows),
                            reference=lambda: reference_value(prev, query, angle, H, W)), iters, 3, flush=True)
    ours, ref = ego.rotate_stack(prev, query, rows), reference_value(prev, query, angle, H, W)
    bwd = event_ms(dict(kernel=lambda: torch.autograd.grad(ours, (prev, query), grad, retain_graph=True),
                        reference=lambda: torch.autograd.grad(ref, (prev, query), grad, retain_graph=True)),
                   iters, 3, flush=True)
    row_map = event_ms(lambda: ego.rotation_rows([angle], H, W, dev), iters, 3, flush=True)
    out = dict(shape=[H, W, C], forward_ms=fwd, backward_ms=bwd, row_map_ms=row_map,
               forward_mb=fwd_bytes / 1e6, backward_mb=bwd_bytes / 1e6)
    out["forward_tb_s"] = fwd_bytes / (fwd["kernel"] * 1e-3) / 1e12
    out["backward_tb_s"] = bwd_bytes / (bwd["kernel"] * 1e-3) / 1e12
    out["forward_share_of_3p35"] = out["forward_tb_s"] * 1e12 / PEAK_BW
    out["backward_share_of_3p35"] = out["backward_tb_s"] * 1e12 / PEAK_BW
    return out


def reseed(seed):
    np.random.seed(seed)
    random.seed(seed)
    torch.manual_seed(seed)


def step_part(dev, args):
    arms = {}
    for on in (False, True):
        model, opt = pretrain.build(dev, seed=args.seed, config=CONFIG, dcn=True, grid_mask=True, image_pipeline=True,
                                    point_pipeline=True, ego_motion=on)
        queues = [pretrain.synthetic_sample(None, seed=args.seed + k, future_frames=model.future_frames, files=True,
                                            poses=True) for k in range(2)]
        arms[on] = (model, opt, queues)
    n = args.warmup + args.steps + 1
    times = {False: [], True: []}
    syncs = {}
    for _ in range(args.rounds):
        for on in (False, True):
            model, opt, queues = arms[on]
            reseed(args.seed)
            loader = pretrain.SampleLoader(model, [queues[k % 2] for k in range(n)], num_workers=args.workers,
                                           prefetch=1, seed=args.seed)
            it = iter(loader)
            torch.cuda.synchronize()
            times[on].append(window_ms(lambda: pretrain.train_step(model, opt, next(it)), args.steps, args.warmup))
            syncs[on] = count_syncs(pretrain.train_step, model, opt, next(it))
            del it, loader
    return dict(config=CONFIG, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                step_ms=dict(off=times[False], on=times[True]),
                step_ms_median=dict(off=float(np.median(times[False])), on=float(np.median(times[True]))),
                host_syncs_per_step=dict(off=syncs[False][0], on=syncs[True][0]),
                sync_sites=dict(off=syncs[False][1], on=syncs[True][1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ego_motion: needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(card=card(), kernel=kernel_part(dev))
    print(json.dumps(res), flush=True)
    if not args.skip_step:
        res["step"] = step_part(dev, args)
    res["card_after"] = card()
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
