"""The OpenScene pre-training step from files (vidar_b200/pretrain.py) on one GPU, one JSON line on stdout.

The `vidar_OpenScene_mini_1_8_3future` preset at full size (8 cameras of 1920 x 1080 JPEGs rescaled to 1280 x 736, a
200 x 200 BEV, 3 history frames, 3 future frames) with the DCNv2 backbone, GridMask and both pipelines, trained from
files through `SampleLoader(num_workers=--workers, prefetch=1)` with the configs' optimizer:
  * ms per step (host clock around --steps steps and a synchronize, after --warmup steps), host syncs per step
    (`gpu_timing.count_syncs` over one more step) and the peak allocation;
  * the device image chain of one frame (8 cameras, photometric + normalise + rescale + pad, one launch, CUDA events)
    against the reference's host statements on the same frame (numpy's photometric float32 math, mmcv's
    normalisation, cv2.resize and cv2.copyMakeBorder per camera; CPU clock).
The line also holds `gpu_timing.card()`.

    python tools/bench_openscene.py [--steps 5] [--warmup 2] [--workers 4] [--out f.jsonl]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gpu_timing import card, count_syncs, event_ms  # noqa: E402

CONFIG = "vidar_OpenScene_mini_1_8_3future"


def host_chain(imgs, plan):
    """The reference's host statements of the OpenScene train chain for one frame (transform_3d.py:98-185 on
    float32, mmcv.imnormalize, mmcv.imresize, mmcv.impad_to_multiple)."""
    import cv2
    out = []
    mean = np.float64(plan.mean.reshape(1, -1))
    for im, d in zip(imgs, plan.photo):
        x = im.astype(np.float32)
        if d.delta is not None:
            x += d.delta
        if d.mode == 1 and d.alpha is not None:
            x *= d.alpha
        hsv = cv2.cvtColor(x, cv2.COLOR_BGR2HSV)
        if d.sat is not None:
            hsv[..., 1] *= d.sat
        if d.hue is not None:
            hsv[..., 0] += d.hue
            hsv[..., 0][hsv[..., 0] > 360] -= 360
            hsv[..., 0][hsv[..., 0] < 0] += 360
        x = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
        if d.mode == 0 and d.alpha is not None:
            x *= d.alpha
        if d.perm is not None:
            x = x[..., list(d.perm)]
        x = cv2.multiply(cv2.subtract(x, mean), 1 / np.float64(plan.std.reshape(1, -1)))
        x = cv2.resize(x, plan.scale_hw[::-1], interpolation=cv2.INTER_LINEAR)
        out.append(cv2.copyMakeBorder(x, 0, plan.pad_hw[0] - x.shape[0], 0, plan.pad_hw[1] - x.shape[1],
                                      cv2.BORDER_CONSTANT, value=0))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    from vidar_b200 import image_aug, pretrain, synthetic
    dev = torch.device("cuda:0")
    line = dict(config=CONFIG, **card())

    # (b) the image chain of one frame
    rng = np.random.default_rng(0)
    imgs = np.stack([synthetic.camera_image(rng, synthetic.NUPLAN_IMG_HW) for _ in range(8)])
    np.random.seed(1)
    results = dict(img=list(imgs), lidar2img=[np.eye(4)] * 8)
    for t in image_aug.config_openscene_pipeline():
        results = t(results)
    src = torch.from_numpy(imgs).to(dev)
    line["image_chain_device_ms"] = event_ms(lambda: image_aug.apply_multiview(src, results), 20, 3)
    t0 = time.perf_counter()
    host = host_chain(imgs, results["img_aug"])
    line["image_chain_host_ms"] = (time.perf_counter() - t0) * 1e3
    got = image_aug.apply_multiview(src, results).cpu().numpy().transpose(0, 2, 3, 1)
    line["image_chain_max_abs_diff_vs_host"] = float(max(np.abs(g - h).max() for g, h in zip(got, host)))

    # (a) the step from files
    n = args.warmup + args.steps + 1
    queues = [pretrain.synthetic_sample(None, frames=4, future_frames=3, points_per_frame=100000, files=True,
                                        openscene=True, seed=s) for s in range(n)]
    np.random.seed(0)
    random.seed(0)
    model, _ = pretrain.build(dev, seed=0, config=CONFIG, dcn=True, grid_mask=True, image_pipeline=True,
                              point_pipeline=True)
    opt = pretrain.config_optimizer(model)
    loader = iter(pretrain.SampleLoader(model, queues, num_workers=args.workers, prefetch=1, seed=0))
    for _ in range(args.warmup):
        pretrain.train_step(model, opt, next(loader))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        loss, _ = pretrain.train_step(model, opt, next(loader))
    torch.cuda.synchronize()
    line["ms_per_step"] = (time.perf_counter() - t0) * 1e3 / args.steps
    line["peak_gb"] = torch.cuda.max_memory_allocated(dev) / 1e9
    syncs, sites = count_syncs(lambda: pretrain.train_step(model, opt, next(loader)))
    line.update(syncs_per_step=syncs, sync_sites=sites, loss=float(loss), steps=args.steps, warmup=args.warmup,
                workers=args.workers)
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(args.out, "a") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
