"""The pre-training image pipeline on one 6-camera 900 x 1600 frame: `vidar_b200.image_aug` (host draws, then two
launches) against the reference's statements (cv2 / PIL / numpy on the host's CPU), at output heights 720, 900 and
1080, with and without the photometric step; then one synthetic pre-training step with `image_pipeline=True`
against the default (float images already on the device), alternated.

  * kernel: CUDA events around `apply_multiview` alone (median of 20, warmed up); the bytes the pass must move
    (read the uint8 frame, write the float32 output) over that time, and over 3.35 TB/s, the H100 SXM data-sheet
    HBM3 bandwidth;
  * host: wall clock from the draws (the four transforms' __call__) to a synchronised device result (median of 20);
  * reference: the reference's statements on this host's CPU for the same draws, one process (median of 3; needs
    cv2 and PIL, as the reference does -- the arm is skipped when they are missing);
  * upload: host-to-device bytes per frame, the uint8 frame against the reference's float32 padded tensor;
  * step: `pretrain.train_step`, image pipeline on against off (median of --steps, alternated).
The card's name, power limit and SM clock are read in the same run.

    python tools/bench_image_aug.py [--steps 5] [--out /tmp/bench_image_aug.json]
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

from oracle import image_aug_ref  # noqa: E402
from tools.gpu_timing import card, event_ms, host_ms  # noqa: E402
from vidar_b200 import image_aug, pretrain  # noqa: E402

N, H, W = 6, 900, 1600
PEAK_BW = 3.35e12


def transforms(h, photo):
    steps = image_aug.config_pipeline(dict(reisze=[h], crop=(0, 0, W, H), H=H, W=W, rand_flip=True))
    return steps if photo else steps[1:]


def frame_results(src_list, steps, seed=0):
    np.random.seed(seed)
    random.seed(seed)
    results = dict(img=src_list, cam2img=[np.eye(4) for _ in range(N)], lidar2cam=[np.eye(4) for _ in range(N)])
    for s in steps:
        results = s(results)
    return results


def has_cv2_pil():
    try:
        import cv2  # noqa: F401
        import PIL  # noqa: F401
        return True
    except ImportError:
        return False


def op_bench(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    src = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
    src_host = src.cpu().numpy()
    res = {}
    for h in (720, 900, 1080):
        for photo in (True, False):
            steps = transforms(h, photo)
            results = frame_results(list(src), steps)
            plan = results["img_aug"]
            hp, wp = plan.pad_hw
            out = image_aug.apply_multiview(src, results)
            # same values first: camera 0 against the closed-form oracle
            want = image_aug_ref.pipeline(src_host[0], plan.photo[0] if photo else None, plan.crop, plan.dims,
                                          plan.flip, plan.mean, plan.std, plan.to_rgb, plan.pad_hw, plan.pad_val)
            assert np.array_equal(out[0].permute(1, 2, 0).cpu().numpy().view(np.uint32), want.view(np.uint32))
            nbytes = src.numel() + out.numel() * 4
            r = dict(out_shape=list(out.shape),
                     kernel_ms=event_ms(lambda: image_aug.apply_multiview(src, results), 20, 3))
            r["algorithmic_bytes"] = nbytes
            r["kernel_GBps"] = nbytes / (r["kernel_ms"] * 1e-3) / 1e9
            r["kernel_bytes_share_of_peak"] = nbytes / (r["kernel_ms"] * 1e-3) / PEAK_BW
            r["host_ms_with_draws"] = host_ms(lambda: image_aug.apply_multiview(
                src, frame_results(list(src), steps)), 20, 3)
            r["h2d_bytes_uint8_frame"] = src.numel()
            r["h2d_bytes_reference_float32"] = N * 3 * hp * wp * 4
            if has_cv2_pil():
                r["reference_cpu_ms_per_frame"] = host_ms(lambda: [image_aug_ref.pipeline_statements(
                    src_host[n], plan.photo[n] if photo else None, plan.crop, plan.dims, plan.flip, plan.mean,
                    plan.std, plan.to_rgb, plan.pad_hw, plan.pad_val[0]) for n in range(N)], 3, 0)
                r["host_cpus"] = os.cpu_count()
            else:
                r["reference_cpu_ms_per_frame"] = "not measured (cv2 or PIL missing)"
            key = f"h{h}_{'photo' if photo else 'nophoto'}"
            res[key] = r
            print(json.dumps({key: r}), flush=True)
    return res


def step_bench(dev, steps):
    model, opt = pretrain.build(dev, None, seed=0, image_pipeline=True)
    raw = pretrain.synthetic_sample(dev, raw_images=True)
    plain = pretrain.synthetic_sample(dev)

    def run(k):
        model.image_transforms = transforms_on if k == "pipeline" else None
        pretrain.train_step(model, opt, raw if k == "pipeline" else plain)

    transforms_on = model.image_transforms
    np.random.seed(0)
    random.seed(0)
    med, ms = host_ms({k: lambda k=k: run(k) for k in ("pipeline", "default")}, steps, 1, raw=True)   # alternating
    model.image_transforms = transforms_on
    return {k: dict(median_ms=med[k], all_ms=ms[k]) for k in med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_aug needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(card=card(), frame=[N, H, W, 3], op=op_bench(dev))
    res["step"] = step_bench(dev, args.steps)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
