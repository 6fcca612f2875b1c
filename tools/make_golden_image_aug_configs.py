"""Write tests/golden/image_aug_configs.npz: the reference's own image transforms for the pipelines of the
memory-efficient pre-training config (PhotoMetricDistortionMultiViewImage -> RandomCropResizeFlipImage ->
NormalizeMultiviewImage -> PadMultiViewImage), the fine-tuning configs (PhotoMetricDistortionMultiViewImage ->
NormalizeMultiviewImage -> PadMultiViewImage, no crop step) and the test pipelines (NormalizeMultiviewImage ->
PadMultiViewImage), loaded through tools/ref_shim.py with mmcv / mmdet stand-ins, on small seeded frames.

The frames are 2 x 45 x 80 BGR images of random 3 x 4 blocks with a saturated and a black patch (so brightness and
contrast push pixels past 255 and below 0; the blocks keep the file small), with the first two cameras of
tools/make_golden_image_aug.py's rig.  They run as a queue (later frames take the resize / crop / flip from
`aug_param`) after seeding numpy's global generator and the stdlib `random`.  Per frame the file holds the output images [N, Hp, Wp, 3] float32, cam2img and lidar2img
(cases with a crop step), the shape keys, and numpy's and `random`'s states after the call.

    python tools/make_golden_image_aug_configs.py
"""
import copy
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden_image_aug import np_state, rig  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "image_aug_configs.npz")

CONFIG_NORM = dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False)
RGB_NORM = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)


N, H, W = 2, 45, 80


def conf(reisze, crop=(0, 0, W, H), H=H, W=W, rand_flip=True):
    return dict(reisze=reisze, crop=crop, H=H, W=W, rand_flip=rand_flip)


def frames(seed, count):
    """count uint8 frames [N, H, W, 3] of random 3 x 4 pixel blocks, with a saturated and a black patch each."""
    rng = np.random.default_rng(200 + seed)
    out = []
    for _ in range(count):
        f = np.kron(rng.integers(0, 256, (N, H // 3, W // 4, 3)), np.ones((1, 3, 4, 1), np.int64))
        f[:, 5:11, 10:20] = 255
        f[:, 30:38, 50:65] = 0
        out.append(f.astype(np.uint8))
    return out


# name -> (seed, frames, photometric, RandomCropResizeFlipImage kwargs or None, normalize kwargs, pad kwargs).
# The 45 x 80 frames stand for nuScenes' 900 x 1600 at a twentieth: heights 36 / 45 / 54 are below, at and above the
# crop's 45 rows, and their widths 64 / 80 / 96 below, at and above its 80 columns.
CASES = {
    "mem_below": (0, 2, True, dict(data_aug_conf=conf([36])), CONFIG_NORM, dict(size_divisor=32)),
    "mem_at": (1, 1, True, dict(data_aug_conf=conf([45])), CONFIG_NORM, dict(size_divisor=32)),
    "mem_above": (12, 1, True, dict(data_aug_conf=conf([54])), CONFIG_NORM, dict(size_divisor=32)),
    "mem_config": (27, 2, True, dict(data_aug_conf=conf([36, 40, 45, 49, 54])), CONFIG_NORM,
                   dict(size_divisor=32)),
    "mem_no_flip": (4, 1, True, dict(data_aug_conf=conf([54], rand_flip=False)), CONFIG_NORM, dict(size_divisor=32)),
    # the conf's H / W set the resize, not the image's; a crop wider and shorter than the resize, rgb, std, size pad
    "mem_conf_hw_rgb": (5, 2, True, dict(data_aug_conf=conf([50], crop=(0, 0, 88, 40), H=50, W=75)), RGB_NORM,
                        dict(size=(48, 96), pad_val=(1.5, -2.0, 3.0))),
    "mem_no_photo": (6, 1, False, dict(data_aug_conf=conf([54])), CONFIG_NORM, dict(size_divisor=32, pad_val=5)),
    "mem_eval": (7, 1, True, dict(data_aug_conf=conf([50], crop=(5, 2, 75, 42)), training=False), CONFIG_NORM,
                 dict(size_divisor=32)),
    "mem_eval_full_crop": (8, 1, False, dict(data_aug_conf=conf([36]), training=False), CONFIG_NORM,
                           dict(size_divisor=32)),
    "finetune": (9, 1, True, None, CONFIG_NORM, dict(size_divisor=32)),
    "finetune_rgb_size": (10, 1, True, None, RGB_NORM, dict(size=(48, 88), pad_val=(1.5, -2.0, 3.0))),
    "finetune_seed11": (11, 1, True, None, dict(mean=[103.530, 116.280, 123.675], std=[2.0, 1.0, 0.5],
                                                to_rgb=True), dict(size_divisor=32, pad_val=2)),
    "test_pipeline": (12, 1, False, None, CONFIG_NORM, dict(size_divisor=32)),
}


def main():
    classes = ref_shim.install_pipelines()
    cam2img, lidar2cam = (a[:N] for a in rig())
    out = {"cam2img": cam2img, "lidar2cam": lidar2cam}
    meta = {}
    for name, (seed, count, photo, crop, norm, pad) in CASES.items():
        steps = (([classes["PhotoMetricDistortionMultiViewImage"]()] if photo else [])
                 + ([classes["RandomCropResizeFlipImage"](**crop)] if crop is not None else [])
                 + [classes["NormalizeMultiviewImage"](**norm), classes["PadMultiViewImage"](**pad)])
        np.random.seed(seed)
        random.seed(seed)
        aug_param = None
        for t, imgs in enumerate(frames(seed, count)):
            results = dict(img=[im.astype(np.float32) for im in imgs], cam2img=[m.copy() for m in cam2img],
                           lidar2cam=[m.copy() for m in lidar2cam])
            if aug_param is not None:
                results["aug_param"] = copy.deepcopy(aug_param)
            for step in steps:
                results = step(results)
            key = f"{name}.{t}"
            out[f"{key}.src"] = imgs
            out[f"{key}.img"] = np.stack(results["img"])
            if crop is not None:
                aug_param = copy.deepcopy(results["aug_param"])
                out[f"{key}.cam2img"] = np.stack(results["cam2img"])
                out[f"{key}.lidar2img"] = np.stack(results["lidar2img"])
                out[f"{key}.flip"] = np.array(aug_param["CropResizeFlipImage_param"][3], bool)
            for k in ("ori_shape", "img_shape", "pad_shape"):
                out[f"{key}.{k}"] = np.array(results[k], np.int64)
            out[f"{key}.np_state"], out[f"{key}.np_gauss"] = np_state()
            out[f"{key}.random_state"] = np.array(random.getstate()[1], np.int64)
        meta[name] = dict(seed=seed, frames=count, photometric=photo, crop=crop, normalize=norm, pad=pad)
    out["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1e6:.2f} MB, {len(CASES)} cases")


if __name__ == "__main__":
    main()
