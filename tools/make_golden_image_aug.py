"""Write tests/golden/image_aug.npz: the reference's own image transforms (datasets/pipelines/transform_3d.py
PhotoMetricDistortionMultiViewImage, NormalizeMultiviewImage, PadMultiViewImage; augmentation.py
CropResizeFlipImage), loaded through tools/ref_shim.py with mmcv / mmdet stand-ins, on small seeded frames.

Each case runs a queue of frames through the transforms, as the dataset does (the first frame draws the crop /
resize / flip, later frames take it from `aug_param`), after seeding numpy's global generator and the stdlib
`random`.  Per frame it stores the output images [N, Hp, Wp, 3] float32, cam2img, lidar2img, the shape keys, and
numpy's and `random`'s states after the call.  The inputs are 3 x 90 x 160 BGR frames of random 6 x 8 blocks with
saturated and black patches (so brightness and contrast push pixels past 255 and below 0), and the same cam2img /
lidar2cam.  The blocks keep the file small (deflate finds their repeats; it does not find smooth gradients').

    python tools/make_golden_image_aug.py
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

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "image_aug.npz")
N, H, W = 3, 90, 160

# name -> (seed, frames, photometric, ida_aug_conf, normalize kwargs, pad kwargs)
CASES = {
    "config": (0, 2, True, dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True),
               dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False), dict(size_divisor=32)),
    "config_seed1": (1, 1, True, dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True),
                     dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False), dict(size_divisor=32)),
    "config_seed5": (5, 1, True, dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True),
                     dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False), dict(size_divisor=32)),
    "outside_rgb_std": (5, 2, True, dict(reisze=[72, 108], crop=(-8, 6, 168, 96), H=90, W=160, rand_flip=True),
                        dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                        dict(size=(128, 224), pad_val=(1.5, -2.0, 3.0))),
    "inside_no_photo": (4, 1, False, dict(reisze=[80], crop=(10, 4, 150, 84), H=90, W=160, rand_flip=True),
                        dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False),
                        dict(size_divisor=32, pad_val=5)),
}


def frames(seed, count):
    """count uint8 frames [N, H, W, 3] of random 6 x 8 pixel blocks, with a saturated and a black patch each."""
    rng = np.random.default_rng(100 + seed)
    out = []
    for _ in range(count):
        f = np.kron(rng.integers(0, 256, (N, H // 6, W // 8, 3)), np.ones((1, 6, 8, 1), np.int64))
        f[:, 10:22, 20:40] = 255
        f[:, 60:75, 100:130] = 0
        out.append(f.astype(np.uint8))
    return out


def rig():
    rng = np.random.default_rng(7)
    cam2img, lidar2cam = [], []
    for _ in range(N):
        k = np.eye(4)
        k[0, 0] = k[1, 1] = rng.uniform(120, 130)
        k[0, 2], k[1, 2] = rng.uniform(75, 85), rng.uniform(40, 50)
        e = np.eye(4)
        e[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        e[:3, 3] = rng.normal(size=3)
        cam2img.append(k)
        lidar2cam.append(e)
    return np.stack(cam2img), np.stack(lidar2cam)


def np_state():
    s = np.random.get_state()
    return np.concatenate([s[1].astype(np.int64), [s[2], s[3]]]), np.float64(s[4])


def main():
    classes = ref_shim.install_pipelines()
    cam2img, lidar2cam = rig()
    out = {"cam2img": cam2img, "lidar2cam": lidar2cam}
    meta = {}
    for name, (seed, count, photo, conf, norm, pad) in CASES.items():
        steps = ([classes["PhotoMetricDistortionMultiViewImage"]()] if photo else []) + [
            classes["CropResizeFlipImage"](data_aug_conf=conf, training=True, debug=False),
            classes["NormalizeMultiviewImage"](**norm), classes["PadMultiViewImage"](**pad)]
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
            aug_param = copy.deepcopy(results["aug_param"])
            key = f"{name}.{t}"
            out[f"{key}.src"] = imgs
            out[f"{key}.img"] = np.stack(results["img"])
            out[f"{key}.cam2img"] = np.stack(results["cam2img"])
            out[f"{key}.lidar2img"] = np.stack(results["lidar2img"])
            for k in ("ori_shape", "img_shape", "pad_shape"):
                out[f"{key}.{k}"] = np.array(results[k], np.int64)
            out[f"{key}.np_state"], out[f"{key}.np_gauss"] = np_state()
            out[f"{key}.random_state"] = np.array(random.getstate()[1], np.int64)
        meta[name] = dict(seed=seed, frames=count, photometric=photo, ida_aug_conf=conf, normalize=norm, pad=pad)
    out["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1e6:.2f} MB, {len(CASES)} cases")


if __name__ == "__main__":
    main()
