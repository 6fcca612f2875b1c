"""Shared inputs of the memory-efficient and fine-tuning image pipeline tests: the golden cases of
tests/golden/image_aug_configs.npz (written by tools/make_golden_image_aug_configs.py from the reference's own
transforms) replayed through vidar_b200.image_aug, and the oracle of both chains: RandomCropResizeFlipImage's
resize-then-crop and the float chain with no crop step, composed of oracle/image_aug_ref.py's steps."""
import copy
import json
import os
import random

import numpy as np

from oracle import image_aug_ref as ref
from vidar_b200 import image_aug

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_aug_configs.npz")


def golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["cases"]))


def transforms(meta):
    pad = dict(meta["pad"])
    if isinstance(pad.get("pad_val"), list):
        pad["pad_val"] = tuple(pad["pad_val"])
    if pad.get("size") is not None:
        pad["size"] = tuple(pad["size"])
    steps = [image_aug.PhotoMetricDistortionMultiViewImage()] if meta["photometric"] else []
    if meta["crop"] is not None:
        steps.append(image_aug.RandomCropResizeFlipImage(**meta["crop"]))
    return steps + [image_aug.NormalizeMultiviewImage(**meta["normalize"]), image_aug.PadMultiViewImage(**pad)]


def replay(z, name, meta):
    """Run the case's frames through the package's transforms after the golden's seeding -> [(results, states)] per
    frame, states = (numpy MT key + pos + has_gauss, cached gaussian, random's state words) after the frame."""
    steps = transforms(meta)
    np.random.seed(meta["seed"])
    random.seed(meta["seed"])
    aug_param, out = None, []
    for t in range(meta["frames"]):
        results = dict(img=list(z[f"{name}.{t}.src"]), cam2img=[m.copy() for m in z["cam2img"]],
                       lidar2cam=[m.copy() for m in z["lidar2cam"]])
        if aug_param is not None:
            results["aug_param"] = copy.deepcopy(aug_param)
        for s in steps:
            results = s(results)
        aug_param = copy.deepcopy(results.get("aug_param"))
        st = np.random.get_state()
        states = (np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4]),
                  np.array(random.getstate()[1], np.int64))
        out.append((results, states))
    return out


# ---------------------------------------------------------------------------------------------------------------
# oracle of the two chains, built on oracle/image_aug_ref.py's steps: closed form (numpy only) and statements form
# (the reference's cv2 / PIL / numpy calls; needs cv2 and PIL)
# ---------------------------------------------------------------------------------------------------------------
def resize_crop_flip(img_u8, dims, box, flip):
    """RandomCropResizeFlipImage's pixels: resize the whole image to dims = (w, h), crop `box` of the resized image
    (zero outside it), FLIP_LEFT_RIGHT -> uint8 [box h, box w, 3]."""
    out = ref.crop(ref.resize(img_u8, *dims), box)
    return np.ascontiguousarray(out[:, ::-1]) if flip else out


def pipeline_resize_crop(img_u8, draw, dims, box, flip, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False, shape=None,
                         pad_val=0):
    """The four steps with RandomCropResizeFlipImage on one uint8 [H, W, 3] BGR image -> float32 [Hp, Wp, 3]."""
    x = np.asarray(img_u8, np.float32)
    if draw is not None:
        x = ref.photometric(x, draw)
    x = resize_crop_flip(ref.to_uint8(x), dims, box, flip).astype(np.float32)
    x = ref.normalize(x, mean, std, to_rgb)
    return x if shape is None else ref.pad(x, shape, pad_val)


def pipeline_float(img_u8, draw, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False, shape=None, pad_val=0):
    """Photometric distortion (draw None: none), normalisation and padding of one uint8 [H, W, 3] BGR image read as
    float32, the distorted pixels unclamped and not cast -> float32 [Hp, Wp, 3]."""
    x = np.asarray(img_u8, np.float32)
    if draw is not None:
        x = ref.photometric(x, draw)
    x = ref.normalize(x, mean, std, to_rgb)
    return x if shape is None else ref.pad(x, shape, pad_val)


def resize_crop_flip_statements(img, dims, box, flip):
    from PIL import Image
    im = Image.fromarray(np.uint8(img)).resize(dims).crop(box)
    if flip:
        im = im.transpose(method=Image.FLIP_LEFT_RIGHT)
    return np.array(im).astype(np.float32)


def pipeline_resize_crop_statements(img_u8, draw, dims, box, flip, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False,
                                    shape=None, pad_val=0):
    x = np.asarray(img_u8, np.float32)
    if draw is not None:
        x = ref.photometric_statements(x, draw)
    x = ref.normalize_statements(resize_crop_flip_statements(x, dims, box, flip), mean, std, to_rgb)
    return x if shape is None else ref.pad_statements(x, shape, pad_val)


def pipeline_float_statements(img_u8, draw, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False, shape=None, pad_val=0):
    x = np.asarray(img_u8, np.float32)
    if draw is not None:
        x = ref.photometric_statements(x, draw)
    x = ref.normalize_statements(x, mean, std, to_rgb)
    return x if shape is None else ref.pad_statements(x, shape, pad_val)


def oracle_frame(src, plan, statements=False):
    """The oracle (closed form, or the reference's statements) on every image of a frame, from its recorded plan of
    either chain -> float32 [N, Hp, Wp, 3]."""
    outs = []
    for n in range(plan.n):
        draw = plan.photo[n] if plan.photo is not None else None
        norm = (plan.mean, plan.std, plan.to_rgb, plan.pad_hw, plan.pad_val)
        if plan.crop is None:
            f = pipeline_float_statements if statements else pipeline_float
            outs.append(f(src[n], draw, *norm))
        else:
            assert plan.crop == (0, 0, src.shape[2], src.shape[1]) and plan.window is not None
            f = pipeline_resize_crop_statements if statements else pipeline_resize_crop
            outs.append(f(src[n], draw, plan.dims, plan.window, plan.flip, *norm))
    return np.stack(outs)
