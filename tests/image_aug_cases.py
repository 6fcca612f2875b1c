"""Shared inputs of the image pipeline tests: the golden cases of tests/golden/image_aug.npz (written by
tools/make_golden_image_aug.py from the reference's own transforms) replayed through vidar_b200.image_aug, and
photometric draws that cover every gate pattern."""
import copy
import itertools
import json
import os
import random

import numpy as np

from vidar_b200 import image_aug
from vidar_b200.image_aug import PhotoDraw

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_aug.npz")


def golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["cases"]))


def transforms(meta):
    steps = [image_aug.PhotoMetricDistortionMultiViewImage()] if meta["photometric"] else []
    pad = dict(meta["pad"])
    if isinstance(pad.get("pad_val"), list):
        pad["pad_val"] = tuple(pad["pad_val"])
    if pad.get("size") is not None:
        pad["size"] = tuple(pad["size"])
    conf = dict(meta["ida_aug_conf"], crop=tuple(meta["ida_aug_conf"]["crop"]))
    return steps + [image_aug.CropResizeFlipImage(data_aug_conf=conf, training=True, debug=False),
                    image_aug.NormalizeMultiviewImage(**meta["normalize"]), image_aug.PadMultiViewImage(**pad)]


def replay(z, name, meta):
    """Run the case's frames through the package's transforms after the golden's seeding -> [(results, states)] per
    frame, states = (numpy MT key + pos + has_gauss, cached gaussian, random's state words) after the frame."""
    steps = transforms(meta)
    np.random.seed(meta["seed"])
    random.seed(meta["seed"])
    aug_param, out = None, []
    for t in range(meta["frames"]):
        src = z[f"{name}.{t}.src"]
        results = dict(img=list(src), cam2img=[m.copy() for m in z["cam2img"]],
                       lidar2cam=[m.copy() for m in z["lidar2cam"]])
        if aug_param is not None:
            results["aug_param"] = copy.deepcopy(aug_param)
        for s in steps:
            results = s(results)
        aug_param = copy.deepcopy(results["aug_param"])
        st = np.random.get_state()
        states = (np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4]),
                  np.array(random.getstate()[1], np.int64))
        out.append((results, states))
    return out


def oracle_frame(ref, src, plan):
    """The closed-form oracle on every image of a frame, from its recorded plan -> float32 [N, Hp, Wp, 3]."""
    H, W = src.shape[1:3]
    box = plan.crop if plan.crop is not None else (0, 0, W, H)
    dims = plan.dims if plan.dims is not None else (W, H)
    outs = []
    for n in range(plan.n):
        draw = plan.photo[n] if plan.photo is not None else None
        outs.append(ref.pipeline(src[n], draw, box, dims, plan.flip, plan.mean, plan.std, plan.to_rgb, plan.pad_hw,
                                 plan.pad_val))
    return np.stack(outs)


def gate_draws(seed=0):
    """PhotoDraws covering every gate pattern (brightness, contrast, saturation, hue, swap) in both modes, with
    factors at and near the ends of the config's ranges."""
    rng = np.random.default_rng(seed)
    perms = list(itertools.permutations(range(3)))
    draws = []
    for gates in itertools.product((0, 1), repeat=5):
        for mode in (0, 1):
            b, c, s, h, p = gates
            draws.append(PhotoDraw(
                delta=float(rng.choice([-32.0, 32.0, rng.uniform(-32, 32)])) if b else None, mode=mode,
                alpha=float(rng.choice([0.5, 1.5, rng.uniform(0.5, 1.5)])) if c else None,
                sat=float(rng.choice([0.5, 1.5, rng.uniform(0.5, 1.5)])) if s else None,
                hue=float(rng.choice([-18.0, 18.0, rng.uniform(-18, 18)])) if h else None,
                perm=perms[int(rng.integers(len(perms)))] if p else None))
    return draws
