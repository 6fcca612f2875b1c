"""The multi-view image pipelines of ViDAR's configs on the H100:

    pre-training (vidar_1_8_nusc_3future.py:279-317):
        PhotoMetricDistortionMultiViewImage -> CropResizeFlipImage(ida_aug_conf) -> NormalizeMultiviewImage
          -> PadMultiViewImage
    memory-efficient pre-training (mem_efficient_vidar_1_8_nusc_3future.py:307-314):
        PhotoMetricDistortionMultiViewImage -> RandomCropResizeFlipImage(ida_aug_conf) -> NormalizeMultiviewImage
          -> PadMultiViewImage
    fine-tuning (vidar_finetune/*, bevformer_base.py) and every nuScenes test pipeline:
        [PhotoMetricDistortionMultiViewImage ->] NormalizeMultiviewImage -> PadMultiViewImage
    OpenScene pre-training and test (vidar_OpenScene_*_3future.py:297-312):
        [PhotoMetricDistortionMultiViewImage ->] NormalizeMultiviewImage -> RandomScaleImageMultiViewImage([2/3])
          -> PadMultiViewImage

The six classes take the reference's constructor arguments (datasets/pipelines/transform_3d.py:7-185,
augmentation.py:10-301).  Used as dataloader transforms, their `__call__(results)` does only the host work: the
same draws from the same generators in the same order (numpy's global generator for the photometric gates and
factors, the crop offset and the flip, the stdlib `random` for the resize, cached in `results['aug_param']` so
that the later frames of a queue reuse it), the `cam2img` / `lidar2img` / `img_norm_cfg` / shape keys as the
reference sets them, and a record of what to do to the pixels in `results['img_aug']`.  `results['img']` is left
as loaded (uint8).

`apply_multiview(img, results)` then runs the recorded chain on the device, on the current stream (csrc/image_aug.cu,
include/vidar_b200.h §x): uint8 [N, H, W, 3] BGR in, float32 [N, 3, Hp, Wp] out, bit for bit what the reference's
cv2 / PIL / numpy statements give.  With a crop step that is two launches, including numpy's wrapping `np.uint8`
cast of pixels that brightness and contrast push past 255 or below 0; without one it is one launch, and the
photometric output reaches the normalisation as unclamped float32, as in the reference.  With a rescale step
(the OpenScene chains) it is one launch too: photometric, normalisation, mmcv.imresize and padding per output pixel.  The per-image draws
travel in the kernel arguments; the resample taps are computed on the host in float64 by Pillow's rules, cached per
(input size, output size, device) and uploaded once from pinned memory without blocking.  No host sync.  CUDA
tensors only.
"""
import random
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib

MAX_IMAGES = 64
MAX_SIDE = 8192
PRECISION_BITS = 22


@dataclass(frozen=True)
class PhotoDraw:
    """One image's photometric draws; None where the step's gate was closed.  `mode` 1 puts contrast before the
    HSV round trip, 0 after it; `perm` is the channel permutation."""
    delta: float = None
    mode: int = 0
    alpha: float = None
    sat: float = None
    hue: float = None
    perm: tuple = None


@dataclass
class ImageAugPlan:
    """What `apply_multiview` does to one frame's images, recorded by the transforms in `results['img_aug']`."""
    n: int
    src_hw: tuple
    photo: list = None                 # [PhotoDraw] per image, or None
    crop: tuple = None                 # (x0, y0, x1, y1)
    dims: tuple = None                 # (w, h) after the resize
    flip: bool = False
    mean: np.ndarray = field(default_factory=lambda: np.zeros(3, np.float32))
    std: np.ndarray = field(default_factory=lambda: np.ones(3, np.float32))
    to_rgb: bool = False
    normalized: bool = False
    pad_hw: tuple = None
    pad_val: tuple = (0.0, 0.0, 0.0)
    window: tuple = None               # (x0, y0, x1, y1) of the resized image, zero outside; None: all of it
    scale_hw: tuple = None             # (h, w) after RandomScaleImageMultiViewImage, or None

    @property
    def hw(self):
        """(h, w) of the images after the steps recorded so far."""
        if self.pad_hw is not None:
            return self.pad_hw
        if self.scale_hw is not None:
            return self.scale_hw
        if self.window is not None:
            return self.window[3] - self.window[1], self.window[2] - self.window[0]
        return (self.dims[1], self.dims[0]) if self.dims is not None else tuple(self.src_hw)


def _plan(results, step):
    """results['img_aug'], created at the first step; raises when `step` comes out of the order the device chain
    runs (photometric, crop / resize / flip, normalise, pad; each at most once)."""
    imgs = results["img"]
    plan = results.get("img_aug")
    if plan is None:
        shapes = {tuple(im.shape) for im in imgs}
        if len(imgs) == 0 or len(shapes) != 1 or len(next(iter(shapes))) != 3 or next(iter(shapes))[2] != 3:
            raise ValueError(f"image pipeline: results['img'] must be images of one [H, W, 3] shape (got {shapes})")
        plan = results["img_aug"] = ImageAugPlan(len(imgs), next(iter(shapes))[:2])
    elif plan.n != len(imgs):
        raise ValueError(f"image pipeline: {len(imgs)} images, the recorded steps saw {plan.n}")
    done = {"photo": plan.photo is not None, "crop": plan.crop is not None, "norm": plan.normalized,
            "scale": plan.scale_hw is not None, "pad": plan.pad_hw is not None}
    order = ["photo", "crop", "norm", "scale", "pad"]
    later = order[order.index(step):]
    if any(done[s] for s in later):
        raise ValueError(f"image pipeline: step '{step}' after {[s for s in order if done[s]]}; the device chain "
                         "runs photometric distortion, crop / resize / flip, normalisation, rescale and padding in "
                         "this order, each at most once")
    return plan


class PhotoMetricDistortionMultiViewImage:
    """transform_3d.py:98-185: per image, numpy draws for brightness, mode, contrast, saturation, hue and the
    channel swap, in the reference's order (contrast before the HSV round trip when mode == 1)."""

    def __init__(self, brightness_delta=32, contrast_range=(0.5, 1.5), saturation_range=(0.5, 1.5), hue_delta=18):
        self.brightness_delta = brightness_delta
        self.contrast_lower, self.contrast_upper = contrast_range
        self.saturation_lower, self.saturation_upper = saturation_range
        self.hue_delta = hue_delta

    def draw(self):
        """One image's draws from numpy's global generator -> PhotoDraw."""
        rnd = np.random
        delta = alpha = sat = hue = perm = None
        if rnd.randint(2):
            delta = rnd.uniform(-self.brightness_delta, self.brightness_delta)
        mode = rnd.randint(2)
        if mode == 1 and rnd.randint(2):
            alpha = rnd.uniform(self.contrast_lower, self.contrast_upper)
        if rnd.randint(2):
            sat = rnd.uniform(self.saturation_lower, self.saturation_upper)
        if rnd.randint(2):
            hue = rnd.uniform(-self.hue_delta, self.hue_delta)
        if mode == 0 and rnd.randint(2):
            alpha = rnd.uniform(self.contrast_lower, self.contrast_upper)
        if rnd.randint(2):
            perm = tuple(int(c) for c in rnd.permutation(3))
        return PhotoDraw(delta, int(mode), alpha, sat, hue, perm)

    def __call__(self, results):
        plan = _plan(results, "photo")
        plan.photo = [self.draw() for _ in range(plan.n)]
        return results


class CropResizeFlipImage:
    """augmentation.py:9-202: one crop / resize / flip per frame, drawn (stdlib `random.choice` for the height,
    `np.random.choice([0, 1])` for the flip when `rand_flip`) or taken from results['aug_param'].  Updates
    `cam2img[:3, :3]` with the crop / resize matrix (which, as in the reference, leaves the flip out) and sets
    `lidar2img = cam2img @ lidar2cam`."""

    def __init__(self, data_aug_conf=None, training=True, debug=False):
        if debug:
            raise ValueError("CropResizeFlipImage: debug=True (drawing projected points into saved images) is not "
                             "supported")
        self.data_aug_conf = data_aug_conf
        self.training = training
        self.debug = debug

    def _sample_augmentation(self, results):
        if "CropResizeFlipImage_param" in results["aug_param"]:
            return results["aug_param"]["CropResizeFlipImage_param"]
        conf = self.data_aug_conf
        crop = conf["crop"]
        resized_h = random.choice(conf["reisze"])
        if not self.training and len(conf["reisze"]) != 1:
            raise ValueError("CropResizeFlipImage: training=False needs exactly one entry in 'reisze'")
        resized_w = resized_h / (crop[3] - crop[1]) * (crop[2] - crop[0])
        resize = resized_h / (crop[3] - crop[1])
        resize_dims = (int(resized_w), int(resized_h))
        flip = False
        if self.training and conf["rand_flip"] and np.random.choice([0, 1]):
            flip = True
        results["aug_param"]["CropResizeFlipImage_param"] = (resize, resize_dims, crop, flip)
        return resize, resize_dims, crop, flip

    def __call__(self, results):
        if "mono_ann_idx" in results:
            raise ValueError("CropResizeFlipImage: the DD3D mono annotations ('mono_ann_idx') are not supported")
        plan = _plan(results, "crop")
        if "aug_param" not in results:
            results["aug_param"] = {}
        resize, resize_dims, crop, flip = self._sample_augmentation(results)
        x0, y0, x1, y1 = (int(round(v)) for v in crop)
        w, h = (int(v) for v in resize_dims)
        if not (0 < x1 - x0 <= MAX_SIDE and 0 < y1 - y0 <= MAX_SIDE and 0 < w <= MAX_SIDE and 0 < h <= MAX_SIDE):
            raise ValueError(f"CropResizeFlipImage: crop {crop} -> {resize_dims} is outside 1..{MAX_SIDE} pixels")
        ida_mat = np.eye(3)
        ida_mat[:2, :2] *= resize
        ida_mat[:2, 2] -= np.array(crop[:2]) * resize
        for i in range(plan.n):
            results["cam2img"][i][:3, :3] = np.matmul(ida_mat, results["cam2img"][i][:3, :3])
        results["lidar2img"] = [np.matmul(results["cam2img"][i], results["lidar2cam"][i])
                                for i in range(len(results["lidar2cam"]))]
        plan.crop, plan.dims, plan.flip = (x0, y0, x1, y1), (w, h), bool(flip)
        return results


class RandomCropResizeFlipImage:
    """augmentation.py:204-301: one resize / crop / flip per frame -- the whole image resized first, then cropped to
    the conf's crop size, zero outside the resized image.  Training draws the height (stdlib `random.choice`), the
    crop's x offset (`np.random.uniform(0, max(0, newW - fW))`, a draw even when the range is empty), the bottom-
    aligned crop's y offset (no draw) and the flip (`np.random.choice([0, 1])` when `rand_flip`); `training=False`
    resizes to the one height and crops with the conf's box.  The result is cached in results['aug_param'] under
    the key CropResizeFlipImage uses.  Updates `cam2img[:3, :3]` with [[r, 0, -crop_x], [0, r, -crop_y]] (the
    translation not scaled, the flip left out, as in the reference) and sets `lidar2img = cam2img @ lidar2cam`."""

    def __init__(self, data_aug_conf=None, training=True):
        self.data_aug_conf = data_aug_conf
        self.training = training

    def _sample_augmentation(self, results):
        if "CropResizeFlipImage_param" in results["aug_param"]:
            return results["aug_param"]["CropResizeFlipImage_param"]
        conf = self.data_aug_conf
        H, W = conf["H"], conf["W"]
        crop = conf["crop"]
        fW, fH = int(crop[2] - crop[0]), int(crop[3] - crop[1])
        resized_h = random.choice(conf["reisze"])
        if self.training:
            resized_w = resized_h / H * W
            resize = resized_h / H
            resize_dims = (int(resized_w), int(resized_h))
            newW, newH = resize_dims
            crop_h = int(max(0, newH - fH))
            crop_w = int(np.random.uniform(0, max(0, newW - fW)))
            crop = (crop_w, crop_h, crop_w + fW, crop_h + fH)
            flip = False
            if conf["rand_flip"] and np.random.choice([0, 1]):
                flip = True
        else:
            if len(conf["reisze"]) != 1:
                raise ValueError("RandomCropResizeFlipImage: training=False needs exactly one entry in 'reisze'")
            resized_w = resized_h / (crop[3] - crop[1]) * (crop[2] - crop[0])
            resize = resized_h / (crop[3] - crop[1])
            resize_dims = (int(resized_w), int(resized_h))
            flip = False
        results["aug_param"]["CropResizeFlipImage_param"] = (resize, resize_dims, crop, flip)
        return resize, resize_dims, crop, flip

    def __call__(self, results):
        plan = _plan(results, "crop")
        if "aug_param" not in results:
            results["aug_param"] = {}
        resize, resize_dims, crop, flip = self._sample_augmentation(results)
        x0, y0, x1, y1 = (int(round(v)) for v in crop)
        w, h = (int(v) for v in resize_dims)
        if not (0 < x1 - x0 <= MAX_SIDE and 0 < y1 - y0 <= MAX_SIDE and 0 < w <= MAX_SIDE and 0 < h <= MAX_SIDE
                and -MAX_SIDE < x0 < w and -MAX_SIDE < y0 < h and x1 > 0 and y1 > 0):
            raise ValueError(f"RandomCropResizeFlipImage: resize to {resize_dims} and crop {crop} need sides in "
                             f"1..{MAX_SIDE} and a crop that overlaps the resized image")
        ida_rot = np.eye(2)
        ida_rot *= resize
        ida_tran = np.zeros(2)
        ida_tran -= np.array(crop[:2])
        ida_mat = np.eye(3)
        ida_mat[:2, :2] = ida_rot
        ida_mat[:2, 2] = ida_tran
        for i in range(plan.n):
            results["cam2img"][i][:3, :3] = np.matmul(ida_mat, results["cam2img"][i][:3, :3])
        results["lidar2img"] = [np.matmul(results["cam2img"][i], results["lidar2cam"][i])
                                for i in range(len(results["lidar2cam"]))]
        H, W = plan.src_hw
        plan.crop, plan.dims, plan.window, plan.flip = (0, 0, W, H), (w, h), (x0, y0, x1, y1), bool(flip)
        return results


class NormalizeMultiviewImage:
    """transform_3d.py:61-95 (mmcv.imnormalize): optional BGR -> RGB, then (x - mean) / std per channel."""

    def __init__(self, mean, std, to_rgb=True):
        self.mean = np.array(mean, dtype=np.float32)
        self.std = np.array(std, dtype=np.float32)
        self.to_rgb = to_rgb
        if self.mean.shape != (3,) or self.std.shape != (3,):
            raise ValueError("NormalizeMultiviewImage: mean and std need 3 values")

    def __call__(self, results):
        plan = _plan(results, "norm")
        plan.mean, plan.std, plan.to_rgb, plan.normalized = self.mean, self.std, bool(self.to_rgb), True
        results["img_norm_cfg"] = dict(mean=self.mean, std=self.std, to_rgb=self.to_rgb)
        return results


class RandomScaleImageMultiViewImage:
    """transform_3d.py:295-327: one scale per call from `scales`, drawn as the reference draws it --
    `np.random.permutation(range(len(scales)))[0]`, one permutation per call even with one scale --, then every
    image resized to (int(h * scale), int(w * scale)) with mmcv.imresize (cv2 INTER_LINEAR), `lidar2img` :=
    diag(scale, scale, 1, 1) @ lidar2img, and `img_shape` / `ori_shape` the resized shapes.  The device step supports
    the configs' 2/3 on sides divisible by 3 (1920 x 1080 -> 1280 x 720); other sizes are rejected here."""

    def __init__(self, scales=[]):
        self.scales = scales
        if len(self.scales) != 1:
            raise ValueError(f"RandomScaleImageMultiViewImage: exactly one scale, as the reference asserts (got "
                             f"{scales})")

    def __call__(self, results):
        plan = _plan(results, "scale")
        rand_scale = self.scales[np.random.permutation(range(len(self.scales)))[0]]
        h, w = plan.hw
        y_size, x_size = int(h * rand_scale), int(w * rand_scale)
        if plan.crop is not None or 2 * h != 3 * y_size or 2 * w != 3 * x_size:
            raise ValueError(f"RandomScaleImageMultiViewImage: {h} x {w} by {rand_scale} -> {y_size} x {x_size}: the "
                             "device chain supports a scale of 2/3 on sides divisible by 3, after no crop step")
        scale_factor = np.eye(4)
        scale_factor[0, 0] *= rand_scale
        scale_factor[1, 1] *= rand_scale
        results["lidar2img"] = [scale_factor @ l2i for l2i in results["lidar2img"]]
        results["img_shape"] = [(y_size, x_size, 3)] * plan.n
        results["ori_shape"] = [(y_size, x_size, 3)] * plan.n
        plan.scale_hw = (y_size, x_size)
        return results


class PadMultiViewImage:
    """transform_3d.py:7-58 (mmcv.impad / impad_to_multiple): bottom / right padding to `size` or to multiples of
    `size_divisor`.  A number `pad_val` fills channel 0 only and leaves 0 in the others, as cv2.copyMakeBorder does
    with a scalar; a 3-tuple fills each channel."""

    def __init__(self, size=None, size_divisor=None, pad_val=0):
        if (size is None) == (size_divisor is None):
            raise ValueError("PadMultiViewImage: give exactly one of size and size_divisor")
        self.size = size
        self.size_divisor = size_divisor
        self.pad_val = pad_val

    def __call__(self, results):
        plan = _plan(results, "pad")
        h, w = plan.hw
        if self.size is not None:
            hp, wp = int(self.size[0]), int(self.size[1])
            if hp < h or wp < w:
                raise ValueError(f"PadMultiViewImage: size {self.size} is smaller than the image ({h}, {w})")
        else:
            d = self.size_divisor
            hp, wp = -(-h // d) * d, -(-w // d) * d
        if hp > MAX_SIDE or wp > MAX_SIDE:
            raise ValueError(f"PadMultiViewImage: padded size ({hp}, {wp}) is over {MAX_SIDE}")
        pv = self.pad_val
        if isinstance(pv, tuple):
            if len(pv) != 3:
                raise ValueError(f"PadMultiViewImage: a tuple pad_val needs 3 values (got {pv})")
            plan.pad_val = tuple(float(v) for v in pv)
        else:
            plan.pad_val = (float(pv), 0.0, 0.0)
        results["ori_shape"] = [(h, w, 3)] * plan.n
        plan.pad_hw = (hp, wp)
        results["img_shape"] = [(hp, wp, 3)] * plan.n
        results["pad_shape"] = [(hp, wp, 3)] * plan.n
        results["pad_fixed_size"] = self.size
        results["pad_size_divisor"] = self.size_divisor
        return results


# ---------------------------------------------------------------------------------------------------------------
# device step
# ---------------------------------------------------------------------------------------------------------------
def bicubic_taps(in_size, out_size):
    """Pillow's antialiased BICUBIC taps (Resample.c precompute_coeffs + normalize_coeffs_8bpc), in float64 in its
    order of operations -> int32 [out_size, 2 + ksize]: per output pixel (xmin, count, weights in 2^-22 units)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    table = np.zeros((out_size, 2 + ksize), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        ws = []
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * ss)
            if t < 1.0:
                ws.append((1.5 * t - 2.5) * t * t + 1)
            elif t < 2.0:
                ws.append((((t - 5) * t + 8) * t - 4) * -0.5)
            else:
                ws.append(0.0)
        total = 0.0
        for v in ws:
            total += v
        table[xx, 0], table[xx, 1] = xmin, xmax
        for x, v in enumerate(ws):
            v = v / total if total != 0.0 else v
            table[xx, 2 + x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
    return table


_TAPS = {}


def _taps(in_size, out_size, device):
    """Device copy of bicubic_taps(in_size, out_size), made once per device from pinned memory without blocking
    (the pinned buffer is kept with it, so the copy never reads freed memory)."""
    key = (in_size, out_size, device)
    if key not in _TAPS:
        host = torch.from_numpy(bicubic_taps(in_size, out_size)).pin_memory()
        _TAPS[key] = (host.to(device, non_blocking=True), host)
    return _TAPS[key][0]


def _check(img, plan, cams):
    """Every argument check of apply_multiview, before any CUDA call; the device check comes last, so the others can
    be tested without a GPU."""
    if not isinstance(plan, ImageAugPlan):
        raise ValueError("apply_multiview: results has no recorded image steps (run the transforms first)")
    if plan.scale_hw is not None and not plan.normalized:
        raise ValueError("apply_multiview: RandomScaleImageMultiViewImage without NormalizeMultiviewImage is not "
                         "supported (the configs rescale the normalised float32 images)")
    if plan.photo is not None and plan.crop is None and not plan.normalized:
        raise ValueError("apply_multiview: photometric distortion without CropResizeFlipImage or "
                         "NormalizeMultiviewImage is not supported (the float32 pixels it makes are the output of "
                         "neither)")
    if not isinstance(img, torch.Tensor):
        raise TypeError(f"apply_multiview: img must be a tensor (got {type(img).__name__})")
    if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[-1] != 3:
        raise ValueError(f"apply_multiview: img must be uint8 [N, H, W, 3] (got {img.dtype} {tuple(img.shape)})")
    if tuple(img.shape[1:3]) != tuple(plan.src_hw):
        raise ValueError(f"apply_multiview: images are {tuple(img.shape[1:3])}, the steps were recorded for "
                         f"{tuple(plan.src_hw)}")
    if len(cams) != img.shape[0] or any(not 0 <= c < plan.n for c in cams) or len(set(cams)) != len(cams):
        raise ValueError(f"apply_multiview: cams {list(cams)} must name the {img.shape[0]} images given, out of "
                         f"{plan.n}")
    if not 1 <= img.shape[0] <= MAX_IMAGES:
        raise ValueError(f"apply_multiview: {img.shape[0]} images per call (at most {MAX_IMAGES})")
    if not img.is_cuda:
        raise RuntimeError("apply_multiview: img must be a CUDA tensor")


def _photo_args(plan, cams):
    """The draws of the images `cams` as the C entry points take them -> (int32 [n, 8], float32 [n, 4]), or Nones."""
    if plan.photo is None:
        return None, None
    photo_i = np.zeros((len(cams), 8), np.int32)
    photo_f = np.zeros((len(cams), 4), np.float32)
    for k, c in enumerate(cams):
        d = plan.photo[c]
        photo_i[k] = (d.delta is not None, d.alpha is not None, d.sat is not None, d.hue is not None, d.mode == 1,
                      *(d.perm or (0, 1, 2)))
        photo_f[k] = [v if v is not None else 0.0 for v in (d.delta, d.alpha, d.sat, d.hue)]
    return photo_i, photo_f


def apply_multiview(img, results, cams=None):
    """Run the steps recorded in results['img_aug'] on img, uint8 [N, H, W, 3] BGR on a CUDA device -> float32
    [N, 3, Hp, Wp], on the current stream.  `cams`: which of the frame's images img holds (default all, in order),
    so a rank can process only its cameras with the frame's draws."""
    plan = results.get("img_aug") if isinstance(results, dict) else None
    cams = list(range(plan.n)) if cams is None and isinstance(plan, ImageAugPlan) else list(cams or [])
    _check(img, plan, cams)
    n, H, W = img.shape[:3]
    photo_i, photo_f = _photo_args(plan, cams)
    mean = np.ascontiguousarray(plan.mean, np.float32)
    stdinv = 1 / plan.std.astype(np.float64)
    pad_val = np.asarray(plan.pad_val, np.float32)
    hp, wp = plan.hw
    img = img.contiguous()
    dev = img.device

    def host(a):
        return None if a is None else a.ctypes.data

    with torch.cuda.device(dev):
        out = torch.empty((n, 3, hp, wp), dtype=torch.float32, device=dev)
        if plan.scale_hw is not None:
            _lib.check(_lib.lib().vidar_image_aug_scale(
                _lib.ptr(img), _lib.ptr(out), n, H, W, host(photo_i), host(photo_f), int(plan.to_rgb), host(mean),
                host(stdinv), host(pad_val), *plan.scale_hw, hp, wp, _lib.stream_ptr(dev)))
            return out
        if plan.crop is None:
            _lib.check(_lib.lib().vidar_image_aug_normalize(
                _lib.ptr(img), _lib.ptr(out), n, H, W, host(photo_i), host(photo_f), int(plan.to_rgb), host(mean),
                host(stdinv), host(pad_val), hp, wp, _lib.stream_ptr(dev)))
            return out
        x0, y0, x1, y1 = plan.crop
        ow, oh = plan.dims
        cw, ch = x1 - x0, y1 - y0
        wx0, wy0, wx1, wy1 = plan.window if plan.window is not None else (0, 0, ow, oh)
        htaps = _taps(cw, ow, dev) if ow != cw else None
        vtaps = _taps(ch, oh, dev) if oh != ch else None
        mid = torch.empty((n, ch, max(min(wx1, ow) - max(wx0, 0), 0), 3), dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().vidar_image_aug_apply(
            _lib.ptr(img), _lib.ptr(mid), _lib.ptr(out), n, H, W, host(photo_i), host(photo_f), x0, y0, cw, ch, ow,
            oh, wx0, wy0, wx1 - wx0, wy1 - wy0, _lib.ptr(htaps), htaps.shape[1] - 2 if htaps is not None else 0,
            _lib.ptr(vtaps), vtaps.shape[1] - 2 if vtaps is not None else 0, int(plan.flip), int(plan.to_rgb),
            host(mean), host(stdinv), host(pad_val), hp, wp, _lib.stream_ptr(dev)))
    return out


CONFIG_IMG_NORM = dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False)   # cfg :50-51


def config_pipeline(ida_aug_conf=None):
    """The four transforms of the pre-training config (vidar_1_8_nusc_3future.py:41-51, 303-314)."""
    conf = ida_aug_conf if ida_aug_conf is not None else dict(
        reisze=[720, 765, 810, 855, 900, 945, 990, 1035, 1080], crop=(0, 0, 1600, 900), H=900, W=1600, rand_flip=True)
    return [PhotoMetricDistortionMultiViewImage(),
            CropResizeFlipImage(data_aug_conf=conf, training=True, debug=False),
            NormalizeMultiviewImage(**CONFIG_IMG_NORM),
            PadMultiViewImage(size_divisor=32)]


def config_test_pipeline():
    """The image transforms of the pre-training config's test_pipeline (vidar_1_8_nusc_3future.py:319-328), after
    LoadMultiViewImageFromFiles: normalisation with the config's img_norm_cfg, then padding to multiples of 32.  No
    draw, no crop or resize: `lidar2img` passes through as the dataset gives it, and `img_shape` is the padded shape."""
    return [NormalizeMultiviewImage(**CONFIG_IMG_NORM), PadMultiViewImage(size_divisor=32)]


def config_openscene_pipeline():
    """The image transforms of the OpenScene configs' train_pipeline (vidar_OpenScene_*_3future.py:297-303), after
    LoadMultiViewImageFromFiles: photometric distortion, normalisation, the rescale by 2/3 and padding to multiples of
    32 -- 1920 x 1080 cameras become 1280 x 720, padded to 1280 x 736.  No crop: `lidar2img` is the dataset's,
    scaled."""
    return [PhotoMetricDistortionMultiViewImage(), NormalizeMultiviewImage(**CONFIG_IMG_NORM),
            RandomScaleImageMultiViewImage(scales=[2 / 3]), PadMultiViewImage(size_divisor=32)]


def config_openscene_test_pipeline():
    """The image transforms of the OpenScene configs' test_pipeline (vidar_OpenScene_*_3future.py:309-311):
    normalisation, the rescale by 2/3 (its one permutation draw per frame) and padding to multiples of 32."""
    return [NormalizeMultiviewImage(**CONFIG_IMG_NORM), RandomScaleImageMultiViewImage(scales=[2 / 3]),
            PadMultiViewImage(size_divisor=32)]
