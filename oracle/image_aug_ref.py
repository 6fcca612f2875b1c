"""The multi-view image pipeline of ViDAR's pre-training configs, restated for the tests:
PhotoMetricDistortionMultiViewImage -> CropResizeFlipImage -> NormalizeMultiviewImage -> PadMultiViewImage
(datasets/pipelines/transform_3d.py:7-185, augmentation.py:10-202), for one image and fixed draws.

Two forms:
  * closed form (numpy only, usable where neither PIL nor cv2 is installed): the float32 HSV formulas of
    cv2.cvtColor with an exact fmaf, the wrapping `np.uint8` cast, Pillow's antialiased bicubic resample as its
    22-bit fixed-point taps, mmcv's imnormalize and impad arithmetic;
  * statements form (`*_statements`): the reference's own cv2 / PIL / numpy calls on the same draws, the CPU
    baseline the closed form is checked against (needs cv2 and PIL).

A draw of the photometric step is any object with the attributes `delta`, `mode`, `alpha`, `sat`, `hue` and
`perm`: None where the step's gate was closed, else the drawn value (Python floats, `mode` 0 or 1, `perm` a
permutation of (0, 1, 2)).
"""
import numpy as np

F32 = np.float32
FLT_EPSILON = F32(np.finfo(np.float32).eps)
HSCALE = F32(6.0) / F32(360.0)                              # cv2's hscale = 6.f / hrange, in float32
SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])
PRECISION_BITS = 22                                         # Pillow's Resample.c for 8-bit images


# ---------------------------------------------------------------------------------------------------------------
# float32 arithmetic
# ---------------------------------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """C's fmaf(a, b, c) on float32 arrays: a*b + c rounded once.  a*b is exact in float64 (24 + 24 bits); the sum
    is made exact-or-odd in float64 (round to odd: an inexact sum gets an odd last bit, moved toward the error
    term), and a round-to-odd result with 53 >= 24 + 2 bits rounds to float32 exactly as the infinitely precise sum
    would."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                            # TwoSum: s + e == p + c exactly
    bits = np.atleast_1d(s).view(np.int64).copy()
    fix = np.atleast_1d((e != 0) & (bits & 1 == 0))
    away = np.atleast_1d((e > 0) == (s >= 0))                # the error points away from zero
    bits[fix] += np.where(away[fix], 1, -1)
    return bits.view(np.float64).reshape(np.shape(s)).astype(F32)


def bgr2hsv(img):
    """cv2.cvtColor(img, COLOR_BGR2HSV) of a float32 [..., 3] image: h in [0, 360], s, v."""
    img = np.asarray(img, F32)
    b, g, r = img[..., 0], img[..., 1], img[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    diff = v - np.minimum(np.minimum(r, g), b)
    s = diff / (np.abs(v) + FLT_EPSILON)
    d = F32(60.0) / (diff + FLT_EPSILON)
    h_r = fmaf(g - b, d, F32(0))
    h_r = np.where(h_r < 0, fmaf(g - b, d, F32(360)), h_r)
    h = np.where(v == r, h_r, np.where(v == g, fmaf(b - r, d, F32(120)), fmaf(r - g, d, F32(240))))
    return np.stack([h, s, v], -1).astype(F32)


def hsv2bgr(img):
    """cv2.cvtColor(img, COLOR_HSV2BGR) of a float32 [..., 3] image with h in degrees."""
    img = np.asarray(img, F32)
    h, s, v = img[..., 0] * HSCALE, img[..., 1], img[..., 2]
    while (h < 0).any():
        h = np.where(h < 0, h + F32(6), h)
    while (h >= 6).any():
        h = np.where(h >= 6, h - F32(6), h)
    sector = np.floor(h)
    h = h - sector
    bad = (sector < 0) | (sector >= 6)
    sector = np.where(bad, 0, sector).astype(np.int64)
    h = np.where(bad, F32(0), h)
    one = F32(1)
    tab = np.stack([v, v * (one - s), v * fmaf(-s, h, one), v * fmaf(-s, one - h, one)], -1)
    idx = SECTORS[sector]                                                   # [..., 3] indices into tab
    out = np.take_along_axis(tab, idx, -1)
    return np.where((s == 0)[..., None], v[..., None], out).astype(F32)


def photometric(img, draw):
    """PhotoMetricDistortionMultiViewImage's pixel math on a float32 [H, W, 3] BGR image for one image's draw."""
    x = np.array(img, F32)
    if draw.delta is not None:
        x = x + F32(draw.delta)
    if draw.mode == 1 and draw.alpha is not None:
        x = x * F32(draw.alpha)
    x = bgr2hsv(x)
    if draw.sat is not None:
        x[..., 1] = x[..., 1] * F32(draw.sat)
    if draw.hue is not None:
        h = x[..., 0] + F32(draw.hue)
        h = np.where(h > 360, h - F32(360), h)
        x[..., 0] = np.where(h < 0, h + F32(360), h)
    x = hsv2bgr(x)
    if draw.mode == 0 and draw.alpha is not None:
        x = x * F32(draw.alpha)
    if draw.perm is not None:
        x = x[..., list(draw.perm)]
    return x.astype(F32)


def to_uint8(x):
    """`np.uint8(x)` of a float32 array on x86-64: truncation toward zero, then the low 8 bits (wraps)."""
    return (np.trunc(np.asarray(x, F32)).astype(np.int64) & 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------
# Pillow's resample (Resample.c: precompute_coeffs, normalize_coeffs_8bpc, ImagingResample{Horizontal,Vertical}_8bpc)
# ---------------------------------------------------------------------------------------------------------------
def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def resample_taps(in_size, out_size):
    """Pillow's BICUBIC taps from in_size to out_size pixels -> (xmin [out] int32, count [out] int32,
    weights [out, ksize] int32 in 2^-22 units).  In float64 in Pillow's order of operations; the weights of an
    output pixel are normalised by their sequential sum."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64) - xmin
    ss = 1.0 / filterscale
    k = np.arange(ksize)
    w = _bicubic(((k[None] + xmin[:, None]) - center[:, None] + 0.5) * ss)
    w = np.where(k[None] < xmax[:, None], w, 0.0)
    ww = np.zeros(out_size)
    for j in range(ksize):                                   # sequential, as the C loop sums
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    scaled = w * (1 << PRECISION_BITS)
    kk = np.trunc(np.where(w < 0, -0.5 + scaled, 0.5 + scaled)).astype(np.int32)
    return xmin.astype(np.int32), xmax.astype(np.int32), kk


def _pass(img, taps, axis):
    """One 8-bit pass of Pillow along `axis` (1 horizontal, 0 vertical) of a uint8 [H, W, C] image."""
    xmin, cnt, kk = taps
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((len(xmin),) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for j in range(kk.shape[1]):
        idx = np.minimum(xmin + j, src.shape[0] - 1)
        wj = np.where(j < cnt, kk[:, j], 0).astype(np.int64)
        acc += src[idx] * wj.reshape((-1,) + (1,) * (src.ndim - 1))
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, out_w, out_h):
    """`Image.fromarray(img).resize((out_w, out_h))` of a uint8 [H, W, 3] image: a horizontal pass, then a vertical
    one, each only when its size changes."""
    h, w = img.shape[:2]
    if out_w != w:
        img = _pass(img, resample_taps(w, out_w), 1)
    if out_h != h:
        img = _pass(img, resample_taps(h, out_h), 0)
    return np.ascontiguousarray(img)


def crop(img, box):
    """PIL `Image.crop(box)` (left, upper, right, lower) of a [H, W, C] image, zero outside the image."""
    x0, y0, x1, y1 = box
    h, w = img.shape[:2]
    out = np.zeros((y1 - y0, x1 - x0) + img.shape[2:], img.dtype)
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, h), max(x0, 0), min(x1, w)
    if sy1 > sy0 and sx1 > sx0:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = img[sy0:sy1, sx0:sx1]
    return out


def crop_resize_flip(img_u8, box, dims, flip):
    """CropResizeFlipImage's pixels: crop, resize to dims = (w, h), FLIP_LEFT_RIGHT -> uint8 [h, w, 3]."""
    out = resize(crop(img_u8, box), *dims)
    return np.ascontiguousarray(out[:, ::-1]) if flip else out


def normalize(img, mean, std, to_rgb):
    """mmcv.imnormalize of a float32 [H, W, 3] image: optional BGR -> RGB, x - f32(mean), f32(double(y) / std)."""
    x = np.asarray(img, F32)
    if to_rgb:
        x = x[..., ::-1]
    stdinv = 1 / np.asarray(std, F32).astype(np.float64)
    y = x - np.asarray(mean, F32)
    return (y.astype(np.float64) * stdinv).astype(F32)


def pad_values(pad_val):
    """Per-channel fill of cv2.copyMakeBorder(value=pad_val) on 3 channels: a number fills channel 0 only."""
    if isinstance(pad_val, (tuple, list)):
        return tuple(float(v) for v in pad_val)
    return (float(pad_val), 0.0, 0.0)


def pad(img, shape, pad_val=0):
    """mmcv.impad(img, shape=shape, pad_val=pad_val): bottom / right padding of a float32 [H, W, 3] image."""
    out = np.empty(tuple(shape[:2]) + img.shape[2:], F32)
    out[...] = np.asarray(pad_values(pad_val), F32)
    out[:img.shape[0], :img.shape[1]] = img
    return out


def pad_shape(h, w, size=None, size_divisor=None):
    """(Hp, Wp) of PadMultiViewImage: `size` as given, or the next multiples of `size_divisor`."""
    if size is not None:
        return int(size[0]), int(size[1])
    return -(-h // size_divisor) * size_divisor, -(-w // size_divisor) * size_divisor


def pipeline(img_u8, draw, box, dims, flip, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False, shape=None, pad_val=0):
    """The four steps on one uint8 [H, W, 3] BGR image (draw None: no photometric step; shape None: no padding) ->
    float32 [Hp, Wp, 3]."""
    x = np.asarray(img_u8, F32)
    if draw is not None:
        x = photometric(x, draw)
    x = crop_resize_flip(to_uint8(x), box, dims, flip).astype(F32)
    x = normalize(x, mean, std, to_rgb)
    return x if shape is None else pad(x, shape, pad_val)


# ---------------------------------------------------------------------------------------------------------------
# statements form: the reference's cv2 / PIL / numpy calls (CPU baseline; needs cv2 and PIL)
# ---------------------------------------------------------------------------------------------------------------
def photometric_statements(img, draw):
    import cv2
    img = np.array(img, F32)
    if draw.delta is not None:
        img += draw.delta
    if draw.mode == 1 and draw.alpha is not None:
        img *= draw.alpha
    img = cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
    if draw.sat is not None:
        img[..., 1] *= draw.sat
    if draw.hue is not None:
        img[..., 0] += draw.hue
        img[..., 0][img[..., 0] > 360] -= 360
        img[..., 0][img[..., 0] < 0] += 360
    img = cv2.cvtColor(img, cv2.COLOR_HSV2BGR)
    if draw.mode == 0 and draw.alpha is not None:
        img *= draw.alpha
    if draw.perm is not None:
        img = img[..., np.asarray(draw.perm)]
    return img


def crop_resize_flip_statements(img, box, dims, flip):
    from PIL import Image
    im = Image.fromarray(np.uint8(img)).crop(box).resize(dims)
    if flip:
        im = im.transpose(method=Image.FLIP_LEFT_RIGHT)
    return np.array(im).astype(np.float32)


def normalize_statements(img, mean, std, to_rgb):
    import cv2
    img = img.copy().astype(np.float32)
    mean = np.float64(np.asarray(mean, F32).reshape(1, -1))
    stdinv = 1 / np.float64(np.asarray(std, F32).reshape(1, -1))
    if to_rgb:
        cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
    cv2.subtract(img, mean, img)
    cv2.multiply(img, stdinv, img)
    return img


def pad_statements(img, shape, pad_val=0):
    import cv2
    return cv2.copyMakeBorder(img, 0, shape[0] - img.shape[0], 0, shape[1] - img.shape[1], cv2.BORDER_CONSTANT,
                              value=pad_val)


def pipeline_statements(img_u8, draw, box, dims, flip, mean=(0, 0, 0), std=(1, 1, 1), to_rgb=False, shape=None,
                        pad_val=0):
    x = np.asarray(img_u8, F32)
    if draw is not None:
        x = photometric_statements(x, draw)
    x = normalize_statements(crop_resize_flip_statements(x, box, dims, flip), mean, std, to_rgb)
    return x if shape is None else pad_statements(x, shape, pad_val)
