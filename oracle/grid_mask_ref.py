"""GridMask's mask (models/utils/grid_mask.py GridMask.forward) restated in numpy, for the tests.

The reference writes stripes into an (int(1.5 h), int(1.5 w)) frame of ones, rotates it with PIL's
`Image.rotate(r)` (nearest, no expand, fill 0) and crops the centre.  Here the rotation is Pillow's nearest affine
transform in closed form: the inverse rotation about the frame's centre, entries rounded to 15 decimals, as 16.16
fixed point with the half-pixel centre folded into the translation; output pixel (Y, X) reads input pixel
  xin = (a2 + Y*a1 + X*a0) >> 16,   yin = (a5 + Y*a4 + X*a3) >> 16      (0 outside the input).
The stripes are tested at (yin, xin) instead of being written, so no (1.5 h, 1.5 w) array is needed either.
"""
import math

import numpy as np


def pillow_rotation(angle, height, width):
    """(a0, a1, a2, a3, a4, a5) of Pillow's `Image.rotate(angle)` on a height x width image."""
    a = -math.radians(angle % 360)
    m = [round(math.cos(a), 15), round(math.sin(a), 15), 0.0, round(-math.sin(a), 15), round(math.cos(a), 15), 0.0]
    cx, cy = width / 2, height / 2
    m[2] = m[0] * -cx + m[1] * -cy + 0.0 + cx
    m[5] = m[3] * -cx + m[4] * -cy + 0.0 + cy

    def fix(v):
        return math.floor(v * 65536.0 + 0.5)
    return (fix(m[0]), fix(m[1]), fix(m[2] + m[0] * 0.5 + m[1] * 0.5), fix(m[3]), fix(m[4]),
            fix(m[5] + m[3] * 0.5 + m[4] * 0.5))


def source_pixels(angle, height, width, ys, xs):
    """Input pixel (yin, xin) that output pixels (ys, xs) of the rotation read, as int64 arrays."""
    a0, a1, a2, a3, a4, a5 = pillow_rotation(angle, height, width)
    ys, xs = np.asarray(ys, np.int64), np.asarray(xs, np.int64)
    return (a5 + ys * a4 + xs * a3) >> 16, (a2 + ys * a1 + xs * a0) >> 16


def rotate_nearest(img, angle):
    """`np.asarray(Image.fromarray(img).rotate(angle))` for a 2-D uint8 array, in closed form."""
    H, W = img.shape
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    yin, xin = source_pixels(angle, H, W, ys, xs)
    inside = (xin >= 0) & (xin < W) & (yin >= 0) & (yin < H)
    out = np.zeros_like(img)
    out[inside] = img[yin[inside], xin[inside]]
    return out


def on_stripe(i, start, d, l, n):
    """Row (or column) i lies on one of the reference's n stripes [d*k + start, d*k + start + l)."""
    r = i - start
    return (r >= 0) & (r // d < n) & (r % d < l)


def grid_mask(h, w, d, l, st_h, st_w, r, use_h, use_w, mode):
    """The reference's [h, w] mask as float32 0 / 1 (after `1 - mask` when mode == 1)."""
    hh, ww = int(1.5 * h), int(1.5 * w)
    ys, xs = np.meshgrid(np.arange(h) + (hh - h) // 2, np.arange(w) + (ww - w) // 2, indexing="ij")
    yin, xin = source_pixels(r, hh, ww, ys, xs)
    inside = (xin >= 0) & (xin < ww) & (yin >= 0) & (yin < hh)
    stripe = np.zeros((h, w), bool)
    if use_h:
        stripe |= on_stripe(yin, st_h, d, l, hh // d)
    if use_w:
        stripe |= on_stripe(xin, st_w, d, l, ww // d)
    mask = (inside & ~stripe).astype(np.float32)
    return 1 - mask if mode == 1 else mask


def pil_mask(h, w, d, l, st_h, st_w, r, use_h, use_w, mode):
    """The same mask made the reference's way, for comparison and timing: the stripes written into a float32
    (1.5 h, 1.5 w) frame of ones row block by row block, then uint8, PIL's rotate and the centre crop."""
    from PIL import Image
    hh, ww = int(1.5 * h), int(1.5 * w)
    frame = np.ones((hh, ww), np.float32)
    for k in range(hh // d if use_h else 0):
        frame[d * k + st_h:min(d * k + st_h + l, hh), :] *= 0
    for k in range(ww // d if use_w else 0):
        frame[:, d * k + st_w:min(d * k + st_w + l, ww)] *= 0
    rotated = np.asarray(Image.fromarray(np.uint8(frame)).rotate(r))
    mask = rotated[(hh - h) // 2:(hh - h) // 2 + h, (ww - w) // 2:(ww - w) // 2 + w].astype(np.float32)
    return 1 - mask if mode == 1 else mask


def apply(x, mask, offset=None):
    """The reference's statements on a CPU tensor x [N, C, h, w]: x * mask, or x * mask + offset * (1 - mask), in
    x's dtype; mask [h, w] (numpy 0 / 1), offset [h, w] (float64 numpy, cast to x's dtype as the reference does)."""
    import torch
    m = torch.from_numpy(np.ascontiguousarray(mask)).to(x.dtype).expand_as(x)
    if offset is None:
        return x * m
    o = torch.from_numpy(offset).to(x.dtype)
    return x * m + o * (1 - m)
