"""ViDAR's GridMask image augmentation (models/utils/grid_mask.py `GridMask`) on the H100: a drop-in module with the
reference's constructor, attributes, `set_prob` and numpy draws, whose mask never exists as a tensor.

The reference builds a (1.5 h, 1.5 w) float32 mask on the host with Python loops, rotates it through PIL, crops it,
uploads it with a blocking `.cuda()` and multiplies.  Here the same global-numpy draws, in the same order (`rand()`
for the prob gate -- also in eval mode --, `randint(2, h)`, `randint(d)` twice, `randint(rotate)`, and `rand(h, w)`
with `offset`), feed one kernel launch (csrc/grid_mask.cu, include/vidar_b200.h §ix) that evaluates the mask per
pixel, PIL's nearest rotation included, and writes `x * mask` (+ `offset * (1 - mask)`) in x's dtype (float32,
float16 or bfloat16): bit for bit what the reference's statements give.  No scratch and no host sync; with `offset`
the [h, w] field is drawn on the host as the reference draws it and uploaded from pinned memory without blocking.
The backward is the same launch on grad_out (d out / d x = mask); no mask is stored.  CUDA tensors only.
"""
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import Function, once_differentiable

from . import _lib

# dtype codes of vidar_grid_mask_apply (VIDAR_DTYPE_F32 / _F16 / _BF16 of include/vidar_b200.h)
DTYPE_CODES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
MAX_SIDE = 8192


@dataclass(frozen=True)
class GridDraw:
    """One call's draws: stripe period d, stripe length l, stripe starts, rotation angle (degrees) and, with
    `offset`, the reference's float64 [h, w] offset field."""
    d: int
    l: int  # noqa: E741  (the reference's name)
    st_h: int
    st_w: int
    r: int
    offset: np.ndarray = None


def _check(x):
    """Every argument check of the op, before any CUDA call; the device check comes last, so the others can be
    tested without a GPU."""
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"grid_mask: x must be a tensor (got {type(x).__name__})")
    if x.dim() != 4:
        raise ValueError(f"grid_mask: x must be 4-D [n, c, h, w] (got shape {tuple(x.shape)})")
    if x.dtype not in DTYPE_CODES:
        raise TypeError(f"grid_mask: x must be float32, float16 or bfloat16 (got {x.dtype})")
    h, w = x.shape[-2:]
    if not (3 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError(f"grid_mask: image size {h} x {w} is outside 3..{MAX_SIDE} x 1..{MAX_SIDE}")
    if x.shape[0] * x.shape[1] >= 2 ** 31:
        raise ValueError(f"grid_mask: n * c = {x.shape[0] * x.shape[1]} is too large")
    if not x.is_cuda:
        raise RuntimeError("grid_mask: x must be a CUDA tensor")


def grid_mask_apply(x, draw, use_h, use_w, mode, offset=None):
    """x [n, c, h, w] (contiguous CUDA) -> x * mask, or x * mask + offset * (1 - mask) with offset [h, w] in x's
    dtype on x's device; mask from `draw` as the reference makes it (`mode == 1` inverts it)."""
    n, c, h, w = x.shape
    out = torch.empty_like(x, memory_format=torch.contiguous_format)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().vidar_grid_mask_apply(
            _lib.ptr(x), _lib.ptr(offset), _lib.ptr(out), DTYPE_CODES[x.dtype], n, c, h, w, draw.d, draw.l,
            draw.st_h, draw.st_w, draw.r, int(bool(use_h)), int(bool(use_w)), int(mode == 1),
            _lib.stream_ptr(x.device)))
    return out


class GridMaskFunction(Function):
    """apply(x, draw, use_h, use_w, mode, offset): out = x * mask (+ offset * (1 - mask)); grad_x = grad_out * mask."""

    @staticmethod
    def forward(ctx, x, draw, use_h, use_w, mode, offset):
        ctx.args = (draw, use_h, use_w, mode)
        return grid_mask_apply(x.contiguous(), draw, use_h, use_w, mode, offset)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        return grid_mask_apply(grad_out.contiguous(), *ctx.args), None, None, None, None, None


class GridMask(nn.Module):
    """models/utils/grid_mask.py `GridMask`: forward(x [n, c, h, w]) -> x with the grid mask applied, or x itself
    when the prob gate fails or in eval mode.  Same constructor, attributes (`l` holds the last stripe length) and
    `set_prob` as the reference; `fp16_enable` is kept, and as in the reference it casts nothing."""

    def __init__(self, use_h, use_w, rotate=1, offset=False, ratio=0.5, mode=0, prob=1.):
        super().__init__()
        self.use_h = use_h
        self.use_w = use_w
        self.rotate = rotate
        self.offset = offset
        self.ratio = ratio
        self.mode = mode
        self.st_prob = prob
        self.prob = prob
        self.fp16_enable = False

    def set_prob(self, epoch, max_epoch):
        self.prob = self.st_prob * epoch / max_epoch

    def _gate(self, training=None):
        """The prob gate: one `rand()`, drawn in eval mode too, as in the reference -> True to mask."""
        training = self.training if training is None else training
        return not (np.random.rand() > self.prob or not training)

    def _draw(self, h, w):
        d = np.random.randint(2, h)
        self.l = min(max(int(d * self.ratio + 0.5), 1), d - 1)
        st_h = np.random.randint(d)
        st_w = np.random.randint(d)
        r = np.random.randint(self.rotate)
        offset = 2 * (np.random.rand(h, w) - 0.5) if self.offset else None
        return GridDraw(int(d), int(self.l), int(st_h), int(st_w), int(r), offset)

    def sample(self, h, w, training=None):
        """The reference's numpy draws of one forward on an h x w image, in its order -> GridDraw, or None when the
        prob gate fails or the module is not training (`training` overrides self.training)."""
        return self._draw(h, w) if self._gate(training) else None

    def masked(self, x, draw):
        """x [n, c, h, w] CUDA with the mask of `draw` (from `sample(h, w)`) applied; differentiable in x (not named
        `apply`, which nn.Module already defines)."""
        _check(x)
        offset = None
        if draw.offset is not None:       # cast on the host as the reference does, then an asynchronous upload
            offset = torch.from_numpy(draw.offset).to(x.dtype).pin_memory().to(x.device, non_blocking=True)
        return GridMaskFunction.apply(x, draw, self.use_h, self.use_w, self.mode, offset)

    def forward(self, x):
        if not self._gate():
            return x
        _check(x)
        return self.masked(x, self._draw(x.shape[-2], x.shape[-1]))
