"""Modulated deformable convolution (DCNv2) on the H100: mmcv's `modulated_deform_conv2d`,
`ModulatedDeformConv2d` and `ModulatedDeformConv2dPack` (registered as `DCNv2`), with the same signatures, constructor
kwargs and parameter names, so the reference's ResNet-101 `dcn=dict(type='DCNv2', deform_groups=1)` layers build from
the unchanged config and an mmcv state_dict loads.

Path (csrc/dcn.cu + csrc/linear_tc.cu):
  forward   the input in channel-last layout; `vidar_dcn_im2col` writes the modulated bilinear samples as columns
            cols [n*Ho*Wo, kh*kw*Cin] (channels fastest); y = cols @ W'^T (+ bias) with W' = weight permuted to
            [Cout, kh, kw, Cin], on the tensor cores (3xTF32 wgmma) when kh*kw*Cin and Cout are multiples of 128
            and kh*kw*Cin <= TC_MAX_K, else the fp32 cuBLAS GEMM.  The output [n*Ho*Wo, Cout] is returned as a channels_last
            [N, Cout, Ho, Wo] view, no copy.
  backward  per chunk of images the columns are recomputed, grad_W' += g^T @ cols (fp32 cuBLAS), then the same buffer
            receives grad_cols = g @ W' (3xTF32 when the shape allows and Cout <= TC_MAX_K) and `vidar_dcn_col2im` turns it into grad_input
            (red.global.add to the four corners), grad_offset and grad_mask (warp sums over the channels).
Columns are computed for chunks of whole images of at most MAX_COLS_BYTES (512 MiB; one image when a single image's
columns are larger), so the scratch does not grow with the batch.  At the reference's 6 x 928 x 1600 input a stage-3
layer's columns are 6 x 5800 x 2304 floats (321 MB) and a stage-4 layer's 160 MB: one chunk each.

Mixed precision (mmcv 1.4.0's amp rule, see ModulatedDeformConv2dFunction): the op computes in the dtype of `offset`,
float32, float16 or bfloat16.  In 16 bits x, offset, mask and the columns are stored in that dtype, the sampling
arithmetic is fp32, and the GEMMs run on cuBLAS in that dtype with fp32 accumulation; the 3xTF32 GEMM is fp32 only.

Only groups == 1 and deform_groups == 1 (every reference config) and CUDA tensors of those three dtypes are supported;
anything else raises, there is no CPU fallback.
"""
import math

import torch
import torch.nn as nn
from torch.amp import custom_bwd, custom_fwd
from torch.autograd.function import Function, once_differentiable
from torch.nn.modules.utils import _pair

from . import _lib
from . import linear as _tc
from .registry import CONV_LAYERS

MAX_COLS_BYTES = 512 << 20
# Longest contraction given to the 3xTF32 GEMM, so the backbone's forwards (K = 2304 / 4608) run on fp32 cuBLAS and the
# tensor cores take grad_cols (K = Cout = 256 / 512).  The limit once fenced off an accumulation error that grew with K
# (6x / 20x torchvision's fp32 error at those forwards); the GEMM now holds fp32 cuBLAS's accuracy at any K
# (tests/test_linear_tc_gpu.py), and whether those forwards are faster on the tensor cores has not been measured.
TC_MAX_K = 1024


def _check_groups(groups, deform_groups):
    if groups != 1 or deform_groups != 1:
        raise ValueError(f"modulated_deform_conv2d supports groups == 1 and deform_groups == 1 only "
                         f"(got groups={groups}, deform_groups={deform_groups})")


def chunk_images(N, per_image_elems, elem_size=4):
    """Images per column chunk: as many as fit in MAX_COLS_BYTES, at least one (`elem_size` bytes per element)."""
    return max(1, min(N, MAX_COLS_BYTES // max(1, elem_size * per_image_elems)))


# dtype codes of vidar_dcn_im2col_half / vidar_dcn_col2im_half (VIDAR_DTYPE_F16 / _BF16 of include/vidar_b200.h)
HALF_DTYPE_CODES = {torch.float16: 1, torch.bfloat16: 2}
_COMPUTE_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def compute_dtype(input, offset, mask, weight, bias=None):
    """The dtype the op computes in, from the dtypes of its five tensors (None for no bias): mmcv's amp rule, the
    dtype of `offset`.  Every tensor must be float32, float16 or bfloat16 (the others are cast to the result);
    anything else raises TypeError."""
    for name, dt in (("input", input), ("offset", offset), ("mask", mask), ("weight", weight), ("bias", bias)):
        if dt is not None and dt not in _COMPUTE_DTYPES:
            raise TypeError(f"modulated_deform_conv2d: {name} must be float32, float16 or bfloat16 (got {dt})")
    return offset


def _gemm(a, w, bias, out, scratch):
    """out [M, Nout] = a [M, K] @ w[Nout, K]^T (+ bias): 3xTF32 wgmma when `scratch` is given, else fp32 cuBLAS."""
    M, K = a.shape
    if scratch is not None:
        _lib.check(_lib.lib().vidar_linear_tf32x3(_lib.ptr(a), _lib.ptr(w), _lib.ptr(bias), _lib.ptr(out),
                                                  _lib.ptr(scratch), M, w.shape[0], K, _lib.stream_ptr(a.device)))
    elif bias is not None:
        torch.addmm(bias, a, w.t(), out=out)
    else:
        torch.mm(a, w.t(), out=out)


def _geometry(x, weight, stride, padding, dilation):
    N, C, H, W = x.shape
    kh, kw = weight.shape[-2:]
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    return (N, C, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw)


class ModulatedDeformConv2dFunction(Function):
    """mmcv.ops.ModulatedDeformConv2dFunction: forward(input, offset, mask, weight, bias=None, stride=1, padding=0,
    dilation=1, groups=1, deform_groups=1).

    Dtypes, restated from mmcv 1.4.0's published `ModulatedDeformConv2dFunction.forward` (its source is not part of
    this project, and this rule has not been run against it): the op computes in cd = offset.dtype, and input, mask,
    weight and bias are cast to cd.  Under autocast the offset conv emits the autocast dtype, so the op runs in it;
    mmcv's fp16 mode (`Fp16OptimizerHook` + `auto_fp16`) is autocast on torch >= 1.6.
      cd = float32             the fp32 path (3xTF32 / fp32 cuBLAS GEMMs), unchanged by this rule.
      cd = float16, bfloat16   x, offset, mask and the columns in cd, sampling arithmetic in fp32 (csrc/dcn.cu, each
                               column element rounded once); y = cols @ W'^T (+ bias) and grad_cols = g @ W' on cuBLAS
                               in cd with fp32 accumulation (the user's allow_fp16/bf16_reduced_precision_reduction
                               settings apply); grad_W' per chunk by `torch.mm(..., out_dtype=torch.float32)`, summed
                               over chunks in fp32; grad_x, grad_offset and grad_mask from col2im in fp32.
      anything else            TypeError (`compute_dtype`).
    The output has dtype cd; each gradient is cast once to its leaf's dtype (an fp32 weight gets an fp32 grad_weight).
    The GEMMs run with autocast disabled, so their dtypes do not depend on the autocast state around the call."""

    @staticmethod
    @custom_fwd(device_type="cuda")
    def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1, deform_groups=1):
        _check_groups(groups, deform_groups)
        for name, t in (("input", input), ("offset", offset), ("mask", mask), ("weight", weight), ("bias", bias)):
            if t is not None and not t.is_cuda:
                raise RuntimeError(f"{name} must be a CUDA tensor")
        cd = compute_dtype(input.dtype, offset.dtype, mask.dtype, weight.dtype, bias.dtype if bias is not None else None)
        ctx.leaf_dtypes = tuple(t.dtype if t is not None else None for t in (input, offset, mask, weight, bias))
        input, mask, weight = input.to(cd), mask.to(cd), weight.to(cd)
        bias = bias.to(cd) if bias is not None else None
        geom = _geometry(input, weight, stride, padding, dilation)
        N, C, H, W, Ho, Wo, kh, kw = geom[:8]
        Cout = weight.shape[0]
        if weight.shape[1] != C:
            raise ValueError(f"modulated_deform_conv2d: weight {tuple(weight.shape)} does not match {C} input channels")
        if Ho <= 0 or Wo <= 0:
            raise ValueError(f"modulated_deform_conv2d: empty output ({Ho} x {Wo}) for input {tuple(input.shape)}")
        K = kh * kw
        if tuple(offset.shape) != (N, 2 * K, Ho, Wo) or tuple(mask.shape) != (N, K, Ho, Wo):
            raise ValueError(f"modulated_deform_conv2d: offset {tuple(offset.shape)} / mask {tuple(mask.shape)} must be "
                             f"{(N, 2 * K, Ho, Wo)} / {(N, K, Ho, Wo)}")
        x = _lib.aligned(input.detach().permute(0, 2, 3, 1).contiguous())        # NHWC; free for channels_last input
        off = _lib.aligned(offset.detach().contiguous())
        msk = _lib.aligned(mask.detach().contiguous())
        w2 = weight.detach().permute(0, 2, 3, 1).reshape(Cout, K * C).contiguous()
        b = bias.detach().contiguous() if bias is not None else None
        ctx.geom, ctx.with_bias = geom, bias is not None
        ctx.save_for_backward(x, off, msk, w2)
        y = torch.empty((N * Ho * Wo, Cout), dtype=cd, device=input.device)
        if N:
            scratch = _split_scratch(w2)
            with torch.autocast("cuda", enabled=False):
                _columns_pass(x, off, msk, geom, lambda cols, rows, n0, nb: _gemm(cols, w2, b, y[rows], scratch))
        return y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2)                       # channels_last strides

    @staticmethod
    @custom_bwd(device_type="cuda")
    @once_differentiable
    def backward(ctx, grad_output):
        with torch.autocast("cuda", enabled=False):
            grads = _backward(ctx, grad_output)
        return tuple(g.to(dt) if g is not None else None for g, dt in zip(grads, ctx.leaf_dtypes)) + (None,) * 5


def _backward(ctx, grad_output):
    """(grad_input, grad_offset, grad_mask, grad_weight, grad_bias), each None where not needed: in fp32 for
    cd = float32; for 16 bits grad_bias and grad_weight are fp32 sums and the sampling gradients come from col2im in
    fp32."""
    x, off, msk, w2 = ctx.saved_tensors
    N, C, H, W, Ho, Wo, kh, kw = ctx.geom[:8]
    Cout, Kc = w2.shape
    half = w2.dtype != torch.float32
    need_x, need_off, need_mask, need_w = ctx.needs_input_grad[:4]
    g = _lib.aligned(grad_output.to(w2.dtype).permute(0, 2, 3, 1).contiguous().view(N * Ho * Wo, Cout))
    gb = None
    if ctx.with_bias and ctx.needs_input_grad[4]:
        gb = g.sum(0, dtype=torch.float32) if half else g.sum(0)
    gw = torch.zeros_like(w2, dtype=torch.float32) if need_w else None
    gx = go = gm = None
    if need_x or need_off or need_mask:
        gx = torch.zeros_like(x, dtype=torch.float32)
        go = torch.empty_like(off, dtype=torch.float32)
        gm = torch.empty_like(msk, dtype=torch.float32)
    if N and (need_w or gx is not None):
        wt = w2 if half else w2.t().contiguous()                                  # fp32: [Kc, Cout], grad_cols = g @ W'
        scratch = None if half else _split_scratch(wt)
        stream = _lib.stream_ptr(x.device)

        def chunk(cols, rows, n0, nb):
            gc = g[rows]
            if gw is not None:
                if half:
                    gw.add_(torch.mm(gc.t(), cols, out_dtype=torch.float32))          # cuBLAS, fp32 out
                else:
                    gw.addmm_(gc.t(), cols)                                           # fp32 cuBLAS
            if gx is not None:
                if half:
                    torch.mm(gc, wt, out=cols)                                        # grad_cols, in place of cols
                else:
                    _gemm(gc, wt, None, cols, scratch)
                _col2im(x, off, msk, cols, gx, go, gm, ctx.geom, n0, nb, stream)

        _columns_pass(x, off, msk, ctx.geom, chunk, recompute=need_w)
    gw = gw.view(Cout, kh, kw, C).permute(0, 3, 1, 2).contiguous() if gw is not None else None
    gx = gx.permute(0, 3, 1, 2) if need_x else None
    return gx, go if need_off else None, gm if need_mask else None, gw, gb


def _split_scratch(w):
    """Split-weight scratch of the 3xTF32 GEMM for weight `w` [Nout, K], or None when the GEMM runs on cuBLAS: 16-bit
    weights, shapes the kernel does not take, and contractions longer than TC_MAX_K."""
    Nout, K = w.shape
    if w.dtype != torch.float32 or not _tc.supported(K, Nout) or K > TC_MAX_K or torch.is_autocast_enabled():
        return None
    return torch.empty(2 * Nout * K, dtype=torch.float32, device=w.device)


def _columns_pass(x, off, msk, geom, fn, recompute=True):
    """Calls fn(cols [nb*Ho*Wo, kh*kw*C], rows, n0, nb) for each chunk of nb images, with the columns of the
    chunk written by vidar_dcn_im2col when `recompute` (else the buffer holds garbage for fn to overwrite)."""
    N, C, H, W, Ho, Wo, kh, kw = geom[:8]
    per_image = Ho * Wo * kh * kw * C
    nb = chunk_images(N, per_image, x.element_size())
    buf = torch.empty(nb * per_image, dtype=x.dtype, device=x.device)
    stream = _lib.stream_ptr(x.device)
    with torch.cuda.device(x.device):
        for n0 in range(0, N, nb):
            b = min(nb, N - n0)
            cols = buf[: b * per_image].view(b * Ho * Wo, kh * kw * C)
            if recompute:
                _im2col(x, off, msk, cols, geom, n0, b, stream)
            rows = slice(n0 * Ho * Wo, (n0 + b) * Ho * Wo)
            fn(cols, rows, n0, b)


def _im2col(x, off, msk, cols, geom, n0, nb, stream):
    L = _lib.lib()
    if x.dtype == torch.float32:
        rc = L.vidar_dcn_im2col(_lib.ptr(x), _lib.ptr(off), _lib.ptr(msk), _lib.ptr(cols), *geom, n0, nb, stream)
    else:
        rc = L.vidar_dcn_im2col_half(_lib.ptr(x), _lib.ptr(off), _lib.ptr(msk), _lib.ptr(cols),
                                     HALF_DTYPE_CODES[x.dtype], *geom, n0, nb, stream)
    _lib.check(rc)


def _col2im(x, off, msk, grad_cols, gx, go, gm, geom, n0, nb, stream):
    L = _lib.lib()
    ptrs = [_lib.ptr(t) for t in (x, off, msk, grad_cols, gx, go, gm)]
    if x.dtype == torch.float32:
        rc = L.vidar_dcn_col2im(*ptrs, *geom, n0, nb, stream)
    else:
        rc = L.vidar_dcn_col2im_half(*ptrs, HALF_DTYPE_CODES[x.dtype], *geom, n0, nb, stream)
    _lib.check(rc)


def modulated_deform_conv2d(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                            deform_groups=1):
    """mmcv.ops.modulated_deform_conv2d (= ModulatedDeformConv2dFunction.apply)."""
    return ModulatedDeformConv2dFunction.apply(input, offset, mask, weight, bias, stride, padding, dilation, groups,
                                               deform_groups)


class ModulatedDeformConv2d(nn.Module):
    """mmcv.ops.ModulatedDeformConv2d: parameters `weight` [out, in // groups, kh, kw] and `bias` [out] (or None).

    Init as restated from mmcv 1.4.0's published code (its source is not part of this project):
    weight ~ uniform(+-1/sqrt(in_channels * kh * kw)), bias = 0."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deform_groups=1, bias=True, deformable_groups=None):
        super().__init__()
        if deformable_groups is not None:            # the name mmcv deprecated in favour of deform_groups
            deform_groups = deformable_groups
        _check_groups(groups, deform_groups)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = _pair(stride), _pair(padding), _pair(dilation)
        self.groups, self.deform_groups = groups, deform_groups
        self.transposed, self.output_padding = False, (0,)
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self.init_weights()

    def init_weights(self):
        stdv = 1.0 / math.sqrt(self.in_channels * self.kernel_size[0] * self.kernel_size[1])
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.zero_()

    def forward(self, x, offset, mask):
        return modulated_deform_conv2d(x, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                       self.groups, self.deform_groups)


@CONV_LAYERS.register_module("DCNv2")
class ModulatedDeformConv2dPack(ModulatedDeformConv2d):
    """mmcv.ops.ModulatedDeformConv2dPack (registry name DCNv2): offsets and mask from `conv_offset`, a Conv2d with
    deform_groups * 3 * kh * kw outputs and the layer's kernel / stride / padding / dilation, zero at init.
    out = conv_offset(x); offset = cat(chunk(out, 3)[:2]) = out[:, :2*kh*kw]; mask = sigmoid(out[:, 2*kh*kw:])."""

    _version = 2

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deform_groups * 3 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=self.stride, padding=self.padding,
                                     dilation=self.dilation, bias=True)
        self.init_weights()

    def init_weights(self):
        super().init_weights()
        if hasattr(self, "conv_offset"):
            self.conv_offset.weight.data.zero_()
            self.conv_offset.bias.data.zero_()

    def forward(self, x):
        out = self.conv_offset(x)
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        return modulated_deform_conv2d(x, offset, torch.sigmoid(mask), self.weight, self.bias, self.stride, self.padding,
                                       self.dilation, self.groups, self.deform_groups)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        version = local_metadata.get("version", None)
        if version is None or version < 2:
            # checkpoints of mmcv's version 1 of this module name the offset conv `conv_offset_mask`
            for suffix in ("weight", "bias"):
                old, new = prefix + "conv_offset_mask." + suffix, prefix + "conv_offset." + suffix
                if new not in state_dict and old in state_dict:
                    state_dict[new] = state_dict.pop(old)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)
