"""InternImage's deformable convolution v3 (DCNv3) on the H100: a drop-in for the compiled `DCNv3` extension of
`ops_dcnv3` (`ext`, so `import DCNv3` becomes `from vidar_b200.dcnv3 import ext as DCNv3`), its `DCNv3Function`, and
the `DCNv3` module with the same constructor kwargs and parameter names, so InternImage checkpoints load.

The op (csrc/dcnv3.cu, include/vidar_b200.h §viii): for every output pixel and group, K = kernel_h*kernel_w
bilinear samples of the channel-last input at the offset kernel grid, weighted by the (softmaxed) mask.  Input,
offset and mask share one dtype, float32, float16 or bfloat16; all arithmetic is fp32, the output is rounded once,
and the gradients come back in that dtype (grad_input is summed in fp32 and cast once).  One kernel launch per
forward and one per backward, on the current stream, with no host sync.  CUDA tensors only: there is no CPU path.
"""
import types
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.amp import custom_bwd, custom_fwd
from torch.autograd.function import Function, once_differentiable

from . import _lib

# dtype codes of vidar_dcnv3_forward / _backward (VIDAR_DTYPE_F32 / _F16 / _BF16 of include/vidar_b200.h)
DTYPE_CODES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def output_size(H, W, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w):
    Ho = (H + 2 * pad_h - (dilation_h * (kernel_h - 1) + 1)) // stride_h + 1
    Wo = (W + 2 * pad_w - (dilation_w * (kernel_w - 1) + 1)) // stride_w + 1
    return Ho, Wo


def _check(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group,
           group_channels, im2col_step, grad_output=None):
    """Every argument check of the op, before any CUDA call; the device check comes last, so the others can be
    tested without a GPU.  Returns (N, H, W, Ho, Wo)."""
    tensors = (("input", input), ("offset", offset), ("mask", mask), ("grad_output", grad_output))
    tensors = tuple((n, t) for n, t in tensors if t is not None)
    for name, t in tensors:
        if t.dtype not in DTYPE_CODES:
            raise TypeError(f"dcnv3: {name} must be float32, float16 or bfloat16 (got {t.dtype})")
        if t.dtype != input.dtype:
            raise TypeError(f"dcnv3: {name} is {t.dtype} but input is {input.dtype}; they must share one dtype")
        if t.dim() != 4:
            raise RuntimeError(f"dcnv3: {name} must be 4-D (got shape {tuple(t.shape)})")
    sizes = (kernel_h, kernel_w, stride_h, stride_w, dilation_h, dilation_w, group, group_channels)
    if min(sizes) <= 0 or pad_h < 0 or pad_w < 0:
        raise RuntimeError(f"dcnv3: kernel, stride, dilation, group and group_channels must be positive and the "
                           f"padding non-negative (got kernel {kernel_h}x{kernel_w}, stride {stride_h}x{stride_w}, "
                           f"pad {pad_h}x{pad_w}, dilation {dilation_h}x{dilation_w}, group {group}, "
                           f"group_channels {group_channels})")
    N, H, W, C = input.shape
    if C != group * group_channels:
        raise RuntimeError(f"dcnv3: input channels and group times group channels do not match: "
                           f"({C} vs {group * group_channels})")
    Ho, Wo = output_size(H, W, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w)
    if N <= 0 or H <= 0 or W <= 0 or Ho <= 0 or Wo <= 0:
        raise RuntimeError(f"dcnv3: empty input or output (input {tuple(input.shape)}, output {Ho} x {Wo})")
    K = kernel_h * kernel_w
    want = {"offset": (N, Ho, Wo, group * K * 2), "mask": (N, Ho, Wo, group * K), "grad_output": (N, Ho, Wo, C)}
    for name, t in tensors[1:]:
        if tuple(t.shape) != want[name]:
            raise RuntimeError(f"dcnv3: {name} must be {want[name]} (got {tuple(t.shape)})")
    if im2col_step <= 0 or N % min(N, im2col_step):
        raise RuntimeError(f"dcnv3: batch({N}) must divide im2col_step({min(N, im2col_step)})")
    for name, t in tensors:
        if not t.is_contiguous():
            raise RuntimeError(f"dcnv3: {name} tensor has to be contiguous")
    for name, t in tensors:
        if not t.is_cuda:
            raise RuntimeError(f"dcnv3: {name} must be a CUDA tensor")
    return N, H, W, Ho, Wo


def dcnv3_forward(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
                  group, group_channels, offset_scale, im2col_step):
    """`DCNv3.dcnv3_forward` -> output [N, Ho, Wo, group*group_channels] in input's dtype."""
    N, H, W, Ho, Wo = _check(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h,
                             dilation_w, group, group_channels, im2col_step)
    out = torch.empty((N, Ho, Wo, group * group_channels), dtype=input.dtype, device=input.device)
    with torch.cuda.device(input.device):
        _lib.check(_lib.lib().vidar_dcnv3_forward(
            _lib.ptr(input), _lib.ptr(offset), _lib.ptr(mask), _lib.ptr(out), DTYPE_CODES[input.dtype], N, H, W,
            group, group_channels, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
            float(offset_scale), int(im2col_step), _lib.stream_ptr(input.device)))
    return out


def dcnv3_backward(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
                   group, group_channels, offset_scale, grad_output, im2col_step):
    """`DCNv3.dcnv3_backward` -> [grad_input, grad_offset, grad_mask] in input's dtype (grad_input summed in fp32)."""
    N, H, W, Ho, Wo = _check(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h,
                             dilation_w, group, group_channels, im2col_step, grad_output)
    grad_input = torch.zeros(input.shape, dtype=torch.float32, device=input.device)
    grad_offset = torch.empty_like(offset)
    grad_mask = torch.empty_like(mask)
    with torch.cuda.device(input.device):
        _lib.check(_lib.lib().vidar_dcnv3_backward(
            _lib.ptr(input), _lib.ptr(offset), _lib.ptr(mask), _lib.ptr(grad_output), _lib.ptr(grad_input),
            _lib.ptr(grad_offset), _lib.ptr(grad_mask), DTYPE_CODES[input.dtype], N, H, W, group, group_channels,
            kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, float(offset_scale),
            int(im2col_step), _lib.stream_ptr(input.device)))
    return [grad_input.to(input.dtype), grad_offset, grad_mask]


# Stand-in for the compiled extension module `DCNv3` of ops_dcnv3.
ext = types.SimpleNamespace(dcnv3_forward=dcnv3_forward, dcnv3_backward=dcnv3_backward)


class DCNv3Function(Function):
    """ops_dcnv3's DCNv3Function: apply(input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
    dilation_h, dilation_w, group, group_channels, offset_scale, im2col_step).  custom_fwd without a cast, as in the
    reference: the op runs in the dtype its tensors have."""

    @staticmethod
    @custom_fwd(device_type="cuda")
    def forward(ctx, input, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w,
                group, group_channels, offset_scale, im2col_step):
        ctx.args = (kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group,
                    group_channels, offset_scale)
        ctx.im2col_step = im2col_step
        output = dcnv3_forward(input, offset, mask, *ctx.args, im2col_step)
        ctx.save_for_backward(input, offset, mask)
        return output

    @staticmethod
    @once_differentiable
    @custom_bwd(device_type="cuda")
    def backward(ctx, grad_output):
        input, offset, mask = ctx.saved_tensors
        grads = dcnv3_backward(input, offset, mask, *ctx.args, grad_output.contiguous(), ctx.im2col_step)
        return (*grads,) + (None,) * 12


class to_channels_first(nn.Module):
    def forward(self, x):
        return x.permute(0, 3, 1, 2)


class to_channels_last(nn.Module):
    def forward(self, x):
        return x.permute(0, 2, 3, 1)


def build_norm_layer(dim, norm_layer, in_format="channels_last", out_format="channels_last", eps=1e-6):
    """'BN' (BatchNorm2d, channels-first inside) or 'LN' (LayerNorm, channels-last inside) between the formats."""
    if norm_layer == "BN":
        layers = ([to_channels_first()] if in_format == "channels_last" else []) + [nn.BatchNorm2d(dim)]
        layers += [to_channels_last()] if out_format == "channels_last" else []
    elif norm_layer == "LN":
        layers = ([to_channels_last()] if in_format == "channels_first" else []) + [nn.LayerNorm(dim, eps=eps)]
        layers += [to_channels_first()] if out_format == "channels_first" else []
    else:
        raise NotImplementedError(f"build_norm_layer does not support {norm_layer}")
    return nn.Sequential(*layers)


def build_act_layer(act_layer):
    acts = {"ReLU": lambda: nn.ReLU(inplace=True), "SiLU": lambda: nn.SiLU(inplace=True), "GELU": nn.GELU}
    if act_layer not in acts:
        raise NotImplementedError(f"build_act_layer does not support {act_layer}")
    return acts[act_layer]()


class CenterFeatureScaleModule(nn.Module):
    def forward(self, query, center_feature_scale_proj_weight, center_feature_scale_proj_bias):
        return F.linear(query, weight=center_feature_scale_proj_weight, bias=center_feature_scale_proj_bias).sigmoid()


class DCNv3(nn.Module):
    """ops_dcnv3's DCNv3 module (InternImage's `core_op`): input and output [N, H, W, channels].

    x = input_proj(input); offsets and mask come from a depthwise conv + norm + activation of the input through the
    `offset` / `mask` Linears, the mask softmaxed over each group's K logits; the op samples x; with
    `center_feature_scale` the result is blended with x by sigmoid(Linear(features)) per group; then output_proj.
    Parameters: dw_conv.0 (depthwise conv), dw_conv.1.* (norm), offset, mask, input_proj, output_proj and, with
    center_feature_scale, center_feature_scale_proj_weight [group, channels] / _bias [group]."""

    def __init__(self, channels=64, kernel_size=3, dw_kernel_size=None, stride=1, pad=1, dilation=1, group=4,
                 offset_scale=1.0, act_layer="GELU", norm_layer="LN", center_feature_scale=False):
        super().__init__()
        if channels % group != 0:
            raise ValueError(f"channels must be divisible by group, but got {channels} and {group}")
        gc = channels // group
        if gc & (gc - 1):
            warnings.warn("DCNv3: channels // group is not a power of 2; the reference's CUDA op prefers one")
        dw_kernel_size = kernel_size if dw_kernel_size is None else dw_kernel_size
        self.offset_scale = offset_scale
        self.channels = channels
        self.kernel_size = kernel_size
        self.dw_kernel_size = dw_kernel_size
        self.stride = stride
        self.dilation = dilation
        self.pad = pad
        self.group = group
        self.group_channels = gc
        self.center_feature_scale = center_feature_scale
        self.dw_conv = nn.Sequential(
            nn.Conv2d(channels, channels, kernel_size=dw_kernel_size, stride=1, padding=(dw_kernel_size - 1) // 2,
                      groups=channels),
            build_norm_layer(channels, norm_layer, "channels_first", "channels_last"),
            build_act_layer(act_layer))
        K = kernel_size * kernel_size
        self.offset = nn.Linear(channels, group * K * 2)
        self.mask = nn.Linear(channels, group * K)
        self.input_proj = nn.Linear(channels, channels)
        self.output_proj = nn.Linear(channels, channels)
        self._reset_parameters()
        if center_feature_scale:
            self.center_feature_scale_proj_weight = nn.Parameter(torch.zeros((group, channels), dtype=torch.float))
            self.center_feature_scale_proj_bias = nn.Parameter(torch.zeros(group, dtype=torch.float))
            self.center_feature_scale_module = CenterFeatureScaleModule()

    def _reset_parameters(self):
        """Offsets and mask logits start at zero; the projections are Xavier-uniform with zero bias."""
        for lin in (self.offset, self.mask):
            nn.init.constant_(lin.weight, 0.0)
            nn.init.constant_(lin.bias, 0.0)
        for lin in (self.input_proj, self.output_proj):
            nn.init.xavier_uniform_(lin.weight)
            nn.init.constant_(lin.bias, 0.0)

    def forward(self, input):
        N, H, W, _ = input.shape
        x = self.input_proj(input)
        x_proj = x
        feat = self.dw_conv(input.permute(0, 3, 1, 2))
        offset = self.offset(feat)
        mask = F.softmax(self.mask(feat).reshape(N, H, W, self.group, -1), -1).reshape(N, H, W, -1).type(x.dtype)
        x = DCNv3Function.apply(x, offset, mask, self.kernel_size, self.kernel_size, self.stride, self.stride,
                                self.pad, self.pad, self.dilation, self.dilation, self.group, self.group_channels,
                                self.offset_scale, 256)
        if self.center_feature_scale:
            scale = self.center_feature_scale_module(feat, self.center_feature_scale_proj_weight,
                                                     self.center_feature_scale_proj_bias)
            scale = scale[..., None].repeat(1, 1, 1, 1, self.group_channels).flatten(-2)
            x = x * (1 - scale) + x_proj * scale
        return self.output_proj(x)
