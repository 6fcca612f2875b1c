"""nn.Linear on the H100 tensor cores with fp32 accuracy (3xTF32, csrc/linear_tc.cu).

The reference runs `value_proj` -- the one dense contraction on the hot path, 6 x 30825 x 256 -> 256 per
SpatialCrossAttention layer (spatial_cross_attention.py:333) -- as an fp32 cuBLAS GEMM.  `linear_tf32x3`
computes the same product with wgmma (TMA-fed, register accumulators) with every operand split into two TF32
parts, three MMAs per K step.  Accuracy is fp32's at every in_features the kernel takes (any multiple of 32 through the
C ABI): per output element, |y - y_fp64| / sum_k |x_k w_k| stays within 2x of fp32 cuBLAS's in max and RMS
(tests/test_linear_tc_gpu.py), far inside the 1e-4 parity bar that a plain TF32 GEMM (~5e-4) misses.
Non-finite inputs: a NaN in a row of x (a row of W) makes that output row (column) NaN and nothing else.  An inf in x
gives NaN where cuBLAS gives inf, because the split's low part is inf - inf.
Backward: grad_input through the same kernel (weight transposed); grad_weight / grad_bias are [N, K]-sized
reductions over all rows and stay on cuBLAS (fp32).
"""
import torch
from torch.autograd.function import Function, once_differentiable

from . import _lib


def supported(in_features, out_features, x=None):
    ok = in_features % 128 == 0 and out_features % 128 == 0      # both directions (forward and grad_input)
    if x is not None:
        ok = ok and x.is_cuda and x.dtype == torch.float32 and not torch.is_autocast_enabled()
    return ok


def _gemm(x2d, weight, bias):
    M, K = x2d.shape
    N = weight.shape[0]
    y = torch.empty((M, N), dtype=torch.float32, device=x2d.device)
    if M == 0:
        return y
    scratch = torch.empty(2 * N * K, dtype=torch.float32, device=x2d.device)
    with torch.cuda.device(x2d.device):
        _lib.check(_lib.lib().vidar_linear_tf32x3(_lib.ptr(x2d), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(y),
                                                  _lib.ptr(scratch), M, N, K, _lib.stream_ptr(x2d.device)))
    return y


class _LinearTF32x3(Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        x2d = _lib.aligned(x.reshape(-1, x.shape[-1]).float().contiguous())
        w = weight.detach().float().contiguous()
        b = bias.detach().float().contiguous() if bias is not None else None
        _lib.require_cuda(x=x2d, weight=w, bias=b)
        y = _gemm(x2d, w, b)
        ctx.save_for_backward(x2d, w)
        ctx.has_bias = bias is not None
        ctx.shape = x.shape
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        x2d, w = ctx.saved_tensors
        g = _lib.aligned(grad_y.reshape(-1, grad_y.shape[-1]).float().contiguous())
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = _gemm(g, w.t().contiguous(), None).view(ctx.shape)          # grad_y @ W
        if ctx.needs_input_grad[1]:
            gw = g.t() @ x2d                                                  # [N, K] reduction over the rows (cuBLAS fp32)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = g.sum(0)
        return gx, gw, gb


def linear_tf32x3(x, weight, bias=None):
    """F.linear(x, weight, bias) for fp32 CUDA tensors with in/out features multiples of 128."""
    if not supported(weight.shape[1], weight.shape[0], x):
        raise RuntimeError("linear_tf32x3 needs fp32 CUDA tensors and in/out features that are multiples of 128")
    return _LinearTF32x3.apply(x, weight, bias)
