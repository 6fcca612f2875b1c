"""fp64 statement of modulated deformable convolution (DCNv2; mmcv's modulated_deform_conv2d, torchvision's
deform_conv2d with a mask), groups = deform_groups = 1, differentiable by autograd.

For output pixel (n, ho, wo) and kernel point k = i * kw + j:
  h = ho * sh - ph + i * dh + offset[n, 2k],  w = wo * sw - pw + j * dw + offset[n, 2k + 1]
  v_c = 0 when h <= -1, h >= H, w <= -1 or w >= W; otherwise the bilinear value of x[n, c] on the floor cell, a corner
        outside [0, H-1] x [0, W-1] adding 0
  y[n, o, ho, wo] = sum_{k, c} weight[o, c, i, j] * mask[n, k] * v_c + bias[o]
The corner weights use the fractional parts h - floor(h), w - floor(w); floor has no gradient, so autograd gives the
one-sided derivative of the bilinear form on the floor cell, and 0 outside the open range.
"""
import torch


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def deform_conv2d(x, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1):
    """x [N, C, H, W], offset [N, 2*kh*kw, Ho, Wo], mask [N, kh*kw, Ho, Wo], weight [O, C, kh, kw], bias [O] or None
    -> y [N, O, Ho, Wo], in the dtype of x (call with fp64 tensors)."""
    sh, sw = _pair(stride)
    ph, pw = _pair(padding)
    dh, dw = _pair(dilation)
    N, C, H, W = x.shape
    O, _, kh, kw = weight.shape
    K = kh * kw
    Ho, Wo = offset.shape[-2:]
    dev, dt = x.device, x.dtype
    i = torch.arange(kh, device=dev).repeat_interleave(kw)          # kernel row of point k
    j = torch.arange(kw, device=dev).repeat(kh)                     # kernel column of point k
    base_h = (torch.arange(Ho, device=dev)[None, :] * sh - ph + i[:, None] * dh).to(dt)       # [K, Ho]
    base_w = (torch.arange(Wo, device=dev)[None, :] * sw - pw + j[:, None] * dw).to(dt)       # [K, Wo]
    off = offset.view(N, K, 2, Ho, Wo)
    h = base_h[None, :, :, None] + off[:, :, 0]                     # [N, K, Ho, Wo]
    w = base_w[None, :, None, :] + off[:, :, 1]
    inside = (h > -1) & (h < H) & (w > -1) & (w < W)
    h0, w0 = torch.floor(h).detach(), torch.floor(w).detach()
    lh, lw = h - h0, w - w0
    flat = x.reshape(N, C, H * W)
    v = 0
    for dy, wy in ((0, 1 - lh), (1, lh)):
        for dx, wx in ((0, 1 - lw), (1, lw)):
            yy, xx = h0 + dy, w0 + dx
            ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long().view(N, 1, -1).expand(N, C, -1)
            corner = flat.gather(2, idx).view(N, C, K, Ho, Wo)
            v = v + torch.where(ok[:, None], (wy * wx)[:, None] * corner, torch.zeros((), dtype=dt, device=dev))
    cols = v * mask[:, None]                                        # [N, C, K, Ho, Wo]
    y = torch.einsum("ock,nckp->nop", weight.reshape(O, C, K), cols.reshape(N, C, K, Ho * Wo)).view(N, O, Ho, Wo)
    if bias is not None:
        y = y + bias.view(1, O, 1, 1)
    return y


def deform_conv2d_backward(x, offset, mask, weight, bias, grad_out, stride=1, padding=0, dilation=1):
    """fp64 gradients (input, offset, mask, weight, bias) of `deform_conv2d` for the upstream gradient grad_out."""
    leaves = [t.detach().double().requires_grad_(True) if t is not None else None for t in (x, offset, mask, weight, bias)]
    y = deform_conv2d(*leaves, stride=stride, padding=padding, dilation=dilation)
    y.backward(grad_out.double())
    return y.detach(), tuple(t.grad if t is not None else None for t in leaves)
