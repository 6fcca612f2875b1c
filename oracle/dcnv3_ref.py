"""CPU oracle for DCNv3 (InternImage's deformable convolution v3 core op).  TEST INFRASTRUCTURE ONLY.

The op is stated from its formula, in differentiable torch, so it runs in fp64 on any device and autograd gives
every gradient.  Layouts are channel-last: input [N, H, W, G*Cg], offset [N, Ho, Wo, G*K*2] as (dx, dy) pairs,
mask [N, Ho, Wo, G*K], output [N, Ho, Wo, G*Cg], K = kh*kw, kernel point p = i*kh + j with i < kw along x.
With s = offset_scale, cw = (dw*(kw-1)) // 2 and ch = (dh*(kh-1)) // 2, point p of (n, ho, wo, g) samples at
    x = wo*sw - pw + cw + (i*dw - cw + dx) * s,   y = ho*sh - ph + ch + (j*dh - ch + dy) * s
(pixels of the unpadded input, no -0.5 shift) and contributes mask * bilinear(input, y, x) when -1 < y < H and
-1 < x < W, both strict; the bilinear form is taken on the floor cell, corners outside the image read 0.
Boundary rule: a sample outside the open range, one exactly on -1 or on H (W) included, contributes nothing and
gets zero for every gradient.  Inside, d/d(x, y) is that of the floor cell's bilinear form: one-sided (from the
right) on integer lines.

Pinning (tests/test_dcnv3_cpu.py): it equals one-level MSDA (`oracle.msda_ref.msda_grid_sample`) on the
zero-padded input at locations ((x + pw + 0.5) / W_pad, (y + ph + 0.5) / H_pad), heads = groups, weights = mask,
everywhere in value and in gradients away from x = -1 / y = -1; and it reproduces the reference's own pure-torch
`dcnv3_core_pytorch` on the golden vectors of tests/golden/dcnv3.npz.
"""
import torch


def output_size(H, W, kh, kw, sh, sw, ph, pw, dh, dw):
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def sample_points(offset, H, W, kh, kw, sh, sw, ph, pw, dh, dw, group, offset_scale):
    """(x, y) [N, Ho, Wo, G, K] of every sample, differentiable in offset."""
    N, Ho, Wo, _ = offset.shape
    K = kh * kw
    dev, dt = offset.device, offset.dtype
    cw, ch = (dw * (kw - 1)) // 2, (dh * (kh - 1)) // 2
    p = torch.arange(K, device=dev)
    i, j = p // kh, p % kh
    off = offset.reshape(N, Ho, Wo, group, K, 2)
    wo = torch.arange(Wo, device=dev).view(1, 1, Wo, 1, 1)
    ho = torch.arange(Ho, device=dev).view(1, Ho, 1, 1, 1)
    x = (wo * sw - pw + cw).to(dt) + ((i * dw - cw).to(dt) + off[..., 0]) * offset_scale
    y = (ho * sh - ph + ch).to(dt) + ((j * dh - ch).to(dt) + off[..., 1]) * offset_scale
    return x, y


def terms(input, offset, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale):
    """The pieces of every sample, [N, Ho, Wo, G, K(, Cg)]: inside (bool), the fractional parts ly, lx (with
    gradients to the offsets) and the four corner values c00, c01, c10, c11 (0 outside the image or the range)."""
    N, H, W, C = input.shape
    G, Cg, K = group, group_channels, kh * kw
    assert C == G * Cg
    Ho, Wo = output_size(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    assert tuple(offset.shape) == (N, Ho, Wo, G * K * 2)
    x, y = sample_points(offset, H, W, kh, kw, sh, sw, ph, pw, dh, dw, G, offset_scale)
    inside = (x > -1) & (y > -1) & (x < W) & (y < H)
    x0, y0 = x.detach().floor(), y.detach().floor()
    img = input.reshape(N, H * W, G, Cg).permute(0, 2, 1, 3)                  # [N, G, HW, Cg]

    def corner(yy, xx):
        ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()           # [N, Ho, Wo, G, K]
        idx = idx.permute(0, 3, 1, 2, 4).reshape(N, G, Ho * Wo * K, 1).expand(N, G, Ho * Wo * K, Cg)
        v = img.gather(2, idx).view(N, G, Ho, Wo, K, Cg).permute(0, 2, 3, 1, 4, 5)
        return v * ok[..., None].to(v.dtype)

    return (inside, y - y0, x - x0, corner(y0, x0), corner(y0, x0 + 1), corner(y0 + 1, x0),
            corner(y0 + 1, x0 + 1))


def dcnv3(input, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale):
    """-> output [N, Ho, Wo, G*Cg] in the inputs' dtype."""
    N, Ho, Wo, _ = offset.shape
    K = kh * kw
    assert tuple(mask.shape) == (N, Ho, Wo, group * K)
    inside, ly, lx, c00, c01, c10, c11 = terms(input, offset, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels,
                                               offset_scale)
    lx, ly = lx[..., None], ly[..., None]
    val = (1 - ly) * (1 - lx) * c00 + (1 - ly) * lx * c01 + ly * (1 - lx) * c10 + ly * lx * c11
    w = mask.reshape(N, Ho, Wo, group, K) * inside.to(mask.dtype)
    return (val * w[..., None]).sum(4).reshape(N, Ho, Wo, -1)


def dcnv3_backward(input, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale,
                   grad_output, dtype=torch.float64):
    """(output, grad_input, grad_offset, grad_mask) of `dcnv3` by autograd, in `dtype`."""
    leaves = [t.detach().to(dtype).requires_grad_(True) for t in (input, offset, mask)]
    out = dcnv3(*leaves, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale)
    out.backward(grad_output.to(dtype))
    return (out.detach(),) + tuple(t.grad for t in leaves)


def as_msda(input, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale):
    """The same op as one-level MSDA arguments: (value [N, Hp*Wp, G, Cg] of the zero-padded input, spatial_shapes
    [[Hp, Wp]], sampling_locations [N, Ho*Wo, G, 1, K, 2], attention_weights [N, Ho*Wo, G, 1, K]), all
    differentiable in input / offset / mask."""
    N, H, W, C = input.shape
    G, Cg, K = group, group_channels, kh * kw
    Hp, Wp = H + 2 * ph, W + 2 * pw
    value = torch.nn.functional.pad(input, (0, 0, pw, pw, ph, ph)).reshape(N, Hp * Wp, G, Cg)
    x, y = sample_points(offset, H, W, kh, kw, sh, sw, ph, pw, dh, dw, G, offset_scale)
    Q = x.shape[1] * x.shape[2]
    loc = torch.stack(((x + pw + 0.5) / Wp, (y + ph + 0.5) / Hp), -1).reshape(N, Q, G, 1, K, 2)
    shapes = torch.tensor([[Hp, Wp]], dtype=torch.int64)
    return value, shapes, loc, mask.reshape(N, Q, G, 1, K)
