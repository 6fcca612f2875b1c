"""Mixed-precision modulated deformable convolution (vidar_b200/dcn.py, csrc/dcn.cu) on the GPU: the float16 and
bfloat16 paths against the fp64 oracle of oracle/dcn_ref.py with elementwise bounds, the dtype rule, the module under
autocast, the DCN backbone under autocast, and the pre-training step with `backbone_autocast`.

Oracle parity.  The oracle runs in fp64 on the inputs after they are rounded to T (x^, o^, m^, W^, b^ and the
upstream gradient g^), so only the op's own rounding is measured.  u is T's unit roundoff (2^-11 fp16, 2^-8 bf16),
e = 2^-24 fp32's, ETA = 2^-25 the largest rounding error of an fp16 subnormal (0 for bf16, whose range is fp32's).
Offsets below 2^-8 in magnitude are set to 0: every other T offset has no bit below 2^-18, so each sample position
h = base + o^ (|h| < 64 here) is exact in fp32 and the kernel samples exactly where the oracle does.  The GEMMs run
with cuBLAS's reduced-precision reductions off, so they accumulate in fp32.  Bounds, all elementwise, with
Kc = kh*kw*C, M = N*Ho*Wo, and abs quantities computed by the oracle on |x^|, o^, |m^|, |W^|, |b^|, |g^| (the bilinear
weights are non-negative, so each is an upper bound on the magnitude of every term the op sums):
- columns: bilinear weights from exact fractional parts (<= 1 rounding each in 1 - l, 1 in the product), four fma
  and the mask product: <= 8 e relative to their abs value; then one rounding to T: u.
- y = cols @ W'^T + b on cuBLAS, products of T values exact in fp32, Kc-term fp32 sum, one rounding to T:
    |y - y*| <= (u + (Kc + 8) e) A + u |y*| + ETA (1 + sum|W^_o|),   A = oracle(|x^|, o^, |m^|, |W^|, |b^|).
- grad_cols = g @ W' (Cout-term fp32 sum, rounded once to T): |gc - gc*| <= (u + Cout e) G + ETA,
  G[n, c, k, p] = sum_o |g^| |W^| (an intermediate, not compared).
- grad_x: col2im adds m w_i gc into fp32 with red.add in any order, at most n terms per element (n counted from
  the samples): (u + (Cout + n + 12) e) Bx + ETA n before the cast to T (u |gx*| + ETA), Bx = grad_input of the
  abs problem.
- grad_mask = sum_c gc v_c, v recomputed in fp32 from x^ (<= 8 e), fp32 warp sum (C / 32 lane steps, 5 shuffle
  levels): (u + (Cout + C + 16) e) Bm + ETA sum_c V_c, then the cast; Bm = grad_mask of the abs problem = sum_c G V,
  V = the bilinear value on |x^|.
- grad_offset = m sum_c gc dv/d(h, w), dv/dh = lw (x11 - x01) + (1 - lw)(x10 - x00) in fp32: the same as grad_mask
  with Bo = |m^| sum_c G D, D = lw (|x01| + |x11|) + (1 - lw)(|x00| + |x10|) (and likewise for w), on kink-free
  coordinates (`_kink_free`: one-sided derivatives legitimately jump on integer lines).
- grad_weight: fp32 cuBLAS output of g^T cols (products exact, M-term sums, one fp32 add per column chunk) and the
  cols' own rounding: (u + (M + N + 8) e) Bw + ETA sum|g^|, then the cast; Bw = grad_weight of the abs problem.
- grad_bias: an fp32 sum of M terms, (M + 2) e sum|g^| + ETA, then the cast.
The bounds are first order; SAFETY = 2 covers the second-order terms.  The largest error-to-bound ratio of each
quantity is printed at the end of the module (pytest -s).

Backbone.  The backbone under autocast with our 16-bit op, the same under autocast with each DCN computed by our
fp32 op on .float() inputs (those the dtype rule gives, the weight included; the output cast to the autocast dtype,
as an op under autocast returns it), and the
backbone in fp32 (TF32 off) as reference, with a mean loss per level (scaled by 512 in fp16): C3-C5 and every
layer3 / layer4 gradient of the 16-bit op are within BACKBONE_FACTOR = 3 of the fp32 op's error (max and L2 norms).
The 16-bit path rounds each column element once more than the fp32 op, in each of the 26 layers, on top of the
roundings the autocast convolutions around it make in both runs; on the H100 the largest ratio over all these
tensors was 2.4 in fp16 and in bf16, mostly 1-2.
"""
import copy

import pytest
import torch

from oracle import dcn_ref
from tests.test_dcn_gpu import SAMPLE, SMALL, _inputs, _kink_free

pytestmark = pytest.mark.gpu

DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
E32 = 2.0 ** -24
SAFETY = 2.0
BACKBONE_FACTOR = 3.0
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest error / bound per quantity:")
    for k in sorted(RATIOS):
        print(f"  {k:32s} {RATIOS[k]:.3e}")


@pytest.fixture
def fp32_accumulation(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_fp16_reduced_precision_reduction", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_bf16_reduced_precision_reduction", False)


def _sampling_abs(xa, off, k, stride, padding, dilation):
    """From |x^| [N, C, H, W] and the offsets: per (n, c, k, ho, wo) the bilinear value V on |x^| and the absolute
    forms Dh, Dw of its derivatives, and the largest number of (sample, corner) terms any input element receives."""
    N, C, H, W = xa.shape
    kh, kw = k
    K = kh * kw
    Ho, Wo = off.shape[-2:]
    dev = xa.device
    o = off.double().view(N, K, 2, Ho, Wo)
    i = torch.arange(kh, device=dev).repeat_interleave(kw)
    j = torch.arange(kw, device=dev).repeat(kh)
    h = (torch.arange(Ho, device=dev)[None, :] * stride[0] - padding[0] + i[:, None] * dilation[0]).double()[None, :, :, None] + o[:, :, 0]
    w = (torch.arange(Wo, device=dev)[None, :] * stride[1] - padding[1] + j[:, None] * dilation[1]).double()[None, :, None, :] + o[:, :, 1]
    inside = (h > -1) & (h < H) & (w > -1) & (w < W)
    h0, w0 = h.floor(), w.floor()
    lh, lw = (h - h0)[:, None], (w - w0)[:, None]
    flat = xa.double().reshape(N, C, H * W)
    hits = torch.zeros(N, H * W, dtype=torch.float64, device=dev)
    c = {}
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = h0 + dy, w0 + dx
            ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long().view(N, -1)
            hits.scatter_add_(1, idx, ok.view(N, -1).double())
            v = flat.gather(2, idx[:, None].expand(N, C, -1)).view(N, C, K, Ho, Wo)
            c[dy, dx] = torch.where(ok[:, None], v, torch.zeros((), dtype=torch.float64, device=dev))
    V = (1 - lh) * (1 - lw) * c[0, 0] + (1 - lh) * lw * c[0, 1] + lh * (1 - lw) * c[1, 0] + lh * lw * c[1, 1]
    Dh = lw * (c[0, 1] + c[1, 1]) + (1 - lw) * (c[0, 0] + c[1, 0])
    Dw = lh * (c[1, 0] + c[1, 1]) + (1 - lh) * (c[0, 0] + c[0, 1])
    return V, Dh, Dw, hits.max().item()


def _within(what, got, ref, bound, keep=None):
    err = (got.detach().double() - ref).abs()
    assert torch.isfinite(got).all(), what
    if keep is not None:
        err, bound = err[keep], bound[keep]
    ratio = torch.where(err > 0, err / bound, 0.0).max().item() if err.numel() else 0.0
    key = what.split(":")[0]
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)
    worst = int((err - bound).argmax()) if err.numel() else 0
    assert ratio <= 1.0, (f"{what}: error {err.flatten()[worst].item():.3e} over its bound "
                          f"{bound.flatten()[worst].item():.3e} (ratio {ratio:.3f})")


def _rounded_inputs(dev, dt, case):
    x, off, mask, w, b, gy = _inputs(dev, **case)
    off = off.to(dt)
    off = off.masked_fill(off.abs() < 2.0 ** -8, 0)
    return [t.to(dt) if t is not None else None for t in (x, off, mask, w, b, gy)]


def _check_against_oracle(dev, dt, misaligned=False, **case):
    from vidar_b200.dcn import modulated_deform_conv2d
    stride, padding, dilation = (case.get(k, (1, 1)) for k in ("stride", "padding", "dilation"))
    k = case.get("k", (3, 3))
    x, off, mask, w, b, gy = _rounded_inputs(dev, dt, case)
    N, C, H, W = x.shape
    O = w.shape[0]
    leaves = [t.clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, w, b)]
    args = list(leaves)
    if misaligned:
        # channels_last input and contiguous offsets 2 bytes past a 16-byte boundary
        buf = torch.empty(x.numel() + 1, dtype=dt, device=dev)
        buf[1:].copy_(x.permute(0, 2, 3, 1).reshape(-1))
        leaves[0] = buf.requires_grad_(True)
        args[0] = leaves[0][1:].view(N, H, W, C).permute(0, 3, 1, 2)
        args[0].retain_grad()
        obuf = torch.empty(off.numel() + 1, dtype=dt, device=dev)
        obuf[1:].copy_(off.reshape(-1))
        leaves[1] = obuf.requires_grad_(True)
        args[1] = leaves[1][1:].view(off.shape)
        args[1].retain_grad()
        assert args[0].data_ptr() % 16 and args[1].data_ptr() % 16
    y = modulated_deform_conv2d(*args, stride, padding, dilation, 1, 1)
    assert y.dtype == dt and y.is_contiguous(memory_format=torch.channels_last)
    y.backward(gy)
    grads = [a.grad if a is not None else None for a in args]
    assert all(g.dtype == dt for g in grads if g is not None)

    geo = dict(stride=stride, padding=padding, dilation=dilation)
    y_ref, ref = dcn_ref.deform_conv2d_backward(x, off, mask, w, b, gy, **geo)
    absb = b.abs() if b is not None else None
    A, (Bx, _, Bm, Bw, _) = dcn_ref.deform_conv2d_backward(x.abs(), off, mask.abs(), w.abs(), absb, gy.abs(), **geo)
    V, Dh, Dw, n = _sampling_abs(x.abs(), off, k, stride, padding, dilation)
    Ho, Wo = y.shape[-2:]
    K, M, P = k[0] * k[1], N * Ho * Wo, Ho * Wo
    G = torch.einsum("ock,nop->nckp", w.abs().double().reshape(O, C, K), gy.abs().double().reshape(N, O, P))
    G = G.view(N, C, K, Ho, Wo)
    m_abs = mask.abs().double()
    Bo = torch.stack([m_abs * (G * Dh).sum(1), m_abs * (G * Dw).sum(1)], 2).view(N, 2 * K, Ho, Wo)
    Vo = torch.stack([m_abs * Dh.sum(1), m_abs * Dw.sum(1)], 2).view(N, 2 * K, Ho, Wo)
    u, eta, Kc = U[dt], ETA[dt], K * C
    sum_g = gy.abs().double().sum()
    tag = f"{dt}".replace("torch.", "")

    w_l1 = w.abs().double().reshape(O, -1).sum(1).view(1, O, 1, 1)
    _within(f"out {tag}: {case}", y, y_ref,
            SAFETY * ((u + (Kc + 8) * E32) * A + u * y_ref.abs() + eta * (1 + w_l1)))
    bounds = {
        "input": (u + (O + n + 12) * E32) * Bx + eta * n,
        "offset": (u + (O + C + 16) * E32) * Bo + eta * Vo,
        "mask": (u + (O + C + 16) * E32) * Bm + eta * V.sum(1),
        "weight": (u + (M + N + 8) * E32) * Bw + eta * sum_g,
        "bias": None if b is None else (M + 2) * E32 * sum_g + eta,
    }
    keep_off = _kink_free(off, stride, padding, dilation, k).to(dev)
    for what, got, r in zip(("input", "offset", "mask", "weight", "bias"), grads, ref):
        if got is None:
            continue
        bound = SAFETY * (bounds[what] + u * r.abs() + eta)
        _within(f"grad_{what} {tag}: {case}", got, r, bound, keep_off if what == "offset" else None)


CASES = {
    # C % 8 == 0: 16-byte, 8-channel loops
    "vec8_c128": dict(N=2, C=128, H=10, W=13, O=128),
    "vec8_c256": dict(N=1, C=256, H=8, W=9, O=64, bias=False),
    # scalar loops: C = 5, and C % 4 == 0 but C % 8 != 0
    "scalar_c5": dict(N=2, C=5, H=9, W=11, O=7, bias=False),
    "scalar_c12": dict(N=1, C=12, H=9, W=10, O=8),
    "stride2": dict(N=2, C=64, H=11, W=14, O=32, stride=(2, 2)),
    "pad0_dil2": dict(N=1, C=64, H=14, W=12, O=32, padding=(0, 0), dilation=(2, 2), bias=False),
    "nonsquare": dict(N=1, C=16, H=9, W=15, O=6, k=(2, 3), stride=(2, 1), padding=(1, 0), dilation=(1, 2)),
    "small_offsets": dict(N=2, C=32, H=8, W=8, O=16, offset_std=0.6),
}


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_oracle(cuda, fp32_accumulation, name, dtype):
    _check_against_oracle(cuda, DTYPES[dtype], **CASES[name])


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_misaligned_views(cuda, fp32_accumulation, dtype):
    _check_against_oracle(cuda, DTYPES[dtype], misaligned=True, N=2, C=16, H=7, W=9, O=8)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_several_column_chunks(cuda, fp32_accumulation, monkeypatch, dtype):
    """5 images in chunks of 2 (+ the remainder 1): a 16-bit chunk holds twice the images of an fp32 one."""
    from vidar_b200 import dcn
    C, H, W = 16, 7, 9
    per_image = H * W * 9 * C
    monkeypatch.setattr(dcn, "MAX_COLS_BYTES", 2 * 2 * per_image + 100)
    assert dcn.chunk_images(5, per_image, 2) == 2 and dcn.chunk_images(5, per_image) == 1
    _check_against_oracle(cuda, DTYPES[dtype], N=5, C=C, H=H, W=W, O=12)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_scalar_fallback_on_misaligned_buffers_gives_the_same_columns(cuda, dtype):
    """The C entry point itself: x and cols 2 bytes off a 16-byte boundary take the scalar loop, which computes each
    column element with the same fp32 operations as the vector loop."""
    from vidar_b200 import _lib, dcn
    dt = DTYPES[dtype]
    x, off, mask, _, _, _ = _rounded_inputs(cuda, dt, dict(N=2, C=16, H=7, W=9, O=8))
    N, C, H, W = x.shape
    xl = x.permute(0, 2, 3, 1).contiguous()
    geom = (N, C, H, W, H, W, 3, 3, 1, 1, 1, 1, 1, 1)
    n = N * H * W * 9 * C
    xb, cb = torch.empty(xl.numel() + 8, dtype=dt, device=cuda), torch.zeros(2 * n + 8, dtype=dt, device=cuda)
    xb[1:1 + xl.numel()].copy_(xl.view(-1))
    L, st = _lib.lib(), _lib.stream_ptr(cuda)
    code = dcn.HALF_DTYPE_CODES[dt]
    _lib.check(L.vidar_dcn_im2col_half(_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cb), code, *geom, 0, N, st))
    _lib.check(L.vidar_dcn_im2col_half(_lib.ptr(xb[1:]), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cb[n + 1:]), code,
                                       *geom, 0, N, st))
    assert torch.equal(cb[:n], cb[n + 1:2 * n + 1])


def test_dtype_rule(cuda):
    from vidar_b200 import _lib
    from vidar_b200.dcn import modulated_deform_conv2d
    x, off, mask, w, b, gy = _inputs(cuda, 2, 16, 6, 7, 8)

    def run(*ts):
        leaves = [t.clone().requires_grad_(True) for t in ts]
        y = modulated_deform_conv2d(*leaves, 1, 1, 1, 1, 1)
        y.backward(gy.to(y.dtype))
        return y, [t.grad for t in leaves]

    # input fp32, offset fp16: computes in fp16, returns fp16, each gradient in its leaf's dtype
    y, g = run(x, off.half(), mask, w, b)
    assert y.dtype == torch.float16 and [t.dtype for t in g] == [torch.float32, torch.float16] + [torch.float32] * 3
    y16, _ = run(x.half(), off.half(), mask.half(), w.half(), b.half())
    assert torch.equal(y, y16)
    # input fp16, offset fp32: the fp32 path, bit-identical to input.float(); grad_input back in fp16
    y, g = run(x.half(), off, mask, w, b)
    yf, gf = run(x.half().float(), off, mask, w, b)
    assert y.dtype == torch.float32 and torch.equal(y, yf) and g[0].dtype == torch.float16
    assert torch.equal(g[3], gf[3]) and torch.equal(g[4], gf[4])
    # an fp32 weight gets an fp32 grad_weight from the bf16 path
    y, g = run(x.bfloat16(), off.bfloat16(), mask.bfloat16(), w, b.bfloat16())
    assert y.dtype == torch.bfloat16 and g[3].dtype == torch.float32 and g[4].dtype == torch.bfloat16
    with pytest.raises(TypeError, match="float32"):
        modulated_deform_conv2d(x, off.double(), mask, w, b, 1, 1, 1, 1, 1)
    with pytest.raises(TypeError, match="float32"):
        modulated_deform_conv2d(x.half(), off.half(), mask, w.double(), b, 1, 1, 1, 1, 1)
    # an unknown dtype code on the C entry points
    xl = x.half().permute(0, 2, 3, 1).contiguous()
    cols = torch.empty(2 * 6 * 7 * 9 * 16, dtype=torch.float16, device=cuda)
    geom = [2, 16, 6, 7, 6, 7, 3, 3, 1, 1, 1, 1, 1, 1, 0, 2]
    L, st = _lib.lib(), _lib.stream_ptr(cuda)
    for code in (0, 3):
        assert L.vidar_dcn_im2col_half(_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cols), code, *geom, st) == 1
        assert b"unsupported dtype" in L.vidar_last_error()
        assert L.vidar_dcn_col2im_half(_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cols), _lib.ptr(x),
                                       _lib.ptr(off), _lib.ptr(mask), code, *geom, st) == 1
        assert b"unsupported dtype" in L.vidar_last_error()
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_pack_module_under_autocast(cuda, dtype):
    from vidar_b200.dcn import ModulatedDeformConv2dPack
    dt = DTYPES[dtype]
    torch.manual_seed(0)
    m = ModulatedDeformConv2dPack(32, 48, 3, padding=1, bias=True).to(cuda)
    g = torch.Generator().manual_seed(1)
    m.conv_offset.weight.data.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * 0.05)
    x = torch.randn(2, 32, 12, 14, generator=g).to(cuda)
    with torch.autocast("cuda", dtype=dt):
        y = m(x)
    assert y.dtype == dt
    (y.float() * torch.linspace(-1, 1, y.numel(), device=cuda).view_as(y)).sum().backward()
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.dtype == torch.float32, n
        assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n


def _fp32_dcn_forward(self, x):
    """ModulatedDeformConv2dPack.forward with our fp32 op inside an autocast region: the inputs the dtype rule gives
    (x, offset, mask and weight in the autocast dtype) converted by .float(), the output returned in the autocast
    dtype as any op under autocast returns it.  Only the op's internal precision differs from the 16-bit path."""
    from vidar_b200.dcn import modulated_deform_conv2d
    out = self.conv_offset(x)
    o1, o2, mask = torch.chunk(out, 3, dim=1)
    y = modulated_deform_conv2d(x.float(), torch.cat((o1, o2), 1).float(), torch.sigmoid(mask).float(),
                                self.weight.to(out.dtype).float(), None, self.stride, self.padding, self.dilation, 1, 1)
    return y.to(out.dtype)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_backbone_under_autocast(cuda, monkeypatch, dtype):
    from vidar_b200.dcn import ModulatedDeformConv2dPack
    from vidar_b200.pretrain import ImageBackbone
    dt = DTYPES[dtype]
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    torch.manual_seed(0)
    base = ImageBackbone(dcn=True)
    g = torch.Generator().manual_seed(1)
    for m in base.modules():            # the conv_offset initialisation of test_dcn_backbone_matches_torchvision_backbone
        if isinstance(m, ModulatedDeformConv2dPack):
            m.conv_offset.weight.data.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * 1e-3)
            m.conv_offset.bias.data.copy_(torch.randn(m.conv_offset.bias.shape, generator=g) * 0.5)
    fp32_dcn = copy.deepcopy(base)
    for m in fp32_dcn.modules():
        if isinstance(m, ModulatedDeformConv2dPack):
            m.forward = _fp32_dcn_forward.__get__(m)
    img = torch.randn(2, 3, 96, 160, generator=g).to(cuda)
    scale = 512.0 if dt == torch.float16 else 1.0          # the reference's static fp16 loss scale
    runs = []
    for model, amp in ((base, True), (fp32_dcn, True), (base, False)):
        model = copy.deepcopy(model).to(cuda).train()
        with torch.autocast("cuda", dtype=dt, enabled=amp):
            feats = model(img)
        feats = [f.float() for f in feats]
        loss = sum((f * torch.linspace(-1, 1, f.numel(), device=cuda).view_as(f)).mean() for f in feats)
        (loss * (scale if amp else 1.0)).backward()
        grads = {n: p.grad.detach() / (scale if amp else 1.0) for n, p in model.named_parameters()
                 if n.startswith(("layer3", "layer4"))}
        runs.append(([f.detach() for f in feats], grads))
    (fa, ga), (fb, gb), (fc, gc) = runs
    assert set(ga) == set(gc) and sum("conv_offset" in n for n in ga) == 2 * 26
    pairs = list(zip(("C3", "C4", "C5"), fa, fb, fc)) + [(n, ga[n], gb[n], gc[n]) for n in sorted(ga)]
    over, worst = [], 0.0
    for what, a, b, c in pairs:
        assert torch.isfinite(a).all() and torch.isfinite(b).all(), what
        for norm in (lambda v: v.abs().max().item(), lambda v: v.norm().item()):
            err, err_fp32_op = norm((a - c).double()), norm((b - c).double())
            worst = max(worst, err / max(err_fp32_op, 1e-30))
            if err > BACKBONE_FACTOR * err_fp32_op:
                over.append(f"{what}: {dtype} op err {err:.3e}, fp32 op err {err_fp32_op:.3e}")
    RATIOS[f"backbone {dtype} err / fp32-op err"] = worst
    assert not over, "\n".join(over)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_pretrain_step_with_backbone_autocast(cuda, dtype):
    from vidar_b200 import pretrain, synthetic
    dt = DTYPES[dtype]
    model, opt = pretrain.build(cuda, None, seed=1, backbone_autocast=dt, **SMALL)
    sample = pretrain.synthetic_sample(cuda, **SAMPLE)
    l2i = sample["lidar2img"].copy()
    l2i[..., 0, :] *= SAMPLE["img_hw"][1] / synthetic.IMG_HW[1]
    l2i[..., 1, :] *= SAMPLE["img_hw"][0] / synthetic.IMG_HW[0]
    sample["lidar2img"] = l2i
    scaler = torch.amp.GradScaler("cuda", init_scale=512.0) if dt == torch.float16 else None
    loss, _ = pretrain.train_step(model, opt, sample, None, scaler=scaler)
    assert torch.isfinite(loss)
    offs = [(n, p) for n, p in model.named_parameters() if "conv_offset" in n]
    assert len(offs) == 2 * 26
    for n, p in offs:
        assert p.grad is not None and p.grad.dtype == torch.float32, n
        assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n
