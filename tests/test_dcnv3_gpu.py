"""DCNv3 on the GPU (vidar_b200/dcnv3.py, csrc/dcnv3.cu): every kernel instantiation against the fp64 oracle of
oracle/dcnv3_ref.py, the 16-bit paths within elementwise bounds derived from their rounding steps, the reference's
own compiled extension (oracle/_ref/ref_dcnv3.so) where it was built, the module (also under autocast), and the launch
rules.

fp32 parity: each output and gradient within 2e-6 of its largest oracle magnitude.  Samples are kept 1e-3 px away
from integer lines (`_kink_free`), where d/d(x, y) of the bilinear form jumps; the boundary cases place samples
exactly on -1, on H and W, and on integer lines, where the kernel's fp32 positions are exact and both sides take the
floor cell's one-sided derivative.

16-bit bounds.  The oracle runs in fp64 on the inputs rounded to T (x^, o^, m^, g^).  Offsets below 2^-8 in magnitude
are set to 0 and images are under 32 px, so every sample position is exact in fp32 and the kernel samples where the
oracle does.  u is T's unit roundoff (2^-11 fp16, 2^-8 bf16), e = 2^-24, ETA = 2^-25 the largest rounding error of an
fp16 subnormal (0 for bf16).  Abs quantities are the oracle's on |x^|, |m^|, |g^| (bilinear weights are non-negative,
so each bounds the magnitude of every term the op sums):
- output: bilinear weights 1 rounding, four fma, one fma per point into the accumulator: (K + 8) e A, then the
  rounding to T: u |y*| + ETA.  A = output of the abs problem.
- grad_input: m g w per term (3 roundings) summed by red.add in any order, n terms at most: (n + 3) e Bx, then the
  cast: u |gx*| + ETA.  Bx = grad_input of the abs problem, n counted from the samples.
- grad_mask: per corner a Cg-term dot d_ab = sum_c g x_ab over vectors and lanes, combined with the four bilinear
  weights (2 roundings each): (Cg + 8) e Bm, then u |gm*| + ETA.
- grad_offset: the same corner dots combined as ly (d11 - d10) + (1 - ly)(d01 - d00) (and likewise for y), then the
  two products by s and m: (Cg + 10) e Bo, then u |go*| + ETA; Bo = |s m| sum_c |g| D with D the abs form
  ly (|x11| + |x10|) + (1 - ly)(|x01| + |x00|).
First-order bounds; SAFETY = 2 covers the second-order terms.
"""
import pytest
import torch

from oracle import dcnv3_ref

pytestmark = pytest.mark.gpu

U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
E32 = 2.0 ** -24
SAFETY = 2.0


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _inputs(N, H, W, G, Cg, k, s, p, d, spread, seed):
    kh, kw = k
    Ho, Wo = dcnv3_ref.output_size(H, W, kh, kw, s[0], s[1], p[0], p[1], d[0], d[1])
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, G * Cg, generator=g)
    off = torch.randn(N, Ho, Wo, G * kh * kw * 2, generator=g) * spread
    mask = torch.softmax(torch.randn(N, Ho, Wo, G, kh * kw, generator=g), -1).reshape(N, Ho, Wo, -1)
    gy = torch.randn(N, Ho, Wo, G * Cg, generator=g)
    return x, off, mask, gy


def _kink_free(off, H, W, args, eps=1e-3):
    """[N, Ho, Wo, G*K*2] bool: both coordinates of the sample are farther than eps from every integer line."""
    x, y = dcnv3_ref.sample_points(off.double().cpu(), H, W, *args[:8], args[8], args[10])
    ok = ((x - x.round()).abs() > eps) & ((y - y.round()).abs() > eps)
    return torch.stack([ok, ok], -1).reshape(off.shape)


def _run(x, off, mask, gy, args, step=256):
    from vidar_b200.dcnv3 import DCNv3Function
    leaves = [t.detach().clone().requires_grad_(True) for t in (x, off, mask)]
    y = DCNv3Function.apply(*leaves, *args, step)
    y.backward(gy)
    return y.detach(), leaves[0].grad, leaves[1].grad, leaves[2].grad


def _close(what, got, ref, keep=None, tol=2e-6):
    err = (got.detach().cpu().double() - ref)
    if keep is not None:
        err = err[keep]
    scale = ref.abs().max().item()
    assert err.abs().max().item() <= tol * max(scale, 1e-30), f"{what}: {err.abs().max().item():.3e} vs {scale:.3e}"


# (N, H, W, G, Cg, kernel, stride, pad, dilation, offset_scale, im2col_step)
FP32_CASES = {
    "cg16_k3": (2, 9, 11, 4, 16, (3, 3), (1, 1), (1, 1), (1, 1), 1.0, 256),
    "cg32_k3_s2": (2, 10, 13, 2, 32, (3, 3), (2, 2), (1, 1), (1, 1), 1.0, 1),
    "cg7_scalar_k5": (3, 9, 8, 3, 7, (5, 5), (1, 1), (2, 2), (1, 1), 1.0, 256),     # N = 3, step clamped to 3
    "cg16_k5_d2_s05": (2, 12, 11, 2, 16, (5, 5), (1, 2), (2, 3), (2, 2), 0.5, 2),
    "cg136_two_runs": (1, 7, 9, 2, 136, (3, 3), (1, 1), (1, 1), (1, 1), 1.0, 256),   # 4 * 32 lanes < 136 channels
    "cg40_scalar_two_runs": (2, 6, 7, 1, 40, (3, 3), (1, 1), (0, 0), (1, 1), 1.5, 256),
    "k3x5_asym": (1, 8, 12, 2, 8, (3, 5), (2, 1), (1, 2), (1, 2), 0.5, 256),
}


@pytest.mark.parametrize("case", list(FP32_CASES))
def test_fp32_matches_the_oracle(dev, case):
    N, H, W, G, Cg, k, s, p, d, scale, step = FP32_CASES[case]
    x, off, mask, gy = _inputs(N, H, W, G, Cg, k, s, p, d, 2.0, seed=sum(map(ord, case)))
    args = (*k, *s, *p, *d, G, Cg, scale)
    y, gx, go, gm = _run(*(t.to(dev) for t in (x, off, mask, gy)), args, step)
    ry, rgx, rgo, rgm = dcnv3_ref.dcnv3_backward(x, off, mask, *args, gy)
    keep = _kink_free(off, H, W, args)
    _close(f"{case} out", y, ry)
    _close(f"{case} grad_input", gx, rgx)
    _close(f"{case} grad_offset", go, rgo, keep)
    _close(f"{case} grad_mask", gm, rgm)


@pytest.mark.parametrize("Cg", [16, 7])
def test_fp32_misaligned_buffers_take_the_scalar_path(dev, Cg):
    N, H, W, G = 2, 7, 8, 2
    x, off, mask, gy = _inputs(N, H, W, G, Cg, (3, 3), (1, 1), (1, 1), (1, 1), 1.5, seed=5)
    args = (3, 3, 1, 1, 1, 1, 1, 1, G, Cg, 1.0)
    xs = torch.empty(x.numel() + 1, device=dev)[1:].view(x.shape)
    xs.copy_(x)
    assert xs.data_ptr() % 16 and xs.is_contiguous()
    y, gx, go, gm = _run(xs, off.to(dev), mask.to(dev), gy.to(dev), args)
    ry, rgx, rgo, rgm = dcnv3_ref.dcnv3_backward(x, off, mask, *args, gy)
    _close("out", y, ry)
    _close("grad_input", gx, rgx)
    _close("grad_offset", go, rgo, _kink_free(off, H, W, args))
    _close("grad_mask", gm, rgm)


@pytest.mark.parametrize("Cg", [16, 5])
def test_samples_on_minus_one_on_the_far_edge_and_inside_the_first_cell(dev, Cg):
    """Zero offsets with a 3x3 kernel, pad 1 put the border samples exactly on x = -1, y = -1, x = W and y = H (all
    dropped, zero gradients) and the others on integer lines; a quarter-pixel shift puts samples in (-1, 0)."""
    N, H, W, G = 1, 6, 7, 2
    x, _, mask, gy = _inputs(N, H, W, G, Cg, (3, 3), (1, 1), (1, 1), (1, 1), 0.0, seed=9)
    args = (3, 3, 1, 1, 1, 1, 1, 1, G, Cg, 1.0)
    for shift in (0.0, 0.25, -0.25):
        off = torch.full((N, H, W, G * 18), shift)
        y, gx, go, gm = _run(*(t.to(dev) for t in (x, off, mask, gy)), args)
        ry, rgx, rgo, rgm = dcnv3_ref.dcnv3_backward(x, off, mask, *args, gy)
        _close(f"shift {shift} out", y, ry)
        _close(f"shift {shift} grad_input", gx, rgx)
        _close(f"shift {shift} grad_offset", go, rgo)
        _close(f"shift {shift} grad_mask", gm, rgm)
        if shift == 0.0:
            px, _ = dcnv3_ref.sample_points(off.double(), H, W, *args[:8], G, 1.0)
            on = (px == -1).unsqueeze(-1).expand(*px.shape, 2).reshape(go.shape)
            assert on.any() and (go.cpu()[on] == 0).all()
            assert (gm.cpu()[(px == -1).reshape(gm.shape)] == 0).all()


def _abs_bounds(xr, offr, mr, gr, args):
    """A, Bx, Bm, Bo (see the module docstring) and n, from the rounded inputs in fp64 on the CPU."""
    xa, ma, ga = xr.abs().double().cpu(), mr.abs().double().cpu(), gr.abs().double().cpu()
    o = offr.double().cpu()
    A, Bx, _, Bm = dcnv3_ref.dcnv3_backward(xa, o, ma, *args, ga)
    kh, kw, sh, sw, ph, pw, dh, dw, G, Cg, s = args
    inside, ly, lx, c00, c01, c10, c11 = dcnv3_ref.terms(xa, o, *args)
    ly, lx = ly[..., None], lx[..., None]
    N, Ho, Wo = o.shape[:3]
    gq = ga.view(N, Ho, Wo, G, 1, Cg)
    mq = ma.view(N, Ho, Wo, G, kh * kw) * abs(s)
    Dx = ly * (c11 + c10) + (1 - ly) * (c01 + c00)
    Dy = lx * (c11 + c01) + (1 - lx) * (c10 + c00)
    Bo = torch.stack([mq * (gq * Dx).sum(-1), mq * (gq * Dy).sum(-1)], -1).reshape(o.shape)
    # n: the most (sample, corner) terms any input element receives
    H, W = xr.shape[1:3]
    px, py = dcnv3_ref.sample_points(o, H, W, kh, kw, sh, sw, ph, pw, dh, dw, G, s)
    hits = torch.zeros(N * H * W, dtype=torch.float64)
    for ddy in (0, 1):
        for ddx in (0, 1):
            yy, xx = py.floor() + ddy, px.floor() + ddx
            ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
            nn_ = torch.arange(N).view(N, 1, 1, 1, 1).expand_as(yy)
            idx = (nn_ * H * W + yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()
            hits.index_add_(0, idx[ok], torch.ones(int(ok.sum()), dtype=torch.float64))
    return A, Bx, Bm, Bo, hits.max().item()


def _within(what, got, ref, bound, keep=None):
    err = (got.detach().cpu().double() - ref).abs()
    assert torch.isfinite(got).all(), what
    if keep is not None:
        err, bound = err[keep], bound[keep]
    worst = int((err - bound).argmax())
    assert (err <= bound).all(), f"{what}: error {err.flatten()[worst]:.3e} over its bound {bound.flatten()[worst]:.3e}"


HALF_CASES = {
    "cg16_k3": (2, 9, 11, 4, 16, (3, 3), (1, 1), (1, 1), (1, 1), 1.0),
    "cg32_k5_s2_d2": (2, 12, 13, 2, 32, (5, 5), (2, 1), (2, 3), (2, 1), 0.5),
    "cg12_scalar": (3, 8, 9, 2, 12, (3, 3), (1, 1), (1, 1), (1, 1), 1.0),
    "cg272_two_runs": (1, 6, 7, 1, 272, (3, 3), (1, 1), (1, 1), (1, 1), 1.0),
}


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["float16", "bfloat16"])
@pytest.mark.parametrize("case", list(HALF_CASES))
def test_16bit_within_rounding_bounds(dev, case, dt):
    N, H, W, G, Cg, k, s, p, d, scale = HALF_CASES[case]
    x, off, mask, gy = _inputs(N, H, W, G, Cg, k, s, p, d, 2.0, seed=sum(map(ord, case)))
    off = off.to(dt)
    off = off.masked_fill(off.abs() < 2.0 ** -8, 0)
    xr, mr, gr = x.to(dt), mask.to(dt), gy.to(dt)
    args = (*k, *s, *p, *d, G, Cg, scale)
    y, gx, go, gm = _run(*(t.to(dev) for t in (xr, off, mr, gr)), args)
    for t in (y, gx, go, gm):
        assert t.dtype == dt
    ry, rgx, rgo, rgm = dcnv3_ref.dcnv3_backward(xr, off, mr, *args, gr)
    A, Bx, Bm, Bo, n = _abs_bounds(xr, off, mr, gr, args)
    u, eta, K = U[dt], ETA[dt], k[0] * k[1]
    _within(f"{case} out", y, ry, SAFETY * ((K + 8) * E32 * A + u * ry.abs()) + eta)
    _within(f"{case} grad_input", gx, rgx, SAFETY * ((n + 3) * E32 * Bx + u * rgx.abs()) + eta)
    _within(f"{case} grad_mask", gm, rgm, SAFETY * ((Cg + 8) * E32 * Bm + u * rgm.abs()) + eta)
    _within(f"{case} grad_offset", go, rgo, SAFETY * ((Cg + 10) * E32 * Bo + u * rgo.abs()) + eta,
            _kink_free(off.float(), H, W, args))


def _reference_ext():
    try:
        from oracle import build_ref_dcnv3
        return build_ref_dcnv3.load()
    except (FileNotFoundError, ImportError, OSError) as e:
        pytest.skip(f"reference DCNv3 extension not built: {e}")


# InternImage-T stages 1 and 3 at the 928 x 1600 input (stem stride 4): C = 64 / 256, group = C / 16, one image
REF_SHAPES = {"T_stage1": (1, 232, 400, 4, 16), "T_stage3": (1, 58, 100, 16, 16)}


@pytest.mark.parametrize("dt", [torch.float32, torch.float16], ids=["float32", "float16"])
@pytest.mark.parametrize("shape", list(REF_SHAPES))
def test_matches_the_reference_extension(dev, shape, dt):
    """Same rounded inputs into both ops; the reference sums grad_input, grad_offset and grad_mask with atomics in no
    fixed order, so the comparison is within a tolerance: 1e-5 (fp32) or 4 units of T's roundoff (fp16) of each
    tensor's largest magnitude."""
    ref = _reference_ext()
    from vidar_b200.dcnv3 import ext
    N, H, W, G, Cg = REF_SHAPES[shape]
    x, off, mask, gy = (t.to(dev, dt) for t in _inputs(N, H, W, G, Cg, (3, 3), (1, 1), (1, 1), (1, 1), 1.0, seed=1))
    args = (3, 3, 1, 1, 1, 1, 1, 1, G, Cg, 1.0)
    ours = [ext.dcnv3_forward(x, off, mask, *args, 256)] + ext.dcnv3_backward(x, off, mask, *args, gy, 256)
    theirs = [ref.dcnv3_forward(x, off, mask, *args, 256)] + list(ref.dcnv3_backward(x, off, mask, *args, gy, 256))
    tol = 1e-5 if dt == torch.float32 else 4 * 2.0 ** -11
    keep = _kink_free(off.float(), H, W, args).to(dev)
    for what, a, b in zip(("out", "grad_input", "grad_offset", "grad_mask"), ours, theirs):
        assert a.dtype == b.dtype == dt, what
        diff = (a.float() - b.float()).abs()
        if what == "grad_offset":
            diff = diff[keep]
        assert diff.max().item() <= tol * b.float().abs().max().item(), f"{shape} {what}: {diff.max().item():.3e}"


def _module_pair(dev, center):
    from vidar_b200 import dcnv3
    torch.manual_seed(3)
    m = dcnv3.DCNv3(channels=64, kernel_size=3, group=4, offset_scale=1.0, center_feature_scale=center)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for n, prm in m.named_parameters():
            prm.copy_(torch.randn(prm.shape, generator=g) * (0.5 if "offset" in n else 0.2))
    return m.to(dev), dcnv3


@pytest.mark.parametrize("center", [False, True])
def test_module_forward_and_backward_match_the_oracle_core(dev, center, monkeypatch):
    import copy
    m, dcnv3 = _module_pair(dev, center)
    ref = copy.deepcopy(m).double().cpu()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 9, 10, 64, generator=g)
    gy = torch.randn(2, 9, 10, 64, generator=g)
    xd = x.to(dev).requires_grad_(True)
    y = m(xd)
    y.backward(gy.to(dev))

    class Oracle(torch.autograd.Function):
        @staticmethod
        def forward(ctx, inp, off, msk, *args):
            ctx.args = args[:-1]
            ctx.save_for_backward(inp, off, msk)
            return dcnv3_ref.dcnv3(inp, off, msk, *ctx.args)

        @staticmethod
        def backward(ctx, go):
            with torch.enable_grad():
                leaves = [t.detach().requires_grad_(True) for t in ctx.saved_tensors]
                out = dcnv3_ref.dcnv3(*leaves, *ctx.args)
                grads = torch.autograd.grad(out, leaves, go)
            return (*grads,) + (None,) * 12

    monkeypatch.setattr(dcnv3, "DCNv3Function", Oracle)
    xc = x.double().requires_grad_(True)
    yr = ref(xc)
    yr.backward(gy.double())
    _close("module out", y, yr.detach(), tol=1e-5)
    _close("module grad_x", xd.grad, xc.grad, tol=1e-4)
    for (n, p), (_, pr) in zip(m.named_parameters(), ref.named_parameters()):
        assert p.grad is not None and p.grad.dtype == torch.float32, n
        _close(f"module grad {n}", p.grad, pr.grad, tol=1e-4)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["float16", "bfloat16"])
def test_module_under_autocast(dev, dt):
    """Under autocast the op runs in the autocast dtype (input_proj and the offset Linear emit it); fp32 parameters
    get fp32 gradients, close to the fp32 module's (normwise, 32 units of T's roundoff)."""
    import copy
    m, _ = _module_pair(dev, True)
    m32 = copy.deepcopy(m)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 9, 10, 64, generator=g).to(dev)
    with torch.autocast("cuda", dtype=dt):
        y = m(x)
    assert y.dtype == dt
    y.float().square().mean().backward()
    y32 = m32(x)
    y32.square().mean().backward()
    u = U[dt]
    assert (y.float() - y32).norm() <= 32 * u * y32.norm()
    for (n, p), (_, p32) in zip(m.named_parameters(), m32.named_parameters()):
        assert p.grad.dtype == torch.float32 and torch.isfinite(p.grad).all(), n
        assert (p.grad - p32.grad).norm() <= 32 * u * p32.grad.norm() + 1e-12, n


def test_one_launch_each_and_no_host_sync(dev):
    from vidar_b200 import _lib
    from vidar_b200.dcnv3 import DCNv3Function
    x, off, mask, gy = (t.to(dev) for t in _inputs(2, 8, 9, 4, 16, (3, 3), (1, 1), (1, 1), (1, 1), 1.0, seed=2))
    leaves = [t.requires_grad_(True) for t in (x, off, mask)]
    args = (3, 3, 1, 1, 1, 1, 1, 1, 4, 16, 1.0, 256)
    DCNv3Function.apply(*leaves, *args).backward(gy)          # warm-up (library load, allocator)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = DCNv3Function.apply(*leaves, *args)
        n1 = _lib.launch_count()
        y.backward(gy)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert n1 - n0 == 1 and _lib.launch_count() - n1 == 1
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        y2 = DCNv3Function.apply(*[t.detach() for t in leaves], *args)
    stream.synchronize()
    assert torch.equal(y2, y.detach())
