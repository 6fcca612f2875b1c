"""The wgmma 3xTF32 Linear (csrc/linear_tc.cu, SURVEY.md 8f-4) against fp64 and against fp32 cuBLAS.

Metric: per output element r = |y - y64| / (sum_k |x_k| |w_k| + |b|), with y64 the fp64 result on the same inputs.
The kernel passes when the max and the RMS of r are both within FACTOR = 2 of what fp32 cuBLAS (`F.linear`, TF32
off) gets on the same inputs.  Why 2: both sum the same fp32 products and differ only in the order of the additions
and in what 3xTF32 drops (x_lo * w_lo, <= 2^-22 of each product); on an H100 that leaves the kernel at 0.2 - 1.5x
cuBLAS's error for rows >= 129, and at up to 1.9x where cuBLAS switches to a more accurate split reduction for a few
rows (M <= 128).  A sum that rounds toward zero, as the tensor core does inside one accumulator, builds an error that
does not cancel: with all 3 K / 8 wgmma chained into one accumulator the RMS ratio was 2.8x at K = 32 and 27x at
K = 4608 (52x for non-negative inputs).  A bar relative to what cuBLAS gets needs no retuning per K.

SHAPES holds every (M, N, K) the forward runs at: a K sweep 32 ... 4608 (K < 128 through the C ABI, which takes any
multiple of 32, `linear.supported` does not), every out_features the callers pass, last row tiles that hold rows of
one or of both consumer warpgroups, tile counts of one, one more than and 2x - 1 the device's SM count (the
persistent loop's second pass and mbarrier phases), and value_proj's 6 x 30825 x 256 -> 256.  A census test runs a
reduced pre-training step and checks that every (N, K) the wgmma kernel sees there is in the table."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

FACTOR = 2.0
FAMILIES = ("randn", "rand", "spike", "tf32_edges")
KS = (32, 64, 96, 128, 256, 384, 512, 1024, 2304, 4608)

# (M, N, K, families).  M may name a tile count relative to the SM count: "sms", "sms+1", "2sms-1" (N = 128, so a
# tile is 128 rows; the last one is ragged and holds rows of both consumer warpgroups).
SHAPES = (
    [(2048, 256, K, FAMILIES) for K in KS]
    + [(1000, N, K, FAMILIES) for N, K in ((128, 128), (128, 512), (512, 128), (512, 256), (256, 512),
                                           (2304, 256), (4608, 512))]
    + [(M, 256, 256, ("randn", "rand")) for M in (1, 63, 64, 65, 127, 128, 129, 191)]
    + [(M, 128, 256, ("randn", "spike")) for M in ("sms", "sms+1", "2sms-1")]
    + [(128, 128, 128, ("randn",)), (30825, 256, 256, ("randn",)), (1000, 256, 128, ("randn",)),
       (77, 128, 384, ("randn", "tf32_edges"))]
    + [(6 * 30825, 256, 256, ("randn", "rand"))]
)
TABLE_PAIRS = {(N, K) for _, N, K, _ in SHAPES}


def _rows(M):
    """M, or the row count whose 128-row tiles number `M` of the SM count (last tile ragged: 91 rows)."""
    if isinstance(M, int):
        return M
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {"sms": sms, "sms+1": sms + 1, "2sms-1": 2 * sms - 1}[M]
    return 128 * tiles - 37


def _tf32_edges(t, g):
    """t with each element's low mantissa bits moved onto a TF32 rounding point: a third exact ties of cvt.rna (low
    13 bits 0x1000), a third rounding up across a binade (the 10 TF32 mantissa bits all ones, low bits >= 0x1000,
    one in 4096 of them also a tie), a third unchanged."""
    bits = t.view(torch.int32)
    mode = torch.randint(0, 3, t.shape, device=t.device, generator=g)
    low = torch.randint(0, 1 << 12, t.shape, device=t.device, generator=g, dtype=torch.int32)
    tie = (bits & ~0x1FFF) | 0x1000
    carry = (bits & ~0x7FFFFF) | 0x7FE000 | 0x1000 | low
    return torch.where(mode == 0, tie, torch.where(mode == 1, carry, bits)).view(torch.float32)


def _inputs(family, M, N, K, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed * 7919 + M * 31 + N * 17 + K)
    if family == "rand":                          # non-negative: no cancellation for a rounding bias to hide behind
        x, w, b = (torch.rand(*s, device=dev, generator=g) for s in ((M, K), (N, K), (N,)))
        return x, w / K ** 0.5, b
    x, w, b = (torch.randn(*s, device=dev, generator=g) for s in ((M, K), (N, K), (N,)))
    w = w / K ** 0.5
    if family == "spike":                         # one element per row 2^20 x the rest: alignment loss
        col = torch.randint(0, K, (M,), device=dev, generator=g)
        x[torch.arange(M, device=dev), col] *= 2.0 ** 20
    elif family == "tf32_edges":
        x, w = _tf32_edges(x, g), _tf32_edges(w, g)
    return x, w, b


def _abi(x, w, b, y=None, scratch=None):
    """y = x w^T + b by `vidar_linear_tf32x3` itself (any K that is a multiple of 32)."""
    from vidar_b200 import _lib
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, device=x.device) if y is None else y
    scratch = torch.empty(2 * N * K, device=x.device) if scratch is None else scratch
    _lib.check(_lib.lib().vidar_linear_tf32x3(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(y), _lib.ptr(scratch),
                                              M, N, K, _lib.stream_ptr(x.device)))
    return y


def _forward(x, w, b):
    from vidar_b200 import linear
    if linear.supported(x.shape[1], w.shape[0], x):
        return linear.linear_tf32x3(x, w, b)
    return _abi(x, w, b)


def _r(y, y64, den):
    return (y.double() - y64).abs() / den.clamp_min(torch.finfo(torch.float64).tiny)


def _stats(r):
    return r.max().item(), r.square().mean().sqrt().item()


def ratios(y, yc, y64, den):
    """(max r / cuBLAS's max r, RMS r / cuBLAS's RMS r) for `y` and the fp32 cuBLAS result `yc`."""
    (m, s), (mc, sc) = _stats(_r(y, y64, den)), _stats(_r(yc, y64, den))
    return m / mc, s / sc, (m, s, mc, sc)


def _assert_like_cublas(what, y, yc, y64, den):
    assert torch.isfinite(y).all(), f"{what}: non-finite output"
    rmax, rrms, (m, s, mc, sc) = ratios(y, yc, y64, den)
    assert rmax <= FACTOR and rrms <= FACTOR, (
        f"{what}: max r {m:.3e} ({rmax:.2f}x cuBLAS {mc:.3e}), RMS r {s:.3e} ({rrms:.2f}x cuBLAS {sc:.3e})")


def forward_ratios(family, M, N, K, dev):
    x, w, b = _inputs(family, M, N, K, dev)
    y = _forward(x, w, b)
    yc = F.linear(x, w, b)
    x64, w64, b64 = x.double(), w.double(), b.double()
    return y, yc, F.linear(x64, w64, b64), F.linear(x64.abs(), w64.abs(), b64.abs())


@pytest.fixture
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.mark.parametrize("M,N,K,families", SHAPES, ids=[f"{M}-{N}-{K}" for M, N, K, _ in SHAPES])
def test_forward_matches_fp64(cuda, no_tf32, M, N, K, families):
    """Each input family of the row with bias, and randn without bias too."""
    M = _rows(M)
    for family in families:
        _assert_like_cublas(f"{family} {M}x{N}x{K}", *forward_ratios(family, M, N, K, cuda))
    x, w, _ = _inputs("randn", M, N, K, cuda)
    x64, w64 = x.double(), w.double()
    _assert_like_cublas(f"no bias {M}x{N}x{K}", _forward(x, w, None), F.linear(x, w), F.linear(x64, w64),
                        F.linear(x64.abs(), w64.abs()))


# (batch dims, N, K): every (N, K) pair of the pre-training step whose grad_input also runs on the kernel, DCN's
# grad_cols as the grad_input of K = 9 Cin, and value_proj's size.
GRAD_SHAPES = [((3, 517), 256, 256), ((1551,), 512, 256), ((1551,), 256, 512), ((1551,), 128, 512),
               ((1551,), 256, 2304), ((1551,), 512, 4608), ((6 * 30825,), 256, 256)]


def test_gradients_match_fp64(cuda, no_tf32):
    """grad_x (the kernel with N and K swapped), grad_w and grad_b against fp64 autograd, with the forward's metric
    and bar: each denominator is the same sum of |terms| (|gy| |w|, |gy|^T |x|, sum |gy|)."""
    from vidar_b200 import linear
    for lead, N, K in GRAD_SHAPES:
        M = int(torch.tensor(lead).prod())
        x, w, b = _inputs("randn", M, N, K, cuda)
        x = x.view(*lead, K)
        gy = torch.randn(*lead, N, device=cuda, generator=torch.Generator(device=cuda).manual_seed(M + 1))
        grads = []
        for fn, dt in ((linear.linear_tf32x3, torch.float32), (F.linear, torch.float32), (F.linear, torch.float64)):
            leaves = [t.detach().to(dt).clone().requires_grad_(True) for t in (x, w, b)]
            fn(*leaves).backward(gy.to(dt))
            grads.append([t.grad.reshape(-1, t.shape[-1]) if t.dim() > 1 else t.grad for t in leaves])
        ours, cublas, ref = grads
        ga, xa, wa = gy.double().abs().reshape(M, N), x.double().abs().reshape(M, K), w.double().abs()
        dens = (ga @ wa, ga.t() @ xa, ga.sum(0))
        for name, a, c, r, den in zip(("grad_x", "grad_w", "grad_b"), ours, cublas, ref, dens):
            _assert_like_cublas(f"{name} {M}x{N}x{K}", a, c, r, den)


@pytest.mark.parametrize("M,N,K", [(191, 256, 96), (1000, 256, 2304)])
def test_power_of_two_scaling_is_exact(cuda, M, N, K):
    """Without bias, x * 2^a and w * 2^b give exactly y * 2^(a + b): every step of the split and the accumulation
    is scale-invariant while nothing leaves fp32's normal range."""
    x, w, _ = _inputs("randn", M, N, K, cuda)
    y0 = _abi(x, w, None)
    for a in (-40, 0, 40):
        for b in (-40, 0, 40):
            y = _abi(x * 2.0 ** a, w * 2.0 ** b, None)
            assert torch.equal(y, y0 * 2.0 ** (a + b)), (a, b)


@pytest.mark.parametrize("M,N,K", [(6 * 30825, 256, 256), (1000, 256, 4608)])
def test_repeated_calls_are_bitwise_identical(cuda, M, N, K):
    x, w, b = _inputs("randn", M, N, K, cuda)
    y1, y2 = _abi(x, w, b), _abi(x, w, b)
    assert torch.equal(y1.view(torch.int32), y2.view(torch.int32))


def _only_row_or_column_differs(y, clean, row=None, col=None, nonfinite=False):
    bad = torch.zeros_like(y, dtype=torch.bool)
    if row is not None:
        bad[row] = True
    if col is not None:
        bad[:, col] = True
    hit = y[bad]
    assert (~torch.isfinite(hit)).all() if nonfinite else torch.isnan(hit).all()
    assert torch.equal(y[~bad].view(torch.int32), clean[~bad].view(torch.int32))


@pytest.mark.parametrize("M,N,K", [(191, 256, 256), (300, 512, 2304)])
def test_nan_and_inf_stay_in_their_row_or_column(cuda, M, N, K):
    """A NaN in row i of x makes row i of y NaN, a NaN in row j of W column j; an inf in x makes its row non-finite
    (NaN where cuBLAS gives inf: x_lo = inf - inf).  Every other element is the clean call's, bit for bit."""
    x, w, b = _inputs("randn", M, N, K, cuda)
    clean = _abi(x, w, b)
    i, j, k = M - 5, N - 3, K // 2 + 1
    for v in (float("nan"), float("inf"), float("-inf")):
        xv = x.clone()
        xv[i, k] = v
        _only_row_or_column_differs(_abi(xv, w, b), clean, row=i, nonfinite=v == v)
    wv = w.clone()
    wv[j, k] = float("nan")
    _only_row_or_column_differs(_abi(x, wv, b), clean, col=j)


FILL = 0x7FBADBAD                                    # a NaN pattern the kernel never writes


@pytest.mark.parametrize("M", [1, 65, 191])
def test_writes_only_y_and_its_scratch(cuda, no_tf32, M):
    """y and the 2 N K split-weight scratch sit in the middle of buffers filled with a NaN pattern, a full row tile of
    N floats on either side of y: only y [M, N] and the scratch change, so no row >= M of a ragged last tile is
    stored.  x and w are not modified."""
    N, K = 256, 96
    x, w, b = _inputs("randn", M, N, K, cuda)
    x0, w0 = x.clone(), w.clone()
    pad = 128 * N
    ybuf = torch.full((pad + M * N + pad,), FILL, dtype=torch.int32, device=cuda)
    sbuf = torch.full((pad + 2 * N * K + pad,), FILL, dtype=torch.int32, device=cuda)
    y = ybuf.view(torch.float32)[pad: pad + M * N].view(M, N)
    _abi(x, w, b, y=y, scratch=sbuf.view(torch.float32)[pad: pad + 2 * N * K])
    torch.cuda.synchronize()
    for buf, n in ((ybuf, M * N), (sbuf, 2 * N * K)):
        assert (buf[:pad] == FILL).all() and (buf[pad + n:] == FILL).all()
        assert (buf[pad: pad + n] != FILL).all()
    assert torch.isfinite(y).all()
    torch.testing.assert_close(y, F.linear(x, w, b), rtol=0, atol=1e-4)
    assert torch.equal(x, x0) and torch.equal(w, w0)


def test_caller_shapes_are_in_the_table(cuda, monkeypatch):
    """A reduced pre-training step with the DCN backbone (the sizes of test_dcn_gpu's pre-training test): every
    (N, K) the wgmma kernel runs at -- attention Linears, the FFN, their grad_input, DCN's grad_cols -- is in
    SHAPES, so the accuracy table keeps covering what the callers pass."""
    from tests.test_dcn_gpu import run_reduced_pretrain_step
    from vidar_b200 import dcn, linear
    seen = set()
    gemm, dcn_gemm = linear._gemm, dcn._gemm

    def linear_gemm(x2d, weight, bias):
        if x2d.shape[0]:
            seen.add((weight.shape[0], x2d.shape[1]))
        return gemm(x2d, weight, bias)

    def dcn_gemm_rec(a, w, bias, out, scratch):
        if scratch is not None:
            seen.add((w.shape[0], a.shape[1]))
        return dcn_gemm(a, w, bias, out, scratch)

    monkeypatch.setattr(linear, "_gemm", linear_gemm)
    monkeypatch.setattr(dcn, "_gemm", dcn_gemm_rec)
    run_reduced_pretrain_step(cuda)
    assert seen, "the step ran no wgmma GEMM"
    assert seen <= TABLE_PAIRS, f"(N, K) run by the step but not in SHAPES: {sorted(seen - TABLE_PAIRS)}"


def test_rejects_unsupported_shapes(cuda):
    from vidar_b200 import linear
    with pytest.raises(RuntimeError):
        linear.linear_tf32x3(torch.randn(4, 100, device=cuda), torch.randn(128, 100, device=cuda))
