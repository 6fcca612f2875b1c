"""The wgmma 3xTF32 Linear (csrc/linear_tc.cu, SURVEY.md 8f-4) against fp64: value_proj's shape
(rows = 30825 per camera, 256 -> 256), ragged row counts (TMA clipping / guarded stores), gradients; and
through SpatialCrossAttention's value_proj.  Tolerance 2e-6 relative to max|y| (fp32 cuBLAS sits at ~1e-6,
a plain TF32 GEMM at ~5e-4)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (30825, 256, 256), (1000, 256, 128), (77, 128, 384), (1, 256, 256)])
def test_forward_matches_fp64(cuda, M, N, K):
    from vidar_b200 import linear
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    y = linear.linear_tf32x3(x.to(cuda), w.to(cuda), b.to(cuda)).cpu().double()
    ref = x.double() @ w.double().t() + b.double()
    err = (y - ref).abs().max().item()
    assert err <= 2e-6 * ref.abs().max().item(), f"max err {err:.3e} vs max|ref| {ref.abs().max().item():.3e}"
    y0 = linear.linear_tf32x3(x.to(cuda), w.to(cuda), None).cpu().double()
    assert (y0 - (ref - b.double())).abs().max().item() <= 2e-6 * ref.abs().max().item()


def test_gradients_match_fp64(cuda):
    from vidar_b200 import linear
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 517, 256, generator=g)
    w = torch.randn(256, 256, generator=g) / 16
    b = torch.randn(256, generator=g)
    gy = torch.randn(3, 517, 256, generator=g)
    xa, wa, ba = (t.to(cuda).requires_grad_(True) for t in (x, w, b))
    linear.linear_tf32x3(xa, wa, ba).backward(gy.to(cuda))
    xd, wd, bd = (t.double().requires_grad_(True) for t in (x, w, b))
    torch.nn.functional.linear(xd, wd, bd).backward(gy.double())
    for a, r, name in ((xa.grad, xd.grad, "grad_x"), (wa.grad, wd.grad, "grad_w"), (ba.grad, bd.grad, "grad_b")):
        err = (a.cpu().double() - r).abs().max().item()
        assert err <= 5e-6 * r.abs().max().item(), f"{name}: {err:.3e} vs {r.abs().max().item():.3e}"


def test_rejects_unsupported_shapes(cuda):
    from vidar_b200 import linear
    with pytest.raises(RuntimeError):
        linear.linear_tf32x3(torch.randn(4, 100, device=cuda), torch.randn(128, 100, device=cuda))
