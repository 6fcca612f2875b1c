"""The gradient bucket kernels (vidar_b200/grad_bucket.py, csrc/grad_bucket.cu) against torch: pack is bitwise
`torch.cat([g.reshape(-1) * s ...])` (zeros for a None gradient) and unpack bitwise its split, for odd numels and
bucket offsets, gradients at storage offsets that are not 16-byte aligned, zero-size tensors, more tensors than one
launch's table holds, and the real parameter list of SyntheticViDAR with the grid's scales; gradients that are not
fp32, not on the GPU or not contiguous are rejected."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TABLE = 1024         # tensors per launch (csrc/grad_bucket.cu kTable)


def _params(numels, cuda, seed, none_every=0):
    """fp32 parameters whose gradients are contiguous views at odd element offsets of one buffer (4-byte aligned
    only); every `none_every`-th has no gradient."""
    g = torch.Generator(device=cuda).manual_seed(seed)
    buf = torch.randn(sum(numels) + 3 * len(numels) + 1, generator=g, device=cuda)
    ps, at = [], 1
    for i, n in enumerate(numels):
        p = torch.nn.Parameter(torch.zeros(n, device=cuda))
        if not (none_every and i % none_every == none_every - 1):
            p.grad = buf[at: at + n]
        at += n + 1 + i % 3
        ps.append(p)
    return ps


def _expected(ps, scales):
    return torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) * s for p, s in zip(ps, scales)])


def _check_unpack(ps, cuda, seed):
    from vidar_b200 import grad_bucket
    total = sum(p.numel() for p in ps)
    bucket = torch.randn(total, generator=torch.Generator(device=cuda).manual_seed(seed), device=cuda)
    before = [None if p.grad is None else p.grad.data_ptr() for p in ps]
    grad_bucket.unpack(bucket, ps)
    off = 0
    for p, b in zip(ps, before):
        assert p.grad is not None and p.grad.shape == p.shape
        if b is not None:
            assert p.grad.data_ptr() == b                     # written in place
        assert torch.equal(p.grad.reshape(-1), bucket[off: off + p.numel()])
        off += p.numel()


def test_pack_unpack_odd_sizes_offsets_and_missing_gradients(cuda):
    from vidar_b200 import _lib, grad_bucket
    numels = [1, 3, 0, 7, 4099, 0, 5, 65537, 2, 1000003, 31, 0, 257]
    ps = _params(numels, cuda, 0, none_every=4)
    assert any(p.grad is None for p in ps) and any(p.grad is not None and p.grad.data_ptr() % 16 for p in ps)
    scales = [1.0 / 3, 0.0, 1.0, -2.5, 0.125, 7.0, 1.0 / 7, 0.5, 3.0, 1.0 / 3, -1.0, 2.0, 1e-3]
    n0 = _lib.launch_count()
    got = grad_bucket.pack(ps, scales)
    assert _lib.launch_count() - n0 == 1
    assert torch.equal(got, _expected(ps, scales))
    out = torch.full_like(got, float("nan"))
    assert grad_bucket.pack(ps, scales, out=out) is out and torch.equal(out, got)
    n0 = _lib.launch_count()
    _check_unpack(ps, cuda, 1)
    assert _lib.launch_count() - n0 == 1


def test_pack_propagates_non_finite_values_like_torch(cuda):
    from vidar_b200 import grad_bucket
    p = torch.nn.Parameter(torch.zeros(6, device=cuda))
    p.grad = torch.tensor([1.0, float("inf"), float("nan"), -float("inf"), 3e38, -0.0], device=cuda)
    for s in (0.0, 2.0, -1.0):
        assert torch.equal(grad_bucket.pack([p], [s]).isnan(), (p.grad * s).isnan())
        e = p.grad * s
        got = grad_bucket.pack([p], [s])
        assert torch.equal(got[~e.isnan()], e[~e.isnan()])


def test_more_tensors_than_one_table(cuda):
    from vidar_b200 import _lib, grad_bucket
    g = torch.Generator().manual_seed(2)
    numels = torch.randint(0, 600, (2 * TABLE + 77,), generator=g).tolist()
    ps = _params(numels, cuda, 3, none_every=9)
    scales = torch.rand(len(ps), generator=g).tolist()
    n0 = _lib.launch_count()
    got = grad_bucket.pack(ps, scales)
    assert _lib.launch_count() - n0 == 3
    assert torch.equal(got, _expected(ps, scales))
    _check_unpack(ps, cuda, 4)


def test_real_parameter_list_with_grid_scales(cuda):
    """Every trainable parameter of the full-size SyntheticViDAR (RN101 + FPN + transformer), random gradients, a few
    None, packed with the scales of a 4 x 2 grid's shard rank 0 and 1."""
    from vidar_b200 import _lib, grad_bucket, pretrain, sharding
    torch.manual_seed(0)
    model = pretrain.SyntheticViDAR().to(cuda)
    model.set_process_group(None)
    for m in (model.backbone, model.neck):
        sharding.mark_partial(m)
    ps = [p for p in model.parameters() if p.requires_grad]
    assert len(ps) > 100
    g = torch.Generator(device=cuda).manual_seed(5)
    for i, p in enumerate(ps):
        p.grad = None if i % 37 == 5 else torch.randn(p.shape, generator=g, device=cuda)
    for shard_rank in (0, 1):
        grid = sharding.Grid(None, 0, shard_rank, 4, 2, None)
        scales = sharding.grid_grad_scales(ps, grid)
        assert set(scales) == ({0.25} if shard_rank == 0 else {0.25, 0.0})
        n0 = _lib.launch_count()
        got = grad_bucket.pack(ps, scales)
        assert _lib.launch_count() - n0 == 1                  # the whole model in one launch
        assert got.numel() == sum(p.numel() for p in ps)
        assert torch.equal(got, _expected(ps, scales))
    _check_unpack(ps, cuda, 6)


def test_rejects_gradients_it_cannot_pack(cuda):
    from vidar_b200 import grad_bucket
    ok = torch.nn.Parameter(torch.zeros(4, 4, device=cuda))
    ok.grad = torch.ones(4, 4, device=cuda)
    half = torch.nn.Parameter(torch.zeros(3, device=cuda, dtype=torch.float16))
    half.grad = torch.ones(3, device=cuda, dtype=torch.float16)
    dbl = torch.nn.Parameter(torch.zeros(3, device=cuda, dtype=torch.float64))
    dbl.grad = torch.ones(3, device=cuda, dtype=torch.float64)
    cpu = torch.nn.Parameter(torch.zeros(3))
    cpu.grad = torch.ones(3)
    strided = torch.nn.Parameter(torch.zeros(4, 4, device=cuda))
    strided.grad = torch.ones(4, 4, device=cuda).t()
    assert not strided.grad.is_contiguous()
    for bad, needle in ((half, "fp32"), (dbl, "fp32"), (cpu, "fp32"), (strided, "contiguous")):
        with pytest.raises(RuntimeError, match=needle):
            grad_bucket.pack([ok, bad], [1.0, 1.0])
        with pytest.raises(RuntimeError, match=needle):
            grad_bucket.unpack(torch.zeros(16 + bad.numel(), device=cuda), [ok, bad])
    with pytest.raises(RuntimeError, match="scales"):
        grad_bucket.pack([ok], [1.0, 2.0])
    with pytest.raises(RuntimeError, match="bucket must be"):
        grad_bucket.unpack(torch.zeros(15, device=cuda), [ok])
