"""The row-map backwards against the plain ops: sca.MSDARowsFunction (rows -> BEV slots, the benchmark's MSDA
stage) against ms_deform_attn, sca.SCARowsFunction (SpatialCrossAttention's fused path) against
MSDeformAttn3DFusedFunction.

Per launch group the plain op runs on the same rows with each row's grad_out set to its pillar's slot gradient
times 1 / #cameras, and zero for rows outside the launch (dead list entries, other sub-slices).  Its gradients
are then what the row map must give; SCARowsFunction's offset / logit gradients are the per-pillar sums over
cameras."""
import pytest
import torch

from tests.inputs import SCA_LEVELS, msda_inputs
from vidar_b200 import msda, sca, synthetic

pytestmark = pytest.mark.gpu

H, C, P = 8, 32, 8


def _row_grad_out(g, inv, idx, count, group, bs, rows):
    cam0, ncl, S, lo, hi = group
    j = torch.arange(rows, device=g.device)
    n = torch.arange(bs * ncl, device=g.device)
    b, cam = n // ncl, cam0 + n % ncl
    q = idx[cam][:, :rows].long() if idx is not None else j.expand(bs * ncl, rows)
    live = ((j // 64) % S >= lo) & ((j // 64) % S < hi)
    live = live.expand(bs * ncl, rows)
    if count is not None:
        live = live & (j[None] < count[cam].long()[:, None])
    go = g[b[:, None], q]                                           # [bs*ncl, rows, H*C]
    if inv is not None:
        go = go * inv[b[:, None], q][..., None]
    return go * live[..., None]


def _check(dev, plan, bs, Qd, groups, shapes, lsi, idx=None, count=None, inv=None, seed=0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    g = torch.randn(bs, Qd, H * C, device=dev, generator=gen)
    leaves = [t.detach().clone().requires_grad_(True) for grp in groups for t in grp]
    slots = sca.MSDARowsFunction.apply(plan, bs, Qd, shapes, lsi, idx, count, inv, *leaves)
    slots.backward(g)
    for k, (group, (v, loc, aw)) in enumerate(zip(plan, groups)):
        go = _row_grad_out(g, inv, idx, count, group, bs, loc.shape[1])
        rv, rl, ra = (t.detach().clone().requires_grad_(True) for t in (v, loc, aw))
        out = msda.MultiScaleDeformableAttnFunction_fp32.apply(rv, shapes, lsi, rl, ra, 64)
        out.backward(go.reshape(out.shape))
        for name, got, want in (("grad_value", leaves[3 * k].grad, rv.grad), ("grad_loc", leaves[3 * k + 1].grad, rl.grad),
                                ("grad_attn", leaves[3 * k + 2].grad, ra.grad)):
            scale = want.abs().max().item()
            err = (got - want).abs().max().item()
            assert err <= 1e-5 * scale, f"group {k} {name}: err {err:.3e} vs max {scale:.3e}"


def _inputs(dev, n, rows, mode, seed):
    d = msda_inputs(B=n, Q=rows, H=H, C=C, levels=SCA_LEVELS, P=P, seed=seed, mode=mode)
    return d["shapes"].to(dev), d["lsi"].to(dev), tuple(d[k].to(dev) for k in ("value", "loc", "attn"))


@pytest.mark.parametrize("mode", ["local", "stress"])
def test_rows_backward_identity_rows(cuda, mode):
    """idx None: row j is pillar j; several tiles and a partial last one; 'stress' puts samples outside the image."""
    cams, Qd = 3, 1000
    shapes, lsi, grp = _inputs(cuda, cams, Qd, mode, seed=1)
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    _check(cuda, sca.unit_plan(1, 0, cams), 1, Qd, [grp], shapes, lsi, inv=inv)


def test_rows_backward_shuffled_idx_count(cuda):
    """A shuffled visible-pillar list per camera with fewer live entries than rows, two batch elements and two
    launch groups (the second starts at camera 2)."""
    cams, bs, Qd = 3, 2, 900
    gen = torch.Generator().manual_seed(3)
    idx = torch.stack([torch.randperm(Qd, generator=gen) for _ in range(cams)]).int().to(cuda)
    count = torch.tensor([700, 333, 0], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (bs, Qd), device=cuda).float()).contiguous()
    plan = [(0, 2, 1, 0, 1), (2, 1, 1, 0, 1)]
    shapes, lsi, g0 = _inputs(cuda, bs * 2, Qd, "local", seed=4)
    _, _, g1 = _inputs(cuda, bs * 1, Qd, "stress", seed=5)
    _check(cuda, plan, bs, Qd, [g0, g1], shapes, lsi, idx=idx, count=count, inv=inv)


def test_rows_backward_sub_slices(cuda):
    """S = 4 interleaved sub-slices of 64 rows, this launch owning [1, 3), with a shuffled list and a count."""
    cams, Qd = 2, 1100
    gen = torch.Generator().manual_seed(6)
    idx = torch.stack([torch.randperm(Qd, generator=gen) for _ in range(cams)]).int().to(cuda)
    count = torch.tensor([1050, 600], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    shapes, lsi, grp = _inputs(cuda, cams, Qd, "local", seed=7)
    _check(cuda, [(0, cams, 4, 1, 3)], 1, Qd, [grp], shapes, lsi, idx=idx, count=count, inv=inv)


def test_rows_backward_bench_size(cuda):
    """The benchmark's shape: 6 cameras x 40 000 rows of SpatialCrossAttention-like sampling locations."""
    d = synthetic.sca_like_inputs(cuda, cams=6, Q=40000, seed=0)
    Qd = 40000
    inv = torch.full((1, Qd), 1.0 / 3.0, device=cuda)
    _check(cuda, sca.unit_plan(1, 0, 6), 1, Qd, [(d["value"], d["loc"], d["attn"])], d["shapes"], d["lsi"], inv=inv)


def _check_sca(dev, cams, Qd, plan, idx=None, count=None, inv=None, seed=0, D=4):
    d = msda_inputs(B=cams, Q=1, H=H, C=C, levels=SCA_LEVELS, P=P, seed=seed)
    shapes, lsi, value = d["shapes"].to(dev), d["lsi"].to(dev), d["value"].to(dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    L = len(SCA_LEVELS)
    ref_cam = torch.rand(cams, 1, Qd, D, 2, device=dev, generator=gen) * 1.2 - 0.1    # some anchors off the image
    offsets = 4.0 * torch.randn(1, Qd, H, L, P, 2, device=dev, generator=gen)
    logits = torch.randn(1, Qd, H, L * P, device=dev, generator=gen)
    g = torch.randn(1, Qd, H * C, device=dev, generator=gen)
    leaves = [t.detach().clone().requires_grad_(True) for t in (offsets, logits)]
    values = [value[cam0:cam0 + ncl].detach().clone().requires_grad_(True) for cam0, ncl, *_ in plan]
    slots = sca.SCARowsFunction.apply(plan, 1, shapes, lsi, ref_cam, *leaves, idx, count, inv, *values)
    slots.backward(g)
    want_off, want_log = torch.zeros_like(offsets), torch.zeros_like(logits)
    for k, group in enumerate(plan):
        cam0, ncl = group[0], group[1]
        go = _row_grad_out(g, inv, idx, count, group, 1, Qd)
        cam = torch.arange(cam0, cam0 + ncl, device=dev)
        q = idx[cam].long() if idx is not None else torch.arange(Qd, device=dev).expand(ncl, Qd)
        rv = value[cam0:cam0 + ncl].detach().clone().requires_grad_(True)
        ro = offsets[0][q].detach().clone().requires_grad_(True)
        rl = logits[0][q].detach().clone().requires_grad_(True)
        out = msda.MSDeformAttn3DFusedFunction.apply(rv, shapes, lsi, ref_cam[cam, 0][torch.arange(ncl, device=dev)[:, None], q],
                                                      ro, rl)
        out.backward(go.reshape(out.shape))
        want_off[0].index_add_(0, q.reshape(-1), ro.grad.reshape(-1, *ro.shape[2:]))
        want_log[0].index_add_(0, q.reshape(-1), rl.grad.reshape(-1, *rl.shape[2:]))
        _close(f"group {k} grad_value", values[k].grad, rv.grad)
    _close("grad_offsets", leaves[0].grad, want_off)
    _close("grad_logits", leaves[1].grad, want_log)


def _close(name, got, want):
    scale = want.abs().max().item()
    err = (got - want).abs().max().item()
    assert err <= 1e-5 * scale, f"{name}: err {err:.3e} vs max {scale:.3e}"


def test_sca_rows_backward_identity_rows(cuda):
    """SCARowsFunction, idx None: row j is pillar j; several tiles and a partial last one."""
    cams, Qd = 3, 1000
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    _check_sca(cuda, cams, Qd, sca.unit_plan(1, 0, cams), inv=inv, seed=11)


def test_sca_rows_backward_shuffled_idx_sub_slices(cuda):
    """SCARowsFunction with shuffled lists, counts below the row count, S = 4 sub-slices and two launch groups."""
    cams, Qd = 3, 1100
    gen = torch.Generator().manual_seed(12)
    idx = torch.stack([torch.randperm(Qd, generator=gen) for _ in range(cams)]).int().to(cuda)
    count = torch.tensor([1050, 600, 333], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    _check_sca(cuda, cams, Qd, [(0, 2, 4, 1, 3), (2, 1, 4, 0, 4)], idx=idx, count=count, inv=inv, seed=13)


def test_sca_rows_backward_bench_size(cuda):
    """SCARowsFunction at SpatialCrossAttention's size: 6 cameras x 40 000 pillars."""
    inv = torch.full((1, 40000), 1.0 / 3.0, device=cuda)
    _check_sca(cuda, 6, 40000, sca.unit_plan(1, 0, 6), inv=inv, seed=14)
