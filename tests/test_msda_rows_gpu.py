"""The row-map entry points (SpatialCrossAttention's rebatch + scatter-add inside the op) against the fp64 oracle:
sca.MSDARowsFunction (rows -> BEV slots, the benchmark's MSDA stage) against oracle/msda_ref.msda_rows,
sca.SCARowsFunction (SpatialCrossAttention's fused path) against msda_ref.msda_sca_rows.  The slots and every
gradient are held to tests/parity.py; grad_sampling_loc / grad_offsets skip samples on a pixel-centre line.

They are also compared with the plain ops at 1e-5 (tighter than parity, shared arithmetic; where the rows take the
tile kernel, grad_sampling_loc / grad_attn_weight must be bit-identical): per launch group
`ms_deform_attn` / MSDeformAttn3DFusedFunction runs on the same rows with each row's grad_out set to its pillar's
slot gradient times 1 / #cameras, and zero for rows outside the launch (dead list entries, other sub-slices).

The cases reach every backward branch of vidar_msda_rows_backward / vidar_msda_sca_rows_backward: the tile kernel
(C = 32, 8 points on 4 levels, K < 2^19) and msda_backward_kernel<CV, .., IDX> otherwise (C = 16 / 64, other L*P,
K >= 2^19), with the forward at all three head widths."""
import pytest
import torch

from oracle import msda_ref
from tests import parity
from tests.inputs import SCA_LEVELS, level_tensors, msda_inputs
from vidar_b200 import _lib, msda, sca, synthetic

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


def _parts(bs, ncl, per_camera, dev):
    """(first camera, cameras, batch elements n = b*ncl + camera) of a launch group, whole or one camera at a time"""
    spans = [(cl, 1) for cl in range(ncl)] if per_camera else [(0, ncl)]
    return [(cl0, m, torch.tensor([b * ncl + cl for b in range(bs) for cl in range(cl0, cl0 + m)], device=dev))
            for cl0, m in spans]


def _oracle_rows(plan, bs, Qd, shapes, idx, count, inv, groups, g, per_camera=False):
    """fp64 slots and per-group (value, loc, attn) gradients of msda_ref.msda_rows on the device.  per_camera: one
    camera at a time (at 6 x 40 000 rows grid_sample's fp64 intermediates are several GB per level)."""
    slots = torch.zeros(g.shape, dtype=torch.float64, device=g.device)
    grads = []
    for (cam0, ncl, S, lo, hi), grp in zip(plan, groups):
        acc = [torch.zeros(t.shape, dtype=torch.float64, device=g.device) for t in grp]
        for cl0, m, sel in _parts(bs, ncl, per_camera, g.device):
            leaves = [t[sel].double().requires_grad_(True) for t in grp]
            s = msda_ref.msda_rows([(cam0 + cl0, m, S, lo, hi)], bs, Qd, shapes, idx, count, inv, [leaves])
            s.backward(g.double())
            slots += s.detach()
            for a, t in zip(acc, leaves):
                a[sel] = t.grad
            del s, leaves
        grads.append(acc)
    return slots, grads


def _close_rows(got_slots, got_grads, ref, shapes, oracle_groups, tag=""):
    rslots, rgrads = ref
    parity.close(got_slots, rslots, f"{tag}slots")
    for k, ((gv, gl, ga), (rv, rl, ra), grp) in enumerate(zip(got_grads, rgrads, oracle_groups)):
        parity.close(gv, rv, f"{tag}group {k} grad_value")
        keep = parity.off_kink(grp[1], shapes.cpu())
        parity.close(gl, rl, f"{tag}group {k} grad_sampling_loc", keep=keep.unsqueeze(-1).expand(rl.shape))
        parity.close(ga, ra, f"{tag}group {k} grad_attn_weight")


def _check(dev, plan, bs, Qd, groups, shapes, lsi, idx=None, count=None, inv=None, seed=0, oracle_groups=None,
           per_camera=False, plain=True):
    """Forward + backward of MSDARowsFunction against the oracle (on `oracle_groups` when given: NaN locations
    there become far-outside ones) and, with `plain`, against ms_deform_attn at 1e-5."""
    HC = groups[0][0].shape[2] * groups[0][0].shape[3]
    gen = torch.Generator(device=dev).manual_seed(seed)
    g = torch.randn(bs, Qd, HC, device=dev, generator=gen)
    leaves = [t.detach().clone().requires_grad_(True) for grp in groups for t in grp]
    slots = sca.MSDARowsFunction.apply(plan, bs, Qd, shapes, lsi, idx, count, inv, *leaves)
    slots.backward(g)
    got = [tuple(t.grad for t in leaves[3 * k:3 * k + 3]) for k in range(len(plan))]
    oracle_groups = groups if oracle_groups is None else oracle_groups
    ref = _oracle_rows(plan, bs, Qd, shapes, idx, count, inv, oracle_groups, g, per_camera)
    _close_rows(slots, got, ref, shapes, oracle_groups)
    del ref
    if not plain:
        return
    for k, (group, (v, loc, aw)) in enumerate(zip(plan, groups)):
        go = _row_grad_out(g, inv, idx, count, group, bs, loc.shape[1])
        rv, rl, ra = (t.detach().clone().requires_grad_(True) for t in (v, loc, aw))
        out = msda.MultiScaleDeformableAttnFunction_fp32.apply(rv, shapes, lsi, rl, ra, 64)
        out.backward(go.reshape(out.shape))
        # the tile kernel's location / attention gradients are msda_backward_kernel's arithmetic: bit-identical.
        # `tile` restates tile_backward_ok in csrc/msda.cu, which picks the tile kernel; keep the two in step.
        K, C_, L, P_ = v.shape[1], v.shape[3], loc.shape[3], loc.shape[4]
        tile = C_ == 32 and P_ == 8 and L * P_ == 32 and K < 2 ** 19
        for name, got_, want in (("grad_value", got[k][0], rv.grad), ("grad_loc", got[k][1], rl.grad),
                                 ("grad_attn", got[k][2], ra.grad)):
            if tile and name != "grad_value":
                assert torch.equal(got_, want), f"group {k} {name}: tile kernel differs from ms_deform_attn"
            else:
                _close(f"group {k} {name}", got_, want)


def _inputs(dev, n, rows, mode, seed, levels=SCA_LEVELS, heads=H, dim=C, points=P):
    d = msda_inputs(B=n, Q=rows, H=heads, C=dim, levels=levels, P=points, seed=seed, mode=mode)
    return d["shapes"].to(dev), d["lsi"].to(dev), tuple(d[k].to(dev) for k in ("value", "loc", "attn"))


def _lists(dev, cams, Qd, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(Qd, generator=gen) for _ in range(cams)]).int().to(dev)


def _inv(dev, bs, Qd, seed):
    gen = torch.Generator().manual_seed(seed)
    return (1.0 / torch.randint(1, 4, (bs, Qd), generator=gen).float()).to(dev).contiguous()


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
    idx = _lists(cuda, cams, Qd, 3)
    count = torch.tensor([700, 333, 0], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (bs, Qd), device=cuda).float()).contiguous()
    plan = [(0, 2, 1, 0, 1), (2, 1, 1, 0, 1)]
    shapes, lsi, g0 = _inputs(cuda, bs * 2, Qd, "local", seed=4)
    _, _, g1 = _inputs(cuda, bs * 1, Qd, "stress", seed=5)
    _check(cuda, plan, bs, Qd, [g0, g1], shapes, lsi, idx=idx, count=count, inv=inv)


def test_rows_backward_sub_slices(cuda):
    """S = 4 interleaved sub-slices of 64 rows, this launch owning [1, 3), with a shuffled list and a count."""
    cams, Qd = 2, 1100
    idx = _lists(cuda, cams, Qd, 6)
    count = torch.tensor([1050, 600], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    shapes, lsi, grp = _inputs(cuda, cams, Qd, "local", seed=7)
    _check(cuda, [(0, cams, 4, 1, 3)], 1, Qd, [grp], shapes, lsi, idx=idx, count=count, inv=inv)


def test_rows_backward_full_tiles(cuda):
    """Live lists of exactly one and two 256-row tiles, and of a single row."""
    cams, Qd = 3, 700
    idx = _lists(cuda, cams, Qd, 8)
    count = torch.tensor([256, 512, 1], dtype=torch.int32, device=cuda)
    shapes, lsi, grp = _inputs(cuda, cams, Qd, "local", seed=9)
    _check(cuda, sca.unit_plan(1, 0, cams), 1, Qd, [grp], shapes, lsi, idx=idx, count=count, inv=_inv(cuda, 1, Qd, 9))


def test_rows_backward_bench_size(cuda):
    """The benchmark's shape: 6 cameras x 40 000 rows of SpatialCrossAttention-like sampling locations."""
    d = synthetic.sca_like_inputs(cuda, cams=6, Q=40000, seed=0)
    Qd = 40000
    inv = torch.full((1, Qd), 1.0 / 3.0, device=cuda)
    _check(cuda, sca.unit_plan(1, 0, 6), 1, Qd, [(d["value"], d["loc"], d["attn"])], d["shapes"], d["lsi"], inv=inv,
           per_camera=True)


# msda_backward_kernel<CV, false, false, true> (and the forward at every CV): shapes the tile kernel does not take
FALLBACK = {
    # name: (cams, bs, Qd, heads, dim, levels, points, shuffled list + count, plan)
    "C16": (2, 2, 600, 8, 16, SCA_LEVELS, 8, True, [(0, 2, 4, 1, 4)]),
    "C64": (3, 1, 500, 4, 64, SCA_LEVELS, 8, False, None),
    "LP4": (2, 2, 700, 8, 32, ((50, 50),), 4, True, [(0, 1, 2, 0, 1), (1, 1, 1, 0, 1)]),
    "LP40": (2, 1, 300, 8, 32, ((24, 40), (12, 20), (6, 10), (3, 5), (1, 1)), 8, False, None),
}


@pytest.mark.parametrize("case", list(FALLBACK))
def test_rows_fallback_kernels(cuda, case):
    cams, bs, Qd, heads, dim, levels, points, listed, plan = FALLBACK[case]
    plan = plan or sca.unit_plan(1, 0, cams)
    idx = _lists(cuda, cams, Qd, 20) if listed else None
    count = torch.tensor([Qd - 37 - 150 * c for c in range(cams)], dtype=torch.int32, device=cuda) if listed else None
    groups = []
    for k, (_, ncl, *_) in enumerate(plan):
        shapes, lsi, grp = _inputs(cuda, bs * ncl, Qd, ("local", "stress")[k % 2], 21 + k, levels, heads, dim, points)
        groups.append(grp)
    _check(cuda, plan, bs, Qd, groups, shapes, lsi, idx=idx, count=count, inv=_inv(cuda, bs, Qd, 22))


# The tile kernel's sort key holds a level pixel (pb = bit length of H_l * W_l) above 13 record bits.  With one head
# of 32 channels K * H * C stays below the vector kernels' 2^25 float-offset limit at these sizes.
EDGES = {
    "pixel-bits-19-tile": ((724, 724), (8, 8), (4, 4), (2, 2)),      # K = 524 260 < 2^19: 32-bit keys
    "K-2^19-fallback": ((725, 725), (8, 8), (4, 4), (2, 2)),         # K = 525 709: the same rows on the fallback
    "sentinel-tile": ((16, 16), (8, 8), (1, 1), (4, 2)),             # powers of two and a 1 x 1 level
}


@pytest.mark.parametrize("case", list(EDGES))
def test_rows_level_size_edges(cuda, case):
    levels = EDGES[case]
    heads = 8 if case.startswith("sentinel") else 1
    Qd = 600
    shapes, lsi, (value, loc, attn) = _inputs(cuda, 1 if heads == 1 else 2, Qd, "local" if heads == 1 else "stress", 30,
                                              levels, heads)
    # At 724 px the fp32 pixel coordinate loc * W - 0.5 has an ulp of 6e-5 px, which alone moves outputs past parity.
    # On a 2^-14 grid it is exact, so what is compared is the kernels' arithmetic, not input rounding.
    grp = (value, torch.round(loc * 16384) / 16384, attn)
    _check(cuda, sca.unit_plan(1, 0, grp[0].shape[0]), 1, Qd, [grp], shapes, lsi, inv=_inv(cuda, 1, Qd, 31))


def test_rows_long_pixel_runs(cuda):
    """Every row of two tiles samples the same 2 x 2 pixels of each level (+-0.3 px): a pixel's run of records spans
    many 128-record group segments.  Every fifth row sits exactly on a pixel centre."""
    cams, Qd = 2, 512
    shapes, lsi, (value, _, attn) = _inputs(cuda, cams, Qd, "local", seed=40)
    gen = torch.Generator().manual_seed(41)
    wh = torch.tensor([[w, h] for h, w in SCA_LEVELS], dtype=torch.float64).view(1, 1, 1, 4, 1, 2)
    corner = torch.floor(wh / 2) - 0.5                                    # pixel coordinate between 4 pixel centres
    px = corner + 0.6 * torch.rand(cams, Qd, H, 4, P, 2, generator=gen, dtype=torch.float64) - 0.3
    px[:, ::5] = torch.floor(corner + 0.5).expand(cams, Qd, H, 4, P, 2)[:, ::5]     # on a pixel centre
    loc = ((px + 0.5) / wh).float().to(cuda)
    _check(cuda, sca.unit_plan(1, 0, cams), 1, Qd, [(value, loc, attn)], shapes, lsi, inv=_inv(cuda, 1, Qd, 42))


@pytest.mark.parametrize("dim", [32, 16], ids=["tile", "fallback"])
def test_rows_nan_and_outside_rows(cuda, dim):
    """Rows whose head-0 locations are NaN (they decide the row's image cell) contribute nothing on head 0; rows
    entirely outside the image contribute nothing.  The oracle gets the NaN locations as far-outside ones."""
    cams, Qd = 2, 700
    shapes, lsi, (value, loc, attn) = _inputs(cuda, cams, Qd, "local", seed=50, dim=dim)
    loc = loc.clone()
    loc[:, ::7, 0] = float("nan")
    loc[:, 3::11] = -3.0
    loc[1, 5::13] = 1e30
    far = torch.where(torch.isnan(loc) | (loc.abs() > 100), 37.5, loc)    # grid_sample wants finite, moderate grids
    _check(cuda, sca.unit_plan(1, 0, cams), 1, Qd, [(value, loc, attn)], shapes, lsi, inv=_inv(cuda, 1, Qd, 51),
           oracle_groups=[(value, far, attn)])


def _sca_inputs(dev, cams, bs, Qd, seed, D=4, heads=H, dim=C, levels=SCA_LEVELS, points=P):
    d = msda_inputs(B=bs * cams, Q=1, H=heads, C=dim, levels=levels, P=points, seed=seed)
    shapes, lsi = d["shapes"].to(dev), d["lsi"].to(dev)
    value = d["value"].to(dev).view(bs, cams, *d["value"].shape[1:])            # [bs, cams, K, H, C]
    gen = torch.Generator(device=dev).manual_seed(seed)
    L = len(levels)
    ref_cam = torch.rand(cams, bs, Qd, D, 2, device=dev, generator=gen) * 1.2 - 0.1    # some anchors off the image
    offsets = 4.0 * torch.randn(bs, Qd, heads, L, points, 2, device=dev, generator=gen)
    logits = torch.randn(bs, Qd, heads, L * points, device=dev, generator=gen)
    g = torch.randn(bs, Qd, heads * dim, device=dev, generator=gen)
    return shapes, lsi, value, ref_cam, offsets, logits, g


def _group_values(value, plan):
    bs = value.shape[0]
    return [value[:, cam0:cam0 + ncl].reshape(bs * ncl, *value.shape[2:]).contiguous() for cam0, ncl, *_ in plan]


def _oracle_sca(plan, bs, shapes, idx, count, inv, ref_cam, offsets, logits, values, g, per_camera=False):
    """fp64 slots, grad_offsets, grad_logits and per-group grad_value of msda_ref.msda_sca_rows on the device."""
    off = offsets.double().requires_grad_(True)
    lg = logits.double().requires_grad_(True)
    slots = torch.zeros(g.shape, dtype=torch.float64, device=g.device)
    gvs = []
    for (cam0, ncl, S, lo, hi), v in zip(plan, values):
        gv = torch.zeros(v.shape, dtype=torch.float64, device=g.device)
        for cl0, m, sel in _parts(bs, ncl, per_camera, g.device):
            vl = v[sel].double().requires_grad_(True)
            s = msda_ref.msda_sca_rows([(cam0 + cl0, m, S, lo, hi)], bs, shapes, idx, count, inv, ref_cam, off, lg, [vl])
            s.backward(g.double())
            slots += s.detach()
            gv[sel] = vl.grad
            del s, vl
        gvs.append(gv)
    return slots, off.grad, lg.grad, gvs


def _offsets_keep(plan, bs, shapes, idx, ref_cam, offsets):
    """[bs, Qd, H, L, P] bool: the pillar's sample is off every pixel-centre line in every camera's row of it."""
    Qd = offsets.shape[1]
    bad = torch.zeros(offsets.shape[:-1], dtype=torch.int32)
    for cam0, ncl, *_ in plan:
        n = torch.arange(bs * ncl, device=offsets.device)
        b, cam = n // ncl, cam0 + n % ncl
        q = idx[cam].long() if idx is not None else torch.arange(Qd, device=offsets.device).expand(bs * ncl, Qd)
        bb = b[:, None].expand_as(q)
        loc = msda_ref.sca_locations(shapes, offsets[bb, q], ref_cam[cam[:, None], bb, q])
        ok = parity.off_kink(loc, shapes.cpu())
        bad.index_put_((bb.cpu(), q.cpu()), (~ok).int(), accumulate=True)
    return bad == 0


def _check_sca(dev, cams, Qd, plan, idx=None, count=None, inv=None, seed=0, D=4, bs=1, heads=H, dim=C,
               levels=SCA_LEVELS, points=P, per_camera=False):
    shapes, lsi, value, ref_cam, offsets, logits, g = _sca_inputs(dev, cams, bs, Qd, seed, D, heads, dim, levels, points)
    gvalues = _group_values(value, plan)
    leaves = [t.detach().clone().requires_grad_(True) for t in (offsets, logits)]
    values = [v.detach().clone().requires_grad_(True) for v in gvalues]
    slots = sca.SCARowsFunction.apply(plan, bs, shapes, lsi, ref_cam, *leaves, idx, count, inv, *values)
    slots.backward(g)

    # against the oracle
    rslots, roff, rlog, rgvs = _oracle_sca(plan, bs, shapes, idx, count, inv, ref_cam, offsets, logits, gvalues, g,
                                           per_camera)
    parity.close(slots, rslots, "slots")
    for k, (v, rv) in enumerate(zip(values, rgvs)):
        parity.close(v.grad, rv, f"group {k} grad_value")
    keep = _offsets_keep(plan, bs, shapes, idx, ref_cam, offsets)
    parity.close(leaves[0].grad, roff, "grad_offsets", keep=keep.unsqueeze(-1).expand(roff.shape))
    parity.close(leaves[1].grad, rlog, "grad_logits")
    del rslots, roff, rlog, rgvs

    # against the fused plain op on the same rows
    want_off, want_log = torch.zeros_like(offsets), torch.zeros_like(logits)
    for k, group in enumerate(plan):
        cam0, ncl = group[0], group[1]
        go = _row_grad_out(g, inv, idx, count, group, bs, Qd)
        n = torch.arange(bs * ncl, device=dev)
        b, cam = n // ncl, cam0 + n % ncl
        q = idx[cam].long() if idx is not None else torch.arange(Qd, device=dev).expand(bs * ncl, Qd)
        bb = b[:, None].expand_as(q)
        rv = gvalues[k].detach().clone().requires_grad_(True)
        ro = offsets[bb, q].detach().clone().requires_grad_(True)
        rl = logits[bb, q].detach().clone().requires_grad_(True)
        out = msda.MSDeformAttn3DFusedFunction.apply(rv, shapes, lsi, ref_cam[cam[:, None], bb, q], ro, rl)
        out.backward(go.reshape(out.shape))
        want_off.index_put_((bb, q), ro.grad, accumulate=True)
        want_log.index_put_((bb, q), rl.grad, accumulate=True)
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
    idx = _lists(cuda, cams, Qd, 12)
    count = torch.tensor([1050, 600, 333], dtype=torch.int32, device=cuda)
    inv = (1.0 / torch.randint(1, 4, (1, Qd), device=cuda).float()).contiguous()
    _check_sca(cuda, cams, Qd, [(0, 2, 4, 1, 3), (2, 1, 4, 0, 4)], idx=idx, count=count, inv=inv, seed=13)


def test_sca_rows_backward_two_batch_elements(cuda):
    """bs = 2 above one tile per batch element: shuffled lists, counts and S = 4 sub-slices."""
    cams, bs, Qd = 3, 2, 1100
    idx = _lists(cuda, cams, Qd, 15)
    count = torch.tensor([1100, 777, 290], dtype=torch.int32, device=cuda)
    _check_sca(cuda, cams, Qd, [(0, 3, 4, 1, 4)], idx=idx, count=count, inv=_inv(cuda, bs, Qd, 15), seed=16, bs=bs)


def test_sca_rows_backward_bench_size(cuda):
    """SCARowsFunction at SpatialCrossAttention's size: 6 cameras x 40 000 pillars."""
    inv = torch.full((1, 40000), 1.0 / 3.0, device=cuda)
    _check_sca(cuda, 6, 40000, sca.unit_plan(1, 0, 6), inv=inv, seed=14, per_camera=True)


# msda_backward_kernel<CV, false, true, true>: head widths other than 32, and 2 levels x 16 points at 32
SCA_FALLBACK = {
    # name: (heads, dim, levels, points, bs, shuffled list + count + S = 4)
    "C16": (8, 16, SCA_LEVELS, 8, 1, False),
    "C64": (4, 64, SCA_LEVELS, 8, 2, True),
    "L2P16": (8, 32, ((58, 100), (15, 25)), 16, 1, True),
}


@pytest.mark.parametrize("case", list(SCA_FALLBACK))
def test_sca_rows_fallback_kernels(cuda, case):
    heads, dim, levels, points, bs, listed = SCA_FALLBACK[case]
    cams, Qd = 3, 600
    idx = _lists(cuda, cams, Qd, 60) if listed else None
    count = torch.tensor([600, 411, 0], dtype=torch.int32, device=cuda) if listed else None
    plan = [(0, 2, 4, 0, 3), (2, 1, 4, 1, 4)] if listed else sca.unit_plan(1, 0, cams)
    _check_sca(cuda, cams, Qd, plan, idx=idx, count=count, inv=_inv(cuda, bs, Qd, 61), seed=62, bs=bs, heads=heads,
               dim=dim, levels=levels, points=points)


# ---- the C ABI: grad_sampling_loc / grad_attn_weight are written for the rows of the launch, nothing else ----------
NAN_BITS = 0x7FC00123          # a quiet NaN with a payload the kernels cannot produce


@pytest.mark.parametrize("dim", [32, 16], ids=["tile", "fallback"])
def test_rows_backward_c_abi_writes_only_live_rows(cuda, dim):
    cams, Qd = 2, 600
    shapes, lsi, (value, loc, attn) = _inputs(cuda, cams, Qd, "local", seed=70, dim=dim)
    idx = _lists(cuda, cams, Qd, 71)
    count = torch.tensor([555, 300], dtype=torch.int32, device=cuda)
    inv = _inv(cuda, 1, Qd, 72)
    g = torch.randn(1, Qd, H * dim, device=cuda, generator=torch.Generator(device=cuda).manual_seed(73))
    L, Pt = loc.shape[3], loc.shape[4]
    K = value.shape[1]
    j = torch.arange(Qd, device=cuda)
    for plan, lidx, lcount in (((0, cams, 4, 1, 3), idx, count), ((0, cams, 1, 0, 1), None, None)):
        cam0, ncl, S, lo, hi = plan
        gv = torch.zeros_like(value)
        gl = torch.full(loc.shape, NAN_BITS, dtype=torch.int32, device=cuda).view(torch.float32)
        ga = torch.full(attn.shape, NAN_BITS, dtype=torch.int32, device=cuda).view(torch.float32)
        P_ = _lib.ptr
        _lib.check(_lib.lib().vidar_msda_rows_backward(
            P_(value), P_(shapes), P_(lsi), P_(loc), P_(attn), P_(lidx), P_(lcount), P_(inv), P_(g), P_(gv), P_(gl),
            P_(ga), 1, ncl, cam0, K, H, dim, L, Qd, Qd, Pt, S, lo, hi, _lib.stream_ptr(cuda)))
        live = (((j // 64) % S >= lo) & ((j // 64) % S < hi)).expand(cams, Qd)
        if lcount is not None:
            live = live & (j[None] < lcount.long()[:, None])
        assert bool((~live).any()) == (lcount is not None)
        for name, t in (("grad_sampling_loc", gl), ("grad_attn_weight", ga)):
            bits = t.view(torch.int32)[~live]
            assert bool((bits == NAN_BITS).all()), f"{name}: a row outside the launch was written"
            assert bool(torch.isfinite(t[live]).all()), f"{name}: a live row was not written"
        _, rgrads = _oracle_rows([plan], 1, Qd, shapes, lidx, lcount, inv, [(value, loc, attn)], g)
        rv, rl, ra = rgrads[0]
        parity.close(gv, rv, "grad_value")
        keep = parity.off_kink(loc, shapes.cpu()) & live.cpu()[..., None, None, None]
        parity.close(gl, rl, "grad_sampling_loc", keep=keep.unsqueeze(-1).expand(rl.shape))
        parity.close(ga, ra, "grad_attn_weight", keep=live.cpu()[..., None, None, None].expand(ra.shape))


# ---- the execution contexts of bench.py: CUDA-graph replay, side streams, scratch pool reuse ---------------------
def _bench_rows_case(dev, seed):
    d = synthetic.sca_like_inputs(dev, cams=6, Q=40000, seed=seed)
    return d["shapes"], d["lsi"], [d["value"], d["loc"], d["attn"]]


@pytest.mark.parametrize("fn", ["msda_rows", "sca_rows"])
def test_rows_cuda_graph_replay(cuda, fn):
    """Forward + backward captured as bench.py captures its step (warm-up on a side stream, leaves created inside the
    capture), at the benchmark shape.  Replays equal the eager run; after new inputs are copied into the captured
    tensors a replay matches the oracle on them (the row order is recomputed from the data, not baked in)."""
    plan, Qd = sca.unit_plan(1, 0, 6), 40000
    inv = _inv(cuda, 1, Qd, 80)
    g = torch.randn(1, Qd, H * C, device=cuda, generator=torch.Generator(device=cuda).manual_seed(81))
    if fn == "msda_rows":
        shapes, lsi, static = _bench_rows_case(cuda, 0)

        def step():
            leaves = [t.detach().requires_grad_(True) for t in static]
            slots = sca.MSDARowsFunction.apply(plan, 1, Qd, shapes, lsi, None, None, inv, *leaves)
            slots.backward(g)
            return [slots.detach()] + [t.grad for t in leaves]
        exact = (2, 3)                       # grad_sampling_loc, grad_attn_weight: plain stores
    else:
        shapes, lsi, value, ref_cam, offsets, logits, _ = _sca_inputs(cuda, 6, 1, Qd, 82)
        static = [_group_values(value, plan)[0], ref_cam, offsets, logits]

        def step():
            v, o, lg = (t.detach().requires_grad_(True) for t in (static[0], static[2], static[3]))
            slots = sca.SCARowsFunction.apply(plan, 1, shapes, lsi, static[1], o, lg, None, None, inv, v)
            slots.backward(g)
            return [slots.detach(), v.grad, o.grad, lg.grad]
        exact = ()                           # offset / logit gradients are reduced over cameras
    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream(device=cuda)
    side.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(cuda).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for r in range(3):
        for t in outs:
            t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for k, (a, b) in enumerate(zip(outs, eager)):
            if k in exact:
                assert torch.equal(a, b), f"replay {r}: output {k} differs from the eager run"
            else:
                parity.close(a, b, f"replay {r}: output {k}")
    # new data in the captured inputs
    if fn == "msda_rows":
        _, _, new = _bench_rows_case(cuda, 5)
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        ref = _oracle_rows(plan, 1, Qd, shapes, None, None, inv, [static], g, per_camera=True)
        _close_rows(outs[0], [outs[1:]], ref, shapes, [static], tag="new inputs: ")
    else:
        _, _, value2, ref2, off2, log2, _ = _sca_inputs(cuda, 6, 1, Qd, 83)
        for t, n in zip(static, (_group_values(value2, plan)[0], ref2, off2, log2)):
            t.copy_(n)
        graph.replay()
        rslots, roff, rlog, rgvs = _oracle_sca(plan, 1, shapes, None, None, inv, static[1], static[2], static[3],
                                               [static[0]], g, per_camera=True)
        parity.close(outs[0], rslots, "new inputs: slots")
        parity.close(outs[1], rgvs[0], "new inputs: grad_value")
        keep = _offsets_keep(plan, 1, shapes, None, static[1], static[2])
        parity.close(outs[2], roff, "new inputs: grad_offsets", keep=keep.unsqueeze(-1).expand(roff.shape))
        parity.close(outs[3], rlog, "new inputs: grad_logits")


def test_rows_on_side_stream(cuda):
    """Forward + backward of both functions issued on a non-default stream."""
    cams, Qd = 3, 900
    shapes, lsi, grp = _inputs(cuda, cams, Qd, "local", seed=90)
    idx, count = _lists(cuda, cams, Qd, 91), torch.tensor([900, 500, 260], dtype=torch.int32, device=cuda)
    s = torch.cuda.Stream(device=cuda)
    s.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(s):
        _check(cuda, [(0, cams, 2, 0, 2)], 1, Qd, [grp], shapes, lsi, idx=idx, count=count, inv=_inv(cuda, 1, Qd, 92),
               plain=False)
        _check_sca(cuda, cams, Qd, [(0, cams, 1, 0, 1)], idx=idx, count=count, inv=_inv(cuda, 1, Qd, 93), seed=94)
    torch.cuda.current_stream(cuda).wait_stream(s)
    torch.cuda.synchronize()


def test_rows_backward_scratch_reuse(cuda):
    """Backward calls back to back at 1000, 40 000 and 1000 rows: the row order's scratch comes from the pool,
    grows, and is reused; each call matches its oracle."""
    cams = 2
    runs = []
    for k, Qd in enumerate((1000, 40000, 1000)):
        shapes, lsi, grp = _inputs(cuda, cams, Qd, "local", seed=100 + k)
        inv = _inv(cuda, 1, Qd, 110 + k)
        g = torch.randn(1, Qd, H * C, device=cuda, generator=torch.Generator(device=cuda).manual_seed(120 + k))
        leaves = [t.detach().clone().requires_grad_(True) for t in grp]
        slots = sca.MSDARowsFunction.apply(sca.unit_plan(1, 0, cams), 1, Qd, shapes, lsi, None, None, inv, *leaves)
        runs.append((Qd, shapes, grp, inv, g, leaves, slots))
    for *_, g, leaves, slots in runs:           # no synchronisation between the three backwards
        slots.backward(g)
    for Qd, shapes, grp, inv, g, leaves, slots in runs:
        ref = _oracle_rows(sca.unit_plan(1, 0, cams), 1, Qd, shapes, None, None, inv, [grp], g, per_camera=True)
        _close_rows(slots, [[t.grad for t in leaves]], ref, shapes, [grp], tag=f"{Qd} rows: ")
