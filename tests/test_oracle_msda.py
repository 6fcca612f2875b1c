"""Pin the MSDA oracle: grid_sample statement == per-corner statement == the same-lineage
implementation shipped in `transformers` (mmcv itself is not in this image)."""
import numpy as np
import pytest
import torch

from oracle import msda_ref
from tests.inputs import level_tensors, msda_inputs

LEVELS = ((9, 13), (5, 7), (3, 4))


def _case(mode, seed):
    return msda_inputs(B=2, Q=37, H=3, C=8, levels=LEVELS, P=4, seed=seed, mode=mode,
                       dtype=torch.float64)


@pytest.mark.parametrize("mode", ["local", "stress"])
def test_grid_sample_equals_explicit_forward_backward(mode):
    d = _case(mode, 1)
    out_gs = msda_ref.msda_grid_sample(d["value"], d["shapes"], d["loc"], d["attn"])
    gv, gl, ga = msda_ref.msda_grid_sample_backward(d["value"], d["shapes"], d["loc"], d["attn"],
                                                    d["grad_out"])
    out, ev, el, ea = msda_ref.msda_explicit(d["value"].numpy(), d["shapes"].numpy(), d["lsi"].numpy(),
                                             d["loc"].numpy(), d["attn"].numpy(), d["grad_out"].numpy())
    np.testing.assert_allclose(out, out_gs.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(ev, gv.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(el, gl.numpy(), rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(ea, ga.numpy(), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("mode", ["local", "stress"])
def test_matches_transformers_deformable_detr(mode):
    tr = pytest.importorskip("transformers.models.deformable_detr.modeling_deformable_detr")
    d = _case(mode, 2)
    ref = tr.MultiScaleDeformableAttention().forward(
        d["value"], d["shapes"], [tuple(x) for x in d["shapes"].tolist()], d["lsi"], d["loc"],
        d["attn"], 64)
    out = msda_ref.msda_grid_sample(d["value"], d["shapes"], d["loc"], d["attn"])
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)


def _rows_problem(seed):
    """Three cameras, two batch elements, shuffled visible lists with counts (one empty), a launch group with
    S = 4 sub-slices owning [1, 3) and a second group of one camera; some pillars are seen by no live row."""
    g = torch.Generator().manual_seed(seed)
    cams, bs, Qd, H, C, L, P, D = 3, 2, 150, 2, 4, 2, 4, 2
    levels = ((6, 5), (3, 2))
    shapes, lsi = level_tensors(levels)
    K = sum(h * w for h, w in levels)
    idx = torch.stack([torch.randperm(Qd, generator=g) for _ in range(cams)]).int()
    count = torch.tensor([140, 0, 97], dtype=torch.int32)
    plan = [(0, 2, 4, 1, 3), (2, 1, 1, 0, 1)]
    seen = torch.zeros(Qd)
    for c in range(cams):
        seen[idx[c, :count[c]].long()] += 1
    assert (seen == 0).any()
    inv = (1.0 / seen.clamp(min=1)).double().expand(bs, Qd).contiguous()
    values = [torch.randn(bs * ncl, K, H, C, generator=g, dtype=torch.float64) for _, ncl, *_ in plan]
    locs = [torch.rand(bs * ncl, Qd, H, L, P, 2, generator=g, dtype=torch.float64) * 1.2 - 0.1 for _, ncl, *_ in plan]
    attns = [torch.rand(bs * ncl, Qd, H, L, P, generator=g, dtype=torch.float64) for _, ncl, *_ in plan]
    ref_cam = torch.rand(cams, bs, Qd, D, 2, generator=g) * 1.2 - 0.1
    offsets = 2.0 * torch.randn(bs, Qd, H, L, P, 2, generator=g)
    logits = torch.randn(bs, Qd, H, L * P, generator=g)
    grad = torch.randn(bs, Qd, H * C, generator=g, dtype=torch.float64)
    return dict(plan=plan, bs=bs, Qd=Qd, shapes=shapes, lsi=lsi, idx=idx, count=count, inv=inv, values=values,
                locs=locs, attns=attns, ref_cam=ref_cam, offsets=offsets, logits=logits, grad=grad)


def _live_rows(group, count, c, rows):
    _, _, S, lo, hi = group
    return [j for j in range(rows) if (count is None or j < int(count[c])) and lo <= (j // 64) % S < hi]


def _rows_explicit(d, locs, attns):
    """The row map stated directly: per (group, b, camera) the live rows, msda_explicit on them, out * inv added
    into the slots of their pillars; (value, loc, attn) gradients per row."""
    shapes, lsi, idx, inv, grad = (d[k].numpy() for k in ("shapes", "lsi", "idx", "inv", "grad"))
    slots = np.zeros(grad.shape)
    grads = []
    for group, v, loc, aw in zip(d["plan"], d["values"], locs, attns):
        cam0, ncl = group[:2]
        v, loc, aw = v.detach().numpy(), loc.detach().numpy(), aw.detach().numpy()
        gv, gl, ga = np.zeros_like(v), np.zeros_like(loc), np.zeros_like(aw)
        for b in range(d["bs"]):
            for cl in range(ncl):
                n, c = b * ncl + cl, cam0 + cl
                js = _live_rows(group, d["count"], c, loc.shape[1])
                if not js:
                    continue
                q = idx[c, js].astype(np.int64)
                s = inv[b, q][:, None]
                out, v_g, l_g, a_g = msda_ref.msda_explicit(v[n:n + 1], shapes, lsi, loc[n:n + 1, js], aw[n:n + 1, js],
                                                            (grad[b, q] * s)[None])
                slots[b, q] += out[0] * s                 # a camera lists a pillar once
                gv[n] += v_g[0]
                gl[n, js], ga[n, js] = l_g[0], a_g[0]
        grads.append((gv, gl, ga))
    return slots, grads


def test_rows_oracle_equals_explicit_row_loop():
    """msda_rows (grid_sample + index_put, autograd) == a Python loop over (b, camera) of msda_explicit."""
    d = _rows_problem(5)
    leaves = [[t.clone().requires_grad_(True) for t in grp] for grp in zip(d["values"], d["locs"], d["attns"])]
    slots = msda_ref.msda_rows(d["plan"], d["bs"], d["Qd"], d["shapes"], d["idx"], d["count"], d["inv"], leaves)
    slots.backward(d["grad"])
    want, wgrads = _rows_explicit(d, d["locs"], d["attns"])
    assert np.abs(want).max() > 0 and (np.abs(want).sum(-1) == 0).any()     # some slots receive nothing
    np.testing.assert_allclose(slots.detach().numpy(), want, rtol=1e-10, atol=1e-12)
    for k, (lv, (gv, gl, ga)) in enumerate(zip(leaves, wgrads)):
        np.testing.assert_allclose(lv[0].grad.numpy(), gv, rtol=1e-10, atol=1e-12, err_msg=f"group {k} grad_value")
        np.testing.assert_allclose(lv[1].grad.numpy(), gl, rtol=1e-9, atol=1e-10, err_msg=f"group {k} grad_loc")
        np.testing.assert_allclose(lv[2].grad.numpy(), ga, rtol=1e-10, atol=1e-12, err_msg=f"group {k} grad_attn")
    # an identity list (idx None) with every row live is the plain op with its output scaled by inv
    v, loc, aw = (t[:2].clone() for t in (d["values"][0], d["locs"][0], d["attns"][0]))
    s = msda_ref.msda_rows([(0, 1, 1, 0, 1)], 2, d["Qd"], d["shapes"], None, None, d["inv"], [(v, loc, aw)])
    torch.testing.assert_close(s, msda_ref.msda_grid_sample(v, d["shapes"], loc, aw) * d["inv"][..., None],
                               rtol=1e-12, atol=1e-12)


def test_sca_rows_oracle_equals_explicit_row_loop():
    """msda_sca_rows (gathered offsets / logits, fp32 location statements, fp64 softmax + sampling, autograd)
    == the same loop with the per-pillar gradients accumulated by hand."""
    d = _rows_problem(6)
    bs, Qd, plan = d["bs"], d["Qd"], d["plan"]
    _, _, H, L, P, _ = d["offsets"].shape
    off = d["offsets"].double().requires_grad_(True)
    lg = d["logits"].double().requires_grad_(True)
    values = [v.clone().requires_grad_(True) for v in d["values"]]
    slots = msda_ref.msda_sca_rows(plan, bs, d["shapes"], d["idx"], d["count"], d["inv"], d["ref_cam"], off, lg, values)
    slots.backward(d["grad"])
    # per row: locations in the module's fp32 statements, weights = softmax in fp64
    wh = torch.stack([d["shapes"][:, 1], d["shapes"][:, 0]], -1).float().view(L, 1, 2)
    locs, attns = [], []
    for cam0, ncl, *_ in plan:
        n = torch.arange(bs * ncl)
        b, cam = n // ncl, cam0 + n % ncl
        q = d["idx"][cam].long()
        o32 = d["offsets"][b[:, None], q] / wh
        r = d["ref_cam"][cam[:, None], b[:, None], q]
        locs.append((o32.view(bs * ncl, Qd, H, L, P // 2, 2, 2) + r.view(bs * ncl, Qd, 1, 1, 1, 2, 2))
                    .view(bs * ncl, Qd, H, L, P, 2).double())
        attns.append(d["logits"][b[:, None], q].double().softmax(-1).view(bs * ncl, Qd, H, L, P))
    want, wgrads = _rows_explicit(d, locs, attns)
    np.testing.assert_allclose(slots.detach().numpy(), want, rtol=1e-10, atol=1e-12)
    g_off, g_lg = np.zeros(off.shape), np.zeros(lg.shape)
    for group, (gv, gl, ga), aw, v in zip(plan, wgrads, attns, values):
        cam0, ncl = group[:2]
        np.testing.assert_allclose(v.grad.numpy(), gv, rtol=1e-10, atol=1e-12)
        aw = aw.numpy().reshape(bs * ncl, Qd, H, L * P)
        ga = ga.reshape(aw.shape)
        gl_ = gl / wh.double().numpy()
        glog = aw * (ga - (aw * ga).sum(-1, keepdims=True))
        for b in range(bs):
            for cl in range(ncl):
                n, c = b * ncl + cl, cam0 + cl
                js = _live_rows(group, d["count"], c, Qd)
                q = d["idx"][c, js].long().numpy()
                np.add.at(g_off[b], q, gl_[n, js])
                np.add.at(g_lg[b], q, glog[n, js])
    np.testing.assert_allclose(off.grad.numpy(), g_off, rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(lg.grad.numpy(), g_lg, rtol=1e-9, atol=1e-12)


def test_out_of_range_samples_contribute_nothing():
    d = _case("local", 3)
    loc = d["loc"].clone()
    loc[:, :, :, 0] = -0.5          # whole level 0 far outside
    loc[:, :, :, 1, :, 0] = 1.5
    base = msda_ref.msda_grid_sample(d["value"], d["shapes"], loc, d["attn"])
    attn = d["attn"].clone()
    attn[:, :, :, 0] = 0
    attn[:, :, :, 1] = 0
    zeroed = msda_ref.msda_grid_sample(d["value"], d["shapes"], d["loc"], attn)
    torch.testing.assert_close(base, zeroed, rtol=1e-12, atol=1e-12)
