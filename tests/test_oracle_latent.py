"""Pin the fp64 LatentRendering oracle (`latent_core_fp64`): against a per-cell, per-waypoint loop that
restates SURVEY.md A.3 with hand-written bilinear weights, against the fp32 `latent_core`, and on its
geometry, which must be exactly the fp32 rays and masks of `latent_core`."""
import numpy as np
import pytest
import torch

from oracle import latent_render_ref as ref

f32 = np.float32


def _ray(Hb, Wb, iy, ix, grid_num, grid_step):
    """One cell's ray in fp32 scalar arithmetic: (cell gx, cell gy, [(gx, gy, phase-1 mask, phase-2 mask)])."""
    with np.errstate(divide="ignore", invalid="ignore"):
        cx, cy = f32(ix + 0.5) / f32(Wb), f32(iy + 0.5) / f32(Hb)
        rx, ry = cx - f32(0.5), cy - f32(0.5)
        nrm = np.sqrt(rx * rx + ry * ry)
        rnx, rny = rx / nrm, ry / nrm
        rnx, rny = (f32(0) if np.isnan(v) else v for v in (rnx, rny))     # the centre cell has no direction
        cgx, cgy = cx * f32(2) - f32(1), cy * f32(2) - f32(1)
        len_cell = np.sqrt(cgx * cgx + cgy * cgy)
        bound = min(f32(1) / abs(rnx), f32(1) / abs(rny))
    tstep = f32(grid_step / (min(Hb, Wb) // 2))
    way = []
    for k in range(grid_num):
        t = f32(k + 0.5) * tstep
        gx = (f32(0.5) + rnx * t) * f32(2) - f32(1)
        gy = (f32(0.5) + rny * t) * f32(2) - f32(1)
        ln = np.sqrt(gx * gx + gy * gy)
        way.append((float(gx), float(gy), bool(ln < len_cell), bool(ln < bound)))
    return float(cgx), float(cgy), way


def _bilerp(m, gx, gy):
    """grid_sample(align_corners=False, zero padding) of the channel-last map m [bs,Hb,Wb,C] at one point."""
    Hb, Wb = m.shape[1], m.shape[2]
    ix, iy = ((gx + 1) * Wb - 1) / 2, ((gy + 1) * Hb - 1) / 2
    x0, y0 = int(np.floor(ix)), int(np.floor(iy))
    wx, wy = ix - x0, iy - y0
    out = torch.zeros(m.shape[0], m.shape[3], dtype=m.dtype)
    for xx, yy, w in ((x0, y0, (1 - wx) * (1 - wy)), (x0 + 1, y0, wx * (1 - wy)),          # nw, ne
                      (x0, y0 + 1, (1 - wx) * wy), (x0 + 1, y0 + 1, wx * wy)):          # sw, se
        if 0 <= xx < Wb and 0 <= yy < Hb:
            out = out + w * m[:, yy, xx]
    return out


def _loop_core(occ, feat, grid_num, grid_step, eps, act):
    """prob_u = a_cell * prod_k (1 - a_k m1_k);  pooled_u,(d,j) = sum_k m2_k p_k f_k / (sum_k m2_k p_k + eps)."""
    bs, Hb, Wb, D = occ.shape
    G = feat.shape[-1] // D
    fn = torch.sigmoid if act == "sigmoid" else (lambda x: 1 - torch.exp(-torch.relu(x)))
    rays = [_ray(Hb, Wb, iy, ix, grid_num, grid_step) for iy in range(Hb) for ix in range(Wb)]
    probs = []
    for cgx, cgy, way in rays:
        p = fn(_bilerp(occ, cgx, cgy))
        for gx, gy, m1, _ in way:
            if m1:
                p = p * (1 - fn(_bilerp(occ, gx, gy)))
        probs.append(p)
    prob = torch.stack(probs, 1).view(bs, Hb, Wb, D)
    pooled = []
    for _, _, way in rays:
        S, N = torch.zeros(bs, D, dtype=occ.dtype), torch.zeros(bs, D, G, dtype=occ.dtype)
        for gx, gy, _, m2 in way:
            if m2:
                pg = _bilerp(prob, gx, gy)
                S = S + pg
                N = N + pg[..., None] * _bilerp(feat, gx, gy).view(bs, D, G)
        pooled.append((N / (S + eps)[..., None]).reshape(bs, D * G))
    return prob, torch.stack(pooled, 1)


def _forward_backward(core, occ, feat, gp, gq, *args):
    o, f = occ.clone().requires_grad_(True), feat.clone().requires_grad_(True)
    p, q = core(o, f, *args)
    (p * gp).sum().add((q * gq).sum()).backward()
    return p.detach(), q.detach(), o.grad, f.grad


def _inputs(bs, Hb, Wb, D, G, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    occ = torch.randn(bs, Hb, Wb, D, generator=g, dtype=dtype) * 1.5
    feat = torch.randn(bs, Hb, Wb, D * G, generator=g, dtype=dtype)
    gp = torch.randn(bs, Hb, Wb, D, generator=g, dtype=dtype)
    gq = torch.randn(bs, Hb * Wb, D * G, generator=g, dtype=dtype)
    return occ, feat, gp, gq


TINY_BEVS = [(2, 2), (3, 3), (3, 4), (5, 5), (4, 7)]
DG = [(1, 1), (2, 4), (4, 2)]


@pytest.mark.parametrize("act", ["sigmoid", "exp"])
@pytest.mark.parametrize("grid_num", [1, 3, 9])
@pytest.mark.parametrize("bev", TINY_BEVS)
def test_fp64_oracle_equals_loop(bev, grid_num, act):
    i = TINY_BEVS.index(bev) + grid_num + (act == "exp")
    D, G = DG[i % len(DG)]
    grid_step = (0.5, 1.0, 0.25)[i % 3]
    occ, feat, gp, gq = _inputs(2, *bev, D, G, seed=i, dtype=torch.float64)
    want = _forward_backward(_loop_core, occ, feat, gp, gq, grid_num, grid_step, 1e-3, act)
    got = _forward_backward(ref.latent_core_fp64, occ, feat, gp, gq, grid_num, grid_step, 1e-3, act)
    for a, b, what in zip(got, want, ("prob", "pooled", "grad occ", "grad feat")):
        assert a.dtype == torch.float64, what
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-12, atol=1e-13 * b.abs().max().item(), err_msg=what)


# the golden cases' core shapes (tests/latent_cases.py): (bs, Hb, Wb, D, G, grid_num, act)
GOLDEN_SHAPES = [(2, 20, 24, 16, 1, 48, "sigmoid"), (2, 20, 24, 4, 2, 40, "exp"), (2, 20, 24, 1, 16, 40, "sigmoid"),
                 (2, 13, 14, 16, 1, 48, "sigmoid"), (2, 13, 14, 8, 2, 40, "exp")]


@pytest.mark.parametrize("bs,Hb,Wb,D,G,grid_num,act", GOLDEN_SHAPES)
def test_fp64_oracle_agrees_with_fp32_oracle(bs, Hb, Wb, D, G, grid_num, act):
    occ, feat, gp, gq = _inputs(bs, Hb, Wb, D, G, seed=Hb * D + G, dtype=torch.float32)
    want = _forward_backward(ref.latent_core_fp64, *(t.double() for t in (occ, feat, gp, gq)), grid_num, 0.5, 1e-3, act)
    got = _forward_backward(ref.latent_core, occ, feat, gp, gq, grid_num, 0.5, 1e-3, act)
    for a, b, what in zip(got, want, ("prob", "pooled", "grad occ", "grad feat")):
        assert a.dtype == torch.float32 and b.dtype == torch.float64, what
        err = (a.double() - b).abs().max().item()
        assert err <= 1e-5 * b.abs().max().item(), f"{what}: max err {err:.3e} vs max|ref| {b.abs().max().item():.3e}"


@pytest.mark.parametrize("Hb,Wb,grid_num,grid_step", [(5, 5, 9, 0.5), (9, 9, 33, 0.25), (3, 4, 3, 2.0), (7, 12, 40, 1.0),
                                                      (13, 6, 17, 0.5), (63, 64, 96, 0.5)])
def test_fp64_oracle_uses_the_fp32_geometry_of_latent_core(monkeypatch, Hb, Wb, grid_num, grid_step):
    """latent_core_fp64 samples with the same fp32 rays whatever its input's precision.  They equal the per-cell
    fp32 scalar statement of the loop above bit for bit (IEEE square roots, as in the kernels), and their masks are
    exactly the masks latent_core uses on fp32 input.  latent_core's waypoints may differ by an ulp: torch's CPU
    fp32 sqrt is not always correctly rounded."""
    seen = []
    geometry = ref.geometry

    def spy(*args, **kw):
        out = geometry(*args, **kw)
        seen.append(out)
        return out

    monkeypatch.setattr(ref, "geometry", spy)
    occ, feat, _, _ = _inputs(1, Hb, Wb, 2, 1, seed=0, dtype=torch.float32)
    ref.latent_core_fp64(occ, feat, grid_num, grid_step)
    ref.latent_core_fp64(occ.double(), feat.double(), grid_num, grid_step)
    ref.latent_core(occ, feat, grid_num, grid_step)
    assert len(seen) == 3
    (grid, m1, m2), (g2, a2, b2), (g_fp32, m1_fp32, m2_fp32) = seen
    assert grid.dtype == torch.float32 and m1.dtype == torch.bool and m2.dtype == torch.bool
    assert torch.equal(g2, grid) and torch.equal(a2, m1) and torch.equal(b2, m2)
    assert torch.equal(m1, m1_fp32) and torch.equal(m2, m2_fp32)
    assert ((g_fp32 - grid).abs() <= 2 ** -20 * grid.abs().clamp(min=1)).all()
    assert not m1[:, -1].any(), "a cell never masks itself"
    for u in range(Hb * Wb):
        cgx, cgy, way = _ray(Hb, Wb, u // Wb, u % Wb, grid_num, grid_step)
        want = torch.tensor([[gx, gy] for gx, gy, _, _ in way] + [[cgx, cgy]], dtype=torch.float32)
        assert torch.equal(grid[u], want), f"cell {u}: waypoints"
        assert m1[u, :-1].tolist() == [w[2] for w in way], f"cell {u}: phase-1 mask"
        assert m2[u].tolist() == [w[3] for w in way], f"cell {u}: phase-2 mask"
