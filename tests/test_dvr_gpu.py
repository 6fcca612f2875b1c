"""Parity of the CUDA ray-casters (through the C ABI) with the CPU oracle, BASELINE
configs[0] (50x50x8, 1k rays), a LiDAR-like 3-frame case and long 4x4xX grids on either side
of the warp kernels' shared-memory budget.  pred/gt: 1e-5 relative (fp64
internally on both sides, fp32 outputs); gradients: 1e-4 relative + fp32-atomic noise."""
import numpy as np
import pytest
import torch

from oracle import dvr_ref
from tests.inputs import dvr_inputs_cfg1, dvr_inputs_lidar, dvr_inputs_outside, dvr_inputs_ties
from vidar_b200 import render

pytestmark = pytest.mark.gpu


def _t(cuda, *arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(cuda) for a in arrs]


def _close(a, b, what, rtol=1e-4, atol_scale=1e-5):
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    scale = np.sqrt((b ** 2).mean()) + 1e-30
    err = np.abs(a - b)
    tol = rtol * np.abs(b) + atol_scale * scale
    assert (err <= tol).all(), f"{what}: max err {err.max():.3e} scale {scale:.3e}, {(err > tol).sum()} bad"


def _long_x_grid(X, seed=21, M=320):
    """A 4 x 4 x X grid (T = 1) on either side of the warp kernels' shared-memory budget.  They keep
    cap = X + Y + Z + 8 records rounded up to 32, 20 B each, for 4 rays per block, and run only while
    that is at most 200 KiB (csrc/dvr.cu, warp_ray_config).  X = 2544: cap 2560, 204 800 B, the last
    size on the warp kernels.  X = 2545: cap 2592, 207 360 B, so every entry point runs one ray per
    thread.  Integer, half-integer and outside-the-grid (x < 0) origins; end points spread along x,
    so many rays close more than MAX_D = 1026 segments, which caps the lists and the fused backward."""
    rng = np.random.default_rng(seed)
    sigma = rng.uniform(0, 0.004, (1, 1, 4, 4, X)).astype(np.float32)
    origin = np.array([[[3.0, 2.0, 1.0], [40.5, 1.5, 2.5], [-6.3, 1.7, 2.2]]], np.float32)
    points = (rng.uniform(0, 1, (1, M, 3)) * np.array([X + 40, 6, 6]) - np.array([20, 1, 1])).astype(np.float32)
    tindex = rng.integers(0, 3, (1, M)).astype(np.float32)
    return sigma, origin, points, tindex


CFG = [("cfg1-int", lambda: dvr_inputs_cfg1(seed=0, integer_origin=True)),
       ("cfg1-frac", lambda: dvr_inputs_cfg1(seed=0, integer_origin=False)),
       ("lidar-3f", lambda: dvr_inputs_lidar(M=3000, T=3, grid=(16, 200, 200), seed=1, pad=24)),
       ("static-T1", lambda: (lambda s, o, p, t: (s[:, :1], o, p, t))(*dvr_inputs_lidar(M=900, T=3, grid=(8, 60, 50), seed=2))),
       ("long-x2544-warp", lambda: _long_x_grid(2544)),
       ("long-x2545-thread", lambda: _long_x_grid(2545))]


@pytest.mark.parametrize("name,make", CFG)
@pytest.mark.parametrize("phase", ["test", "train"])
def test_render_forward(cuda, name, make, phase):
    sigma, origin, points, tindex = make()
    rp, rg = dvr_ref.render_forward(sigma, origin, points, tindex, None, phase)
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    pred, gt = render.dvr.render_forward(s, o, p, t, list(sigma.shape[1:]), phase)
    assert ((pred.cpu().numpy() == -1) == (rp == -1)).all()
    _close(pred, rp, "pred_dist", rtol=1e-5)
    _close(gt, rg, "gt_dist", rtol=1e-5)


@pytest.mark.parametrize("name,make", CFG)
@pytest.mark.parametrize("loss", ["l1", "l2", "absrel"])
def test_render_with_loss_gradient(cuda, name, make, loss):
    sigma, origin, points, tindex = make()
    rp, rg, rgrad = dvr_ref.render(sigma, origin, points, tindex, loss)
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    pred, gt, grad = render.dvr.render(s, o, p, t, loss)
    _close(pred, rp, "pred_dist", rtol=1e-5)
    _close(gt, rg, "gt_dist", rtol=1e-5)
    _close(grad, rgrad, "grad_sigma")


@pytest.mark.parametrize("name,make", CFG)
def test_dvxlr_lists_and_scatter(cuda, name, make):
    sigma, origin, points, tindex = make()
    rng = np.random.default_rng(7)
    regul = rng.standard_normal(sigma.shape).astype(np.float32)
    ref = dvr_ref.dvxlr_render(sigma, origin, points, tindex, regul)
    s, o, p, t, r = _t(cuda, sigma, origin, points, tindex, regul)
    out = render.dvxlr_v2.render_v2(s, o, p, t, r)
    for a, b, w in zip(out, ref, ["pred", "gt", "dd_dsigma", "indices", "ray_pred", "indicator"]):
        if w in ("indices", "indicator", "ray_pred"):
            np.testing.assert_array_equal(a.cpu().numpy(), b, err_msg=w)
        else:
            _close(a, b, w, rtol=1e-5 if w != "dd_dsigma" else 1e-4)
    v1 = render.dvxlr.render(s, o, p, t)
    for a, b in zip(v1, out[:4]):
        assert torch.equal(a, b)
    assert v1[2].shape[-1] == 1026 and v1[3].shape[-2:] == (1026, 3)
    # scatter kernels
    gp = rng.standard_normal(ref[0].shape).astype(np.float32)
    grp = rng.standard_normal(ref[4].shape).astype(np.float32)
    em = gp[..., None] * ref[2]
    rg1, rg2 = dvr_ref.dvxlr_get_grad_sigma(em, ref[3], tindex, sigma, ref[5], grp)
    emt, idx, ind, grpt = _t(cuda, em, ref[3], ref[5], grp)
    g1, g2 = render.dvxlr_v2.get_grad_sigma_v2(emt, idx, t, s, ind, grpt)
    _close(g1, rg1, "grad_sigma(v2)")
    _close(g2, rg2, "grad_sigma_regul")
    (g0,) = render.dvxlr.get_grad_sigma(emt, idx, t, s)
    _close(g0, rg1, "grad_sigma(v1)")


@pytest.mark.parametrize("name,make", CFG)
def test_autograd_layers_fused_equals_lists_equals_oracle(cuda, name, make):
    sigma, origin, points, tindex = make()
    rng = np.random.default_rng(9)
    gp = rng.standard_normal(points.shape[:2]).astype(np.float32)
    (rgrad,) = dvr_ref.dvxlr_autograd_backward(sigma, origin, points, tindex, gp)
    rp, rg = dvr_ref.dvxlr_forward(sigma, origin, points, tindex)
    s, o, p, t, gpt = _t(cuda, sigma, origin, points, tindex, gp)
    for layer in (render.DifferentiableVoxelRendering, render.DifferentiableVoxelRenderingLayerLists.apply):
        sg = s.clone().requires_grad_(True)
        pred, gt = layer(sg, o, p, t)
        _close(pred, rp, "pred", rtol=1e-5)
        _close(gt, rg, "gt", rtol=1e-5)
        (pred * gpt).sum().backward()
        _close(sg.grad, rgrad, "grad_sigma")
    # V2: second gradient path through ray_pred
    regul = rng.standard_normal(sigma.shape).astype(np.float32)
    ref = dvr_ref.dvxlr_render(sigma, origin, points, tindex, regul)
    grp = (rng.standard_normal(ref[4].shape) * (ref[5] >= 0)).astype(np.float32)
    rg1, rg2 = dvr_ref.dvxlr_autograd_backward(sigma, origin, points, tindex, gp, regul, grp)
    sg = s.clone().requires_grad_(True)
    rr = torch.from_numpy(regul).to(cuda).requires_grad_(True)
    pred, gt, ray_pred, indicator = render.DifferentiableVoxelRenderingV2(sg, o, p, t, rr)
    np.testing.assert_array_equal(indicator.cpu().numpy(), ref[5])
    np.testing.assert_array_equal(ray_pred.detach().cpu().numpy(), ref[4])
    ((pred * gpt).sum() + (ray_pred * torch.from_numpy(grp).to(cuda)).sum()).backward()
    _close(sg.grad, rg1, "grad_sigma(v2)")
    _close(rr.grad, rg2, "grad_sigma_regul(v2)")


def test_init_and_errors(cuda):
    sigma, origin, points, tindex = dvr_inputs_cfg1(seed=4)
    p, t = _t(cuda, points, tindex)
    occ = render.dvr.init(p, t, [1, 8, 50, 50])
    np.testing.assert_array_equal(occ.cpu().numpy(), dvr_ref.init(points, tindex, [1, 8, 50, 50]))
    assert torch.equal(render.dvxlr.init(p, t, [1, 8, 50, 50]), occ)
    s, o = _t(cuda, sigma, origin)
    with pytest.raises(ValueError, match="UNKNOWN PHASE NAME"):
        render.dvr.render_forward(s, o, p, t, [1, 8, 50, 50], "val")
    with pytest.raises(RuntimeError, match="must be contiguous"):
        render.dvr.render(s, o, p.transpose(0, 1).transpose(0, 1)[:, ::2], t[:, ::2], "l1")
    # empty ray set
    pe = torch.zeros(1, 0, 3, device=cuda)
    te = torch.zeros(1, 0, device=cuda)
    pred, gt = render.dvr.render_forward(s, o, pe, te, [1, 8, 50, 50], "test")
    assert pred.shape == (1, 0)


def test_full_size_properties(cuda):
    """BASELINE configs[2] size: sigma [1,3,16,200,200], 30k rays.  Size-independent checks:
    zero density -> pred == exit distance == clamped gt bound; huge density -> pred == first
    crossing; gradient mass == directional derivative; a strided subset against the oracle."""
    sigma, origin, points, tindex = dvr_inputs_lidar(M=30000, T=3, seed=0)
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    z = torch.zeros_like(s)
    pred0, gt_train = render.dvr.render_forward(z, o, p, t, [3, 16, 200, 200], "train")
    _, gt_test = render.dvr.render_forward(z, o, p, t, [3, 16, 200, 200], "test")
    assert torch.equal(gt_train, torch.minimum(gt_test, pred0))
    sub = slice(0, 30000, 97)
    rp, rg, rgrad = dvr_ref.render(sigma, origin, points[:, sub], tindex[:, sub], "l2")
    pred, gt, grad = render.dvr.render(s, o, p[:, sub].contiguous(), t[:, sub].contiguous(), "l2")
    _close(pred, rp, "pred subset", rtol=1e-5)
    _close(grad, rgrad, "grad subset")
    # directional derivative of sum(pred) along a random direction, fused autograd op
    sg = s.clone().requires_grad_(True)
    pr, _ = render.DifferentiableVoxelRendering(sg, o, p, t)
    pr.sum().backward()
    direction = torch.randn_like(s)
    eps = 1e-2
    pp, _ = render.DifferentiableVoxelRendering(s + eps * direction, o, p, t)
    pm, _ = render.DifferentiableVoxelRendering(s - eps * direction, o, p, t)
    fd = ((pp - pm).double().sum() / (2 * eps)).item()
    an = (sg.grad.double() * direction.double()).sum().item()
    assert fd == pytest.approx(an, rel=2e-3)


def test_origin_outside_volume_uses_serial_path_and_matches_oracle(cuda):
    sigma, origin, points, tindex = dvr_inputs_outside()
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    for phase in ("test", "train"):
        rp, rg = dvr_ref.render_forward(sigma, origin, points, tindex, None, phase)
        pred, gt = render.dvr.render_forward(s, o, p, t, list(sigma.shape[1:]), phase)
        a, b = pred.cpu().numpy(), rp
        assert (np.isnan(a) == np.isnan(b)).all() and ((a == -1) == (b == -1)).all()
        ok = ~np.isnan(b)
        _close(a[ok], b[ok], f"pred {phase}", rtol=1e-5)
        _close(gt.cpu().numpy()[ok], rg[ok], f"gt {phase}", rtol=1e-5)
    assert 0.05 < (rp == -1).mean() < 0.95          # both outcomes are exercised
    rp, rg, rgrad = dvr_ref.render(sigma, origin, points, tindex, "l1")
    pred, gt, grad = render.dvr.render(s, o, p, t, "l1")
    ok = ~np.isnan(rp)
    _close(pred.cpu().numpy()[ok], rp[ok], "pred render", rtol=1e-5)
    fin = np.isfinite(rgrad)
    _close(grad.cpu().numpy()[fin], rgrad[fin], "grad_sigma")


def test_all_padded_and_single_ray(cuda):
    sigma, origin, points, tindex = dvr_inputs_cfg1(seed=3, M=64, pad=0)
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    t_pad = torch.full_like(t, -1.0)
    pred, gt, grad = render.dvr.render(s, o, p, t_pad, "l2")
    assert float(pred.max()) == -1 and float(gt.max()) == -1 and float(grad.abs().sum()) == 0
    pred1, gt1, _ = render.dvr.render(s, o, p[:, :1].contiguous(), t[:, :1].contiguous(), "l2")
    rp, rg, _ = dvr_ref.render(sigma, origin, points[:, :1], tindex[:, :1], "l2")
    _close(pred1, rp, "single ray", rtol=1e-5)


def test_warp_per_ray_voxel_mismatch_rate(cuda):
    """The warp-per-ray kernels take crossing times from fma(i, tDelta, tMax0) and the rounded path
    voxel from round(fma(last, d, v0)) (csrc/dvr.cu header): a branch decision can differ from the
    serial reference's only on near-exact ties.  Randomised rays from integer, half-integer and generic
    origins -- the tie-prone cases -- against the C oracle: a different voxel shows up as a pred
    difference far above 1e-12; the count must be zero at the ray-caster tolerance."""
    sigma, origin, points, tindex = dvr_inputs_ties()
    Z, Y, X = sigma.shape[2:]
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    bad = 0
    for phase in ("test", "train"):
        rp, rg = dvr_ref.render_forward(sigma, origin, points, tindex, None, phase)
        pred, gt = render.dvr.render_forward(s, o, p, t, [3, Z, Y, X], phase)
        a = pred.cpu().numpy()
        assert ((a == -1) == (rp == -1)).all()
        bad += int((np.abs(a - rp) > 1e-5 * np.maximum(1.0, np.abs(rp))).sum())
    rp, rg, rgrad = dvr_ref.render(sigma, origin, points, tindex, "l1")
    pred, gt, grad = render.dvr.render(s, o, p, t, "l1")
    bad += int((np.abs(pred.cpu().numpy() - rp) > 1e-5 * np.maximum(1.0, np.abs(rp))).sum())
    assert bad == 0, f"{bad} rays took a different voxel sequence than the reference"
    _close(grad, rgrad, "grad_sigma")


def test_large_grid_needs_shared_memory_opt_in_for_both_kernels(cuda):
    """X+Y+Z > ~600: the warp-per-ray kernels need more than 48 KB of dynamic shared memory; the
    opt-in must be applied to render_forward's AND render's instantiation (same function-pointer type)."""
    rng = np.random.default_rng(5)
    Z, Y, X, M = 8, 420, 400, 1500
    sigma = rng.uniform(0, 0.05, (1, 1, Z, Y, X)).astype(np.float32)
    origin = np.array([[[200.3, 210.7, 4.2]]], np.float32)
    points = (rng.uniform(0, 1, (1, M, 3)) * np.array([X, Y, Z])).astype(np.float32)
    tindex = np.zeros((1, M), np.float32)
    s, o, p, t = _t(cuda, sigma, origin, points, tindex)
    rp, rg = dvr_ref.render_forward(sigma, origin, points, tindex, None, "train")
    pred, gt = render.dvr.render_forward(s, o, p, t, [1, Z, Y, X], "train")
    _close(pred, rp, "pred (large grid, render_forward)", rtol=1e-5)
    rp2, rg2, rgrad = dvr_ref.render(sigma, origin, points, tindex, "l2")
    pred2, gt2, grad = render.dvr.render(s, o, p, t, "l2")
    _close(pred2, rp2, "pred (large grid, render)", rtol=1e-5)
    _close(grad, rgrad, "grad_sigma (large grid)")


def test_tie_prone_rays_equal_reference_cuda_golden(cuda):
    """The tie-prone rays against what the REFERENCE's own CUDA binary returned for them
    (tests/golden/dvr_ties.npz, tools/make_golden_dvr.py): pred / gt of render_forward, render and the dvxlr
    autograd forward, every ray."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "dvr_ties.npz"))
    s, o, p, t = _t(cuda, g["sigma"], g["origin"], g["points"], g["tindex"])
    grid = list(g["sigma"].shape[1:])
    for ph in ("test", "train"):
        pred, gt = render.dvr.render_forward(s, o, p, t, grid, ph)
        _close(pred, g[f"fwd_{ph}_pred"], f"render_forward {ph} pred", rtol=1e-5)
        _close(gt, g[f"fwd_{ph}_gt"], f"render_forward {ph} gt", rtol=1e-5)
    pred, gt, _ = render.dvr.render(s, o, p, t, "l1")
    _close(pred, g["render_l1_pred"], "render pred", rtol=1e-5)
    sg = s.clone().requires_grad_(True)
    pr, gtd = render.DifferentiableVoxelRendering(sg, o, p, t)
    _close(pr, g["dvxlr_pred"], "dvxlr pred", rtol=1e-5)
    _close(gtd, g["dvxlr_gt"], "dvxlr gt", rtol=1e-5)
    gp = torch.from_numpy(g["grad_pred"]).to(cuda)
    pr.backward(gp)
    _close(sg.grad, g["scatter_grad_sigma_v1"], "dvxlr autograd grad_sigma vs the reference's list scatter")
