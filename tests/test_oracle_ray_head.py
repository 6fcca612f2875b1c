"""Pin oracle/ray_head_ref.py against the reference's own methods (tests/golden/ray_head.npz,
made by tools/make_golden_ray_head.py)."""
import os

import numpy as np
import torch

from oracle import ray_head_ref as ref
from tests import ray_cases as rc

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ray_head.npz")


def test_grid_features_ce_and_gradients_match_reference():
    g = np.load(GOLD)
    c = rc.case()
    sig = [s.clone().requires_grad_(True) for s in c["sigma"]]
    r_mask, r_feat, r_w, r_len = ref.grid_features(c["origin"], c["gt"], c["tindex"], sig, rc.LOSS_W,
                                                   rc.STEP, rc.NUM_WAY)
    np.testing.assert_array_equal(r_mask.numpy(), g["r_mask"])
    np.testing.assert_allclose(r_feat.detach().numpy(), g["r_feat"], rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(r_w.numpy(), g["r_w"])
    np.testing.assert_allclose(r_len.numpy(), g["r_len"], rtol=1e-6)
    loss = ref.ce_loss(r_feat, r_w)
    np.testing.assert_allclose(loss.detach().numpy(), g["loss"], rtol=1e-6)
    loss.backward()
    np.testing.assert_allclose(sig[0].grad.numpy(), g["grad_sigma0"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(sig[1].grad.numpy(), g["grad_sigma1"], rtol=1e-5, atol=1e-7)


def test_decode_matches_reference():
    g = np.load(GOLD)
    c = rc.case()
    sigma = c["sigma"][-1]
    for b in range(rc.BS):
        for f in range(rc.FRAMES):
            sel = c["tindex"][b] == f
            pred, idx = ref.decode_frame(sigma[b, f], c["origin"][b, f], c["gt"][b][sel], rc.NUM_WAY, rc.STEP)
            np.testing.assert_array_equal(idx.numpy(), g["decode_idx"][b][sel.numpy()])
            np.testing.assert_allclose(pred.numpy(), g["decode_pred"][b][sel.numpy()], rtol=1e-6)


# ---- the fp64 oracle (sample_fp64, ce_fp64, gumbel_fp64, argmax_fp64) on the same golden case -------------
def _frames(c, b):
    """The case's tindex as the int32 frame the kernels take: -1 for padding rows."""
    return c["tindex"][b].to(torch.int32)


def _frame_major(frame, keep):
    """Row order of _get_grid_features: frame-major, original order inside a frame, rows `keep` only."""
    idx = keep.nonzero().squeeze(-1)
    return idx[torch.argsort(frame[idx], stable=True)]


def test_sample_fp64_reproduces_fp32_oracle_and_golden():
    g = np.load(GOLD)
    c = rc.case()
    feats = []
    for lvl, sig in enumerate(c["sigma"]):
        for b in range(rc.BS):
            frame = _frames(c, b)
            lg, ln, vd, absw = ref.sample_fp64(sig[b], c["origin"][b], c["gt"][b], frame, rc.NUM_WAY, rc.STEP, True)
            for f in range(rc.FRAMES):
                sel = frame == f
                lg32, ln32, vd32 = ref.sample_frame(sig[b, f], c["origin"][b, f], c["gt"][b][sel], rc.NUM_WAY, rc.STEP)
                assert torch.equal(vd[sel], vd32)
                assert torch.equal(torch.isinf(lg[sel]), torch.isinf(lg32))
                fin = torch.isfinite(lg32)
                err = (lg32.double() - lg[sel])[fin].abs()
                assert (err <= 16 * ref.U32 * absw[sel][fin] + 1e-30).all(), err.max()
                np.testing.assert_array_max_ulp(ln[sel].numpy(), ln32.numpy(), maxulp=1)
            assert not vd[frame < 0].any() and torch.isinf(lg[frame < 0]).all() and (ln[frame < 0] == 0).all()
            order = _frame_major(frame, vd)
            feats.append((lg[order], ln[order], absw[order]))
    r_feat = torch.stack([lg for lg, _, _ in feats], 0)
    np.testing.assert_array_equal(np.where(np.isinf(r_feat[0].numpy()), -np.inf, 0.0), g["r_mask"])
    fin = torch.isfinite(r_feat)
    bound = 16 * ref.U32 * torch.stack([a for _, _, a in feats], 0)
    assert ((torch.from_numpy(g["r_feat"]).double() - r_feat).abs()[fin] <= bound[fin] + 1e-30).all()
    np.testing.assert_array_max_ulp(feats[0][1].numpy(), g["r_len"], maxulp=1)


def test_ce_fp64_and_its_gradient_match_golden():
    g = np.load(GOLD)
    c = rc.case()
    b = 0
    frame = _frames(c, b)
    w = torch.tensor(rc.LOSS_W, dtype=torch.float64)          # [frame, level]
    outs = [ref.ce_fp64(sig[b], c["origin"][b], c["gt"][b], frame, rc.NUM_WAY, rc.STEP) for sig in c["sigma"]]
    wr = torch.stack([torch.where(o.valid, w[frame.clamp(min=0).long(), lvl], 0.0) for lvl, o in enumerate(outs)])
    den = wr.sum().clamp(min=1)
    loss = sum((o.ce * wr[lvl]).sum() for lvl, o in enumerate(outs)) / den
    np.testing.assert_allclose(loss.item(), g["loss"], rtol=2e-6)
    order = _frame_major(frame, outs[0].valid)
    np.testing.assert_allclose(torch.stack([o.ce[order] for o in outs]).numpy(), g["ce_per_ray"], rtol=2e-6, atol=1e-6)
    for lvl, sig in enumerate(c["sigma"]):
        got = ref.ce_fp64(sig[b], c["origin"][b], c["gt"][b], frame, rc.NUM_WAY, rc.STEP, wr[lvl] / den).scatter
        np.testing.assert_allclose(got.grad.numpy(), g[f"grad_sigma{lvl}"][b], rtol=1e-5, atol=1e-7)


def test_argmax_fp64_matches_golden_decode():
    g = np.load(GOLD)
    c = rc.case()
    sigma = c["sigma"][-1]
    for b in range(rc.BS):
        frame = _frames(c, b)
        out = ref.argmax_fp64(sigma[b], c["origin"][b], c["gt"][b], frame, rc.NUM_WAY, rc.STEP)
        sel = (frame >= 0).numpy()
        np.testing.assert_array_equal(out.index.numpy()[sel], g["decode_idx"][b][sel])
        np.testing.assert_array_equal(out.depth.numpy()[sel], g["decode_pred"][b][sel])
        assert (out.index[~sel] == 0).all() and (out.depth[~sel] == 0).all()


# ---- the oracle's closed-form gradients against fp64 autograd through the same corners -----------------------
def _autograd_logits(sig64, origin, points, frame, num_way, step, with_gt):
    nf = sig64.shape[0]
    f, live = ref.ray_frames(frame, points.shape[0], nf)
    length, masked, coord, gin = ref.waypoints(origin, points, f, sig64.shape[1:], num_way, step, with_gt)
    idx, w = ref.corners(coord, sig64.shape[1:])
    v = sig64.reshape(nf, -1)[f.clamp(0, nf - 1)[:, None, None], idx.clamp(min=0)]
    return (torch.where(idx >= 0, v, 0.0) * w).sum(-1), length, masked, gin, live


def _small_case(seed=0, R=300, nf=3, grid=(5, 13, 29)):
    gen = torch.Generator().manual_seed(seed)
    Z, Y, X = grid
    size = torch.tensor([X, Y, Z], dtype=torch.float32)
    sigma = torch.randn(nf, Z, Y, X, generator=gen) * 2
    origin = size * (0.3 + 0.4 * torch.rand(nf, 3, generator=gen))
    points = size * (1.3 * torch.rand(R, 3, generator=gen) - 0.15)
    frame = torch.randint(-1, nf + 1, (R,), generator=gen).to(torch.int32)      # -1 and nf are skipped
    return sigma, origin, points, frame


def test_closed_form_gradients_equal_fp64_autograd():
    sigma, origin, points, frame = _small_case()
    nw, step = 40, 0.7
    gen = torch.Generator().manual_seed(1)
    s64 = sigma.double().requires_grad_(True)
    # ray_sample backward
    logit, _, masked, gin, live = _autograd_logits(s64, origin, points, frame, nw, step, True)
    gl = torch.randn(logit.shape, generator=gen)
    keep = live[:, None] & ~masked
    (gs,) = torch.autograd.grad((torch.where(keep, logit, 0.0) * gl.double()).sum(), s64, retain_graph=True)
    sc = ref.sample_backward_fp64(sigma, origin, points, frame, gl, nw, step, True)
    torch.testing.assert_close(sc.grad, gs, rtol=1e-12, atol=1e-12)
    assert (sc.mag >= sc.grad.abs()).all() and (sc.err == 0).all() and sc.count.sum() > 0
    # cross entropy
    gce = torch.randn(points.shape[0], generator=gen)
    ok = live & gin
    ce = torch.logsumexp(torch.where(masked, float("-inf"), logit), -1) - logit[:, 0]
    (gs,) = torch.autograd.grad((torch.where(ok, ce, 0.0) * gce.double()).sum(), s64, retain_graph=True)
    out = ref.ce_fp64(sigma, origin, points, frame, nw, step, gce)
    torch.testing.assert_close(out.scatter.grad, gs, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(out.ce, torch.where(ok, ce, 0.0).detach(), rtol=1e-14, atol=1e-14)
    assert torch.equal(out.valid, ok) and 0 < ok.sum() < ok.numel()
    # gumbel: the reference statements on the fp64 waypoint logits, with the arg-max over logit + noise
    noise = -torch.empty(points.shape[0], nw).exponential_(generator=gen).log()
    gd = torch.randn(points.shape[0], generator=gen)
    lg = torch.where(masked, float("-inf"), logit)[:, 1:]
    _, length, *_ = _autograd_logits(s64, origin, points, frame, nw, step, False)
    pick = (lg + noise.double()).argmax(-1)
    pred = length.gather(1, pick[:, None])[:, 0].double()
    e = torch.exp(lg - lg.max(-1, keepdim=True)[0])
    prob = (e * (length > pred[:, None].float())).sum(-1) / e.sum(-1)
    dist = (1 - prob.detach() + prob) * pred
    live_wp = ok & ~masked[:, 1:].all(-1)
    (gs,) = torch.autograd.grad((torch.where(live_wp, dist, 0.0) * gd.double()).sum(), s64)
    out = ref.gumbel_fp64(sigma, origin, points, frame, nw, step, noise, gd)
    torch.testing.assert_close(out.scatter.grad, gs, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(out.dist[live_wp].double(), dist[live_wp].detach(), rtol=0, atol=0)
    assert torch.equal(out.index[ok], pick[ok])
    assert 0 < live_wp.sum() and (ok & ~live_wp).sum() == out.dist[ok].isnan().sum()
