"""The head's dense Chamfer term on the GPU (ray_head.dense_chamfer_loss, csrc/dense_chamfer.cu): against goldens
from the reference's own loss and the fp64 oracle, against the per-pair loop it replaces inside
ViDARRayHead.loss, and its batch properties (no host sync, fixed launch count, repeatable bits)."""
import numpy as np
import pytest
import torch

from oracle import dense_chamfer_ref
from tests import dense_chamfer_cases as dc
from tests.test_dense_chamfer_cpu import GOLD, golden_case
from vidar_b200 import _lib, ray_head
from vidar_b200.head import ViDARRayHead

pytestmark = pytest.mark.gpu


def _grad_ok(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool((np.abs(a - b) <= 1e-4 * np.abs(b) + 1e-5 * np.abs(b).max()).all())


def _op(cuda, args):
    t = {k: torch.from_numpy(np.asarray(args[k], np.float32)).to(cuda).contiguous()
         for k in ("dist", "points", "origin", "gt", "gt_tindex")}
    dist = t.pop("dist").requires_grad_(True)
    loss = ray_head.dense_chamfer_loss(dist, t["points"], t["origin"], t["gt"], t["gt_tindex"], args["grid"],
                                       args["frame_weights"], args["weight_sum"], args["eval_within_grid"],
                                       args["pc_range"])
    loss.backward()
    return float(loss.detach()), dist.grad.cpu().numpy()


@pytest.mark.parametrize("name", dc.NAMES)
def test_op_matches_reference_golden_and_oracle(cuda, name):
    args, loss, grad = golden_case(np.load(GOLD), name)
    got_loss, got_grad = _op(cuda, args)
    f32 = {k: (np.asarray(v, np.float32) if isinstance(v, np.ndarray) else v) for k, v in args.items()}
    o_loss, o_grad = dense_chamfer_ref.dense_chamfer(**f32)
    for want_loss, want_grad, what in ((loss, grad, "golden"), (o_loss, o_grad, "oracle")):
        assert abs(got_loss - want_loss) <= 1e-5 * abs(want_loss), (what, got_loss, want_loss)
        assert _grad_ok(got_grad, want_grad), (what, np.abs(got_grad - want_grad).max())


def _head_inputs(cuda, bs, F, seed, H=100, W=100, Z=16, per_frame=8000, num_way=64):
    g = torch.Generator().manual_seed(seed)
    pc = [-50.0, -50.0, -4.0, 50.0, 50.0, 4.0]
    preds = torch.randn(F, 1, bs, H * W, Z, generator=g).to(cuda)
    lo, hi = torch.tensor([-52.0, -52.0, -4.5]), torch.tensor([52.0, 52.0, 4.5])
    gt = []
    for _ in range(bs):
        n = per_frame * (F + 1)                                  # frame F is not predicted
        xyz = lo + (hi - lo) * torch.rand(n, 3, generator=g)
        t = torch.randint(0, F + 1, (n, 1), generator=g).float()
        gt.append(torch.cat([xyz, torch.rand(n, 1, generator=g), t], 1).to(cuda))
    origin = (2.0 * torch.randn(bs, F, 3, generator=g)).to(cuda)
    R = (H // 4) * (W // 4) * (Z // 4) * F
    noise = (-torch.empty(bs, R, num_way).exponential_(generator=g).log()).to(cuda)
    kw = dict(start_idx=0, tgt_bev_h=H, tgt_bev_w=W, tgt_pc_range=pc, pred_frame_num=F, batched_origin_points=origin)
    return preds, gt, kw, noise


def _head(F, num_way=64, **kw):
    lw = np.array([[1.0], [0.8], [1.2], [0.6]][:F])
    return ViDARRayHead(ray_grid_num=num_way, use_ce_loss=False, use_dist_loss=False, loss_weight=lw, **kw)


def _dense(cuda, head, preds, gt, kw, noise, F):
    p = preds.clone().requires_grad_(True)
    out = head.loss(dict(next_bev_preds=p, valid_frames=list(range(F))), gt, gumbels={"dense": noise}, **kw)
    loss = out["loss.dense_voxel"]
    loss.backward()
    return float(loss.detach()), p.grad


def test_head_dense_term_batched_equals_per_pair_loop(cuda):
    preds, gt, kw, noise = _head_inputs(cuda, bs=2, F=4, seed=0)
    res = []
    for fused in (True, False):
        head = _head(4)
        head.fuse_dense_chamfer = fused
        res.append(_dense(cuda, head, preds, gt, kw, noise, 4))
    (l1, g1), (l0, g0) = res
    assert np.isfinite(l1) and abs(l1 - l0) <= 1e-6 * abs(l0), (l1, l0)
    err = (g1 - g0).abs().max().item()
    assert err <= 1e-5 * g0.abs().max().item(), f"grad wrt next_bev_preds: {err:.3e} vs {g0.abs().max().item():.3e}"


def test_gt_without_pred_points_is_nan_on_both_paths(cuda):
    """eval_within_grid with a metre range that no voxel-unit ray end point falls in: every pair has GT points
    and no pred point."""
    preds, gt, kw, noise = _head_inputs(cuda, bs=1, F=2, seed=1, H=40, W=40, Z=8, per_frame=500, num_way=32)
    kw["tgt_pc_range"] = [-60.0, -60.0, -8.0, -1.0, -1.0, -1.0]
    gt = [torch.cat([p[:, :3] * torch.tensor([0.5, 0.5, 0.5], device=cuda) - torch.tensor([30.0, 30.0, 4.5], device=cuda),
                     p[:, 3:]], 1) for p in gt]
    vals = []
    for fused in (True, False):
        head = _head(2, num_way=32, eval_within_grid=True)
        head.fuse_dense_chamfer = fused
        out = head.loss(dict(next_bev_preds=preds, valid_frames=[0, 1]), gt, gumbels={"dense": noise}, **kw)
        vals.append(float(out["loss.dense_voxel"]))
    assert np.isnan(vals[0]) and np.isnan(vals[1]), vals


def _op_inputs(cuda, bs, F, R0=2500, M=9000, seed=0):
    g = torch.Generator().manual_seed(seed)
    ext = torch.tensor([100.0, 100.0, 16.0])
    dist = 40.0 * torch.rand(bs, F * R0, generator=g)
    dist[torch.rand(bs, F * R0, generator=g) < 0.1] = 0.0
    pts = torch.rand(bs, F * R0, 3, generator=g) * ext
    origin = ext / 2 + torch.randn(bs, F, 3, generator=g)
    gt = torch.rand(bs, M, 3, generator=g) * (ext + 2) - 1
    tindex = torch.randint(-1, F + 1, (bs, M), generator=g).float()
    return [t.to(cuda).contiguous() for t in (dist, pts, origin, gt, tindex)]


def _op_call(inputs, F, **kw):
    dist, pts, origin, gt, tindex = inputs
    return ray_head.dense_chamfer_loss(dist, pts, origin, gt, tindex, (100, 100, 16), [1.0 + 0.1 * f for f in range(F)],
                                       float(sum(1.0 + 0.1 * f for f in range(F))), **kw)


def test_launch_count_is_independent_of_batch_and_frames(cuda):
    counts = []
    for bs, F in ((1, 2), (2, 4)):
        inputs = _op_inputs(cuda, bs, F, seed=bs)
        inputs[0].requires_grad_(True)
        n0 = _lib.launch_count()
        _op_call(inputs, F).backward()
        counts.append(_lib.launch_count() - n0)
    assert counts[0] == counts[1] == 8, counts


def test_two_calls_are_bit_identical(cuda):
    inputs = _op_inputs(cuda, 2, 4, seed=5)
    a, pa = _op_call(inputs, 4, return_pairs=True)
    b, pb = _op_call(inputs, 4, return_pairs=True)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)) and torch.equal(pa.view(torch.int64), pb.view(torch.int64))
    # and the op agrees with the oracle at this size
    want, _ = dense_chamfer_ref.dense_chamfer(*[t.cpu().numpy() for t in inputs], (100, 100, 16),
                                              [1.0 + 0.1 * f for f in range(4)], sum(1.0 + 0.1 * f for f in range(4)))
    assert abs(float(a) - want) <= 1e-5 * abs(want), (float(a), want)


def test_shipped_configuration_has_no_host_sync(cuda):
    """CE + dense (use_dist_loss=False, default noise), forward and backward."""
    preds, gt, kw, _ = _head_inputs(cuda, bs=2, F=2, seed=2, H=40, W=40, Z=8, per_frame=2000, num_way=32)
    head = ViDARRayHead(ray_grid_num=32, loss_weight=np.array([[1.0], [0.5]]))
    p = preds.clone().requires_grad_(True)

    def step():
        out = head.loss(dict(next_bev_preds=p, valid_frames=[0, 1]), gt, **kw)
        sum(out.values()).backward()
        return out
    step()                                          # warm the allocators and the library's pool
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert set(out) == {"regularization.loss", "loss.dense_voxel"}
    assert all(np.isfinite(float(v)) for v in out.values())


def test_ce_with_padded_rays_equals_ce_over_compacted_rays(cuda):
    g = torch.Generator().manual_seed(4)
    F, Z, Y, X, M = 3, 8, 30, 26, 4000
    sigma = torch.randn(2, F, Z, Y, X, generator=g).to(cuda)
    origin = (torch.tensor([X / 2, Y / 2, Z / 2]) + torch.randn(2, F, 3, generator=g)).to(cuda)
    pts = torch.rand(2, M, 3, generator=g) * torch.tensor([X + 2.0, Y + 2.0, Z + 1.0]) - 1
    t = torch.randint(-1, F + 2, (2, M), generator=g).float()                # -1 and F, F+1: no predicted frame
    t[:, ::7] = 1.5                                                           # not a frame index either
    pts[t < 0] = float("nan")
    pts, t = pts.to(cuda), t.to(cuda)
    lw = np.array([[0.5], [1.0], [2.0]])
    s1 = sigma.clone().requires_grad_(True)
    ce = ray_head.ce_regularization_loss(origin, pts, t, [s1], lw, 1.0, 24)
    ce.backward()
    s2 = sigma.clone().requires_grad_(True)
    num, den = 0, 0
    w = torch.tensor(lw, dtype=torch.float32, device=cuda)
    for b in range(2):
        p, fr = ray_head._frame_sorted_rays(pts[b], t[b], F)
        c, valid = ray_head.ray_ce(s2[b], origin[b], p, fr, 24, 1.0)
        wr = w[fr.long(), 0] * valid
        num, den = num + (c * wr).sum(), den + wr.sum()
    ref = num / torch.clamp(den, min=1)
    ref.backward()
    assert abs(float(ce) - float(ref)) <= 1e-6 * abs(float(ref))
    err = (s1.grad - s2.grad).abs().max().item()
    assert err <= 1e-5 * s2.grad.abs().max().item(), err
