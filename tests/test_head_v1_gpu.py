"""ViDARRayHeadV1 (every head frame in one batched pass) on the GPU against goldens from the REFERENCE
ViDARHeadV1.loss / get_point_cloud_prediction (tools/make_golden_head_v1.py) and against its own per-head-frame
loop (fuse_head_frames=False)."""
import os

import numpy as np
import pytest
import torch

from tests import head_v1_cases as hc
from tests.parity import close
from vidar_b200 import _lib, ray_head
from vidar_b200.head import ViDARRayHeadV1

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "head_v1.npz")


def _setup(cuda, name, bs=hc.BS, head_frames=hc.HEAD_FRAMES):
    c = hc.case(name, bs=bs)
    kw = dict(hc.HEAD_KW)
    if head_frames != hc.HEAD_FRAMES:      # keep the current frame and one future frame, fewer history frames
        kw.update(pred_history_frame_num=head_frames - 2, per_frame_loss_weight=kw["per_frame_loss_weight"][-head_frames:])
    head = ViDARRayHeadV1(loss_weight=c["loss_weight"], **kw)
    preds = c["pred_dict"]["next_bev_preds"][:, :, -head_frames:].contiguous().to(cuda).requires_grad_(True)
    pd = dict(c["pred_dict"], next_bev_preds=preds)
    gt = [p.to(cuda) for p in c["gt_points"]]
    return head, pd, gt, c["img_metas"]


def _noise(g, name, cuda):
    """The reference's Gumbel draws in the per-head-frame layout ({'dense': [bs, frames*R0, K]} per loss index).
    Frames of zero weight, whose noise changes nothing, get zeros."""
    src = hc.SAME_DRAWS.get(name, name)
    V = len(hc.CASES[name]["valid_frames"])
    R0 = (hc.BEV_H // 4) * (hc.BEV_W // 4) * (hc.Z // 4)
    out = []
    for idx in range(hc.HEAD_FRAMES):
        noise = torch.zeros(hc.BS, V * R0, hc.RAY_GRID_NUM)
        frames = hc.weighted_frames(src, idx)
        if frames:
            stored = torch.from_numpy(g[f"{src}/gumbel_dense_{idx}"])
            for k, t in enumerate(frames):
                noise[:, t * R0:(t + 1) * R0] = stored[:, k * R0:(k + 1) * R0]
        out.append({"dense": noise.to(cuda)})
    return out


def _ref_grad(g, name):
    """Reference gradient in the last intermediate output (see head_v1_cases.SAME_DRAWS)."""
    src = hc.SAME_DRAWS.get(name)
    if src is None:
        return g[f"{name}/grad_preds_last"]
    phf = hc.HEAD_KW["pred_history_frame_num"]
    ref = np.zeros_like(g[f"{src}/grad_preds_last"])
    ref[:, phf] = g[f"{src}/grad_preds_last"][:, phf]
    return ref


def _run(head, pd, gt, metas, gumbels=None):
    losses = head.loss(pd, gt, pred_frame_num=None, img_metas=metas, gumbels=gumbels, **hc.CALL_KW)
    sum(losses.values()).backward()
    return losses, pd["next_bev_preds"].grad


@pytest.mark.parametrize("name", list(hc.CASES))
def test_loss_keys_and_gradient_match_reference(cuda, name):
    g = np.load(GOLD)
    head, pd, gt, metas = _setup(cuda, name)
    losses, grad = _run(head, pd, gt, metas, _noise(g, name, cuda))
    ref_keys = {k.split("/", 2)[2] for k in g.files if k.startswith(f"{name}/loss/")}
    assert set(losses) == ref_keys and len(ref_keys) == 2 * hc.HEAD_FRAMES
    for k, v in losses.items():
        np.testing.assert_allclose(float(v.detach()), float(g[f"{name}/loss/{k}"]), rtol=1e-4, err_msg=k)
    ref = _ref_grad(g, name)
    err = np.abs(grad[:, -1].cpu().numpy() - ref).max()
    assert err <= 1e-4 * np.abs(ref).max(), f"grad wrt next_bev_preds: max err {err:.3e} vs {np.abs(ref).max():.3e}"
    assert float(grad[:, :-1].abs().sum()) == 0          # only the last intermediate output is supervised


@pytest.mark.parametrize("name", ["shipped", "valid_0_2"])
def test_point_cloud_prediction_matches_reference(cuda, name):
    g = np.load(GOLD)
    head, pd, gt, metas = _setup(cuda, name)
    with torch.no_grad():
        dec = head.get_point_cloud_prediction(pd, gt, img_metas=metas, **hc.CALL_KW)
    np.testing.assert_allclose(dec["origin"].cpu().numpy(), g[f"{name}/origin"], rtol=1e-5, atol=1e-5)
    n = 0
    for key in ("pred_pcds", "gt_pcds"):
        for b in range(hc.BS):
            for t in range(len(pd["valid_frames"])):
                ref = g[f"{name}/{key}_{b}_{t}"]
                out = dec[key][b][t].cpu().numpy()
                assert out.shape == ref.shape
                np.testing.assert_allclose(out, ref, rtol=1e-4, atol=1e-4)
                n += ref.shape[0]
    assert n > 100


@pytest.mark.parametrize("name", list(hc.CASES))
def test_batched_equals_per_head_frame_loop(cuda, name):
    g = np.load(GOLD)
    res = []
    for fused in (True, False):
        head, pd, gt, metas = _setup(cuda, name)
        head.fuse_head_frames = fused
        losses, grad = _run(head, pd, gt, metas, _noise(g, name, cuda))
        res.append(({k: float(v.detach()) for k, v in losses.items()}, grad.clone()))
    assert res[0][0].keys() == res[1][0].keys()
    for k, v in res[1][0].items():
        assert abs(res[0][0][k] - v) <= 1e-5 * abs(v), (k, res[0][0][k], v)
    close(res[0][1], res[1][1], "grad wrt next_bev_preds")


def test_alignment_equals_masked_statements(cuda):
    """_get_reference_gt_points (one alignment op) returns the rows and origins of the reference's boolean-mask
    statements, bit for bit, in the same order."""
    head, pd, gt, metas = _setup(cuda, "shipped")
    vf = np.array(pd["valid_frames"])
    src, tgt = vf + hc.HISTORY_QUEUE_LENGTH - 3 + 1, vf + hc.HISTORY_QUEUE_LENGTH
    rows, origin = head._get_reference_gt_points(gt, src, tgt, metas)
    rows_t, origin_t = head._align_torch(gt, src, tgt, metas)
    assert torch.equal(origin, origin_t) and tuple(origin.shape) == (hc.BS, len(vf), 3)
    for a, b in zip(rows, rows_t):
        assert a.shape == b.shape and a.shape[0] > 100
        assert torch.equal(a, b)


def test_shipped_configuration_runs_without_host_sync(cuda):
    head, pd, gt, metas = _setup(cuda, "shipped")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = head.loss(pd, gt, pred_frame_num=None, img_metas=metas, **hc.CALL_KW)
        sum(losses.values()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(np.isfinite(float(v.detach())) for v in losses.values())


def test_launch_count_is_fixed():
    cuda = torch.device("cuda")
    counts = []
    for bs, head_frames, name in ((1, 5, "shipped"), (2, 5, "shipped"), (1, 3, "valid_0_2")):
        head, pd, gt, metas = _setup(cuda, name, bs=bs, head_frames=head_frames)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        _run(head, pd, gt, metas)
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - n0)
    assert counts[0] == counts[1] == counts[2], counts


def test_zero_weight_pairs_are_skipped(cuda, monkeypatch):
    seen = {}
    gumbel, chamfer = ray_head.gumbel_distance, ray_head.dense_chamfer_group_loss

    def rec_gumbel(sigma, origin, points, frame, *a):
        seen["rays"] = points.shape[0]
        return gumbel(sigma, origin, points, frame, *a)

    def rec_chamfer(dist, points, origin, gt, gt_tindex, grid, pairs, *a, **k):
        seen["pairs"] = len(pairs)
        return chamfer(dist, points, origin, gt, gt_tindex, grid, pairs, *a, **k)

    monkeypatch.setattr(ray_head, "gumbel_distance", rec_gumbel)
    monkeypatch.setattr(ray_head, "dense_chamfer_group_loss", rec_chamfer)
    head, pd, gt, metas = _setup(cuda, "shipped")
    _run(head, pd, gt, metas)
    R0 = (hc.BEV_H // 4) * (hc.BEV_W // 4) * (hc.Z // 4)
    # 4 weighted frames of the current head frame + the first frame of each of the 4 auxiliary ones
    assert seen == {"rays": 8 * R0 * hc.BS, "pairs": 8 * hc.BS}


def test_two_calls_give_the_same_loss_bits(cuda):
    g = np.load(GOLD)
    out = []
    for _ in range(2):
        head, pd, gt, metas = _setup(cuda, "shipped")
        losses, _ = _run(head, pd, gt, metas, _noise(g, "shipped", cuda))
        out.append(torch.stack([v.detach() for v in losses.values()]).cpu())
    assert torch.equal(out[0], out[1])
