"""The point pipeline on the H100 (csrc/point_pipeline.cu through vidar_b200.point_pipeline.gather_gt_points):
bit for bit the reference's own statements (tests/golden/point_pipeline.npz) and the oracle, in the compact and the
padded forms; the device's per-frame counts equal the host's; repeatable bytes; no host sync on the padded path;
the heads' loss and evaluation take the padded form as they take the reference's tensor; and the pre-training
harness builds its gt_points this way."""
import numpy as np
import pytest
import torch

from oracle import point_pipeline_ref as ref
from tests import point_pipeline_cases as cases
from vidar_b200 import point_pipeline as pp

pytestmark = pytest.mark.gpu

Z, METAS = cases.golden()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def cuda():
    return torch.device("cuda", 0)


@pytest.mark.parametrize("meta", METAS, ids=[m["name"] for m in METAS])
def test_device_equals_golden_and_oracle(meta, cuda, tmp_path):
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    plans = [pp.frame_plan(r) for r in gathered]
    want = Z[f"{meta['name']}.gt"]
    compact = pp.gather_gt_points(gathered, meta["ego_mask"], cuda, compact=True).cpu().numpy()
    assert compact.shape == want.shape and np.array_equal(bits(compact), bits(want))
    padded, counts = pp.gather_gt_points(gathered, meta["ego_mask"], cuda, return_counts=True)
    padded = padded.cpu().numpy()
    oracle_padded = ref.gather(plans, meta["ego_mask"], padded=True)
    assert padded.shape == (1,) + oracle_padded.shape
    assert np.array_equal(bits(padded[0]), bits(oracle_padded))                 # NaN rows included
    assert np.array_equal(bits(padded[0][~np.isnan(padded[0, :, 0])]), bits(want))
    host_merged = [sum(s.n_keep for s in p.current()) for p in plans]
    assert counts.cpu().numpy()[:, 0].tolist() == host_merged
    assert np.array_equal(counts.cpu().numpy(), ref.counts(plans))


def test_repeatable_and_no_sync_on_padded_path(cuda, tmp_path):
    meta = next(m for m in METAS if m["name"] == "queue3")
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    a = pp.gather_gt_points(gathered, meta["ego_mask"], cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = pp.gather_gt_points(gathered, meta["ego_mask"], cuda)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))


def test_launches_do_not_depend_on_frames(cuda, tmp_path):
    from vidar_b200 import _lib
    meta = next(m for m in METAS if m["name"] == "queue3")
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    n = []
    for frames in (gathered[:1], gathered):
        n0 = _lib.launch_count()
        pp.gather_gt_points(frames, meta["ego_mask"], cuda)
        n.append(_lib.launch_count() - n0)
    assert n[0] == n[1]


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return bool(np.array_equal(np.asarray(a), np.asarray(b)))


def test_heads_take_the_padded_form(cuda, tmp_path):
    """The padded gt_points (NaN rows inside and after each frame's rows) give the heads' losses and evaluation
    bit for bit what the compact reference tensor gives: a 9-frame queue (the config case's frame repeated) against
    ViDARRayHeadV1's shipped structure and ViDARRayHead."""
    from tests import head_v1_cases as hc
    from vidar_b200.head import ViDARRayHead, ViDARRayHeadV1
    meta = METAS[0]
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    queue = gathered * hc.N_FRAMES
    padded = pp.gather_gt_points(queue, meta["ego_mask"], cuda)
    compact = pp.gather_gt_points(queue, meta["ego_mask"], cuda, compact=True)
    assert torch.isnan(padded).any()
    c = hc.case("shipped", bs=1)
    v1 = ViDARRayHeadV1(loss_weight=c["loss_weight"], **hc.HEAD_KW)
    pd = dict(c["pred_dict"], next_bev_preds=c["pred_dict"]["next_bev_preds"].to(cuda))
    res = []
    for gt in (padded, [compact]):
        torch.manual_seed(0)
        losses = v1.loss(pd, gt, pred_frame_num=None, img_metas=c["img_metas"], **hc.CALL_KW)
        ev = v1.evaluate(pd, gt, img_metas=c["img_metas"], **hc.CALL_KW)
        res.append((losses, ev))
    assert _same(res[0][0], res[1][0])
    assert _same(res[0][1], res[1][1])
    head = ViDARRayHead(ray_grid_num=hc.RAY_GRID_NUM, ray_grid_step=1.0, use_ce_loss=True, use_dist_loss=False,
                        use_dense_loss=True, loss_weight=[[1.0]] * 4)
    g = torch.Generator(device=cuda).manual_seed(1)
    pd0 = dict(next_bev_preds=torch.randn(4, 1, 1, hc.BEV_H * hc.BEV_W, hc.Z, device=cuda, generator=g),
               valid_frames=[0, 1, 2, 3])
    res = []
    for gt in (padded, [compact]):
        torch.manual_seed(0)
        losses = head.loss(pd0, gt, 0, hc.BEV_H, hc.BEV_W, hc.PC_RANGE, pred_frame_num=4)
        ev = head.evaluate(pd0, gt, 0, hc.BEV_H, hc.BEV_W, hc.PC_RANGE)
        res.append((losses, ev))
    assert _same(res[0][0], res[1][0])
    assert _same(res[0][1], res[1][1])


SMALL = dict(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(40, 40), ray_grid_num=64)


def test_pretrain_step_builds_gt_points_on_the_device(cuda):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(cuda, None, seed=1, point_pipeline=True, **SMALL)
    sample = pretrain.synthetic_sample(cuda, frames=2, img_hw=(96, 160), rays_per_frame=500,
                                       future_frames=SMALL["future_frames"], bev_hw=SMALL["bev_hw"], raw_points=True,
                                       points_per_frame=5000)
    np.random.seed(0)
    loss, _ = pretrain.train_step(model, opt, sample)
    assert torch.isfinite(loss)
    gt = model.gt_points_of(sample["point_infos"], training=True)
    assert gt.shape[0] == 1 and gt.shape[2] == 5
    frames = gt[0, :, 4][~torch.isnan(gt[0, :, 0])]
    assert set(frames.unique().tolist()) == set(float(i) for i in range(1 + SMALL["future_frames"]))
