"""ViDAR evaluation in one batched device pass (ViDARRayHead.evaluate / evaluate_device, csrc/eval_metrics.cu
vidar_eval_decode_clouds): against the reference's own decoded clouds scored by the oracle, against the unfused path
frame_metrics(get_point_cloud_prediction(...)) table row by row, its failure, host syncs, launches, determinism, and
SyntheticViDAR.forward_test."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_ref
from tests import head_cases as hc
from tests import head_v1_cases as hc1
from vidar_b200 import _lib, evaluate
from vidar_b200.head import ViDARRayHead, ViDARRayHeadV1

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "head.npz")
GOLD_V1 = os.path.join(os.path.dirname(__file__), "golden", "head_v1.npz")
V1_DECODED = ("shipped", "no_prev_bev", "valid_0_2")
# library launches of evaluate_device (DESIGN.md 4.9): arg-max 1 + cloud decode 3 + prologue 1 + NN search 2 +
# metrics 2; ViDARRayHeadV1 adds the GT alignment's 3
LAUNCHES, LAUNCHES_V1 = 9, 12


# ------------------------------------------------------------------ inputs
def _base(cuda, **head_kw):
    c = hc.case()
    head = ViDARRayHead(loss_weight=c["loss_weight"], **dict(hc.HEAD_KW, **head_kw))
    args = (dict(next_bev_preds=c["pred_dict"]["next_bev_preds"].to(cuda), valid_frames=[0, 1]),
            [p.to(cuda) for p in c["gt_points"]])
    kw = dict(hc.CALL_KW, batched_origin_points=c["origin"].to(cuda))
    return head, args, kw


def _v1(cuda, name):
    c = hc1.case(name)
    head = ViDARRayHeadV1(loss_weight=c["loss_weight"], **hc1.HEAD_KW)
    pd = dict(c["pred_dict"], next_bev_preds=c["pred_dict"]["next_bev_preds"].to(cuda))
    return head, (pd, [p.to(cuda) for p in c["gt_points"]]), dict(hc1.CALL_KW, img_metas=c["img_metas"])


# anisotropic voxels (1 m x 0.8 m x 1.5 m), like the shipped grid's 0.512 m x 0.512 m x 0.5 m
SEEDED_PC = [-10.0, -8.0, -3.0, 10.0, 8.0, 3.0]
SEEDED_H, SEEDED_W, SEEDED_Z = 20, 20, 4


def _seeded(cuda, bs=2, Fp=3, valid_frames=None, start_idx=0, within=False, seed=0):
    """bs samples of ragged GT rows in shuffled frame order (frames 0 .. Fp, the last one not predicted), one row at
    the origin of its frame (gt_dist == 0), sample 1 without rows of frame start_idx + 1 (an empty cloud), some rows
    outside pc_range."""
    g = torch.Generator().manual_seed(seed)
    preds = torch.randn(Fp, 2, bs, SEEDED_H * SEEDED_W, SEEDED_Z, generator=g)
    origin = 0.6 * torch.randn(bs, Fp, 3, generator=g)
    lo, hi = torch.tensor(SEEDED_PC[:3]) - 1.0, torch.tensor(SEEDED_PC[3:]) + 1.0
    gt = []
    for b in range(bs):
        n = 400 + 90 * b
        xyz = lo + (hi - lo) * torch.rand(n, 3, generator=g)
        t = torch.randint(0, Fp + 1, (n, 1), generator=g).float()
        if b == 1:
            t[t == start_idx + 1] = Fp
        t[5] = start_idx
        xyz[5] = origin[b, 0]
        gt.append(torch.cat([xyz, torch.rand(n, 1, generator=g), t], 1).to(cuda))
    head = ViDARRayHead(ray_grid_num=16, ray_grid_step=0.75, loss_weight=np.ones((Fp, 1)), eval_within_grid=within)
    pd = dict(next_bev_preds=preds.to(cuda), valid_frames=list(range(Fp)) if valid_frames is None else valid_frames)
    kw = dict(start_idx=start_idx, tgt_bev_h=SEEDED_H, tgt_bev_w=SEEDED_W, tgt_pc_range=SEEDED_PC,
              batched_origin_points=origin.to(cuda))
    return head, (pd, gt), kw


SEEDED = {
    "shuffled_padded": dict(),
    "subset_start_1": dict(valid_frames=[0, 2], start_idx=1),
    "start_1": dict(start_idx=1),
    "within_grid": dict(within=True),
    "bs1_f2": dict(bs=1, Fp=2),
}


def _unfused_table(head, args, kw):
    dec = head.get_point_cloud_prediction(*args, **kw)
    return evaluate.frame_metrics_device(dec["pred_pcds"], dec["gt_pcds"], dec["origin"], kw["tgt_pc_range"]), dec


EXACT, SUMS = [2, 4, 6, 7], [0, 1, 3, 5]       # counts and flags; fp64 sums of l1, absrel and both Chamfer terms


def _assert_same_table(fused, unfused):
    """Counts and flags bit for bit; the sums to 1e-6 relative.  The unfused path takes each norm
    sqrt(sum(r ** 2)) with torch's CUDA sum over the 3 coordinates, whose addition order follows the row's alignment
    in memory; the kernel always adds (x^2 + y^2) + z^2, so a point can differ in its last bit."""
    a, b = fused.cpu().numpy(), unfused.cpu().numpy()
    assert a.shape == b.shape
    np.testing.assert_array_equal(a[:, EXACT], b[:, EXACT])
    np.testing.assert_allclose(a[:, SUMS], b[:, SUMS], rtol=1e-6, atol=0)


# ------------------------------------------------------------------ 1. against the reference
def _check_against_oracle(ret, pred_pcds, gt_pcds, origin, pc_range):
    ref = eval_ref.frame_metrics(pred_pcds, gt_pcds, origin, pc_range)
    assert ret.keys() == ref.keys()
    for k, d in ref.items():
        assert ret[k]["count"] == d["count"] == len(pred_pcds)
        for m in ("chamfer_distance", "l1_error", "absrel_error"):
            np.testing.assert_allclose(ret[k][m], d[m], rtol=1e-4, err_msg=f"{k} {m}")


def test_base_head_matches_oracle_on_reference_clouds(cuda):
    g = np.load(GOLD)
    head, args, kw = _base(cuda)
    ret = head.evaluate(*args, **kw)
    clouds = {key: [[g[f"{key}_{b}_{t}"] for t in range(hc.FRAMES)] for b in range(hc.BS)]
              for key in ("pred_pcds", "gt_pcds")}
    _check_against_oracle(ret, clouds["pred_pcds"], clouds["gt_pcds"], hc.case()["origin"].numpy(), hc.PC_RANGE)


@pytest.mark.parametrize("name", V1_DECODED)
def test_v1_head_matches_oracle_on_reference_clouds(cuda, name):
    g = np.load(GOLD_V1)
    if f"{name}/pred_pcds_0_0" not in g.files:
        pytest.skip(f"no decoded clouds for {name}")
    head, args, kw = _v1(cuda, name)
    ret = head.evaluate(*args, **kw)
    F = len(hc1.CASES[name]["valid_frames"])
    clouds = {key: [[g[f"{name}/{key}_{b}_{t}"] for t in range(F)] for b in range(hc1.BS)]
              for key in ("pred_pcds", "gt_pcds")}
    _check_against_oracle(ret, clouds["pred_pcds"], clouds["gt_pcds"], g[f"{name}/origin"], hc1.PC_RANGE)


# ------------------------------------------------------------------ 2. against the unfused path
def test_base_head_table_equals_unfused(cuda):
    head, args, kw = _base(cuda)
    unfused, _ = _unfused_table(head, args, kw)
    _assert_same_table(head.evaluate_device(*args, **kw), unfused)


@pytest.mark.parametrize("name", V1_DECODED)
def test_v1_head_table_equals_unfused(cuda, name):
    head, args, kw = _v1(cuda, name)
    unfused, _ = _unfused_table(head, args, kw)
    _assert_same_table(head.evaluate_device(*args, **kw), unfused)


@pytest.mark.parametrize("name", list(SEEDED))
def test_seeded_table_equals_unfused(cuda, name):
    head, args, kw = _seeded(cuda, **SEEDED[name])
    unfused, dec = _unfused_table(head, args, kw)
    fused = head.evaluate_device(*args, **kw)
    _assert_same_table(fused, unfused)
    sizes = [[int(p.shape[0]) for p in row] for row in dec["gt_pcds"]]
    assert sum(map(sum, sizes)) > 100
    if name != "bs1_f2":
        assert sizes[1][1] == 0                              # sample 1 has no GT rows of frame start_idx + 1
        ret = head.evaluate(*args, **kw)
        key = f"frame.{1 + kw['start_idx']}"
        assert ret[key]["count"] == len(sizes) and np.isnan(ret[key]["l1_error"])


def test_seeded_row_at_the_origin_is_left_out(cuda):
    head, (pd, gt), kw = _seeded(cuda)
    dec = head.get_point_cloud_prediction(pd, gt, **kw)
    # every other row of frame 0 of sample 0 has gt_dist > 0 (within_grid is off)
    assert int((gt[0][:, -1] == 0).sum()) - 1 == int(dec["gt_pcds"][0][0].shape[0])
    assert bool(torch.isfinite(dec["gt_pcds"][0][0]).all())


# ------------------------------------------------------------------ 3. failure
def test_no_kept_pred_point_raises_like_the_unfused_path(cuda):
    head, args, kw = _base(cuda, ray_grid_step=1e-4)      # every waypoint within 2e-3 m of the origin
    with pytest.raises(ValueError) as unfused:
        dec = head.get_point_cloud_prediction(*args, **kw)
        evaluate.frame_metrics(dec["pred_pcds"], dec["gt_pcds"], dec["origin"], kw["tgt_pc_range"])
    with pytest.raises(ValueError) as fused:
        head.evaluate(*args, **kw)
    assert str(fused.value) == str(unfused.value) and "no pred point" in str(fused.value)


# ------------------------------------------------------------------ 4. host syncs and launches
def _device_part(head, args, kw):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = head.evaluate_device(*args, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


def test_device_part_has_no_host_sync_and_a_fixed_launch_count(cuda):
    counts = []
    for bs in (1, 2):
        for Fp in (2, 3):
            head, args, kw = _seeded(cuda, bs=bs, Fp=Fp)
            out, n = _device_part(head, args, kw)
            assert tuple(out.shape) == (bs * Fp, evaluate.FIELDS)
            counts.append(n)
    assert counts == [LAUNCHES] * 4, counts
    for name in ("shipped", "valid_0_2"):
        _, n = _device_part(*_v1(cuda, name))
        assert n == LAUNCHES_V1, (name, n)


# ------------------------------------------------------------------ 5. determinism
def test_two_calls_give_the_same_bits(cuda):
    for head, args, kw in (_seeded(cuda, within=True), _v1(cuda, "shipped")):
        a = head.evaluate_device(*args, **kw).cpu()
        b = head.evaluate_device(*args, **kw).cpu()
        assert torch.equal(a, b)


# ------------------------------------------------------------------ 6. the model
SMALL = dict(encoder_layers=3, decoder_layers=2, future_frames=2, bev_hw=(40, 40), ray_grid_num=64)
FUTURE = 6
SAMPLE = dict(frames=2, img_hw=(96, 160), rays_per_frame=800, future_frames=FUTURE, bev_hw=(40, 40))


def test_synthetic_forward_test(cuda, monkeypatch):
    from vidar_b200 import pretrain
    model, _ = pretrain.build(cuda, None, seed=1, **SMALL)
    s = pretrain.synthetic_sample(cuda, **SAMPLE)
    (ret,) = model.forward_test(s["img"], s["lidar2img"], s["gt_points"], future_frames=FUTURE)
    assert list(ret) == [f"frame.{t}" for t in range(1 + FUTURE)]
    for k, d in ret.items():
        assert d["count"] == 1 and all(np.isfinite(d[m]) for m in ("chamfer_distance", "l1_error", "absrel_error")), k

    # the same prediction scored through the reference-signature API
    pred = model.predict_future(s["img"], s["lidar2img"], FUTURE)
    assert tuple(pred["next_bev_preds"].shape[:3]) == (1 + FUTURE, 2, model.pred_frame_num)
    monkeypatch.setattr(model, "predict_future", lambda *a, **k: pred)
    (fused,) = model.forward_test(s["img"], s["lidar2img"], s["gt_points"], future_frames=FUTURE)
    cur = dict(pred, next_bev_preds=pred["next_bev_preds"][:, :, model.history_frames])
    dec = model.ray_head.get_point_cloud_prediction(cur, s["gt_points"], 0, model.bev_h, model.bev_w, pretrain.PC_RANGE)
    ref = evaluate.frame_metrics(dec["pred_pcds"], dec["gt_pcds"], dec["origin"], pretrain.PC_RANGE)
    assert fused.keys() == ref.keys()
    for k, d in ref.items():
        assert fused[k]["count"] == d["count"]
        for m in ("chamfer_distance", "l1_error", "absrel_error"):
            np.testing.assert_allclose(fused[k][m], d[m], rtol=1e-6, err_msg=f"{k} {m}")
