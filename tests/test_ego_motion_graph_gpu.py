"""The ego-motion graph on the GPU (`SyntheticViDAR(ego_motion=True)`), at the reduced size of the other pre-training
tests, against independent statements:
  * `predict_future` equals a restatement of the reference's own statements over the same fused modules: the shift
    from get_bev_features (pageable new_tensor, torchvision `rotate` about [100, 100] on the permuted previous BEV,
    the can_bus through can_bus_mlp), BEVFormerEncoder.forward's value schedule with CustomBEVFormerEncoder's restack
    after the LatentRendering layer, `_align_bev_coordnates` with ref_to_history updated per roll-out (vidar.py:
    196-238, 339-363), and the future head's can_bus_mlp over future_can_bus[k][:, (0, 1, 2, 17)];
  * a queue whose first frames come from another scene equals the same sample without those frames, bit for bit;
  * from files with poses, the loader's prefetch 0 and 1 give bit-identical losses;
  * `pretrain.evaluate` with ego motion equals per-sample `forward_test` plus `summarize` bit for bit;
  * sharded over 2 GPUs (skipped on one) the ego-motion step equals the single-GPU one."""
import os
import random

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=3, bev_hw=(40, 40), ray_grid_num=64)
HW = (90, 160)


@pytest.fixture
def exact():
    saved = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
             torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = saved


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def _eval_model(dev, **kw):
    from vidar_b200 import pretrain
    model, _ = pretrain.build(dev, seed=1, config="vidar_1_8_nusc_3future", **dict(SMALL, **kw), ego_motion=True)
    return model.eval()


# ---- restatement of the reference's statements -------------------------------------------------------------------
def _ref_encode(model, feats, shapes, lsi, meta, prev_bev):
    """transformer.py:114-157 + encoder.py:196-243 for bs 1 over the model's own layers."""
    from torchvision.transforms.functional import rotate

    from vidar_b200 import bev_geometry, pretrain
    H, W = model.bev_h, model.bev_w
    Q, dev = H * W, feats.device
    if not meta["prev_bev_exists"]:
        prev_bev = None
    bev_queries = model.bev_embedding.weight
    delta_lidar = np.linalg.inv(meta["lidar2global_rotation"]) @ np.array(meta["can_bus"][:3])
    shift = bev_queries.new_tensor([[delta_lidar[0] / 0.512 / W, delta_lidar[1] / 0.512 / H]])      # bs, xy
    if prev_bev is not None:
        tmp = rotate(prev_bev[0].reshape(H, W, -1).permute(2, 0, 1), meta["can_bus"][-1], center=[100, 100])
        prev_bev = tmp.permute(1, 2, 0).reshape(Q, 1, -1)[:, 0][None]
    can_bus = model.can_bus_mlp(bev_queries.new_tensor([meta["can_bus"]]))
    bev_query = bev_queries[None] + can_bus[:, None]
    bev_pos = model.positional_encoding(1)
    ref_3d = bev_geometry.get_reference_points(H, W, pretrain.PC_RANGE[5] - pretrain.PC_RANGE[2], 4, dim="3d",
                                               bs=1, device=dev)
    ref_2d = bev_geometry.get_reference_points(H, W, dim="2d", bs=1, device=dev)
    ref_cam, bev_mask = bev_geometry.point_sampling(ref_3d, pretrain.PC_RANGE, [meta])
    shift_ref_2d = ref_2d.clone()
    shift_ref_2d += shift[:, None, None, :]
    if prev_bev is not None:
        prev_bev = torch.stack([prev_bev, bev_query], 1).reshape(2, Q, -1)
        hybrid = torch.stack([shift_ref_2d, ref_2d], 1).reshape(2, Q, 1, 2)
    else:
        hybrid = torch.stack([ref_2d, ref_2d], 1).reshape(2, Q, 1, 2)
    bev_shapes, bev_lsi = torch.tensor([[H, W]], device=dev), torch.tensor([0], device=dev)
    for layer in model.encoder:
        value = prev_bev if prev_bev is not None else torch.stack([bev_query, bev_query], 1).reshape(2, Q, -1)
        output = layer(bev_query, feats, bev_pos, hybrid, value, shapes, lsi, ref_cam, bev_mask, bev_shapes, bev_lsi)
        bev_query = output
        if prev_bev is not None and layer.latent_render is not None:
            prev_bev = torch.stack([prev_bev[:1], bev_query], 1).reshape(2, Q, -1)
    return bev_query


def _ref_predict(model, img, lidar2img, metas, future_frames):
    """vidar.py:392-437 (forward_test's prediction) over the restated encoder, with _align_bev_coordnates."""
    from vidar_b200 import bev_geometry, pretrain
    H, W = model.bev_h, model.bev_w
    T = img.shape[1]
    prev_bev = None
    for t in range(T):
        meta = dict(lidar2img=np.asarray(lidar2img[0]), img_shape=[(img.shape[-2], img.shape[-1], 3)], **metas[t])
        feats, shapes, lsi = model.extract_feat(img[:, t])
        prev_bev = _ref_encode(model, feats, shapes, lsi, meta, prev_bev)
    ref_bev = prev_bev
    cur = metas[T - 1]
    feats = [ref_bev.unsqueeze(0).repeat(len(model.bev_pred_head), 1, 1, 1)]
    prev_input = ref_bev.unsqueeze(1)
    r2h = ref_bev.new_tensor(np.array([[cur["ref_lidar_to_cur_lidar"]]]))                       # [bs, 1, 4, 4]
    dev = ref_bev.device
    for k in range(1, future_frames + 1):
        future2ref = r2h.new_tensor(np.array([cur["future2ref_lidar_transform"][k]]))
        ref2future = r2h.new_tensor(np.array([cur["ref2future_lidar_transform"][k]]))
        f2h = torch.matmul(future2ref.unsqueeze(1), r2h)
        grids = bev_geometry.get_bev_grids(H, W, 1, device=dev).view(1, 1, -1, 2)
        coords = bev_geometry.bev_grids_to_coordinates(grids, pretrain.PC_RANGE)
        coords = torch.matmul(torch.cat([coords, torch.ones_like(coords[..., :2])], -1), f2h)[..., :2]
        aligned, _ = bev_geometry.bev_coords_to_grids(coords, H, W, pretrain.PC_RANGE)
        ref_points = ((aligned + 1) / 2.).permute(0, 2, 1, 3)                                       # [bs, Q, 1, 2]
        tgt_points = grids[:, -1][:, :, None]
        can_bus = ref_bev.new_tensor(np.array([cur["future_can_bus"][k]])[:, (0, 1, 2, 17)])
        query = model.future_bev_embedding.weight[None] + model.future_can_bus_mlp(can_bus)[:, None]
        prev = (prev_input + model.prev_frame_embedding[None, :, None, :]).view(1, -1, 256)
        bev_pos = model.future_positional_encoding(1)
        shapes_, lsi_ = torch.tensor([[H, W]], device=dev), torch.tensor([0], device=dev)
        inter = []
        for layer in model.decoder:
            query = layer(query, prev, bev_pos, tgt_points, ref_points, shapes_, lsi_)
            inter.append(query)
        feats.append(torch.stack(inter))
        prev_input = inter[-1].unsqueeze(1)
        r2h = torch.cat([r2h, ref2future.unsqueeze(1)], 1)[:, 1:]
    return model.forward_head(torch.stack(feats, 0))


def _sample(dev, frames=4, future=3, seed=0, scene_change=None):
    from vidar_b200 import pretrain
    return pretrain.synthetic_sample(dev, frames=frames, img_hw=(96, 160), rays_per_frame=800, seed=seed,
                                     bev_hw=(40, 40), future_frames=future, poses=True, scene_change=scene_change)


def test_predict_future_equals_the_reference_statements(cuda, exact):
    model = _eval_model(cuda)
    sample = _sample(cuda, seed=3)
    metas = sample["pose_metas"]
    assert all(m["prev_bev_exists"] for m in metas[1:]) and abs(metas[-1]["can_bus"][-1]) > 0.1
    with torch.no_grad():
        got = model.predict_future(sample["img"], sample["lidar2img"], 3, pose_metas=metas)["next_bev_preds"]
        ref = _ref_predict(model, sample["img"], sample["lidar2img"], metas, 3)
    scale = float(ref.abs().max())
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5 * scale)
    # the metas matter at this size: with the can_bus zeroed (no shift, no rotation) the prediction is far off
    with torch.no_grad():
        still = [dict(m, can_bus=np.zeros(18)) for m in metas]
        moved = model.predict_future(sample["img"], sample["lidar2img"], 3, pose_metas=still)["next_bev_preds"]
    assert (moved - ref).abs().max() > 100 * (got - ref).abs().max() + 1e-6


def test_queue_from_another_scene_equals_the_sample_without_it(cuda, exact):
    from vidar_b200 import ego_motion, synthetic
    model = _eval_model(cuda)
    full = _sample(cuda, frames=4, future=3, seed=7, scene_change=2)
    assert [m["prev_bev_exists"] for m in full["pose_metas"]] == [False, True, False, True]
    drive = synthetic.drive(4 + 3, 7, scene_change=2)[2:]
    short = ego_motion.queue_metas([dict(f, img_filename=()) for f in drive[:2]] + drive[2:])
    with torch.no_grad():
        a = model.predict_future(full["img"], full["lidar2img"], 3, pose_metas=full["pose_metas"])["next_bev_preds"]
        b = model.predict_future(full["img"][:, 2:], full["lidar2img"], 3, pose_metas=short)["next_bev_preds"]
    assert torch.equal(a, b)


def _files_model(dev, lr=2e-4, **kw):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(dev, seed=1, config="vidar_1_8_nusc_3future", lr=lr, grid_mask=True,
                                image_pipeline=True, point_pipeline=True, ego_motion=True, **SMALL, **kw)
    model.image_transforms[1].data_aug_conf = dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160,
                                                   rand_flip=True)
    return model, opt


def test_loader_prefetch_gives_identical_losses_with_poses(cuda, exact):
    from vidar_b200 import pretrain
    queues = [pretrain.synthetic_sample(None, frames=4, img_hw=HW, future_frames=3, points_per_frame=4000, seed=s,
                                        files=True, poses=True, scene_change=1 if s == 1 else None) for s in range(3)]
    losses = {}
    for prefetch in (0, 1):
        model, opt = _files_model(cuda, lr=0.0)
        loader = pretrain.SampleLoader(model, queues, num_workers=1, prefetch=prefetch, seed=9)
        _seed(5)
        out = []
        for sample in loader:
            assert "future_can_bus" in sample["img_metas"][-1][0]
            torch.manual_seed(11)
            loss, _ = pretrain.train_step(model, opt, sample)
            out.append(loss.cpu())
        losses[prefetch] = out
    assert len(losses[0]) == 3 and all(torch.equal(a, b) for a, b in zip(losses[0], losses[1])), losses
    assert all(torch.isfinite(x) for x in losses[0])


def test_evaluate_equals_per_sample_forward_test_with_ego_motion(cuda, exact):
    from vidar_b200 import evaluate, pretrain
    model, _ = pretrain.build(cuda, seed=1, config="vidar_1_8_nusc_3future", grid_mask=True, point_pipeline=True,
                              ego_motion=True, **SMALL)
    model.eval()
    queues = pretrain.synthetic_scene(4, 3, 3, img_hw=HW, points_per_frame=4000, seed=2, poses=True)
    _seed(5)
    loader = pretrain.SampleLoader(model, queues, num_workers=0, prefetch=0, test_mode=True)
    ref = evaluate.summarize([model.forward_test(s["img"], None, s["gt_points"], future_frames=3,
                                                 img_metas=s["img_metas"])[0] for s in loader])
    for prefetch in (0, 1):
        _seed(5)
        got = pretrain.evaluate(model, queues, future_frames=3, prefetch=prefetch)
        assert got.keys() == ref.keys()
        for frame in ref:
            for k, v in ref[frame].items():
                assert np.array_equal(np.float64(got[frame][k]), np.float64(v), equal_nan=True), (prefetch, frame, k)
    assert ref["frame.0"]["count"] > 0


def _grads(model, sample):
    model.zero_grad(set_to_none=True)
    torch.manual_seed(11)
    losses = model.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"], draws=(-1, None),
                                 pose_metas=sample["pose_metas"])
    loss = sum(losses.values())
    loss.backward()
    return float(loss.detach()), {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sample = _sample(dev, seed=4)
    res = []
    for group in (None, dist.group.WORLD):
        model, _ = pretrain.build(dev, group, seed=1, config="vidar_1_8_nusc_3future", ego_motion=True, **SMALL)
        r = _grads(model, sample)
        if group is not None:
            sharding.allreduce_partial_grads(model, dist.group.WORLD)
            r = (r[0], {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None})
        res.append(r)
    if rank == 0:
        torch.save(res, out)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_ego_motion_step_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "e.pt")
    mp.spawn(_worker, args=(2, 29480 + os.getpid() % 100, out), nprocs=2, join=True)
    (l1, g1), (l2, g2) = torch.load(out, weights_only=False)
    assert abs(l1 - l2) <= 1e-4 * abs(l1)
    assert set(g1) == set(g2)
    for n in g1:
        scale = float(g1[n].abs().max())
        torch.testing.assert_close(g2[n], g1[n], rtol=2e-3, atol=2e-4 * scale + 1e-9, msg=lambda m: f"{n}: {m}")
