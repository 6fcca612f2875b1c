"""The OpenScene (nuPlan) pre-training inputs and presets on CPU:
  * the .pcd parse, the nuPlan point transforms and RandomScaleImageMultiViewImage against the reference's own
    statements (tests/golden/openscene.npz, tools/make_golden_openscene.py): points, raised exception classes,
    lidar2img, shapes and numpy's state;
  * the restatement of cv2's INTER_LINEAR 2/3 rescale that the device chain computes equals cv2 on this machine;
  * the 8-camera OpenScene preset sharded over 4 and 8 gloo ranks equals the single-process graph in fp64."""
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "openscene.npz")


@pytest.fixture(scope="module")
def gold():
    g = np.load(GOLDEN)
    return g, json.loads(str(g["meta"]))


def _state_row():
    st = np.random.get_state()
    return np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4])


def test_pcd_parse_matches_the_reference(gold):
    from vidar_b200 import point_pipeline as pp
    g, meta = gold
    for name in ("pcd_small", "pcd_garbage"):
        got = pp.parse_pcd(g[f"{name}.bytes"].tobytes())
        want = g[f"{name}.points"]
        assert got.dtype == np.float32 and got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want).view(np.uint32)), name
    for name, err in meta["errors"].items():
        with pytest.raises(getattr(__builtins__, err, None) or eval(err)):
            pp.parse_pcd(g[f"bad_{name}.bytes"].tobytes())


def test_nuplan_point_transforms_match_the_reference(gold, tmp_path):
    from vidar_b200 import point_pipeline as pp
    g, meta = gold
    q = meta["queue"]
    steps = [pp.LoadNuPlanPointsFromFile("LIDAR"), pp.LoadNuPlanPointsFromMultiSweeps(**q["sweeps_kwargs"]),
             pp.CustomVoxelBasedPointSampler(**q["sampler_kwargs"])]
    np.random.seed(q["seed"])
    states = []
    for f in range(q["frames"]):
        path = tmp_path / f"{f}.pcd"
        g[f"queue.{f}.bytes"].tofile(path)
        results = dict(pts_filename=str(path), timestamp=1.0 + f, sweeps=[])
        for s in steps:
            results = s(results)
            states.append(_state_row()[0])
            if s is steps[1]:
                plan = results["pts_aug"]
                assert len(plan.segments) == 1 and plan.segments[0].filt is None
                seg = plan.segments[0]
                # the reference's points after the multi-sweep step: column 4 := 0, the last column := 0
                raw = seg.raw.copy()
                raw[:, 4] = seg.time
                raw[:, 5] = np.float32(q["sweeps_kwargs"]["hard_sweeps_timestamp"])
                want = g[f"queue.{f}.sweeps_out"]
                assert np.array_equal(raw.view(np.uint32), want.view(np.uint32))
        assert results["pts_aug"].perm.shape == (seg.raw.shape[0],)
    assert np.array_equal(np.stack(states), g["queue.states"])


def test_openscene_pipelines_follow_the_config():
    from vidar_b200 import image_aug, point_pipeline as pp
    load, sweeps, sampler = pp.config_openscene_train_pipeline()
    assert isinstance(load, pp.LoadNuPlanPointsFromFile) and sweeps.sweeps_num == 0 and sweeps.pad_empty_sweeps
    assert sampler.grid == (102, 102, 8) and sampler.max_voxels == 50000
    names = [type(t).__name__ for t in image_aug.config_openscene_pipeline()]
    assert names == ["PhotoMetricDistortionMultiViewImage", "NormalizeMultiviewImage",
                     "RandomScaleImageMultiViewImage", "PadMultiViewImage"]
    assert [type(t).__name__ for t in image_aug.config_openscene_test_pipeline()] == names[1:]
    with pytest.raises(ValueError):
        pp.LoadNuPlanPointsFromMultiSweeps(sweeps_num=2, use_dim=[0, 1, 2, 3, 4, 5])
    with pytest.raises(ValueError):
        image_aug.RandomScaleImageMultiViewImage(scales=[0.5, 2 / 3])


def test_random_scale_matches_the_reference(gold):
    from vidar_b200 import image_aug
    g, meta = gold
    imgs = [np.zeros((96, 150, 3), np.uint8)] * 2
    results = dict(img=imgs, lidar2img=[g["scale.lidar2img_in0"], g["scale.lidar2img_in1"]])
    np.random.seed(meta["scale"]["seed"])
    for t in image_aug.config_openscene_test_pipeline()[:2]:
        results = t(results)
    k, gauss = _state_row()
    assert np.array_equal(k, g["scale.state"]) and gauss == g["scale.gauss"]
    for i in range(2):
        assert np.array_equal(results["lidar2img"][i], g[f"scale.lidar2img{i}"])
    assert [list(s) for s in results["img_shape"]] == meta["scale"]["img_shape"]
    assert [list(s) for s in results["ori_shape"]] == meta["scale"]["ori_shape"]
    assert results["img_aug"].scale_hw == (64, 100)


def rescale_restated(img):
    """cv2.resize(img, 2/3, INTER_LINEAR) on float32 HWC as cv2 with IPP computes it (the device chain's statements):
    along x within each source row, then between the rows, each a + t * (b - a) with one fused multiply-add."""
    H, W = img.shape[:2]
    oh, ow = H * 2 // 3, W * 2 // 3

    def taps(n):
        d = np.arange(n)
        return (3 * d) // 2, np.where(d % 2 == 1, np.float32(0.75), np.float32(0.25)).astype(np.float32)

    def lerp(a, b, t):             # the product exact in float64, one rounding: an fma
        return (t.astype(np.float64) * (b - a).astype(np.float32) + a).astype(np.float32)

    sx, fx = taps(ow)
    sy, fy = taps(oh)
    rows = lerp(img[:, sx], img[:, sx + 1], fx[None, :, None])
    return lerp(rows[sy], rows[sy + 1], fy[:, None, None])


@pytest.mark.parametrize("hw", [(96, 150), (1080, 1920)])
def test_rescale_restatement_equals_cv2(gold, hw):
    cv2 = pytest.importorskip("cv2")
    g, _ = gold
    rng = np.random.default_rng(7)
    img = (rng.standard_normal((*hw, 3)) * 80).astype(np.float32)
    want = cv2.resize(img, (hw[1] * 2 // 3, hw[0] * 2 // 3), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(rescale_restated(img).view(np.uint32), want.view(np.uint32))
    for i in range(2):                                       # and the reference's own mmcv.imresize call
        assert np.array_equal(rescale_restated(g[f"scale.img{i}"]), g[f"scale.out{i}"])


def test_openscene_presets():
    from vidar_b200 import pretrain
    for name in pretrain.OPENSCENE_CONFIGS:
        cfg = pretrain.CONFIGS[name]
        assert (cfg["num_cams"], cfg["history_frames"], cfg["future_frames"], cfg["decoder_layers"]) == (8, 3, 3, 3)
        assert cfg["frame_loss_weight"] == ((1.0,),) * 4 + ((0.0,),) and cfg["openscene"]
    m = pretrain.SyntheticViDAR(**dict(pretrain.CONFIGS[pretrain.OPENSCENE_CONFIGS[0]], bev_hw=(8, 8),
                                       encoder_layers=1, ray_grid_num=16, image_pipeline=True, point_pipeline=True))
    assert m.pred_frame_num == 1 and m.cams_embeds.shape[0] == 8
    assert type(m.point_transforms[0][0]).__name__ == "LoadNuPlanPointsFromFile"
    assert type(m.image_transforms[2]).__name__ == "RandomScaleImageMultiViewImage"


# ---- sharded 8-camera graph (follows tests/test_pretrain_configs_cpu.py) ----
FRAMES, IMG = 4, (32, 64)


def _model():
    from vidar_b200 import pretrain
    from tests.test_pretrain_sharding_cpu import BEV
    torch.manual_seed(3)
    cfg = dict(pretrain.CONFIGS["vidar_OpenScene_mini_1_8_3future"], encoder_layers=2, decoder_layers=1, latent_layer=-1,
               bev_hw=BEV, ray_grid_num=16)
    m = pretrain.SyntheticViDAR(**cfg)
    gen = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if ("sampling_offsets" in n or "attention_weights" in n) and p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=gen) / p.shape[-1] ** 0.5)
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0

    def loss(pred_dict, *a, loss_weight=None, **k):
        p = pred_dict["next_bev_preds"]
        w = torch.as_tensor(loss_weight[: p.shape[0], 0], dtype=p.dtype).view(-1, *[1] * (p.dim() - 1))
        return {"stand_in": (w * p * torch.linspace(0.5, 1.5, p.shape[-1], dtype=p.dtype)).square().mean()}
    m.ray_head.loss = loss
    return m.double()


def _step(m, group):
    from vidar_b200 import sharding
    m.set_process_group(group)
    m.zero_grad(set_to_none=True)
    img = torch.randn(1, FRAMES, 8, 3, *IMG, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    lidar2img = torch.eye(4).repeat(1, 8, 1, 1).numpy()
    losses = m.forward_train(img, lidar2img, [torch.zeros(4, 6)], can_bus=torch.zeros(1, 18, dtype=torch.float64),
                             draws=(-1, None))
    loss = sum(losses.values())
    loss.backward()
    if group is not None:
        sharding.allreduce_partial_grads(m, group)
    return loss.detach(), {n: (None if p.grad is None else p.grad.clone()) for n, p in m.named_parameters()
                           if p.requires_grad}


def _install_8_camera_ops(sharded):
    """tests/test_pretrain_sharding_cpu.py's CPU stand-ins, with its seeded projection drawn for 8 cameras."""
    from tests.test_pretrain_sharding_cpu import D, _install_cpu_ops
    from vidar_b200 import pretrain
    _install_cpu_ops(sharded)

    def point_sampling(ref_3d, pc_range, img_metas):
        g = torch.Generator().manual_seed(5)
        Q = ref_3d.shape[2]
        ref_cam = (torch.rand(8, 1, Q, D, 2, generator=g) * 1.2 - 0.1).to(ref_3d.dtype)
        return ref_cam, torch.rand(8, 1, Q, D, generator=g) < 0.25
    pretrain.bev_geometry.point_sampling = point_sampling


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _install_8_camera_ops(sharded=True)
    res = _step(_model(), dist.group.WORLD)
    if rank in (0, world - 1):
        torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [4, 8])
def test_sharded_openscene_preset_equals_single_process(tmp_path, world):
    out = str(tmp_path / "os.pt")
    mp.spawn(_worker, args=(world, 29800 + os.getpid() % 150 + world, out), nprocs=world, join=True)
    _install_8_camera_ops(sharded=False)
    loss, grads = _step(_model(), None)
    assert all(g is not None for g in grads.values())
    for rank in (0, world - 1):
        got_loss, got = torch.load(f"{out}.{rank}", weights_only=False)
        torch.testing.assert_close(got_loss, loss, rtol=1e-9, atol=1e-12)
        for n, g in grads.items():
            scale = float(g.abs().max())
            torch.testing.assert_close(got[n], g, rtol=1e-6, atol=1e-8 * scale + 1e-16, msg=lambda m_: f"{n}: {m_}")
