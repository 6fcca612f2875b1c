"""The image pipeline on the H100 (csrc/image_aug.cu through vidar_b200.image_aug.apply_multiview): bit for bit the
closed-form oracle (oracle/image_aug_ref.py) at the config's nine output sizes with and without the flip, for every
photometric gate pattern in both modes, at odd sizes, crops reaching outside the frame, BGR -> RGB, std != 1 and the
`size` pad; bit for bit the reference's own transforms (tests/golden/image_aug.npz); no host sync and two launches
per call; and the pre-training harness feeds its backbone exactly the oracle pipeline's images."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import image_aug_ref as ref
from tests import image_aug_cases as cases
from vidar_b200 import _lib
from vidar_b200.image_aug import ImageAugPlan, apply_multiview

pytestmark = pytest.mark.gpu

MEAN, STD = (103.530, 116.280, 123.675), (1.0, 1.0, 1.0)


def plan_for(src, photo, box, dims, flip, mean=MEAN, std=STD, to_rgb=False, pad_hw=None, pad_val=(0.0, 0.0, 0.0)):
    return dict(img_aug=ImageAugPlan(n=src.shape[0], src_hw=tuple(src.shape[1:3]), photo=photo, crop=box, dims=dims,
                                     flip=flip, mean=np.array(mean, np.float32), std=np.array(std, np.float32),
                                     to_rgb=to_rgb, normalized=True, pad_hw=pad_hw, pad_val=pad_val))


def device_hwc(src, results, cuda):
    out = apply_multiview(torch.from_numpy(src).to(cuda), results)
    return out.permute(0, 2, 3, 1).cpu().numpy()


def mismatches(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    return int((np.ascontiguousarray(got).view(np.uint32) != np.ascontiguousarray(want).view(np.uint32)).sum())


@pytest.fixture(scope="module")
def full_frame():
    """One 6-camera 900 x 1600 frame with bright and dark blocks, and six different photometric draws."""
    rng = np.random.default_rng(0)
    src = rng.integers(0, 256, (6, 900, 1600, 3), dtype=np.uint8)
    src[:, 100:200, 300:500] = rng.integers(230, 256, (6, 100, 200, 3))
    src[:, 600:700, 900:1100] = rng.integers(0, 20, (6, 100, 200, 3))
    draws = cases.gate_draws(2)[::11][:6]
    u8 = [ref.to_uint8(ref.photometric(src[n].astype(np.float32), draws[n])) for n in range(6)]
    return src, draws, u8


@pytest.mark.parametrize("h", [720, 765, 810, 855, 900, 945, 990, 1035, 1080])
def test_config_sizes_equal_the_oracle(cuda, full_frame, h):
    src, draws, u8 = full_frame
    w = int(h / 900 * 1600)
    hp, wp = ref.pad_shape(h, w, size_divisor=32)
    resized = [ref.resize(u, w, h) for u in u8]
    for flip in (False, True):
        got = device_hwc(src, plan_for(src, draws, (0, 0, 1600, 900), (w, h), flip, pad_hw=(hp, wp)), cuda)
        for n in range(6):
            r = resized[n][:, ::-1] if flip else resized[n]
            want = ref.pad(ref.normalize(r.astype(np.float32), MEAN, STD, False), (hp, wp))
            assert mismatches(got[n], want) == 0, (h, flip, n)


def test_every_gate_pattern_and_mode_equals_the_oracle(cuda):
    draws = cases.gate_draws(3)
    rng = np.random.default_rng(4)
    src = rng.integers(0, 256, (len(draws), 45, 80, 3), dtype=np.uint8)
    src[:, :5] = 255
    src[:, 5:10] = 0
    results = plan_for(src, draws, (0, 0, 80, 45), (96, 54), True, pad_hw=(64, 96))
    got = device_hwc(src, results, cuda)
    want = cases.oracle_frame(ref, src, results["img_aug"])
    assert mismatches(got, want) == 0


@pytest.mark.parametrize("box,dims,flip,to_rgb,std,pad_hw,pad_val", [
    ((-8, 6, 168, 96), (211, 108), True, True, (58.395, 57.12, 57.375), (128, 224), (1.5, -2.0, 3.0)),
    ((-30, -20, 200, 120), (97, 51), False, False, (2.0, 1.0, 0.5), (64, 128), (5.0, 0.0, 0.0)),
    ((10, 4, 150, 84), (140, 80), True, False, STD, (96, 160), (0.0, 0.0, 0.0)),          # no resample pass
    ((0, 0, 160, 90), (160, 77), False, True, STD, None, (0.0, 0.0, 0.0)),                # vertical only, no pad
    ((0, 0, 160, 90), (123, 90), True, False, STD, (96, 128), (0.0, 0.0, 0.0)),           # horizontal only
    ((3, 1, 164, 92), (1, 1), False, False, STD, (7, 3), (0.0, 0.0, 0.0)),
    ((0, 0, 160, 90), (333, 187), True, True, (0.5, 0.25, 3.0), (192, 352), (0.0, 0.0, 0.0)),
])
def test_odd_sizes_crops_and_options_equal_the_oracle(cuda, box, dims, flip, to_rgb, std, pad_hw, pad_val):
    rng = np.random.default_rng(sum(dims))
    src = rng.integers(0, 256, (6, 90, 160, 3), dtype=np.uint8)
    draws = cases.gate_draws(5)[1::10][:6]
    for photo in (draws, None):
        results = plan_for(src, photo, box, dims, flip, std=std, to_rgb=to_rgb, pad_hw=pad_hw, pad_val=pad_val)
        got = device_hwc(src, results, cuda)
        assert mismatches(got, cases.oracle_frame(ref, src, results["img_aug"])) == 0, photo is None


def test_golden_equals_the_reference_transforms(cuda):
    z, meta = cases.golden()
    for name, m in meta.items():
        for t, (results, _) in enumerate(cases.replay(z, name, m)):
            got = device_hwc(z[f"{name}.{t}.src"], results, cuda)
            assert mismatches(got, z[f"{name}.{t}.img"]) == 0, (name, t)


def test_camera_subset_uses_the_frames_draws(cuda):
    rng = np.random.default_rng(6)
    src = rng.integers(0, 256, (6, 45, 80, 3), dtype=np.uint8)
    results = plan_for(src, cases.gate_draws(6)[:6], (0, 0, 80, 45), (64, 36), True, pad_hw=(64, 64))
    full = device_hwc(src, results, cuda)
    part = apply_multiview(torch.from_numpy(src[[4, 1]]).to(cuda), results, cams=[4, 1])
    assert mismatches(part.permute(0, 2, 3, 1).cpu().numpy(), full[[4, 1]]) == 0


def test_no_host_sync_and_two_launches(cuda):
    src = torch.randint(0, 256, (6, 900, 1600, 3), dtype=torch.uint8, device=cuda)
    results = plan_for(src, cases.gate_draws(7)[:6], (0, 0, 1600, 900), (1440, 810), True, pad_hw=(832, 1440))
    apply_multiview(src, results)                                # warm up: taps upload, pinned allocator
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = apply_multiview(src, results)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() - n0 <= 2
    torch.cuda.synchronize()
    assert out.shape == (6, 3, 832, 1440) and torch.isfinite(out).all()


SMALL = dict(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(20, 20), ray_grid_num=32)
SMALL_CONF = dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True)


def small_pipeline_model(device, group=None):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(device, group, seed=1, image_pipeline=True, **SMALL)
    model.image_transforms[1].data_aug_conf = SMALL_CONF
    sample = pretrain.synthetic_sample(device, frames=3, img_hw=(90, 160), rays_per_frame=300, future_frames=1,
                                       bev_hw=(20, 20), raw_images=True)
    return model, opt, sample


def run_recorded(model, opt, sample, seed):
    """One train_step with numpy and `random` seeded -> (backbone inputs per frame, img_metas per frame)."""
    import random

    from vidar_b200 import pretrain
    seen, metas = [], []
    hook = model.backbone.stem[0].register_forward_hook(lambda mod, inp, out: seen.append(inp[0].detach().clone()))
    encode = model.encode
    model.encode = lambda feats, shapes, lsi, img_metas, *a: (metas.append(img_metas), encode(feats, shapes, lsi,
                                                                                              img_metas, *a))[1]
    np.random.seed(seed)
    random.seed(seed)
    loss, _ = pretrain.train_step(model, opt, sample)
    hook.remove()
    del model.encode
    assert torch.isfinite(loss)
    return seen, metas


def oracle_frames(model, sample, seed):
    import random
    np.random.seed(seed)
    random.seed(seed)
    frames = model.frame_transforms(sample["img"], sample["cam2img"], sample["lidar2cam"])
    src = sample["img"][0].cpu().numpy()
    return frames, [cases.oracle_frame(ref, src[t], r["img_aug"]).transpose(0, 3, 1, 2) for t, r in enumerate(frames)]


def test_pretrain_harness_runs_the_pipeline_on_every_frame(cuda):
    model, opt, sample = small_pipeline_model(cuda)
    seen, metas = run_recorded(model, opt, sample, 10)
    frames, want = oracle_frames(model, sample, 10)
    assert len(seen) == 3 and len(metas) == 3
    dims = frames[0]["img_aug"].dims
    for t in range(3):
        assert frames[t]["img_aug"].dims == dims and frames[t]["img_aug"].flip == frames[0]["img_aug"].flip
        assert torch.equal(seen[t].cpu(), torch.from_numpy(np.ascontiguousarray(want[t]))), t
        scale = dims[1] / 90
        k = sample["cam2img"][0].copy()
        k[:, :2, :3] *= scale
        assert np.array_equal(metas[t][0]["lidar2img"], np.stack(frames[t]["lidar2img"]))
        np.testing.assert_allclose(metas[t][0]["lidar2img"], k @ sample["lidar2cam"][0], rtol=1e-12, atol=1e-9)
        assert metas[t][0]["img_shape"][0] == tuple(want[t].shape[2:]) + (3,)


def test_pipeline_off_leaves_the_model_unchanged(cuda):
    from vidar_b200 import pretrain
    on, _ = pretrain.build(cuda, None, seed=1, image_pipeline=True, **SMALL)
    off, _ = pretrain.build(cuda, None, seed=1, **SMALL)
    assert off.image_transforms is None
    assert on.state_dict().keys() == off.state_dict().keys()
    assert all(torch.equal(a, b) for a, b in zip(on.state_dict().values(), off.state_dict().values()))


def test_pipeline_needs_bs_1_and_raw_frames(cuda):
    model, _, sample = small_pipeline_model(cuda)
    with pytest.raises(ValueError, match="bs 1"):
        model.frame_transforms(sample["img"].expand(2, *sample["img"].shape[1:]), sample["cam2img"],
                               sample["lidar2cam"])
    with pytest.raises(ValueError, match="cam2img"):
        model.frame_transforms(sample["img"], None, None)


def _sharded_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    dev = torch.device("cuda", rank)
    model, opt, sample = small_pipeline_model(dev, dist.group.WORLD)
    seen, metas = run_recorded(model, opt, sample, 10)
    torch.save(dict(cams=model.my_backbone_cams, seen=[s.cpu() for s in seen],
                    lidar2img=[m[0]["lidar2img"] for m in metas]), f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_camera_sharded_harness_equals_single_process(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "sharded")
    mp.spawn(_sharded_worker, args=(2, 29040 + os.getpid() % 200, out), nprocs=2, join=True)
    model, opt, sample = small_pipeline_model(cuda)
    seen, metas = run_recorded(model, opt, sample, 10)
    covered = set()
    for rank in range(2):
        r = torch.load(f"{out}.{rank}", weights_only=False)
        covered |= set(r["cams"])
        for t in range(3):
            assert np.array_equal(r["lidar2img"][t], metas[t][0]["lidar2img"])
            if r["cams"]:
                assert torch.equal(r["seen"][t], seen[t][r["cams"]].cpu()), (rank, t)
    assert covered == set(range(6))
