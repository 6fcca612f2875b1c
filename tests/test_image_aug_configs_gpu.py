"""The memory-efficient pre-training chain (RandomCropResizeFlipImage) and the fine-tuning chain (photometric
distortion straight into normalisation) on the H100, through vidar_b200.image_aug.apply_multiview: bit for bit the
reference's own transforms (tests/golden/image_aug_configs.npz); bit for bit the closed-form oracle on a full
6 x 900 x 1600 frame at the config's nine heights with and without the flip and at two crop offsets, and for the
fine-tuning chain; camera subsets; no host sync, two launches with a crop step and one without."""
import numpy as np
import pytest
import torch

from oracle import image_aug_ref as ref
from tests import image_aug_cases as cases
from tests import image_aug_configs_cases as cfg_cases
from vidar_b200 import _lib
from vidar_b200.image_aug import ImageAugPlan, apply_multiview

pytestmark = pytest.mark.gpu

MEAN, STD = (103.530, 116.280, 123.675), (1.0, 1.0, 1.0)
CONFIG_HEIGHTS = [720, 765, 810, 855, 900, 945, 990, 1035, 1080]


def plan_for(src, photo, dims=None, window=None, flip=False, mean=MEAN, std=STD, to_rgb=False, pad_hw=None,
             pad_val=(0.0, 0.0, 0.0)):
    """A recorded plan of RandomCropResizeFlipImage's chain (dims given) or of the chain without a crop step."""
    n, H, W = src.shape[:3]
    return dict(img_aug=ImageAugPlan(n=n, src_hw=(H, W), photo=photo, crop=(0, 0, W, H) if dims else None, dims=dims,
                                     flip=flip, mean=np.array(mean, np.float32), std=np.array(std, np.float32),
                                     to_rgb=to_rgb, normalized=True, pad_hw=pad_hw, pad_val=pad_val, window=window))


def device_hwc(src, results, cuda, cams=None):
    x = src[cams] if cams is not None else src
    out = apply_multiview(torch.from_numpy(np.ascontiguousarray(x)).to(cuda), results, cams)
    return out.permute(0, 2, 3, 1).cpu().numpy()


def mismatches(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    return int((np.ascontiguousarray(got).view(np.uint32) != np.ascontiguousarray(want).view(np.uint32)).sum())


def test_golden_equals_the_reference_transforms(cuda):
    z, meta = cfg_cases.golden()
    for name, m in meta.items():
        for t, (results, _) in enumerate(cfg_cases.replay(z, name, m)):
            got = device_hwc(z[f"{name}.{t}.src"], results, cuda)
            assert mismatches(got, z[f"{name}.{t}.img"]) == 0, (name, t)


@pytest.fixture(scope="module")
def full_frame():
    """One 6-camera 900 x 1600 frame with bright and dark blocks, six photometric draws, and the distorted pixels
    after numpy's uint8 cast."""
    rng = np.random.default_rng(10)
    src = rng.integers(0, 256, (6, 900, 1600, 3), dtype=np.uint8)
    src[:, 100:200, 300:500] = rng.integers(230, 256, (6, 100, 200, 3))
    src[:, 600:700, 900:1100] = rng.integers(0, 20, (6, 100, 200, 3))
    draws = cases.gate_draws(12)[::11][:6]
    u8 = [ref.to_uint8(ref.photometric(src[n].astype(np.float32), draws[n])) for n in range(6)]
    return src, draws, u8


@pytest.mark.parametrize("h", CONFIG_HEIGHTS)
def test_config_sizes_equal_the_oracle(cuda, full_frame, h):
    """The window is 900 x 1600 of the resized image: bottom rows zero below 900, the bottom 900 rows above it, right
    columns zero below 1600 (left ones after the flip), a drawn x offset above it."""
    src, draws, u8 = full_frame
    w = int(h / 900 * 1600)
    hp, wp = ref.pad_shape(900, 1600, size_divisor=32)
    resized = [ref.resize(u, w, h) for u in u8]
    crop_h, span = max(0, h - 900), max(0, w - 1600)
    for crop_w in sorted({span // 3, max(span - 1, 0)}):
        box = (crop_w, crop_h, crop_w + 1600, crop_h + 900)
        for flip in (False, True):
            got = device_hwc(src, plan_for(src, draws, (w, h), box, flip, pad_hw=(hp, wp)), cuda)
            for n in range(6):
                r = ref.crop(resized[n], box)
                r = r[:, ::-1] if flip else r
                want = ref.pad(ref.normalize(r.astype(np.float32), MEAN, STD, False), (hp, wp))
                assert mismatches(got[n], want) == 0, (h, crop_w, flip, n)


@pytest.mark.parametrize("to_rgb,std,pad_hw,pad_val", [(False, STD, (928, 1600), (0.0, 0.0, 0.0)),
                                                       (True, (58.395, 57.12, 57.375), (912, 1632), (1.5, -2.0, 3.0))])
def test_finetune_chain_equals_the_oracle(cuda, full_frame, to_rgb, std, pad_hw, pad_val):
    src, draws, _ = full_frame
    for photo in (draws, None):
        results = plan_for(src, photo, to_rgb=to_rgb, std=std, pad_hw=pad_hw, pad_val=pad_val)
        got = device_hwc(src, results, cuda)
        for n in range(6):
            want = cfg_cases.pipeline_float(src[n], photo[n] if photo else None, MEAN, std, to_rgb, pad_hw, pad_val)
            assert mismatches(got[n], want) == 0, (photo is None, n)


def test_every_gate_pattern_in_both_chains_equals_the_oracle(cuda):
    draws = cases.gate_draws(13)
    rng = np.random.default_rng(14)
    src = rng.integers(0, 256, (len(draws), 45, 80, 3), dtype=np.uint8)
    src[:, :5] = 255
    src[:, 5:10] = 0
    for results in (plan_for(src, draws, (96, 54), (7, 9, 87, 54), True, pad_hw=(64, 96)),
                    plan_for(src, draws, (64, 36), (0, 0, 80, 45), False, to_rgb=True, pad_hw=(64, 96)),
                    plan_for(src, draws, to_rgb=True, std=(2.0, 1.0, 0.5), pad_hw=(48, 96), pad_val=(1.0, 2.0, 3.0))):
        got = device_hwc(src, results, cuda)
        assert mismatches(got, cfg_cases.oracle_frame(src, results["img_aug"])) == 0


@pytest.mark.parametrize("chain", ["mem_efficient", "finetune"])
def test_camera_subset_uses_the_frames_draws(cuda, chain):
    rng = np.random.default_rng(15)
    src = rng.integers(0, 256, (6, 45, 80, 3), dtype=np.uint8)
    draws = cases.gate_draws(16)[:6]
    results = (plan_for(src, draws, (96, 54), (5, 9, 85, 54), True, pad_hw=(64, 96)) if chain == "mem_efficient"
               else plan_for(src, draws, pad_hw=(64, 96)))
    full = device_hwc(src, results, cuda)
    assert mismatches(device_hwc(src, results, cuda, cams=[4, 1]), full[[4, 1]]) == 0


@pytest.mark.parametrize("chain,launches", [("mem_efficient", 2), ("finetune", 1)])
def test_no_host_sync_and_launch_count(cuda, chain, launches):
    src = torch.randint(0, 256, (6, 900, 1600, 3), dtype=torch.uint8, device=cuda)
    draws = cases.gate_draws(17)[:6]
    results = (plan_for(src, draws, (1856, 1044), (100, 144, 1700, 1044), True, pad_hw=(928, 1600))
               if chain == "mem_efficient" else plan_for(src, draws, pad_hw=(928, 1600)))
    apply_multiview(src, results)                                # warm up: taps upload, pinned allocator
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = apply_multiview(src, results)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() - n0 == launches
    torch.cuda.synchronize()
    assert out.shape == (6, 3, 928, 1600) and torch.isfinite(out).all()
