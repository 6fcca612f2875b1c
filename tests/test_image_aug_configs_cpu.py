"""The memory-efficient pre-training chain (RandomCropResizeFlipImage: resize, then crop) and the fine-tuning chain
(photometric distortion straight into normalisation) without a GPU: the package's transforms make the reference's
draws, leave numpy and `random` in the same state and set the same keys as tests/golden/image_aug_configs.npz; the
closed-form oracle equals that golden and the reference's cv2 / PIL / numpy statements with 0 differing bits; and
argument errors raise before any CUDA call."""
import numpy as np
import pytest
import torch

from tests import image_aug_cases as cases
from tests import image_aug_configs_cases as cfg_cases
from vidar_b200 import image_aug

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")

MEAN, STD = (103.530, 116.280, 123.675), (1.0, 1.0, 1.0)


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    return int((a.view(np.uint8) != b.view(np.uint8)).sum())


@pytest.fixture(scope="module")
def gold():
    return cfg_cases.golden()


def test_golden_covers_the_cases(gold):
    """Heights below, at and above the crop, both flips, a queue, training=False and the float chains."""
    z, meta = gold
    plans = [(name, results["img_aug"]) for name, m in meta.items()
             for results, _ in cfg_cases.replay(z, name, m)]
    crop = [p for _, p in plans if p.crop is not None]
    wh = [(p.dims[1], p.window[3] - p.window[1]) for p in crop]
    assert {h < fh for h, fh in wh} == {True, False} and any(h == fh for h, fh in wh)
    assert {p.dims[0] < p.window[2] - p.window[0] for p in crop} == {True, False}
    assert {p.flip for p in crop} == {True, False}
    assert any(m["frames"] > 1 and m["crop"] is not None for m in meta.values())
    assert any(m["crop"] is not None and m["crop"].get("training") is False for m in meta.values())
    assert any(p.crop is None and p.photo is not None for _, p in plans)
    assert any(p.crop is None and p.photo is None for _, p in plans)


def test_draws_states_and_keys_equal_the_reference(gold):
    z, meta = gold
    for name, m in meta.items():
        for t, (results, (np_key, np_gauss, rnd)) in enumerate(cfg_cases.replay(z, name, m)):
            key = f"{name}.{t}"
            assert np.array_equal(np_key, z[f"{key}.np_state"]) and np_gauss == z[f"{key}.np_gauss"], key
            assert np.array_equal(rnd, z[f"{key}.random_state"]), key
            if m["crop"] is not None:
                assert np.array_equal(np.stack(results["cam2img"]), z[f"{key}.cam2img"]), key
                assert np.array_equal(np.stack(results["lidar2img"]), z[f"{key}.lidar2img"]), key
                assert results["img_aug"].flip == bool(z[f"{key}.flip"]), key
            else:
                assert "lidar2img" not in results and "aug_param" not in results, key
            for k in ("ori_shape", "img_shape", "pad_shape"):
                assert np.array_equal(np.array(results[k]), z[f"{key}.{k}"]), (key, k)
            assert all(im.dtype == np.uint8 for im in results["img"]), "results['img'] must stay uint8"


def test_oracle_and_statements_reproduce_the_golden(gold):
    z, meta = gold
    for name, m in meta.items():
        for t, (results, _) in enumerate(cfg_cases.replay(z, name, m)):
            src, want = z[f"{name}.{t}.src"], z[f"{name}.{t}.img"]
            assert bits_equal(cfg_cases.oracle_frame(src, results["img_aug"]), want) == 0, (name, t)
            assert bits_equal(cfg_cases.oracle_frame(src, results["img_aug"], statements=True), want) == 0, \
                (name, t)


@pytest.mark.parametrize("dims,box,flip", [((128, 72), (0, 0, 160, 90), True), ((192, 108), (17, 18, 177, 108), False),
                                           ((192, 108), (32, 18, 192, 108), True), ((160, 90), (0, 0, 160, 90), False),
                                           ((175, 100), (10, 5, 150, 85), True), ((144, 81), (-5, -3, 171, 83), True)])
def test_resize_crop_flip_matches_pil(dims, box, flip):
    img = np.random.default_rng(1).integers(0, 256, (90, 160, 3), np.uint8)
    assert bits_equal(cfg_cases.resize_crop_flip(img, dims, box, flip),
                      cfg_cases.resize_crop_flip_statements(img, dims, box, flip).astype(np.uint8)) == 0


@pytest.mark.parametrize("std,to_rgb,shape,pad_val", [(STD, False, None, 0), ((58.395, 57.12, 57.375), True, (96, 192),
                                                                              (1.5, -2.0, 3.0)),
                                                      ((2.0, 1.0, 0.5), True, (96, 176), 2)])
def test_float_chain_matches_statements_for_every_gate_pattern(std, to_rgb, shape, pad_val):
    img = np.random.default_rng(5).integers(0, 256, (16, 64, 3), np.uint8)
    img[0, :8] = 255
    img[1, :8] = 0
    for d in cases.gate_draws(4) + [None]:
        kw = dict(mean=MEAN, std=std, to_rgb=to_rgb, shape=shape, pad_val=pad_val)
        got = cfg_cases.pipeline_float(img, d, **kw)
        assert bits_equal(got, cfg_cases.pipeline_float_statements(img, d, **kw)) == 0, d
    # brightness and contrast push the float chain past 255 and below 0, with no cast
    hot = cfg_cases.pipeline_float(img, image_aug.PhotoDraw(delta=32.0, mode=1, alpha=1.5), MEAN, STD)
    cold = cfg_cases.pipeline_float(img, image_aug.PhotoDraw(delta=-32.0, mode=1, alpha=0.5), MEAN, STD)
    assert (hot + np.float32(MEAN) > 255).any() and (cold + np.float32(MEAN) < 0).any()


@pytest.mark.parametrize("dims,box,flip", [((192, 108), (13, 18, 173, 108), True), ((128, 72), (0, 0, 160, 90), False)])
def test_resize_crop_pipeline_matches_statements(dims, box, flip):
    img = np.random.default_rng(8).integers(0, 256, (90, 160, 3), np.uint8)
    for d in cases.gate_draws(1)[::5]:
        kw = dict(mean=MEAN, std=(2.0, 1.0, 0.5), to_rgb=True, shape=(96, 192), pad_val=1)
        assert bits_equal(cfg_cases.pipeline_resize_crop(img, d, dims, box, flip, **kw),
                          cfg_cases.pipeline_resize_crop_statements(img, d, dims, box, flip, **kw)) == 0


def frame_results(n=2, hw=(90, 160)):
    return dict(img=[np.zeros(hw + (3,), np.uint8)] * n, cam2img=[np.eye(4) for _ in range(n)],
                lidar2cam=[np.eye(4) for _ in range(n)])


def run(steps, results=None):
    results = frame_results() if results is None else results
    for s in steps:
        results = s(results)
    return results


def test_random_crop_draws_and_matrices():
    conf = dict(reisze=[72, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True)
    np.random.seed(3)
    r = run([image_aug.RandomCropResizeFlipImage(conf)])
    resize, dims, crop, flip = r["aug_param"]["CropResizeFlipImage_param"]
    plan = r["img_aug"]
    assert plan.crop == (0, 0, 160, 90) and plan.dims == dims and plan.window == tuple(crop) and plan.hw == (90, 160)
    want = np.array([[resize, 0, -crop[0], 0], [0, resize, -crop[1], 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    assert np.array_equal(r["cam2img"][0], want) and np.array_equal(r["lidar2img"][1], want)
    # a later frame of the queue draws nothing
    state = np.random.get_state()[1].copy()
    r2 = run([image_aug.RandomCropResizeFlipImage(conf)], dict(frame_results(), aug_param=r["aug_param"]))
    assert np.array_equal(np.random.get_state()[1], state) and r2["img_aug"].window == plan.window


def test_argument_errors_raise_without_a_gpu():
    conf = dict(reisze=[72], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=False)
    with pytest.raises(TypeError):
        image_aug.RandomCropResizeFlipImage(conf, debug=False)
    with pytest.raises(ValueError, match="exactly one"):
        run([image_aug.RandomCropResizeFlipImage(dict(conf, reisze=[72, 90]), training=False)])
    with pytest.raises(ValueError, match="overlaps"):
        run([image_aug.RandomCropResizeFlipImage(dict(conf, crop=(200, 0, 360, 90)), training=False)])
    with pytest.raises(ValueError, match="order"):
        run([image_aug.RandomCropResizeFlipImage(conf), image_aug.CropResizeFlipImage(conf)])
    with pytest.raises(ValueError, match="order"):
        run([image_aug.NormalizeMultiviewImage(MEAN, STD), image_aug.RandomCropResizeFlipImage(conf)])
    with pytest.raises(ValueError, match="without CropResizeFlipImage"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8),
                                  run([image_aug.PhotoMetricDistortionMultiViewImage(),
                                       image_aug.PadMultiViewImage(size_divisor=32)]))
    finetune = run([image_aug.PhotoMetricDistortionMultiViewImage(), image_aug.NormalizeMultiviewImage(MEAN, STD),
                    image_aug.PadMultiViewImage(size_divisor=32)])
    with pytest.raises(ValueError, match="uint8"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3), finetune)
    with pytest.raises(ValueError, match="cams"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8), finetune, cams=[0, 2])
    for results in (finetune, run([image_aug.RandomCropResizeFlipImage(conf)])):
        with pytest.raises(ValueError, match="recorded for"):
            image_aug.apply_multiview(torch.zeros(2, 90, 161, 3, dtype=torch.uint8), results)
        with pytest.raises(RuntimeError, match="CUDA"):
            image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8), results)
