"""The image pipeline's host side and its closed-form oracle (oracle/image_aug_ref.py), without a GPU: the oracle
equals the reference's cv2 / PIL / numpy statements bit for bit (resample, HSV both ways, normalisation, padding,
the wrapping uint8 cast), it reproduces the golden written by the reference's own transforms, and the package's
transforms make the reference's draws, leave numpy and `random` in the same state and set the same keys.  Argument
errors raise before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import image_aug_ref as ref
from tests import image_aug_cases as cases
from vidar_b200 import image_aug
from vidar_b200.image_aug import PhotoDraw

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")

CONFIG_HEIGHTS = [720, 765, 810, 855, 900, 945, 990, 1035, 1080]


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    return int((a.view(np.uint8) != b.view(np.uint8)).sum())


def pil_resize(img, w, h):
    return np.asarray(Image.fromarray(img).resize((w, h)))


@pytest.fixture(scope="module")
def frame():
    return np.random.default_rng(0).integers(0, 256, (900, 1600, 3), dtype=np.uint8)


@pytest.mark.parametrize("h", CONFIG_HEIGHTS)
def test_resample_matches_pillow_at_config_sizes(frame, h):
    w = int(h / 900 * 1600)
    assert bits_equal(ref.resize(frame, w, h), pil_resize(frame, w, h)) == 0


@pytest.mark.parametrize("size", [(1600, 700), (1600, 1111), (1234, 900), (2001, 900), (37, 11), (161, 93),
                                  (1, 1), (3, 2000)])
def test_resample_matches_pillow_one_axis_and_odd_sizes(size):
    img = np.random.default_rng(sum(size)).integers(0, 256, (90 if size[1] < 900 else 900, 160 if size[0] < 1234
                                                                                          else 1600, 3), np.uint8)
    assert bits_equal(ref.resize(img, *size), pil_resize(img, *size)) == 0


@pytest.mark.parametrize("box,dims,flip", [((0, 0, 160, 90), (128, 72), True), ((-10, 5, 150, 100), (211, 108), False),
                                           ((10, 4, 150, 84), (140, 80), True), ((-30, -20, 200, 120), (97, 51), True),
                                           ((0, 0, 160, 90), (160, 90), False)])
def test_crop_resize_flip_matches_pil(box, dims, flip):
    img = np.random.default_rng(1).integers(0, 256, (90, 160, 3), np.uint8)
    assert bits_equal(ref.crop_resize_flip(img, box, dims, flip),
                      ref.crop_resize_flip_statements(img, box, dims, flip).astype(np.uint8)) == 0


def test_package_taps_equal_the_oracle_taps():
    for n_in, n_out in [(1600, 1280), (1600, 1920), (900, 720), (900, 1080), (90, 72), (160, 211), (11, 37), (5, 1)]:
        xmin, cnt, kk = ref.resample_taps(n_in, n_out)
        t = image_aug.bicubic_taps(n_in, n_out)
        assert np.array_equal(t[:, 0], xmin) and np.array_equal(t[:, 1], cnt) and np.array_equal(t[:, 2:], kk)


def hsv_inputs():
    """BGR float32 rows of width 1024 (a multiple of cv2's vector width): random values over the photometric range,
    grey pixels, two equal channels in every position, negative v, small integers (ties)."""
    rng = np.random.default_rng(2)
    x = (rng.random((64, 1024, 3)) * 480 - 48).astype(np.float32)
    x[0] = x[0, :, :1]                                   # grey
    x[1, :, 1] = x[1, :, 0]
    x[2, :, 2] = x[2, :, 1]
    x[3, :, 0] = x[3, :, 2]
    x[4] = -np.abs(x[4])                                 # negative v
    x[5:9] = rng.integers(-3, 4, (4, 1024, 3))           # ties and zeros
    x[9] = np.round(x[9])
    return x


def test_bgr2hsv_matches_cv2():
    x = hsv_inputs()
    assert bits_equal(ref.bgr2hsv(x), cv2.cvtColor(x, cv2.COLOR_BGR2HSV)) == 0


def test_hsv2bgr_matches_cv2():
    rng = np.random.default_rng(3)
    hsv = cv2.cvtColor(hsv_inputs(), cv2.COLOR_BGR2HSV)
    hsv[..., 1] *= np.float32(1.5)
    hsv[10:20, :, 0] = (rng.random((10, 1024)) * 360).astype(np.float32)
    hsv[20, :, 0] = np.float32(360)
    hsv[21, :, 0] = np.float32(0)
    hsv[22, :, 0] = np.resize(np.arange(0, 361, 60, dtype=np.float32), 1024)          # sector boundaries
    hsv[23, :, 0] = np.nextafter(hsv[22, :, 0], np.float32(0))
    hsv[24, :, 1] = 0                                                                # s == 0
    assert bits_equal(ref.hsv2bgr(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)) == 0


def test_fmaf_emulation_is_exact():
    libm = ctypes.CDLL("libm.so.6")
    libm.fmaf.restype, libm.fmaf.argtypes = ctypes.c_float, [ctypes.c_float] * 3
    rng = np.random.default_rng(4)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) * np.float32(10.0) ** rng.integers(-8, 8, 20000)
               .astype(np.float32) for _ in range(3))
    want = np.array([libm.fmaf(*v) for v in zip(a.tolist(), b.tolist(), c.tolist())], np.float32)
    assert bits_equal(ref.fmaf(a, b, c), want) == 0


def test_photometric_matches_statements_for_every_gate_pattern():
    img = np.random.default_rng(5).integers(0, 256, (16, 64, 3)).astype(np.float32)
    img[0, :8] = 255
    img[1, :8] = 0
    for d in cases.gate_draws():
        assert bits_equal(ref.photometric(img, d), ref.photometric_statements(img, d)) == 0, d


def test_uint8_cast_wraps_like_numpy():
    x = np.arange(-48 * 64, 431 * 64 + 1, dtype=np.float32) / np.float32(64)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(ref.to_uint8(x), np.uint8(x))
    assert ref.to_uint8(np.float32([260.7, -3.2]))[0] == 4 and ref.to_uint8(np.float32([-3.2]))[0] == 253


@pytest.mark.parametrize("std,to_rgb", [((1.0, 1.0, 1.0), False), ((58.395, 57.12, 57.375), True)])
def test_normalize_matches_imnormalize(std, to_rgb):
    img = np.random.default_rng(6).integers(0, 256, (32, 48, 3)).astype(np.float32)
    mean = (103.530, 116.280, 123.675)
    assert bits_equal(ref.normalize(img, mean, std, to_rgb), ref.normalize_statements(img, mean, std, to_rgb)) == 0


@pytest.mark.parametrize("pad_val", [0, 5, 2.5, (1.5, -2.0, 3.0)])
def test_pad_matches_copy_make_border(pad_val):
    img = np.random.default_rng(7).random((30, 41, 3)).astype(np.float32)
    assert bits_equal(ref.pad(img, (32, 64), pad_val), ref.pad_statements(img, (32, 64), pad_val)) == 0


@pytest.mark.parametrize("box,dims,flip", [((0, 0, 160, 90), (192, 108), True), ((-8, 6, 168, 96), (140, 72), False)])
def test_pipeline_matches_statements(box, dims, flip):
    img = np.random.default_rng(8).integers(0, 256, (90, 160, 3), np.uint8)
    for d in cases.gate_draws(1)[::5]:
        kw = dict(mean=(103.53, 116.28, 123.675), std=(2.0, 1.0, 0.5), to_rgb=True, shape=(128, 224), pad_val=1)
        assert bits_equal(ref.pipeline(img, d, box, dims, flip, **kw),
                          ref.pipeline_statements(img, d, box, dims, flip, **kw)) == 0


@pytest.fixture(scope="module")
def gold():
    return cases.golden()


def test_oracle_reproduces_the_golden(gold):
    z, meta = gold
    for name, m in meta.items():
        for t, (results, _) in enumerate(cases.replay(z, name, m)):
            got = cases.oracle_frame(ref, z[f"{name}.{t}.src"], results["img_aug"])
            assert bits_equal(got, z[f"{name}.{t}.img"]) == 0, (name, t)


def test_draws_states_and_keys_equal_the_reference(gold):
    z, meta = gold
    for name, m in meta.items():
        for t, (results, (np_key, np_gauss, rnd)) in enumerate(cases.replay(z, name, m)):
            key = f"{name}.{t}"
            assert np.array_equal(np_key, z[f"{key}.np_state"]) and np_gauss == z[f"{key}.np_gauss"], key
            assert np.array_equal(rnd, z[f"{key}.random_state"]), key
            assert np.array_equal(np.stack(results["cam2img"]), z[f"{key}.cam2img"]), key
            assert np.array_equal(np.stack(results["lidar2img"]), z[f"{key}.lidar2img"]), key
            for k in ("ori_shape", "img_shape", "pad_shape"):
                assert np.array_equal(np.array(results[k]), z[f"{key}.{k}"]), (key, k)
            assert all(im.dtype == np.uint8 for im in results["img"]), "results['img'] must stay uint8"


def recorded(steps=None, n=2, hw=(90, 160)):
    results = dict(img=[np.zeros(hw + (3,), np.uint8)] * n, cam2img=[np.eye(4)] * n, lidar2cam=[np.eye(4)] * n)
    conf = dict(reisze=[72], crop=(0, 0, hw[1], hw[0]), H=hw[0], W=hw[1], rand_flip=False)
    for s in steps if steps is not None else [image_aug.PhotoMetricDistortionMultiViewImage(),
                                              image_aug.CropResizeFlipImage(conf),
                                              image_aug.NormalizeMultiviewImage([0, 0, 0], [1, 1, 1]),
                                              image_aug.PadMultiViewImage(size_divisor=32)]:
        results = s(results)
    return results


def test_argument_errors_raise_without_a_gpu():
    with pytest.raises(ValueError, match="debug"):
        image_aug.CropResizeFlipImage(dict(), debug=True)
    with pytest.raises(TypeError):
        image_aug.CropResizeFlipImage(dict(), unknown=1)
    with pytest.raises(ValueError, match="exactly one"):
        image_aug.PadMultiViewImage()
    results = recorded()
    with pytest.raises(ValueError, match="order"):
        image_aug.PhotoMetricDistortionMultiViewImage()(results)
    with pytest.raises(ValueError, match="without CropResizeFlipImage"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8),
                                  recorded([image_aug.PhotoMetricDistortionMultiViewImage()]))
    with pytest.raises(ValueError, match="uint8"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3), results)
    with pytest.raises(ValueError, match="recorded for"):
        image_aug.apply_multiview(torch.zeros(2, 90, 161, 3, dtype=torch.uint8), results)
    with pytest.raises(ValueError, match="cams"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8), results, cams=[0, 2])
    with pytest.raises(ValueError, match="no recorded"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8), dict(img=[]))
    with pytest.raises(RuntimeError, match="CUDA"):
        image_aug.apply_multiview(torch.zeros(2, 90, 160, 3, dtype=torch.uint8), results)


def test_pad_size_mode_and_shapes():
    conf = dict(reisze=[72], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=False)
    r = recorded([image_aug.CropResizeFlipImage(conf), image_aug.PadMultiViewImage(size=(80, 130), pad_val=2)])
    assert r["ori_shape"] == [(72, 128, 3)] * 2 and r["img_shape"] == [(80, 130, 3)] * 2
    assert r["img_aug"].pad_val == (2.0, 0.0, 0.0) and r["pad_fixed_size"] == (80, 130)
    with pytest.raises(ValueError, match="smaller"):
        recorded([image_aug.CropResizeFlipImage(conf), image_aug.PadMultiViewImage(size=(70, 130))])


def test_photo_draw_record_is_a_draw_of_the_oracle():
    d = image_aug.PhotoMetricDistortionMultiViewImage().draw()
    assert isinstance(d, PhotoDraw) and d.mode in (0, 1)
