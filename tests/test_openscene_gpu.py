"""The OpenScene (nuPlan) inputs on the GPU, with 8 cameras of 1920 x 1080:
  * `apply_multiview` of the OpenScene train chain (photometric, normalise, rescale by 2/3, pad) and test chain
    against cv2: the test chain equals cv2.resize of mmcv's normalisation bit for bit; the train chain equals the
    device's own photometric + normalisation output (the nuScenes test-chain kernel) rescaled by the host
    restatement of cv2's INTER_LINEAR, which tests/test_openscene_cpu.py holds equal to cv2;
  * `jpeg.decode_frames` on 1920 x 1080 4:2:0 and 4:2:2 files (1080 is not a multiple of 16) against cv2.imread;
  * `gather_gt_points` on the golden nuPlan queue against the reference's union2one (6 columns);
  * a full OpenScene step from files: backbone inputs, gt_points and loss bit-identical to the in-step pipelines fed
    cv2.imread frames;
  * `evaluate` equal to per-sample `forward_test` plus `summarize`, and the submission files byte-equal to a
    restatement of the reference's `_save_prediction`."""
import os
import random

import numpy as np
import pytest
import torch

from tests.test_openscene_cpu import GOLDEN, rescale_restated

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=2, bev_hw=(40, 40), ray_grid_num=64)
NAME = "vidar_OpenScene_mini_1_8_3future"


@pytest.fixture
def exact():
    saved = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
             torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = saved


def _frame(rng, n=8):
    from vidar_b200 import synthetic
    return np.stack([synthetic.camera_image(rng, synthetic.NUPLAN_IMG_HW) for _ in range(n)])


def test_test_chain_equals_cv2(cuda):
    import cv2
    from vidar_b200 import image_aug
    imgs = _frame(np.random.default_rng(1))
    results = dict(img=list(imgs), lidar2img=[np.eye(4)] * 8)
    for t in image_aug.config_openscene_test_pipeline():
        results = t(results)
    out = image_aug.apply_multiview(torch.from_numpy(imgs).to(cuda), results).cpu().numpy()
    assert out.shape == (8, 3, 736, 1280)
    mean = np.array(image_aug.CONFIG_IMG_NORM["mean"], np.float32)
    for i, im in enumerate(imgs):
        norm = cv2.multiply(cv2.subtract(im.astype(np.float32), np.float64(mean.reshape(1, -1))),
                            1 / np.float64(np.ones((1, 3))))
        want = cv2.resize(norm, (1280, 720), interpolation=cv2.INTER_LINEAR)
        want = cv2.copyMakeBorder(want, 0, 16, 0, 0, cv2.BORDER_CONSTANT, value=0)
        assert np.array_equal(out[i].transpose(1, 2, 0), want), i


def test_train_chain_is_the_photometric_output_rescaled(cuda):
    from vidar_b200 import image_aug
    rng = np.random.default_rng(2)
    imgs = _frame(rng)
    np.random.seed(4)
    results = dict(img=list(imgs), lidar2img=[np.eye(4)] * 8)
    for t in image_aug.config_openscene_pipeline():
        results = t(results)
    assert results["img_shape"][0] == (736, 1280, 3) and results["lidar2img"][0][0, 0] == 2 / 3
    src = torch.from_numpy(imgs).to(cuda)
    out = image_aug.apply_multiview(src, results).cpu().numpy()
    # the same draws without the rescale: the nuScenes test-chain kernel's photometric + normalisation
    plan = results["img_aug"]
    flat = dict(img=list(imgs), img_aug=image_aug.ImageAugPlan(8, (1080, 1920), photo=plan.photo, mean=plan.mean,
                                                              std=plan.std, normalized=True, pad_hw=(1080, 1920)))
    norm = image_aug.apply_multiview(src, flat).cpu().numpy()
    for i in range(8):
        want = rescale_restated(norm[i].transpose(1, 2, 0))
        got = out[i].transpose(1, 2, 0)
        assert np.array_equal(got[:720], want) and not got[720:].any(), i
    # and only the cameras asked for, with their own draws
    part = image_aug.apply_multiview(src[[5, 2]], results, [5, 2]).cpu().numpy()
    assert np.array_equal(part, out[[5, 2]])


@pytest.mark.parametrize("sampling", ["420", "422"])
def test_decode_frames_1920x1080(cuda, tmp_path, sampling):
    import cv2
    from vidar_b200 import jpeg
    factor = dict(zip(("420", "422"), (cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422)))
    imgs = _frame(np.random.default_rng(3), 3)
    names = []
    for i, im in enumerate(imgs):
        names.append(str(tmp_path / f"{i}.jpg"))
        assert cv2.imwrite(names[-1], im, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           factor[sampling]])
    frames = [jpeg.LoadMultiViewImageFromFiles(to_float32=True)(dict(img_filename=names))]
    (out,) = jpeg.decode_frames(frames, cuda)
    want = np.stack([cv2.imread(n, cv2.IMREAD_UNCHANGED) for n in names])
    assert out.shape == (3, 1080, 1920, 3) and np.array_equal(out.cpu().numpy(), want)


def test_gather_gt_points_six_columns_match_the_reference(cuda, tmp_path):
    import json
    from vidar_b200 import point_pipeline as pp, pretrain
    g = np.load(GOLDEN)
    q = json.loads(str(g["meta"]))["queue"]
    steps = pp.config_openscene_train_pipeline()
    np.random.seed(q["seed"])
    frames = []
    for f in range(q["frames"]):
        path = tmp_path / f"{f}.pcd"
        g[f"queue.{f}.bytes"].tofile(path)
        frames.append(pretrain.run_point_transforms(steps, [dict(pts_filename=str(path), timestamp=1.0 + f,
                                                                  sweeps=[])])[0])
    got = pp.gather_gt_points(frames, q["ego_mask"], cuda, compact=True).cpu().numpy()
    want = g["queue.gt"]
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the test chain: LoadNuPlanPointsFromFile only, column 4 the raw ring
    raw = pp.read_pcd(str(tmp_path / "0.pcd"))
    test = pp.gather_gt_points([dict(points=raw)], None, cuda, compact=True).cpu().numpy()
    assert np.array_equal(test[:, :5], raw[:, :5]) and (test[:, 5] == 0).all()


def _model(dev):
    from vidar_b200 import pretrain
    return pretrain.build(dev, seed=1, config=NAME, grid_mask=True, image_pipeline=True, point_pipeline=True, **SMALL)


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def _recorded(model, forward):
    seen, gts = [], []
    hook = model.backbone.stem[0].register_forward_hook(lambda m, inp, out: seen.append(inp[0].detach().clone()))
    loss_fn = model.ray_head.loss
    model.ray_head.loss = lambda pred, gt, *a, **k: (gts.append(gt), loss_fn(pred, gt, *a, **k))[1]
    try:
        torch.manual_seed(11)
        loss = sum(forward().values()).detach().cpu()
    finally:
        hook.remove()
        del model.ray_head.loss
    return loss, [s.cpu() for s in seen], gts[0].detach().cpu()


def test_step_from_files_equals_the_in_step_pipelines(cuda, exact):
    import cv2
    from vidar_b200 import pretrain
    model, _ = _model(cuda)
    queue = pretrain.synthetic_sample(None, frames=4, future_frames=3, points_per_frame=4000, files=True,
                                      openscene=True)
    _seed(3)
    draws = model.host_draws(4)
    img = torch.from_numpy(np.stack([[cv2.imread(n, cv2.IMREAD_UNCHANGED) for n in f["img_filename"]]
                                     for f in queue if "img_filename" in f]))[None].to(cuda)
    cam2img, lidar2cam = np.stack(queue[0]["cam2img"])[None], np.stack(queue[0]["lidar2cam"])[None]
    infos = [f for f in queue if "pts_filename" in f]
    _seed(40)
    loss_ref, seen_ref, gt_ref = _recorded(model, lambda: model.forward_train(
        img, None, None, cam2img=cam2img, lidar2cam=lidar2cam, point_infos=infos, draws=draws))
    assert seen_ref[-1].shape == (8, 3, 736, 1280) and gt_ref.shape[-1] == 6
    for prefetch in (0, 1):
        _seed(40)
        sample = next(iter(pretrain.SampleLoader(model, [queue], num_workers=0, prefetch=prefetch)))
        loss, seen, gt = _recorded(model, lambda: model.forward_train(
            sample["img"], None, sample["gt_points"], img_metas=sample["img_metas"], draws=draws))
        assert len(seen) == 4 and all(torch.equal(a, b) for a, b in zip(seen, seen_ref)), prefetch
        assert torch.equal(gt.nan_to_num(-1e30), gt_ref.nan_to_num(-1e30)), prefetch
        assert torch.equal(loss, loss_ref) and torch.isfinite(loss), (prefetch, float(loss), float(loss_ref))
    _seed(41)
    sample = next(iter(pretrain.SampleLoader(model, [queue], num_workers=1, prefetch=1)))
    loss, _ = pretrain.train_step(model, pretrain.config_optimizer(model), sample)
    assert torch.isfinite(loss)


def test_evaluate_and_submission(cuda, exact, tmp_path):
    from vidar_b200 import evaluate, pretrain
    model, _ = _model(cuda)
    model.eval()
    future = 2
    queues = pretrain.synthetic_scene(3, 4, future, points_per_frame=3000, seed=5, openscene=True)
    got = pretrain.evaluate(model, queues, future_frames=future, prefetch=1, ego_mask=(0.0, 0.0, 0.0, 0.0),
                            submission_path=str(tmp_path / "sub"))
    loader = pretrain.SampleLoader(model, queues, num_workers=0, prefetch=0, test_mode=True,
                                   ego_mask=(0.0, 0.0, 0.0, 0.0))
    rows, files = [], {}
    for s in loader:
        rows.append(model.forward_test(s["img"], None, s["gt_points"], future_frames=future,
                                       img_metas=s["img_metas"])[0])
        # the reference's _save_prediction, per frame t > 0 (vidar.py:491-519)
        pred = model.predict_future(s["img"], None, future, img_metas=s["img_metas"])
        dec = model.ray_head.get_point_cloud_prediction(model._current_head_frame(pred), s["gt_points"], 0,
                                                        model.bev_h, model.bev_w, pretrain.PC_RANGE)
        name = queues[s["index"]][3]["sample_idx"]
        for t in range(1, future + 1):
            r_depth = torch.sqrt((dec["pred_pcds"][0][t] ** 2).sum(1)).cpu().numpy()
            files[f"{name}_{t}.txt"] = "".join("%f\n" % d for d in r_depth)
    want = evaluate.summarize(rows)
    assert got == want
    assert sorted(os.listdir(tmp_path / "sub")) == sorted(files)
    for n, text in files.items():
        assert (tmp_path / "sub" / n).read_text() == text, n
    assert any(len(t) for t in files.values())
