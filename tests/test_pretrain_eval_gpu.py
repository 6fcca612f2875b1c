"""Evaluation from files on the GPU (`SampleLoader(..., test_mode=True)`, `pretrain.evaluate`), at the reduced size of
the other pre-training tests, GridMask on (its eval-mode draws are made), cuDNN deterministic:
  * the test-mode loader's pixels are bit-identical to the test chain run by `apply_multiview` on `cv2.imread` frames
    and to (img - mean) / std padded in numpy; its gt_points equal `gt_points_of(point_infos, False)`; its metas carry
    the queue's lidar2img, the padded img_shape and the camera file names;
  * `evaluate` over 4 consecutive samples of a scene equals per-sample `forward_test` plus `summarize` bit for bit,
    with prefetch 0 and 1, leaves numpy's generator where the per-sample loop leaves it, runs the backbone
    frames + (N - 1) times instead of N x frames, and converts the metric tables on the host once per call (neither
    `frame_metrics_host` nor `ray_head.evaluate` runs per sample);
  * two scenes back to back: one more backbone pass at the boundary, and the same summary;
  * on 2 GPUs (skipped on one): grid 2 x 1 equals the single-GPU summary exactly, grid 1 x 2 to the relative
    tolerance of the sharded loader test (1e-4)."""
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
DEFAULT = "vidar_1_8_nusc_3future"
FRAMES, FUTURE = 3, 3


@pytest.fixture
def exact():
    """cuDNN's deterministic algorithms and no TF32, restored afterwards."""
    saved = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
             torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = saved


def _model(dev, grid=None):
    from vidar_b200 import pretrain
    model, _ = pretrain.build(dev, seed=1, config=DEFAULT, grid=grid, grid_mask=True, point_pipeline=True, **SMALL)
    return model.eval()


def _scene(n, seed=0):
    from vidar_b200 import pretrain
    return pretrain.synthetic_scene(n, FRAMES, FUTURE, img_hw=HW, points_per_frame=4000, seed=seed)


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def _per_sample(model, queues):
    """The loop evaluate replaces: the test-mode loader, forward_test per sample, summarize."""
    from vidar_b200 import evaluate, pretrain
    loader = pretrain.SampleLoader(model, queues, num_workers=0, prefetch=0, test_mode=True)
    return evaluate.summarize([model.forward_test(s["img"], None, s["gt_points"], future_frames=FUTURE,
                                                  img_metas=s["img_metas"])[0] for s in loader])


def _assert_same(got, ref, what):
    assert got.keys() == ref.keys() and len(ref) == 1 + FUTURE, what
    for frame in ref:
        assert got[frame].keys() == ref[frame].keys(), what
        for k, v in ref[frame].items():
            assert np.array_equal(np.float64(got[frame][k]), np.float64(v), equal_nan=True), (what, frame, k,
                                                                                             got[frame][k], v)
    assert ref["frame.0"]["count"] > 0 and np.isfinite(ref["frame.0"]["chamfer_distance"]), ref


class _Passes:
    """Counts backbone passes (one stem call per extract_feat)."""

    def __init__(self, model):
        self.n = 0
        self.hook = model.backbone.stem[0].register_forward_hook(self)

    def __call__(self, *_):
        self.n += 1


def test_test_mode_pixels_points_and_metas(cuda, exact):
    import cv2

    from vidar_b200 import image_aug, pretrain
    model = _model(cuda)
    queue = _scene(1)[0]
    sample = next(iter(pretrain.SampleLoader(model, [queue], num_workers=0, prefetch=1, test_mode=True)))
    mean = np.float32([103.530, 116.280, 123.675])
    image_frames = [f for f in queue if "img_filename" in f]
    assert len(sample["img"]) == FRAMES
    for t, f in enumerate(image_frames):
        raw = np.stack([cv2.imread(n, cv2.IMREAD_UNCHANGED) for n in f["img_filename"]])
        results = pretrain.run_image_transforms(image_aug.config_test_pipeline(), [dict(img=list(raw))])[0]
        chain = image_aug.apply_multiview(torch.from_numpy(raw).to(cuda), results)
        ref = np.zeros((6, 3, 96, 160), np.float32)
        ref[:, :, :90] = ((raw.astype(np.float32) - mean) / np.float32(1.0)).transpose(0, 3, 1, 2)
        got = sample["img"][t]
        assert got.dtype == torch.float32 and tuple(got.shape) == (6, 3, 96, 160)
        assert torch.equal(got, chain), t
        assert np.array_equal(got.cpu().numpy(), ref), t
        meta = sample["img_metas"][t][0]
        assert np.array_equal(meta["lidar2img"], np.stack(f["lidar2img"]))
        assert meta["img_shape"] == [(96, 160, 3)] * 6 and meta["filename"] == f["img_filename"]
    want = model.gt_points_of([f for f in queue if "pts_filename" in f], False)
    assert torch.equal(sample["gt_points"].nan_to_num(-1e30), want.nan_to_num(-1e30))


def test_evaluate_equals_per_sample_forward_test(cuda, exact, monkeypatch):
    from vidar_b200 import evaluate, pretrain
    model = _model(cuda)
    queues = _scene(4)
    passes = _Passes(model)
    _seed(5)
    ref = _per_sample(model, queues)
    ref_state = np.random.get_state()[1].copy()
    assert passes.n == 4 * FRAMES
    host_calls = {"frame_metrics_host": 0, "ray_head.evaluate": 0}
    frame_metrics_host, ray_evaluate = evaluate.frame_metrics_host, model.ray_head.evaluate

    def counted_host(*a, **k):
        host_calls["frame_metrics_host"] += 1
        return frame_metrics_host(*a, **k)

    def counted_evaluate(*a, **k):
        host_calls["ray_head.evaluate"] += 1
        return ray_evaluate(*a, **k)

    monkeypatch.setattr(evaluate, "frame_metrics_host", counted_host)
    monkeypatch.setattr(model.ray_head, "evaluate", counted_evaluate)
    for prefetch in (0, 1):
        passes.n = 0
        host_calls.update({k: 0 for k in host_calls})
        _seed(5)
        got = pretrain.evaluate(model, queues, future_frames=FUTURE, prefetch=prefetch)
        _assert_same(got, ref, f"prefetch={prefetch}")
        assert np.array_equal(np.random.get_state()[1], ref_state), prefetch     # GridMask's draws, as without reuse
        assert passes.n == FRAMES + 3, (prefetch, passes.n)
        assert host_calls == {"frame_metrics_host": 1, "ray_head.evaluate": 0}, host_calls
    passes.hook.remove()


def test_scene_boundary_misses_the_cache(cuda, exact):
    from vidar_b200 import pretrain
    model = _model(cuda)
    queues = _scene(2, seed=0) + _scene(2, seed=1)
    _seed(6)
    ref = _per_sample(model, queues)
    passes = _Passes(model)
    _seed(6)
    got = pretrain.evaluate(model, queues, future_frames=FUTURE, prefetch=1)
    passes.hook.remove()
    assert passes.n == 2 * (FRAMES + 1), passes.n                              # frames + (N - 1) + 1
    _assert_same(got, ref, "two scenes")


def _grid_worker(rank, world, shard, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    grid = sharding.make_grid(shard)
    model = _model(dev, grid)
    _seed(7)
    got = pretrain.evaluate(model, _scene(4) + _scene(1, seed=1), future_frames=FUTURE, prefetch=1, grid=grid)
    torch.save(got, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("shard", [1, 2])
def test_grid_equals_single_gpu(cuda, exact, tmp_path, shard):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from vidar_b200 import pretrain
    out = str(tmp_path / "eval")
    mp.spawn(_grid_worker, args=(2, shard, 29660 + os.getpid() % 200 + shard, out), nprocs=2, join=True)
    model = _model(cuda)
    _seed(7)
    ref = pretrain.evaluate(model, _scene(4) + _scene(1, seed=1), future_frames=FUTURE, prefetch=1)
    for rank in range(2):
        got = torch.load(f"{out}.{rank}", weights_only=False)
        if shard == 1:
            _assert_same(got, ref, f"grid 2x1 rank {rank}")
            continue
        assert got.keys() == ref.keys()
        for frame in ref:
            for k, v in ref[frame].items():
                assert abs(got[frame][k] - v) <= 1e-4 * abs(v), (rank, frame, k, got[frame][k], v)
