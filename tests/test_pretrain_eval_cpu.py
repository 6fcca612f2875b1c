"""Evaluation from files without a GPU:
  * the test-mode `SampleLoader`'s host half runs the config's test chain: no photometric step and no crop in the
    plan, `lidar2img` as the queue gives it, the padded `img_shape`, the GT frames through LoadPointsFromFile only,
    and no draw from numpy or `random`;
  * `synthetic_scene`'s sliding windows: neighbours share frames - 1 image frames' files, every sample has
    1 + future_frames GT frames, and lidar2img = cam2img @ lidar2cam;
  * `pretrain.summarize_tables` over gloo at 2 and 4 ranks, for every (replica x shard) grid, with CPU tables: the
    replica split, the all-gather and the summary equal `evaluate.summarize` of the per-sample ret_dicts in dataset
    order, also with N not divisible by R and with a replica whose block is empty; the first failing sample's
    exception is raised on every rank;
  * `pretrain.evaluate` rejects a queue with too few GT frames before any work."""
import os
import random

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SMALL = dict(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(20, 20), ray_grid_num=32)
HW = (90, 160)


def _model():
    from vidar_b200 import pretrain
    model, _ = pretrain.build("cpu", None, seed=1, point_pipeline=True, **SMALL)
    return model


def _rng_state():
    return np.random.get_state()[1].copy(), random.getstate()


def test_test_mode_host_half_is_the_test_chain():
    from vidar_b200 import point_pipeline, pretrain
    model = _model()
    assert model.image_transforms is None                       # the test mode needs no image pipeline
    queue = pretrain.synthetic_scene(1, 3, 2, img_hw=HW, points_per_frame=500, seed=4)[0]
    loader = pretrain.SampleLoader(model, [queue], num_workers=0, prefetch=0, test_mode=True)
    np.random.seed(7)
    random.seed(7)
    before = _rng_state()
    host = next(iter(loader.host_loader))
    after = _rng_state()
    assert np.array_equal(before[0], after[0]) and before[1] == after[1]
    image_frames = [f for f in queue if "img_filename" in f]
    assert len(host["frames"]) == 3
    for r, f in zip(host["frames"], image_frames):
        plan = r["img_aug"]
        assert plan.photo is None and plan.crop is None and plan.dims is None and not plan.flip
        assert plan.normalized and not plan.to_rgb
        assert np.array_equal(plan.mean, np.float32([103.530, 116.280, 123.675])) and np.all(plan.std == 1)
        assert plan.pad_hw == (96, 160) and plan.pad_val == (0.0, 0.0, 0.0)
        assert r["img_shape"] == [(96, 160, 3)] * 6
        assert len(r["lidar2img"]) == 6
        for got, want in zip(r["lidar2img"], f["lidar2img"]):
            assert got.dtype == np.float64 and np.array_equal(got, want)
        assert list(r["filename"]) == f["img_filename"]
        assert [rec.name for rec in r["img_jpeg"]] == f["img_filename"]
    gt_frames = [f for f in queue if "pts_filename" in f]
    assert len(host["points"]) == 3
    want = pretrain.run_point_transforms(point_pipeline.config_test_pipeline(), gt_frames)
    for got, ref in zip(host["points"], want):
        assert "pts_aug" not in got and np.array_equal(got["points"], ref["points"])
        assert got["points"].shape[1] == 5
    # the queue's own dicts are left as they were
    assert "img_aug" not in queue[0] and "points" not in queue[-1]


def test_test_mode_needs_the_point_pipeline_and_lidar2img():
    from vidar_b200 import pretrain
    model, _ = pretrain.build("cpu", None, seed=1, **SMALL)
    with pytest.raises(ValueError, match="point_pipeline"):
        pretrain.SampleLoader(model, [], 0, 0, test_mode=True)
    queue = [dict(f) for f in pretrain.synthetic_scene(1, 2, 1, cams=2, img_hw=HW, points_per_frame=100)[0]]
    del queue[0]["lidar2img"]
    with pytest.raises(ValueError, match="lidar2img"):
        pretrain.SampleLoader(_model(), [queue], 0, 0, test_mode=True).dataset[0]


def test_synthetic_scene_windows_share_frames():
    from vidar_b200 import pretrain
    n, frames, future = 4, 3, 2
    queues = pretrain.synthetic_scene(n, frames, future, cams=2, img_hw=HW, points_per_frame=100, seed=1)
    assert len(queues) == n
    images = [[tuple(f["img_filename"]) for f in q if "img_filename" in f] for q in queues]
    points = [[f["pts_filename"] for f in q if "pts_filename" in f] for q in queues]
    for i, q in enumerate(queues):
        assert len(images[i]) == frames and len(points[i]) == 1 + future
        assert len(q) == frames + future
        # the current (last image) frame is the first GT frame; earlier image frames carry no points
        assert [("img_filename" in f, "pts_filename" in f) for f in q] == \
            [(True, False)] * (frames - 1) + [(True, True)] + [(False, True)] * future
        for f in q[:frames]:
            for c2i, l2c, l2i in zip(f["cam2img"], f["lidar2cam"], f["lidar2img"]):
                assert l2i.dtype == np.float64 and np.array_equal(l2i, c2i @ l2c)
    for i in range(n - 1):
        assert images[i][1:] == images[i + 1][:-1]                  # frames - 1 shared image frames
        assert images[i][0] not in images[i + 1] and images[i + 1][-1] not in images[i]
        assert points[i][1:] == points[i + 1][:-1]
    assert len({name for q in images for f in q for name in f}) == 2 * (n + frames - 1)
    for name in images[0][0]:
        assert os.path.isfile(name)


def test_synthetic_queue_is_unchanged_by_the_scene_split():
    """`synthetic_sample(files=True)`'s queue keeps its layout: GT frames from the current frame on."""
    from vidar_b200 import pretrain
    queue = pretrain.synthetic_sample(None, frames=3, cams=2, img_hw=HW, future_frames=2, points_per_frame=100,
                                      files=True)
    assert [("img_filename" in f, "pts_filename" in f) for f in queue] == \
        [(True, False), (True, False), (True, True), (False, True), (False, True)]


def test_evaluate_rejects_a_short_queue():
    from vidar_b200 import pretrain
    model = _model()
    queues = pretrain.synthetic_scene(2, 2, 2, cams=2, img_hw=HW, points_per_frame=100)
    queues[1] = queues[1][:-1]
    with pytest.raises(ValueError, match="sample 1 has 2 GT frames"):
        pretrain.evaluate(model, queues, future_frames=2)
    with pytest.raises(ValueError, match="sample 0 has 3 GT frames"):
        pretrain.evaluate(model, queues, future_frames=6)


# ---- the replica split, gather and summary over gloo ----------------------------------------------------------
FRAMES = 3


def _tables(n, seed=0, fail=()):
    """[n * FRAMES, 8] float64 metric rows (evaluate.FIELDS); `fail`: (sample, frame, flags) to set."""
    g = np.random.default_rng(seed)
    t = np.zeros((n * FRAMES, 8))
    t[:, 2] = g.integers(0, 50, n * FRAMES)                             # count (some 0: nan ray errors)
    t[:, 0] = g.uniform(0, 30, n * FRAMES) * t[:, 2]
    t[:, 1] = g.uniform(0, 2, n * FRAMES) * t[:, 2]
    t[:, 4], t[:, 6] = g.integers(0, 40, n * FRAMES), g.integers(1, 40, n * FRAMES)
    t[:, 3], t[:, 5] = g.uniform(0, 9, n * FRAMES) * t[:, 4], g.uniform(0, 9, n * FRAMES) * t[:, 6]
    for i, f, flags in fail:
        t[i * FRAMES + f, 7] = flags
    return torch.from_numpy(t)


def _per_sample_summary(table, n):
    from vidar_b200 import evaluate
    return evaluate.summarize([evaluate.frame_metrics_host(table[i * FRAMES:(i + 1) * FRAMES], 1, FRAMES)
                               for i in range(n)])


FAIL = ((3, 2, 2), (3, 1, 1 << 4), (4, 0, 1))       # sample 3 fails first, at frame 1 (NO_PRED: a ValueError)


def _worker(rank, world, shard, port, cases, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from vidar_b200 import pretrain, sharding
    grid = sharding.make_grid(shard)
    got = []
    for n, fail in cases:
        full = _tables(n, seed=n, fail=fail)
        lo, hi = sharding.shard_range(n, grid.replica, grid.replicas)
        block = full[lo * FRAMES:hi * FRAMES].clone()
        if grid.shard_rank:                          # only shard rank 0's block may be read
            block.fill_(-1.0)
        try:
            got.append(("ok", pretrain.summarize_tables(block, n, FRAMES, grid)))
        except Exception as e:                       # noqa: BLE001  (the test compares the exception)
            got.append((type(e).__name__, str(e)))
    torch.save(got, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,shard", [(2, 1), (2, 2), (4, 1), (4, 2)])
def test_replica_gather_equals_dataset_order_summary(tmp_path, world, shard):
    from vidar_b200 import pretrain
    replicas = world // shard
    # N divisible by R, N not divisible, N < R (an empty block), and a failing sample
    cases = [(2 * replicas, ()), (2 * replicas + 1, ()), (replicas - 1, ()), (7, FAIL)]
    out = str(tmp_path / "eval")
    mp.spawn(_worker, args=(world, shard, 29700 + os.getpid() % 200 + 7 * world + shard, cases, out), nprocs=world,
             join=True)
    for k, (n, fail) in enumerate(cases):
        full = _tables(n, seed=n, fail=fail)
        if fail:
            with pytest.raises(ValueError) as err:
                pretrain.summarize_tables(full, n, FRAMES)
            want = ("ValueError", str(err.value))
            assert "sample 3, frame 1" in want[1]
        else:
            want = ("ok", _per_sample_summary(full, n))
        for rank in range(world):
            got = torch.load(f"{out}.{rank}", weights_only=False)[k]
            assert got[0] == want[0], (n, rank, got)
            if got[0] == "ok":
                assert got[1].keys() == want[1].keys(), (n, rank)
                for frame, metrics in want[1].items():
                    for m, v in metrics.items():
                        assert np.array_equal(np.float64(got[1][frame][m]), np.float64(v), equal_nan=True), \
                            (n, rank, frame, m, got[1][frame][m], v)
            else:
                assert got[1] == want[1], (n, rank)


def test_single_process_summary_is_the_per_sample_summary():
    from vidar_b200 import pretrain
    for n in (1, 5):
        full = _tables(n, seed=n)
        got, want = pretrain.summarize_tables(full, n, FRAMES), _per_sample_summary(full, n)
        assert got.keys() == want.keys() and len(got) == FRAMES
        for frame in want:
            for m in want[frame]:
                assert np.array_equal(np.float64(got[frame][m]), np.float64(want[frame][m]), equal_nan=True)
    assert pretrain.summarize_tables(torch.zeros(0, 8, dtype=torch.float64), 0, FRAMES) == {}
    with pytest.raises(ValueError, match="table"):
        pretrain.summarize_tables(_tables(2), 3, FRAMES)
