"""`pretrain.SampleLoader`'s host half and `synthetic_sample(..., files=True)`, without a GPU:
  * the sample files: baseline 4:2:0 JPEGs of the camera size, one results dict per queue frame;
  * with num_workers=0 the loader's draws are those of `gt_points_of` + `frame_transforms` in the step, in order and
    value, from the same generator states, and leave the generators in the same state;
  * worker seeding follows mmdet's worker_init_fn (seed + rank * num_workers + worker_id): a run is reproducible,
    and other seeds give other plans;
  * a progressive or truncated camera file fails in the worker with the file's name."""
import random
import re

import numpy as np
import pytest
import torch

SMALL = dict(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(20, 20), ray_grid_num=32)
SMALL_CONF = dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True)
HW = (90, 160)


def _model():
    from vidar_b200 import pretrain
    model, _ = pretrain.build("cpu", None, seed=1, image_pipeline=True, point_pipeline=True, **SMALL)
    model.image_transforms[1].data_aug_conf = SMALL_CONF
    return model


def _queue(seed=0, frames=3):
    from vidar_b200 import pretrain
    return pretrain.synthetic_sample(None, frames=frames, img_hw=HW, future_frames=SMALL["future_frames"],
                                     points_per_frame=1500, seed=seed, files=True)


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def _rng_state():
    return np.random.get_state()[1].copy(), random.getstate()


def _image_key(frames):
    out = []
    for r in frames:
        p = r["img_aug"]
        out.append((p.photo, p.crop, p.dims, p.flip, p.pad_hw, np.stack(r["lidar2img"]).tobytes(), r["img_shape"]))
    return out


def _point_key(frames):
    return [(r["pts_aug"].perm.tobytes(), [s.n_keep for s in r["pts_aug"].segments]) for r in frames]


def test_sample_files_are_the_queues_results_dicts():
    import cv2

    from vidar_b200 import jpeg, pretrain
    queue = pretrain.synthetic_sample(None, frames=2, cams=2, future_frames=2, points_per_frame=100, files=True)
    assert len(queue) == 2 + 2
    assert [("img_filename" in f, "pts_filename" in f) for f in queue] == [(True, False), (True, True),
                                                                          (False, True), (False, True)]
    for f in queue[:2]:
        assert len(f["img_filename"]) == len(f["cam2img"]) == len(f["lidar2cam"]) == 2
        for name in f["img_filename"]:
            with open(name, "rb") as fh:
                h = jpeg.parse(fh.read(), name)
            assert (h.H, h.W, h.hv) == (900, 1600, (2, 2))
            assert cv2.imread(name, cv2.IMREAD_UNCHANGED).shape == (900, 1600, 3)
    assert all(len(f["sweeps"]) == 2 for f in queue[1:])


def test_loader_without_workers_draws_as_the_step():
    import cv2

    from vidar_b200 import pretrain
    model = _model()
    queue = _queue()
    loader = pretrain.SampleLoader(model, [queue], num_workers=0, prefetch=0)
    _seed(21)
    host = next(iter(loader.host_loader))
    after_loader = _rng_state()

    # the step's host halves, in forward_train's order: gt_points_of, then frame_transforms
    seen = []
    model.gather_points = seen.append
    img = torch.from_numpy(np.stack([[cv2.imread(n, cv2.IMREAD_UNCHANGED) for n in f["img_filename"]]
                                     for f in queue if "img_filename" in f]))[None]
    _seed(21)
    model.gt_points_of([f for f in queue if "pts_filename" in f], True)
    frames = model.frame_transforms(img, np.stack(queue[0]["cam2img"])[None], np.stack(queue[0]["lidar2cam"])[None])
    after_step = _rng_state()

    assert _point_key(host["points"]) == _point_key(seen[0])
    assert _image_key(host["frames"]) == _image_key(frames)
    assert np.array_equal(after_loader[0], after_step[0]) and after_loader[1] == after_step[1]
    # the loader parsed the files: records of every camera, the pixels deferred to the device
    for r, f in zip(host["frames"], [f for f in queue if "img_filename" in f]):
        assert [rec.name for rec in r["img_jpeg"]] == f["img_filename"]
    # the queue's own dicts are not changed by the transforms
    assert np.array_equal(np.stack(queue[0]["cam2img"]), np.stack(_queue()[0]["cam2img"]))


def _plans(model, samples, num_workers, seed, rank=0):
    from vidar_b200 import pretrain
    loader = pretrain.SampleLoader(model, samples, num_workers=num_workers, prefetch=0, seed=seed, rank=rank)
    return [(_image_key(h["frames"]), _point_key(h["points"])) for h in loader.host_loader]


def test_worker_seeding_is_reproducible():
    from vidar_b200 import pretrain
    model = _model()
    queue = _queue()
    samples = [queue] * 4
    a = _plans(model, samples, 2, seed=5)
    b = _plans(model, samples, 2, seed=5)
    assert a == b
    c = _plans(model, samples, 2, seed=6)
    assert all(x != y for x, y in zip(a, c))
    assert len({repr(x) for x in a}) == 4                        # each sample has its own draws
    # mmdet's scheme: worker w of rank r draws from seed + r * num_workers + w; samples go round-robin
    ds = pretrain.SampleLoader(model, samples, 0, 0).dataset
    for rank in (0, 1):
        got = a if rank == 0 else _plans(model, samples, 2, seed=5, rank=1)
        for w in range(2):
            _seed(5 + rank * 2 + w)
            torch.manual_seed(5 + rank * 2 + w)
            for i in (w, w + 2):
                h = ds[i]
                assert got[i] == (_image_key(h["frames"]), _point_key(h["points"])), (rank, w, i)


@pytest.mark.parametrize("kind", ["progressive", "truncated"])
def test_bad_camera_file_fails_in_the_worker_with_its_name(tmp_path, kind):
    import cv2

    from vidar_b200 import pretrain
    model = _model()
    queue = [dict(f) for f in _queue()]
    good = queue[1]["img_filename"][4]
    bad = str(tmp_path / f"{kind}.jpg")
    if kind == "progressive":
        cv2.imwrite(bad, cv2.imread(good, cv2.IMREAD_UNCHANGED), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    else:
        with open(good, "rb") as fh:
            data = fh.read()
        with open(bad, "wb") as fh:
            fh.write(data[:len(data) // 2])
    queue[1]["img_filename"] = queue[1]["img_filename"][:4] + [bad] + queue[1]["img_filename"][5:]
    loader = pretrain.SampleLoader(model, [queue], num_workers=1, prefetch=0)
    with pytest.raises(ValueError, match=re.escape(bad)):
        next(iter(loader.host_loader))


def test_loader_needs_both_pipelines():
    from vidar_b200 import pretrain
    model, _ = pretrain.build("cpu", None, seed=1, image_pipeline=True, **SMALL)
    with pytest.raises(ValueError, match="point_pipeline"):
        pretrain.SampleLoader(model, [], 0, 0)
