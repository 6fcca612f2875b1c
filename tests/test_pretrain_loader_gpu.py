"""`pretrain.SampleLoader` on the GPU, at the reduced size of the other pre-training tests, GridMask on:
  * from the same files, the loader with prefetch=0, the loader with prefetch=1 and the in-step pipelines
    (`image_pipeline=True` fed cv2.imread frames, `point_pipeline=True` fed the point infos) give bit-identical
    backbone inputs, gt_points and losses, for the default preset and the memory-efficient one; the parameter
    gradients agree to the tolerance of the other step tests, as the backward's scatter sums (atomics) are not
    bit-reproducible from run to run even on identical inputs;
  * three consecutive prefetched steps, each loss equal to that of the unprefetched run.  This catches a step
    that reads its sample before the side stream's work on it is done (a missing event wait shows on the first
    step, whose sample is launched just before it).  It does not isolate `record_stream`: the side stream's wait on
    the step's stream at each launch already orders the reuse of a dropped sample's blocks;
  * `forward_test` on a loader sample equals `forward_test` on the same pipelined frames, metas and gt_points fed
    through the plain tensor path;
  * sharded over 2 GPUs (skipped on one), each rank decodes only its backbone cameras and the step equals the
    single-GPU one."""
import os
import random

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=3, bev_hw=(40, 40), ray_grid_num=64)
SMALL_CONF = dict(reisze=[72, 90, 108], crop=(0, 0, 160, 90), H=90, W=160, rand_flip=True)
HW = (90, 160)
DEFAULT = "vidar_1_8_nusc_3future"
MEM = "mem_efficient_vidar_1_8_nusc_3future"


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


def _model(dev, name, group=None, lr=2e-4):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(dev, group, seed=1, config=name, lr=lr, grid_mask=True, image_pipeline=True,
                                point_pipeline=True, **SMALL)
    model.image_transforms[1].data_aug_conf = SMALL_CONF
    return model, opt


def _queue(name, seed=0):
    from vidar_b200 import pretrain
    return pretrain.synthetic_sample(None, frames=4, img_hw=HW, future_frames=pretrain.CONFIGS[name]["future_frames"],
                                     points_per_frame=4000, seed=seed, files=True)


def _seed(s):
    np.random.seed(s)
    random.seed(s)


def _grads(model, forward):
    model.zero_grad(set_to_none=True)
    torch.manual_seed(11)                         # the dense loss's gumbel noise
    loss = sum(forward().values())
    loss.backward()
    return loss.detach().cpu(), {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}


def _recorded(model, forward):
    """_grads plus every backbone input and the gt_points the loss saw."""
    seen, gts = [], []
    hook = model.backbone.stem[0].register_forward_hook(lambda m, inp, out: seen.append(inp[0].detach().clone()))
    loss_fn = model.ray_head.loss
    model.ray_head.loss = lambda pred, gt, *a, **k: (gts.append(gt), loss_fn(pred, gt, *a, **k))[1]
    try:
        loss, grads = _grads(model, forward)
    finally:
        hook.remove()
        del model.ray_head.loss
    return loss, grads, [s.cpu() for s in seen], gts[0].detach().cpu()


def _assert_grads_close(got, ref, what):
    assert set(got) == set(ref), what
    for n in ref:
        scale = float(ref[n].abs().max())
        torch.testing.assert_close(got[n], ref[n], rtol=2e-3, atol=2e-4 * scale + 1e-9, msg=lambda m: f"{what} {n}: {m}")


def _in_step(model, queue, draws):
    """The step's own pipelines on cv2.imread frames of the same files."""
    import cv2
    dev = model.bev_embedding.weight.device
    img = torch.from_numpy(np.stack([[cv2.imread(n, cv2.IMREAD_UNCHANGED) for n in f["img_filename"]]
                                     for f in queue if "img_filename" in f]))[None].to(dev)
    cam2img, lidar2cam = np.stack(queue[0]["cam2img"])[None], np.stack(queue[0]["lidar2cam"])[None]
    infos = [f for f in queue if "pts_filename" in f]
    return lambda: model.forward_train(img, None, None, cam2img=cam2img, lidar2cam=lidar2cam, point_infos=infos,
                                       draws=draws)


def _loaded(model, sample, draws):
    return lambda: model.forward_train(sample["img"], None, sample["gt_points"], img_metas=sample["img_metas"],
                                       draws=draws)


@pytest.mark.parametrize("name", [DEFAULT, MEM])
def test_loader_equals_the_in_step_pipelines(cuda, exact, name):
    from vidar_b200 import pretrain
    model, _ = _model(cuda, name)
    queue = _queue(name)
    _seed(3)
    draws = model.host_draws(4)
    _seed(40)
    loss_ref, grads_ref, seen_ref, gt_ref = _recorded(model, _in_step(model, queue, draws))
    assert len(seen_ref) == 4
    for prefetch in (0, 1):
        _seed(40)                                  # num_workers=0: the dataset draws from this process's generators
        sample = next(iter(pretrain.SampleLoader(model, [queue], num_workers=0, prefetch=prefetch)))
        assert [tuple(t.shape[:2]) for t in sample["img"]] == [(6, 3)] * 4
        loss, grads, seen, gt = _recorded(model, _loaded(model, sample, draws))
        assert len(seen) == 4 and all(torch.equal(a, b) for a, b in zip(seen, seen_ref)), (name, prefetch)
        assert torch.equal(gt.nan_to_num(-1e30), gt_ref.nan_to_num(-1e30)), (name, prefetch)
        assert torch.equal(loss, loss_ref), (name, prefetch, float(loss), float(loss_ref))
        _assert_grads_close(grads, grads_ref, f"{name} prefetch={prefetch}")


def test_prefetched_steps_equal_unprefetched_ones(cuda, exact):
    """lr = 0 keeps the parameters, so each step's loss depends on its own sample only."""
    from vidar_b200 import pretrain
    queues = [_queue(DEFAULT, seed=s) for s in range(3)]
    losses = {}
    for prefetch in (0, 1):
        model, opt = _model(cuda, DEFAULT, lr=0.0)
        loader = pretrain.SampleLoader(model, queues, num_workers=1, prefetch=prefetch, seed=9)
        _seed(5)
        out = []
        for k, sample in enumerate(loader):
            torch.manual_seed(100 + k)
            out.append(pretrain.train_step(model, opt, sample)[0].clone())
        losses[prefetch] = torch.stack(out).cpu()
    assert losses[0].shape == (3,) and torch.isfinite(losses[0]).all()
    assert len(set(losses[0].tolist())) == 3                       # three different samples
    assert torch.equal(losses[1], losses[0]), (losses[1], losses[0])


def _flat(ret):
    out = {}
    for frame, metrics in ret[0].items():
        for k, v in metrics.items():
            out[f"{frame}.{k}"] = np.float64(v)
    return out


def test_forward_test_takes_a_loader_sample(cuda, exact, monkeypatch):
    from vidar_b200 import pretrain
    model, _ = _model(cuda, DEFAULT)
    model.eval()
    _seed(40)
    sample = next(iter(pretrain.SampleLoader(model, [_queue(DEFAULT)], num_workers=0, prefetch=1)))
    _seed(41)
    got = _flat(model.forward_test(sample["img"], None, sample["gt_points"], future_frames=3,
                                   img_metas=sample["img_metas"]))
    # the plain tensor path on the same frames: the queue's frames share one crop / resize, so one lidar2img
    l2i = [m[0]["lidar2img"] for m in sample["img_metas"]]
    assert all(np.array_equal(a, l2i[0]) for a in l2i)
    monkeypatch.setattr(model, "image_transforms", None)
    monkeypatch.setattr(model, "point_transforms", None)
    _seed(41)
    ref = _flat(model.forward_test(torch.stack(sample["img"])[None], l2i[0][None], sample["gt_points"],
                                   future_frames=3))
    assert got.keys() == ref.keys() and len(got) >= 4
    for k in ref:
        assert np.array_equal(got[k], ref[k], equal_nan=True), (k, got[k], ref[k])


def _sharded_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    model, _ = _model(dev, DEFAULT, dist.group.WORLD)
    _seed(40)
    sample = next(iter(pretrain.SampleLoader(model, [_queue(DEFAULT)], num_workers=0, prefetch=1)))
    shapes = [tuple(t.shape) for t in sample["img"]]
    model.zero_grad(set_to_none=True)
    torch.manual_seed(11)
    loss = sum(model.forward_train(sample["img"], None, sample["gt_points"], img_metas=sample["img_metas"],
                                   draws=(-1, None)).values())
    loss.backward()
    sharding.allreduce_partial_grads(model, dist.group.WORLD)
    grads = {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}
    torch.save(dict(cams=model.my_backbone_cams, shapes=shapes, loss=float(loss), grads=grads), f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_loader_decodes_each_ranks_cameras(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from vidar_b200 import pretrain
    out = str(tmp_path / "loader")
    mp.spawn(_sharded_worker, args=(2, 29460 + os.getpid() % 200, out), nprocs=2, join=True)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    model, _ = _model(cuda, DEFAULT)
    _seed(40)
    sample = next(iter(pretrain.SampleLoader(model, [_queue(DEFAULT)], num_workers=0, prefetch=1)))
    loss, grads = _grads(model, _loaded(model, sample, (-1, None)))
    covered = []
    for rank in range(2):
        r = torch.load(f"{out}.{rank}", weights_only=False)
        covered += list(r["cams"])
        assert all(s[0] == len(r["cams"]) for s in r["shapes"]), (rank, r["shapes"])
        assert abs(r["loss"] - float(loss)) <= 1e-4 * abs(float(loss)), (rank, r["loss"], float(loss))
        _assert_grads_close(r["grads"], grads, f"rank {rank}")
    assert sorted(covered) == list(range(6))
