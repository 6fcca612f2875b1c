"""The pre-training step under a (replica x shard) grid on two GPUs (skipped on one), at the reduced size of
tests/test_pretrain_gpu.py: 2 x 1 (two replicas, one sample each) against the two single-GPU steps on those samples,
and 1 x 2 (one sample sharded over both) against the sharded path of `allreduce_partial_grads`.  Gradients after the
sync to 1e-5; after one `train_step(..., grid=grid)` the parameters are bitwise identical on both ranks."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=3, decoder_layers=2, future_frames=2, bev_hw=(40, 40), ray_grid_num=64)
SAMPLE = dict(frames=2, img_hw=(96, 160), rays_per_frame=800, future_frames=2, bev_hw=(40, 40))


def _grads(model, sample, sync=None):
    model.zero_grad(set_to_none=True)
    losses = model.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"])
    sum(losses.values()).backward()
    if sync is not None:
        sync()
    return {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.allow_tf32 = False          # the comparison is about the sync, not about TF32 algorithms
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {}
    for shard in (1, 2):
        grid = sharding.make_grid(shard)
        model, opt = pretrain.build(dev, grid=grid, seed=1, **SMALL)
        sample = pretrain.synthetic_sample(dev, seed=grid.replica, **SAMPLE)
        got = _grads(model, sample, lambda: sharding.allreduce_grid_grads(model, grid))
        if shard == 1:                                 # the mean of the two single-GPU steps
            ref_model, _ = pretrain.build(dev, None, seed=1, **SMALL)
            singles = [_grads(ref_model, pretrain.synthetic_sample(dev, seed=r, **SAMPLE)) for r in range(2)]
            ref = {n: (singles[0][n] + singles[1][n]) / 2 for n in singles[0]}
        else:                                          # the existing sharded path
            ref_model, _ = pretrain.build(dev, dist.group.WORLD, seed=1, **SMALL)
            ref = _grads(ref_model, sample, lambda: sharding.allreduce_partial_grads(ref_model, dist.group.WORLD))
        pretrain.train_step(model, opt, sample, grid=grid)
        flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
        other = flat.clone()
        dist.broadcast(other, src=0)
        res[shard] = (got, ref, torch.equal(flat, other))
    torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_grid_steps_on_two_gpus(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "g.pt")
    mp.spawn(_worker, args=(2, 29540 + os.getpid() % 100, out), nprocs=2, join=True)
    for rank in range(2):
        res = torch.load(f"{out}.{rank}", weights_only=False)
        for shard, (got, ref, identical) in res.items():
            assert identical, f"{2 // shard}x{shard} rank {rank}: parameters differ across ranks after a step"
            assert set(got) >= set(ref)
            for n in ref:
                scale = float(ref[n].abs().max())
                torch.testing.assert_close(got[n], ref[n], rtol=1e-5, atol=1e-5 * scale + 1e-9,
                                           msg=lambda m: f"{2 // shard}x{shard} rank {rank} {n}: {m}")
