"""The configs' optimizer in the (replica x shard) pre-training step on two GPUs (skipped on one), at the reduced size
of tests/test_pretrain_gpu.py: at 2 x 1 and 1 x 2, two `train_step(..., grid=grid)`s with `pretrain.config_optimizer`
leave the parameters bitwise identical on both ranks, and within 1e-6 of torch's AdamW over the same
`paramwise_groups` after clip_grad_norm_(35), stepped on one GPU from the same start with the gradients the grid
synchronised."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=3, decoder_layers=2, future_frames=2, bev_hw=(40, 40), ray_grid_num=64)
SAMPLE = dict(frames=2, img_hw=(96, 160), rays_per_frame=800, future_frames=2, bev_hw=(40, 40))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import optim, pretrain, sharding
    res = {}
    for shard in (1, 2):
        grid = sharding.make_grid(shard)
        model, _ = pretrain.build(dev, grid=grid, seed=1, **SMALL)
        opt = pretrain.config_optimizer(model)
        ref_p = [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in model.parameters()]
        groups = optim.paramwise_groups(model, 2e-4, 0.01, {"backbone": dict(lr_mult=0.1)})
        ref = torch.optim.AdamW([dict(g, params=[q]) for g, q in zip(groups, ref_p)], lr=2e-4, weight_decay=0.01,
                                foreach=False)
        captured = []
        opt.register_step_pre_hook(lambda o, a, k: captured.append([None if p.grad is None else p.grad.clone()
                                                                     for p in model.parameters()]))
        sample = pretrain.synthetic_sample(dev, seed=grid.replica, **SAMPLE)
        for _ in range(2):
            pretrain.train_step(model, opt, sample, grid=grid)
            for q, g in zip(ref_p, captured[-1]):
                q.grad = g
            torch.nn.utils.clip_grad_norm_([q for q in ref_p if q.grad is not None], 35.0)
            ref.step()
        flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
        other = flat.clone()
        dist.broadcast(other, src=0)
        err = max(float((p.detach() - q.detach()).abs().max()) / max(float(q.detach().abs().max()), 1e-30)
                  for p, q in zip(model.parameters(), ref_p) if p.numel())
        res[shard] = (torch.equal(flat, other), err)
    torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_config_optimizer_under_a_grid_on_two_gpus(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "o.pt")
    mp.spawn(_worker, args=(2, 29640 + os.getpid() % 100, out), nprocs=2, join=True)
    for rank in range(2):
        for shard, (identical, err) in torch.load(f"{out}.{rank}", weights_only=False).items():
            assert identical, f"{2 // shard}x{shard} rank {rank}: parameters differ across ranks"
            assert err <= 1e-6, f"{2 // shard}x{shard} rank {rank}: {err:.3e} from torch's step"
