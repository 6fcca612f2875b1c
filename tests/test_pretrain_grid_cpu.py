"""The synthetic pre-training graph under a (replica x shard) process grid (`sharding.make_grid`) over gloo on CPU:
world 4 as 2 x 2 and 4 x 1, world 8 as 4 x 2 and 2 x 4.  Each replica trains on its own sample, sharded over its shard
group.  Against the single-process graph on each replica's sample:
  * every rank's loss is its replica's single-process loss;
  * after the grid's gradient sync every parameter gradient is the mean over replicas of the single-process
    gradients;
  * after two AdamW steps (`pretrain.train_step(..., grid=grid)`) every parameter is bitwise identical on all ranks.
2 x 4 has shard groups that are not the world and cameras shared by two ranks: camera groups made from group-local
ranks, or a feature broadcast from a group-local source rank, fail it.

Host logic only, with the CPU stand-ins of tests/test_pretrain_sharding_cpu.py for the CUDA ops, in fp64; the
gradient bucket's pack / unpack kernels are restated in torch (`torch.cat` of grad * scale, and its split)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_pretrain_sharding_cpu import CAMS, IMG, _install_cpu_ops, _model


def _install_torch_bucket():
    from vidar_b200 import grad_bucket

    def pack(params, scales, out=None):
        return torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) * s
                          for p, s in zip(params, scales)])

    def unpack(bucket, params):
        off = 0
        for p in params:
            v = bucket[off: off + p.numel()].view_as(p)
            if p.grad is None:
                p.grad = v.clone()
            else:
                p.grad.copy_(v)
            off += p.numel()
        return params
    grad_bucket.pack, grad_bucket.unpack = pack, unpack


def _sample(replica):
    g = torch.Generator().manual_seed(100 + replica)
    return dict(img=torch.randn(1, 2, CAMS, 3, IMG[0], IMG[1], generator=g, dtype=torch.float64),
                lidar2img=torch.eye(4).repeat(1, CAMS, 1, 1).numpy(), gt_points=[torch.zeros(4, 4)],
                can_bus=torch.zeros(1, 18, dtype=torch.float64))


def _loss_and_grads(m, sample):
    losses = m.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"], can_bus=sample["can_bus"])
    loss = sum(losses.values())
    loss.backward()
    return loss.detach()


def _worker(rank, world, shard, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from vidar_b200 import pretrain, sharding
    _install_cpu_ops(sharded=True)
    _install_torch_bucket()
    grid = sharding.make_grid(shard)
    assert (grid.replica, grid.shard_rank, grid.replicas) == (rank // shard, rank % shard, world // shard)
    m = _model()                                   # the same seed on every rank: the replicas start alike
    m.set_process_group(grid.group)
    sample = _sample(grid.replica)
    loss = _loss_and_grads(m, sample)
    sharding.allreduce_grid_grads(m, grid)
    res = dict(loss=loss, replica=grid.replica)
    if rank in (0, world - 1):
        res["grads"] = {n: p.grad.clone() for n, p in m.named_parameters() if p.requires_grad}
    opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=1e-3, weight_decay=0.01)
    probe = {n: p.detach().clone() for n, p in m.named_parameters() if n in ("cams_embeds", "prev_frame_embedding")}
    for _ in range(2):
        pretrain.train_step(m, opt, sample, grid=grid)
    flat = torch.cat([p.detach().reshape(-1) for p in m.parameters()])
    ref = flat.clone()
    dist.broadcast(ref, src=0)
    res["identical"] = torch.equal(flat, ref)
    res["moved"] = all(not torch.equal(p, dict(m.named_parameters())[n]) for n, p in probe.items())
    torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,shard", [(4, 2), (4, 1), (8, 2), (8, 4)], ids=["2x2", "4x1", "4x2", "2x4"])
def test_grid_step_equals_replica_mean_of_single_process_steps(tmp_path, world, shard):
    out = str(tmp_path / "grid.pt")
    mp.spawn(_worker, args=(world, shard, 29300 + os.getpid() % 150 + 10 * world + shard, out), nprocs=world,
             join=True)
    _install_cpu_ops(sharded=False)
    replicas = world // shard
    single = []
    for r in range(replicas):
        m = _model().set_process_group(None)
        loss = _loss_and_grads(m, _sample(r))
        single.append((loss, {n: p.grad for n, p in m.named_parameters() if p.requires_grad}))
    assert all(g is not None for _, gr in single for g in gr.values())
    mean = {n: sum(gr[n] for _, gr in single) / replicas for n in single[0][1]}
    scale = {n: float(g.abs().max()) for n, g in mean.items()}
    for rank in range(world):
        res = torch.load(f"{out}.{rank}", weights_only=False)
        assert res["replica"] == rank // shard
        torch.testing.assert_close(res["loss"], single[res["replica"]][0], rtol=1e-9, atol=1e-12,
                                   msg=lambda m_: f"{replicas}x{shard} rank {rank} loss: {m_}")
        assert res["identical"], f"{replicas}x{shard} rank {rank}: parameters differ from rank 0 after two steps"
        assert res["moved"], f"{replicas}x{shard} rank {rank}: the optimizer did not change the parameters"
        if "grads" in res:
            assert set(res["grads"]) == set(mean)
            for n, g in mean.items():
                torch.testing.assert_close(res["grads"][n], g, rtol=1e-6, atol=1e-8 * scale[n] + 1e-16,
                                           msg=lambda m_: f"{replicas}x{shard} rank {rank} grad {n}: {m_}")
