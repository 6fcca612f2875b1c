"""The ego-motion pre-training graph (`SyntheticViDAR(ego_motion=True)`) sharded over 4 and 8 gloo ranks on CPU
against the single-process graph, in fp64: the loss and EVERY parameter gradient after `allreduce_partial_grads`.
TSA and the decoder are replicated, so every rank builds the same row map and the same shifted / aligned reference
points from the same metas; this checks that the camera-sharded graph around them still sums to the single-process
one.  The CUDA ops are replaced as in tests/test_pretrain_sharding_cpu.py, and the rotate-and-stack op by a torch
gather (`_rotate_stack_cpu`); the row map itself is built by the package's own code on the CPU."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_pretrain_sharding_cpu import BEV, CAMS, IMG, _install_cpu_ops


def _rotate_stack_cpu(prev, query, rows):
    """value[2b] = prev[b, rows[b]] (zeros where rows < 0), value[2b + 1] = query[b]."""
    bs, Q, C = prev.shape
    idx = rows.clamp(min=0).long()[..., None].expand(-1, -1, C)
    rotated = prev.gather(1, idx) * (rows >= 0)[..., None].to(prev.dtype)
    return torch.stack([rotated, query], 1).reshape(bs * 2, Q, C)


def _install():
    from vidar_b200 import ego_motion
    ego_motion.rotate_stack = _rotate_stack_cpu


def _model():
    from vidar_b200 import pretrain
    torch.manual_seed(3)
    m = pretrain.SyntheticViDAR(num_cams=CAMS, encoder_layers=2, decoder_layers=2, future_frames=2, history_frames=1,
                                latent_layer=-1, bev_hw=BEV, ray_grid_num=16, ego_motion=True)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if ("sampling_offsets" in n or "attention_weights" in n) and p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[-1] ** 0.5)
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0

    def loss(pred_dict, *a, **k):
        p = pred_dict["next_bev_preds"]
        return {"stand_in": (p * torch.linspace(0.5, 1.5, p.shape[-1], dtype=p.dtype)).square().mean()}
    m.ray_head.loss = loss
    return m.double()


def _pose_metas():
    from vidar_b200 import ego_motion, synthetic
    drive = synthetic.drive(4, seed=11)
    return ego_motion.queue_metas([dict(f, img_filename=()) for f in drive[:2]] + drive[2:])


def _step(m, group):
    from vidar_b200 import sharding
    m.set_process_group(group)
    m.zero_grad(set_to_none=True)
    g = torch.Generator().manual_seed(6)
    img = torch.randn(1, 2, CAMS, 3, IMG[0], IMG[1], generator=g, dtype=torch.float64)
    lidar2img = torch.eye(4).repeat(1, CAMS, 1, 1).numpy()
    losses = m.forward_train(img, lidar2img, [torch.zeros(4, 4)], pose_metas=_pose_metas())
    loss = sum(losses.values())
    loss.backward()
    if group is not None:
        sharding.allreduce_partial_grads(m, group)
    return loss.detach(), {n: (None if p.grad is None else p.grad.clone()) for n, p in m.named_parameters() if p.requires_grad}


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _install_cpu_ops(sharded=True)
    _install()
    res = _step(_model(), dist.group.WORLD)
    if rank in (0, world - 1, 3 % world):
        torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_the_drive_moves_and_turns():
    metas = _pose_metas()
    assert metas[1]["prev_bev_exists"] and abs(metas[1]["can_bus"][-1]) > 0.1
    from vidar_b200 import ego_motion
    assert np.abs(ego_motion.bev_shift(metas[1:], *BEV)).max() > 1e-3


@pytest.fixture
def restored():
    """The CPU stand-ins patch package modules in this process: put the originals back afterwards."""
    from vidar_b200 import bev_geometry, ego_motion
    from vidar_b200.modules import deform_attn
    saved = [(deform_attn, "msda_apply"), (bev_geometry, "point_sampling"), (ego_motion, "rotate_stack")]
    saved = [(m, n, getattr(m, n)) for m, n in saved]
    yield
    for m, n, v in saved:
        setattr(m, n, v)


@pytest.mark.parametrize("world", [4, 8])
def test_sharded_ego_motion_graph_equals_single_process(tmp_path, world, restored):
    out = str(tmp_path / "ego.pt")
    mp.spawn(_worker, args=(world, 29300 + os.getpid() % 200 + world, out), nprocs=world, join=True)
    _install_cpu_ops(sharded=False)
    _install()
    loss, grads = _step(_model(), None)
    assert all(g is not None for g in grads.values())
    scale = {n: float(g.abs().max()) for n, g in grads.items()}
    for rank in sorted({0, world - 1, 3 % world}):
        l, gr = torch.load(f"{out}.{rank}", weights_only=False)
        torch.testing.assert_close(l, loss, rtol=1e-9, atol=1e-12, msg=lambda m_: f"world {world} rank {rank} loss: {m_}")
        for n, g in grads.items():
            assert gr[n] is not None, (rank, n)
            torch.testing.assert_close(gr[n], g, rtol=1e-6, atol=1e-8 * scale[n] + 1e-16,
                                       msg=lambda m_: f"world {world} rank {rank} grad {n}: {m_}")
