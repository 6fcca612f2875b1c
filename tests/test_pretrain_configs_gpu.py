"""The training regimes of `pretrain.CONFIGS` on the GPU, at the reduced size of tests/test_pretrain_gpu.py:
  * every preset takes two steps with finite losses, and every trainable parameter gets a finite gradient;
  * under the full-set 1-future preset the encoder's parameters get gradient from the backwarded history frame as
    well as from the current one: it differs from a step with that frame frozen (whose loss is the same), while the
    backbone's gradient, from the current frame only, does not;
  * the same preset with MSDA and the LatentRendering core swapped for the oracle's torch formulas (what bench.py's
    `--impl reference` swaps) agrees with the fused graph to the tolerance of tests/test_pretrain_gpu.py;
  * sharded over 2 GPUs (skipped on one) it equals the single-GPU step."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

SMALL = dict(encoder_layers=3, bev_hw=(40, 40), ray_grid_num=64)
FULL = "vidar_full_nusc_1future"


def _sample(dev, name, seed=0):
    from vidar_b200 import pretrain
    return pretrain.synthetic_sample(dev, frames=4, img_hw=(96, 160), rays_per_frame=800, seed=seed, bev_hw=(40, 40),
                                     future_frames=pretrain.CONFIGS[name]["future_frames"])


def _grads(model, sample, draws, sync=None):
    model.zero_grad(set_to_none=True)
    torch.manual_seed(11)                         # the dense loss's gumbel noise
    losses = model.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"], draws=draws)
    loss = sum(losses.values())
    loss.backward()
    if sync is not None:
        sync()
    return float(loss.detach()), {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}


def _assert_grads_close(got, ref, what):
    assert set(got) == set(ref), what
    for n in ref:
        scale = float(ref[n].abs().max())
        torch.testing.assert_close(got[n], ref[n], rtol=2e-3, atol=2e-4 * scale + 1e-9, msg=lambda m: f"{what} {n}: {m}")


@pytest.mark.parametrize("name", ["vidar_1_8_nusc_3future", FULL, "vidar_1_8_nusc_1future",
                                  "mem_efficient_vidar_1_8_nusc_3future"])
def test_each_preset_takes_a_step(cuda, name):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(cuda, None, seed=1, config=name, **SMALL)
    sample = _sample(cuda, name)
    np.random.seed(0)
    loss, stages = pretrain.train_step(model, opt, sample, None, record=True)
    assert torch.isfinite(loss), name
    assert "cur.encoder" in dict(stages) and "optimizer" in dict(stages)
    missing = [n for n, p in model.named_parameters() if p.requires_grad and p.grad is None]
    assert not missing, (name, missing)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None), name
    loss2, _ = pretrain.train_step(model, opt, sample, None)
    assert torch.isfinite(loss2), name


def test_full_set_encoder_learns_from_the_history_frame(cuda):
    from vidar_b200 import pretrain
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, _ = pretrain.build(cuda, None, seed=1, config=FULL, **SMALL)
    sample = _sample(cuda, FULL)
    for drop in (-1, 1, 2):
        model.backward_history_frames = 1
        loss1, g1 = _grads(model, sample, (drop, None))
        model.backward_history_frames = 0
        loss0, g0 = _grads(model, sample, (drop, None))
        assert abs(loss1 - loss0) <= 1e-6 * abs(loss0), (drop, loss1, loss0)
        enc = [n for n in g1 if n.startswith("encoder.")]
        changed = [n for n in enc if not torch.allclose(g1[n], g0[n], rtol=1e-3, atol=0)]
        # every encoder weight that sees the history BEV or the images (TSA, SCA) gets the history frame's share
        assert any("cross_attn" in n for n in changed) and any("self_attn" in n for n in changed), (drop, changed)
        for n in g1:
            if n.startswith(("backbone.", "neck.")):
                scale = float(g0[n].abs().max())
                torch.testing.assert_close(g1[n], g0[n], rtol=2e-3, atol=2e-4 * scale + 1e-9,
                                           msg=lambda m: f"drop {drop} {n}: {m}")


def _oracle_ops(monkeypatch, model):
    """MSDA and the LatentRendering core through the oracle's torch statements, the fused epilogues off."""
    from oracle import latent_render_ref, msda_ref
    from vidar_b200.modules import deform_attn, latent_rendering

    def msda_eager(value, shapes, lsi, loc, attn, im2col_step):
        return msda_ref.msda_grid_sample(value, shapes, loc, attn)
    act = {0: "exp", 1: "sigmoid"}

    def core_eager(occ, feat, grid_num, grid_step, eps, act_id, group=None):
        return latent_render_ref.latent_core(occ, feat, grid_num, grid_step, eps, act[act_id])
    monkeypatch.setattr(deform_attn, "msda_apply", msda_eager)
    monkeypatch.setattr(latent_rendering, "latent_render_core", core_eager)
    for layer in model.encoder:
        monkeypatch.setattr(layer.cross_attn, "fuse_rebatch", False)
        monkeypatch.setattr(layer.cross_attn.deformable_attention, "fuse_epilogue", False)
        if layer.latent_render is not None:
            monkeypatch.setattr(layer.latent_render, "fuse_projections", False)


def test_full_set_fused_graph_matches_oracle_ops(cuda, monkeypatch):
    from vidar_b200 import pretrain
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, _ = pretrain.build(cuda, None, seed=1, config=FULL, **SMALL)
    sample = _sample(cuda, FULL)
    loss, grads = _grads(model, sample, (1, None))
    with monkeypatch.context() as mp_:
        _oracle_ops(mp_, model)
        loss_ref, grads_ref = _grads(model, sample, (1, None))
    assert abs(loss - loss_ref) <= 1e-4 * abs(loss_ref), (loss, loss_ref)
    _assert_grads_close(grads, grads_ref, "fused vs oracle")


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sample = _sample(dev, FULL)
    res = []
    for group in (None, dist.group.WORLD):
        model, _ = pretrain.build(dev, group, seed=1, config=FULL, **SMALL)
        sync = None if group is None else (lambda m=model: sharding.allreduce_partial_grads(m, dist.group.WORLD))
        res.append(_grads(model, sample, (1, None), sync))
    if rank == 0:
        torch.save(res, out)
    dist.barrier()
    dist.destroy_process_group()


def test_full_set_sharded_step_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "c.pt")
    mp.spawn(_worker, args=(2, 29880 + os.getpid() % 100, out), nprocs=2, join=True)
    (l1, g1), (l2, g2) = torch.load(out, weights_only=False)
    assert abs(l1 - l2) <= 1e-4 * abs(l1)
    _assert_grads_close(g2, g1, "sharded vs single")
