"""The training regimes of `pretrain.CONFIGS` on CPU:
  * forward_train's own numpy draws (`SyntheticViDAR.host_draws`) equal a restatement of the reference's order
    (vidar.py:262-281 and :333-338) on a seeded RandomState, and the default graph draws nothing;
  * the full-set 1-future regime (the last history frame's encoder with gradient, random history drop, no decoder)
    sharded over 4 and 8 gloo ranks equals the single-process graph for drop_prev_index -1, 1 and 2: loss and every
    parameter gradient after `allreduce_partial_grads`; its encoder gradients differ from a step with the history
    frame frozen (the loss does not), so a backwarded frame run under no_grad fails;
  * a step with drop_prev_index = k equals a step on the same sample without its first k frames and no drop.

Host logic only, in fp64, with the CPU stand-ins of tests/test_pretrain_sharding_cpu.py for the CUDA ops."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_pretrain_sharding_cpu import BEV, CAMS, _install_cpu_ops

IMG = (32, 64)
FRAMES = 4                                  # 3 history frames + the current one, as in every config


def _restated_draws(rs, cfg, num_frames):
    """forward_train's draws in its order: A1's rand, A2's rand and randint, the supervised future frame."""
    rs.rand()
    drop = -1
    if rs.rand() < cfg.get("drop_prev_rate", 0.0):
        end = cfg.get("drop_prev_end_idx") or num_frames
        drop = int(rs.randint(1, end))
    future = cfg.get("future_frames", 3)
    supervised = None
    if future > 0 and not cfg.get("supervise_all_future", True):
        supervised = [int(rs.choice(np.arange(1, future + 1), 1)[0])]
    return drop, supervised


@pytest.mark.parametrize("name", ["vidar_1_8_nusc_3future", "vidar_full_nusc_1future", "vidar_1_8_nusc_1future",
                                  "mem_efficient_vidar_1_8_nusc_3future"])
def test_preset_draw_sequence_restates_forward_train(name):
    from vidar_b200 import pretrain
    cfg = pretrain.CONFIGS[name]
    m = pretrain.SyntheticViDAR(**dict(cfg, bev_hw=(8, 8), encoder_layers=1, ray_grid_num=16))
    seen = set()
    for seed in range(300):
        np.random.seed(seed)
        got = m.host_draws(FRAMES)
        after = np.random.rand()                    # the stream continues where the restatement's does
        rs = np.random.RandomState(seed)
        want = _restated_draws(rs, cfg, FRAMES)
        assert got == want, (name, seed)
        assert after == rs.rand(), (name, seed)
        seen.add((got[0], None if got[1] is None else got[1][0]))
    drops = {d for d, _ in seen}
    if cfg.get("drop_prev_rate", 0.0) > 0:
        assert drops == {-1, 1, 2}, drops           # randint(1, 3): both drop indices occur
    else:
        assert drops == {-1}
    if not cfg.get("supervise_all_future", True):
        assert {f for _, f in seen} == {1, 2, 3}


def test_default_graph_draws_nothing():
    from vidar_b200 import pretrain
    m = pretrain.SyntheticViDAR(bev_hw=(8, 8), encoder_layers=1, decoder_layers=1, future_frames=1)
    assert m.reference_draws is False
    np.random.seed(7)
    before = np.random.get_state()
    assert m.host_draws(FRAMES) == (-1, None)
    after = np.random.get_state()
    assert np.array_equal(after[1], before[1]) and after[2:] == before[2:]


def test_presets_build_their_heads_and_reject_bad_options():
    from vidar_b200 import pretrain
    small = dict(bev_hw=(8, 8), encoder_layers=3, ray_grid_num=16)
    m = pretrain.SyntheticViDAR(**dict(pretrain.CONFIGS["vidar_full_nusc_1future"], **small))
    assert len(m.decoder) == 0 and len(m.bev_pred_head) == 1 and m.pred_frame_num == 5
    assert m.prev_frame_embedding is None and not any(n.startswith("future_") for n, _ in m.named_parameters())
    assert m.encoder[2].latent_render.grid_step == 0.5
    m = pretrain.SyntheticViDAR(**dict(pretrain.CONFIGS["mem_efficient_vidar_1_8_nusc_3future"], **small))
    assert len(m.decoder) == 3 and m.pred_frame_num == 1 and m.encoder[2].latent_render.grid_step == 1.0
    with pytest.raises(ValueError):
        pretrain.SyntheticViDAR(backward_history_frames=2, **small)
    with pytest.raises(ValueError):
        pretrain.SyntheticViDAR(future_frames=2, decoder_layers=0, **small)
    with pytest.raises(ValueError):
        pretrain.SyntheticViDAR(drop_prev_rate=0.1, reference_draws=False, **small)
    with pytest.raises(ValueError):
        pretrain.SyntheticViDAR(per_frame_loss_weight=(1.0, 1.0), **small)
    with pytest.raises(ValueError):
        pretrain.build("cpu", config="vidar_full_nusc_2future")


# ---- the full-set regime, sharded and single-process ---------------------------------------------------------------
def _model():
    from vidar_b200 import pretrain
    torch.manual_seed(3)
    cfg = dict(pretrain.CONFIGS["vidar_full_nusc_1future"], num_cams=CAMS, encoder_layers=2, latent_layer=-1,
               bev_hw=BEV, ray_grid_num=16)
    m = pretrain.SyntheticViDAR(**cfg)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():                 # the default init zeroes the offset / weight Linears of every attention
        for n, p in m.named_parameters():
            if ("sampling_offsets" in n or "attention_weights" in n) and p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[-1] ** 0.5)
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0

    def loss(pred_dict, *a, loss_weight=None, **k):       # a replicated stand-in for the CUDA ray losses
        p = pred_dict["next_bev_preds"]
        w = torch.as_tensor(loss_weight[: p.shape[0], 0], dtype=p.dtype).view(-1, *[1] * (p.dim() - 1))
        return {"stand_in": (w * p * torch.linspace(0.5, 1.5, p.shape[-1], dtype=p.dtype)).square().mean()}
    m.ray_head.loss = loss
    return m.double()


def _img():
    g = torch.Generator().manual_seed(6)
    return torch.randn(1, FRAMES, CAMS, 3, IMG[0], IMG[1], generator=g, dtype=torch.float64)


def _step(m, group, drop, img=None, backward=1):
    from vidar_b200 import sharding
    m.set_process_group(group)
    m.backward_history_frames = backward
    m.zero_grad(set_to_none=True)
    img = _img() if img is None else img
    lidar2img = torch.eye(4).repeat(1, CAMS, 1, 1).numpy()
    losses = m.forward_train(img, lidar2img, [torch.zeros(4, 4)], can_bus=torch.zeros(1, 18, dtype=torch.float64),
                             draws=(drop, None))
    loss = sum(losses.values())
    loss.backward()
    if group is not None:
        sharding.allreduce_partial_grads(m, group)
    return loss.detach(), {n: (None if p.grad is None else p.grad.clone()) for n, p in m.named_parameters()
                           if p.requires_grad}


DROPS = (-1, 1, 2)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _install_cpu_ops(sharded=True)
    m = _model()
    res = {drop: _step(m, dist.group.WORLD, drop) for drop in DROPS}
    if rank in (0, 3 % world):                     # rank 3 of 8 owns no camera's backbone
        torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def _close(a, b, what):
    scale = {n: float(g.abs().max()) for n, g in b.items() if g is not None}
    assert set(a) == set(b), what
    for n, g in b.items():
        if g is None:
            assert a[n] is None, (what, n)
            continue
        assert a[n] is not None, (what, n)
        torch.testing.assert_close(a[n], g, rtol=1e-6, atol=1e-8 * scale[n] + 1e-16, msg=lambda m_: f"{what} {n}: {m_}")


@pytest.mark.parametrize("world", [4, 8])
def test_sharded_full_set_regime_equals_single_process(tmp_path, world):
    out = str(tmp_path / "cfg.pt")
    mp.spawn(_worker, args=(world, 29500 + os.getpid() % 150 + world, out), nprocs=world, join=True)
    _install_cpu_ops(sharded=False)
    m = _model()
    single = {drop: _step(m, None, drop) for drop in DROPS}
    for drop, (loss, grads) in single.items():
        # every trainable parameter is on the graph (no decoder is built); the backbone only through the current frame
        assert all(g is not None for g in grads.values()), drop
    # the backwarded frame's encoder pass carries gradient: freezing it keeps the loss and changes the encoder's
    loss, grads = single[-1]
    loss0, grads0 = _step(m, None, -1, backward=0)
    torch.testing.assert_close(loss0, loss, rtol=1e-12, atol=0)
    enc = [n for n in grads if n.startswith("encoder.") and "cross_attn" in n]
    assert enc and all(not torch.allclose(grads0[n], grads[n], rtol=1e-6, atol=0) for n in enc)
    for n in grads:
        if n.startswith(("backbone.", "neck.", "cams_embeds", "level_embeds")):
            torch.testing.assert_close(grads0[n], grads[n], rtol=1e-9, atol=1e-15, msg=lambda m_: f"{n}: {m_}")
    for rank in sorted({0, 3 % world}):
        res = torch.load(f"{out}.{rank}", weights_only=False)
        for drop in DROPS:
            loss, grads = single[drop]
            torch.testing.assert_close(res[drop][0], loss, rtol=1e-9, atol=1e-12,
                                       msg=lambda m_: f"world {world} rank {rank} drop {drop} loss: {m_}")
            _close(res[drop][1], grads, f"world {world} rank {rank} drop {drop} grad")


@pytest.mark.parametrize("k", [1, 2])
def test_dropped_frames_are_the_same_as_absent_frames(k):
    """drop_prev_index = k discards the BEV of history frames 0 .. k-1: the step equals one on frames k .. T-1."""
    _install_cpu_ops(sharded=False)
    m = _model()
    img = _img()
    loss, grads = _step(m, None, k, img)
    loss_cut, grads_cut = _step(m, None, -1, img[:, k:].contiguous())
    torch.testing.assert_close(loss, loss_cut, rtol=0, atol=0)
    _close(grads, grads_cut, f"drop {k}")
    # and it is a different step from keeping the frames
    loss_all, _ = _step(m, None, -1, img)
    assert not torch.equal(loss_all, loss)
