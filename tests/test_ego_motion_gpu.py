"""Ego motion on the GPU (vidar_b200/ego_motion.py, csrc/bev_rotate.cu, `SyntheticViDAR(ego_motion=True)`):
  * the rotate-and-stack kernel equals the reference's statements -- torchvision's nearest `rotate` of the [C, H, W]
    view about [100, 100], permute, stack with the query -- bit for bit, and its backward equals torch autograd through
    them up to the order of the fp32 sums, bit-identical from call to call;
  * with no motion the shift is zero, the row map the identity, and the ego-motion encoder equals itself with the
    alignment skipped, bit for bit;
  * every preset takes a step with ego_motion=True, every trainable parameter getting a finite gradient;
  * a step with ego motion makes no more host syncs than one without."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ANGLES = [0.0, 0.013, -0.013, 1.9, -1.9, 5.0, 45.0, 179.3]
SMALL = dict(encoder_layers=3, bev_hw=(40, 40), ray_grid_num=64)


def _reference_value(prev, query, angle, hw):
    """transformer.py:137-150 and encoder.py:225-227 for bs 1."""
    from torchvision.transforms.functional import rotate
    H, W = hw
    tmp = prev[0].reshape(H, W, -1).permute(2, 0, 1)
    tmp = rotate(tmp, angle, center=[100, 100])
    rotated = tmp.permute(1, 2, 0).reshape(H * W, -1)[None]
    return torch.stack([rotated, query], 1).reshape(2, H * W, -1)


@pytest.mark.parametrize("hw", [(200, 200), (50, 50)])
@pytest.mark.parametrize("angle", ANGLES)
def test_rotate_stack_forward_equals_torchvision(cuda, hw, angle):
    from vidar_b200 import ego_motion as ego
    g = torch.Generator(device=cuda).manual_seed(int(angle * 1000) % 997)
    Q = hw[0] * hw[1]
    prev = torch.randn(1, Q, 256, device=cuda, generator=g)
    query = torch.randn(1, Q, 256, device=cuda, generator=g)
    rows = ego.rotation_rows([angle], *hw, cuda)
    got = ego.rotate_stack(prev, query, rows)
    assert torch.equal(got, _reference_value(prev, query, angle, hw))
    if angle == 0.0:
        assert torch.equal(rows[0].long(), torch.arange(Q, device=cuda))


@pytest.mark.parametrize("hw", [(200, 200), (50, 50)])
@pytest.mark.parametrize("angle", [0.013, -1.9, 45.0, 179.3])
def test_rotate_stack_backward_equals_autograd(cuda, hw, angle):
    from vidar_b200 import ego_motion as ego
    g = torch.Generator(device=cuda).manual_seed(5)
    Q = hw[0] * hw[1]
    prev = torch.randn(1, Q, 256, device=cuda, generator=g, requires_grad=True)
    query = torch.randn(1, Q, 256, device=cuda, generator=g, requires_grad=True)
    grad = torch.randn(2, Q, 256, device=cuda, generator=g)
    ref = torch.autograd.grad(_reference_value(prev, query, angle, hw), (prev, query), grad)
    rows = ego.rotation_rows([angle], *hw, cuda)
    got = torch.autograd.grad(ego.rotate_stack(prev, query, rows), (prev, query), grad)
    again = torch.autograd.grad(ego.rotate_stack(prev, query, rows), (prev, query), grad)
    torch.testing.assert_close(got[0], ref[0], rtol=1e-6, atol=1e-6)
    assert torch.equal(got[1], ref[1])
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])


def _still_metas(T=2):
    from vidar_b200 import ego_motion as ego, synthetic
    d = synthetic.drive(T + 1, 0)
    for f in d:                                   # parked: every frame has the first frame's pose
        f.update({k: d[0][k] for k in ("ego2global_translation", "ego2global_rotation", "can_bus")})
    return ego.queue_metas([dict(f, img_filename=()) for f in d[:T]] + d[T:])


def test_zero_motion_is_the_identity(cuda, monkeypatch):
    from vidar_b200 import ego_motion as ego, pretrain
    metas = _still_metas()
    assert not ego.bev_shift(metas, 40, 40).any()
    assert all(m["can_bus"][-1] == 0 for m in metas)
    torch.manual_seed(0)
    model = pretrain.SyntheticViDAR(num_cams=2, encoder_layers=3, decoder_layers=1, future_frames=1, history_frames=1,
                                    bev_hw=(40, 40), ray_grid_num=64, ego_motion=True).to(cuda).eval()
    model.set_process_group(None)
    sample = pretrain.synthetic_sample(cuda, frames=2, cams=2, img_hw=(96, 160), rays_per_frame=100, bev_hw=(40, 40),
                                       future_frames=1)
    frame_metas = [dict(lidar2img=np.asarray(sample["lidar2img"][0]), img_shape=[(96, 160, 3)], **metas[1])]
    with torch.no_grad():
        feats, shapes, lsi = model.extract_feat(sample["img"][:, 1])
        prev = torch.randn(1, 1600, 256, device=cuda)
        aligned = model.encode(feats, shapes, lsi, frame_metas, None, prev)
        monkeypatch.setattr(ego, "rotate_stack", lambda p, q, rows: torch.stack([p, q], 1).reshape(2, *p.shape[1:]))
        monkeypatch.setattr(ego, "bev_shift", lambda m, h, w: np.zeros((len(m), 2)))
        skipped = model.encode(feats, shapes, lsi, frame_metas, None, prev)
    assert torch.equal(aligned, skipped)


@pytest.mark.parametrize("name", ["vidar_1_8_nusc_3future", "vidar_full_nusc_1future", "vidar_1_8_nusc_1future",
                                  "mem_efficient_vidar_1_8_nusc_3future"])
def test_each_preset_takes_a_step_with_ego_motion(cuda, name):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(cuda, None, seed=1, config=name, ego_motion=True, **SMALL)
    sample = pretrain.synthetic_sample(cuda, frames=4, img_hw=(96, 160), rays_per_frame=800, bev_hw=(40, 40),
                                       future_frames=pretrain.CONFIGS[name]["future_frames"], poses=True)
    np.random.seed(0)
    loss, _ = pretrain.train_step(model, opt, sample, None)
    assert torch.isfinite(loss), name
    missing = [n for n, p in model.named_parameters() if p.requires_grad and p.grad is None]
    assert not missing, (name, missing)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None), name
    if model.future_frames:
        assert model.future_can_bus_mlp[0].weight.grad.abs().sum() > 0


def test_ego_motion_adds_no_host_sync(cuda):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from tools import gpu_timing
    from vidar_b200 import pretrain
    counts = {}
    for on in (False, True):
        model, opt = pretrain.build(cuda, None, seed=1, config="vidar_1_8_nusc_3future", ego_motion=on, **SMALL)
        sample = pretrain.synthetic_sample(cuda, frames=4, img_hw=(96, 160), rays_per_frame=800, bev_hw=(40, 40),
                                           poses=on)
        np.random.seed(0)
        pretrain.train_step(model, opt, sample, None)                  # warm-up
        np.random.seed(0)
        counts[on], sites = gpu_timing.count_syncs(pretrain.train_step, model, opt, sample, None)
    assert counts[True] <= counts[False], (counts, sites)
