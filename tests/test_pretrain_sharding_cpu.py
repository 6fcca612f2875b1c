"""The whole synthetic pre-training graph (vidar_b200/pretrain.py: RN101 + FPN, BEV encoder, future decoder, head)
sharded over 4 and 8 gloo ranks on CPU against the single-process graph: loss and EVERY parameter gradient after
`allreduce_partial_grads`, in both sharding modes (camera / cell sharding only, and with the row-sharded encoder and
decoder).  8 ranks exercise what a 2-GPU run does not: cameras cut into four sub-slices, two ranks that own no
camera's backbone (their backbone gradients are None), chains of 2-rank camera groups.

Host logic only -- the CUDA ops are replaced on this GPU-less host: the sampling op by the CPU oracle, the
camera-sharded slot kernel by the module's own per-camera attention over the rank's (camera, 64-row sub-slice) units,
`point_sampling` by seeded random projections, the ray loss by a plain differentiable function of the head output.
LatentRendering is left out of the graph (its sharding has its own GPU tests)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

BEV = (16, 16)
IMG = (64, 96)
CAMS, D = 6, 4


def _install_cpu_ops(sharded):
    from oracle import msda_ref
    from vidar_b200 import pretrain, sca
    from vidar_b200.modules import deform_attn

    def apply(value, shapes, lsi, loc, attn, im2col_step):
        return msda_ref.msda_grid_sample(value, shapes, loc, attn)
    deform_attn.msda_apply = apply

    def point_sampling(ref_3d, pc_range, img_metas):
        g = torch.Generator().manual_seed(5)
        Q = ref_3d.shape[2]
        ref_cam = (torch.rand(CAMS, 1, Q, D, 2, generator=g) * 1.2 - 0.1).to(ref_3d.dtype)
        mask = torch.rand(CAMS, 1, Q, D, generator=g) < 0.25          # ~70 % of the pillars per camera: 2-3 sub-slices
        return ref_cam, mask
    pretrain.bev_geometry.point_sampling = point_sampling

    def slots_of_my_units(self, query, value, ref_cam, bev_mask, shapes, lsi):
        """What the row-indirect kernel computes: every (camera, visible row) of this rank's units through the
        camera attention, added into the pillar's slot, divided by the number of cameras that see the pillar."""
        da = self.deformable_attention
        w, r = self._world()
        hit = bev_mask[:, 0].sum(-1) > 0
        count = torch.clamp((bev_mask.sum(-1) > 0).permute(1, 2, 0).sum(-1), min=1.0)
        slots = torch.zeros_like(query)
        for cam0, ncl, S, lo, hi in sca.unit_plan(w, r, value.shape[0]):
            for c in range(cam0, cam0 + ncl):
                idx = hit[c].nonzero().squeeze(-1)
                sl = (torch.arange(idx.numel()) // sca.SLICE_ROWS) % S
                sel = idx[(sl >= lo) & (sl < hi)]
                if sel.numel():
                    out = da(query=query[:, sel], value=value[c].permute(1, 0, 2), reference_points=ref_cam[c][:, sel],
                             spatial_shapes=shapes, level_start_index=lsi)
                    slots = slots.index_add(1, sel, out)
        return slots / count[..., None]
    if sharded:
        deform_attn.SpatialCrossAttention._fusable = lambda self, *a: True
        deform_attn.SpatialCrossAttention._slots_fused = slots_of_my_units


def _model():
    from vidar_b200 import pretrain
    torch.manual_seed(3)
    m = pretrain.SyntheticViDAR(num_cams=CAMS, encoder_layers=2, decoder_layers=2, future_frames=2, history_frames=1,
                                latent_layer=-1, bev_hw=BEV, ray_grid_num=16)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():                 # the default init zeroes the offset / weight Linears of every attention
        for n, p in m.named_parameters():
            if ("sampling_offsets" in n or "attention_weights" in n) and p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[-1] ** 0.5)
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0

    def loss(pred_dict, *a, **k):         # stands in for the CUDA ray losses: any replicated function of the head output
        p = pred_dict["next_bev_preds"]
        return {"stand_in": (p * torch.linspace(0.5, 1.5, p.shape[-1], dtype=p.dtype)).square().mean()}
    m.ray_head.loss = loss
    return m.double()                     # fp64: the comparison below is about the sharding logic, not about fp32 summation order


def _step(m, group, row_sharded):
    from vidar_b200 import sharding
    m.set_process_group(group, row_sharded=row_sharded)
    m.zero_grad(set_to_none=True)
    g = torch.Generator().manual_seed(6)
    img = torch.randn(1, 2, CAMS, 3, IMG[0], IMG[1], generator=g, dtype=torch.float64)
    lidar2img = torch.eye(4).repeat(1, CAMS, 1, 1).numpy()
    losses = m.forward_train(img, lidar2img, [torch.zeros(4, 4)], can_bus=torch.zeros(1, 18, dtype=torch.float64))
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
    m = _model()
    res = {}
    for row_sharded in (False, True):
        res[row_sharded] = _step(m, dist.group.WORLD, row_sharded)
    if rank in (0, world - 1, 3 % world):          # rank 3 of 8 owns no camera's backbone
        torch.save(res, f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [4, 8])
def test_sharded_pretraining_graph_equals_single_process(tmp_path, world):
    out = str(tmp_path / "pre.pt")
    mp.spawn(_worker, args=(world, 29700 + os.getpid() % 200 + world, out), nprocs=world, join=True)
    _install_cpu_ops(sharded=False)
    loss, grads = _step(_model(), None, False)
    assert all(g is not None for g in grads.values())
    scale = {n: float(g.abs().max()) for n, g in grads.items()}
    for rank in sorted({0, world - 1, 3 % world}):
        res = torch.load(f"{out}.{rank}", weights_only=False)
        for row_sharded in (False, True):
            l, gr = res[row_sharded]
            torch.testing.assert_close(l, loss, rtol=1e-9, atol=1e-12, msg=lambda m_: f"world {world} rank {rank} rows {row_sharded} loss: {m_}")
            for n, g in grads.items():
                assert gr[n] is not None, (rank, row_sharded, n)
                torch.testing.assert_close(gr[n], g, rtol=1e-6, atol=1e-8 * scale[n] + 1e-16,
                                           msg=lambda m_: f"world {world} rank {rank} rows {row_sharded} grad {n}: {m_}")


def test_model_as_constructed_runs_every_camera_on_one_rank():
    """A `SyntheticViDAR` used without `set_process_group` has the layout of no group: its backbone runs every
    camera and every camera's features are filled."""
    from vidar_b200 import pretrain
    torch.manual_seed(0)
    m = pretrain.SyntheticViDAR(num_cams=2, encoder_layers=1, decoder_layers=1, future_frames=1, history_frames=1,
                                latent_layer=-1, bev_hw=(8, 8), ray_grid_num=16)
    assert m.backbone_cams() == [0, 1]
    with torch.no_grad():
        feats, shapes, lsi = m.extract_feat(torch.randn(1, 2, 3, *IMG))
    assert shapes.tolist() == [[8, 12], [4, 6], [2, 3], [1, 2]] and lsi.tolist() == [0, 96, 120, 126]
    assert feats.shape == (2, 128, 1, 256)
    assert all(feats[c].abs().sum() > 0 for c in range(2))
