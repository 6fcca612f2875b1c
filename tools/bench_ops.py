"""Per-op timings on one H100: this repo's kernels next to the reference's own PyTorch code
run eagerly on the same GPU (test infrastructure; not the graded bench line).
    python tools/bench_ops.py > gpurun_out/ops.json
MSDA eager = the grid_sample formula of mmcv's multi_scale_deformable_attn_pytorch (oracle
restatement) on CUDA; ray sampler+CE eager = oracle restatement of vidar_head_base.py on CUDA."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import msda_ref  # noqa: E402
from tools.gpu_timing import card, window_ms  # noqa: E402
from vidar_b200 import msda, ray_head  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    out = {"card": card()}
    # ---- MSDA, one camera of the SCA workload
    d = bench.sca_like_inputs(dev, cams=1)

    def ours():
        v = d["value"].requires_grad_(True)
        o = msda.MultiScaleDeformableAttnFunction_fp32.apply(v, d["shapes"], d["lsi"], d["loc"].requires_grad_(True),
                                                             d["attn"].requires_grad_(True), 64)
        o.backward(d["grad_out"])

    def eager():
        v = d["value"].detach().requires_grad_(True)
        o = msda_ref.msda_grid_sample(v, d["shapes"].cpu(), d["loc"].detach().requires_grad_(True),
                                      d["attn"].detach().requires_grad_(True))
        o.backward(d["grad_out"])

    out["msda_1cam_40000q_fwd_bwd_ms"] = {"vidar_b200": window_ms(ours, 10, 3), "torch_eager_grid_sample": window_ms(eager, 3, 1)}
    # ---- TSA shape: B=2, 1 level 200x200, P=4
    g = torch.Generator(device=dev).manual_seed(0)
    val = torch.randn(2, 40000, 8, 32, device=dev, generator=g)
    loc = torch.rand(2, 40000, 8, 1, 4, 2, device=dev, generator=g)
    aw = torch.softmax(torch.randn(2, 40000, 8, 4, device=dev, generator=g), -1).view(2, 40000, 8, 1, 4)
    shp = torch.tensor([[200, 200]], device=dev)
    lsi = torch.tensor([0], device=dev)
    go = torch.randn(2, 40000, 256, device=dev, generator=g)

    def tsa():
        v = val.detach().requires_grad_(True)
        o = msda.MultiScaleDeformableAttnFunction_fp32.apply(v, shp, lsi, loc.detach().requires_grad_(True),
                                                             aw.detach().requires_grad_(True), 64)
        o.backward(go)

    def tsa_eager():
        v = val.detach().requires_grad_(True)
        o = msda_ref.msda_grid_sample(v, shp.cpu(), loc.detach().requires_grad_(True), aw.detach().requires_grad_(True))
        o.backward(go)
    out["msda_tsa_B2_Q40000_fwd_bwd_ms"] = {"vidar_b200": window_ms(tsa, 10, 3), "torch_eager_grid_sample": window_ms(tsa_eager, 3, 1)}

    # ---- head ray sampler + CE: 3 frames 16x200x200, 30k rays, 512 waypoints
    from tests.test_ray_head_gpu import _big_case
    from oracle import ray_head_ref
    sigma, origin, pts, frame = (t.to(dev) for t in _big_case(dev))

    def ce_ours():
        s = sigma.detach().requires_grad_(True)
        ce, valid = ray_head.ray_ce(s, origin, pts, frame, 512, 1.0)
        ce.sum().backward()

    def ce_eager():
        s = sigma.detach().requires_grad_(True)
        tot = 0
        for f in range(3):
            sel = frame == f
            lg, ln, vd = ray_head_ref.sample_frame(s[f], origin[f], pts[sel], 512, 1.0)
            tot = tot - torch.log_softmax(lg[vd], -1)[:, 0].sum()
        tot.backward()

    import oracle.ray_head_ref as rr
    _orig = rr.torch.tensor
    out["ray_ce_30k_rays_512wp_fwd_bwd_ms"] = {"vidar_b200": window_ms(ce_ours, 10, 3)}
    try:
        torch.set_default_device(dev)
        out["ray_ce_30k_rays_512wp_fwd_bwd_ms"]["torch_eager_reference_formula"] = window_ms(ce_eager, 3, 1)
    except Exception as e:
        out["ray_ce_30k_rays_512wp_fwd_bwd_ms"]["torch_eager_reference_formula"] = f"failed: {e}"
    finally:
        torch.set_default_device("cpu")
    # ---- LatentRendering core: 200x200 BEV, 16 heights, 256 waypoints
    from oracle import latent_render_ref
    from vidar_b200.modules.latent_rendering import latent_render_core
    g2 = torch.Generator(device=dev).manual_seed(1)
    occ = torch.randn(1, 200, 200, 16, device=dev, generator=g2)
    feat = torch.randn(1, 200, 200, 16, device=dev, generator=g2)

    def lr_ours():
        o, f = occ.detach().requires_grad_(True), feat.detach().requires_grad_(True)
        p, q = latent_render_core(o, f, 256, 0.5, 1e-3, 1)
        (p.sum() + q.sum()).backward()

    def lr_eager():
        o, f = occ.detach().requires_grad_(True), feat.detach().requires_grad_(True)
        p, q = latent_render_ref.latent_core(o, f, 256, 0.5, 1e-3, "sigmoid")
        (p.sum() + q.sum()).backward()

    out["latent_render_core_200x200x16_256wp_fwd_bwd_ms"] = {"vidar_b200": window_ms(lr_ours, 10, 3)}
    try:
        torch.set_default_device(dev)
        out["latent_render_core_200x200x16_256wp_fwd_bwd_ms"]["torch_eager_reference_formula"] = window_ms(lr_eager, 3, 1)
    except Exception as e:
        out["latent_render_core_200x200x16_256wp_fwd_bwd_ms"]["torch_eager_reference_formula"] = f"failed: {e}"
    finally:
        torch.set_default_device("cpu")
    # ---- LatentRendering MODULE (BASELINE configs[2]b): fused projections vs cuBLAS Linears around the same core
    import vidar_b200.modules  # noqa: F401
    from vidar_b200.registry import build_attention
    torch.manual_seed(0)
    mod = build_attention(bench.LR_CFG).to(dev)
    emb = torch.randn(1, 200, 200, 256, device=dev, generator=g2)
    gemb = torch.randn(1, 200, 200, 256, device=dev, generator=g2)

    def module_step():
        e = emb.detach().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        mod(e).backward(gemb)

    rec = {}
    for fused in (True, False):
        mod.fuse_projections = fused
        rec["fused_projections" if fused else "cublas_linears_around_core"] = window_ms(module_step, 20, 3)
    out["latent_rendering_module_200x200x256_fwd_bwd_ms"] = rec
    # ---- MSDeformableAttention3D module (the per-camera attention of SCA), 6 cameras x 10000 visible pillars:
    #      softmax / sampling-location arithmetic inside the kernel vs materialised like the reference
    att = build_attention(dict(type="MSDeformableAttention3D", embed_dims=256, num_points=8, num_levels=4)).to(dev)
    att.sampling_offsets.weight.data.normal_(0, 0.02)
    att.attention_weights.weight.data.normal_(0, 0.02)
    shapes3 = torch.tensor(bench.LEVELS, dtype=torch.int64, device=dev)
    lsi3 = torch.cat([shapes3.new_zeros(1), (shapes3[:, 0] * shapes3[:, 1]).cumsum(0)[:-1]])
    K3 = int((shapes3[:, 0] * shapes3[:, 1]).sum())
    q3 = torch.randn(6, 10000, 256, device=dev, generator=g2)
    v3 = torch.randn(6, K3, 256, device=dev, generator=g2)
    r3 = torch.rand(6, 10000, 4, 2, device=dev, generator=g2)
    go3 = torch.randn(6, 10000, 256, device=dev, generator=g2)

    def att_step():
        qq, vv = q3.detach().requires_grad_(True), v3.detach().requires_grad_(True)
        att.zero_grad(set_to_none=True)
        att(qq, vv, vv, reference_points=r3, spatial_shapes=shapes3, level_start_index=lsi3).backward(go3)

    rec = {}
    for fused in (True, False):
        att.fuse_epilogue = fused
        rec["fused_epilogue" if fused else "materialised_loc_and_weights"] = window_ms(att_step, 10, 3)
    out["msdeformattn3d_module_6cams_10000q_fwd_bwd_ms"] = rec
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
