"""Seeded module-level case for LatentRendering goldens/tests."""
import torch

CFG = dict(type="LatentRendering", embed_dims=64, num_pred_fcs=0, pred_height=16, grid_num=48,
           grid_step=0.5, reduction=4, act="sigmoid")
CFG_EXP = dict(type="LatentRendering", embed_dims=64, num_pred_fcs=1, pred_height=4, grid_num=40,
               grid_step=0.5, reduction=8, act="exp")      # 8 channels / 4 heights: G = 2
CFG_D1 = dict(type="LatentRendering", embed_dims=64, num_pred_fcs=0, pred_height=1, grid_num=40,
              grid_step=0.5, reduction=4, act="sigmoid")    # the class defaults' shape: 1 height, 16 channels
# shapes the fused projection kernels (csrc/latent_proj.cu) take: the shipped configuration
# (vidar_1_8_nusc_3future.py:159-161) and a 128-wide / 8-height / exp variant (G = 2)
CFG_FUSED = dict(type="LatentRendering", embed_dims=256, num_pred_fcs=0, pred_height=16, grid_num=48,
                 grid_step=0.5, reduction=16, act="sigmoid")
CFG_FUSED_EXP = dict(type="LatentRendering", embed_dims=128, num_pred_fcs=0, pred_height=8, grid_num=40,
                     grid_step=0.5, reduction=8, act="exp")
BEV = (20, 24)
BEV_FUSED = (13, 14)          # 2 x 182 rows: not a multiple of the kernels' 32-row tiles


def seeded_state(module, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, p in sorted(module.state_dict().items()):
        scale = 0.5 if name.endswith("bias") else 1.5 / (p.shape[-1] ** 0.5)
        sd[name] = torch.randn(p.shape, generator=g) * scale
    return sd


def case(seed=0, bs=2, bev=BEV, embed_dims=64):
    g = torch.Generator().manual_seed(seed)
    return dict(embed=torch.randn(bs, bev[0], bev[1], embed_dims, generator=g),
                grad=torch.randn(bs, bev[0], bev[1], embed_dims, generator=g))


def proj_inputs(rows, E, D, A=16, seed=0, device="cpu"):
    """fp32 operands of the four projection kernels with non-zero means and gradients of mixed scale
    (each gradient column scaled by 10^[-3, 1)), so that a relative-to-max tolerance would hide errors
    on small columns and only elementwise bounds can judge them."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g)
    scale = lambda n: 10.0 ** (torch.rand(n, generator=g) * 4 - 3)
    t = dict(x=2 + rnd(rows, E), w_occ=rnd(D, E) / 16, b_occ=rnd(D), w_feat=rnd(A, E) / 16, b_feat=rnd(A),
             w_b=rnd(E, A) / 4 + 0.1, b_b=rnd(E), pooled=1 + rnd(rows, A), prob=torch.rand(rows, D, generator=g),
             g_occ=(0.5 + rnd(rows, D)) * scale(D), g_feat=(0.5 + rnd(rows, A)) * scale(A),
             g_out=(0.5 + rnd(rows, E)) * scale(E))
    return {k: v.to(device) for k, v in t.items()}
