"""LatentRendering module on the fused CUDA core (vidar_b200/csrc/latent_render.cu).

Same registry name, constructor kwargs, parameter names (`unsup_raymarching_head.*`,
`lora_a.*`, `lora_b.*`), call signature and numerics as
projects/mmdet3d_plugin/bevformer/modules/ray_operations/latent_rendering.py:37-162; it is
instantiated from the `latent_render=dict(...)` kwarg of the encoder/decoder layers
(encoder_v2.py:81-82) and called as `latent_render(query.view(bs, bev_h, bev_w, C))`.

The ray-marching -- grid_sample x3, masks, cumprod, normalisation, pooling in the reference -- is
a custom op (two kernels forward, two backward) that never materialises the [bs, 16, 40000, 257]
tensors.  With the shipped configuration (`num_pred_fcs=0`, embed_dims 256, pred_height 16,
reduction 16: vidar_1_8_nusc_3future.py:159-161) the three Linear layers and the final product
are fused around it as well (csrc/latent_proj.cu): the whole module is six kernels forward+
backward instead of ~35, and one autograd node (`_FusedLatentRendering`) that can shard the BEV
cells over a process group.  Other configurations keep the Linear layers as PyTorch ops (cuBLAS)
around the custom core.  CUDA only.
"""
import torch
from torch.autograd.function import once_differentiable
import torch.nn as nn

from .. import _lib
from ..registry import ATTENTION, BaseModule

_ACT = {"exp": 0, "sigmoid": 1}


def _shard(n, group):
    """(world, c0, count): this rank's contiguous share [c0, c0 + count) of n BEV cells over `group`; all of them
    when `group` is None, has one rank or no process group is initialised."""
    if group is None:
        return 1, 0, n
    import torch.distributed as dist
    from ..sharding import shard_range
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return 1, 0, n
    lo, hi = shard_range(n, dist.get_rank(group), world)
    return world, lo, hi - lo


class _LatentRenderCore(torch.autograd.Function):
    """(occ [bs,Hb,Wb,D], feat [bs,Hb,Wb,D*G]) -> (prob [bs,Hb,Wb,D], pooled [bs,Hb*Wb,D*G]).

    With `group` of more than one rank the BEV cells are sharded over its ranks (SURVEY.md 8e).  Inputs and
    outputs are replicated; each rank marches only its contiguous share of the cells and the 2.56 MB maps are
    all-reduced between the phases:
      forward : prob(local cells) -> all_reduce(prob) -> pooled(local cells) -> all_reduce(pooled)
      backward: pool-bwd(local) -> all_reduce(grad_prob_map, grad_feat) -> prob-bwd(local)
                -> all_reduce(grad_occ).
    Upstream gradients must be replicated (they are: everything after this op is)."""

    @staticmethod
    def forward(ctx, occ, feat, grid_num, grid_step, eps, act, group):
        import torch.distributed as dist
        _lib.require_cuda(occ=occ.contiguous(), feat=feat.contiguous())
        occ, feat = occ.float().contiguous(), feat.float().contiguous()
        bs, Hb, Wb, D = occ.shape
        Ca = feat.shape[-1]
        if feat.shape[:3] != occ.shape[:3] or Ca % D != 0:
            raise RuntimeError("feat must be [bs, Hb, Wb, pred_height * k]")
        world, c0, n = _shard(bs * Hb * Wb, group)
        alloc = torch.zeros if world > 1 else torch.empty           # other ranks' cells enter the all-reduce as 0
        prob = alloc(tuple(occ.shape), dtype=torch.float32, device=occ.device)
        pooled = alloc((bs, Hb * Wb, Ca), dtype=torch.float32, device=occ.device)
        # the forward's sums, read by the backward instead of a second march (3 x 2.56 MB); only this rank's cells
        # are filled / read
        aux = torch.empty((3,) + tuple(occ.shape), dtype=torch.float32, device=occ.device)
        L = _lib.lib()
        with torch.cuda.device(occ.device):
            st = _lib.stream_ptr(occ.device)
            _lib.check(L.vidar_latent_prob_forward(_lib.ptr(occ), _lib.ptr(prob), _lib.ptr(aux), bs, D, Hb, Wb,
                                                   int(grid_num), float(grid_step), int(act), c0, n, st))
            if world > 1:
                dist.all_reduce(prob, group=group)
            _lib.check(L.vidar_latent_pool_forward(_lib.ptr(prob), _lib.ptr(feat), _lib.ptr(pooled), _lib.ptr(aux), bs, D,
                                                   Ca // D, Hb, Wb, int(grid_num), float(grid_step), float(eps), c0, n, st))
            if world > 1:
                dist.all_reduce(pooled, group=group)
        ctx.save_for_backward(occ, feat, prob, pooled, aux)
        ctx.cfg = (int(grid_num), float(grid_step), float(eps), int(act), group, world, c0, n)
        return prob, pooled

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_prob, grad_pooled):
        import torch.distributed as dist
        occ, feat, prob, pooled, aux = ctx.saved_tensors
        grid_num, grid_step, eps, act, group, world, c0, n = ctx.cfg
        bs, Hb, Wb, D = occ.shape
        Ca = feat.shape[-1]
        grad_pooled = grad_pooled.float().contiguous()
        both = None
        if world > 1:
            # one buffer [2, ...] so the two partial maps travel in a single all-reduce
            both = torch.zeros((2,) + tuple(occ.shape), dtype=torch.float32, device=occ.device) if Ca == D else None
            gpm = both[0] if both is not None else torch.zeros_like(occ)
            gfe = both[1] if both is not None else torch.zeros_like(feat)
        else:
            # the total gradient reaching the prob map starts as the upstream grad_prob; phase 2 adds to it
            gpm = torch.empty_like(occ).copy_(grad_prob)
            gfe = torch.zeros_like(feat)
        grad_occ = torch.zeros_like(occ)
        L = _lib.lib()
        with torch.cuda.device(occ.device):
            st = _lib.stream_ptr(occ.device)
            _lib.check(L.vidar_latent_pool_backward(_lib.ptr(prob), _lib.ptr(feat), _lib.ptr(pooled), _lib.ptr(aux),
                                                    _lib.ptr(grad_pooled), _lib.ptr(gpm), _lib.ptr(gfe), bs, D, Ca // D,
                                                    Hb, Wb, grid_num, grid_step, eps, c0, n, st))
            if world > 1:
                if both is not None:
                    dist.all_reduce(both, group=group)
                else:
                    dist.all_reduce(gpm, group=group)
                    dist.all_reduce(gfe, group=group)
                gpm = (gpm + grad_prob.float()).contiguous()
            _lib.check(L.vidar_latent_prob_backward(_lib.ptr(occ), _lib.ptr(aux), _lib.ptr(gpm), _lib.ptr(grad_occ), bs, D,
                                                    Hb, Wb, grid_num, grid_step, act, c0, n, st))
            if world > 1:
                dist.all_reduce(grad_occ, group=group)
        return grad_occ, gfe.clone() if both is not None else gfe, None, None, None, None, None


class _FusedLatentRendering(torch.autograd.Function):
    """The whole module as one node: embed [bs,Hb,Wb,E] + the six Linear parameters -> out.

      forward : proj_in(rows) -> [all_reduce occ|feat] -> prob(cells) -> [all_reduce prob]
                -> pool(cells) -> proj_out(rows) -> [all_gather out]
      backward: proj_out_bwd(rows) -> pool_bwd(cells) -> [all_reduce grad_prob_map|grad_feat]
                -> prob_bwd(cells) -> [all_reduce grad_occ] -> proj_in_bwd(rows)
                -> [all_gather grad_embed, all_reduce parameter grads]
    Bracketed steps only when `group` has more than one rank: every rank then owns a contiguous
    share of the bs*Hb*Wb rows/cells (SURVEY.md 8e); inputs, outputs and all returned gradients are
    replicated, so the node is a drop-in for the single-GPU one."""

    @staticmethod
    def forward(ctx, embed, w_occ, b_occ, w_feat, b_feat, w_b, b_b, grid_num, grid_step, eps, act, group, rows_io=None):
        """`rows_io` = (bs, Hb, Wb): `embed` holds only THIS RANK's rows [n, E] of the [bs*Hb*Wb, E] BEV grid and
        only its rows of the output are returned (row-wise consumers -- LayerNorm, FFN -- need no more): the two
        41 MB all-gathers of the replicated mode disappear."""
        import torch.distributed as dist
        from ..sharding import gather_rows
        _lib.require_cuda(embed=embed.contiguous())
        params = [p.detach().float().contiguous() for p in (w_occ, b_occ, w_feat, b_feat, w_b, b_b)]
        w_occ, b_occ, w_feat, b_feat, w_b, b_b = params
        D, A = w_occ.shape[0], w_feat.shape[0]
        if rows_io is not None:
            bs, Hb, Wb = rows_io
            E = embed.shape[-1]
        else:
            bs, Hb, Wb, E = embed.shape
        R = bs * Hb * Wb
        world, c0, n = _shard(R, group)
        c1 = c0 + n
        if rows_io is not None:
            if embed.numel() != n * E:
                raise RuntimeError(f"rows_io: expected this rank's {n} rows of {E} channels, got {tuple(embed.shape)}")
            x_l = embed.detach().float().contiguous().view(n, E)
        else:
            x_l = embed.detach().float().contiguous().view(R, E)[c0:c1]
        dev = embed.device
        even = world > 1 and R % world == 0           # equal contiguous shards: all-gather instead of zero-padded all-reduce
        alloc = torch.zeros if (world > 1 and not even) else torch.empty
        flat = alloc(R * (D + A), dtype=torch.float32, device=dev)       # occ | feat in one buffer: one collective
        occ, feat = flat[: R * D].view(R, D), flat[R * D:].view(R, A)
        prob = alloc((R, D), dtype=torch.float32, device=dev)
        pooled = torch.empty((R, A), dtype=torch.float32, device=dev)    # only this rank's rows are filled / read
        aux = torch.empty((3, R, D), dtype=torch.float32, device=dev)
        out_l = torch.empty((n, E), dtype=torch.float32, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            if even:
                # this rank's [occ rows | feat rows] contiguous -> ONE all-gather, then two strided copies into the maps
                mine = torch.empty(n * (D + A), dtype=torch.float32, device=dev)
                o_l, f_l = mine[: n * D].view(n, D), mine[n * D:].view(n, A)
                _lib.check(L.vidar_latent_proj_in_forward(_lib.ptr(x_l), _lib.ptr(w_occ), _lib.ptr(b_occ), _lib.ptr(w_feat),
                                                          _lib.ptr(b_feat), _lib.ptr(o_l), _lib.ptr(f_l), n, E, D, A, st))
                gathered = torch.empty(world * n * (D + A), dtype=torch.float32, device=dev)
                dist.all_gather_into_tensor(gathered, mine, group=group)
                g2 = gathered.view(world, n * (D + A))
                occ.view(world, n * D).copy_(g2[:, : n * D])
                feat.view(world, n * A).copy_(g2[:, n * D:])
            else:
                _lib.check(L.vidar_latent_proj_in_forward(_lib.ptr(x_l), _lib.ptr(w_occ), _lib.ptr(b_occ), _lib.ptr(w_feat),
                                                          _lib.ptr(b_feat), _lib.ptr(occ[c0:c1]), _lib.ptr(feat[c0:c1]), n, E, D, A, st))
                if world > 1:
                    dist.all_reduce(flat, group=group)
            _lib.check(L.vidar_latent_prob_forward(_lib.ptr(occ), _lib.ptr(prob), _lib.ptr(aux), bs, D, Hb, Wb,
                                                   int(grid_num), float(grid_step), int(act), c0, n, st))
            if even:
                dist.all_gather_into_tensor(prob.view(-1), prob[c0:c1].clone().view(-1), group=group)
            elif world > 1:
                dist.all_reduce(prob, group=group)
            _lib.check(L.vidar_latent_pool_forward(_lib.ptr(prob), _lib.ptr(feat), _lib.ptr(pooled), _lib.ptr(aux), bs, D,
                                                   A // D, Hb, Wb, int(grid_num), float(grid_step), float(eps), c0, n, st))
            _lib.check(L.vidar_latent_proj_out_forward(_lib.ptr(pooled[c0:c1]), _lib.ptr(prob[c0:c1]), _lib.ptr(w_b),
                                                       _lib.ptr(b_b), _lib.ptr(out_l), n, E, D, A, st))
            out = out_l if rows_io is not None else gather_rows(out_l, world, R, group)
        ctx.save_for_backward(x_l, occ, feat, prob, pooled, aux, *params)
        ctx.cfg = (int(grid_num), float(grid_step), float(eps), int(act), group, world, c0, n, (bs, Hb, Wb, E, D, A),
                   rows_io is not None)
        return out if rows_io is not None else out.view(bs, Hb, Wb, E)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        import torch.distributed as dist
        from ..sharding import gather_rows
        x_l, occ, feat, prob, pooled, aux, w_occ, b_occ, w_feat, b_feat, w_b, b_b = ctx.saved_tensors
        grid_num, grid_step, eps, act, group, world, c0, n, (bs, Hb, Wb, E, D, A), rows_io = ctx.cfg
        R, c1 = bs * Hb * Wb, c0 + n
        dev = x_l.device
        g_l = grad_out.float().contiguous().view(n, E) if rows_io else grad_out.float().contiguous().view(R, E)[c0:c1]
        # parameter gradients in one buffer (one all-reduce when sharded): w_occ b_occ w_feat b_feat w_b b_b
        sizes = [D * E, D, A * E, A, E * A, E]
        pg = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        g_w_occ, g_b_occ, g_w_feat, g_b_feat, g_w_b, g_b_b = torch.split(pg, sizes)
        g_pooled = torch.empty((R, A), dtype=torch.float32, device=dev)       # rows [c0, c1) used
        g_prob = torch.empty((n, D), dtype=torch.float32, device=dev)
        maps = torch.zeros(R * (D + A), dtype=torch.float32, device=dev)      # grad_prob_map | grad_feat
        gpm, gfe = maps[: R * D].view(R, D), maps[R * D:].view(R, A)
        grad_occ = torch.zeros((R, D), dtype=torch.float32, device=dev)
        gx_l = torch.empty((n, E), dtype=torch.float32, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            _lib.check(L.vidar_latent_proj_out_backward(_lib.ptr(g_l), _lib.ptr(pooled[c0:c1]), _lib.ptr(prob[c0:c1]),
                                                        _lib.ptr(w_b), _lib.ptr(b_b), _lib.ptr(g_pooled[c0:c1]), _lib.ptr(g_prob),
                                                        _lib.ptr(g_w_b), _lib.ptr(g_b_b), n, E, D, A, st))
            _lib.check(L.vidar_latent_pool_backward(_lib.ptr(prob), _lib.ptr(feat), _lib.ptr(pooled), _lib.ptr(aux),
                                                    _lib.ptr(g_pooled), _lib.ptr(gpm), _lib.ptr(gfe), bs, D, A // D,
                                                    Hb, Wb, grid_num, grid_step, eps, c0, n, st))
            if world > 1:
                dist.all_reduce(maps, group=group)
            gpm[c0:c1] += g_prob          # prob's direct use in the final product (this rank's cells)
            _lib.check(L.vidar_latent_prob_backward(_lib.ptr(occ), _lib.ptr(aux), _lib.ptr(gpm), _lib.ptr(grad_occ), bs, D,
                                                    Hb, Wb, grid_num, grid_step, act, c0, n, st))
            if world > 1:
                dist.all_reduce(grad_occ, group=group)
            _lib.check(L.vidar_latent_proj_in_backward(_lib.ptr(x_l), _lib.ptr(w_occ), _lib.ptr(w_feat),
                                                       _lib.ptr(grad_occ[c0:c1]), _lib.ptr(gfe[c0:c1]), _lib.ptr(gx_l),
                                                       _lib.ptr(g_w_occ), _lib.ptr(g_b_occ), _lib.ptr(g_w_feat),
                                                       _lib.ptr(g_b_feat), n, E, D, A, st))
            if world > 1:
                dist.all_reduce(pg, group=group)
            gx = gx_l if rows_io else gather_rows(gx_l, world, R, group).view(bs, Hb, Wb, E)
        return (gx, g_w_occ.view(D, E), g_b_occ, g_w_feat.view(A, E), g_b_feat, g_w_b.view(E, A), g_b_b,
                None, None, None, None, None, None)


def fused_projection_supported(E, D, A):
    """Shapes csrc/latent_proj.cu handles (the shipped configuration is E=256, D=16, A=16)."""
    return (E in (128, 256) and A == 16 and A % D == 0 and (D + A) % 4 == 0 and D + A <= 32
            and E % D == 0 and (E // D) % 4 == 0 and 128 % (E // D) == 0)


def latent_render_core(occ, feat, grid_num, grid_step, eps, act, group=None):
    """(occ, feat) -> (prob, pooled).  `group`: a torch.distributed process group over which the BEV
    cells are sharded (None or a 1-rank group = single GPU)."""
    return _LatentRenderCore.apply(occ, feat, grid_num, grid_step, eps, act, group)


@ATTENTION.register_module()
class LatentRendering(BaseModule):
    """Ray-marching adaptor ("latent rendering") of ViDAR, latent_rendering.py:37-162."""

    def __init__(self, embed_dims=256, num_pred_fcs=2, pred_height=1, grid_num=128, grid_step=0.5,
                 reduction=16, act="exp", viz_response=False, init_cfg=None):
        super().__init__(init_cfg)
        self.embed_dims = embed_dims
        self.num_pred_fcs = num_pred_fcs
        self.grid_num = grid_num
        self.grid_step = grid_step
        self.viz_response = viz_response
        self.act = act
        branch = []
        for _ in range(self.num_pred_fcs):
            branch.append(nn.Linear(self.embed_dims, self.embed_dims))
            branch.append(nn.LayerNorm(self.embed_dims))
            branch.append(nn.ReLU(inplace=True))
        branch.append(nn.Linear(self.embed_dims, pred_height))
        self.unsup_raymarching_head = nn.Sequential(*branch)
        self.pred_height = pred_height
        self.lora_a = nn.Linear(self.embed_dims, self.embed_dims // reduction)
        self.lora_b = nn.Linear(self.embed_dims // reduction, self.embed_dims)
        self.process_group = None     # set to a process group to shard the BEV cells over its ranks
        self.fuse_projections = True  # False: keep the Linear layers as PyTorch ops around the CUDA core

    def forward_rows(self, embed_rows, bs, bev_h, bev_w, eps=1e-3):
        """Row-sharded call: `embed_rows` [n, embed_dims] are THIS RANK's rows (`sharding.shard_range` of the
        bs*bev_h*bev_w BEV rows over `process_group`); returns the same rows of the output.  The small
        occupancy / feature / prob maps (2.56 MB each) are exchanged inside, the 41 MB grid never is."""
        head = self.unsup_raymarching_head
        if not (len(head) == 1 and fused_projection_supported(self.embed_dims, self.pred_height, self.lora_a.out_features)
                and embed_rows.is_cuda and embed_rows.dtype == torch.float32):
            raise RuntimeError("forward_rows needs the fused configuration (num_pred_fcs=0, E in {128,256}, 16 feature channels)")
        return _FusedLatentRendering.apply(embed_rows, head[0].weight, head[0].bias, self.lora_a.weight, self.lora_a.bias,
                                           self.lora_b.weight, self.lora_b.bias, self.grid_num, self.grid_step, eps,
                                           _ACT[self.act], self.process_group, (bs, bev_h, bev_w))

    def forward(self, embed, eps=1e-3, **kwargs):
        """embed [bs, bev_h, bev_w, embed_dims] -> same shape."""
        if self.act not in _ACT:
            raise NotImplementedError("Only support exp or sigmoid activation_fn for now.")
        bs, bev_h, bev_w, _ = embed.shape
        head = self.unsup_raymarching_head
        if (self.fuse_projections and len(head) == 1 and embed.is_cuda and embed.dtype == torch.float32
                and not torch.is_autocast_enabled()
                and fused_projection_supported(self.embed_dims, self.pred_height, self.lora_a.out_features)
                and all(p is not None for p in (head[0].bias, self.lora_a.bias, self.lora_b.bias))):
            return _FusedLatentRendering.apply(embed, head[0].weight, head[0].bias, self.lora_a.weight, self.lora_a.bias,
                                               self.lora_b.weight, self.lora_b.bias, self.grid_num, self.grid_step, eps,
                                               _ACT[self.act], self.process_group)
        occ = head(embed)                                   # [bs, h, w, pred_height]   (:94)
        feat = self.lora_a(embed)                           # [bs, h, w, embed/reduction] (:134)
        prob, pooled = latent_render_core(occ, feat, self.grid_num, self.grid_step, eps, _ACT[self.act],
                                          self.process_group)
        out = self.lora_b(pooled).view(bs, bev_h, bev_w, self.embed_dims)       # (:153-155)
        out = out.view(bs, bev_h, bev_w, self.pred_height, -1) * prob.view(bs, bev_h, bev_w, self.pred_height, 1)
        return out.view(bs, bev_h, bev_w, self.embed_dims)
