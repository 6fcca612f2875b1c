"""The angular-bundle phase 2 backward of csrc/latent_render.cu (VEC 4, G 1), with the per-cell phase 1 backward behind
it, against the fp64 oracle `latent_core_fp64`, at the bench shape and at the bundle's edges: cell counts that are not a
multiple of the bundle, cell ranges that start and end inside a bundle, bundles across a batch-element boundary,
non-square BEVs, and small BEVs where many corners fall outside a bundle's box.  Also the fused module under CUDA
graph capture and on a side stream, since the cell order's scratch is allocated stream-ordered."""
import pytest
import torch

from oracle import latent_render_ref as ref
from tests.parity import close
from tests.test_latent_core_gpu import ACT, EPS, _abi_core, _check_core, _inputs, _oracle
from vidar_b200 import _lib
from vidar_b200.sharding import shard_range


@pytest.fixture(scope="module")
def bench_shape_oracle():
    occ, feat, gp, gq = _inputs(1, 200, 200, 16, 1, seed=7)
    _, _, ((go64, gf64, gt64),) = _oracle(occ, feat, (gp,), gq, 256, 0.5, "sigmoid")
    return (occ, feat, gp, gq), (go64, gf64, gt64)


@pytest.mark.gpu
def test_bench_shape(cuda, bench_shape_oracle):
    """1 x 200 x 200, pred_height 16, one channel per height, grid_num 256, step 0.5, sigmoid: bench.py's core."""
    (occ, feat, gp, gq), (go64, gf64, gt64) = bench_shape_oracle
    *_, total, go, gf = _abi_core(cuda, occ, feat, gp, gq, 256, 0.5, "sigmoid")
    close(total, gt64, "grad_prob_total")
    close(go, go64, "grad occ")
    close(gf, gf64, "grad feat")


# (bs, Hb, Wb, D, grid_num, grid_step, act): G = 1 so both backward kernels take the bundle path
EDGES = {
    "ncells_not_multiple": (1, 9, 12, 16, 40, 0.5, "sigmoid"),     # 108 cells: last bundle of 12
    "bs2": (2, 37, 41, 16, 60, 0.5, "exp"),                      # bundles across the batch-element boundary
    "150x200": (1, 150, 200, 16, 200, 0.5, "sigmoid"),
    "200x150": (1, 200, 150, 16, 200, 0.5, "sigmoid"),
    "d4_odd": (1, 31, 33, 4, 48, 0.5, "sigmoid"),                # centre cell, 1 lane per waypoint
    "d32": (2, 24, 20, 32, 40, 0.5, "exp"),                      # 8 lanes per waypoint, 80 KB of shared memory
    # small BEVs: a bundle spans a wide angle, many corners leave the 4 x 4 box
    "2x2": (3, 2, 2, 16, 9, 0.5, "sigmoid"),
    "3x3": (2, 3, 3, 16, 12, 0.25, "exp"),
    "9x12": (2, 9, 12, 8, 30, 1.0, "sigmoid"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGES))
def test_bundle_edges(cuda, name):
    bs, Hb, Wb, D, grid_num, grid_step, act = EDGES[name]
    _check_core(cuda, bs, Hb, Wb, D, 1, grid_num, grid_step, act, seed=Hb * 31 + Wb)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 7])
def test_sharded_ranges_at_200x200(cuda, world):
    """The phase-wise backward entry points on shard_range's cuts, which start and end inside bundles, summed over
    the ranks as the all-reduces do, against the oracle."""
    bs, Hb, Wb, D, grid_num, grid_step, act = 1, 200, 200, 16, 64, 0.5, "sigmoid"
    total = bs * Hb * Wb
    occ, feat, gp, gq = _inputs(bs, Hb, Wb, D, 1, seed=world)
    _, _, ((go64, gf64, _),) = _oracle(occ, feat, (gp,), gq, grid_num, grid_step, act)
    L, st, P = _lib.lib(), _lib.stream_ptr(cuda), _lib.ptr
    o, f, gpd, gqd = (t.to(cuda) for t in (occ, feat, gp, gq))
    prob, pooled, aux = torch.empty_like(o), torch.empty(bs, Hb * Wb, D, device=cuda), torch.empty(3, bs, Hb, Wb, D, device=cuda)
    _lib.check(L.vidar_latent_prob_forward(P(o), P(prob), P(aux), bs, D, Hb, Wb, grid_num, grid_step, ACT[act], 0, total, st))
    _lib.check(L.vidar_latent_pool_forward(P(prob), P(f), P(pooled), P(aux), bs, D, 1, Hb, Wb, grid_num, grid_step, EPS, 0,
                                           total, st))
    ranges = [shard_range(total, r, world) for r in range(world)]
    assert world == 2 or any((hi - lo) % 32 for lo, hi in ranges)
    gpm, gfe = torch.zeros_like(o), torch.zeros_like(f)
    for lo, hi in ranges:
        _lib.check(L.vidar_latent_pool_backward(P(prob), P(f), P(pooled), P(aux), P(gqd), P(gpm), P(gfe), bs, D, 1, Hb, Wb,
                                                grid_num, grid_step, EPS, lo, hi - lo, st))
    gtot, go = gpm + gpd, torch.zeros_like(o)
    for lo, hi in ranges:
        _lib.check(L.vidar_latent_prob_backward(P(o), P(aux), P(gtot), P(go), bs, D, Hb, Wb, grid_num, grid_step,
                                                ACT[act], lo, hi - lo, st))
    close(gfe, gf64, f"world {world}: grad feat")
    close(go, go64, f"world {world}: grad occ")


def _module(cuda):
    import vidar_b200.modules  # noqa: F401
    from vidar_b200.registry import build_attention
    torch.manual_seed(0)
    return build_attention(dict(type="LatentRendering", embed_dims=256, num_pred_fcs=0, pred_height=16, grid_num=64,
                                grid_step=0.5, reduction=16, act="sigmoid")).to(cuda)


def _eager(mod, emb, gout):
    e = emb.detach().clone().requires_grad_(True)
    mod.zero_grad(set_to_none=True)
    out = mod(e)
    out.backward(gout)
    return out.detach(), e.grad.detach(), mod.lora_a.weight.grad.detach().clone()


@pytest.mark.gpu
def test_module_cuda_graph(cuda):
    """Forward + backward captured in one CUDA graph as bench.py does, replayed, then replayed on new inputs."""
    mod = _module(cuda)
    g = torch.Generator(device=cuda).manual_seed(1)
    emb = torch.randn(1, 60, 50, 256, device=cuda, generator=g)
    gout = torch.randn(1, 60, 50, 256, device=cuda, generator=g)
    s_emb, s_gout = emb.clone(), gout.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _eager(mod, s_emb, s_gout)                       # warm-up off the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    x = s_emb.detach().requires_grad_(True)
    mod.zero_grad(set_to_none=True)
    with torch.cuda.graph(graph):
        out = mod(x)
        out.backward(s_gout)
    for k in range(2):
        if k:
            s_emb.copy_(torch.randn(1, 60, 50, 256, device=cuda, generator=g))
            s_gout.copy_(torch.randn(1, 60, 50, 256, device=cuda, generator=g))
        graph.replay()
        torch.cuda.synchronize()
        want_out, want_gx, want_gw = _eager(mod, s_emb, s_gout)
        assert torch.equal(out.detach(), want_out), f"replay {k}: output"
        close(x.grad, want_gx.double(), f"replay {k}: grad embed")
    del graph


@pytest.mark.gpu
def test_side_stream(cuda):
    mod = _module(cuda)
    g = torch.Generator(device=cuda).manual_seed(2)
    emb = torch.randn(1, 40, 45, 256, device=cuda, generator=g)
    gout = torch.randn(1, 40, 45, 256, device=cuda, generator=g)
    want = _eager(mod, emb, gout)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = _eager(mod, emb, gout)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(got[0], want[0])
    for a, b, w in zip(got[1:], want[1:], ("grad embed", "grad lora_a")):
        close(a, b.double(), w)
