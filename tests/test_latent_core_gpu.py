"""LatentRendering core (vidar_b200/csrc/latent_render.cu) against the fp64 oracle `latent_core_fp64`.

Covers every <VEC, G> instantiation of the pool kernels and both VEC of the prob kernels, BEVs with and
without a centre cell, the march bounds over grid_step / grid_num, saturated activations (exactly-zero
transmittance factors), the `aux` buffer the forward fills and the backward reads through the C ABI, and the
phase-wise entry points on cell ranges, the way the cell-sharded core calls them."""
import os
import re

import pytest
import torch

from oracle import latent_render_ref as ref
from tests.parity import close
from vidar_b200 import _lib
from vidar_b200.modules.latent_rendering import latent_render_core
from vidar_b200.sharding import shard_range

ACT = {"exp": 0, "sigmoid": 1}
EPS = 1e-3
NAN = float("nan")
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vidar_b200", "csrc", "latent_render.cu")


def vec_of(D, G):
    """check_lr's lane layout: a lane takes 4 heights when D % 4 == 0 and G <= 4, else 1."""
    return 4 if D % 4 == 0 and G <= 4 else 1


# (D, G, VEC, act): all 8 pool instantiations <VEC, G> and both prob instantiations <VEC>
MATRIX = [(16, 1, 4, "sigmoid"), (32, 1, 4, "exp"), (8, 2, 4, "sigmoid"), (4, 4, 4, "exp"), (32, 4, 4, "sigmoid"),
          (1, 1, 1, "exp"), (2, 2, 1, "sigmoid"), (2, 4, 1, "exp"), (4, 8, 1, "sigmoid"), (16, 8, 1, "exp"),
          (1, 16, 1, "sigmoid"), (32, 16, 1, "exp")]
MATRIX_IDS = [f"D{D}-G{G}-vec{v}-{a}" for D, G, v, a in MATRIX]


def test_matrix_covers_every_instantiation():
    src = open(SRC).read()
    assert "vec = (D % 4 == 0 && G <= 4) ? 4 : 1;" in src, "the VEC rule changed: update vec_of and MATRIX"
    body = src[src.index("#define LR_DISPATCH_VG"):src.index("} while (0)", src.index("#define LR_DISPATCH_VG"))]
    dispatched = {(int(v), int(g)) for v, g in re.findall(r"KERNEL<(\d+), (\d+)>", body)}
    assert len(dispatched) == 8
    assert {(vec_of(D, G), G) for D, G, _, _ in MATRIX} == dispatched
    assert all(vec_of(D, G) == v for D, G, v, _ in MATRIX)
    assert {a for *_, a in MATRIX} == set(ACT)


def _inputs(bs, Hb, Wb, D, G, seed):
    g = torch.Generator().manual_seed(seed)
    occ = torch.randn(bs, Hb, Wb, D, generator=g) * 1.5
    feat = torch.randn(bs, Hb, Wb, D * G, generator=g)
    gp = torch.randn(bs, Hb, Wb, D, generator=g)
    gq = torch.randn(bs, Hb * Wb, D * G, generator=g)
    return occ, feat, gp, gq


def _oracle(occ, feat, gps, gq, grid_num, grid_step, act):
    """fp64 prob, pooled and, for each upstream grad_prob in gps (with grad_pooled gq), (grad occ, grad feat,
    total gradient reaching the prob map)."""
    o, f = occ.double().requires_grad_(True), feat.double().requires_grad_(True)
    p, q = ref.latent_core_fp64(o, f, grid_num, grid_step, EPS, act)
    grads = [torch.autograd.grad((p, q), (o, f, p), (gp.double(), gq.double()), retain_graph=True) for gp in gps]
    return p.detach(), q.detach(), grads


def _check_core(cuda, bs, Hb, Wb, D, G, grid_num, grid_step, act, seed, occ=None):
    """latent_render_core forward, then its backward with a non-zero grad_prob and with grad_prob = 0 (which
    leaves only the phase-2 -> prob map -> occ path), all against the oracle."""
    occ_r, feat, gp, gq = _inputs(bs, Hb, Wb, D, G, seed)
    occ = occ_r if occ is None else occ
    gps = (gp, torch.zeros_like(gp))
    p64, q64, grads64 = _oracle(occ, feat, gps, gq, grid_num, grid_step, act)
    o, f = occ.to(cuda).requires_grad_(True), feat.to(cuda).requires_grad_(True)
    p, q = latent_render_core(o, f, grid_num, grid_step, EPS, ACT[act])
    tag = f"bs{bs} {Hb}x{Wb} D{D} G{G} n{grid_num} step{grid_step} {act}"
    close(p, p64, f"{tag}: prob")
    close(q, q64, f"{tag}: pooled")
    for gp_, (go64, gf64, _), what in zip(gps, grads64, ("grad_prob", "grad_prob=0")):
        go, gf = torch.autograd.grad((p, q), (o, f), (gp_.to(cuda), gq.to(cuda)), retain_graph=True)
        close(go, go64, f"{tag} {what}: grad occ")
        close(gf, gf64, f"{tag} {what}: grad feat")
    return occ, feat, gp, gq


@pytest.mark.gpu
@pytest.mark.parametrize("D,G,vec,act", MATRIX, ids=MATRIX_IDS)
def test_instantiation_matrix(cuda, D, G, vec, act):
    assert vec_of(D, G) == vec
    i = MATRIX.index((D, G, vec, act))
    _check_core(cuda, 2, 9 + i % 3, 10 + i % 2, D, G, 40, 0.5, act, seed=100 + i)


# (bs, Hb, Wb, D, G, grid_num, grid_step, act).  Waypoints per warp step WPI = 32 / (D / VEC).
GEOMETRY = {
    "odd_x_odd": (1, 9, 9, 16, 1, 33, 0.5, "sigmoid"),         # centre cell; grid_num = 4 WPI + 1
    "odd_x_even": (3, 9, 12, 4, 2, 31, 0.25, "exp"),           # grid_num = WPI - 1
    "even_x_odd": (1, 12, 9, 16, 1, 3, 1.0, "sigmoid"),        # grid_num clamps both marches
    "wide": (3, 6, 17, 1, 16, 65, 2.0, "exp"),                 # grid_num = 2 WPI + 1, far past the border
    "tall": (1, 17, 6, 8, 2, 2, 0.5, "sigmoid"),               # grid_num clamps both marches
    "2x2": (3, 2, 2, 16, 1, 9, 0.5, "exp"),
    "3x3": (1, 3, 3, 32, 1, 5, 0.25, "sigmoid"),               # centre cell; WPI = 4
    "odd_x_odd_exp": (3, 7, 11, 2, 8, 47, 1.0, "exp"),         # centre cell, VEC 1
    "63x64": (1, 63, 64, 16, 1, 96, 0.5, "sigmoid"),           # rays past the border from every cell
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GEOMETRY))
def test_geometry(cuda, name):
    bs, Hb, Wb, D, G, grid_num, grid_step, act = GEOMETRY[name]
    _check_core(cuda, bs, Hb, Wb, D, G, grid_num, grid_step, act, seed=len(name) * 7 + Hb)


def _planted(bs, Hb, Wb, D, act, seed):
    """occ with blocks of +40 (1 - a == 0 exactly, in fp32 and fp64), -40 (a ~ 0) and ~15 (1 - a ~ 3e-7, what
    the backward divides by); under exp a block of occ <= 0 (a == 0, zero relu gradient).  One +40 block covers
    only the even heights, so rays of one cell see different zero counts per height."""
    g = torch.Generator().manual_seed(seed)
    occ = torch.randn(bs, Hb, Wb, D, generator=g) * 1.5
    occ[:, 10:14, 10:14] = 40.0
    occ[:, 2:6, 9:12, 0::2] = 40.0
    occ[:, 3:7, 1:5] = -40.0
    occ[:, 11:15, 2:6] = 15.0 + torch.rand(bs, 4, 4, D, generator=g) - 0.5
    if act == "exp":
        occ[:, 7:9, 12:15] = -torch.rand(bs, 2, 3, D, generator=g)
    return occ


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["sigmoid", "exp"])
@pytest.mark.parametrize("D,G", [(4, 2), (2, 4)], ids=["vec4", "vec1"])
def test_saturated_activations(cuda, D, G, act):
    bs, Hb, Wb, grid_num, grid_step = 2, 16, 16, 40, 0.5
    occ = _planted(bs, Hb, Wb, D, act, seed=D + G)
    # the case reaches rays with 0, 1 and >= 2 exactly-zero factors, and factors 1 - a below 1e-6
    grid, m1, _ = ref.geometry(Hb, Wb, grid_num, grid_step, sqrt=ref.sqrt_rn)
    x = torch.nn.functional.grid_sample(occ.double().permute(0, 3, 1, 2), grid.double()[None].expand(bs, -1, -1, -1),
                                        align_corners=False)
    f = 1 - (torch.sigmoid(x) if act == "sigmoid" else 1 - torch.exp(-torch.relu(x)))
    zeros = ((f == 0) & m1).sum(-1)
    assert (zeros == 0).any() and (zeros == 1).any() and (zeros >= 2).any()
    assert (((f > 0) & (f < 1e-6)) & m1).any()
    _check_core(cuda, bs, Hb, Wb, D, G, grid_num, grid_step, act, seed=D + G, occ=occ)


def _abi_core(cuda, occ, feat, gp, gq, grid_num, grid_step, act):
    """The four phase entry points on all cells, in the single-GPU core's order: prob and pool forward, then the pool
    backward into a copy of grad_prob and the prob backward from that sum.  The forward's outputs start as NaN, so a
    cell left unwritten shows.  Returns prob, pooled, aux, grad_prob_total, grad occ, grad feat."""
    bs, Hb, Wb, D = occ.shape
    G = feat.shape[-1] // D
    L, st, P = _lib.lib(), _lib.stream_ptr(cuda), _lib.ptr
    o, f, gpd, gqd = (t.to(cuda) for t in (occ, feat, gp, gq))
    cells, a = bs * Hb * Wb, ACT[act]
    prob, pooled = torch.full_like(o, NAN), torch.full((bs, Hb * Wb, D * G), NAN, device=cuda)
    aux = torch.full((3,) + tuple(o.shape), NAN, device=cuda)
    _lib.check(L.vidar_latent_prob_forward(P(o), P(prob), P(aux), bs, D, Hb, Wb, grid_num, grid_step, a, 0, cells, st))
    _lib.check(L.vidar_latent_pool_forward(P(prob), P(f), P(pooled), P(aux), bs, D, G, Hb, Wb, grid_num, grid_step, EPS,
                                           0, cells, st))
    total, go, gf = gpd.clone(), torch.zeros_like(o), torch.zeros_like(f)
    _lib.check(L.vidar_latent_pool_backward(P(prob), P(f), P(pooled), P(aux), P(gqd), P(total), P(gf), bs, D, G, Hb, Wb,
                                            grid_num, grid_step, EPS, 0, cells, st))
    _lib.check(L.vidar_latent_prob_backward(P(o), P(aux), P(total), P(go), bs, D, Hb, Wb, grid_num, grid_step, a, 0,
                                            cells, st))
    return prob, pooled, aux, total, go, gf


@pytest.mark.gpu
@pytest.mark.parametrize("D,G,vec,act", MATRIX, ids=MATRIX_IDS)
def test_aux_written_and_read_by_backward(cuda, D, G, vec, act):
    """The forward fills every cell of aux, and the backward that reads aux and pooled matches the oracle."""
    bs, Hb, Wb, grid_num, grid_step = 2, 7, 10, 24, 0.5
    i = MATRIX.index((D, G, vec, act))
    occ, feat, gp, gq = _inputs(bs, Hb, Wb, D, G, seed=200 + i)
    p64, q64, ((go64, gf64, gt64),) = _oracle(occ, feat, (gp,), gq, grid_num, grid_step, act)
    prob, pooled, aux, total, go, gf = _abi_core(cuda, occ, feat, gp, gq, grid_num, grid_step, act)
    assert not aux.isnan().any(), "aux not fully written"
    close(prob, p64, "prob")
    close(pooled, q64, "pooled")
    close(total, gt64, "grad_prob_total")
    close(go, go64, "grad occ")
    close(gf, gf64, "grad feat")


def _range_sets(total, HW):
    sets = {f"world{w}": [shard_range(total, r, w) for r in range(w)] for w in (2, 3, 7)}
    # a single first cell, a range across the batch-element boundary, a single last cell, an empty range at the end
    sets["hand"] = [(0, 1), (1, HW - 1), (HW - 1, HW + 1), (HW + 1, total - 1), (total - 1, total), (total, total)]
    return sets


@pytest.mark.gpu
@pytest.mark.parametrize("D,G,act", [(4, 4, "sigmoid"), (2, 8, "exp")], ids=["vec4", "vec1"])
def test_cell_ranges(cuda, D, G, act):
    """The four phase-wise entry points over sets of cell ranges that partition the bs*Hb*Wb cells, as
    _ShardedLatentRenderCore runs them on each rank: every range writes exactly its own cells, bit-identical to
    the full-range call, and reads aux only there (aux is NaN elsewhere); the all-reduces between the phases
    become sums of the per-range buffers."""
    bs, Hb, Wb, grid_num, grid_step = 2, 9, 11, 30, 0.5
    HW, total = Hb * Wb, bs * Hb * Wb
    occ, feat, gp, gq = _inputs(bs, Hb, Wb, D, G, seed=300 + D)
    p64, q64, ((go64, gf64, _),) = _oracle(occ, feat, (gp,), gq, grid_num, grid_step, act)
    L, st, P = _lib.lib(), _lib.stream_ptr(cuda), _lib.ptr
    o, f, gpd, gqd = (t.to(cuda) for t in (occ, feat, gp, gq))
    a = ACT[act]

    def prob_fwd(prob, aux, c0, n):
        _lib.check(L.vidar_latent_prob_forward(P(o), P(prob), P(aux), bs, D, Hb, Wb, grid_num, grid_step, a, c0, n, st))

    def pool_fwd(prob, pooled, aux, c0, n):
        _lib.check(L.vidar_latent_pool_forward(P(prob), P(f), P(pooled), P(aux), bs, D, G, Hb, Wb, grid_num, grid_step,
                                               EPS, c0, n, st))

    def pool_bwd(prob, pooled, aux, gpm, gfe, c0, n):
        _lib.check(L.vidar_latent_pool_backward(P(prob), P(f), P(pooled), P(aux), P(gqd), P(gpm), P(gfe), bs, D, G, Hb,
                                                Wb, grid_num, grid_step, EPS, c0, n, st))

    def prob_bwd(aux, gtot, go, c0, n):
        _lib.check(L.vidar_latent_prob_backward(P(o), P(aux), P(gtot), P(go), bs, D, Hb, Wb, grid_num, grid_step, a,
                                                c0, n, st))

    def nan(*shape):
        return torch.full(shape, NAN, device=cuda)

    # the full range
    prob, pooled, aux = nan(bs, Hb, Wb, D), nan(bs, HW, D * G), nan(3, bs, Hb, Wb, D)
    prob_fwd(prob, aux, 0, total)
    pool_fwd(prob, pooled, aux, 0, total)
    gpm, gfe, go = torch.zeros_like(o), torch.zeros_like(f), torch.zeros_like(o)
    pool_bwd(prob, pooled, aux, gpm, gfe, 0, total)
    prob_bwd(aux, gpm + gpd, go, 0, total)
    close(prob, p64, "prob")
    close(pooled, q64, "pooled")
    close(go, go64, "grad occ")
    close(gfe, gf64, "grad feat")
    cells = lambda t: t.reshape(total, -1)                       # [total, channels] view of a map
    aux_cells = lambda t: t.reshape(3, total, D)

    for name, ranges in _range_sets(total, HW).items():
        assert ranges[0][0] == 0 and ranges[-1][1] == total and all(r[1] == s[0] for r, s in zip(ranges, ranges[1:]))
        prob_sum, auxes = torch.zeros_like(prob), []
        for lo, hi in ranges:
            pr, ax = nan(bs, Hb, Wb, D), nan(3, bs, Hb, Wb, D)
            n0 = _lib.launch_count()
            prob_fwd(pr, ax, lo, hi - lo)
            assert _lib.launch_count() - n0 == (hi > lo)
            assert torch.equal(cells(pr)[lo:hi], cells(prob)[lo:hi]), f"{name} [{lo},{hi}): prob"
            assert torch.equal(aux_cells(ax)[:2, lo:hi], aux_cells(aux)[:2, lo:hi]), f"{name} [{lo},{hi}): aux"
            assert cells(pr)[:lo].isnan().all() and cells(pr)[hi:].isnan().all(), f"{name} [{lo},{hi}): prob outside"
            assert aux_cells(ax)[:, :lo].isnan().all() and aux_cells(ax)[:, hi:].isnan().all()
            cells(prob_sum)[lo:hi] += cells(pr)[lo:hi]
            auxes.append(ax)
        assert torch.equal(prob_sum, prob), f"{name}: summed prob"
        pooled_sum = torch.zeros_like(pooled)
        for (lo, hi), ax in zip(ranges, auxes):
            pq = nan(bs, HW, D * G)
            n0 = _lib.launch_count()
            pool_fwd(prob_sum, pq, ax, lo, hi - lo)
            assert _lib.launch_count() - n0 == (hi > lo)
            assert torch.equal(cells(pq)[lo:hi], cells(pooled)[lo:hi]), f"{name} [{lo},{hi}): pooled"
            assert torch.equal(aux_cells(ax)[2, lo:hi], aux_cells(aux)[2, lo:hi]), f"{name} [{lo},{hi}): aux sums"
            assert cells(pq)[:lo].isnan().all() and cells(pq)[hi:].isnan().all(), f"{name} [{lo},{hi}): pooled outside"
            assert aux_cells(ax)[2, :lo].isnan().all() and aux_cells(ax)[2, hi:].isnan().all()
            cells(pooled_sum)[lo:hi] += cells(pq)[lo:hi]
        assert torch.equal(pooled_sum, pooled), f"{name}: summed pooled"
        gpm_sum, gfe_sum, go_sum = torch.zeros_like(o), torch.zeros_like(f), torch.zeros_like(o)
        for (lo, hi), ax in zip(ranges, auxes):
            gpm_r, gfe_r = torch.zeros_like(o), torch.zeros_like(f)
            n0 = _lib.launch_count()
            pool_bwd(prob_sum, pooled_sum, ax, gpm_r, gfe_r, lo, hi - lo)
            assert _lib.launch_count() - n0 == (hi > lo)
            gpm_sum += gpm_r
            gfe_sum += gfe_r
        gtot = gpm_sum + gpd
        for (lo, hi), ax in zip(ranges, auxes):
            go_r = torch.zeros_like(o)
            n0 = _lib.launch_count()
            prob_bwd(ax, gtot, go_r, lo, hi - lo)
            assert _lib.launch_count() - n0 == (hi > lo)
            if hi == lo:
                assert not go_r.any()
            go_sum += go_r
        close(gpm_sum, gpm, f"{name}: summed grad_prob_map vs full range")
        close(gfe_sum, gfe, f"{name}: summed grad feat vs full range")
        close(go_sum, go, f"{name}: summed grad occ vs full range")
        close(gfe_sum, gf64, f"{name}: summed grad feat")
        close(go_sum, go64, f"{name}: summed grad occ")


@pytest.mark.gpu
@pytest.mark.parametrize("c0,n", [(0, 199), (198, 1), (5, 194), (199, 1), (-1, 2), (3, -1), (-5, -5), (0, -1),
                                  (1, 2 ** 62), (2 ** 62, 1)])
def test_bad_cell_ranges_are_rejected(cuda, c0, n):
    bs, Hb, Wb, D, G = 2, 9, 11, 4, 2          # 198 cells
    t = torch.zeros(bs * Hb * Wb * D * G * 3, device=cuda)
    L, st, P = _lib.lib(), _lib.stream_ptr(cuda), _lib.ptr
    n0 = _lib.launch_count()
    calls = (lambda: L.vidar_latent_prob_forward(P(t), P(t), P(t), bs, D, Hb, Wb, 8, 0.5, 1, c0, n, st),
             lambda: L.vidar_latent_pool_forward(P(t), P(t), P(t), P(t), bs, D, G, Hb, Wb, 8, 0.5, EPS, c0, n, st),
             lambda: L.vidar_latent_pool_backward(P(t), P(t), P(t), P(t), P(t), P(t), P(t), bs, D, G, Hb, Wb, 8, 0.5, EPS,
                                                  c0, n, st),
             lambda: L.vidar_latent_prob_backward(P(t), P(t), P(t), P(t), bs, D, Hb, Wb, 8, 0.5, 1, c0, n, st))
    for call in calls:
        with pytest.raises(RuntimeError, match="bad cell range"):
            _lib.check(call())
    assert _lib.launch_count() == n0
