"""LatentRendering's fused projections (csrc/latent_proj.cu) past their first persistent round.

Each kernel's grid is capped at (SMs x blocks per SM) blocks that loop over row tiles, and the backward
kernels carry the weight- and bias-gradient sums in registers from tile to tile.  Row counts are derived
from the card's SM count and each kernel's tile and blocks per SM (oracle/encoder_front_ref.py
`proj_launch`): the bench's 40 000 rows, 80 000 (two samples), exactly two full rounds, one round -+ 1
row and a ragged last round.  Inputs have non-zero means and gradients of mixed scale, and every output
is held to its elementwise bound (the module docstring of oracle/encoder_front_ref.py) times SAFETY = 2
against an fp64 reference.  Gradient buffers start non-zero and the backward runs twice on them: the C
ABI adds (grad_W +=).  The largest error / bound per quantity is printed at the end (pytest -s).
"""
import pytest
import torch

from oracle import encoder_front_ref as efr
from tests import latent_cases as lc
import vidar_b200.modules  # noqa: F401  (registers the classes)
from vidar_b200 import _lib
from vidar_b200.modules import latent_rendering as lr
from vidar_b200.registry import build_attention

pytestmark = pytest.mark.gpu
SAFETY = 2.0
RATIOS = {}
KERNELS = ("proj_in_fwd", "proj_in_bwd", "proj_out_fwd", "proj_out_bwd")
ACC = ("grad_w_occ", "grad_b_occ", "grad_w_feat", "grad_b_feat", "grad_w_b", "grad_b_b")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest error / bound per quantity:")
    for k in sorted(RATIOS):
        print(f"  {k:36s} {RATIOS[k]:.3e}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _round(kernel, sms):
    return efr.proj_launch(kernel, 1 << 40, sms)[1]


def _rows(case, sms):
    rb, rf = _round("proj_in_bwd", sms), _round("proj_in_fwd", sms)
    rows = {"bench": 40000, "bs2": 80000, "two_rounds": 2 * rb, "round-1": rb - 1, "round+1": rb + 1,
            "ragged": 2 * rf + 777}[case]
    # the coverage each count claims
    if case in ("bench", "bs2"):
        for k in KERNELS:
            assert rows >= 2 * _round(k, sms), k              # every kernel runs two full rounds and more
    elif case == "two_rounds":
        assert all(rows == 2 * _round(k, sms) for k in ("proj_in_bwd", "proj_out_bwd"))
    elif case in ("round-1", "round+1"):
        assert abs(rows - _round("proj_out_bwd", sms)) == 1
    else:
        assert all(rows > 2 * _round(k, sms) and rows % _round(k, sms) % 32 for k in KERNELS)
    return rows


def _check(got, want, bound, key):
    err = (got.double() - want).abs()
    ratio = float((err / (SAFETY * bound)).max())
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)
    assert ratio < 1, f"{key}: error / bound {ratio:.3e}"


@pytest.mark.parametrize("case,E,D", [(c, 256, 16) for c in ("bench", "bs2", "two_rounds", "round-1", "round+1", "ragged")]
                         + [(c, E, D) for E, D in ((128, 8), (256, 4)) for c in ("bench", "round+1", "ragged")])
def test_projection_kernels_past_one_round(cuda, case, E, D):
    sms = _sms()
    rows, A = _rows(case, sms), 16
    t = lc.proj_inputs(rows, E, D, A, seed=rows + E + D, device=cuda)
    d = {k: v.double() for k, v in t.items()}
    ref = efr.proj_reference(**d)
    g = torch.Generator(device=cuda).manual_seed(7)
    shapes = dict(grad_w_occ=(D, E), grad_b_occ=(D,), grad_w_feat=(A, E), grad_b_feat=(A,), grad_w_b=(E, A), grad_b_b=(E,))
    acc0 = {k: torch.randn(s, generator=g, device=cuda) for k, s in shapes.items()}
    buf = {k: v.clone() for k, v in acc0.items()}
    L, st, P = _lib.lib(), _lib.stream_ptr(cuda), _lib.ptr
    out = {k: torch.empty(rows, n, device=cuda) for k, n in (("occ", D), ("feat", A), ("out", E))}
    _lib.check(L.vidar_latent_proj_in_forward(P(t["x"]), P(t["w_occ"]), P(t["b_occ"]), P(t["w_feat"]), P(t["b_feat"]),
                                              P(out["occ"]), P(out["feat"]), rows, E, D, A, st))
    _lib.check(L.vidar_latent_proj_out_forward(P(t["pooled"]), P(t["prob"]), P(t["w_b"]), P(t["b_b"]), P(out["out"]),
                                               rows, E, D, A, st))

    def backward():
        r = {k: torch.empty(rows, n, device=cuda) for k, n in (("grad_embed", E), ("grad_pooled", A), ("grad_prob", D))}
        _lib.check(L.vidar_latent_proj_in_backward(P(t["x"]), P(t["w_occ"]), P(t["w_feat"]), P(t["g_occ"]), P(t["g_feat"]),
                                                   P(r["grad_embed"]), P(buf["grad_w_occ"]), P(buf["grad_b_occ"]),
                                                   P(buf["grad_w_feat"]), P(buf["grad_b_feat"]), rows, E, D, A, st))
        _lib.check(L.vidar_latent_proj_out_backward(P(t["g_out"]), P(t["pooled"]), P(t["prob"]), P(t["w_b"]), P(t["b_b"]),
                                                    P(r["grad_pooled"]), P(r["grad_prob"]), P(buf["grad_w_b"]),
                                                    P(buf["grad_b_b"]), rows, E, D, A, st))
        return r

    first = backward()
    after1 = {k: v.clone() for k, v in buf.items()}
    second = backward()
    tag = f"E{E} D{D}"
    bounds = efr.proj_bounds(d, sms, {k: v.double() for k, v in acc0.items()})
    for k in ("occ", "feat", "out"):
        _check(out[k], ref[k], bounds[k], f"{k} {tag}")
    for k in ("grad_embed", "grad_pooled", "grad_prob"):
        _check(first[k], ref[k], bounds[k], f"{k} {tag}")
        assert torch.equal(first[k], second[k]), k           # written, not accumulated
    # one backward on a non-zero buffer, then a second one on top of it
    bounds2 = efr.proj_bounds(d, sms, {k: acc0[k].double() + ref[k] for k in ACC})
    for k in ACC:
        _check(after1[k], acc0[k].double() + ref[k], bounds[k], f"{k} {tag}")
        _check(buf[k], acc0[k].double() + 2 * ref[k], bounds[k] + bounds2[k], f"{k} (twice) {tag}")


def test_module_at_bench_size_fused_vs_unfused(cuda, monkeypatch):
    """[1, 200, 200, 256], the shipped shape: the module with its projections fused against the same
    module with torch Linears around the same core.  Each output / gradient may differ by SAFETY x the
    projection bound (computed from the unfused run's intermediates) plus the core's tolerance of
    tests/test_latent_gpu.py (1e-4 of max |.| for values, 2e-4 for gradients), since the two paths feed
    the core slightly different occupancy and feature maps."""
    m = build_attention(lc.CFG_FUSED)
    m.load_state_dict(lc.seeded_state(m, 31))
    m.to(cuda)
    g = torch.Generator().manual_seed(32)
    embed = (2 + torch.randn(1, 200, 200, 256, generator=g)).to(cuda)
    grad = ((0.5 + torch.randn(1, 200, 200, 256, generator=g)) * 10.0 ** (torch.rand(256, generator=g) * 4 - 3)).to(cuda)

    def run(fused):
        m.fuse_projections = fused
        m.zero_grad(set_to_none=True)
        e = embed.clone().requires_grad_(True)
        o = m(e)
        o.backward(grad)
        return o.detach(), e.grad, {n: p.grad.clone() for n, p in m.named_parameters()}

    n0 = _lib.launch_count()
    out_f, ge_f, gp_f = run(True)
    assert _lib.launch_count() - n0 == 8                     # the fused path ran: 4 projection + 4 core kernels
    # unfused run, keeping the projections' operands
    keep = {}
    core = lr.latent_render_core

    def core_keep(occ, feat, *a, **k):
        occ.retain_grad()
        feat.retain_grad()
        prob, pooled = core(occ, feat, *a, **k)
        prob.retain_grad()
        pooled.retain_grad()
        keep.update(occ=occ, feat=feat, prob=prob, pooled=pooled)
        return prob, pooled

    monkeypatch.setattr(lr, "latent_render_core", core_keep)
    out_u, ge_u, gp_u = run(False)
    E, D, A = 256, 16, 16
    rows = 40000
    dd = lambda v: v.detach().double().reshape(rows, -1)
    head, la, lb = m.unsup_raymarching_head[0], m.lora_a, m.lora_b
    d = dict(x=dd(embed), w_occ=head.weight.double(), b_occ=head.bias.double(), w_feat=la.weight.double(),
             b_feat=la.bias.double(), w_b=lb.weight.double(), b_b=lb.bias.double(), pooled=dd(keep["pooled"]),
             prob=dd(keep["prob"]), g_occ=dd(keep["occ"].grad), g_feat=dd(keep["feat"].grad), g_out=dd(grad))
    b = efr.proj_bounds({k: v.detach() for k, v in d.items()}, _sms())
    pairs = [("out", out_f, out_u, b["out"], 1e-4), ("grad_embed", ge_f, ge_u, b["grad_embed"], 2e-4)]
    names = {"unsup_raymarching_head.0.weight": "grad_w_occ", "unsup_raymarching_head.0.bias": "grad_b_occ",
             "lora_a.weight": "grad_w_feat", "lora_a.bias": "grad_b_feat", "lora_b.weight": "grad_w_b",
             "lora_b.bias": "grad_b_b"}
    assert set(names) == set(gp_f)
    pairs += [(names[n], gp_f[n], gp_u[n], b[names[n]], 2e-4) for n in names]
    for key, f, u, bnd, core_tol in pairs:
        f, u = f.double().reshape(bnd.shape), u.double().reshape(bnd.shape)
        tol = SAFETY * bnd + core_tol * u.abs().max()
        ratio = float(((f - u).abs() / tol).max())
        RATIOS[f"module {key}"] = ratio
        assert ratio < 1, f"module {key}: fused vs unfused error / tolerance {ratio:.3e}"
