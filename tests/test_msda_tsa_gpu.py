"""vidar_msda_tsa_* (msda.MSDeformAttnQueueFusedFunction): TemporalSelfAttention's and the future decoder's sampling
with the softmax, the sampling-location arithmetic and the queue mean inside the kernel.

The op is checked against an fp64 statement of the modules' own arithmetic (softmax of the logits, offsets / (W, H)
+ reference points, oracle/msda_ref.py's grid_sample MSDA, mean over the queue), with the gradients of value,
offsets and logits by autograd through it, at the tolerances of tests/parity.py.  The sampling locations keep the
value of the fp32 statement, as in the other MSDA oracle tests: fp32 input quantisation moves a point by up to
~1e-5 px at 200 x 200, which is the size of the tolerance's floor.  grad_offsets inherits
grad_sampling_loc's discontinuity on pixel-centre lines: samples within 1e-4 px of one are excluded, as in
tests/test_msda_gpu.py.  Then each module's fused path against its `fuse_epilogue = False` path with the same
weights, the row-sharded TSA, the path selection and the absence of host syncs."""
import numpy as np
import pytest
import torch

from oracle import msda_ref
from tests import module_cases as mc
from tests import parity
from tests.inputs import level_tensors
import vidar_b200.modules  # noqa: F401  (registers the classes)
from vidar_b200 import msda
from vidar_b200.modules import deform_attn
from vidar_b200.registry import build_attention

pytestmark = pytest.mark.gpu
Fn = msda.MSDeformAttnQueueFusedFunction
BEV = ((200, 200),)


def _inputs(B, G, Q, H, C, levels, P, seed, off_scale=3.0, logit_scale=2.0, ref_lo=-0.1, ref_hi=1.1, device="cuda"):
    L = len(levels)
    shapes, lsi = level_tensors(levels)
    K = int((shapes[:, 0] * shapes[:, 1]).sum())
    g = torch.Generator().manual_seed(seed)
    d = dict(value=torch.randn(B * G, K, H, C, generator=g),
             ref=torch.rand(B * G, Q, L, 2, generator=g) * (ref_hi - ref_lo) + ref_lo,
             offsets=off_scale * torch.randn(B, Q, H, G, L, P, 2, generator=g),
             logits=logit_scale * torch.randn(B, Q, H, G, L * P, generator=g),
             grad=torch.randn(B, Q, H * C, generator=g), shapes=shapes, lsi=lsi)
    return {k: v.to(device) for k, v in d.items()}


def _oracle(d):
    """out [B, Q, H*C], the sampling locations [B*G, Q, H, L, P, 2], and the gradients of value, offsets and logits
    by autograd, all in fp64.  The locations take the value of the modules' fp32 statement, which the kernel
    reproduces bit for bit (as msda_ref.sca_locations does for SpatialCrossAttention), so both sample the same
    points; their derivative with respect to the offsets is 1 / (W_l, H_l)."""
    v, off, lg = (d[k].double().requires_grad_(True) for k in ("value", "offsets", "logits"))
    B, Q, H, G, L, P, _ = off.shape
    shapes = d["shapes"]
    wh = torch.stack([shapes[:, 1], shapes[:, 0]], -1)[None, None, None, :, None, :]
    w = lg.softmax(-1).permute(0, 3, 1, 2, 4).reshape(B * G, Q, H, L, P)
    o = off.permute(0, 3, 1, 2, 4, 5, 6).reshape(B * G, Q, H, L, P, 2)
    loc32 = d["ref"][:, :, None, :, None, :] + o.detach().float() / wh.float()
    loc = loc32.double() + (o - o.detach()) / wh.double()
    out = msda_ref.msda_grid_sample(v, shapes, loc, w).view(B, G, Q, -1).mean(1)
    out.backward(d["grad"].double())
    return out.detach(), loc.detach(), v.grad, off.grad, lg.grad


def _shifted(t):
    """t's values in a view whose data pointer is 4 bytes past a 16-byte boundary (differentiable)."""
    buf = torch.zeros(t.numel() + 1, device=t.device, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16
    return v


def _run(d, shift=()):
    v, off, lg = (t.clone().requires_grad_(True) for t in (d["value"], d["offsets"], d["logits"]))
    x = dict(value=v, offsets=off, logits=lg, ref=d["ref"])
    x = {k: _shifted(t) if k in shift else t for k, t in x.items()}
    out = Fn.apply(x["value"], d["shapes"], d["lsi"], x["ref"], x["offsets"], x["logits"])
    out.backward(d["grad"])
    torch.cuda.synchronize()
    return out.detach(), v.grad, off.grad, lg.grad


def _check(d, res):
    out, gv, goff, glg = res
    rout, rloc, rgv, rgoff, rglg = _oracle(d)
    parity.close(out, rout, "output")
    parity.close(gv, rgv, "grad_value")
    parity.close(glg, rglg, "grad_logits")
    B, Q, H, G, L, P, _ = d["offsets"].shape
    keep = parity.off_kink(rloc, d["shapes"]).view(B, G, Q, H, L, P).permute(0, 2, 3, 1, 4, 5)
    assert keep.float().mean() > 0.995
    parity.close(goff, rgoff, "grad_offsets", keep=keep[..., None].expand(-1, -1, -1, -1, -1, -1, 2).cpu())


CASES = [
    # B, G, Q, H, C, levels, P
    pytest.param(1, 2, 40000, 8, 32, BEV, 4, id="tsa-bs1"),                          # TemporalSelfAttention
    pytest.param(2, 2, 40000, 8, 32, BEV, 4, id="tsa-bs2"),
    pytest.param(1, 1, 40000, 8, 32, BEV, 4, id="decoder-self"),                     # future decoder, L*P = 4
    pytest.param(1, 1, 40000, 8, 32, BEV * 2, 4, id="decoder-cross"),                # two history frames, L*P = 8
    pytest.param(2, 1, 900, 8, 32, BEV, 4, id="detection-decoder"),
    pytest.param(1, 2, 3000, 16, 16, ((50, 60),), 4, id="C16"),                      # G*L*P = 8 at 8 lanes per group
    pytest.param(1, 1, 3000, 16, 16, ((50, 60),), 4, id="C16-single"),               # L*P = 4 < 8 groups: one per warp
    pytest.param(1, 2, 3000, 4, 64, ((50, 60),), 4, id="C64"),
    pytest.param(1, 2, 37, 1, 32, ((20, 30),), 4, id="partial-warp"),                # 37 items, 4 per warp
    pytest.param(3, 1, 37, 2, 32, ((20, 30),), 4, id="partial-warp-lp4"),
    pytest.param(1, 3, 301, 8, 32, ((20, 30),), 4, id="G3"),                         # G*L*P = 12: one item per warp
    pytest.param(1, 1, 301, 8, 32, ((20, 30), (10, 15), (5, 8), (3, 4)), 8, id="LP32"),
    pytest.param(2, 2, 301, 8, 32, ((20, 30),), 1, id="LP1"),
    pytest.param(1, 2, 301, 8, 32, ((20, 30), (10, 15)), 8, id="LP16"),
]


@pytest.mark.parametrize("B,G,Q,H,C,levels,P", CASES)
def test_op_matches_fp64_oracle(cuda, B, G, Q, H, C, levels, P):
    d = _inputs(B, G, Q, H, C, levels, P, seed=B * 7 + G * 131 + Q + C)
    _check(d, _run(d))


def test_samples_outside_the_map(cuda):
    """Offsets of ten pixels and more and reference points well outside [0, 1]: many samples have some or all of their
    corners outside the image."""
    d = _inputs(2, 2, 500, 8, 32, ((20, 30),), 4, seed=3, off_scale=12.0, ref_lo=-0.5, ref_hi=1.5)
    B, Q, H, G, L, P, _ = d["offsets"].shape
    _, loc, _, _, _ = _oracle(d)
    px = loc * torch.tensor([30.0, 20.0], dtype=torch.float64, device=loc.device) - 0.5
    outside = ((px <= -1) | (px >= torch.tensor([30.0, 20.0], dtype=torch.float64, device=loc.device))).any(-1)
    assert 0.2 < outside.double().mean().item() < 0.9
    _check(d, _run(d))


def test_saturated_logits(cuda):
    d = _inputs(1, 2, 500, 8, 32, ((20, 30),), 4, seed=4)
    sign = torch.where(torch.rand(d["logits"].shape, device=cuda) < 0.5, -1.0, 1.0)
    d["logits"] = 80.0 * sign
    d["logits"][0, :10] = 80.0                  # ties at the maximum
    d["logits"][0, 10:20] = -80.0
    res = _run(d)
    assert all(torch.isfinite(t).all() for t in res)
    _check(d, res)


def test_misaligned_views(cuda):
    """Views whose storage offsets are not 16-byte aligned are copied, not read misaligned."""
    d = _inputs(1, 2, 301, 8, 32, ((20, 30),), 4, seed=5)
    _check(d, _run(d, shift=("value", "offsets", "logits", "ref")))


def test_argument_errors(cuda):
    d = _inputs(1, 2, 10, 8, 32, ((4, 5),), 4, seed=6)
    with pytest.raises(RuntimeError, match="bs \\* num_queue"):
        Fn.apply(d["value"][:1], d["shapes"], d["lsi"], d["ref"], d["offsets"], d["logits"])
    with pytest.raises(RuntimeError, match="reference_points"):
        Fn.apply(d["value"], d["shapes"], d["lsi"], d["ref"][:, :, :, :1], d["offsets"], d["logits"])
    big = _inputs(1, 2, 10, 8, 32, ((4, 5),), 16, seed=6)           # G*L*P = 32 is the limit ...
    Fn.apply(big["value"], big["shapes"], big["lsi"], big["ref"], big["offsets"], big["logits"])
    over = _inputs(1, 3, 10, 8, 32, ((4, 5),), 16, seed=6)          # ... 48 is over it
    with pytest.raises(RuntimeError, match="at most 32"):
        Fn.apply(over["value"], over["shapes"], over["lsi"], over["ref"], over["offsets"], over["logits"])
    assert Fn.supported(1, 4, 2, 32) and Fn.supported(2, 4, 1, 64) and Fn.supported(4, 8, 1, 16)
    assert not Fn.supported(1, 3, 1, 32) and not Fn.supported(2, 8, 4, 32) and not Fn.supported(1, 4, 2, 24)


# ---- modules: fused against fuse_epilogue = False ------------------------------------------------------------------

def _module(cfg, seed, cuda):
    m = build_attention(cfg)
    m.load_state_dict(mc.seeded_state(m, seed))
    return m.eval().to(cuda)


def _both_paths(m, run):
    res = []
    for fused in (True, False):
        m.fuse_epilogue = fused
        m.zero_grad(set_to_none=True)
        res.append(list(run()) + [p.grad.clone() for _, p in sorted(m.named_parameters())])
    m.fuse_epilogue = True
    return res


def _assert_equal_paths(m, res, names):
    names = list(names) + [n for n, _ in sorted(m.named_parameters())]
    assert len(names) == len(res[0])
    for a, b, w in zip(res[0], res[1], names):
        err = (a - b).abs().max().item()
        assert err <= 2e-5 * b.abs().max().item() + 1e-7, f"{w}: {err:.3e} vs {b.abs().max().item():.3e}"


def _spy(monkeypatch):
    calls = []
    real = deform_attn.msda_queue_fused_apply
    monkeypatch.setattr(deform_attn, "msda_queue_fused_apply", lambda *a: calls.append(1) or real(*a))
    return calls


@pytest.mark.parametrize("prev_bev", [True, False])
def test_tsa_fused_equals_reference_statements(cuda, prev_bev, monkeypatch):
    m = _module(mc.TSA_CFG, 11, cuda)
    c = {k: v.to(cuda) for k, v in mc.tsa_case(bs=2).items()}
    calls = _spy(monkeypatch)

    def run():
        q = c["query"].clone().requires_grad_(True)
        if prev_bev:
            kv = c["value"].clone().requires_grad_(True)
            out = m(q, None, kv, query_pos=c["query_pos"], reference_points=c["reference_points"],
                    spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
            out.backward(c["grad"])
            return out.detach(), q.grad, kv.grad
        out = m(q, None, None, query_pos=c["query_pos"], reference_points=c["reference_points"],
                spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
        out.backward(c["grad"])
        return out.detach(), q.grad

    res = _both_paths(m, run)
    assert len(calls) == 1
    _assert_equal_paths(m, res, ["out", "grad query", "grad value"][:3 if prev_bev else 2])


@pytest.mark.parametrize("frames", [1, 2])
def test_prediction_attention_fused_equals_reference_statements(cuda, frames, monkeypatch):
    cfg = dict(mc.PRED_CFG, num_levels=frames)
    m = _module(cfg, 12, cuda)
    c = {k: v.to(cuda) for k, v in mc.pred_case(bs=2, frames=frames).items()}
    calls = _spy(monkeypatch)
    res = _both_paths(m, lambda: mc.run_module(m, "pred", c, device=cuda))
    assert len(calls) == 1
    _assert_equal_paths(m, res, ["out", "grad query", "grad value"])


def test_custom_attention_fused_equals_reference_statements(cuda, monkeypatch):
    m = _module(mc.CUSTOM_CFG, 13, cuda)
    c = {k: v.to(cuda) for k, v in mc.custom_case(bs=2, nq=900).items()}
    calls = _spy(monkeypatch)
    res = _both_paths(m, lambda: mc.run_module(m, "custom", c, device=cuda))
    assert len(calls) == 1
    _assert_equal_paths(m, res, ["out", "grad query", "grad value"])


def test_row_sharded_tsa_equals_rows_of_the_full_call(cuda, monkeypatch):
    m = _module(mc.TSA_CFG, 11, cuda)
    c = {k: v.to(cuda) for k, v in mc.tsa_case(bs=1).items()}
    calls = _spy(monkeypatch)
    kw = dict(spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
    full = m(c["query"], None, c["value"], query_pos=c["query_pos"], reference_points=c["reference_points"], **kw)
    for lo, hi in ((0, 37), (37, 100), (50, 51)):
        rows = m(c["query"][:, lo:hi], None, c["value"], query_pos=c["query_pos"][:, lo:hi],
                 reference_points=c["reference_points"][:, lo:hi], row_range=(lo, hi), **kw)
        torch.testing.assert_close(rows, full[:, lo:hi], rtol=1e-6, atol=1e-6)
    assert len(calls) == 4


def test_path_selection(cuda, monkeypatch):
    """The fused op runs for fp32 CUDA tensors with 2-D reference points at a supported shape; autocast, 4-D box
    reference points, an unsupported L*P and fuse_epilogue = False take the reference's statements."""
    calls = _spy(monkeypatch)
    tsa = _module(mc.TSA_CFG, 11, cuda)
    c = {k: v.to(cuda) for k, v in mc.tsa_case().items()}
    kw = dict(spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
    tsa(c["query"], None, c["value"], reference_points=c["reference_points"], **kw)
    assert len(calls) == 1
    with torch.autocast("cuda", dtype=torch.float16):
        tsa(c["query"], None, c["value"], reference_points=c["reference_points"], **kw)
    boxes = torch.cat([c["reference_points"], 0.2 * torch.ones_like(c["reference_points"])], -1)
    tsa(c["query"], None, c["value"], reference_points=boxes, **kw)
    tsa.fuse_epilogue = False
    tsa(c["query"], None, c["value"], reference_points=c["reference_points"], **kw)
    assert len(calls) == 1
    odd = _module(dict(mc.TSA_CFG, num_points=3), 11, cuda)           # L*P = 3
    odd(c["query"], None, c["value"], reference_points=c["reference_points"], **kw)
    assert len(calls) == 1
    custom = _module(mc.CUSTOM_CFG, 14, cuda)
    for boxes, n in ((True, 1), (False, 2)):
        cc = {k: v.to(cuda) for k, v in mc.custom_case(boxes=boxes).items()}
        mc.run_module(custom, "custom", cc, device=cuda)
        assert len(calls) == n


@pytest.mark.parametrize("kind", ["tsa", "pred"])
def test_default_path_has_no_host_sync(cuda, kind):
    cfg, case = {"tsa": (mc.TSA_CFG, mc.tsa_case), "pred": (mc.PRED_CFG, mc.pred_case)}[kind]
    m = _module(cfg, 11, cuda)
    c = {k: v.to(cuda) for k, v in case().items()}
    q = c["query"].clone().requires_grad_(True)
    kv = c["value"].clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m(q, None, kv, query_pos=c["query_pos"], reference_points=c["reference_points"],
                spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
        out.backward(c["grad"])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(q.grad).all() and torch.isfinite(kv.grad).all()
    assert np.isfinite(float(out.sum()))
