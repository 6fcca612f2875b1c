"""DCNv3 without a GPU: the fp64 oracle (oracle/dcnv3_ref.py) against the MSDA oracle and the reference's own
pure-torch op (tests/golden/dcnv3.npz), the module's parameters and forward against the reference module, every
argument check of vidar_b200.dcnv3, and the signatures of its `ext` stand-in."""
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import dcnv3_ref, msda_ref
from vidar_b200 import dcnv3

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dcnv3.npz")
CORE_CASES = ("k3", "k3_s2_d2", "k5_far", "k3_p0_s2")


def _golden():
    return np.load(GOLDEN)


def _args(a):
    """The golden's int args -> (kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale)."""
    return tuple(int(v) for v in a[:10]) + (a[10] / 1000.0,)


def _inputs(N, H, W, G, Cg, k, s, p, d, spread, seed, dtype=torch.float64):
    kh, kw = k
    Ho, Wo = dcnv3_ref.output_size(H, W, kh, kw, s[0], s[1], p[0], p[1], d[0], d[1])
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, G * Cg, generator=g, dtype=dtype)
    off = torch.randn(N, Ho, Wo, G * kh * kw * 2, generator=g, dtype=dtype) * spread
    mask = torch.rand(N, Ho, Wo, G * kh * kw, generator=g, dtype=dtype)
    gy = torch.randn(N, Ho, Wo, G * Cg, generator=g, dtype=dtype)
    return x, off, mask, gy


@pytest.mark.parametrize("name", CORE_CASES)
def test_oracle_matches_the_reference_pytorch_core(name):
    """The reference core builds its base grid in fp32 (torch.linspace(..., dtype=torch.float32) / W), so its sample
    positions carry fp32 rounding (~1e-7 px): agreement to 1e-5, where a wrong point order, centre or boundary rule
    is off by O(1)."""
    z = _golden()
    args = _args(z[f"core/{name}/args"])
    x, off, m = (torch.from_numpy(z[f"core/{name}/{k}"]) for k in ("input", "offset", "mask"))
    y = dcnv3_ref.dcnv3(x, off, m, *args)
    ref = torch.from_numpy(z[f"core/{name}/output"])
    assert (y - ref).abs().max().item() <= 1e-5 * (1 + ref.abs().max().item())


def test_golden_cases_sample_off_the_image():
    z = _golden()
    off_image = 0
    for name in CORE_CASES:
        kh, kw, sh, sw, ph, pw, dh, dw, G, Cg, s = _args(z[f"core/{name}/args"])
        x = torch.from_numpy(z[f"core/{name}/input"])
        px, py = dcnv3_ref.sample_points(torch.from_numpy(z[f"core/{name}/offset"]), x.shape[1], x.shape[2], kh, kw,
                                         sh, sw, ph, pw, dh, dw, G, s)
        off_image += int(((px <= -1) | (py <= -1) | (px >= x.shape[2]) | (py >= x.shape[1])).sum())
    assert off_image > 100


@pytest.mark.parametrize("k,s,p,d,scale", [((3, 3), (1, 1), (1, 1), (1, 1), 1.0), ((3, 5), (2, 1), (0, 2), (2, 1), 0.5),
                                           ((5, 5), (1, 2), (2, 2), (1, 1), 1.5)])
def test_oracle_equals_one_level_msda_on_the_padded_input(k, s, p, d, scale):
    x, off, mask, gy = _inputs(2, 7, 9, 2, 3, k, s, p, d, 2.0, seed=11)
    args = (*k, *s, *p, *d, 2, 3, scale)
    out, gx, go, gm = dcnv3_ref.dcnv3_backward(x, off, mask, *args, gy)
    leaves = [t.clone().requires_grad_(True) for t in (x, off, mask)]
    value, shapes, loc, attn = dcnv3_ref.as_msda(*leaves, *args)
    y = msda_ref.msda_grid_sample(value, shapes, loc, attn).reshape(out.shape)
    y.backward(gy)
    assert (y - out).abs().max().item() <= 1e-12
    assert (leaves[0].grad - gx).abs().max().item() <= 1e-12
    assert (leaves[2].grad - gm).abs().max().item() <= 1e-12
    px, py = dcnv3_ref.sample_points(off, 7, 9, *args[:8], 2, scale)
    keep = torch.stack([px != -1, py != -1], -1).all(-1, keepdim=True).expand(*px.shape, 2).reshape(go.shape)
    assert (leaves[1].grad - go)[keep].abs().max().item() <= 1e-12


def test_a_sample_exactly_on_minus_one_gets_zero_gradients_where_msda_does_not():
    """One point at x = -1 (y inside): DCNv3 drops it; MSDA on the padded input interpolates toward pixel 0."""
    x, off, mask, gy = _inputs(1, 4, 5, 1, 2, (1, 1), (1, 1), (0, 0), (1, 1), 0.0, seed=3)
    off[0, 1, 0, 0] = -1.0          # pixel (ho=1, wo=0): x = 0 - 1 = -1
    off[0, 2, 3, 1] = 2.0           # pixel (ho=2, wo=3): y = 4 = H, on the far edge
    args = (1, 1, 1, 1, 0, 0, 1, 1, 1, 2, 1.0)
    out, gx, go, gm = dcnv3_ref.dcnv3_backward(x, off, mask, *args, gy)
    assert out[0, 1, 0].abs().max() == 0 and out[0, 2, 3].abs().max() == 0
    assert go[0, 1, 0].abs().max() == 0 and gm[0, 1, 0].abs().max() == 0
    assert go[0, 2, 3].abs().max() == 0 and gm[0, 2, 3].abs().max() == 0
    leaves = [t.clone().requires_grad_(True) for t in (x, off, mask)]
    value, shapes, loc, attn = dcnv3_ref.as_msda(*leaves, *args)
    msda_ref.msda_grid_sample(value, shapes, loc, attn).reshape(out.shape).backward(gy)
    assert leaves[1].grad[0, 1, 0, 0].abs().item() > 0


def test_state_dict_matches_the_reference_module():
    z = _golden()
    m = dcnv3.DCNv3(channels=32, kernel_size=3, group=2, offset_scale=1.0, center_feature_scale=True)
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in z["state/keys"]]
    for (k, v), shape in zip(sd.items(), z["state/shapes"]):
        assert list(v.shape) == [int(s) for s in shape if s >= 0], k
    plain = dcnv3.DCNv3(channels=32, group=2)
    assert set(sd) - set(plain.state_dict()) == {"center_feature_scale_proj_weight", "center_feature_scale_proj_bias"}


class _OracleFunction:
    """DCNv3Function with the fp64 oracle as the core, so the module's own code runs on the CPU."""

    @staticmethod
    def apply(x, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale, im2col_step):
        return dcnv3_ref.dcnv3(x, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels, offset_scale)


def test_module_forward_matches_the_reference_module(monkeypatch):
    z = _golden()
    monkeypatch.setattr(dcnv3, "DCNv3Function", _OracleFunction)
    m = dcnv3.DCNv3(channels=32, kernel_size=3, group=2, offset_scale=1.0, center_feature_scale=True).double()
    params = {k[len("module/param/"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("module/param/")}
    m.load_state_dict(params)
    with torch.no_grad():
        y = m(torch.from_numpy(z["module/x"]))
    ref = torch.from_numpy(z["module/out"])
    assert (y - ref).abs().max().item() <= 1e-5 * (1 + ref.abs().max().item())      # the fp32 grid, as above


def test_module_constructor_checks():
    with pytest.raises(ValueError, match="divisible"):
        dcnv3.DCNv3(channels=30, group=4)
    with pytest.warns(UserWarning, match="power of 2"):
        dcnv3.DCNv3(channels=24, group=2)
    with pytest.raises(NotImplementedError):
        dcnv3.DCNv3(channels=16, group=2, norm_layer="GN")
    m = dcnv3.DCNv3(channels=16, group=2, norm_layer="BN", act_layer="ReLU")
    assert isinstance(m.dw_conv[1][0], torch.nn.BatchNorm2d)


ARGS = (3, 3, 1, 1, 1, 1, 1, 1, 2, 4, 1.0)


def _valid(N=2, H=5, W=6, dtype=torch.float32):
    x = torch.zeros(N, H, W, 8, dtype=dtype)
    off = torch.zeros(N, H, W, 2 * 9 * 2, dtype=dtype)
    mask = torch.zeros(N, H, W, 2 * 9, dtype=dtype)
    gy = torch.zeros(N, H, W, 8, dtype=dtype)
    return x, off, mask, gy


@pytest.mark.parametrize("fn", ["forward", "backward"])
def test_argument_checks_run_before_any_cuda_call(fn):
    def call(x, off, mask, gy, args=ARGS, step=256):
        if fn == "forward":
            return dcnv3.ext.dcnv3_forward(x, off, mask, *args, step)
        return dcnv3.ext.dcnv3_backward(x, off, mask, *args, gy, step)

    x, off, mask, gy = _valid()
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        call(x, off, mask, gy)
    for bad in (torch.float64, torch.int32):
        with pytest.raises(TypeError, match="float32, float16 or bfloat16"):
            call(x.to(bad), off.to(bad), mask.to(bad), gy.to(bad))
    with pytest.raises(TypeError, match="share one dtype"):
        call(x, off.half(), mask, gy)
    with pytest.raises(TypeError, match="share one dtype"):
        call(x.bfloat16(), off.bfloat16(), mask.half(), gy.bfloat16())
    with pytest.raises(RuntimeError, match="group times group channels"):
        call(x, off, mask, gy, args=ARGS[:8] + (2, 3, 1.0))
    with pytest.raises(RuntimeError, match="offset must be"):
        call(x, off[..., :-2].contiguous(), mask, gy)
    with pytest.raises(RuntimeError, match="mask must be"):
        call(x, off, mask[:, :4].contiguous(), gy)
    with pytest.raises(RuntimeError, match="4-D"):
        call(x[0], off, mask, gy)
    with pytest.raises(RuntimeError, match="contiguous"):
        call(x, off.transpose(1, 2).contiguous().transpose(1, 2), mask, gy)
    with pytest.raises(RuntimeError, match="must divide im2col_step"):
        x3, o3, m3, g3 = _valid(N=3)
        call(x3, o3, m3, g3, step=2)
    with pytest.raises(RuntimeError, match="must divide im2col_step"):
        call(x, off, mask, gy, step=0)
    with pytest.raises(RuntimeError, match="positive"):
        call(x, off, mask, gy, args=(3, 3, 0, 1) + ARGS[4:])
    with pytest.raises(RuntimeError, match="empty"):
        call(x, off, mask, gy, args=(9, 9, 1, 1, 0, 0, 1, 1, 2, 4, 1.0))
    # N = 3 with the module's im2col_step = 256 is valid: the step is clamped to the batch
    x3, o3, m3, g3 = _valid(N=3)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        call(x3, o3, m3, g3, step=256)
    if fn == "backward":
        with pytest.raises(RuntimeError, match="grad_output must be"):
            call(x, off, mask, gy[:, :, :, :4].contiguous())
        with pytest.raises(TypeError, match="share one dtype"):
            call(x, off, mask, gy.half())


def test_dtype_codes_match_the_header():
    import re

    from vidar_b200 import _lib
    with open(_lib.HEADER) as fh:
        src = fh.read()
    codes = dict(re.findall(r"#define VIDAR_DTYPE_(\w+) (\d+)", src) + re.findall(r"VIDAR_DTYPE_(F32) = (\d+)", src))
    assert {k: int(v) for k, v in codes.items()} == {"F32": dcnv3.DTYPE_CODES[torch.float32],
                                                     "F16": dcnv3.DTYPE_CODES[torch.float16],
                                                     "BF16": dcnv3.DTYPE_CODES[torch.bfloat16]}


def test_ext_has_the_compiled_modules_signatures():
    fwd = list(inspect.signature(dcnv3.ext.dcnv3_forward).parameters)
    bwd = list(inspect.signature(dcnv3.ext.dcnv3_backward).parameters)
    geom = ["kernel_h", "kernel_w", "stride_h", "stride_w", "pad_h", "pad_w", "dilation_h", "dilation_w", "group",
            "group_channels", "offset_scale"]
    assert fwd == ["input", "offset", "mask", *geom, "im2col_step"]
    assert bwd == ["input", "offset", "mask", *geom, "grad_output", "im2col_step"]
    assert len(inspect.signature(dcnv3.DCNv3Function.forward).parameters) == 16        # ctx + 15
