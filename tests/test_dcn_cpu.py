"""Modulated deformable convolution (DCNv2) without a GPU: the fp64 oracle against torchvision, the mmcv-compatible
modules and registry, the argument contracts of the Python and C entry points, and the DCN backbone's structure."""
import ctypes
import hashlib

import pytest
import torch

from oracle import dcn_ref
from vidar_b200 import _lib


def _case(N, C, H, W, O, k, stride, padding, dilation, offset_std, integer=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    kh, kw = k
    Ho = (H + 2 * padding[0] - (dilation[0] * (kh - 1) + 1)) // stride[0] + 1
    Wo = (W + 2 * padding[1] - (dilation[1] * (kw - 1) + 1)) // stride[1] + 1
    x = torch.randn(N, C, H, W, generator=g, dtype=torch.float64)
    off = torch.randn(N, 2 * kh * kw, Ho, Wo, generator=g, dtype=torch.float64) * offset_std
    if integer:
        off = off.round()
    mask = torch.rand(N, kh * kw, Ho, Wo, generator=g, dtype=torch.float64)
    w = torch.randn(O, C, kh, kw, generator=g, dtype=torch.float64) / (C * kh * kw) ** 0.5
    b = torch.randn(O, generator=g, dtype=torch.float64)
    gy = torch.randn(N, O, Ho, Wo, generator=g, dtype=torch.float64)
    return x, off, mask, w, b, gy


CASES = {
    "3x3": dict(N=2, C=5, H=9, W=11, O=4, k=(3, 3), stride=(1, 1), padding=(1, 1), dilation=(1, 1), offset_std=3.0),
    "stride2": dict(N=1, C=3, H=10, W=9, O=2, k=(3, 3), stride=(2, 2), padding=(1, 1), dilation=(1, 1), offset_std=3.0),
    "pad0_dil2": dict(N=2, C=4, H=12, W=10, O=3, k=(3, 3), stride=(1, 1), padding=(0, 0), dilation=(2, 2), offset_std=3.0),
    "nonsquare": dict(N=1, C=3, H=8, W=13, O=5, k=(2, 3), stride=(2, 1), padding=(1, 0), dilation=(1, 2), offset_std=3.0),
    "small_offsets": dict(N=2, C=6, H=7, W=7, O=3, k=(3, 3), stride=(1, 1), padding=(1, 1), dilation=(1, 1), offset_std=0.7),
    "integer": dict(N=1, C=4, H=8, W=8, O=2, k=(3, 3), stride=(1, 1), padding=(1, 1), dilation=(1, 1), offset_std=2.0,
                    integer=True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_torchvision_fp64(name):
    import torchvision
    x, off, mask, w, b, gy = _case(**CASES[name])
    p = CASES[name]
    H, W = x.shape[-2:]
    # the cases reach outside the image and the (-1, 0) / (H-1, H) bands the floor cell handles specially
    kh, kw = p["k"]
    Ho, Wo = off.shape[-2:]
    hh = (torch.arange(Ho)[None, :] * p["stride"][0] - p["padding"][0] +
          torch.arange(kh).repeat_interleave(kw)[:, None] * p["dilation"][0]).double()[None, :, :, None] + off[:, 0::2]
    if p["offset_std"] > 1 and not p.get("integer"):
        assert ((hh <= -1) | (hh >= H)).any() and (((hh > -1) & (hh < 0)) | ((hh > H - 1) & (hh < H))).any()
    leaves_ref = [t.clone().requires_grad_(True) for t in (x, off, mask, w, b)]
    leaves_tv = [t.clone().requires_grad_(True) for t in (x, off, mask, w, b)]
    y_ref = dcn_ref.deform_conv2d(*leaves_ref, stride=p["stride"], padding=p["padding"], dilation=p["dilation"])
    xt, ot, mt, wt, bt = leaves_tv
    y_tv = torchvision.ops.deform_conv2d(xt, ot, wt, bt, stride=p["stride"], padding=p["padding"],
                                         dilation=p["dilation"], mask=mt)
    assert (y_ref - y_tv).abs().max().item() <= 1e-10
    y_ref.backward(gy)
    y_tv.backward(gy)
    # A sample exactly on h = -1 (w = -1) is outside the open range: its d/dh (d/dw) is 0 here, as in mmcv, while
    # torchvision takes the derivative from the right there.  Only integer offsets land on it.
    ww = (torch.arange(Wo)[None, :] * p["stride"][1] - p["padding"][1] +
          torch.arange(kw).repeat(kh)[:, None] * p["dilation"][1]).double()[None, :, None, :] + off[:, 1::2]
    edge = torch.stack([hh == -1, ww == -1], 2).view_as(off)
    assert edge.any() == bool(p.get("integer"))
    assert (leaves_ref[1].grad[edge] == 0).all()
    for what, a, t in zip(("input", "offset", "mask", "weight", "bias"), leaves_ref, leaves_tv):
        ga, gt = (a.grad, t.grad) if what != "offset" else (a.grad[~edge], t.grad[~edge])
        err = (ga - gt).abs().max().item()
        assert err <= 1e-10 * max(1.0, gt.abs().max().item()), f"{name} grad_{what}: {err:.3e}"


def test_pack_module_parameters_and_init():
    from vidar_b200.dcn import ModulatedDeformConv2d, ModulatedDeformConv2dPack
    torch.manual_seed(0)
    m = ModulatedDeformConv2dPack(16, 32, 3, stride=2, padding=1, dilation=1, bias=False)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == {"weight": (32, 16, 3, 3), "conv_offset.weight": (27, 16, 3, 3), "conv_offset.bias": (27,)}
    assert m.bias is None and m.conv_offset.stride == (2, 2) and m.conv_offset.padding == (1, 1)
    assert m.conv_offset.weight.abs().max().item() == 0 and m.conv_offset.bias.abs().max().item() == 0
    bound = 1 / (16 * 9) ** 0.5
    assert 0 < m.weight.abs().max().item() <= bound
    mb = ModulatedDeformConv2d(8, 4, (3, 2), bias=True)
    assert set(mb.state_dict()) == {"weight", "bias"} and mb.bias.abs().max().item() == 0
    assert mb.kernel_size == (3, 2) and mb.stride == (1, 1) and mb.deform_groups == 1
    # an mmcv state_dict loads, also one of the module's first version (`conv_offset_mask`)
    src = ModulatedDeformConv2dPack(16, 32, 3, padding=1, bias=True)
    sd = {k: torch.randn_like(v) for k, v in src.state_dict().items()}
    src.load_state_dict(sd)
    from collections import OrderedDict
    old = OrderedDict((k.replace("conv_offset.", "conv_offset_mask."), v) for k, v in sd.items())
    old._metadata = {"": {"version": 1}}
    dst = ModulatedDeformConv2dPack(16, 32, 3, padding=1, bias=True)
    dst.load_state_dict(old)
    assert all(torch.equal(dst.state_dict()[k], v) for k, v in sd.items())


def test_registry_builds_dcnv2_like_mmdet_resnet():
    from vidar_b200.dcn import ModulatedDeformConv2dPack
    from vidar_b200.registry import CONV_LAYERS, build_conv_layer
    assert CONV_LAYERS.get("DCNv2") is ModulatedDeformConv2dPack
    cfg = dict(type="DCNv2", deform_groups=1)
    m = build_conv_layer(cfg, 256, 256, kernel_size=3, stride=1, padding=1, dilation=1, bias=False)
    assert isinstance(m, ModulatedDeformConv2dPack) and cfg == dict(type="DCNv2", deform_groups=1)
    assert m.weight.shape == (256, 256, 3, 3) and m.bias is None and m.conv_offset.out_channels == 27
    assert type(build_conv_layer(None, 3, 8, 3)) is torch.nn.Conv2d
    with pytest.raises(KeyError):
        build_conv_layer(dict(type="DCNv9"), 3, 8, 3)


def test_unsupported_groups_and_cpu_tensors_raise():
    from vidar_b200.dcn import ModulatedDeformConv2dPack, modulated_deform_conv2d
    with pytest.raises(ValueError, match="deform_groups"):
        ModulatedDeformConv2dPack(16, 16, 3, padding=1, deform_groups=2)
    with pytest.raises(ValueError, match="groups"):
        ModulatedDeformConv2dPack(16, 16, 3, padding=1, groups=2)
    x, off, mask, w, b, _ = (t.float() for t in _case(**CASES["3x3"]))
    with pytest.raises(ValueError, match="groups"):
        modulated_deform_conv2d(x, off, mask, w, b, 1, 1, 1, 1, 2)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        modulated_deform_conv2d(x, off, mask, w, b, 1, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        ModulatedDeformConv2dPack(5, 4, 3, padding=1)(x)


def test_c_entry_points_report_bad_arguments():
    """Validated before any launch: every call returns VIDAR_E_INVALID with a message (a dummy non-null address
    stands in for device memory; nothing is touched)."""
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    geom = [2, 16, 10, 12, 10, 12, 3, 3, 1, 1, 1, 1, 1, 1]        # N C H W Ho Wo kh kw sh sw ph pw dh dw

    def g(**k):
        names = ["N", "C", "H", "W", "Ho", "Wo", "kh", "kw", "sh", "sw", "ph", "pw", "dh", "dw", "n0", "nb"]
        vals = dict(zip(names, geom + [0, 2]))
        vals.update(k)
        return [vals[n] for n in names]

    cases = [
        (L.vidar_dcn_im2col, (N, X, X, X, *g(), N), b"null pointer"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(C=0), N), b"bad sizes"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(sh=0), N), b"bad sizes"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(Ho=9), N), b"does not match the convolution"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(sh=2), N), b"does not match the convolution"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(n0=1, nb=2), N), b"bad image range"),
        (L.vidar_dcn_im2col, (X, X, X, X, *g(nb=-1), N), b"bad image range"),
        (L.vidar_dcn_col2im, (X, X, X, X, X, N, X, *g(), N), b"null pointer"),
        (L.vidar_dcn_col2im, (X, X, X, X, X, X, X, *g(dw=2), N), b"does not match the convolution"),
        (L.vidar_dcn_col2im, (X, X, X, X, X, X, X, *g(n0=3, nb=0), N), b"bad image range"),
    ]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, args, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())
    # an empty image range is a no-op
    assert L.vidar_dcn_im2col(X, X, X, X, *g(nb=0), N) == 0
    assert L.vidar_dcn_col2im(X, X, X, X, X, X, X, *g(n0=2, nb=0), N) == 0


def test_dcn_backbone_structure():
    from vidar_b200.dcn import ModulatedDeformConv2dPack
    from vidar_b200.pretrain import ImageBackbone
    plain, dcn = ImageBackbone(), ImageBackbone(dcn=True)
    found = sorted(n for n, m in dcn.named_modules() if isinstance(m, ModulatedDeformConv2dPack))
    want = sorted([f"layer3.{i}.conv2" for i in range(23)] + [f"layer4.{i}.conv2" for i in range(3)])
    assert found == want
    for name in ("layer2", "layer3", "layer4"):
        b0 = getattr(dcn, name)[0]
        assert b0.conv1.stride == (2, 2) and b0.conv2.stride == (1, 1) and b0.downsample[0].stride == (2, 2)   # caffe
        p0 = getattr(plain, name)[0]
        assert p0.conv1.stride == (1, 1) and p0.conv2.stride == (2, 2)                                         # pytorch
    for name in ("layer3", "layer4"):
        for blk in getattr(dcn, name):
            c = blk.conv2
            assert c.kernel_size == (3, 3) and c.padding == (1, 1) and c.stride == (1, 1) and c.bias is None
            assert c.in_channels == c.out_channels == blk.conv1.out_channels
    # the plain backbone keeps its parameters; the DCN one adds exactly the 26 offset convs
    extra = set(dcn.state_dict()) - set(plain.state_dict())
    assert extra == {f"{n}.conv_offset.{s}" for n in want for s in ("weight", "bias")}


# sha256 over the sorted "name shape" lines of SyntheticViDAR().state_dict() before the DCN option existed
SYNTHETIC_VIDAR_KEYS_SHA256 = "8391508c2ff19fc0205712a937d6a942258b158475ac677dfa493ff5d461d8e4"


def test_default_model_state_dict_is_unchanged():
    from vidar_b200.pretrain import SyntheticViDAR
    sd = SyntheticViDAR().state_dict()
    lines = "\n".join(f"{k} {tuple(v.shape)}" for k, v in sorted(sd.items()))
    assert hashlib.sha256(lines.encode()).hexdigest() == SYNTHETIC_VIDAR_KEYS_SHA256
