"""Write tests/golden/dcnv3.npz from the reference's OWN pure-torch DCNv3 (`dcnv3_core_pytorch` of
ops_dcnv3/functions/dcnv3_func.py) and its module classes (ops_dcnv3/modules/dcnv3.py), loaded from the reference
checkout through tools/ref_shim.py with a stub `DCNv3` extension module in sys.modules (the compiled extension is
neither needed nor built here).  Test infrastructure: nothing of the reference is copied, only its outputs.

Contents (all fp64 unless noted):
  core/<case>/{input,offset,mask,output} and core/<case>/args [kh, kw, sh, sw, ph, pw, dh, dw, group, group_channels,
  offset_scale * 1000] for seeded cases covering stride 2, dilation 2, offset_scale != 1 and samples off the image;
  state/keys, state/shapes: the DCNv3 module's state_dict (center_feature_scale=True) as names and shapes padded with -1 to 4 dims;
  module/x, module/out, module/param/<name>: DCNv3_pytorch (same parameters as DCNv3) on seeded non-zero
  parameters, the reference module's forward in fp64.
The reference core pads W by pad_h and H by pad_w, so its cases use pad_h == pad_w (as the module always does).

    python tools/make_golden_dcnv3.py
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ref_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dcnv3.npz")
# (name, N, H, W, kernel, stride, pad, dilation, group, group_channels, offset_scale, offset spread)
CASES = [
    ("k3", 2, 9, 11, 3, 1, 1, 1, 2, 8, 1.0, 2.0),
    ("k3_s2_d2", 2, 12, 10, 3, 2, 2, 2, 2, 4, 0.5, 2.5),
    ("k5_far", 1, 8, 9, 5, 1, 2, 1, 3, 4, 1.5, 4.0),
    ("k3_p0_s2", 3, 7, 8, 3, 2, 0, 1, 1, 5, 2.0, 1.5),
]


def load_reference():
    ref_shim.install()
    sys.modules.setdefault("DCNv3", types.ModuleType("DCNv3"))        # the compiled extension: never called here
    for sub in ("backbones", "backbones.ops_dcnv3"):
        m = types.ModuleType(f"vidar_ref.{sub}")
        m.__path__ = [os.path.join(ref_shim.REF_BEVFORMER, *sub.split("."))]
        sys.modules[f"vidar_ref.{sub}"] = m
    func = importlib.import_module("vidar_ref.backbones.ops_dcnv3.functions.dcnv3_func")
    mods = importlib.import_module("vidar_ref.backbones.ops_dcnv3.modules.dcnv3")
    return func, mods


def main():
    func, mods = load_reference()
    g = torch.Generator().manual_seed(2024)
    out = {}
    for name, N, H, W, k, s, p, d, G, Cg, scale, spread in CASES:
        Ho = (H + 2 * p - (d * (k - 1) + 1)) // s + 1
        Wo = (W + 2 * p - (d * (k - 1) + 1)) // s + 1
        K = k * k
        x = torch.randn(N, H, W, G * Cg, generator=g, dtype=torch.float64)
        off = torch.randn(N, Ho, Wo, G * K * 2, generator=g, dtype=torch.float64) * spread
        mask = torch.softmax(torch.randn(N, Ho, Wo, G, K, generator=g, dtype=torch.float64), -1).reshape(N, Ho, Wo, -1)
        y = func.dcnv3_core_pytorch(x, off, mask, k, k, s, s, p, p, d, d, G, Cg, scale)
        for key, t in (("input", x), ("offset", off), ("mask", mask), ("output", y)):
            out[f"core/{name}/{key}"] = t.numpy()
        out[f"core/{name}/args"] = np.array([k, k, s, s, p, p, d, d, G, Cg, round(scale * 1000)], np.int64)

    ref = mods.DCNv3(channels=32, kernel_size=3, group=2, offset_scale=1.0, center_feature_scale=True)
    sd = ref.state_dict()
    out["state/keys"] = np.array(list(sd))
    out["state/shapes"] = np.array([list(v.shape) + [-1] * (4 - v.dim()) for v in sd.values()], np.int64)

    torch.manual_seed(7)
    mod = mods.DCNv3_pytorch(channels=32, kernel_size=3, group=2, offset_scale=1.0, center_feature_scale=True).double()
    with torch.no_grad():
        for n, prm in mod.named_parameters():
            prm.copy_(torch.randn(prm.shape, generator=g, dtype=torch.float64) * (0.5 if "offset" in n else 0.2))
    mod.eval()
    x = torch.randn(2, 10, 12, 32, generator=g, dtype=torch.float64)
    with torch.no_grad():
        y = mod(x)
    out["module/x"] = x.numpy()
    out["module/out"] = y.numpy()
    for n, prm in mod.state_dict().items():
        out[f"module/param/{n}"] = prm.numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays")


if __name__ == "__main__":
    main()
