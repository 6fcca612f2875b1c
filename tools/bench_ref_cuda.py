"""Same-box GPU baseline: the REFERENCE's own CUDA ray-casters (oracle/_ref, compiled for
sm_90a by oracle/build_ref.py) next to this repo's kernels on BASELINE configs[2]
(sigma [1,3,16,200,200], 30000 rays), plus a direct output comparison.  Run on a GPU box:
    python tools/bench_ref_cuda.py > gpurun_out/ref_cuda.json
The reference synchronises the device inside every call; timings are wall-clock around
calls bracketed by torch.cuda.synchronize (median of 20 after 5 warm-ups)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402
from tests.inputs import dvr_inputs_lidar  # noqa: E402
from tools.gpu_timing import card, host_ms  # noqa: E402
from vidar_b200 import render  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    sigma, origin, points, tindex = dvr_inputs_lidar(M=30000, T=3, seed=0)
    s, o, p, t = (torch.from_numpy(x).to(dev) for x in (sigma, origin, points, tindex))
    grid = [3, 16, 200, 200]
    rd, rx, rx2 = build_ref.load("ref_dvr"), build_ref.load("ref_dvxlr"), build_ref.load("ref_dvxlr_v2")
    gp = torch.randn(1, 30000, device=dev)
    out = {"config": "sigma[1,3,16,200,200], 30000 rays, 3 frames", "gpu": card(), "ms": {}}

    def ref_dvxlr_fb():
        pred, gt, dd, idx = rx.render(s, o, p, t)
        em = gp[..., None] * dd
        return rx.get_grad_sigma(em, idx, t, s)[0]

    def our_dvxlr_fb():
        sg = s.detach().requires_grad_(True)
        pred, gt = render.DifferentiableVoxelRendering(sg, o, p, t)
        pred.backward(gp)
        return sg.grad

    cases = {
        "dvr.render_forward": (lambda: rd.render_forward(s, o, p, t, grid, "train"),
                               lambda: render.dvr.render_forward(s, o, p, t, grid, "train")),
        "dvr.render(l2)": (lambda: rd.render(s, o, p, t, "l2"), lambda: render.dvr.render(s, o, p, t, "l2")),
        "dvxlr.render(lists)": (lambda: rx.render(s, o, p, t), lambda: render.dvxlr.render(s, o, p, t)),
        "dvxlr fwd+bwd (autograd layer)": (ref_dvxlr_fb, our_dvxlr_fb),
    }
    for name, (ref, ours) in cases.items():
        out["ms"][name] = {"reference_cuda": host_ms(ref, 20, 5), "vidar_b200": host_ms(ours, 20, 5)}
        out["ms"][name]["speedup"] = out["ms"][name]["reference_cuda"] / out["ms"][name]["vidar_b200"]

    # direct comparison of outputs, full size
    a = rd.render_forward(s, o, p, t, grid, "train")
    b = render.dvr.render_forward(s, o, p, t, grid, "train")
    cmp = {"render_forward_pred_maxrel": float(((a[0] - b[0]).abs() / a[0].abs().clamp_min(1e-6)).max())}
    a = rx.render(s, o, p, t)
    b = render.dvxlr.render(s, o, p, t)
    cmp["dvxlr_pred_maxrel"] = float(((a[0] - b[0]).abs() / a[0].abs().clamp_min(1e-6)).max())
    cmp["dvxlr_indices_equal"] = bool(torch.equal(a[3], b[3]))
    cmp["dvxlr_dd_maxabs"] = float((a[2] - b[2]).abs().max())
    cmp["dvxlr_dd_scale"] = float(a[2].abs().max())
    ga, gb = ref_dvxlr_fb(), our_dvxlr_fb()
    cmp["dvxlr_grad_sigma_maxabs"] = float((ga - gb).abs().max())
    cmp["dvxlr_grad_sigma_scale"] = float(ga.abs().max())
    out["compare_full_size"] = cmp
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
