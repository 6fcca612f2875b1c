"""BASELINE.json configs[1], [2] and the configs[4] sweep on ONE H100: per-op time, units/s and
algorithmic GB/s (SURVEY.md 8d byte counts) -> JSON on stdout.  Test infrastructure."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tests.inputs import dvr_inputs_lidar  # noqa: E402
from tools.gpu_timing import card, window_ms  # noqa: E402
from vidar_b200 import msda, ray_head, render  # noqa: E402
from vidar_b200.modules.latent_rendering import latent_render_core  # noqa: E402

dev = torch.device("cuda:0")
PEAK = bench.peaks()[0]


def row(ms, units, bytes_):
    return {"ms": ms, "units_per_s": units / (ms * 1e-3), "GBps": bytes_ / (ms * 1e-3) / 1e9,
            "pct_of_hbm_peak": 100 * bytes_ / (ms * 1e-3) / 1e9 / PEAK}


def msda_sca(Q):
    d = bench.sca_like_inputs(dev, cams=6, Q=Q)
    gv = torch.zeros_like(d["value"])
    gl, ga = torch.empty_like(d["loc"]), torch.empty_like(d["attn"])
    f = lambda: msda.ext_module.ms_deform_attn_forward(d["value"], d["shapes"], d["lsi"], d["loc"], d["attn"], im2col_step=64)
    def b():
        gv.zero_()
        msda.ext_module.ms_deform_attn_backward(d["value"], d["shapes"], d["lsi"], d["loc"], d["attn"], d["grad_out"], gv, gl, ga, im2col_step=64)
    fb, bb = bench.msda_algorithmic_bytes(6 * Q, 6)
    samples = 6 * Q * 8 * 32
    return {"fwd": row(window_ms(f, 10, 3), samples, fb), "bwd": row(window_ms(b, 10, 3), samples, bb)}


def msda_tsa(n):
    g = torch.Generator(device=dev).manual_seed(0)
    Q = n * n
    val = torch.randn(2, Q, 8, 32, device=dev, generator=g)
    loc = torch.rand(2, Q, 8, 1, 4, 2, device=dev, generator=g)
    aw = torch.softmax(torch.randn(2, Q, 8, 4, device=dev, generator=g), -1).view(2, Q, 8, 1, 4)
    shp, lsi = torch.tensor([[n, n]], device=dev), torch.tensor([0], device=dev)
    go = torch.randn(2, Q, 256, device=dev, generator=g)
    gv, gl, ga = torch.zeros_like(val), torch.empty_like(loc), torch.empty_like(aw)
    f = lambda: msda.ext_module.ms_deform_attn_forward(val, shp, lsi, loc, aw, im2col_step=64)
    def b():
        gv.zero_()
        msda.ext_module.ms_deform_attn_backward(val, shp, lsi, loc, aw, go, gv, gl, ga, im2col_step=64)
    vb = 2 * Q * 256 * 4
    fb = vb + 2 * Q * (8 * 4 * 3 * 4 + 1024)
    bbytes = 3 * vb + 2 * Q * (8 * 4 * 3 * 4 * 2 + 1024)
    return {"fwd": row(window_ms(f, 10, 3), 2 * Q * 8 * 4, fb), "bwd": row(window_ms(b, 10, 3), 2 * Q * 8 * 4, bbytes)}


def latent(n):
    g = torch.Generator(device=dev).manual_seed(1)
    occ = torch.randn(1, n, n, 16, device=dev, generator=g)
    feat = torch.randn(1, n, n, 16, device=dev, generator=g)
    def fb():
        o, f = occ.detach().requires_grad_(True), feat.detach().requires_grad_(True)
        p, q = latent_render_core(o, f, 256, 0.5, 1e-3, 1)
        (p.sum() + q.sum()).backward()
    return row(window_ms(fb, 10, 3), n * n, 2 * n * n * 256 * 4 + 3 * n * n * 256 * 4)     # module bytes: 82 MB fwd + 123 MB bwd at n=200


def rays(M, T):
    sigma, origin, points, tindex = dvr_inputs_lidar(M=M, T=T, seed=0)
    s, o, p, t = (torch.from_numpy(x).to(dev) for x in (sigma, origin, points, tindex))
    vol = T * 16 * 200 * 200 * 4
    r = lambda: render.dvr.render(s, o, p, t, "l2")
    fr = t[0].to(torch.int32).contiguous()
    def ce():
        sg = s[0].detach().requires_grad_(True)
        c, v = ray_head.ray_ce(sg, o[0].contiguous(), p[0].contiguous(), fr, 512, 1.0)
        c.sum().backward()
    return {"dvr.render(l2)": row(window_ms(r, 10, 3), M, 3 * vol + 24 * M), "ray_sampler+CE fwd+bwd": row(window_ms(ce, 10, 3), M, 3 * vol + 20 * M)}


out = {"gpu": card(), "hbm_peak_GBps": PEAK,
       "msda_sca_6cam": {f"Q={Q}": msda_sca(Q) for Q in (10000, 40000)},
       "msda_tsa_B2": {f"bev={n}x{n}": msda_tsa(n) for n in (100, 200, 400)},
       "latent_render_core_fwd_bwd": {f"bev={n}x{n}": latent(n) for n in (100, 200, 400)},
       "rays": {f"M={M},frames={T}": rays(M, T) for M in (10000, 30000, 100000) for T in (1, 3, 6)}}
print(json.dumps(out, indent=1))
