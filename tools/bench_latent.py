"""LatentRendering kernels at the bench configuration (1 x 200 x 200, pred_height 16, one feature channel per
height, grid_num 256, grid_step 0.5, sigmoid), one entry point at a time:

    python tools/bench_latent.py [--iters 200] [--json out.json] [--counts-only]

Each entry point of csrc/latent_render.cu is timed with CUDA events around every launch, after warm-up, with the
L2 flushed before each launch (as the MSDA stage leaves it in bench.py).  The backward entry points run with the
forward's aux buffer, as the module does; the whole fused module forward + backward is timed the same way.  Prints
the card name and power limit, the 64-byte reductions the backward kernels send per map -- one per (cell, waypoint,
corner) for the per-cell scatter, one per touched box pixel plus one per out-of-box corner for angular bundles --
computed on the CPU from the geometry (the phase 1 backward keeps its per-cell scatter; its bundle count is what
the scheme would send), and one JSON line.
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gpu_timing import card, event_ms  # noqa: E402

HB, WB, D, G, GRID_NUM, STEP, EPS, ACT = 200, 200, 16, 1, 256, 0.5, 1e-3, 1
BOX = 4                      # box side of a bundle's footprint at one waypoint
ANGLE_BITS = 20              # angle bins of the cell order (2^20, csrc/latent_render.cu kAngleBits)


def reduction_counts(Hb=HB, Wb=WB, grid_num=GRID_NUM, step=STEP, bundles=(32, 64)):
    """64-byte reductions per map of the two backward kernels: per-cell scatter vs angular bundles of B cells."""
    from oracle.latent_render_ref import geometry, sqrt_rn
    grid, m1, m2 = geometry(Hb, Wb, grid_num, step, sqrt=sqrt_rn)
    g = grid[:, :grid_num].numpy()
    ix = ((g[..., 0] + np.float32(1)) * np.float32(Wb) - np.float32(1)) * np.float32(0.5)
    iy = ((g[..., 1] + np.float32(1)) * np.float32(Hb) - np.float32(1)) * np.float32(0.5)
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    masks = {"pool_bwd": m2.numpy(), "prob_bwd": m1[:, :grid_num].numpy()}
    cy, cx = np.divmod(np.arange(Hb * Wb), Wb)
    ang = np.arctan2((2 * cy + 1 - Hb).astype(np.float32), (2 * cx + 1 - Wb).astype(np.float32))
    nbin = 1 << ANGLE_BITS
    key = np.minimum(((ang.astype(np.float64) + math.pi) * (nbin / (2 * math.pi))).astype(np.int64), nbin - 1)
    order = np.argsort(key, kind="stable")
    out = {}
    for name, m in masks.items():
        corners = [(x0 + dx, y0 + dy) for dy in (0, 1) for dx in (0, 1)]
        inimg = [m & (x >= 0) & (x < Wb) & (y >= 0) & (y < Hb) for x, y in corners]
        old = int(sum(a.sum() for a in inimg))
        res = {"per_cell": old}
        for B in bundles:
            n = len(order)
            pad = (-n) % B
            idx = np.concatenate([order, np.full(pad, -1)]).reshape(-1, B)
            live = idx >= 0
            sel = np.where(live, idx, 0)
            mk = m[sel] & live[..., None]                              # [nb, B, K]
            big = np.int64(1) << 40
            bx = np.where(mk, x0[sel], big).min(1, keepdims=True)
            by = np.where(mk, y0[sel], big).min(1, keepdims=True)
            bits = np.zeros(mk.shape[::2], dtype=np.int64)           # [nb, K] touched box pixels
            direct = 0
            for (x, y), a in zip(corners, inimg):
                xs, ys, a = x[sel], y[sel], a[sel] & live[..., None]
                inbox = a & (xs - bx < BOX) & (ys - by < BOX)
                direct += int((a & ~inbox).sum())
                sh = np.where(inbox, (ys - by) * BOX + (xs - bx), 0)
                bits |= np.bitwise_or.reduce(np.where(inbox, np.int64(1) << sh, 0), axis=1)
            flush = int(np.unpackbits(bits.astype(">u8").view(np.uint8)).sum())
            res[f"bundle{B}"] = flush + direct
            res[f"bundle{B}_out_of_box"] = direct
        out[name] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--counts-only", action="store_true")
    ap.add_argument("--profile", action="store_true", help="also print torch.profiler's kernel table of the backward")
    a = ap.parse_args()

    counts = reduction_counts()
    for k, v in counts.items():
        s = ", ".join(f"{n} {c / 1e6:.3f} M" for n, c in v.items())
        print(f"[bench_latent] {k} 64-B reductions per map: {s}")
    result = {"counts_per_map": counts}
    if a.counts_only:
        print(json.dumps(result))
        return

    from vidar_b200 import _lib
    import bench
    import vidar_b200.modules  # noqa: F401
    from vidar_b200.registry import build_attention
    dev = torch.device("cuda:0")
    name = card()
    print(f"[bench_latent] card: {name}")
    L = _lib.lib()
    P = _lib.ptr
    g = torch.Generator(device=dev).manual_seed(0)
    R = HB * WB
    occ = torch.randn(1, HB, WB, D, device=dev, generator=g) * 1.5
    feat = torch.randn(1, HB, WB, D * G, device=dev, generator=g)
    gq = torch.randn(R, D * G, device=dev, generator=g)
    prob, pooled = torch.empty(R, D, device=dev), torch.empty(R, D * G, device=dev)
    aux = torch.empty(3, R, D, device=dev)
    gpm, gfe, gocc = (torch.zeros(R, D, device=dev) for _ in range(3))
    st = _lib.stream_ptr(dev)
    calls = {
        "latent_prob_fwd": lambda: L.vidar_latent_prob_forward(P(occ), P(prob), P(aux), 1, D, HB, WB, GRID_NUM, STEP, ACT,
                                                               0, R, st),
        "latent_pool_fwd": lambda: L.vidar_latent_pool_forward(P(prob), P(feat), P(pooled), P(aux), 1, D, G, HB, WB,
                                                               GRID_NUM, STEP, EPS, 0, R, st),
        "latent_pool_bwd": lambda: L.vidar_latent_pool_backward(P(prob), P(feat), P(pooled), P(aux), P(gq), P(gpm), P(gfe),
                                                                1, D, G, HB, WB, GRID_NUM, STEP, EPS, 0, R, st),
        "latent_prob_bwd": lambda: L.vidar_latent_prob_backward(P(occ), P(aux), P(gpm), P(gocc), 1, D, HB, WB, GRID_NUM,
                                                                STEP, ACT, 0, R, st),
    }
    times = {}

    def record(k, fn, iters):
        med, ms = event_ms(fn, iters, a.warmup, flush=True, sync=False, raw=True)
        times[k] = {"mean_ms": statistics.fmean(ms), "median_ms": med}

    for k, fn in calls.items():
        record(k, lambda fn=fn: _lib.check(fn()), a.iters)

    if a.profile:
        # kernel split of the backward entry points (cell order + bundle kernel), in a run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                _lib.check(calls["latent_pool_bwd"]())
                _lib.check(calls["latent_prob_bwd"]())
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12, max_name_column_width=70))

    torch.manual_seed(0)
    mod = build_attention(bench.LR_CFG).to(dev)
    emb = torch.randn(1, HB, WB, 256, device=dev, generator=g)
    gemb = torch.randn(1, HB, WB, 256, device=dev, generator=g)

    def step():
        e = emb.detach().requires_grad_(True)
        mod.zero_grad(set_to_none=True)
        mod(e).backward(gemb)
    record("module_fwd_bwd", step, a.iters // 4)
    for k, v in times.items():
        print(f"[bench_latent] {k:16s} {v['median_ms']:.4f} ms median, {v['mean_ms']:.4f} ms mean")
    result.update(card=name, iters=a.iters, times=times)
    line = json.dumps(result)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
