"""The row-map MSDA (vidar_b200.sca) at the bench shape -- 6 cameras x 40 000 rows, SCA levels, H = 8, C = 32,
P = 8 -- one entry point at a time:

    python tools/bench_msda_rows.py [--iters 20] [--json out.json]
    python tools/bench_msda_rows.py --count

GPU mode times MSDARowsFunction's forward and backward with CUDA events around every call (median after warm-up),
the tile kernel msda_backward_tile_kernel and the row-order kernels alone (torch.profiler kernel time, in a run of
its own), and SCARowsFunction's backward at 6 cameras x 40 000 pillars.  It prints the card name and power limit
and one JSON line.

--count needs no GPU: from the seeded bench inputs of camera 0 (generated on the CPU) and the tile kernel's row
order it counts, per pyramid level and in numpy, the records each scheme sorts and the grad_value line reductions
its sorted-run pass sends -- one record per corner (the runs of equal pixels in each 128-record group segment) and
one record per horizontally adjacent corner pair (the distinct valid pixels of each 64-record segment's pairs).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gpu_timing import card, event_ms  # noqa: E402
from vidar_b200 import synthetic  # noqa: E402

CAMS, Q, H, C, P = 6, 40000, 8, 32, 8
LEVELS = synthetic.SCA_LEVELS
TILE_ROWS = 256                      # csrc/msda.cu kTileRows
GROUPS = 64                          # 8-lane groups of the sorted-run pass (512 threads)


# ---- counts (CPU) ------------------------------------------------------------------------------------------------
def row_order(loc):
    """loc [Q, H, L, P, 2] of one camera -> the tile kernel's row order: a stable sort by the 16 x 16 image cell of
    the mean of head 0's sampling locations (rows_key_kernel)."""
    lp = loc[:, 0].reshape(loc.shape[0], -1, 4)             # float4 pairs of (x, y) samples, as the kernel reads them
    sx = np.zeros(loc.shape[0], np.float32)
    sy = np.zeros(loc.shape[0], np.float32)
    for i in range(lp.shape[1]):
        sx += lp[:, i, 0] + lp[:, i, 2]
        sy += lp[:, i, 1] + lp[:, i, 3]
    s = np.float32(16.0 / (loc.shape[2] * loc.shape[3]))
    kx = np.clip(np.trunc(sx * s), 0, 15).astype(np.int64)
    ky = np.clip(np.trunc(sy * s), 0, 15).astype(np.int64)
    return np.argsort(ky * 16 + kx, kind="stable")


def decode(lx, ly, Hl, Wl):
    """decode_sample in fp32: unclamped (h_low, w_low) and the corner validity masks."""
    h_im = ly * np.float32(Hl) - np.float32(0.5)
    w_im = lx * np.float32(Wl) - np.float32(0.5)
    inside = (h_im > -1) & (w_im > -1) & (h_im < Hl) & (w_im < Wl)
    hl = np.floor(h_im).astype(np.int64)
    wl = np.floor(w_im).astype(np.int64)
    h0, h1 = inside & (hl >= 0), inside & (hl + 1 <= Hl - 1)
    w0, w1 = inside & (wl >= 0), inside & (wl + 1 <= Wl - 1)
    return hl, wl, h0, h1, w0, w1


def distinct_per_segment(seg, key, valid):
    """number of distinct (segment, key) among valid entries"""
    return int(np.unique(seg[valid] * (1 << 32) + key[valid]).size)


def count_level(loc_t, l, Hl, Wl):
    """loc_t [tiles, 256, H, L, P, 2] in row order -> (corner records, corner reductions, pair records,
    pair reductions) of level l over every (tile, head)."""
    xy = np.moveaxis(loc_t[:, :, :, l], 2, 1)               # [tiles, H, 256, P, 2]: one (tile, head) per CTA
    xy = xy.reshape(-1, TILE_ROWS * P, 2)
    cta = xy.shape[0]
    hl, wl, h0, h1, w0, w1 = decode(xy[..., 0], xy[..., 1], Hl, Wl)
    none = np.int64(1) << 40

    # one record per corner: (top-left, top-right, bottom-left, bottom-right) pixels
    px = [(hl, wl, h0 & w0), (hl, wl + 1, h0 & w1), (hl + 1, wl, h1 & w0), (hl + 1, wl + 1, h1 & w1)]
    ck = np.stack([np.where(v, h * Wl + w, none) for h, w, v in px], -1).reshape(cta, -1)
    ck.sort(axis=1)
    seg = np.broadcast_to(np.arange(ck.shape[1]) // (ck.shape[1] // GROUPS), ck.shape) + \
        np.arange(cta)[:, None] * GROUPS
    corner_red = distinct_per_segment(seg.ravel(), ck.ravel(), ck.ravel() != none)

    # one record per corner pair, keyed by its left pixel in a row padded by one column: x' = w_low + 1
    W1 = Wl + 1
    rows = [(hl, h0), (hl + 1, h1)]
    pk = np.stack([np.where(v & (w0 | w1), h * W1 + wl + 1, none) for h, v in rows], -1).reshape(cta, -1)
    pk.sort(axis=1)
    seg = np.broadcast_to(np.arange(pk.shape[1]) // (pk.shape[1] // GROUPS), pk.shape) + \
        np.arange(cta)[:, None] * GROUPS
    live = pk != none
    # the pair keyed k touches slots k (left pixel) and k + 1 (right pixel); slot x' = 0 is the padding column
    slots = np.concatenate([pk[live], pk[live] + 1])
    sseg = np.concatenate([seg[live], seg[live]])
    real = slots % W1 != 0
    pair_red = distinct_per_segment(sseg, slots, real)
    return ck.size, corner_red, pk.size, pair_red


def counts():
    d = synthetic.sca_like_inputs("cpu", cams=1, Q=Q, seed=0)
    loc = d["loc"][0].numpy()                               # [Q, H, L, P, 2]
    loc = loc[row_order(loc)]
    tiles = -(-Q // TILE_ROWS)
    pad = np.full((tiles * TILE_ROWS - Q,) + loc.shape[1:], -10.0, np.float32)   # rows past the last: no sample
    loc_t = np.concatenate([loc, pad]).reshape(tiles, TILE_ROWS, *loc.shape[1:])
    out = []
    print(f"camera 0, {Q} rows, {tiles} tiles x {H} heads; per level: records sorted / line reductions sent")
    print(f"{'level':>10} {'corner recs':>12} {'corner reds':>12} {'pair recs':>12} {'pair reds':>12} {'reds ratio':>10}")
    for l, (Hl, Wl) in enumerate(LEVELS):
        cr, cred, pr, pred = count_level(loc_t, l, Hl, Wl)
        out.append(dict(level=f"{Hl}x{Wl}", corner_records=cr, corner_reductions=cred, pair_records=pr,
                        pair_reductions=pred))
        print(f"{Hl:>4}x{Wl:<5} {cr:>12} {cred:>12} {pr:>12} {pred:>12} {pred / cred:>10.3f}")
    tot = {k: sum(o[k] for o in out) for k in out[0] if k != "level"}
    print(f"{'total':>10} {tot['corner_records']:>12} {tot['corner_reductions']:>12} {tot['pair_records']:>12} "
          f"{tot['pair_reductions']:>12} {tot['pair_reductions'] / tot['corner_reductions']:>10.3f}")
    return {"camera": 0, "levels": out, "total": tot}


# ---- timings (GPU) -----------------------------------------------------------------------------------------------
def _kernel_ms(fn, names, calls):
    """profiler kernel time per call of the kernels whose names contain one of `names`"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    tot = {n: 0.0 for n in names}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        for n in names:
            if n in e.key:
                tot[n] += t
    return {n: v / calls / 1000.0 for n, v in tot.items()}


def timings(iters, warmup):
    from vidar_b200 import sca
    dev = torch.device("cuda", 0)
    d = synthetic.sca_like_inputs(dev, cams=CAMS, Q=Q, seed=0)
    plan = sca.unit_plan(1, 0, CAMS)
    inv = torch.full((1, Q), 1.0 / CAMS, device=dev)
    g = torch.randn(1, Q, H * C, device=dev, generator=torch.Generator(device=dev).manual_seed(11))
    static = [d["value"], d["loc"], d["attn"]]
    # forward and backward alternate, so each backward is timed alone on the slots of the forward before it
    graph = []

    def forward():
        leaves = [t.detach().requires_grad_(True) for t in static]
        return sca.MSDARowsFunction.apply(plan, 1, Q, d["shapes"], d["lsi"], None, None, inv, *leaves)

    out = {"card": card(), "shape": f"{CAMS} cameras x {Q} rows, H={H} C={C} L={len(LEVELS)} P={P}"}
    ms = event_ms({"fwd": lambda: graph.append(forward()), "bwd": lambda: graph.pop().backward(g)}, iters, warmup,
                  sync=False)
    out["rows_fwd_ms"], out["rows_bwd_ms"] = ms["fwd"], ms["bwd"]
    k = _kernel_ms(lambda: forward().backward(g), ["msda_backward_tile_kernel", "rows_key_kernel", "rows_scan_kernel",
                                                   "rows_scatter_kernel"], 5)
    out["tile_kernel_ms"] = k.pop("msda_backward_tile_kernel")
    out["row_order_kernels_ms"] = sum(k.values())

    # SCARowsFunction (fused softmax / sampling-location epilogue) at 6 cameras x 40 000 pillars
    gen = torch.Generator(device=dev).manual_seed(14)
    ref_cam = torch.rand(CAMS, 1, Q, 4, 2, device=dev, generator=gen) * 1.2 - 0.1
    offsets = 4.0 * torch.randn(1, Q, H, len(LEVELS), P, 2, device=dev, generator=gen)
    logits = torch.randn(1, Q, H, len(LEVELS) * P, device=dev, generator=gen)

    def sca_fwd():
        o, lg, v = (t.detach().requires_grad_(True) for t in (offsets, logits, d["value"]))
        graph.append(sca.SCARowsFunction.apply(plan, 1, d["shapes"], d["lsi"], ref_cam, o, lg, None, None, inv, v))

    out["sca_rows_bwd_ms"] = event_ms({"fwd": sca_fwd, "bwd": lambda: graph.pop().backward(g)}, iters, warmup,
                                      sync=False)["bwd"]
    print(f"card: {out['card']}")
    for key in ("rows_fwd_ms", "rows_bwd_ms", "tile_kernel_ms", "row_order_kernels_ms", "sca_rows_bwd_ms"):
        print(f"{key:>22}: {out[key]:.3f}")
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--count", action="store_true", help="also count records and reductions per level (CPU only)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="write the result here as well")
    args = ap.parse_args()
    res = {}
    if args.count:
        res["counts"] = counts()
    if torch.cuda.is_available():
        res["timings"] = timings(args.iters, args.warmup)
    elif not args.count:
        sys.exit("bench_msda_rows.py: timings need a CUDA device (use --count for the CPU counts)")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
