"""Time TemporalSelfAttention and the future decoder's self- and cross-attention with the fused prologue
(`fuse_epilogue = True`: vidar_msda_tsa_*, softmax / sampling locations / queue mean inside the kernel) against the
reference's statements around the plain op (`fuse_epilogue = False`), at the shipped shapes: bs 1, a 200x200 BEV,
embed 256, 8 heads, 4 points; TSA with a queue of 2 and one level, the decoder's self-attention with one level and
its cross-attention with two history frames as levels.

For each module it times forward and forward + backward of the whole module (value_proj, the Linears, sampling,
output_proj) with CUDA events, the L2 flushed before each call, alternating fused and unfused, median of --iters
after --warmup; and the peak memory allocated during one forward + backward.  The card's name, power limit and SM
clock are read in the same run.

    python tools/bench_msda_tsa.py [--iters 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import vidar_b200.modules  # noqa: E402,F401  (registers the classes)
from tools.gpu_timing import card, event_ms  # noqa: E402
from vidar_b200.registry import build_attention  # noqa: E402

E, BEV = 256, (200, 200)
Q = BEV[0] * BEV[1]


def levels(n):
    s = torch.tensor([BEV] * n, dtype=torch.int64, device="cuda")
    hw = s[:, 0] * s[:, 1]
    return s, torch.cat([hw.new_zeros(1), hw.cumsum(0)[:-1]])


def setup(kind):
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if kind == "tsa":
        m = build_attention(dict(type="TemporalSelfAttention", embed_dims=E, num_levels=1, dropout=0.0))
        shapes, lsi = levels(1)
        value, ref = rnd(2, Q, E), torch.rand(2, Q, 1, 2, device="cuda", generator=g)
    else:
        nl = 1 if kind == "decoder_self" else 2
        m = build_attention(dict(type="PredictionMSDeformableAttention", embed_dims=E, num_levels=nl, dropout=0.0))
        shapes, lsi = levels(nl)
        value, ref = rnd(1, Q * nl, E), torch.rand(1, Q, nl, 2, device="cuda", generator=g)
    m = m.cuda().train()
    with torch.no_grad():        # trained-like offsets of a few pixels and non-uniform weights
        m.sampling_offsets.weight.normal_(0, 0.02, generator=g)
        m.attention_weights.weight.normal_(0, 0.05, generator=g)
    query, pos, grad = rnd(1, Q, E), 0.1 * rnd(1, Q, E), rnd(1, Q, E)
    value.requires_grad_(True)
    query.requires_grad_(True)
    kw = dict(query_pos=pos, reference_points=ref, spatial_shapes=shapes, level_start_index=lsi)

    def fwd():
        return m(query, None, value, **kw)

    def fwd_bwd():
        fwd().backward(grad)

    return m, fwd, fwd_bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    res = {"card": card(), "iters": args.iters}
    print(res["card"], flush=True)
    for kind in ("tsa", "decoder_self", "decoder_cross"):
        m, fwd, fwd_bwd = setup(kind)
        row = {}
        for what, fn in (("forward", fwd), ("forward+backward", fwd_bwd)):
            ctx = torch.no_grad if what == "forward" else torch.enable_grad

            def call(fused, fn=fn, ctx=ctx):
                m.fuse_epilogue = fused
                m.zero_grad(set_to_none=True)
                with ctx():
                    fn()

            ms = event_ms({f: lambda f=f: call(f) for f in (True, False)}, args.iters, args.warmup, flush=True)
            for fused in (True, False):
                row[f"{what} {'fused' if fused else 'unfused'} ms"] = round(ms[fused], 4)
        for fused in (True, False):
            m.fuse_epilogue = fused
            m.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fwd_bwd()
            torch.cuda.synchronize()
            row[f"peak MB {'fused' if fused else 'unfused'}"] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        res[kind] = row
        print(kind, json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
