"""GridMask at the pre-training shape (6 x 3 x 928 x 1600): the reference's statements (numpy stripes + PIL rotate +
crop on the host, a pageable `.cuda()` upload, `1 - mask`, `x * mask`) against `vidar_b200.grid_mask.GridMask`
(one launch), in fp32 and fp16, then one synthetic pre-training step with `grid_mask=True` under each, alternated.

  * host: wall clock around one call that ends in torch.cuda.synchronize() (median of 20, warmed up);
  * kernel: CUDA events around the device work alone (median of 20): the new kernel, or the reference's
    `1 - mask` and multiply on an uploaded mask; its algorithmic bytes (read x, write out) over 3.35 TB/s, the H100
    SXM data-sheet HBM3 bandwidth;
  * blocking: behind a ~50 ms device sleep, how long the host takes to return from the call, and whether the call
    makes a synchronising CUDA call (tools/gpu_timing.py's count_syncs) -- observed, not assumed;
  * step: `pretrain.train_step` with the cfg's GridMask (prob forced to 1 so every step masks), device op vs
    reference statements, alternated.
The card's name, power limit and SM clock are read in the same run.

    python tools/bench_grid_mask.py [--steps 5] [--out /tmp/bench_grid_mask.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import grid_mask_ref  # noqa: E402
from tools.gpu_timing import card, count_syncs, event_ms, host_ms  # noqa: E402
from vidar_b200 import grid_mask, pretrain  # noqa: E402

SHAPE = (6, 3, 928, 1600)
PEAK_BW = 3.35e12
CFG = dict(use_h=True, use_w=True, rotate=1, offset=False, ratio=0.5, mode=1, prob=0.7)


def reference_statements(module, x, draw):
    """The reference's forward from its draws on: host mask, blocking upload, `1 - mask`, multiply."""
    n, c, h, w = x.shape
    mask = grid_mask_ref.pil_mask(h, w, draw.d, draw.l, draw.st_h, draw.st_w, draw.r, module.use_h, module.use_w, 0)
    mask = torch.from_numpy(mask).to(x.dtype).cuda()
    if module.mode == 1:
        mask = 1 - mask
    return (x.view(-1, h, w) * mask.expand_as(x.view(-1, h, w))).view(n, c, h, w)


def blocking(fn):
    """(host ms to return from fn behind a ~50 ms device sleep, whether fn makes a synchronising CUDA call)."""
    torch.cuda.synchronize()
    torch.cuda._sleep(50_000_000)
    t0 = time.perf_counter()
    fn()
    ret = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    return ret, count_syncs(fn)[0] > 0


def op_bench(dev):
    res = {}
    m = grid_mask.GridMask(**dict(CFG, prob=1.0)).train()
    for dt in (torch.float32, torch.float16):
        x = torch.randn(SHAPE, device=dev).to(dt)
        np.random.seed(0)
        draw = m.sample(*SHAPE[-2:])
        # same values first
        assert torch.equal(m.masked(x, draw), reference_statements(m, x, draw))
        dev_mask = torch.from_numpy(grid_mask_ref.pil_mask(*SHAPE[-2:], draw.d, draw.l, draw.st_h, draw.st_w,
                                                           draw.r, True, True, 0)).to(dt).to(dev)
        nbytes = 2 * x.numel() * x.element_size()
        r = {}
        for name, fn in (("reference", lambda: reference_statements(m, x, draw)), ("device", lambda: m.masked(x, draw))):
            r[name] = dict(host_ms=host_ms(fn, 20, 3))
        # with the draws included, as a forward call makes them (the reference's numpy draws are the same)
        r["device"]["host_ms_with_draws"] = host_ms(lambda: m(x), 20, 3)
        r["reference"]["kernel_ms"] = event_ms(lambda: x * (1 - dev_mask).expand_as(x), 20, 3)
        r["device"]["kernel_ms"] = event_ms(lambda: grid_mask.grid_mask_apply(x, draw, True, True, 1), 20, 3)
        for name in r:
            r[name]["kernel_bytes_share_of_peak"] = nbytes / (r[name]["kernel_ms"] * 1e-3) / PEAK_BW
            ret, synced = blocking(lambda: (reference_statements(m, x, draw) if name == "reference"
                                            else m.masked(x, draw)))
            r[name]["host_return_ms_behind_50ms_sleep"] = ret
            r[name]["syncs"] = synced
        r["algorithmic_bytes"] = nbytes
        res[str(dt).split(".")[-1]] = r
        print(json.dumps({str(dt): r}), flush=True)
    return res


def step_bench(dev, steps):
    model, opt = pretrain.build(dev, None, seed=0, grid_mask=True)
    model.grid_mask.prob = 1.0
    sample = pretrain.synthetic_sample(dev)
    device_masked = model.grid_mask.masked
    paths = {"device": device_masked, "reference": lambda x, draw: reference_statements(model.grid_mask, x, draw)}

    def run(k):
        model.grid_mask.masked = paths[k]
        pretrain.train_step(model, opt, sample)

    np.random.seed(0)
    med, ms = host_ms({k: lambda k=k: run(k) for k in paths}, steps, 1, raw=True)     # alternating
    model.grid_mask.masked = device_masked
    return {k: dict(median_ms=med[k], all_ms=ms[k]) for k in paths}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grid_mask needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(card=card(), shape=list(SHAPE), op=op_bench(dev))
    res["step"] = step_bench(dev, args.steps)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
