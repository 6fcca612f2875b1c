"""The pre-training configs' optimizer stage on one GPU, one JSON document on stdout: gradient clip to a total norm
of 35 and AdamW over the harness's full parameter list (SyntheticViDAR, full size: every parameter in the
optimizer, 560 of them trainable with real-size random gradients whose norm is above 35, so the clip is active).

Variants, each run alone on the same parameters, gradients and fresh state:
  (a) mmcv's form of the configs: `optim.paramwise_groups` (one group per tensor, backbone at lr_mult 0.1) +
      torch.optim.AdamW + clip_grad_norm_ + float(norm) for the log;
  (b) `pretrain.build()`'s optimizer: one torch.optim.AdamW group + clip_grad_norm_;
  (c) torch.optim.AdamW(fused=True), one group, + clip_grad_norm_;
  (d) `optim.AdamW(paramwise_groups(...), max_grad_norm=35)` (`pretrain.config_optimizer`).
Per variant: host wall clock to a synchronised result (median of --iters), CUDA-event time of the call with calls
queued back to back (median; it includes the host's time when the host cannot keep ahead), kernels launched per
step and the sum of their durations (torch.profiler, one call), host syncs per step; for (d) also the bytes the step
must move (gradient read twice, parameter / exp_avg / exp_avg_sq read and written: 32 B per element) over its kernel
time, against the 3.35 TB/s data-sheet bandwidth, and the host time of `step()` alone (no sync).
Then the `"optimizer"` stage of the full 1 x 1 pre-training step (`train_step(record=True)`) with `config_optimizer`
and with `build()`'s optimizer, alternating step by step on one model.  The card's name and power limit are read in
the same run.

    python tools/bench_optim.py [--iters 20] [--warmup 3] [--steps 5] [--out f.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gpu_timing import card, count_syncs, cpu_ms, cuda_kernels, event_ms, host_ms  # noqa: E402

PEAK_BW = 3.35e12          # H100 SXM data-sheet HBM3 bandwidth
KEYS = {"backbone": dict(lr_mult=0.1)}


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=20, help="timed calls per variant (median)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed calls per variant first")
    ap.add_argument("--steps", type=int, default=5, help="pre-training steps per optimizer in the stage comparison")
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    return ap.parse_args(argv)


def variants(model, lr=2e-4):
    from vidar_b200 import optim
    trainable = [p for p in model.parameters() if p.requires_grad]

    def clipped(opt, sync=False):
        def step():
            norm = torch.nn.utils.clip_grad_norm_(trainable, 35.0)
            if sync:
                float(norm)
            opt.step()
        return step

    def make(name):
        if name == "a_mmcv_paramwise_torch":
            opt = torch.optim.AdamW(optim.paramwise_groups(model, lr, 0.01, KEYS), lr=lr, weight_decay=0.01)
            return opt, clipped(opt, sync=True)
        if name == "b_harness_single_group":
            opt = torch.optim.AdamW(trainable, lr=lr, weight_decay=0.01)
            return opt, clipped(opt)
        if name == "c_torch_fused":
            opt = torch.optim.AdamW(trainable, lr=lr, weight_decay=0.01, fused=True)
            return opt, clipped(opt)
        opt = optim.AdamW(optim.paramwise_groups(model, lr, 0.01, KEYS), lr=lr, weight_decay=0.01, max_grad_norm=35)
        return opt, opt.step
    return make, trainable


def main(argv=None):
    args = parse(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim needs a CUDA device")
    from vidar_b200 import _lib, pretrain
    dev = torch.device("cuda:0")
    out = dict(card=card(), iters=args.iters, warmup=args.warmup, variants={})
    torch.manual_seed(0)
    model = pretrain.SyntheticViDAR().to(dev)
    make, trainable = variants(model)
    g = torch.Generator(device=dev).manual_seed(1)
    grads = [torch.randn(p.shape, generator=g, device=dev) * 0.01 for p in trainable]
    elems = sum(p.numel() for p in trainable)
    norm = float(torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(x) for x in grads])))
    out.update(parameters=sum(1 for _ in model.parameters()), trainable=len(trainable), elements=elems, grad_norm=norm)
    start = [p.detach().clone() for p in model.parameters()]

    def reset():
        with torch.no_grad():
            for p, s in zip(model.parameters(), start):
                p.copy_(s)
        for p, x in zip(trainable, grads):
            p.grad = x.clone()

    for name in ("a_mmcv_paramwise_torch", "b_harness_single_group", "c_torch_fused", "d_vidar_adamw"):
        reset()
        opt, step = make(name)
        row = dict(host_ms=host_ms(step, args.iters, args.warmup),
                   event_ms=event_ms(step, args.iters, args.warmup, sync=False))
        row["kernels"], row["kernel_ms"] = cuda_kernels(step)
        row["host_syncs"] = count_syncs(step)[0]
        if name == "d_vidar_adamw":
            n0 = _lib.launch_count()
            step()
            row["vidar_launches"] = _lib.launch_count() - n0
            row["step_host_ms"] = cpu_ms(step, args.iters, 1)      # enqueue only
            torch.cuda.synchronize()
            nbytes = 32 * elems
            row["bytes"] = nbytes
            row["achieved_TBps"] = nbytes / (row["kernel_ms"] * 1e-3) / 1e12       # over the kernels' own time
            row["share_of_3.35TBps"] = row["achieved_TBps"] * 1e12 / PEAK_BW
        out["variants"][name] = row
        del opt, step
        torch.cuda.empty_cache()
        print(name, json.dumps(row), file=sys.stderr, flush=True)

    # the "optimizer" stage of the full pre-training step, the two optimizers alternating on one model
    for p in model.parameters():
        p.grad = None
    del grads, start
    torch.cuda.empty_cache()
    model, torch_opt = pretrain.build(dev, None, seed=0)
    opts = dict(build_torch_adamw=torch_opt, config_optimizer=pretrain.config_optimizer(model))
    sample = pretrain.synthetic_sample(dev)
    stage = {k: [] for k in opts}
    for i in range(args.steps + 1):
        for k, o in opts.items():
            _, stages = pretrain.train_step(model, o, sample, None, record=True)
            if i:                                   # the first step of each is warm-up
                stage[k].append(dict(stages)["optimizer"])
    out["pretrain_optimizer_stage_ms"] = {k: dict(median=statistics.median(v), all=v) for k, v in stage.items()}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
