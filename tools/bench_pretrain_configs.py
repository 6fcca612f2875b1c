"""The pre-training step (vidar_b200/pretrain.py, full size, one GPU) under each training regime of
`pretrain.CONFIGS`, one JSON line per preset on stdout:

  * ms per step: CUDA events around each `train_step`, median over --steps after --warmup (`gpu_timing.event_ms`);
  * per-stage ms of one more step (`train_step(..., record=True)`): backbone and encoder of each computed history
    frame, the current frame, the future decoder, head + loss, backward, optimizer -- with that step's drop index
    and supervised future frames, which decide which stages it has;
  * the step's peak allocation (`peak_mem_gb`, torch.cuda.max_memory_allocated over the timed steps);
  * the card's name, power limit and SM clock, read in the same run.

numpy is seeded with --seed before the presets' steps, so the drop index and the supervised future frame vary from
step to step as in training, the same way in every run.

    python tools/bench_pretrain_configs.py [--configs a,b] [--steps 5] [--warmup 2] [--out f.jsonl]
    python tools/bench_pretrain_configs.py --dry-run         # the presets, no GPU
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


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0], formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", default=None, help="comma-separated preset names (default: every preset)")
    ap.add_argument("--steps", type=int, default=5, help="timed steps per preset")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps per preset first")
    ap.add_argument("--seed", type=int, default=0, help="model, sample and numpy seed")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    ap.add_argument("--dry-run", action="store_true", help="print the presets and exit (no GPU needed)")
    args = ap.parse_args(argv)
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    return args


def presets(spec):
    from vidar_b200 import pretrain
    names = list(pretrain.CONFIGS) if spec is None else spec.split(",")
    bad = [n for n in names if n not in pretrain.CONFIGS]
    if bad:
        raise SystemExit(f"unknown presets {bad}; one of {sorted(pretrain.CONFIGS)}")
    return {n: pretrain.CONFIGS[n] for n in names}


def run(name, args, dev):
    from vidar_b200 import pretrain
    model, opt = pretrain.build(dev, seed=args.seed, config=name)
    sample = pretrain.synthetic_sample(dev, seed=args.seed, future_frames=model.future_frames)
    np.random.seed(args.seed)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = event_ms(lambda: pretrain.train_step(model, opt, sample), args.steps, args.warmup)
    peak = torch.cuda.max_memory_allocated()
    state = np.random.get_state()                 # the recorded step's drop index and supervised future frames
    drop, supervised = model.host_draws(sample["img"].shape[1])
    np.random.set_state(state)
    _, stages = pretrain.train_step(model, opt, sample, record=True)
    line = dict(config=name, steps=args.steps, warmup=args.warmup, ms_per_step=ms,
                stages_ms={k: round(v, 3) for k, v in stages}, stages_drop_prev_index=drop,
                stages_supervised_future=supervised, peak_mem_gb=peak / 2**30, **card())
    del model, opt, sample
    torch.cuda.empty_cache()
    return line


def main(argv=None):
    args = parse(argv)
    chosen = presets(args.configs)
    if args.dry_run:
        for name, cfg in chosen.items():
            print(json.dumps(dict(config=name, steps=args.steps, warmup=args.warmup, preset=cfg)))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_pretrain_configs needs a CUDA device")
    dev = torch.device("cuda", 0)
    for name in chosen:
        line = run(name, args, dev)
        print(json.dumps(line), flush=True)
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "a") as fh:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
