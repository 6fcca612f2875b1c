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

--from-files builds each preset with the DCNv2 backbone, GridMask and both pipelines on, and times three steps on
the same card in the same run, each as ms per step of --steps back-to-back steps between two CUDA events (after
--warmup), so a step's share of the loader's work counts wherever it lands:
  * `files_prefetch_ms`: `pretrain.SampleLoader` over camera JPEGs and LiDAR files (`synthetic_sample(...,
    files=True)`), --workers DataLoader workers, the next sample's decode and pipelines prefetched on a side stream;
  * `files_no_prefetch_ms`: the same with prefetch=0, the device half on the step's stream at the start of each step;
  * `synthetic_ms`: the in-step pipelines on uint8 frames and point files already in memory
    (`synthetic_sample(..., raw_images=True, raw_points=True)`), the host half on the training process.
numpy, `random` and torch are re-seeded with --seed at the start of each arm, so the model's own draws (drop index,
supervised future frame, GridMask) are the same step for step in every arm.  The two loader arms also see the same
dataset draws (their workers are seeded alike); the in-step arm draws its crop / resize / flip from the training
process's generators, so its resize heights differ from theirs.  It also reports per-stage ms of one more
prefetched step, the peak allocation of each arm, the worker count and the host's CPU count.

    python tools/bench_pretrain_configs.py [--configs a,b] [--steps 5] [--warmup 2] [--out f.jsonl]
    python tools/bench_pretrain_configs.py --from-files [--workers 4] [--configs a,b]
    python tools/bench_pretrain_configs.py --dry-run         # the presets, no GPU
"""
import argparse
import json
import os
import random
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
    ap.add_argument("--from-files", action="store_true",
                    help="DCNv2, GridMask and the pipelines on: the loader from files (with and without prefetch) "
                         "against the in-step pipelines")
    ap.add_argument("--workers", type=int, default=4, help="DataLoader workers with --from-files")
    ap.add_argument("--dry-run", action="store_true", help="print the presets and exit (no GPU needed)")
    args = ap.parse_args(argv)
    if args.steps < 1 or args.warmup < 0 or args.workers < 0:
        ap.error("--steps must be >= 1, --warmup and --workers >= 0")
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


def reseed(seed):
    """numpy, `random` and torch seeded alike at the start of each --from-files arm, so that every arm makes the same
    model draws (drop index, supervised future frame, GridMask) step for step."""
    np.random.seed(seed)
    random.seed(seed)
    torch.manual_seed(seed)


def run_from_files(name, args, dev):
    from tools.gpu_timing import window_ms
    from vidar_b200 import pretrain
    model, opt = pretrain.build(dev, seed=args.seed, config=name, dcn=True, grid_mask=True, image_pipeline=True,
                                point_pipeline=True)
    queues = [pretrain.synthetic_sample(None, seed=args.seed + k, future_frames=model.future_frames, files=True)
              for k in range(2)]
    n = args.warmup + args.steps + 1
    samples = [queues[k % 2] for k in range(n)]
    line = dict(config=name, steps=args.steps, warmup=args.warmup, dcn=True, grid_mask=True, pipelines=True,
                workers=args.workers, cpus=os.cpu_count(), affinity=len(os.sched_getaffinity(0)),
                jpeg_kb_per_image=sum(os.path.getsize(p) for p in queues[0][0]["img_filename"]) / 6e3)
    for prefetch, key in ((1, "files_prefetch"), (0, "files_no_prefetch")):
        reseed(args.seed)
        loader = pretrain.SampleLoader(model, samples, num_workers=args.workers, prefetch=prefetch, seed=args.seed)
        it = iter(loader)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        line[f"{key}_ms"] = window_ms(lambda: pretrain.train_step(model, opt, next(it)), args.steps, args.warmup)
        line[f"{key}_peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2**30
        if prefetch:
            _, stages = pretrain.train_step(model, opt, next(it), record=True)
            line["files_prefetch_stages_ms"] = {k: round(v, 3) for k, v in stages}
        del it, loader
    sample = pretrain.synthetic_sample(dev, seed=args.seed, future_frames=model.future_frames, raw_images=True,
                                       raw_points=True)
    reseed(args.seed)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    line["synthetic_ms"] = window_ms(lambda: pretrain.train_step(model, opt, sample), args.steps, args.warmup)
    line["synthetic_peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2**30
    _, stages = pretrain.train_step(model, opt, sample, record=True)
    line["synthetic_stages_ms"] = {k: round(v, 3) for k, v in stages}
    line.update(card())
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
        line = (run_from_files if args.from_files else run)(name, args, dev)
        print(json.dumps(line), flush=True)
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "a") as fh:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
