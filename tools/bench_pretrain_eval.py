"""Evaluation from files (vidar_b200/pretrain.py) at full size on one GPU, one JSON line on stdout.

The `vidar_1_8_nusc_3future` preset with the DCNv2 backbone, GridMask and the point pipeline, evaluated over one scene
(`pretrain.synthetic_scene`): --samples consecutive samples of --frames image frames of 6 x 900 x 1600 camera JPEGs
(the test queue: queue_length 4 previous frames and the current one) and 1 + --future GT frames each, --future
roll-outs, --workers DataLoader workers.  Two arms, alternated --rounds times after one untimed call of each on a
2-sample scene:
  (a) `per_sample`: the test-mode `SampleLoader`, `forward_test` per sample, then `evaluate.summarize`;
  (b) `evaluate`: `pretrain.evaluate`, with its feature reuse and one host conversion per call.
Each arm reports ms per sample (host clock around the whole call and a synchronize, `gpu_timing.host_ms`, median over
the rounds, divided by --samples), host syncs per sample and their file:line sites (`gpu_timing.count_syncs`, one more
call), backbone passes per call and the peak allocation; the line also holds `gpu_timing.card()` and whether the two
arms' summaries are equal.

    python tools/bench_pretrain_eval.py [--samples 12] [--rounds 3] [--workers 4] [--out f.jsonl]
    python tools/bench_pretrain_eval.py --dry-run      # both arms at a tiny size on the CPU side, no timing
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

from tools.gpu_timing import card, count_syncs, host_ms  # noqa: E402

CONFIG = "vidar_1_8_nusc_3future"


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0], formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--samples", type=int, default=12, help="samples of the timed scene")
    ap.add_argument("--frames", type=int, default=5, help="image frames per sample (queue_length + 1)")
    ap.add_argument("--future", type=int, default=6, help="future frames (the test_future_frame_num)")
    ap.add_argument("--rounds", type=int, default=3, help="timed calls of each arm, alternated")
    ap.add_argument("--workers", type=int, default=4, help="DataLoader workers")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    ap.add_argument("--dry-run", action="store_true",
                    help="build both arms' inputs at a tiny size and check their plans, without a GPU")
    args = ap.parse_args(argv)
    if args.samples < 1 or args.frames < 1 or args.future < 0 or args.rounds < 1 or args.workers < 0:
        ap.error("--samples, --frames, --rounds >= 1; --future, --workers >= 0")
    return args


def _same(a, b):
    return a.keys() == b.keys() and all(
        a[f].keys() == b[f].keys() and all(np.array_equal(np.float64(a[f][k]), np.float64(b[f][k]), equal_nan=True)
                                           for k in a[f]) for f in a)


def dry_run(args):
    """The scene and the test-mode loader's host half at 90 x 160 on 2 cameras: what the GPU run will read."""
    from vidar_b200 import pretrain
    model, _ = pretrain.build("cpu", seed=args.seed, config=CONFIG, grid_mask=True, point_pipeline=True,
                              encoder_layers=1, bev_hw=(20, 20), ray_grid_num=32, num_cams=2)
    queues = pretrain.synthetic_scene(3, args.frames, args.future, cams=2, img_hw=(90, 160), points_per_frame=500,
                                      seed=args.seed)
    loader = pretrain.SampleLoader(model, queues, num_workers=0, prefetch=0, test_mode=True)
    hosts = list(loader.host_loader)
    shared = [len(set(tuple(r["filename"]) for r in a["frames"]) & set(tuple(r["filename"]) for r in b["frames"]))
              for a, b in zip(hosts, hosts[1:])]
    return dict(dry_run=True, config=CONFIG, samples=len(hosts), frames=args.frames, future=args.future,
                gt_frames=[len(h["points"]) for h in hosts], shared_frames_between_neighbours=shared,
                pad_hw=hosts[0]["frames"][0]["img_aug"].pad_hw, workers=args.workers)


def main(argv=None):
    args = parse(argv)
    if args.dry_run:
        print(json.dumps(dry_run(args)), flush=True)
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_pretrain_eval needs a CUDA device")
    from vidar_b200 import evaluate, pretrain
    dev = torch.device("cuda", 0)
    model, _ = pretrain.build(dev, seed=args.seed, config=CONFIG, dcn=True, grid_mask=True, point_pipeline=True)
    model.eval()
    warm = pretrain.synthetic_scene(2, args.frames, args.future, seed=args.seed + 1)
    scene = pretrain.synthetic_scene(args.samples, args.frames, args.future, seed=args.seed)
    passes = [0]
    model.backbone.stem[0].register_forward_hook(lambda *_: passes.__setitem__(0, passes[0] + 1))
    out = {}

    def per_sample(queues):
        loader = pretrain.SampleLoader(model, queues, num_workers=args.workers, prefetch=0, seed=args.seed,
                                       test_mode=True)
        out["per_sample"] = evaluate.summarize([model.forward_test(s["img"], None, s["gt_points"],
                                                                   future_frames=args.future,
                                                                   img_metas=s["img_metas"])[0] for s in loader])

    def evaluate_arm(queues):
        out["evaluate"] = pretrain.evaluate(model, queues, future_frames=args.future, num_workers=args.workers,
                                            prefetch=0, seed=args.seed)

    arms = dict(per_sample=per_sample, evaluate=evaluate_arm)
    line = dict(config=CONFIG, dcn=True, grid_mask=True, samples=args.samples, frames=args.frames,
                future=args.future, rounds=args.rounds, workers=args.workers, cpus=os.cpu_count(), prefetch=0)
    for name, fn in arms.items():                                   # warm-up: compile caches, the loaders' workers
        fn(warm)
    ms = host_ms({k: (lambda f=f: f(scene)) for k, f in arms.items()}, args.rounds, 0)
    summaries = {}
    for name, fn in arms.items():
        np.random.seed(args.seed)
        random.seed(args.seed)
        passes[0] = 0
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        syncs, sites = count_syncs(fn, scene)
        summaries[name] = out[name]
        line[f"{name}_ms_per_sample"] = ms[name] / args.samples
        line[f"{name}_syncs_per_sample"] = syncs / args.samples
        line[f"{name}_sync_sites"] = sites
        line[f"{name}_backbone_passes"] = passes[0]
        line[f"{name}_peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2**30
    line["summaries_equal"] = _same(summaries["per_sample"], summaries["evaluate"])
    line["summary"] = summaries["evaluate"]
    line.update(card())
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "a") as fh:
            fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
