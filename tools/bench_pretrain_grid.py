"""The synthetic pre-training step (vidar_b200/pretrain.py, full size) under every (replica x shard) process grid the
world allows, alternated step by step in one launch, one JSON document on rank 0's stdout:

  * per grid R x S: ms per step (host clock around `train_step`, which ends in a device synchronise; median over
    steps, the slowest rank), samples per second (R samples per step), the grad-sync stage's ms (`train_step`'s
    recorded stages: pack, the one all-reduce, unpack), the model's resident bytes (parameters, gradients, AdamW
    state) and the step's peak allocation above them;
  * the sync's kernels alone on rank 0's real parameter list: pack and unpack (`vidar_b200.grad_bucket`), with and
    without their host-side table build, against the `torch.cat` of grad * scale and one copy per parameter they
    replace (CUDA events around each call, median), and the kernels' bytes over the 3.35 TB/s data-sheet bandwidth;
  * the card's name, power limit and SM clock of every rank, read in the same run.

Each replica draws its own sample (`synthetic_sample(seed=base + replica)`, numpy seeded per replica).

    torchrun --nproc_per_node 8 tools/bench_pretrain_grid.py [--shards 1,2,4,8] [--steps 5] [--warmup 2] [--out f.json]
    python tools/bench_pretrain_grid.py --dry-run --world 8     # the grids and the plan, no GPU
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.gpu_timing import card, event_ms, host_ms  # noqa: E402

PEAK_BW = 3.35e12          # H100 SXM data-sheet HBM3 bandwidth


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0], formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shards", default=None,
                    help="comma-separated shard sizes S (each must divide the world); default: every divisor")
    ap.add_argument("--steps", type=int, default=5, help="timed steps per grid")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps per grid first")
    ap.add_argument("--seed", type=int, default=0, help="base seed: replica r draws with base + r")
    ap.add_argument("--out", default=None, help="also write the JSON document here (rank 0)")
    ap.add_argument("--dry-run", action="store_true", help="print the grids for --world and exit (no GPU needed)")
    ap.add_argument("--world", type=int, default=None, help="world size of a dry run (default: $WORLD_SIZE or 1)")
    args = ap.parse_args(argv)
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    return args


def shard_sizes(world, spec):
    sizes = [s for s in range(1, world + 1) if world % s == 0] if spec is None else [int(s) for s in spec.split(",")]
    bad = [s for s in sizes if s < 1 or world % s]
    if bad:
        raise SystemExit(f"shard sizes {bad} do not divide the world size {world}")
    return sizes


def resident_bytes(model, opt):
    ts = [p for p in model.parameters()] + [p.grad for p in model.parameters() if p.grad is not None]
    ts += [v for st in opt.state.values() for v in st.values() if torch.is_tensor(v) and v.is_cuda]
    return sum(t.numel() * t.element_size() for t in ts)


def sync_kernels(model, grid):
    """pack / unpack against torch.cat of grad * scale and one copy_ per parameter, on the model's real gradients."""
    from vidar_b200 import _lib, grad_bucket, sharding
    ps = [p for p in model.parameters() if p.requires_grad and p.grad is not None]
    scales = sharding.grid_grad_scales(ps, grid)
    bucket = grad_bucket.pack(ps, scales)
    assert torch.equal(bucket, torch.cat([p.grad.reshape(-1) * s for p, s in zip(ps, scales)]))

    def torch_unpack():
        off = 0
        for p in ps:
            p.grad.copy_(bucket[off: off + p.numel()].view_as(p.grad))
            off += p.numel()

    # the kernels behind a prepared table: what pack / unpack cost beyond their host-side table build
    ptr, numel, offset, device = grad_bucket._table(ps, False)
    sc = np.asarray(scales, np.float32)
    lib, st = _lib.lib(), _lib.stream_ptr(device)
    ms = event_ms({"pack": lambda: grad_bucket.pack(ps, scales, out=bucket),
                   "unpack": lambda: grad_bucket.unpack(bucket, ps),
                   "pack_kernel": lambda: lib.vidar_grad_bucket_pack(ptr.ctypes.data, numel.ctypes.data,
                                                                     offset.ctypes.data, sc.ctypes.data, len(ps),
                                                                     _lib.ptr(bucket), bucket.numel(), st),
                   "unpack_kernel": lambda: lib.vidar_grad_bucket_unpack(_lib.ptr(bucket), bucket.numel(),
                                                                         ptr.ctypes.data, numel.ctypes.data,
                                                                         offset.ctypes.data, len(ps), st),
                   "torch_cat": lambda: torch.cat([p.grad.reshape(-1) * s for p, s in zip(ps, scales)]),
                   "torch_copies": torch_unpack}, 20, 3)
    nbytes = 2 * bucket.numel() * 4                   # read and write every element once
    share = {k: nbytes / (ms[k] * 1e-3) / PEAK_BW for k in ("pack_kernel", "unpack_kernel")}
    return dict(tensors=len(ps), bucket_mb=bucket.numel() * 4 / 2**20, ms=ms, bytes=nbytes,
                kernel_share_of_hbm_peak=share)


def main(argv=None):
    args = parse(argv)
    if args.dry_run:
        world = args.world or int(os.environ.get("WORLD_SIZE", "1"))
        sizes = shard_sizes(world, args.shards)
        print(json.dumps(dict(world=world, grids=[f"{world // s}x{s}" for s in sizes], steps=args.steps,
                              warmup=args.warmup, seed=args.seed)))
        return
    import torch.distributed as dist

    from vidar_b200 import pretrain, sharding
    if not torch.cuda.is_available():
        raise SystemExit("bench_pretrain_grid needs CUDA devices (launch with torchrun)")
    if "WORLD_SIZE" not in os.environ:                # plain `python`: a world of one
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29511", RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    world, rank = dist.get_world_size(), dist.get_rank()
    sizes = shard_sizes(world, args.shards)
    runs = {}
    for s in sizes:                                   # every rank makes every grid's groups, in the same order
        grid = sharding.make_grid(s)
        model, opt = pretrain.build(dev, grid=grid, seed=args.seed)
        np.random.seed(args.seed + grid.replica)
        sample = pretrain.synthetic_sample(dev, seed=args.seed + grid.replica)
        runs[f"{grid.replicas}x{s}"] = dict(grid=grid, model=model, opt=opt, sample=sample, sync=[], peak=[])

    def step(r):
        torch.cuda.synchronize()
        start = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _, stages = pretrain.train_step(r["model"], r["opt"], r["sample"], grid=r["grid"], record=True)
        r["sync"].append(dict(stages)["grad_sync"])
        r["peak"].append(torch.cuda.max_memory_allocated() - start)

    card_before = card()
    med, all_ms = host_ms({k: (lambda r=r: step(r)) for k, r in runs.items()}, args.steps, args.warmup, raw=True)
    grids = {}
    for k, r in runs.items():
        sync = r["sync"][args.warmup:]
        mine = dict(ms_per_step=med[k], grad_sync_ms=float(np.median(sync)),
                    step_peak_mb=max(r["peak"]) / 2**20, resident_mb=resident_bytes(r["model"], r["opt"]) / 2**20)
        every = [None] * world
        dist.all_gather_object(every, mine)
        slowest = max(every, key=lambda d: d["ms_per_step"])
        g = r["grid"]
        grids[k] = dict(replicas=g.replicas, shard_size=g.shard_size, samples_per_step=g.replicas,
                        ms_per_step=slowest["ms_per_step"], samples_per_s=g.replicas / (slowest["ms_per_step"] / 1e3),
                        grad_sync_ms=max(d["grad_sync_ms"] for d in every),
                        step_peak_mb=max(d["step_peak_mb"] for d in every),
                        resident_mb=max(d["resident_mb"] for d in every), rank0_all_ms=all_ms[k])
    first = next(iter(runs.values()))
    kernels = sync_kernels(first["model"], first["grid"])
    cards = [None] * world
    dist.all_gather_object(cards, dict(before=card_before, after=card()))
    if rank == 0:
        doc = dict(world=world, steps=args.steps, warmup=args.warmup, grids=grids, sync_kernels_rank0=kernels,
                   cards=cards)
        print(json.dumps(doc))
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "w") as fh:
                json.dump(doc, fh, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
