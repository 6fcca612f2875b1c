"""Timing and card readout for the benchmark scripts under tools/.

Four statistics, kept apart because the tools report different ones:
  event_ms   CUDA events around each call, median;
  window_ms  CUDA events around `iters` back-to-back calls, divided by `iters`;
  host_ms    a host clock around each call and a torch.cuda.synchronize(), median;
  cpu_ms     a host clock around each call of host-only work, median.
An absolute time is only worth something with the card it was measured on, so every tool records `card()` in the
same run."""
import os
import statistics
import subprocess
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_flush = None                        # 256 MB, five times the H100's 50 MB L2


def card():
    """{gpu, power_limit, sm_clock, sm_clock_max} of the current device as nvidia-smi reports them; only read.
    Without a working nvidia-smi: torch's device name and "unknown"."""
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", f"--id=GPU-{props.uuid}"],
                             capture_output=True, text=True, timeout=30, check=True).stdout
        gpu, power, sm, sm_max = (f.strip() for f in out.strip().split(","))
    except (OSError, subprocess.SubprocessError, ValueError):
        gpu, power, sm, sm_max = props.name, "unknown", "unknown", "unknown"
    return dict(gpu=gpu, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


def _median_ms(fns, iters, warmup, raw, call, read=float):
    single = callable(fns)
    if single:
        fns = {None: fns}
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(iters):
        for k, fn in fns.items():
            out[k].append(call(fn))
    torch.cuda.synchronize()
    ms = {k: [read(t) for t in v] for k, v in out.items()}
    med = {k: statistics.median(v) for k, v in ms.items()}
    if single:
        med, ms = med[None], ms[None]
    return (med, ms) if raw else med


def event_ms(fns, iters, warmup, flush=False, sync=True, raw=False):
    """Median ms between CUDA events recorded around each call, after `warmup` calls.  `fns` is one zero-argument
    callable, or a dict of them run alternating (the result is then a dict of medians).  raw=True returns (median,
    the ms of every call).

    sync=True synchronises after each call, so every call starts on an idle device and the host's time to its first
    launch counts.  sync=False queues the calls back to back, so the events bracket each call's device work alone.
    flush=True zeroes a 256 MB buffer before each call, outside the events, so every call starts from a cold L2."""
    global _flush
    if flush and _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def call(fn):
        if flush:
            _flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        if sync:
            b.synchronize()
        return a, b

    return _median_ms(fns, iters, warmup, raw, call, lambda ab: ab[0].elapsed_time(ab[1]))


def host_ms(fns, iters, warmup, raw=False):
    """Median ms of time.perf_counter around each call and the torch.cuda.synchronize() after it; `fns`, `warmup`
    and `raw` as in event_ms.  For calls that end on the host, where device events would miss the host's share."""
    def call(fn):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    return _median_ms(fns, iters, warmup, raw, call)


def cpu_ms(fns, iters, warmup, raw=False):
    """Median ms of time.perf_counter around each call, with no synchronise in the window: for host-only work (file
    reads, parsing, packing, a CPU decoder).  `fns`, `warmup` and `raw` as in event_ms."""
    def call(fn):
        t0 = time.perf_counter()
        fn()
        return (time.perf_counter() - t0) * 1e3

    return _median_ms(fns, iters, warmup, raw, call)


def window_ms(fn, iters, warmup):
    """ms per call of `iters` back-to-back calls between two CUDA events, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def count_syncs(fn, *args):
    """(host syncs of fn(*args) under torch.cuda.set_sync_debug_mode("warn"), the sorted file:line sites)."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    syncs = [w for w in rec if "called a synchronizing CUDA operation" in str(w.message)]
    return len(syncs), sorted({f"{os.path.relpath(w.filename, ROOT)}:{w.lineno}" for w in syncs})


def cuda_kernels(fn, *args):
    """(GPU kernels fn(*args) launches, every library's, and the sum of their durations in ms) from torch.profiler's
    CUDA activity, memcpy and memset records excluded.  The sum is device time spent in kernels, without the gaps
    between them."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(*args)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.lower().startswith(("memcpy", "memset"))]
    return len(kernels), sum(e.time_range.elapsed_us() for e in kernels) / 1e3
