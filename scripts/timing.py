"""The measurement protocol of the scripts/*_time.py scripts: the card a number was measured on, CUDA-event timings,
rounds of alternated variants, and the library's per-stage device times and launch counts.  Importing it puts the
repository root on sys.path, so that the scripts can import dss_b200 and tests.util when run from any directory."""
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dss_b200 import _lib  # noqa: E402


def card():
    """{"name", "power_limit", "max_sm_clock"} of the first GPU as nvidia-smi reports them ("700.00 W", "1980 MHz");
    the CUDA device name and "unknown" when nvidia-smi cannot be read."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def events_ms(fn, n):
    """ms per call of n back-to-back calls of fn between one pair of CUDA events, from an idle device (so the window
    holds the calls' host time too) to the end of the last call."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def median_ms(fn, warmup, iters):
    """The median of iters per-call CUDA-event times after warmup untimed calls (the upper middle one for an even
    iters)."""
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def alternate(variants, rounds, steps, warmup):
    """{name: callable} -> {name: [ms per call in each round]}.  Every variant is warmed up with warmup calls; then each
    of the rounds times steps calls of every variant in turn (events_ms), so that a drift of the clocks or of the
    host's load is shared by all the variants."""
    for fn in variants.values():
        events_ms(fn, warmup)
    ms = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            ms[k].append(events_ms(fn, steps))
    return ms


def spread(xs):
    """(median, min, max)"""
    return statistics.median(xs), min(xs), max(xs)


def paired(xs, ys):
    """The per-round differences ys - xs of two variants timed in the same rounds."""
    return [y - x for x, y in zip(xs, ys)]


def stage_ms(fn, steps, device):
    """{stage: device ms per call} of the library's profiled stages over steps calls of fn; profiling is off again
    afterwards."""
    _lib.profile_enable(True, device)
    _lib.profile_reset(device)
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    st = _lib.profile_read(device)
    _lib.profile_enable(False, device)
    return {k: ms / steps for k, (ms, _) in st.items()}


def launches(fn, device):
    """The library's kernel launches of one call of fn, counted after a first call that warms it up."""
    fn()
    torch.cuda.synchronize()
    before = _lib.launch_count(device)
    fn()
    return _lib.launch_count(device) - before
