"""Timing helpers of the measurement scripts (tests/*_bench.py): the card a number was measured on, a device-event
window and alternated windows."""
import statistics
import subprocess

import torch


def card():
    """(device name, "power limit, max SM clock") of cuda:0, read from nvidia-smi ("unknown" when it cannot be read)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = "unknown"
    return torch.cuda.get_device_name(0), q


def window_ms(fn, iters):
    """Mean ms per call of `iters` calls of `fn`, between two device events, then a synchronise."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def alternate(fns: dict, reps: int, iters: int, warmup: int = 2) -> dict:
    """Median and spread (max - min) of `reps` windows of `iters` calls per function, after `warmup` calls of each; the
    order of the functions is reversed every other window, so a drift of the clock over a round does not favour
    whichever runs first."""
    for f in fns.values():   # warm-up: descriptor cache, module load
        window_ms(f, warmup)
    t = {k: [] for k in fns}
    for i in range(reps):
        for k in (list(fns) if i % 2 == 0 else list(fns)[::-1]):
            t[k].append(window_ms(fns[k], iters))
    return {k: round(statistics.median(v), 4) for k, v in t.items()} | {
        f"{k}_spread": round(max(v) - min(v), 4) for k, v in t.items()}
