"""What the measurement scripts under tools/ share: the card a number was measured on, CUDA-event timing and peak memory."""
import subprocess

import torch


def gpu_info():
    """(name, power limit, maximum SM clock) of GPU 0, as nvidia-smi reports them ("unknown" where it cannot)."""
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, clock = [s.strip() for s in q.split(",")]
    except (OSError, subprocess.SubprocessError, ValueError):
        power, clock = "unknown", "unknown"
    return name, power, clock


def time_ms(fn, seconds, warmup, iters=None, min_iters=1):
    """Mean ms per call of `fn` after `warmup` calls, from CUDA events around a batch of calls: `iters` calls when given, else
    as many as fill `seconds` by the time of one timed call (at least `min_iters`)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if iters is None:
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        iters = max(min_iters, int(seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_mib(fn):
    """The peak of the CUDA memory allocated while `fn` runs, above what was allocated before it, in MiB."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20
