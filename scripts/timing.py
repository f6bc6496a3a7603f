"""How the scripts under scripts/ take a time on the GPU: the one module that does.

* back to back (`back_to_back_us`): `warm` calls, a synchronise, then CUDA events around `n` calls of `fn`; µs per
  call, best of `reps` windows.  After the synchronise the first event is timestamped at once and the last one when the
  last command ends, so the window spans the same wall interval a host clock around the loop and a final synchronise
  would: for device-bound loops (commands queued faster than they run) and host-bound ones (the stepped route, whose
  Python loop waits on the GPU) alike.
* L2 flushed (`flushed_us`): before each call the 256 MiB `zero_()` bench.py writes before every timed step (more than
  the 50 MB L2 of an H100), CUDA events around the call alone; the per-call times, for the caller's median (or mean).
* alternating (`alternate_us`): a dict of variants timed back to back in turn, interleaved within every round so that
  a slow phase of the shared host hits all of them; every sample per variant.
* host call cost (`host_us`): the host clock around `n` calls after a warm-up — the issue cost of `command()` or the
  round trip of `command_host()`, the only thing a host clock times here.
* the card (`card`, `emit`): its name, power limit and max SM clock, which belong beside every absolute number.

Every measurement needs a CUDA device and raises without one; nothing falls back to a CPU timing."""
import functools
import json
import subprocess
import time

import torch


def _cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("timing needs a CUDA device")


def _window_us(fn, n):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def back_to_back_us(fn, n, warm=20, reps=5):
    """µs per call of `fn`, best of `reps` windows of `n` back-to-back calls after `warm` calls."""
    _cuda()
    for _ in range(warm):
        fn()
    return min(_window_us(fn, n) for _ in range(reps))


def alternate_us(variants, rounds, warm=20, reps=1):
    """{name: [µs per call, one sample per round]} for variants {name: (fn, n)}: in every round each variant in turn,
    `back_to_back_us(fn, n, warm, reps)`.  The warm-up comes before every turn: a variant's first calls after another
    one's run cold."""
    samples = {k: [] for k in variants}
    for _ in range(rounds):
        for k, (fn, n) in variants.items():
            samples[k].append(back_to_back_us(fn, n, warm, reps))
    return samples


@functools.cache
def _flush_buffer():
    return torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def flush_l2():
    """Enqueue bench.py's L2 flush: a 256 MiB zero_(), its buffer allocated once per process."""
    _cuda()
    _flush_buffer().zero_()


def flushed_us(fn, n, warm=5):
    """µs of each of `n` calls of `fn`, the L2 flushed before each one."""
    _cuda()
    for _ in range(warm):
        fn()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in evs:
        flush_l2()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) * 1e3 for a, b in evs]


def median(ts):
    return sorted(ts)[len(ts) // 2]


def host_us(fn, n, warm=20):
    """µs of host time per call of `fn`, over `n` calls after `warm` calls; no synchronise before or after, so that it
    also times calls on a controller whose resident grid never lets the device go idle."""
    _cuda()
    for _ in range(warm):
        fn()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t0) / n * 1e6


def card():
    """'name, power limit, max SM clock' of the first GPU; the device name alone where the query fails."""
    _cuda()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name()


def emit(out):
    """Print a script's one JSON line, with the card added."""
    print(json.dumps({"gpu": card(), **out}))
