"""What the measurement scripts in tools/ share: the repository root on sys.path (on import), the device, the card's identity
and the two clocks.  A time is only worth something with the card's name and power limit read in the same run, so every
script that prints a time prints gpu_identity beside it."""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def cuda_device(tool):
    assert torch.cuda.is_available(), "tools/%s needs a CUDA device; there is no CPU fallback" % tool
    return torch.device("cuda", 0)


def gpu_identity(dev):
    """(torch's name of the card, nvidia-smi's "name, power limit" line, nvidia-smi's (name, power limit)).  The query only
    reads; where nvidia-smi cannot run, the line says why and the pair is None."""
    name = torch.cuda.get_device_name(dev)
    try:
        q = ["nvidia-smi", "-i", str(torch.device(dev).index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"]
        smi = subprocess.run(q, capture_output=True, text=True, timeout=20, check=True).stdout.strip()
    except Exception as exc:
        return name, "nvidia-smi unavailable: %s" % exc, None
    fields = tuple(s.strip() for s in smi.split(","))
    return name, smi, fields if len(fields) == 2 else None


def _chain(ev, first, then):
    ev[0].record()
    out = [first()]
    for i, fn in enumerate(then):
        ev[i + 1].record()
        out.append(fn(out[-1]))
    ev[-1].record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in zip(ev, ev[1:])], out


_STAGE_EVENTS = []


def stages_ms(first, *then):
    """([ms of each stage], [result of each stage]) of first() and then each later stage called with the result before it.
    One CUDA event on the current stream between consecutive stages and one synchronise at the end, so a stage queued
    behind a running one is timed from when its work starts on the device.  Every result is held until the end.  The events
    are made once and reused: an event is created at its first record(), and after a stage that ends in a read-back that
    creation would fall inside the next bracket."""
    _STAGE_EVENTS.extend(torch.cuda.Event(enable_timing=True) for _ in range(len(then) + 2 - len(_STAGE_EVENTS)))
    return _chain(_STAGE_EVENTS[:len(then) + 2], first, then)


def event_ms(fn):
    """(ms, result) of one call of fn, bracketed by two new CUDA events on the current stream and a synchronise."""
    (ms,), (out,) = _chain([torch.cuda.Event(enable_timing=True) for _ in range(2)], fn, ())
    return ms, out


def host_ms(fn):
    """(ms, result) of one call of fn on the host clock, with the device synchronised before and after: the whole call,
    host work and copies included."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def alternate(variants, reps, warmup=1, clock=event_ms):
    """Times {name: fn}: `warmup` rounds whose times are dropped, then `reps` rounds, each round calling every variant once in
    turn so that they all see the same clocks.  Returns {name: [ms of each timed call]}.  Results are dropped as they come:
    held across calls, pinned host buffers would make the next call allocate afresh."""
    ms = {k: [] for k in variants}
    for r in range(warmup + reps):
        for k, fn in variants.items():
            t, _ = clock(fn)
            if r >= warmup:
                ms[k].append(t)
    return ms
