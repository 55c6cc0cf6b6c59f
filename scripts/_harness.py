"""How the measurement scripts measure: the card that ran, the timers, and the reference camera.

Every script under scripts/ imports this module first (``import _harness``); when a script runs as
``python scripts/x.py``, scripts/ is sys.path[0], and the import puts the repository root on sys.path.

A time is only worth something with the card it was measured on, so each script prints ``card()`` first.
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# The reference camera (config.yml:1-3): intrinsics and frame height, width.
REFERENCE_K = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)
REFERENCE_HW = (1544, 2064)


def smi(fields, device=None):
    """nvidia-smi's ``--query-gpu=<fields>`` for the torch device (the current one if None).

    nvidia-smi numbers the cards its own way and ignores CUDA_VISIBLE_DEVICES, so its index 0 need not be torch's
    cuda:0; the card is selected by its UUID instead."""
    uuid = torch.cuda.get_device_properties(device).uuid
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", f"GPU-{uuid}"],
                          capture_output=True, text=True, check=True, timeout=60).stdout.strip()


def card(device=None):
    """One line naming the card that runs the measurement: name, power limit, maximum SM clock."""
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device: these scripts time the GPU and do not fall back to the CPU")
    try:
        return smi("name,power.limit,clocks.max.sm", device)
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(device)}, power limit not read: {e}"


def _event():
    return torch.cuda.Event(enable_timing=True)


def synced_ms(fn, reps, warmup):
    """CUDA-event ms of each of `reps` calls of `fn`, each timed alone: the next call starts after this one ends."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = _event(), _event()
    ts = []
    for _ in range(reps):
        start.record()
        fn()
        end.record()
        end.synchronize()
        ts.append(start.elapsed_time(end))
    return ts


def queued_ms(fn, reps, warmup):
    """CUDA-event ms of each of `reps` calls of `fn` queued back to back, with one wait after the last."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(_event(), _event()) for _ in range(reps)]
    for start, end in ev:
        start.record()
        fn()
        end.record()
    torch.cuda.synchronize()
    return [start.elapsed_time(end) for start, end in ev]


def wall_ms(fn, reps, warmup):
    """Host-clock ms of each of `reps` calls of `fn`, from a synchronised device to the end of its work."""
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def summary(ts):
    """Median, min and max of the times `ts` in ms, and their count, on one line."""
    ts = np.asarray(ts)
    return f"median {np.median(ts):9.3f} ms  min {ts.min():9.3f}  max {ts.max():9.3f}  (n={len(ts)})"
