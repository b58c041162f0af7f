"""The measuring shared by the development benchmarks in this directory (bench.py keeps its own timing).

Protocol, for every number these tools print:
  - Our kernels and torch's run on one created CUDA stream (setup()): the legacy default stream cannot be captured,
    and CUDA events recorded on that one stream time both.
  - window(fn, window_ms, reps): WARMUP = 3 calls (module loads, cuDNN's algorithm choice, first-use allocations) and
    a synchronise; one host-timed call then sizes a window of about `window_ms` of back-to-back calls, the count
    clamped to [MIN_ITERS, MAX_ITERS] = [1, 5000] (a call longer than the window still runs once; a call of a few
    microseconds does not run for minutes).  Then `reps` such windows between two CUDA events on the current stream.
    It returns the median ms per call over the windows and the median SM clock sampled (NVML) while they ran.
  - alternate(fns, window_ms, reps): the implementations under comparison take turns, one window each per round, so
    that a drifting clock or a neighbour's load falls on all of them alike.
  - The card's name, enforced power limit and maximum SM clock are read (NVML) in the same process as the timings and
    printed beside them.
  - Shares of peak divide by DATASHEET: NVIDIA's data-sheet figures, bounds that are never measured here.
"""
from __future__ import annotations

import json
import threading
import time

import numpy as np

WARMUP = 3
MIN_ITERS, MAX_ITERS = 1, 5000

# NVIDIA's data sheet for the H100 SXM (a card allowed up to 700 W): HBM3 bandwidth in GB/s, dense tensor-core
# (BF16, TF32) and CUDA-core (FP32) rates in TFLOP/s
DATASHEET = {"hbm_gbps": 3350.0, "bf16_tflops": 989.0, "tf32_tflops": 495.0, "fp32_tflops": 67.0}

_clock = None       # the Clock that setup() starts; window() arms it while its windows run


class Clock(threading.Thread):
    """median SM clock (NVML) while armed"""

    def __init__(self, index):
        super().__init__(daemon=True)
        import pynvml
        pynvml.nvmlInit()
        self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(index)
        self.samples, self.armed = [], threading.Event()

    def run(self):
        while True:
            if self.armed.is_set():
                self.samples.append(int(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM)))
            time.sleep(0.002)

    def take(self):
        s, self.samples = self.samples, []
        return float(np.median(s)) if s else float("nan")

    def card(self):
        nv, h = self.nv, self.h
        name = nv.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                "sm_max_mhz": int(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))}


def setup(**header):
    """(Device on a created stream that torch also uses, card record); starts the Clock and prints the header line:
    card, SM count and `header` (the data-sheet bounds the tool divides by)"""
    global _clock
    import torch

    import neuronika_b200 as nk
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    dev = nk.Device(0, stream=stream.cuda_stream)
    _clock = Clock(0)
    _clock.start()
    card = _clock.card()
    print(json.dumps({"card": card, "sm_count": dev.sm_count, **header}), flush=True)
    return dev, card


def window(fn, window_ms, reps):
    """(median ms per call over `reps` windows of back-to-back calls, each about `window_ms` long; median SM MHz)"""
    import torch
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    iters = int(min(MAX_ITERS, max(MIN_ITERS, window_ms / ((time.perf_counter() - t0) * 1e3))))
    _clock.armed.set()
    per = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / iters)
    _clock.armed.clear()
    return float(np.median(per)), _clock.take()


def alternate(fns, window_ms, reps):
    """({name: median ms per call}, median SM MHz) over `reps` rounds, one window per function per round"""
    res, mhz = {k: [] for k in fns}, []
    for _ in range(reps):
        for k, fn in fns.items():
            ms, m = window(fn, window_ms, 1)
            res[k].append(ms)
            mhz.append(m)
    return {k: float(np.median(v)) for k, v in res.items()}, float(np.nanmedian(mhz))


def capture(dev, step, arena_bytes):
    """the captured graph of `step`, recorded with an arena of `arena_bytes` after two eager steps (first-use
    allocations cannot be captured) and a synchronise"""
    step()
    step()
    dev.synchronize()
    with dev.capture(arena_bytes) as cap:
        step()
    return cap.graph


def kernel_ms(fn, groups, trace=None):
    """{group: ms per call} of the kernels whose names contain one of the group's substrings (the first group that
    matches takes a kernel; copies and memsets count in none), from a torch.profiler pass over 10 calls after the
    warm-up; `trace`: a path for the chrome trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
    if trace:
        prof.export_chrome_trace(trace)
    out = dict.fromkeys(groups, 0.0)
    for e in prof.key_averages():
        if "Memcpy" in e.key or "Memset" in e.key:
            continue
        hit = next((g for g, keys in groups.items() if any(k in e.key for k in keys)), None)
        if hit is not None:
            out[hit] += e.device_time_total / 10e3     # us over 10 calls -> ms per call
    return out
