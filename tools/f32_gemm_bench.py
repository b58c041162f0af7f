#!/usr/bin/env python
"""f32 GEMMs on the CUDA cores and the tensor cores (development tool; bench.py measures the flagship workload).

For every shape below, nk_gemm with f32 operands and an f32 C in each f32 mode (Device.f32_matmul: "ieee" = the SIMT
kernel, "tf32", "tf32x3"), beside torch.matmul in f32 with torch.backends.cuda.matmul.allow_tf32 off and on, on the same
GPU in the same process.  The variants alternate, one window each, `--reps` times; the median is reported as ms per
call and TFLOP/s (2 M N K over the time).  Shapes: NT / NN / TN at 4096^3 and the f32 MLP's forward GEMMs at batch 8192
(8192 x 1024 -> 4096, 8192 x 4096 -> 4096, 8192 x 4096 -> 10, all NT).

A separate torch.profiler pass per shape and mode splits the tf32 calls into the operand pack kernel and the GEMM
kernel: the pack's share of the call, and its bandwidth against the 3.35 TB/s HBM3 data-sheet figure (bytes = every
operand element read once and its packed copy written once, ceil4(K) or ceil4(3K) floats per row).

Then a captured f32 training step (zero_grad -> forward -> backward -> SGD) of the 1024-4096-4096-10 MLP (ReLU, softmax,
mse) at batch 8192, one graph per mode, replayed alternately: ms per step.

Card name, power limit and the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/f32_gemm_bench.py [--reps 3] [--window-ms 150] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gemm_sweep import Clock  # noqa: E402

SHAPES = [("NT", 4096, 4096, 4096), ("NN", 4096, 4096, 4096), ("TN", 4096, 4096, 4096),
          ("NT", 8192, 4096, 1024), ("NT", 8192, 4096, 4096), ("NT", 8192, 10, 4096)]
MODES = ("ieee", "tf32", "tf32x3")
HBM_BYTES_PER_S = 3.35e12


def timed(torch, fn, clock, window_ms):
    """ms per call over one window of back-to-back calls (after a short warm-up), and the median SM clock meanwhile"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    iters = int(min(2000, max(3, window_ms / ((time.perf_counter() - t0) * 1e3))))
    clock.armed.set()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    clock.armed.clear()
    return e0.elapsed_time(e1) / iters, clock.take()


def gemm_variants(nk, dev, torch, form, M, N, K):
    """{variant: callable} for one shape; our operands and torch's hold the same values"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(0)
    ta, tb = form[0] == "T", form[1] == "T"
    a = rng.uniform(-1, 1, (K, M) if ta else (M, K)).astype(np.float32)
    b = rng.uniform(-1, 1, (N, K) if tb else (K, N)).astype(np.float32)
    A, B, C = dev.from_ndarray(a), dev.from_ndarray(b), dev.zeros((M, N))
    tA, tB = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    opa, opb = (tA.t() if ta else tA), (tB.t() if tb else tB)

    def ours(mode):
        def run():
            dev.f32_matmul(mode)
            ops.gemm(A, B, C, trans_a=ta, trans_b=tb)
        return run

    def theirs(tf32):
        def run():
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.matmul(opa, opb)
        return run

    v = {m: ours(m) for m in MODES}
    v["torch_f32"] = theirs(False)
    v["torch_tf32"] = theirs(True)
    return v


def pack_share(torch, fn, M, N, K, mode, out_dir):
    """(pack ms, gemm ms, pack GB/s) per call from a torch.profiler pass over 10 calls"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
    pack = gemm = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "tf32_pack" in e.key:
            pack += t
        elif "tf32_gemm" in e.key:
            gemm += t
    pack, gemm = pack / 10e3, gemm / 10e3    # us total over 10 calls -> ms per call
    kp = K * (3 if mode == "tf32x3" else 1)
    ldp = (kp + 3) // 4 * 4
    bytes_ = 4 * (M + N) * (K + ldp)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, f"f32_gemm_{M}x{N}x{K}_{mode}.trace.json"))
    return pack, gemm, (bytes_ / (pack * 1e-3) / 1e9) if pack > 0 else float("nan")


def mlp_step(nk, dev, mode, batch=8192, sizes=(1024, 4096, 4096, 10)):
    """the captured f32 training step of the MLP in `mode` (captured after one eager warm-up step)"""
    rng = np.random.default_rng(1)
    layers = [nk.nn.Linear(dev, a, b, rng=rng) for a, b in zip(sizes[:-1], sizes[1:])]
    opt = nk.optim.StochasticGD.new(0.01)
    for l in layers:
        for p in l.parameters():
            opt.register(p)
    X = nk.from_ndarray(dev, rng.uniform(-1, 1, (batch, sizes[0])).astype(np.float32))
    Tt = nk.from_ndarray(dev, np.eye(sizes[-1], dtype=np.float32)[rng.integers(0, sizes[-1], batch)])

    def step():
        opt.zero_grad()
        h = X
        for i, l in enumerate(layers):
            h = l.forward(h)
            h = h.relu() if i < len(layers) - 1 else h.softmax(1)
        loss = h.mse_loss(Tt)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    dev.f32_matmul(mode)
    step()
    dev.synchronize()
    with dev.capture(6 << 30) as cap:
        step()
    dev.f32_matmul("ieee")
    return cap.graph, layers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=150.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="", help="directory for the profiler traces (none when empty)")
    args = ap.parse_args()
    import torch

    import neuronika_b200 as nk

    if args.out:
        os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()        # a created stream: the legacy default stream cannot be captured
    torch.cuda.set_stream(stream)
    dev = nk.Device(0, stream=stream.cuda_stream)
    clock = Clock(0)
    clock.start()
    card = clock.card()
    print(json.dumps({"card": card, "sm_count": dev.sm_count}), flush=True)
    for form, M, N, K in SHAPES:
        v = gemm_variants(nk, dev, torch, form, M, N, K)
        times = {k: [] for k in v}
        mhz = []
        for _ in range(args.reps):
            for name, fn in v.items():
                ms, m = timed(torch, fn, clock, args.window_ms)
                times[name].append(ms)
                mhz.append(m)
        flop = 2.0 * M * N * K
        row = {"form": form, "M": M, "N": N, "K": K, "card": card["name"], "power_limit_w": card["power_limit_w"],
               "sm_mhz_median": float(np.nanmedian(mhz))}
        for name, ts in times.items():
            ms = float(np.median(ts))
            row[name] = {"ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1)}
        for mode in ("tf32", "tf32x3"):
            pack, gemm, gbs = pack_share(torch, v[mode], M, N, K, mode, args.out)
            row[mode].update({"pack_ms": round(pack, 4), "gemm_kernel_ms": round(gemm, 4),
                              "pack_share": round(pack / (pack + gemm), 3) if pack + gemm > 0 else None,
                              "pack_gbs": round(gbs, 1), "pack_hbm_fraction": round(gbs * 1e9 / HBM_BYTES_PER_S, 3),
                              "gemm_kernel_tflops": round(flop / gemm / 1e9, 1) if gemm > 0 else None})
        row["tf32x3_over_simt"] = round(row["ieee"]["ms"] / row["tf32x3"]["ms"], 2)
        print(json.dumps(row), flush=True)
        del v
        torch.backends.cuda.matmul.allow_tf32 = False

    graphs = {m: mlp_step(nk, dev, m) for m in MODES}
    times = {m: [] for m in MODES}
    mhz = []
    for _ in range(args.reps):
        for m, (g, _) in graphs.items():
            ms, c = timed(torch, g.launch, clock, max(args.window_ms, 300.0))
            times[m].append(ms)
            mhz.append(c)
    row = {"mlp_step": "1024-4096-4096-10 f32, batch 8192, captured", "card": card["name"],
           "power_limit_w": card["power_limit_w"], "sm_mhz_median": float(np.nanmedian(mhz))}
    for m in MODES:
        row[m + "_ms"] = round(float(np.median(times[m])), 3)
    print(json.dumps(row), flush=True)
    for g, _ in graphs.values():
        g.close()
    clock.halt.set()


if __name__ == "__main__":
    main()
