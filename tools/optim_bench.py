#!/usr/bin/env python
"""Optimizer step benchmark: the default (per-parameter) Adam against the capturable (multi-tensor) Adam (development
tool; bench.py measures the flagship workload).

Both paths are captured (Device.capture) and replayed, in alternating windows of `--window-ms`, timed with CUDA events
(Device.timer_start / timer_stop).  Parameters are bf16 with f32 gradients, no master weights.  Parameter sets:
  - mlp:  config 4's MLP 1024-4096-4096-10 (6 tensors);
  - lstm: the README's 2-layer bidirectional LSTM at N = 256, I = H = 1024 (16 tensors: per layer and direction W_ih,
          W_hh, b_ih, b_hh);
  - many: 256 tensors of 4096 elements.
Reported per set, one JSON line each: us per optimizer step (median of the windows), kernels per step (the captured
graph's kernel count), and GB/s from the bytes Adam must move per element -- w read + written (2 x 2 B), g read and the
penalised gradient written back (2 x 4 B), exp_avg and exp_avg_sq read + written (4 x 4 B): 28 B -- against the H100
SXM's 3.35 TB/s.  Then one captured training step of the mlp set (batch 8192, MSE) with Adam + StepLR, default vs
capturable, in ms per step and kernels per step.  Card name and power limit are printed beside the numbers.

    python tools/optim_bench.py [--reps 7] [--window-ms 200]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBPS = 3.35
BYTES_PER_ELEM = 2 * 2 + 2 * 4 + 4 * 4


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # the numbers stand without it, but say so
        return {"gpu": "unknown (%s)" % e, "power_limit": "unknown"}


def shapes(name):
    if name == "mlp":
        dims = [1024, 4096, 4096, 10]
        return [s for i in range(3) for s in ((dims[i + 1], dims[i]), (dims[i + 1],))]
    if name == "lstm":
        h, out = 1024, []
        for layer in range(2):
            i = 1024 if layer == 0 else 2 * h
            for _ in range(2):
                out += [(4 * h, i), (4 * h, h), (4 * h,), (4 * h,)]
        return out
    return [(4096,)] * 256


def timed(dev, launch, window_ms):
    """ms per launch over a window of about window_ms"""
    dev.timer_start()
    launch()
    one = max(dev.timer_stop(), 1e-3)
    n = max(3, int(window_ms / one))
    dev.timer_start()
    for _ in range(n):
        launch()
    return dev.timer_stop() / n


def optimizer_rows(nk, dev, args):
    from neuronika_b200 import optim
    rows = []
    for name in ("mlp", "lstm", "many"):
        rng = np.random.default_rng(0)
        graphs = {}
        for mode in ("default", "capturable"):
            ps = [nk.from_ndarray(dev, rng.uniform(-0.1, 0.1, s).astype(np.float32), nk.BF16).requires_grad(nk.F32)
                  for s in shapes(name)]
            for p in ps:
                p.grad_array().copy_from(rng.normal(0, 1e-3, p.shape).astype(np.float32))
            opt = optim.Adam.new(1e-4, capturable=(mode == "capturable"))
            for p in ps:
                opt.register(p)
            opt.step()
            with dev.capture(1 << 20) as cap:
                opt.step()
            graphs[mode] = (cap.graph, ps, opt)
        times = {m: [] for m in graphs}
        for _ in range(args.reps):
            for m, (g, _, _) in graphs.items():
                times[m].append(timed(dev, g.launch, args.window_ms))
        elems = sum(int(np.prod(s)) for s in shapes(name))
        row = {"set": name, "tensors": len(shapes(name)), "elements": elems, "bytes_per_elem": BYTES_PER_ELEM}
        for m, (g, _, _) in graphs.items():
            us = 1e3 * float(np.median(times[m]))
            row[m] = {"us_per_step": round(us, 2), "kernels_per_step": g.kernel_count,
                      "GB_s": round(elems * BYTES_PER_ELEM / (us * 1e-6) / 1e9, 1),
                      "share_of_3.35_TB_s": round(elems * BYTES_PER_ELEM / (us * 1e-6) / (HBM_TBPS * 1e12), 3)}
        row["capturable_over_default"] = round(row["capturable"]["us_per_step"] / row["default"]["us_per_step"], 3)
        rows.append(row)
        for g, _, _ in graphs.values():
            g.close()
    return rows


def training_row(nk, dev, args):
    from neuronika_b200 import nn, optim
    from neuronika_b200.optim import lr_scheduler as S
    graphs = {}
    for mode in ("default", "capturable"):
        rng = np.random.default_rng(1)
        dims = [1024, 4096, 4096, 10]
        layers = [nn.Linear(dev, dims[i], dims[i + 1], dtype=nk.BF16, grad_dtype=nk.F32, rng=rng) for i in range(3)]
        x = nk.from_ndarray(dev, rng.uniform(-1, 1, (8192, 1024)).astype(np.float32), nk.BF16)
        t = nk.from_ndarray(dev, rng.uniform(0, 1, (8192, 10)).astype(np.float32), nk.BF16)
        h = x
        for i, l in enumerate(layers):
            h = l.forward(h)
            if i < 2:
                h = h.relu()
        loss = h.mse_loss(t)
        opt = optim.Adam.new(1e-4, capturable=(mode == "capturable"))
        for l in layers:
            for p in l.parameters():
                opt.register(p)
        sched = S.StepLR(opt, 100, 0.9)

        def step(loss=loss, opt=opt, sched=sched):
            opt.zero_grad()
            loss.forward()
            loss.backward(1.0)
            opt.step()
            sched.step()
        step()
        with dev.capture(4 << 30) as cap:
            step()
        graphs[mode] = (cap.graph, layers, loss, x, t)
    times = {m: [] for m in graphs}
    for _ in range(args.reps):
        for m, (g, *_rest) in graphs.items():
            times[m].append(timed(dev, g.launch, args.window_ms))
    row = {"set": "mlp training step (batch 8192, MSE, Adam + StepLR)"}
    for m, (g, *_rest) in graphs.items():
        row[m] = {"ms_per_step": round(float(np.median(times[m])), 4), "kernels_per_step": g.kernel_count}
    for g, *_rest in graphs.values():
        g.close()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--window-ms", type=float, default=200.0)
    args = ap.parse_args()
    import neuronika_b200 as nk
    dev = nk.Device(0)
    info = card()
    for row in optimizer_rows(nk, dev, args):
        print(json.dumps({**info, **row}), flush=True)
    print(json.dumps({**info, **training_row(nk, dev, args)}), flush=True)


if __name__ == "__main__":
    main()
