#!/usr/bin/env python
"""Optimizer step benchmark: one optimizer's step over three parameter sets, and a training step with it (development
tool; bench.py measures the flagship workload).

Each step is captured (Device.capture) and replayed in windows of `--window-ms`, timed with CUDA events.  Parameters
are bf16 with f32 gradients, no master weights.  `--optimizer`: sgd (no momentum, as bench.py's configs 4 and 5), adam,
rmsprop (centered, momentum 0.9) or adagrad.  Parameter sets:
  - mlp:  config 4's MLP 1024-4096-4096-10 (6 tensors);
  - lstm: the README's 2-layer bidirectional LSTM at N = 256, I = H = 1024 (16 tensors: per layer and direction W_ih,
          W_hh, b_ih, b_hh);
  - many: 256 tensors of 4096 elements.
Reported per set, one JSON line each: us per optimizer step (median of the windows, and their min and max), kernels per
step (the captured graph's kernel count), and GB/s from the bytes the optimizer must move per element -- w read +
written (2 x 2 B), g read (4 B) and, except for plain SGD, the penalised gradient written back (4 B), and each f32
state array read + written (2 x 4 B) -- against the H100 SXM's 3.35 TB/s.  Then one captured training step of the mlp
set (batch 8192, MSE) with the optimizer and StepLR, in ms per step and kernels per step.  Card name, power limit and
the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/optim_bench.py [--optimizer adam] [--reps 7] [--window-ms 200]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, capture, setup, window  # noqa: E402

BYTES_PER_ELEM = {"sgd": 2 * 2 + 4, "adam": 2 * 2 + 2 * 4 + 4 * 4, "rmsprop": 2 * 2 + 2 * 4 + 6 * 4,
                  "adagrad": 2 * 2 + 2 * 4 + 2 * 4}


def make_opt(family, lr, **kw):
    from neuronika_b200 import optim
    if family == "sgd":
        return optim.StochasticGD.new(lr, **kw)
    if family == "adam":
        return optim.Adam.new(lr, **kw)
    if family == "rmsprop":
        return optim.RMSProp.new(lr, momentum=0.9, centered=True, **kw)
    return optim.Adagrad.new(lr, **kw)


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


def windows(launch, args):
    """(ms per launch of each of `args.reps` windows, median SM MHz)"""
    runs = [window(launch, args.window_ms, 1) for _ in range(args.reps)]
    return [ms for ms, _ in runs], float(np.nanmedian([mhz for _, mhz in runs]))


def optimizer_rows(nk, dev, args):
    rows = []
    for name in ("mlp", "lstm", "many"):
        rng = np.random.default_rng(0)
        ps = [nk.from_ndarray(dev, rng.uniform(-0.1, 0.1, s).astype(np.float32), nk.BF16).requires_grad(nk.F32)
              for s in shapes(name)]
        for p in ps:
            p.grad_array().copy_from(rng.normal(0, 1e-3, p.shape).astype(np.float32))
        opt = make_opt(args.optimizer, 1e-4)
        for p in ps:
            opt.register(p)
        graph = capture(dev, opt.step, 1 << 20)
        times, mhz = windows(graph.launch, args)
        elems = sum(int(np.prod(s)) for s in shapes(name))
        bpe = BYTES_PER_ELEM[args.optimizer]
        us = 1e3 * float(np.median(times))
        rows.append({"optimizer": args.optimizer, "set": name, "tensors": len(shapes(name)), "elements": elems,
                     "bytes_per_elem": bpe, "us_per_step": round(us, 2),
                     "us_min_max": [round(1e3 * min(times), 2), round(1e3 * max(times), 2)],
                     "kernels_per_step": graph.kernel_count, "GB_s": round(elems * bpe / (us * 1e-6) / 1e9, 1),
                     "share_of_3.35_TB_s": round(elems * bpe / (us * 1e-6) / 1e9 / DATASHEET["hbm_gbps"], 3),
                     "median_sm_mhz": mhz})
        graph.close()
    return rows


def training_row(nk, dev, args):
    from neuronika_b200 import nn
    from neuronika_b200.optim import lr_scheduler as S
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
    opt = make_opt(args.optimizer, 1e-4)
    for l in layers:
        for p in l.parameters():
            opt.register(p)
    sched = S.StepLR(opt, 100, 0.9)

    def step():
        opt.zero_grad()
        loss.forward()
        loss.backward(1.0)
        opt.step()
        sched.step()
    graph = capture(dev, step, 4 << 30)
    times, mhz = windows(graph.launch, args)
    row = {"optimizer": args.optimizer, "set": "mlp training step (batch 8192, MSE, StepLR)",
           "ms_per_step": round(float(np.median(times)), 4), "ms_min_max": [round(min(times), 4), round(max(times), 4)],
           "kernels_per_step": graph.kernel_count, "median_sm_mhz": mhz}
    graph.close()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--optimizer", default="adam", choices=sorted(BYTES_PER_ELEM))
    args = ap.parse_args()
    import neuronika_b200 as nk
    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    info = {"gpu": card["name"], "power_limit": card["power_limit_w"]}
    for row in optimizer_rows(nk, dev, args):
        print(json.dumps({**info, **row}), flush=True)
    print(json.dumps({**info, **training_row(nk, dev, args)}), flush=True)


if __name__ == "__main__":
    main()
