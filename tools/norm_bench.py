#!/usr/bin/env python
"""Normalization benchmark (development tool; bench.py measures the flagship workload).

For each case, csrc/nk_norm.cu against torch CUDA (cuDNN batch norm, torch's native layer norm) on the same tensors in
the same process, the two alternating window by window, timed with CUDA events:
  forward           ours: nk_batch_norm_fwd in training mode (running statistics updated) / nk_layer_norm_fwd;
                    torch: F.batch_norm(training=True) / F.layer_norm;
  forward+backward  the forward, then ours: nk_*_norm_bwd writing dx, dw and db (beta 0); torch: torch.autograd.grad
                    of a fresh forward for x, weight and bias.
Bytes are the least the algorithm moves: the batch-norm forward reads x twice (statistics, then apply: these maps do not
fit the 50 MB L2) and writes y; its backward reads g and x twice and writes dx; the layer-norm forward reads x once and
writes y (a row fits on chip); its backward reads g and x once and writes dx.  GB/s are reported beside the 3.35 TB/s
HBM3 data-sheet bound of the H100 SXM.  Card name, power limit and the median SM clock during the timed windows (NVML)
are printed beside the numbers.

    python tools/norm_bench.py [--reps 5] [--window-ms 200] [--only bn2d_cfg5_c32]
    python tools/norm_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, setup  # noqa: E402

# name: (kind, shape, dtypes); layer norm normalizes the last dim
CASES = {
    "bn2d_cfg5_c32": ("bn", (4096, 32, 32, 32), ("bf16", "f32")),
    "bn2d_cfg5_c64": ("bn", (4096, 64, 32, 32), ("bf16", "f32")),
    "bn2d_resnet_56x56": ("bn", (256, 64, 56, 56), ("bf16",)),
    "bn1d_8192x4096": ("bn", (8192, 4096), ("bf16", "f32")),
    "ln_8192x1024": ("ln", (8192, 1024), ("bf16", "f32")),
    "ln_4096x4096": ("ln", (4096, 4096), ("bf16", "f32")),
    "ln_32768x768": ("ln", (32768, 768), ("bf16", "f32")),
}


def traffic(kind, shape, esize):
    """(forward bytes, forward+backward bytes) from the shapes"""
    n = int(np.prod(shape))
    fwd = (3 if kind == "bn" else 2) * n * esize
    bwd = (5 if kind == "bn" else 3) * n * esize
    return fwd, fwd + bwd


def run_case(dev, card, name, dtype, reps, window_ms):
    import torch
    import torch.nn.functional as F

    import neuronika_b200 as nk
    from neuronika_b200 import ops
    kind, shape, _ = CASES[name]
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float32
    ndt = nk.BF16 if dtype == "bf16" else nk.F32
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, generator=gen, device="cuda", dtype=tdt)
    g = torch.randn(shape, generator=gen, device="cuda", dtype=tdt)
    c = shape[1] if kind == "bn" else shape[-1]
    # ours takes w and b in x's dtype; cuDNN's batch norm takes a bf16 input with f32 parameters
    pdt = torch.float32 if kind == "bn" else tdt
    w = torch.ones(c, device="cuda", dtype=pdt, requires_grad=True)
    b = torch.zeros(c, device="cuda", dtype=pdt, requires_grad=True)
    wrap = lambda t, dt=ndt: nk.CuArray(dev, tuple(t.shape), dt, ptr=t.data_ptr(), owner=t)
    X, G = wrap(x), wrap(g)
    W, B = dev.full((c,), 1.0, ndt), dev.zeros((c,), ndt)
    Y = dev.zeros(shape, ndt)
    DX, DW, DB = dev.zeros(shape, ndt), dev.zeros((c,), ndt), dev.zeros((c,), ndt)
    if kind == "bn":
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        RM, RV = dev.zeros((c,), nk.F32), dev.full((c,), 1.0, nk.F32)
        SM, SR = dev.zeros((c,), nk.F32), dev.zeros((c,), nk.F32)

        def ours_f():
            ops.batch_norm(X, W, B, RM, RV, True, out=Y, save_mean=SM, save_rstd=SR)

        def ours_fb():
            ours_f()
            ops.batch_norm_bwd(G, X, SM, SR, W, DX, DW, DB, True)

        torch_f = lambda: F.batch_norm(x, rm, rv, w.detach(), b.detach(), True)

        def torch_fb():
            xr = x.detach().requires_grad_(True)
            torch.autograd.grad(F.batch_norm(xr, rm, rv, w, b, True), (xr, w, b), g)
    else:
        cols = shape[-1]
        SM, SR = dev.zeros((shape[0],), nk.F32), dev.zeros((shape[0],), nk.F32)

        def ours_f():
            ops.layer_norm(X, cols, W, B, out=Y, save_mean=SM, save_rstd=SR)

        def ours_fb():
            ours_f()
            ops.layer_norm_bwd(G, X, cols, SM, SR, W, DX, DW, DB)

        torch_f = lambda: F.layer_norm(x, (cols,), w.detach(), b.detach())

        def torch_fb():
            xr = x.detach().requires_grad_(True)
            torch.autograd.grad(F.layer_norm(xr, (cols,), w, b), (xr, w, b), g)

    fns = {"ours_fwd": ours_f, "torch_fwd": torch_f, "ours_fwdbwd": ours_fb, "torch_fwdbwd": torch_fb}
    med, mhz = alternate(fns, window_ms, reps)
    fb, fbb = traffic(kind, shape, 2 if dtype == "bf16" else 4)
    return {"case": name, "dtype": dtype, "shape": list(shape),
            "ours_fwd_us": med["ours_fwd"] * 1e3, "torch_fwd_us": med["torch_fwd"] * 1e3,
            "ours_fwd_GBps": fb / med["ours_fwd"] / 1e6, "torch_fwd_GBps": fb / med["torch_fwd"] / 1e6,
            "ours_fwdbwd_us": med["ours_fwdbwd"] * 1e3, "torch_fwdbwd_us": med["torch_fwdbwd"] * 1e3,
            "ours_fwdbwd_GBps": fbb / med["ours_fwdbwd"] / 1e6,
            "torch_fwdbwd_GBps": fbb / med["torch_fwdbwd"] / 1e6,
            "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--only", default=None)
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args()
    names = [a.only] if a.only else list(CASES)
    if a.dry_run:
        for n in names:
            kind, shape, dts = CASES[n]
            for d in dts:
                print(n, d, "bytes fwd / fwd+bwd:", traffic(kind, shape, 2 if d == "bf16" else 4))
        return
    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for n in names:
        for d in CASES[n][2]:
            r = run_case(dev, card, n, d, a.reps, a.window_ms)
            print(json.dumps(r))
            print("  %-20s %-4s fwd ours %8.1f us %6.0f GB/s (%2.0f %%) | torch %8.1f us | %4.2fx    fwd+bwd ours %8.1f us "
                  "%6.0f GB/s (%2.0f %%) | torch %8.1f us | %4.2fx" % (
                      n, d, r["ours_fwd_us"], r["ours_fwd_GBps"], 100 * r["ours_fwd_GBps"] / DATASHEET["hbm_gbps"],
                      r["torch_fwd_us"], r["torch_fwd_us"] / r["ours_fwd_us"], r["ours_fwdbwd_us"],
                      r["ours_fwdbwd_GBps"], 100 * r["ours_fwdbwd_GBps"] / DATASHEET["hbm_gbps"], r["torch_fwdbwd_us"],
                      r["torch_fwdbwd_us"] / r["ours_fwdbwd_us"]), flush=True)


if __name__ == "__main__":
    main()
