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

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, kernel_ms, setup  # noqa: E402

SHAPES = [("NT", 4096, 4096, 4096), ("NN", 4096, 4096, 4096), ("TN", 4096, 4096, 4096),
          ("NT", 8192, 4096, 1024), ("NT", 8192, 4096, 4096), ("NT", 8192, 10, 4096)]
MODES = ("ieee", "tf32", "tf32x3")


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


def pack_share(fn, M, N, K, mode, out_dir):
    """(pack ms, gemm ms, pack GB/s) per call from a torch.profiler pass"""
    trace = os.path.join(out_dir, f"f32_gemm_{M}x{N}x{K}_{mode}.trace.json") if out_dir else None
    ms = kernel_ms(fn, {"pack": ("tf32_pack",), "gemm": ("tf32_gemm",)}, trace)
    pack, gemm = ms["pack"], ms["gemm"]
    kp = K * (3 if mode == "tf32x3" else 1)
    ldp = (kp + 3) // 4 * 4
    bytes_ = 4 * (M + N) * (K + ldp)
    return pack, gemm, (bytes_ / (pack * 1e-3) / 1e9) if pack > 0 else float("nan")


def mlp_step(nk, dev, mode, batch=8192, sizes=(1024, 4096, 4096, 10)):
    """the captured f32 training step of the MLP in `mode`"""
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
    graph = capture(dev, step, 6 << 30)
    dev.f32_matmul("ieee")
    return graph, layers


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
    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"], tf32_datasheet_tflops=DATASHEET["tf32_tflops"],
                      fp32_datasheet_tflops=DATASHEET["fp32_tflops"])
    for form, M, N, K in SHAPES:
        v = gemm_variants(nk, dev, torch, form, M, N, K)
        times, mhz = alternate(v, args.window_ms, args.reps)
        flop = 2.0 * M * N * K
        row = {"form": form, "M": M, "N": N, "K": K, "card": card["name"], "power_limit_w": card["power_limit_w"],
               "sm_mhz_median": mhz}
        for name, ms in times.items():
            row[name] = {"ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1)}
        for mode in ("tf32", "tf32x3"):
            pack, gemm, gbs = pack_share(v[mode], M, N, K, mode, args.out)
            row[mode].update({"pack_ms": round(pack, 4), "gemm_kernel_ms": round(gemm, 4),
                              "pack_share": round(pack / (pack + gemm), 3) if pack + gemm > 0 else None,
                              "pack_gbs": round(gbs, 1), "pack_hbm_fraction": round(gbs / DATASHEET["hbm_gbps"], 3),
                              "gemm_kernel_tflops": round(flop / gemm / 1e9, 1) if gemm > 0 else None})
        row["tf32x3_over_simt"] = round(row["ieee"]["ms"] / row["tf32x3"]["ms"], 2)
        print(json.dumps(row), flush=True)
        del v
        torch.backends.cuda.matmul.allow_tf32 = False

    graphs = {m: mlp_step(nk, dev, m) for m in MODES}
    times, mhz = alternate({m: g.launch for m, (g, _) in graphs.items()}, max(args.window_ms, 300.0), args.reps)
    row = {"mlp_step": "1024-4096-4096-10 f32, batch 8192, captured", "card": card["name"],
           "power_limit_w": card["power_limit_w"], "sm_mhz_median": mhz}
    for m in MODES:
        row[m + "_ms"] = round(times[m], 3)
    print(json.dumps(row), flush=True)
    for g, _ in graphs.values():
        g.close()


if __name__ == "__main__":
    main()
