#!/usr/bin/env python
"""f32 convolutions on the CUDA cores and the tensor cores (development tool; bench.py measures the flagship workload).

For every shape below, the convolution with f32 operands in each f32 convolution mode (Device.f32_conv: "ieee" = the
direct CUDA-core kernels, "tf32", "tf32x3" = the im2col engine of csrc/nk_conv_tf32.cu), beside torch's F.conv1d/2d/3d
in f32 with torch.backends.cudnn.allow_tf32 off and on (cudnn.benchmark on), on the same GPU in the same process.  Two
passes per shape: the forward alone, and forward + backward with the input, the weight and the bias differentiable (dX,
dW and db).  The variants alternate, one window each, `--reps` times; the median is reported as ms per call and
TFLOP/s (2 N Cout L K per product: one for the forward, three for forward + backward).  The 2-D rows run the 2-D entry
points on an input padded once beforehand (nn.Conv2d pads through its own graph node); the 1-D / 3-D rows run the
convolution layers (nk_conv_layer_nd_*) with the padding folded into the gather; torch pads inside its convolution.

Shapes: config 5's two Conv2d layers (3->32 and 32->64, k3, pad 1, 32x32, N 4096), the config 3 stem (3->64 k3 p0,
224x224, N 64), Conv1d 256->256 (k3, zero pad 1, N 64, L 4096) and Conv3d 64->64 (k3, replicative pad 1, N 8, 32^3).
The ieee path takes up to seconds per call at these sizes: each window runs at least one call.

A separate torch.profiler pass per shape and tf32 mode splits a forward + backward call into the gathers and packs
(tf32_im2col_kernel, tf32_pack_kernel), the GEMM (tf32_gemm_kernel) and the rest (col2im, the dW reduction, db).

Then a captured f32 training step of config 5's ConvNet (Conv2d 3->32 p1, ReLU, Conv2d 32->64 p1, ReLU, Linear
65536->10, softmax, mse, SGD; batch 4096; f32_matmul stays "ieee"), one graph per convolution mode, each captured,
replayed for a window and released in turn: ms per step.

Card name, power limit and the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/f32_conv_bench.py [--reps 3] [--window-ms 300] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, kernel_ms, setup, window  # noqa: E402

MODES = ("ieee", "tf32", "tf32x3")
# name: (x shape, Cout, kernel, padding, padding mode)
SHAPES = {
    "config5_conv1 3->32 k3 p1 32x32 N4096": ((4096, 3, 32, 32), 32, (3, 3), (1, 1), "zero"),
    "config5_conv2 32->64 k3 p1 32x32 N4096": ((4096, 32, 32, 32), 64, (3, 3), (1, 1), "zero"),
    "config3_stem 3->64 k3 p0 224x224 N64": ((64, 3, 224, 224), 64, (3, 3), (0, 0), "zero"),
    "conv1d 256->256 k3 zero-pad1 L4096 N64": ((64, 256, 4096), 256, (3,), (1,), "zero"),
    "conv3d 64->64 k3 replicative-pad1 32^3 N8": ((8, 64, 32, 32, 32), 64, (3, 3, 3), (1, 1, 1), "replicative"),
}
TORCH_PAD = {"zero": "zeros", "replicative": "replicate"}
# kernel groups of the profiler split ("" takes every other kernel)
SPLIT = {"gather_pack": ("tf32_im2col", "tf32_pack"), "gemm": ("tf32_gemm",), "other": ("",)}


def variants(nk, dev, torch, xs, cout, k, pad, pmode):
    """({variant: forward callable}, {variant: forward + backward callable}, flop of one product); our operands and
    torch's hold the same values"""
    import torch.nn.functional as F
    from neuronika_b200 import ops
    nsp = len(k)
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, xs).astype(np.float32)
    w = (rng.uniform(-1, 1, (cout, xs[1]) + k) / math.sqrt(xs[1] * math.prod(k))).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, cout).astype(np.float32)
    out = tuple(s + 2 * p - kk + 1 for s, p, kk in zip(xs[2:], pad, k))
    L, K = math.prod(out), xs[1] * math.prod(k)
    flop = 2.0 * xs[0] * cout * L * K
    g = rng.uniform(-1, 1, (xs[0], cout) + out).astype(np.float32)
    W, G = dev.from_ndarray(w), dev.from_ndarray(g)
    if nsp == 2:
        xp = np.pad(x, [(0, 0), (0, 0)] + [(p, p) for p in pad])
        X, B = dev.from_ndarray(xp), dev.from_ndarray(b.reshape(cout, 1, 1))
        Y, DX, DW, DB = dev.zeros(g.shape), dev.zeros(xp.shape), dev.zeros(w.shape), dev.zeros((cout, 1, 1))

        def fwd():
            ops.conv2d(X, W, bias=B, out=Y)

        def bwd():
            ops.conv2d_bwd_input(DX, G, W, beta=0.0)
            ops.conv2d_bwd_kernel(DW, G, X, beta=0.0, dbias=DB)
    else:
        X, B = dev.from_ndarray(x), dev.from_ndarray(b)
        Y, DX, DW, DB = dev.zeros(g.shape), dev.zeros(xs), dev.zeros(w.shape), dev.zeros((cout,))
        mc = "constant" if pmode == "zero" else pmode

        def fwd():
            ops.conv_layer_nd(X, W, pad, mc, 0.0, bias=B, out=Y)

        def bwd():
            ops.conv_layer_nd_bwd_input(DX, G, W, pad, mc, beta=0.0)
            ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, mc, 0.0, beta=0.0, dbias=DB)

    tx = torch.from_numpy(x).cuda().requires_grad_(True)
    tw = torch.from_numpy(w).cuda().requires_grad_(True)
    tb = torch.from_numpy(b).cuda().requires_grad_(True)
    tg = torch.from_numpy(g).cuda()
    conv = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}[nsp]

    def t_fwd():
        if pmode == "zero":
            return conv(tx, tw, tb, padding=pad)
        return conv(F.pad(tx, [p for q in reversed(pad) for p in (q, q)], mode=TORCH_PAD[pmode]), tw, tb)

    def ours(mode, both):
        def run():
            dev.f32_conv(mode)
            fwd()
            if both:
                bwd()
        return run

    def theirs(tf32, both):
        def run():
            torch.backends.cudnn.allow_tf32 = tf32
            if both:
                torch.autograd.grad(t_fwd(), (tx, tw, tb), tg)
            else:
                with torch.no_grad():
                    t_fwd()
        return run

    vf, vb = {}, {}
    for both, v in ((False, vf), (True, vb)):
        for m in MODES:
            v[m] = ours(m, both)
        v["torch_f32"] = theirs(False, both)
        v["torch_tf32"] = theirs(True, both)
    return vf, vb, flop


def convnet_step(nk, dev, mode, batch=4096):
    """config 5's ConvNet in f32, its training step captured in `mode`"""
    rng = np.random.default_rng(1)
    c1 = nk.nn.Conv2d(dev, 3, 32, (3, 3), padding=(1, 1), rng=rng)
    c2 = nk.nn.Conv2d(dev, 32, 64, (3, 3), padding=(1, 1), rng=rng)
    head = nk.nn.Linear(dev, 64 * 32 * 32, 10, rng=rng)
    opt = nk.optim.StochasticGD.new(0.01)
    for p in c1.parameters() + c2.parameters() + head.parameters():
        opt.register(p)
    X = nk.from_ndarray(dev, rng.uniform(-1, 1, (batch, 3, 32, 32)).astype(np.float32))
    Tt = nk.from_ndarray(dev, np.eye(10, dtype=np.float32)[rng.integers(0, 10, batch)])

    def step():
        opt.zero_grad()
        h = c2.forward(c1.forward(X).relu()).relu()
        loss = head.forward(h.flatten()).softmax(1).mse_loss(Tt)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    dev.f32_conv(mode)
    graph = capture(dev, step, 24 << 30)
    kern = dev.last_conv_kernel
    dev.f32_conv("ieee")
    return graph, kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="", help="directory for the profiler traces (none when empty)")
    args = ap.parse_args()
    import torch

    import neuronika_b200 as nk

    if args.out:
        os.makedirs(args.out, exist_ok=True)
    torch.backends.cudnn.benchmark = True
    dev, card = setup(tf32_datasheet_tflops=DATASHEET["tf32_tflops"], fp32_datasheet_tflops=DATASHEET["fp32_tflops"])
    for name, (xs, cout, k, pad, pmode) in SHAPES.items():
        vf, vb, flop = variants(nk, dev, torch, xs, cout, k, pad, pmode)
        for what, v, products in (("fwd", vf, 1), ("fwd+bwd", vb, 3)):
            times, mhz = alternate(v, args.window_ms, args.reps)
            row = {"shape": name, "pass": what, "card": card["name"], "power_limit_w": card["power_limit_w"],
                   "sm_mhz_median": mhz}
            for key, ms in times.items():
                row[key] = {"ms": round(ms, 4), "tflops": round(products * flop / ms / 1e9, 2)}
            if what == "fwd+bwd":
                for mode in ("tf32", "tf32x3"):
                    trace = f"f32_conv_{name.split()[0]}_{mode}.trace.json"
                    sp = kernel_ms(v[mode], SPLIT, os.path.join(args.out, trace) if args.out else None)
                    total = sum(sp.values())
                    row[mode].update({k2 + "_ms": round(t, 4) for k2, t in sp.items()})
                    row[mode]["gather_pack_share"] = round(sp["gather_pack"] / total, 3) if total > 0 else None
                row["tf32_speedup_over_ieee"] = round(row["ieee"]["ms"] / row["tf32"]["ms"], 1)
            print(json.dumps(row), flush=True)
        del vf, vb
        torch.backends.cudnn.allow_tf32 = True
        torch.cuda.empty_cache()

    # one captured graph (and its arena) alive at a time: each mode is captured, timed and released in turn
    times = {m: [] for m in MODES}
    kern = {}
    mhz = []
    for _ in range(args.reps):
        for m in MODES:
            g, kern[m] = convnet_step(nk, dev, m)
            ms, c = window(g.launch, max(args.window_ms, 300.0), 1)
            g.close()
            times[m].append(ms)
            mhz.append(c)
    row = {"convnet_step": "config 5 ConvNet f32, batch 4096, captured", "card": card["name"],
           "power_limit_w": card["power_limit_w"], "sm_mhz_median": float(np.nanmedian(mhz))}
    for m in MODES:
        row[m + "_ms"] = round(float(np.median(times[m])), 3)
        row[m + "_conv_kernel"] = kern[m]
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
