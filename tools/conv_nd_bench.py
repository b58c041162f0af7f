#!/usr/bin/env python
"""1-D / 3-D convolution layer benchmark (development tool; bench.py measures the flagship workload).

Three implementations of the same bf16 layer y = conv(pad(x), W) + b, on the same data, alternating window by window:
  node       variable.conv_layer: one graph node, the im2col + wgmma engine with the padding in the column gather
  cuda_core  the composed graph x.pad(..) -> W.convolution(..) + b: the CUDA-core gather kernels of nk_convnd_*
  cudnn      torch F.conv1d / F.conv3d in bf16 (cudnn.benchmark on; replicate padding through F.pad, as nn.Conv3d does)
each timed for the forward and for forward + backward (input, weight and bias all differentiable, bf16 gradients).
Shapes (FLOPs from the shapes, 2.N.Cout.L_out.Cin.prod(k) per product; forward = 1 product, backward = 2 more):
  conv1d      Conv1d 256 -> 256, k 3, zero pad 1, N 64, L 4096
  conv3d      Conv3d 64 -> 64, k 3, replicative pad 1, N 8, 32^3
  conv3d_stem Conv3d 3 -> 32, k 3, zero pad 1, N 8, 64^3 (K = 81: bounded by HBM, not by the tensor cores)
The column buffer of the node (bf16, N.Lp.Kp elements) is reported beside; the node's output is checked against
cuDNN's before timing.  Card name, power limit and the median SM clock during the timed windows (NVML) are printed with
the numbers.

    python tools/conv_nd_bench.py [--reps 3] [--window-ms 200]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, setup  # noqa: E402

# name: (N, Cin, Cout, sample extents, kernel, padding, mode)
CASES = {
    "conv1d": (64, 256, 256, (4096,), (3,), (1,), "zero"),
    "conv3d": (8, 64, 64, (32, 32, 32), (3, 3, 3), (1, 1, 1), "replicative"),
    "conv3d_stem": (8, 3, 32, (64, 64, 64), (3, 3, 3), (1, 1, 1), "zero"),
}


def case_fns(nk, dev, torch, n, cin, cout, sp, k, pad, mode):
    from neuronika_b200 import variable as V
    F = torch.nn.functional
    rng = np.random.default_rng(0)
    nsp = len(sp)
    bound = 1.0 / math.sqrt(cin * math.prod(k))
    xa = rng.uniform(-1, 1, (n, cin) + sp).astype(np.float32)
    wa = rng.uniform(-bound, bound, (cout, cin) + k).astype(np.float32)
    ba = rng.uniform(-bound, bound, (cout,) + (1,) * nsp).astype(np.float32)

    def params():
        return [nk.from_ndarray(dev, a, nk.BF16).requires_grad() for a in (xa, wa, ba)]

    x, w, b = params()
    y = V.conv_layer(x, w, b, pad, mode)
    xc, wc, bc = params()
    yc = wc.convolution(xc.pad(pad, 0.0, mode=mode), (1,) * nsp, (1,) * nsp, 1) + bc

    xt, wt, bt = (torch.tensor(a, device="cuda", dtype=torch.bfloat16, requires_grad=True) for a in (xa, wa, ba.ravel()))
    conv = F.conv1d if nsp == 1 else F.conv3d
    if mode == "zero":
        tfwd = lambda: conv(xt, wt, bt, padding=pad)
    else:
        widths = [p for p in reversed(pad) for _ in range(2)]
        tfwd = lambda: conv(F.pad(xt, widths, mode="replicate"), wt, bt)
    yt = tfwd()
    gt = torch.ones_like(yt)

    def tstep():
        tfwd().backward(gt)

    def node_step():
        y.forward()
        y.backward(1.0)

    def core_step():
        yc.forward()
        yc.backward(1.0)

    y.forward()
    got = torch.tensor(y.data(), device="cuda")
    want = yt.float()
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 2e-2, ("node vs cudnn", err)
    lo = (n * cout * yt[0, 0].numel())                      # N.Cout.L_out
    flops = 2 * lo * cin * math.prod(k)
    L = yt[0, 0].numel()
    cols = n * ((L + 7) // 8 * 8) * ((cin * math.prod(k) + 7) // 8 * 8) * 2
    fwd = {"node": y.forward, "cuda_core": yc.forward, "cudnn": tfwd}
    both = {"node": node_step, "cuda_core": core_step, "cudnn": tstep}
    return fwd, both, flops, cols, err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    torch.backends.cudnn.benchmark = True
    dev, card = setup(bf16_datasheet_tflops=DATASHEET["bf16_tflops"])
    for name in args.cases.split(","):
        n, cin, cout, sp, k, pad, mode = CASES[name]
        fwd, both, flops, cols, err = case_fns(nk, dev, torch, n, cin, cout, sp, k, pad, mode)
        for direction, fns, fl in (("forward", fwd, flops), ("forward+backward", both, 3 * flops)):
            ms, mhz = alternate(fns, args.window_ms, args.reps)
            tf = {key: round(fl / v / 1e9, 1) for key, v in ms.items()}
            print(json.dumps({
                "case": name, "direction": direction, "N": n, "cin": cin, "cout": cout, "extent": list(sp),
                "kernel": list(k), "padding": list(pad), "mode": mode, "gflop": round(fl / 1e9, 1),
                "column_buffer_mb": round(cols / 1e6, 1), "node_vs_cudnn_max_rel_err": round(err, 5),
                "ms": {key: round(v, 4) for key, v in ms.items()}, "tflops": tf,
                "node_vs_cuda_core": round(ms["cuda_core"] / ms["node"], 2),
                "node_vs_cudnn": round(ms["cudnn"] / ms["node"], 3),
                "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        del fwd, both
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
