#!/usr/bin/env python
"""Pooling benchmark (development tool; bench.py measures the flagship workload).

For each case below, in bf16 and in f32, csrc/nk_pool.cu against torch CUDA on the same tensors in the same process,
the two alternating window by window:
  forward           ours: nk_*_pool_nd_fwd (the max pool writing its int32 indices, as in training);
                    torch: F.max_pool*d(return_indices=True) / F.avg_pool*d / F.adaptive_avg_pool*d;
  forward+backward  the forward, then ours: nk_*_pool_nd_bwd with beta 0; torch: torch.autograd.grad of a fresh
                    forward (the same two kernels).
Bytes are counted from the shapes: the forward reads x and writes y (plus the indices, 4 bytes per output for ours,
8 for torch's int64); the backward reads g (and the indices) and writes dx.  GB/s are reported beside the 3.35 TB/s
HBM3 data-sheet bound of the H100 SXM.

Then one captured training step of config 5's ConvNet (bench.py: Conv2d 3->32 p1 -> ReLU -> Conv2d 32->64 p1 -> ReLU
-> Linear 65536->10 -> softmax -> mse, batch 4096, bf16 data, f32 gradients, SGD) beside the same network with a
MaxPool2d(2) after each ReLU (Linear 4096->10): ms per step and captured kernels.  Card name, power limit and the
median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/pool_bench.py [--reps 5] [--window-ms 200]
    python tools/pool_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402

# name: (kind, input shape, kernel, stride, padding)  (adaptive: kernel = output size)
CASES = {
    "maxpool2d_k3s2p1_resnet_stem": ("max", (256, 64, 112, 112), (3, 3), (2, 2), (1, 1)),
    "maxpool2d_k2": ("max", (4096, 32, 32, 32), (2, 2), (2, 2), (0, 0)),
    "maxpool1d_k3s2p1": ("max", (64, 256, 4096), (3,), (2,), (1,)),
    "avgpool3d_k2": ("avg", (8, 64, 32, 32, 32), (2, 2, 2), (2, 2, 2), (0, 0, 0)),
    "adaptiveavgpool2d_1_7x7": ("adaptive", (256, 2048, 7, 7), (1, 1), None, None),
    "adaptiveavgpool2d_1_32x32": ("adaptive", (4096, 64, 32, 32), (1, 1), None, None),
}


def out_shape(kind, shape, k, s, p):
    if kind == "adaptive":
        return shape[:2] + tuple(k)
    return shape[:2] + tuple((L + 2 * pp - kk) // ss + 1 for L, kk, ss, pp in zip(shape[2:], k, s, p))


def traffic(kind, shape, oshape, esize):
    """{impl: (forward bytes, backward bytes)} from the shapes"""
    n, m = int(np.prod(shape)), int(np.prod(oshape))
    out = {}
    for impl, isz in (("ours", 4), ("torch", 8)):
        ib = m * isz if kind == "max" else 0
        out[impl] = ((n + m) * esize + ib, (n + m) * esize + ib)
    return out


def case(nk, dev, torch, kind, shape, k, s, p, dt):
    """{impl: forward fn}, {impl: forward + backward fn} on the same tensors"""
    import torch.nn.functional as F

    from neuronika_b200 import ops
    ndt = nk.BF16 if dt == torch.bfloat16 else nk.F32
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, device="cuda", generator=gen).to(dt)
    oshape = out_shape(kind, shape, k, s, p)
    y = torch.empty(oshape, device="cuda", dtype=dt)
    g = torch.randn(oshape, device="cuda", generator=gen).to(dt)
    dx = torch.empty_like(x)
    wrap = lambda a, d: nk.CuArray(dev, tuple(a.shape), d, ptr=a.data_ptr(), owner=a)
    xv, yv, gv, dxv = wrap(x, ndt), wrap(y, ndt), wrap(g, ndt), wrap(dx, ndt)
    xr = x.detach().requires_grad_(True)
    nsp = len(shape) - 2
    if kind == "max":
        idx = torch.empty(oshape, device="cuda", dtype=torch.int32)
        iv = wrap(idx, nk.F32)
        tf = {1: F.max_pool1d, 2: F.max_pool2d, 3: F.max_pool3d}[nsp]
        ours_f = lambda: ops.max_pool_nd(xv, k, s, p, idx=iv, out=yv)
        ours_b = lambda: ops.max_pool_nd_bwd(dxv, gv, iv, k, s, p, beta=0.0)
        torch_f = lambda: tf(x, k, s, p, return_indices=True)
        torch_fb = lambda: torch.autograd.grad(tf(xr, k, s, p, return_indices=True)[0], xr, g)
    elif kind == "avg":
        tf = {1: F.avg_pool1d, 2: F.avg_pool2d, 3: F.avg_pool3d}[nsp]
        ours_f = lambda: ops.avg_pool_nd(xv, k, s, p, out=yv)
        ours_b = lambda: ops.avg_pool_nd_bwd(dxv, gv, k, s, p, beta=0.0)
        torch_f = lambda: tf(x, k, s, p)
        torch_fb = lambda: torch.autograd.grad(tf(xr, k, s, p), xr, g)
    else:
        tf = {1: F.adaptive_avg_pool1d, 2: F.adaptive_avg_pool2d, 3: F.adaptive_avg_pool3d}[nsp]
        ours_f = lambda: ops.adaptive_avg_pool_nd(xv, k, out=yv)
        ours_b = lambda: ops.adaptive_avg_pool_nd_bwd(dxv, gv, beta=0.0)
        torch_f = lambda: tf(x, k)
        torch_fb = lambda: torch.autograd.grad(tf(xr, k), xr, g)
    # the two agree on the forward
    ours_f()
    dev.synchronize()
    ref = torch_f()
    ref = ref[0] if isinstance(ref, tuple) else ref
    assert torch.allclose(y.float(), ref.float(), rtol=1e-2, atol=1e-2), kind
    fwd = {"ours": ours_f, "torch": torch_f}
    fb = {"ours": lambda: (ours_f(), ours_b()), "torch": torch_fb}
    return fwd, fb, oshape


def convnet_step(nk, dev, pooled, batch=4096):
    """config 5's ConvNet step, or the same network with MaxPool2d(2) after each ReLU, captured"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    feat = 64 * 8 * 8 if pooled else 65536
    shapes = [(32, 3, 3, 3), (32, 1, 1), (64, 32, 3, 3), (64, 1, 1), (10, feat), (10,)]
    fans = [27, 27, 288, 288, feat, feat]
    params = [nk.from_ndarray(dev, rng.uniform(-1 / np.sqrt(f), 1 / np.sqrt(f), sh).astype(np.float32), nk.BF16)
              .requires_grad(nk.F32) for sh, f in zip(shapes, fans)]
    x = nk.from_ndarray(dev, rng.uniform(0, 1, (batch, 3, 32, 32)).astype(np.float32), nk.BF16)
    t = nk.from_ndarray(dev, np.eye(10, dtype=np.float32)[rng.integers(0, 10, batch)], nk.BF16)
    opt = optim.StochasticGD.new(0.01)
    for q in params:
        opt.register(q)
    pool = nk.nn.MaxPool2d(2)

    def step():
        opt.zero_grad()
        h = (params[0].convolution(x.pad((1, 1)), (1, 1), (1, 1), 1) + params[1]).relu()
        if pooled:
            h = pool.forward(h)
        h = (params[2].convolution(h.pad((1, 1)), (1, 1), (1, 1), 1) + params[3]).relu()
        if pooled:
            h = pool.forward(h)
        loss = (h.flatten().mm_t(params[4]) + params[5]).softmax(1).mse_loss(t)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    return capture(dev, step, 24 << 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dry-run", action="store_true", help="print the byte counts; no device")
    args = ap.parse_args()
    if args.dry_run:
        for name, (kind, shape, k, s, p) in CASES.items():
            oshape = out_shape(kind, shape, k, s, p)
            for dname, es in (("f32", 4), ("bf16", 2)):
                print(json.dumps({"case": name, "dtype": dname, "shape": shape, "out": oshape,
                                  "bytes": traffic(kind, shape, oshape, es)}))
        return
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for name, (kind, shape, k, s, p) in CASES.items():
        for dname, dt in (("bf16", torch.bfloat16), ("f32", torch.float32)):
            fwd, fb, oshape = case(nk, dev, torch, kind, shape, k, s, p, dt)
            nbytes = traffic(kind, shape, oshape, 2 if dt == torch.bfloat16 else 4)
            for direction, fns in (("forward", fwd), ("forward+backward", fb)):
                ms, mhz = alternate(fns, args.window_ms, args.reps)
                b = {i: nbytes[i][0] + (nbytes[i][1] if direction != "forward" else 0) for i in ms}
                gbps = {i: round(b[i] / v / 1e6, 1) for i, v in ms.items()}
                print(json.dumps({
                    "case": name, "dtype": dname, "direction": direction, "shape": shape, "out": oshape, "bytes": b,
                    "us": {i: round(v * 1e3, 1) for i, v in ms.items()}, "gbps": gbps,
                    "share_of_hbm": {i: round(v / DATASHEET["hbm_gbps"], 3) for i, v in gbps.items()},
                    "ours_vs_torch": round(ms["torch"] / ms["ours"], 3),
                    "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
            del fwd, fb
            torch.cuda.empty_cache()
    graphs = {"config5_convnet": convnet_step(nk, dev, False), "config5_convnet_maxpool": convnet_step(nk, dev, True)}
    ms, mhz = alternate({k: g.launch for k, g in graphs.items()}, args.window_ms, args.reps)
    for k, g in graphs.items():
        print(json.dumps({"case": k, "batch": 4096, "dtype": "bf16", "grad_dtype": "f32", "ms_per_step": round(ms[k], 4),
                          "kernels_per_step": g.kernel_count, "median_sm_mhz": mhz, "card": card["name"],
                          "power_limit_w": card["power_limit_w"]}), flush=True)
        g.close()


if __name__ == "__main__":
    main()
