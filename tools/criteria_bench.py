#!/usr/bin/env python
"""Criteria and dropout benchmark (development tool; bench.py measures the flagship workload).

For mae, bce, bce_with_logits, kldiv and dropout over n = 2^26 elements (a (2^13, 2^13) tensor) in f32 and in bf16,
the forward and the backward of csrc/nk_criteria.cu / csrc/nk_dropout.cu against torch's counterparts on the same
tensors in the same process, the two alternating window by window:
  forward   F.l1_loss / F.binary_cross_entropy / F.binary_cross_entropy_with_logits / F.kl_div(reduction='batchmean')
            (Mean) and F.dropout(training=True);
  backward  what torch's autograd runs for that loss (torch.autograd.grad on a retained graph: the backward kernels
            alone), dx in the operands' dtype.
Bytes are counted from the shapes, for each implementation's own traffic: a loss forward reads x and t; a loss
backward reads x and t and writes dx (kldiv's reads only t); dropout's forward reads x and writes y plus the keep mask
-- n/8 bytes here, n bytes (one bool per element) for torch -- and its backward reads g and the mask and writes dx.
GB/s are reported beside the 3.35 TB/s HBM3 data-sheet bound of the H100 SXM.

Then one captured training step (zero_grad -> forward -> backward -> SGD) of an MLP Linear(1024 -> 4096) -> ReLU ->
dropout(0.5) -> Linear(4096 -> 1) -> bce_with_logits, batch 4096, bf16 data and f32 gradients: ms per step and the
captured kernel count.  Card name, power limit and the median SM clock during the timed windows (NVML) are printed
beside the numbers.

    python tools/criteria_bench.py [--log2n 26] [--reps 5] [--window-ms 200]
    python tools/criteria_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402

OPS = ["mae", "bce", "bce_with_logits", "kldiv", "dropout"]


def traffic(op, n, esize):
    """{impl: (forward bytes, backward bytes)} from the shapes"""
    if op == "dropout":
        return {"ours": (2 * n * esize + n // 8, 2 * n * esize + n // 8),
                "torch": (2 * n * esize + n, 2 * n * esize + n)}
    bwd = (2 if op == "kldiv" else 3) * n * esize
    return {"ours": (2 * n * esize, bwd), "torch": (2 * n * esize, bwd)}


def operands(torch, op, shape, dt, gen):
    x = torch.rand(shape, device="cuda", generator=gen)
    t = torch.rand(shape, device="cuda", generator=gen)
    if op == "bce":
        x = x * 0.98 + 0.01
    elif op == "bce_with_logits":
        x = 4 * torch.randn(shape, device="cuda", generator=gen)
    elif op == "kldiv":
        x = torch.log(x * 0.99 + 0.01)
    elif op == "mae":
        x, t = torch.randn(shape, device="cuda", generator=gen), torch.randn(shape, device="cuda", generator=gen)
    return x.to(dt).contiguous(), t.to(dt).contiguous()


def case(nk, dev, torch, op, shape, dt):
    """(forward fns, backward fns) of one (op, dtype), ours and torch's on the same tensors"""
    import torch.nn.functional as F

    from neuronika_b200 import ops
    ndt = nk.BF16 if dt == torch.bfloat16 else nk.F32
    gen = torch.Generator(device="cuda").manual_seed(0)
    x, t = operands(torch, op, shape, dt, gen)
    n = x.numel()
    wrap = lambda a, d, s=None: nk.CuArray(dev, tuple(s or a.shape), d, ptr=a.data_ptr(), owner=a)
    xv, tv = wrap(x, ndt), wrap(t, ndt)
    dx = torch.empty_like(x)
    dxv = wrap(dx, ndt)
    xr = x.detach().requires_grad_(True)
    if op == "dropout":
        y = torch.empty_like(x)
        yv = wrap(y, ndt)
        mask = torch.empty(((n + 31) // 32,), dtype=torch.int32, device="cuda")
        mv = wrap(mask, nk.F32)
        g = torch.randn(shape, device="cuda", generator=gen).to(dt)
        gv = wrap(g, ndt)
        ty = F.dropout(xr, 0.5, training=True)
        fwd = {"ours": lambda: ops.dropout(xv, 0.5, mv, out=yv), "torch": lambda: F.dropout(x, 0.5, training=True)}
        bwd = {"ours": lambda: ops.dropout_bwd(dxv, mv, gv, 0.5, beta=0.0),
               "torch": lambda: torch.autograd.grad(ty, xr, g, retain_graph=True)}
        return fwd, bwd
    fn = {"mae": lambda a, b: F.l1_loss(a, b),
          "bce": lambda a, b: F.binary_cross_entropy(a, b),
          "bce_with_logits": lambda a, b: F.binary_cross_entropy_with_logits(a, b),
          "kldiv": lambda a, b: F.kl_div(a, b, reduction="batchmean")}[op]
    loss = torch.empty((), device="cuda")
    lv = wrap(loss, nk.F32, ())
    one = torch.ones((), device="cuda")
    ov = wrap(one, nk.F32, ())
    tl = fn(xr, t)
    fwd = {"ours": lambda: ops.criterion(op, xv, tv, True, out=lv), "torch": lambda: fn(x, t)}
    bwd = {"ours": lambda: ops.criterion_bwd(op, dxv, xv, tv, ov, True, beta=0.0),
           "torch": lambda: torch.autograd.grad(tl, xr, retain_graph=True)}
    # the two agree on the loss (bce's ln clamps and kldiv's batch mean are torch's too)
    ops.criterion(op, xv, tv, True, out=lv)
    dev.synchronize()
    ref = float(fn(x.float(), t.float()))
    assert abs(float(loss) - ref) <= 1e-3 * abs(ref) + 1e-6, (op, float(loss), ref)
    return fwd, bwd


def mlp_step(nk, dev, batch=4096, n_in=1024, hidden=4096):
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    l1 = nk.nn.Linear(dev, n_in, hidden, nk.BF16, grad_dtype=nk.F32, rng=rng)
    l2 = nk.nn.Linear(dev, hidden, 1, nk.BF16, grad_dtype=nk.F32, rng=rng)
    drop = nk.nn.Dropout(0.5)
    opt = optim.StochasticGD.new(1e-3)
    for p in l1.parameters() + l2.parameters():
        opt.register(p)
    x = nk.from_ndarray(dev, rng.standard_normal((batch, n_in)).astype(np.float32), nk.BF16)
    t = nk.from_ndarray(dev, (rng.uniform(0, 1, (batch, 1)) < 0.5).astype(np.float32), nk.BF16)

    def step():
        opt.zero_grad()
        loss = l2.forward(drop.forward(l1.forward(x).relu())).bce_with_logits(t)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    dev.manual_seed(0)
    return capture(dev, step, 2 << 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=26)
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dry-run", action="store_true", help="print the byte counts; no device")
    args = ap.parse_args()
    n = 1 << args.log2n
    shape = (1 << (args.log2n // 2), 1 << (args.log2n - args.log2n // 2))
    if args.dry_run:
        for op in OPS:
            for name, es in (("f32", 4), ("bf16", 2)):
                print(json.dumps({"op": op, "dtype": name, "n": n, "shape": list(shape), "bytes": traffic(op, n, es)}))
        return
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for op in OPS:
        for dname, dt in (("f32", torch.float32), ("bf16", torch.bfloat16)):
            fwd, bwd = case(nk, dev, torch, op, shape, dt)
            nbytes = traffic(op, n, 2 if dt == torch.bfloat16 else 4)
            for k, (direction, fns) in enumerate((("forward", fwd), ("backward", bwd))):
                ms, mhz = alternate(fns, args.window_ms, args.reps)
                gbps = {i: round(nbytes[i][k] / v / 1e6, 1) for i, v in ms.items()}
                print(json.dumps({
                    "op": op, "dtype": dname, "direction": direction, "n": n,
                    "bytes": {i: nbytes[i][k] for i in ms}, "us": {i: round(v * 1e3, 2) for i, v in ms.items()},
                    "gbps": gbps, "share_of_hbm": {i: round(v / DATASHEET["hbm_gbps"], 3) for i, v in gbps.items()},
                    "ours_vs_torch": round(ms["torch"] / ms["ours"], 3),
                    "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
            del fwd, bwd
            torch.cuda.empty_cache()
    g = mlp_step(nk, dev)
    ms, mhz = alternate({"step": g.launch}, args.window_ms, args.reps)
    print(json.dumps({
        "case": "mlp_dropout_bce_with_logits", "batch": 4096, "layers": [1024, 4096, 1], "p": 0.5,
        "dtype": "bf16", "grad_dtype": "f32", "ms_per_step": round(ms["step"], 4), "kernels_per_step": g.kernel_count,
        "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
    g.close()


if __name__ == "__main__":
    main()
