#!/usr/bin/env python
"""Concatenation benchmark (development tool; bench.py measures the flagship workload).

Cases, forward and backward, each against torch.cat / torch.stack on the same tensors in the same process, the two
alternating window by window:
  sequence    cat of 32 x (1024, 2048) bf16 along axis 0; backward into f32 gradients
  channels    cat of 2 x (256, 64, 56, 56) bf16 along axis 1; backward into bf16 gradients
  interleave  stack of 3 x (2^24,) f32 along axis 1 (runs of one element); backward into f32 gradients
Bytes are counted from the shapes: every element is read once and written once (the backward overwrites, beta = 0).
torch's backward is what its autograd does for cat / stack: split (or unbind) the gradient and copy each slice into
the operand's gradient.  GB/s are reported beside the 3.35 TB/s HBM3 data-sheet bound of the H100 SXM.

Then the sequence head that motivates the op: T = 32 hidden states (N = 256, H = 1024, bf16, f32 gradients) into a
Linear(1024 -> 1024) head with an mse loss, (a) T per-step heads whose losses are added, against (b) `cat` along axis
0 -> one head -> one loss.  Each is one step (zero_grad -> forward -> backward -> SGD on the head) captured with
Device.capture and replayed; ms per step and the captured kernel count are reported.
Card name, power limit and the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/cat_bench.py [--reps 5] [--window-ms 200]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402


def copy_case(nk, dev, torch, name, shapes, axis, dt, gdt, stack):
    """(fwd fns, bwd fns, fwd bytes, bwd bytes, check) for one case; ours and torch's work on the same tensors"""
    from neuronika_b200 import ops
    tdt = {nk.BF16: torch.bfloat16, nk.F32: torch.float32}
    g = torch.Generator(device="cuda").manual_seed(0)
    xs = [torch.randn(s, device="cuda", generator=g).to(tdt[dt]) for s in shapes]
    wrap = lambda t, d, s=None: nk.CuArray(dev, tuple(s or t.shape), d, ptr=t.data_ptr(), owner=t)
    if stack:
        views = [wrap(x, dt, x.shape[:axis] + (1,) + x.shape[axis:]) for x in xs]
        y = torch.stack(xs, axis)
    else:
        views = [wrap(x, dt) for x in xs]
        y = torch.cat(xs, axis)
    cat_axis = axis
    yv = wrap(y, dt)
    gt = torch.randn(y.shape, device="cuda", generator=g).to(tdt[dt])
    gv = wrap(gt, dt)
    dxs = [torch.empty(x.shape, device="cuda", dtype=tdt[gdt]) for x in xs]
    dxv = [wrap(d, gdt, v.shape) for d, v in zip(dxs, views)]
    zeros = [0.0] * len(xs)
    lens = [v.shape[cat_axis] for v in views]

    def ours_fwd():
        ops.cat(views, cat_axis, out=yv)

    def torch_fwd():
        (torch.stack if stack else torch.cat)(xs, axis, out=y)

    def ours_bwd():
        ops.cat_bwd(dxv, gv, cat_axis, zeros)

    def torch_bwd():
        parts = torch.unbind(gt, axis) if stack else torch.split(gt, lens, axis)
        for d, p in zip(dxs, parts):
            d.copy_(p)

    n = sum(x.numel() for x in xs)
    fb = 2 * n * y.element_size()
    bb = n * (gt.element_size() + dxs[0].element_size())

    def check():
        ours_fwd()
        want = (torch.stack if stack else torch.cat)(xs, axis)
        assert torch.equal(y.view(torch.int16) if dt == nk.BF16 else y, want.view(torch.int16) if dt == nk.BF16 else want)
        ours_bwd()
        parts = torch.unbind(gt, axis) if stack else torch.split(gt, lens, axis)
        for d, p in zip(dxs, parts):
            assert torch.equal(d, p.to(d.dtype))

    return {"ours": ours_fwd, "torch": torch_fwd}, {"ours": ours_bwd, "torch": torch_bwd}, fb, bb, check


def head_step(nk, dev, T, n, hidden, use_cat):
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    head = nk.nn.Linear(dev, hidden, hidden, nk.BF16, grad_dtype=nk.F32, rng=rng)
    opt = optim.StochasticGD.new(1e-3)
    for p in head.parameters():
        opt.register(p)
    hs = [nk.from_ndarray(dev, rng.uniform(-1, 1, (n, hidden)).astype(np.float32), nk.BF16).requires_grad(nk.F32)
          for _ in range(T)]
    tg = [nk.from_ndarray(dev, rng.uniform(-1, 1, (n, hidden)).astype(np.float32), nk.BF16) for _ in range(T)]
    tgt = tg[0].cat(tg[1:], 0)
    tgt.forward()

    def step():
        opt.zero_grad()
        for h in hs:
            h.zero_grad()
        if use_cat:
            loss = head.forward(hs[0].cat(hs[1:], 0)).mse_loss(tgt)
        else:
            loss = None
            for h, t in zip(hs, tg):
                l_ = head.forward(h).mse_loss(t)
                loss = l_ if loss is None else loss + l_
        loss.forward()
        loss.backward(1.0)
        opt.step()

    return capture(dev, step, 4 << 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    cases = [("sequence", [(1024, 2048)] * 32, 0, nk.BF16, nk.F32, False),
             ("channels", [(256, 64, 56, 56)] * 2, 1, nk.BF16, nk.BF16, False),
             ("interleave", [(1 << 24,)] * 3, 1, nk.F32, nk.F32, True)]
    for name, shapes, axis, dt, gdt, stack in cases:
        fwd, bwd, fb, bb, check = copy_case(nk, dev, torch, name, shapes, axis, dt, gdt, stack)
        check()
        for direction, fns, nbytes in (("forward", fwd, fb), ("backward", bwd, bb)):
            ms, mhz = alternate(fns, args.window_ms, args.reps)
            gbps = {k: round(nbytes / v / 1e6, 1) for k, v in ms.items()}
            print(json.dumps({
                "case": name, "direction": direction, "op": "stack" if stack else "cat", "operands": len(shapes),
                "shape": list(shapes[0]), "axis": axis, "bytes": nbytes,
                "us": {k: round(v * 1e3, 2) for k, v in ms.items()}, "gbps": gbps,
                "share_of_hbm": {k: round(v / DATASHEET["hbm_gbps"], 3) for k, v in gbps.items()},
                "ours_vs_torch": round(ms["torch"] / ms["ours"], 3),
                "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        del fwd, bwd
        torch.cuda.empty_cache()
    T, n, hidden = 32, 256, 1024
    per_step = head_step(nk, dev, T, n, hidden, use_cat=False)
    catted = head_step(nk, dev, T, n, hidden, use_cat=True)
    ms, mhz = alternate({"per_step_heads": per_step.launch, "cat_one_head": catted.launch}, args.window_ms, args.reps)
    print(json.dumps({
        "case": "sequence_head", "T": T, "N": n, "H": hidden, "dtype": "bf16", "grad_dtype": "f32",
        "ms_per_step": {k: round(v, 4) for k, v in ms.items()},
        "kernels_per_step": {"per_step_heads": per_step.kernel_count, "cat_one_head": catted.kernel_count},
        "speedup_cat": round(ms["per_step_heads"] / ms["cat_one_head"], 3),
        "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
    per_step.close()
    catted.close()


if __name__ == "__main__":
    main()
