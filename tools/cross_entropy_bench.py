#!/usr/bin/env python
"""Cross-entropy benchmark (development tool; bench.py measures the flagship workload).

For each case below, three implementations on the same tensors in the same process, alternating window by window:
  fused        ours: nk_cross_entropy_fwd, then nk_cross_entropy_bwd with beta 0 (dx in x's dtype);
  composition  ours: nk_log_softmax_fwd + nk_nll_fwd, then nk_nll_bwd + nk_log_softmax_bwd (2-D inputs only: nll takes
               (N, C));
  torch        F.cross_entropy, and torch.autograd.grad of it for forward + backward.
Each is timed for the forward alone and for forward + backward.  Bytes are counted from the shapes: the forward reads
x and the f32 targets, the backward reads x, the targets and the f32 lse and writes dx; GB/s are reported beside the
3.35 TB/s HBM3 data-sheet bound of the H100 SXM.  The fused kernels' traffic is the floor of the three.

Then one captured language-model training step (Embedding -> LSTM -> reshape -> Linear -> loss, SGD; V = 10 000,
E = H = 650, T = 35, N = 256, bf16 data, f32 gradients) with the loss as cross_entropy and as log_softmax -> nll_loss:
ms per step and captured kernels.  Card name, power limit and the median SM clock during the timed windows (NVML) are
printed beside the numbers.

    python tools/cross_entropy_bench.py [--reps 5] [--window-ms 200]
    python tools/cross_entropy_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402

# name: (x shape, dtype)
CASES = {
    "config4_8192x10_f32": ((8192, 10), "f32"),
    "lm_8960x10000_bf16": ((8960, 10000), "bf16"),
    "llama_4096x32000_bf16": ((4096, 32000), "bf16"),
    "gpt2_8192x50257_bf16": ((8192, 50257), "bf16"),
    "few_long_rows_16x262144_bf16": ((16, 262144), "bf16"),
    "segmentation_8x19x512x512_f32": ((8, 19, 512, 512), "f32"),
}


def traffic(shape, esize):
    """(forward bytes, backward bytes): the forward reads x and the f32 targets; the backward reads x, the targets and
    the f32 lse and writes dx (x's dtype)"""
    n, c = shape[0], shape[1]
    pos = n * int(np.prod(shape[2:], dtype=np.int64)) if len(shape) > 2 else n
    elems = pos * c
    return elems * esize + 4 * pos, 2 * elems * esize + 8 * pos


def case(nk, dev, torch, shape, xdt):
    import torch.nn.functional as F

    from neuronika_b200 import ops
    tdt = torch.bfloat16 if xdt == "bf16" else torch.float32
    ndt = nk.BF16 if xdt == "bf16" else nk.F32
    n, c = shape[0], shape[1]
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(shape, device="cuda", generator=gen) * 2).to(tdt)
    tshape = (n,) + tuple(shape[2:])
    t = torch.randint(0, c, tshape, device="cuda", generator=gen).float()
    tl = t.long()
    dx = torch.empty(shape, device="cuda", dtype=tdt)
    wrap = lambda a, d: nk.CuArray(dev, tuple(a.shape), d, ptr=a.data_ptr(), owner=a)
    xv, tv, dxv = wrap(x, ndt), wrap(t, nk.F32), wrap(dx, ndt)
    loss, lse, denom = dev.zeros((), nk.F32), dev.zeros((t.numel(),), nk.F32), dev.zeros((), nk.F32)
    one = dev.from_ndarray(np.ones((), np.float32))
    fused_f = lambda: ops.cross_entropy(xv, tv, out=loss, lse=lse, denom=denom)
    fused_b = lambda: ops.cross_entropy_bwd(dxv, xv, tv, lse, denom, one, beta=0.0)
    xr = x.detach().requires_grad_(True)
    torch_f = lambda: F.cross_entropy(x, tl)
    torch_fb = lambda: torch.autograd.grad(F.cross_entropy(xr, tl), xr)
    fwd = {"fused": fused_f, "torch": torch_f}
    fb = {"fused": lambda: (fused_f(), fused_b()), "torch": torch_fb}
    fused_f()
    fused_b()
    dev.synchronize()
    want = F.cross_entropy(x.float(), tl)
    assert abs(float(loss.as_ndarray()) - float(want)) <= 1e-4 * abs(float(want)), "loss differs from torch"
    if len(shape) == 2:
        logp, nll, dlogp = wrap(torch.empty_like(x), ndt), dev.zeros((), nk.F32), wrap(torch.empty_like(x), ndt)
        comp_f = lambda: (ops.softmax(xv, 1, out=logp, log=True), ops.nll(logp, tv, out=nll))
        comp_b = lambda: (ops.nll_bwd(dlogp, tv, one, beta=0.0), ops.softmax_bwd(dxv, logp, dlogp, 1, beta=0.0, log=True))
        fwd["composition"] = comp_f
        fb["composition"] = lambda: (comp_f(), comp_b())
    return fwd, fb


def lm_step(nk, dev, fused, V=10000, E=650, T=35, N=256):
    """the language-model step of embedding_bench.py, captured, with the loss as cross_entropy (fused) or as
    log_softmax -> nll_loss"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    emb = nk.nn.Embedding(dev, V, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    lstm = nk.nn.LSTM(dev, E, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    head = nk.nn.Linear(dev, E, V, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    params = emb.parameters() + lstm.parameters() + head.parameters()
    I = nk.from_ndarray(dev, rng.integers(0, V, (T, N)).astype(np.float32))
    TG = nk.from_ndarray(dev, rng.integers(0, V, T * N).astype(np.float32))
    c0, h0 = nk.zeros(dev, (N, E), nk.BF16), nk.zeros(dev, (N, E), nk.BF16)
    opt = optim.StochasticGD.new(0.01)
    for q in params:
        opt.register(q)

    def step():
        opt.zero_grad()
        out, _ = lstm.forward((c0, h0), emb.forward(I))
        logits = head.forward(out.reshape(T * N, E))
        loss = logits.cross_entropy(TG) if fused else logits.log_softmax(1).nll_loss(TG)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    return capture(dev, step, 8 << 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dry-run", action="store_true", help="print the byte counts; no device")
    args = ap.parse_args()
    if args.dry_run:
        for name, (shape, xdt) in CASES.items():
            fb, bb = traffic(shape, 2 if xdt == "bf16" else 4)
            print(json.dumps({"case": name, "shape": shape, "dtype": xdt, "forward_bytes": fb, "backward_bytes": bb,
                              "fwd+bwd_bytes": fb + bb}))
        return
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for name, (shape, xdt) in CASES.items():
        fwd, fb = case(nk, dev, torch, shape, xdt)
        fbytes, bbytes = traffic(shape, 2 if xdt == "bf16" else 4)
        for direction, fns, nbytes in (("forward", fwd, fbytes), ("fwd+bwd", fb, fbytes + bbytes)):
            ms, mhz = alternate(fns, args.window_ms, args.reps)
            rec = {"case": name, "shape": shape, "dtype": xdt, "direction": direction, "bytes": nbytes,
                   "us": {k: round(v * 1e3, 1) for k, v in ms.items()},
                   "fused_gbps": round(nbytes / ms["fused"] / 1e6, 1),
                   "fused_share_of_hbm": round(nbytes / ms["fused"] / 1e6 / DATASHEET["hbm_gbps"], 3),
                   "fused_vs_torch": round(ms["torch"] / ms["fused"], 3)}
            if "composition" in ms:
                rec["fused_vs_composition"] = round(ms["composition"] / ms["fused"], 3)
            rec.update({"median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]})
            print(json.dumps(rec), flush=True)
        del fwd, fb
        torch.cuda.empty_cache()
    graphs = {"lm_step_cross_entropy": lm_step(nk, dev, True), "lm_step_log_softmax_nll": lm_step(nk, dev, False)}
    ms, mhz = alternate({k: g.launch for k, g in graphs.items()}, args.window_ms, args.reps)
    for k, g in graphs.items():
        print(json.dumps({"case": k, "V": 10000, "E": 650, "T": 35, "N": 256, "dtype": "bf16", "grad_dtype": "f32",
                          "ms_per_step": round(ms[k], 4), "kernels_per_step": g.kernel_count, "median_sm_mhz": mhz,
                          "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        g.close()


if __name__ == "__main__":
    main()
