#!/usr/bin/env python
"""Gradient-clipping benchmark (development tool; bench.py measures the flagship workload).

For each parameter set below, our optim.clip_grad_norm_ against torch CUDA's clip_grad_norm_(foreach=True) on
gradients of the same shapes and dtypes, alternating window by window, CUDA events on the stream both run on:
  eager     one call per iteration, host work included (ours: ctypes, the 0-d total, the partials workspace);
  captured  the call recorded once (our Device.capture, torch.cuda.graph) and replayed: what it adds to a captured step.
Each set runs twice: max_norm above the total (no clip: ours reads the gradients once and skips the scale pass) and
max_norm = 0 (every call clips and writes every gradient).  Bytes: n*s for the norm pass, plus 2*n*s when clipping;
reported as GB/s beside the 3.35 TB/s HBM3 data-sheet bound of the H100 SXM.

Then the captured language-model step of cross_entropy_bench.py (Embedding -> LSTM -> reshape -> Linear ->
cross_entropy, SGD; V = 10 000, E = H = 650, T = 35, N = 256, bf16 data, f32 gradients) with and without
clip_grad_norm_(0.25) before the optimizer step: ms per step and captured kernels.  Card name, power limit and the
median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/clip_bench.py [--reps 5] [--window-ms 200]
    python tools/clip_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402

V_, E_, T_, N_ = 10000, 650, 35, 256
_MLP = [(4096, 1024), (4096,), (4096, 4096), (4096,), (10, 4096), (10,)]
_LM = [(V_, E_), (4 * E_, E_), (4 * E_, E_), (4 * E_,), (4 * E_,), (V_, E_), (V_,)]
# name: ([shapes], data dtype, gradient dtype)
SETS = {
    "mlp_config4_f32": (_MLP, "f32", "f32"),            # bench.py config 4: 1024-4096-4096-10
    "lm_bf16_weights_f32_grads": (_LM, "bf16", "f32"),  # the language model of cross_entropy_bench.py
    "256x4096_f32": ([(4096,)] * 256, "f32", "f32"),
    "mlp_config4_bf16": (_MLP, "bf16", "bf16"),
}


def numel(shapes):
    return sum(int(np.prod(s)) for s in shapes)


def traffic(shapes, gdt, clip):
    s = 2 if gdt == "bf16" else 4
    n = numel(shapes)
    return n * s * (3 if clip else 1)


def param_set(nk, dev, torch, shapes, dt, gdt, seed):
    """our parameters and torch's, with the same gradient values"""
    from neuronika_b200 import _lib as L
    tdt = torch.bfloat16 if gdt == "bf16" else torch.float32
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ours, theirs = [], []
    for s in shapes:
        g = (torch.randn(s, device="cuda", generator=gen) * 1e-3).to(tdt)
        p = nk.zeros(dev, s, nk.BF16 if dt == "bf16" else nk.F32).requires_grad(nk.BF16 if gdt == "bf16" else nk.F32)
        arr = p.grad_array()
        L.check(L.lib.nk_d2d(dev.ctx, arr.ptr, C.c_void_p(g.data_ptr()), arr.nbytes), dev.ctx)   # same stream as g's
        t = torch.nn.Parameter(torch.zeros(s, device="cuda", dtype=tdt))
        t.grad = g.clone()
        ours.append(p)
        theirs.append(t)
    dev.synchronize()
    return ours, theirs


def captured(nk, dev, torch, ours, theirs, max_norm):
    from neuronika_b200 import optim
    ours_graph = capture(dev, lambda: optim.clip_grad_norm_(ours, max_norm), 64 << 20)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.nn.utils.clip_grad_norm_(theirs, max_norm, foreach=True)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        torch.nn.utils.clip_grad_norm_(theirs, max_norm, foreach=True)
    return ours_graph, g


def lm_step(nk, dev, clip, V=V_, E=E_, T=T_, N=N_):
    """the language-model step of cross_entropy_bench.py, captured, with clip_grad_norm_(0.25) before the step or not"""
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
    keep = []

    def step():
        opt.zero_grad()
        out, _ = lstm.forward((c0, h0), emb.forward(I))
        loss = head.forward(out.reshape(T * N, E)).cross_entropy(TG)
        loss.forward()
        loss.backward(1.0)
        if clip:
            keep.append(optim.clip_grad_norm_(params, 0.25))
        opt.step()

    graph = capture(dev, step, 8 << 30)
    total = float(keep[-1].as_ndarray()) if clip else None
    return graph, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--dry-run", action="store_true", help="print the byte counts; no device")
    args = ap.parse_args()
    if args.dry_run:
        for name, (shapes, dt, gdt) in SETS.items():
            print(json.dumps({"set": name, "tensors": len(shapes), "elements": numel(shapes), "grad_dtype": gdt,
                              "norm_bytes": traffic(shapes, gdt, False), "clip_bytes": traffic(shapes, gdt, True)}))
        return
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk
    from neuronika_b200 import optim

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for name, (shapes, dt, gdt) in SETS.items():
        ours, theirs = param_set(nk, dev, torch, shapes, dt, gdt, 0)
        t_ours = float(optim.get_total_norm(ours).as_ndarray())
        t_theirs = float(torch.nn.utils.get_total_norm([t.grad for t in theirs]))
        assert abs(t_ours - t_theirs) <= (1e-2 if gdt == "bf16" else 1e-5) * t_theirs, (t_ours, t_theirs)  # bf16: torch rounds its norms to bf16
        for clip in (False, True):
            max_norm = 0.0 if clip else 1e30
            g_ours, g_theirs = captured(nk, dev, torch, ours, theirs, max_norm)
            fns = {"ours_eager": lambda: optim.clip_grad_norm_(ours, max_norm),
                   "torch_eager": lambda: torch.nn.utils.clip_grad_norm_(theirs, max_norm, foreach=True),
                   "ours_captured": g_ours.launch, "torch_captured": g_theirs.replay}
            ms, mhz = alternate(fns, args.window_ms, args.reps)
            nbytes = traffic(shapes, gdt, clip)
            print(json.dumps({
                "set": name, "tensors": len(shapes), "elements": numel(shapes), "grad_dtype": gdt, "clip": clip,
                "bytes": nbytes, "us": {k: round(v * 1e3, 1) for k, v in ms.items()},
                "ours_captured_gbps": round(nbytes / ms["ours_captured"] / 1e6, 1),
                "ours_captured_share_of_hbm": round(nbytes / ms["ours_captured"] / 1e6 / DATASHEET["hbm_gbps"], 3),
                "captured_vs_torch": round(ms["torch_captured"] / ms["ours_captured"], 3),
                "eager_vs_torch": round(ms["torch_eager"] / ms["ours_eager"], 3),
                "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
            g_ours.close()
            del g_theirs
        del ours, theirs
        torch.cuda.empty_cache()
    graphs = {}
    for clip in (False, True):
        graphs["lm_step_clip" if clip else "lm_step"] = lm_step(nk, dev, clip)
    ms, mhz = alternate({k: g.launch for k, (g, _) in graphs.items()}, args.window_ms, args.reps)
    for k, (g, total) in graphs.items():
        print(json.dumps({"case": k, "V": V_, "E": E_, "T": T_, "N": N_, "dtype": "bf16", "grad_dtype": "f32",
                          "ms_per_step": round(ms[k], 4), "kernels_per_step": g.kernel_count,
                          "captured_total_norm": total, "median_sm_mhz": mhz, "card": card["name"],
                          "power_limit_w": card["power_limit_w"]}), flush=True)
    print(json.dumps({"case": "lm_step_clip_overhead", "ms": round(ms["lm_step_clip"] - ms["lm_step"], 4),
                      "share": round(ms["lm_step_clip"] / ms["lm_step"] - 1.0, 4)}), flush=True)
    for g, _ in graphs.values():
        g.close()


if __name__ == "__main__":
    main()
