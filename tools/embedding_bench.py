#!/usr/bin/env python
"""Embedding benchmark (development tool; bench.py measures the flagship workload).

For each case below, csrc/nk_embedding.cu against torch CUDA on the same tensors in the same process, the two
alternating window by window:
  forward           ours: nk_embedding_fwd; torch: F.embedding;
  backward          ours: nk_embedding_bwd with beta 0 into the weight's gradient; torch: torch.autograd.grad of the
                    weight through F.embedding (its sort-based dense backward), which also runs the forward;
                    so the torch column of the backward is forward + backward, and ours is reported both ways.
Bytes are counted from the shapes: the forward reads n*e weight elements and the ids and writes n*e; the backward
reads g and the ids and writes all v*e rows of dw (beta = 0).  GB/s are reported beside the 3.35 TB/s HBM3
data-sheet bound of the H100 SXM.

Then one captured language-model training step (Embedding -> LSTM -> reshape -> Linear -> log_softmax -> nll, SGD;
V = 10 000, E = H = 650, T = 35, N = 256, bf16 data, f32 gradients) beside the same step with the embedding done as
the one-hot workaround (a (T*N, V) one-hot operand times the (V, E) weight): ms per step and captured kernels.  Card
name, power limit and the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/embedding_bench.py [--reps 5] [--window-ms 200]
    python tools/embedding_bench.py --dry-run      # the byte counts only, no device
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DATASHEET, alternate, capture, setup  # noqa: E402

# name: (v, e, ids shape, id distribution, weight dtype); gradients are f32
CASES = {
    "gpt2_v50257_e768_8x1024": (50257, 768, (8, 1024), "uniform", "bf16"),
    "llama_v32000_e4096_4x2048": (32000, 4096, (4, 2048), "uniform", "bf16"),
    "ptb_v10000_e650_35x256_zipf_f32": (10000, 650, (35, 256), "zipf", "f32"),
    "ptb_v10000_e650_35x256_zipf_bf16": (10000, 650, (35, 256), "zipf", "bf16"),
    "all_equal_n2^20_e768": (50257, 768, (1 << 20,), "equal", "bf16"),
}


def traffic(v, e, n, esize):
    """(forward bytes, backward bytes) from the shapes; ids are f32, the gradient f32"""
    return (2 * n * e * esize + 4 * n, n * e * 4 + 4 * n + v * e * 4)


def make_ids(kind, rng, n, v):
    if kind == "uniform":
        return rng.integers(0, v, n).astype(np.float32)
    if kind == "zipf":
        return np.minimum(rng.zipf(1.2, n) - 1, v - 1).astype(np.float32)
    return np.full(n, v // 2, np.float32)


def case(nk, dev, torch, v, e, shape, kind, wdt):
    import torch.nn.functional as F

    from neuronika_b200 import ops
    tdt = torch.bfloat16 if wdt == "bf16" else torch.float32
    ndt = nk.BF16 if wdt == "bf16" else nk.F32
    rng = np.random.default_rng(0)
    n = int(np.prod(shape))
    ids = make_ids(kind, rng, n, v)
    gen = torch.Generator(device="cuda").manual_seed(0)
    w = torch.randn(v, e, device="cuda", generator=gen).to(tdt)
    idf = torch.from_numpy(ids).cuda()
    idl = idf.long()
    y = torch.empty(n, e, device="cuda", dtype=tdt)
    g = torch.randn(n, e, device="cuda", generator=gen)
    dw = torch.empty(v, e, device="cuda", dtype=torch.float32)
    wrap = lambda a, d, s=None: nk.CuArray(dev, tuple(s or a.shape), d, ptr=a.data_ptr(), owner=a)
    wv, yv, iv, gv, dwv = wrap(w, ndt), wrap(y, ndt), wrap(idf, nk.F32), wrap(g, nk.F32), wrap(dw, nk.F32)
    wr = w.float().detach().requires_grad_(True)      # torch: f32 master weight for an f32 gradient
    wb = w.detach().requires_grad_(True)
    ours_f = lambda: ops.embedding(wv, iv, out=yv)
    ours_b = lambda: ops.embedding_bwd(dwv, iv, gv, beta=0.0)
    torch_f = lambda: F.embedding(idl, w)
    torch_fb = lambda: torch.autograd.grad(F.embedding(idl, wr if wdt == "f32" else wb), wr if wdt == "f32" else wb,
                                           g.to(tdt))
    ours_f()
    ours_b()
    dev.synchronize()
    assert torch.equal(y, torch_f()), "forward differs from torch"
    ref = torch.autograd.grad(F.embedding(idl, wr), wr, g)[0]
    # a row of 2^20 summed terms differs from torch's order by up to ~1e-4 of the largest partial sum
    assert torch.allclose(dw, ref, rtol=1e-3, atol=1e-4 * float(ref.abs().max()) + 1e-3), "backward differs from torch"
    return ({"ours": ours_f, "torch": torch_f},
            {"ours": ours_b, "ours_fwd+bwd": lambda: (ours_f(), ours_b()), "torch": torch_fb}, n)


def lm_step(nk, dev, onehot, V=10000, E=650, T=35, N=256):
    """the language-model step, captured; onehot: the embedding as a (T*N, V) one-hot operand times the weight"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    emb = nk.nn.Embedding(dev, V, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    lstm = nk.nn.LSTM(dev, E, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    head = nk.nn.Linear(dev, E, V, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    params = emb.parameters() + lstm.parameters() + head.parameters()
    ids = rng.integers(0, V, (T, N))
    I = nk.from_ndarray(dev, ids.astype(np.float32))
    if onehot:
        oh = np.zeros((T * N, V), np.float32)
        oh[np.arange(T * N), ids.reshape(-1)] = 1.0
        OH = nk.from_ndarray(dev, oh, nk.BF16)
        del oh
    TG = nk.from_ndarray(dev, rng.integers(0, V, T * N).astype(np.float32))
    c0, h0 = nk.zeros(dev, (N, E), nk.BF16), nk.zeros(dev, (N, E), nk.BF16)
    opt = optim.StochasticGD.new(0.01)
    for q in params:
        opt.register(q)

    def step():
        opt.zero_grad()
        x = OH.mm(emb.weight).reshape(T, N, E) if onehot else emb.forward(I)
        out, _ = lstm.forward((c0, h0), x)
        loss = head.forward(out.reshape(T * N, E)).log_softmax(1).nll_loss(TG)
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
        for name, (v, e, shape, kind, wdt) in CASES.items():
            n = int(np.prod(shape))
            print(json.dumps({"case": name, "v": v, "e": e, "n": n, "bytes": traffic(v, e, n, 2 if wdt == "bf16" else 4)}))
        return
    args.window_ms = max(150.0, args.window_ms)
    import torch

    import neuronika_b200 as nk

    dev, card = setup(hbm_datasheet_gbps=DATASHEET["hbm_gbps"])
    for name, (v, e, shape, kind, wdt) in CASES.items():
        fwd, bwd, n = case(nk, dev, torch, v, e, shape, kind, wdt)
        fb, bb = traffic(v, e, n, 2 if wdt == "bf16" else 4)
        for direction, fns, nbytes in (("forward", fwd, fb), ("backward", bwd, bb)):
            ms, mhz = alternate(fns, args.window_ms, args.reps)
            print(json.dumps({
                "case": name, "dtype": wdt, "grad_dtype": "f32", "direction": direction, "v": v, "e": e, "n": n,
                "bytes": nbytes, "us": {i: round(t * 1e3, 1) for i, t in ms.items()},
                "ours_gbps": round(nbytes / ms["ours"] / 1e6, 1),
                "ours_share_of_hbm": round(nbytes / ms["ours"] / 1e6 / DATASHEET["hbm_gbps"], 3),
                "ours_vs_torch": round(ms["torch"] / ms["ours"], 3),
                "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        del fwd, bwd
        torch.cuda.empty_cache()
    graphs = {"lm_step_embedding": lm_step(nk, dev, False), "lm_step_onehot_gemm": lm_step(nk, dev, True)}
    ms, mhz = alternate({k: g.launch for k, g in graphs.items()}, args.window_ms, args.reps)
    for k, g in graphs.items():
        print(json.dumps({"case": k, "V": 10000, "E": 650, "T": 35, "N": 256, "dtype": "bf16", "grad_dtype": "f32",
                          "ms_per_step": round(ms[k], 4), "kernels_per_step": g.kernel_count, "median_sm_mhz": mhz,
                          "card": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        g.close()


if __name__ == "__main__":
    main()
