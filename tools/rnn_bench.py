#!/usr/bin/env python
"""LSTM / GRU training-step benchmark (development tool; bench.py measures the flagship workload).

Workload: a sequence of T = 32 steps, bf16 parameters with f32 gradients, the input a `Var`, h0 = c0 = 0, the loss the
mse of h_T against a seeded target.  One step is zero_grad -> forward -> backward -> SGD, captured once with
Device.capture and replayed.  Shapes (N, I, H) = (256, 1024, 1024) and (1024, 2048, 2048), LSTM and GRU.  Three variants
of the same computation: "fused" unrolls nn.LSTMCell / nn.GRUCell (one node per time step), "composed" unrolls the cell
written with primitives, "sequence" is nn.LSTM / nn.GRU (one node for the whole sequence).

Reported per configuration, in one JSON line each:
  - ms per sequence and per time step, and kernel launches per time step (the captured graph's kernel count / T);
  - the cell's GEMMs alone (the same five products per step, timed back to back: x.W_ih^T + b, h.W_hh^T + b,
    dW_ih, dW_hh, dh), as TFLOP/s from FLOPs counted from the shapes, and their share of the step;
  - the gate kernels alone (forward and backward, CUDA events over many launches) as GB/s against HBM, from the bytes
    each must move (f32 gates, bf16 states / gradients) counted from the shapes;
  - in the same process and alternating with it: the same cell composed from primitives through the graph API
    (chunks + sigmoid / tanh + mul / add, intended gate assignment), also captured and replayed, and
    torch.nn.LSTMCell / GRUCell in bf16 on the same GPU in an eager loop ("torch_eager_bf16") and torch.nn.LSTM / GRU
    (cuDNN) in bf16 on the whole sequence ("torch_cudnn_bf16");
  - the sequence layer's GEMMs alone, in two groups: the products that run once over all T*N rows (x.W_ih^T + b, dW_ih,
    dW_hh) and the 2T sequential ones that stay N rows tall (h.W_hh^T + b forward, dG.W_hh backward), as ms per sequence
    and as shares of the sequence layer's step.
Then one more JSON line per configuration ("stacked"): nn.LSTM / nn.GRU unidirectional, bidirectional and 2 layers x
bidirectional on the same sequence (the loss on the last time step of the last layer's output), each beside
torch.nn.LSTM / GRU(num_layers, bidirectional) in bf16 (cuDNN); the ratio bidirectional / (2 x unidirectional) (below 1:
the two directions' batched step GEMM and step kernel cost less than two layers' worth) and the launches per time step.
Each of these three captured steps reserves a 12 GiB capture arena (what the GRU's 2 layers x 2 directions at N = 1024
need), 36 GiB of device memory in all while a row is measured: run it on a card that has that much free.
Card name, power limit and the median SM clock during the timed windows (NVML) are printed beside the numbers.

    python tools/rnn_bench.py [--reps 5] [--window-ms 200] [--stacked-only]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import alternate, capture, setup, window  # noqa: E402

T = 32
SHAPES = [(256, 1024, 1024), (1024, 2048, 2048)]


def composed_cell(kind, cell, state, x, n, hidden):
    """the cell written as the reference writes it (intended LSTM gate assignment), through the graph API"""
    if kind == "lstm":
        c, h = state
        gates = x.mm_t(cell.weight_ih) + cell.bias_ih + h.mm_t(cell.weight_hh) + cell.bias_hh
        i, f, g, o = gates.chunks((n, hidden))
        c2 = f.sigmoid() * c + i.sigmoid() * g.tanh()
        return c2, o.sigmoid() * c2.tanh()
    ig = x.mm_t(cell.weight_ih) + cell.bias_ih
    hg = state.mm_t(cell.weight_hh) + cell.bias_hh
    ir, iz, i_n = ig.chunks((n, hidden))
    hr, hz, hn = hg.chunks((n, hidden))
    r, z = (hr + ir).sigmoid(), (hz + iz).sigmoid()
    nn = (i_n + hn * r).tanh()
    return (state - nn) * z + nn


def graph_step(nk, dev, kind, n, n_in, hidden, variant):
    """the captured step of one variant ("fused", "composed" or "sequence")"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    composed, sequence = variant == "composed", variant == "sequence"
    if sequence:
        cls = nk.nn.LSTM if kind == "lstm" else nk.nn.GRU
    else:
        cls = nk.nn.LSTMCell if kind == "lstm" else nk.nn.GRUCell
    cell = cls(dev, n_in, hidden, nk.BF16, grad_dtype=nk.F32, rng=rng)
    opt = optim.StochasticGD.new(1e-3)
    for p in cell.parameters():
        opt.register(p)
    xs = [nk.from_ndarray(dev, rng.uniform(-1, 1, (n, n_in)).astype(np.float32), nk.BF16) for _ in range(T)]
    zero = nk.zeros(dev, (n, hidden), nk.BF16)
    tgt = nk.from_ndarray(dev, rng.uniform(-0.5, 0.5, (n, hidden)).astype(np.float32), nk.BF16)
    if sequence:
        x_seq = nk.from_ndarray(dev, np.stack([x.data() for x in xs]), nk.BF16)
        tgt_seq = nk.from_ndarray(dev, tgt.data().reshape(1, n, hidden), nk.BF16)

    def step():
        opt.zero_grad()
        state = (zero, zero) if kind == "lstm" else zero
        if sequence:
            out = cell.forward(state, x_seq)
            h_last = (out[0] if kind == "lstm" else out).chunks((1, n, hidden))[T - 1]      # output[T-1] is h_T
            loss = h_last.mse_loss(tgt_seq)
        else:
            for x in xs:
                state = composed_cell(kind, cell, state, x, n, hidden) if composed else cell.forward(state, x)
            loss = (state[1] if kind == "lstm" else state).mse_loss(tgt)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    return capture(dev, step, 8 << 30)


def torch_step(torch, kind, n, n_in, hidden):
    g = torch.Generator(device="cuda").manual_seed(0)
    cell = (torch.nn.LSTMCell if kind == "lstm" else torch.nn.GRUCell)(n_in, hidden).cuda().to(torch.bfloat16)
    opt = torch.optim.SGD(cell.parameters(), lr=1e-3)
    xs = [(torch.rand(n, n_in, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16) for _ in range(T)]
    tgt = (torch.rand(n, hidden, device="cuda", generator=g) - 0.5).to(torch.bfloat16)
    zero = torch.zeros(n, hidden, device="cuda", dtype=torch.bfloat16)

    def step():
        opt.zero_grad(set_to_none=False)
        state = (zero, zero) if kind == "lstm" else zero
        for x in xs:
            state = cell(x, state)
        h = state[0] if kind == "lstm" else state          # torch returns (h, c)
        torch.nn.functional.mse_loss(h, tgt).backward()
        opt.step()
    return step


def torch_cudnn_step(torch, kind, n, n_in, hidden, layers=1, bidirectional=False):
    g = torch.Generator(device="cuda").manual_seed(0)
    dirs = 2 if bidirectional else 1
    layer = (torch.nn.LSTM if kind == "lstm" else torch.nn.GRU)(n_in, hidden, num_layers=layers,
                                                                bidirectional=bidirectional).cuda().to(torch.bfloat16)
    opt = torch.optim.SGD(layer.parameters(), lr=1e-3)
    x = (torch.rand(T, n, n_in, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    tgt = (torch.rand(n, dirs * hidden, device="cuda", generator=g) - 0.5).to(torch.bfloat16)
    zero = torch.zeros(layers * dirs, n, hidden, device="cuda", dtype=torch.bfloat16)

    def step():
        opt.zero_grad(set_to_none=False)
        out, _ = layer(x, (zero, zero) if kind == "lstm" else zero)
        torch.nn.functional.mse_loss(out[-1], tgt).backward()
        opt.step()
    return step


STACKED = [("unidirectional", 1, False), ("bidirectional", 1, True), ("2_layers_bidirectional", 2, True)]


def stacked_step(nk, dev, kind, n, n_in, hidden, layers, bidirectional):
    """the captured step of nn.LSTM / nn.GRU(num_layers, bidirectional); the loss on the last layer's output[T-1]"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(0)
    dirs = 2 if bidirectional else 1
    stacked = layers > 1 or bidirectional
    m = (nk.nn.LSTM if kind == "lstm" else nk.nn.GRU)(dev, n_in, hidden, nk.BF16, grad_dtype=nk.F32, rng=rng,
                                                       num_layers=layers, bidirectional=bidirectional)
    opt = optim.StochasticGD.new(1e-3)
    for p in m.parameters():
        opt.register(p)
    x = nk.from_ndarray(dev, rng.uniform(-1, 1, (T, n, n_in)).astype(np.float32), nk.BF16)
    zero = nk.zeros(dev, (layers * dirs, n, hidden) if stacked else (n, hidden), nk.BF16)
    tgt = nk.from_ndarray(dev, rng.uniform(-0.5, 0.5, (1, n, dirs * hidden)).astype(np.float32), nk.BF16)

    def step():
        opt.zero_grad()
        out = m.forward((zero, zero), x) if kind == "lstm" else m.forward(zero, x)
        y = out[0] if (kind == "lstm" or stacked) else out
        loss = y.chunks((1, n, dirs * hidden))[T - 1].mse_loss(tgt)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    return capture(dev, step, 12 << 30)   # the GRU's 2 layers x 2 directions at N = 1024, H = 2048 take ~9 GiB


def stacked_row(nk, dev, torch, args, card, kind, n, n_in, hidden):
    graphs = {name: stacked_step(nk, dev, kind, n, n_in, hidden, layers, bi) for name, layers, bi in STACKED}
    cudnn = {name: torch_cudnn_step(torch, kind, n, n_in, hidden, layers, bi) for name, layers, bi in STACKED}
    fns = {}
    for name, _, _ in STACKED:
        fns[name], fns[name + "_torch_cudnn_bf16"] = graphs[name].launch, cudnn[name]
    med, mhz = alternate(fns, args.window_ms, args.reps)
    print(json.dumps({
        "cell": kind, "variant": "stacked", "N": n, "I": n_in, "H": hidden, "T": T,
        "ms_per_sequence": {k: round(v, 3) for k, v in med.items()},
        "launches_per_time_step": {name: round(graphs[name].kernel_count / T, 2) for name, _, _ in STACKED},
        "bidirectional_over_2x_unidirectional": round(med["bidirectional"] / (2 * med["unidirectional"]), 3),
        "speedup_vs_torch_cudnn_bf16": {name: round(med[name + "_torch_cudnn_bf16"] / med[name], 2)
                                        for name, _, _ in STACKED},
        "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"],
    }), flush=True)
    for g in graphs.values():
        g.close()


def sequence_gemms(nk, dev, kind, n, n_in, hidden):
    """the sequence layer's products of one training step in two groups: (whole-sequence fn, sequential fn)"""
    from neuronika_b200 import ops
    G = (4 if kind == "lstm" else 3) * hidden
    r = lambda *s: dev.from_ndarray(np.random.default_rng(1).uniform(-1, 1, s).astype(np.float32), nk.BF16)
    x, hs, h, w_ih, w_hh, b = r(T * n, n_in), r((T - 1) * n, hidden), r(n, hidden), r(G, n_in), r(G, hidden), r(G)
    gates, dg = dev.zeros((T * n, G), nk.F32), r(T * n, G)
    gates_t, dg_t, dg_rest = gates.slice_flat(0, (n, G)), dg.slice_flat(0, (n, G)), dg.slice_flat(n * G, ((T - 1) * n, G))
    dw_ih, dw_hh, dh = dev.zeros((G, n_in), nk.F32), dev.zeros((G, hidden), nk.F32), dev.zeros((n, hidden), nk.F32)

    def whole():
        ops.gemm(x, w_ih, gates, trans_b=True, bias=b)
        ops.gemm(dg_rest, hs, dw_hh, trans_a=True)
        ops.gemm(dg_t, h, dw_hh, trans_a=True, beta=1.0)
        ops.gemm(dg, x, dw_ih, trans_a=True)

    def sequential():
        for _ in range(T):
            ops.gemm(h, w_hh, gates_t, trans_b=True, bias=b, beta=1.0)
        for _ in range(T):
            ops.gemm(dg_t, w_hh, dh)
    return whole, sequential


def gemm_only(nk, dev, torch, kind, n, n_in, hidden):
    """the five products of one cell step, back to back"""
    from neuronika_b200 import ops
    G = (4 if kind == "lstm" else 3) * hidden
    r = lambda *s: dev.from_ndarray(np.random.default_rng(1).uniform(-1, 1, s).astype(np.float32), nk.BF16)
    x, h, w_ih, w_hh, b = r(n, n_in), r(n, hidden), r(G, n_in), r(G, hidden), r(G)
    gates, dg = dev.zeros((n, G), nk.F32), r(n, G)
    dw_ih, dw_hh, dh = dev.zeros((G, n_in), nk.F32), dev.zeros((G, hidden), nk.F32), dev.zeros((n, hidden), nk.BF16)

    def run():
        ops.gemm(x, w_ih, gates, trans_b=True, bias=b)
        ops.gemm(h, w_hh, gates, trans_b=True, bias=b, beta=1.0)
        ops.gemm(dg, x, dw_ih, trans_a=True, beta=1.0)
        ops.gemm(dg, h, dw_hh, trans_a=True, beta=1.0)
        ops.gemm(dg, w_hh, dh)
    flops = 2.0 * n * G * (n_in + hidden) * 2 + 2.0 * n * G * hidden
    return run, flops


def gate_kernels(nk, dev, kind, n, hidden):
    """(fwd fn, fwd bytes, bwd fn, bwd bytes)"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(2)
    s = lambda: dev.from_ndarray(rng.uniform(-1, 1, (n, hidden)).astype(np.float32), nk.BF16)
    if kind == "lstm":
        gates = dev.from_ndarray(rng.standard_normal((n, 4 * hidden)).astype(np.float32))
        c, dh, dc = s(), s(), s()
        co, ho, dcp = dev.zeros((n, hidden), nk.BF16), dev.zeros((n, hidden), nk.BF16), dev.zeros((n, hidden), nk.BF16)
        dg = dev.zeros((n, 4 * hidden), nk.BF16)
        fwd = lambda: ops.lstm_cell(gates, c, co, ho)
        bwd = lambda: ops.lstm_cell_bwd(dg, gates, c, dh, dc, dcp, beta_dc=0.0)
        return fwd, n * hidden * (16 + 2 + 4), bwd, n * hidden * (16 + 2 * 3 + 8 + 2)
    ig = dev.from_ndarray(rng.standard_normal((n, 3 * hidden)).astype(np.float32))
    hg = dev.from_ndarray(rng.standard_normal((n, 3 * hidden)).astype(np.float32))
    h, dh = s(), s()
    ho, dhp = dev.zeros((n, hidden), nk.BF16), dev.zeros((n, hidden), nk.BF16)
    di, dhg = dev.zeros((n, 3 * hidden), nk.BF16), dev.zeros((n, 3 * hidden), nk.BF16)
    fwd = lambda: ops.gru_cell(ig, hg, h, ho)
    bwd = lambda: ops.gru_cell_bwd(di, dhg, ig, hg, h, dh, dhp, beta_dh=0.0)
    return fwd, n * hidden * (24 + 2 + 2), bwd, n * hidden * (24 + 2 * 2 + 12 + 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stacked-only", action="store_true", help="only the stacked / bidirectional rows")
    args = ap.parse_args()
    import torch

    import neuronika_b200 as nk

    dev, card = setup(T=T)
    for kind in ("lstm", "gru"):
        for n, n_in, hidden in SHAPES:
            if args.stacked_only:
                stacked_row(nk, dev, torch, args, card, kind, n, n_in, hidden)
                continue
            fused = graph_step(nk, dev, kind, n, n_in, hidden, "fused")
            comp = graph_step(nk, dev, kind, n, n_in, hidden, "composed")
            seq = graph_step(nk, dev, kind, n, n_in, hidden, "sequence")
            teager = torch_step(torch, kind, n, n_in, hidden)
            tcudnn = torch_cudnn_step(torch, kind, n, n_in, hidden)
            med, mhz = alternate({"fused": fused.launch, "composed": comp.launch, "sequence": seq.launch,
                                  "torch_eager_bf16": teager, "torch_cudnn_bf16": tcudnn}, args.window_ms, args.reps)
            gem, flops = gemm_only(nk, dev, torch, kind, n, n_in, hidden)
            gms, _ = window(gem, args.window_ms / 4, args.reps)
            whole, sequential = sequence_gemms(nk, dev, kind, n, n_in, hidden)
            wms, _ = window(whole, args.window_ms / 4, args.reps)
            sms, _ = window(sequential, args.window_ms / 4, args.reps)
            fwd, fb, bwd, bb = gate_kernels(nk, dev, kind, n, hidden)
            fms, _ = window(fwd, args.window_ms / 4, args.reps)
            bms, _ = window(bwd, args.window_ms / 4, args.reps)
            print(json.dumps({
                "cell": kind, "N": n, "I": n_in, "H": hidden, "T": T,
                "ms_per_sequence": {k: round(v, 3) for k, v in med.items()},
                "ms_per_time_step": {k: round(v / T, 4) for k, v in med.items()},
                "launches_per_time_step": {"fused": round(fused.kernel_count / T, 2),
                                           "composed": round(comp.kernel_count / T, 2),
                                           "sequence": round(seq.kernel_count / T, 2)},
                "speedup_fused_vs_composed": round(med["composed"] / med["fused"], 2),
                "speedup_fused_vs_torch_eager_bf16": round(med["torch_eager_bf16"] / med["fused"], 2),
                "speedup_sequence_vs_fused": round(med["fused"] / med["sequence"], 2),
                "speedup_sequence_vs_torch_cudnn_bf16": round(med["torch_cudnn_bf16"] / med["sequence"], 2),
                "sequence_whole_gemms_ms": round(wms, 3), "sequence_sequential_gemms_ms": round(sms, 3),
                "sequential_gemm_share_of_sequence_step": round(sms / med["sequence"], 3),
                "whole_gemm_share_of_sequence_step": round(wms / med["sequence"], 3),
                "gemm_only_ms_per_time_step": round(gms, 4),
                "gemm_tflops": round(flops / gms / 1e9, 1),
                "gemm_share_of_fused_step": round(gms * T / med["fused"], 3),
                "gate_fwd_us": round(fms * 1e3, 2), "gate_fwd_gbps": round(fb / fms / 1e6, 1),
                "gate_bwd_us": round(bms * 1e3, 2), "gate_bwd_gbps": round(bb / bms / 1e6, 1),
                "median_sm_mhz": mhz, "card": card["name"], "power_limit_w": card["power_limit_w"],
            }), flush=True)
            fused.close()
            comp.close()
            seq.close()
            stacked_row(nk, dev, torch, args, card, kind, n, n_in, hidden)


if __name__ == "__main__":
    main()
