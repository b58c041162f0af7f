#!/usr/bin/env python
"""Where the time of the wgmma GEMM engine goes: a K sweep of the three GEMM forms of the Linear 4096->4096 step.

    python tools/gemm_sweep.py                    # writes a header and one JSON line (and a table on stderr)
    python tools/gemm_sweep.py --root OTHER_TREE  # the same sweep against another build of the package

The three forms exactly as the step calls them (nk_gemm_bias_act):
    NT  y(bf16)  = x.W^T + b(bf16)       NN  dX(bf16) = G.W       TN  dW(f32) = G^T.X
at M = N = 4096 and K in {1024, 2048, 4096, 8192}, on seeded random bf16 operands, timed with CUDA events over many
launches after a warm-up.  Every CTA of the persistent grid runs the same number of 128 x 256 tiles, so a linear fit
time = a.K + b per form splits the launch into
    a . 64 / tiles_per_cta   time per 64-deep k-block per tile -- the main loop -- against the ideal 1024 tensor-core
                             cycles (2.128.256.64 FLOP at 4096 dense bf16 FLOP per cycle and SM) at the sampled SM clock;
    b / tiles_per_cta        the fixed cost per tile: epilogue, pipeline refill, launch.
torch.matmul / linear (cuBLAS) on the same shapes and dtypes is timed the same way as the attainable figure on the card.
Device name, power limit and the median SM clock (NVML) are printed beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

from measure import setup, window

KS = (1024, 2048, 4096, 8192)
MN = 4096
BLOCK_M, BLOCK_N, BLOCK_K = 128, 256, 64
CYCLES_PER_KBLOCK = 2 * BLOCK_M * BLOCK_N * BLOCK_K / 4096     # dense bf16: 4096 FLOP per cycle and SM on H100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="package tree to import (default: this repository)")
    ap.add_argument("--window-ms", type=float, default=100.0, help="length of one timed window of back-to-back calls")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cublas", action="store_true")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch

    import neuronika_b200 as nk
    from neuronika_b200 import ops

    dev, card = setup()
    sm = dev.sm_count
    tiles = (MN // BLOCK_M) * (MN // BLOCK_N)
    waves = -(-tiles // sm)
    grid = -(-tiles // waves)
    tiles_per_cta = tiles / grid

    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *shape: (torch.rand(*shape, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)

    def wrap(t):
        """a CuArray view of a torch tensor (same memory)"""
        return nk.CuArray(dev, tuple(t.shape), nk.BF16 if t.dtype == torch.bfloat16 else nk.F32, ptr=t.data_ptr(), owner=t)

    bias = rnd(MN)
    y16 = torch.empty(MN, MN, device="cuda", dtype=torch.bfloat16)
    y32 = torch.empty(MN, MN, device="cuda", dtype=torch.float32)
    rows = {}
    for form in ("nt_fwd_bias_bf16out", "nn_dx_bf16out", "tn_dw_f32out"):
        rows[form] = []
        for K in KS:
            if form.startswith("nt"):          # x (M, K) . W (N, K)^T + b
                a, b = rnd(MN, K), rnd(MN, K)
                own = lambda: ops.gemm(A, B, C16, trans_b=True, bias=Bias)
                ref = lambda: torch.nn.functional.linear(a, b, bias)
            elif form.startswith("nn"):        # G (M, K) . W (K, N)
                a, b = rnd(MN, K), rnd(K, MN)
                own = lambda: ops.gemm(A, B, C16)
                ref = lambda: torch.matmul(a, b)
            else:                              # G (K, M)^T . X (K, N), f32 out
                a, b = rnd(K, MN), rnd(K, MN)
                own = lambda: ops.gemm(A, B, C32, trans_a=True)
                ref = lambda: torch.mm(a.t(), b, out_dtype=torch.float32)
            A, B, C16, C32, Bias = wrap(a), wrap(b), wrap(y16), wrap(y32), wrap(bias)
            ms, mhz = window(own, args.window_ms, args.reps)
            row = {"K": K, "ms": round(ms, 5), "sm_mhz": mhz, "kcycles": round(ms * mhz, 1),
                   "tflops": round(2.0 * MN * MN * K / ms / 1e9, 1), "kernel": dev.last_gemm_kernel}
            if not args.no_cublas:
                try:
                    cms, cmhz = window(ref, args.window_ms, args.reps)
                    row.update(cublas_ms=round(cms, 5), cublas_sm_mhz=cmhz, cublas_kcycles=round(cms * cmhz, 1),
                               cublas_tflops=round(2.0 * MN * MN * K / cms / 1e9, 1))
                except Exception as e:  # noqa: BLE001 -- an older torch without out_dtype: leave the column out
                    row["cublas_error"] = repr(e)[:120]
            rows[form].append(row)
            del a, b, A, B
    torch.cuda.synchronize()

    fits = {}
    for form, rs in rows.items():
        k = np.array([r["K"] for r in rs], float)
        fit = {}
        for key in ("ms", "cublas_ms"):
            if not all(key in r for r in rs):
                continue
            a, b = np.polyfit(k, np.array([r[key] for r in rs]), 1)
            mhz = float(np.median([r["sm_mhz" if key == "ms" else "cublas_sm_mhz"] for r in rs]))
            kblock_us = a * BLOCK_K / tiles_per_cta * 1e3
            # the same fit in SM cycles (time x the clock sampled during that point): a power-limited card changes its
            # clock from point to point, which bends a fit in time
            ck = "kcycles" if key == "ms" else "cublas_kcycles"
            ac, bc = np.polyfit(k, np.array([r[ck] for r in rs]), 1)
            kblock_cyc = ac * 1e3 * BLOCK_K / tiles_per_cta
            fit[key.replace("ms", "fit")] = {
                "slope_us_per_kblock_per_tile": round(kblock_us, 4),
                "ideal_us_per_kblock_at_clock": round(CYCLES_PER_KBLOCK / mhz, 4),
                "main_loop_frac_of_tensor_rate": round(CYCLES_PER_KBLOCK / mhz / kblock_us, 4),
                "intercept_us_per_tile": round(b / tiles_per_cta * 1e3, 3), "intercept_ms": round(b, 5),
                "sm_mhz": mhz,
                "slope_cycles_per_kblock_per_tile": round(kblock_cyc, 1),
                "main_loop_frac_of_tensor_rate_cycles": round(CYCLES_PER_KBLOCK / kblock_cyc, 4),
                "intercept_kcycles_per_tile": round(bc / tiles_per_cta, 2)}
        fits[form] = fit
    out = {"what": "K sweep of the Linear step's three GEMM forms at M = N = 4096; fit time = a.K + b",
           "card": card, "sm_count": sm, "grid": grid, "tiles_per_cta": tiles_per_cta,
           "window_ms": args.window_ms, "reps": args.reps, "root": os.path.abspath(args.root), "rows": rows, "fits": fits}
    for form, rs in rows.items():
        print(form, file=sys.stderr)
        for r in rs:
            print(f"  K={r['K']:5d}  own {r['ms']:.4f} ms {r['tflops']:6.1f} TF/s @{r['sm_mhz']:.0f} MHz   "
                  f"cublas {r.get('cublas_ms', float('nan')):.4f} ms {r.get('cublas_tflops', float('nan')):6.1f} TF/s",
                  file=sys.stderr)
        for key, f in fits[form].items():
            print(f"  {key}: {json.dumps(f)}", file=sys.stderr)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
