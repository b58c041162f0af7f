"""The 1-D / 3-D convolution layers' im2col engine (nk_conv_gemm_nd_*, nk_conv_gemm.cu) at the places where it branches,
checked EXACTLY rather than within a rounding bound.

Exact arithmetic: the operands are small integers (x, w, g, bias, fill and the accumulated-into old values in {-2..2},
most of them sparse) or one-hot kernels, so every product is exact, and as long as every partial sum is an integer of at
most 2^24 an f32 sum of them is exact in any order (the wgmma accumulators, the f32 column gradients, the split
reduction of dW, f32 atomics).  A bf16 output is then exact when |value| <= 256, an f32 one when |value| <= 2^20 (the
limits these tests keep, with room).  The largest partial sum any summation order can form is sum|terms|, which the
oracle computes on absolute values; `exact_regime` asserts it is within the limit for every output of every call, so an
edit that takes a case out of the exact regime fails loudly instead of passing on a rounding.  Inside the regime every
result must EQUAL the float64 oracle, and the tensor-core engine, the bf16 layer under conv_engine("direct") and the f32
CUDA-core layer must give identical results.

Covered:
  - the padding map (pad_src_index) of all four modes in 1-D and 3-D at its limits: reflective pad = len - 1,
    replicative pad > len and len = 1, a kernel wider than the unpadded input, an output extent of 1, and a dilation
    whose taps read only the padding (y = fill.sum(w) + b, dX = beta.dx0);
  - the three gather branches of im2col_nd_kernel, one at a time, with one-hot kernels: y[:, o] is then a strided window
    of the padded input, compared bit for bit with nk_padnd_fwd's output on the same device operand, including fills
    that bf16 cannot represent (0.1, -1/3);
  - the tile boundaries of the three batched GEMMs (BLOCK_M 128, BLOCK_K 64, block_n 64 / 128 / 256) over Cout, K and L,
    in 1-D and 3-D, and through the 2-D entry points that share the same drivers;
  - the applicability rules (K = 8 / 9, Cout 7 / 12, x, g and out= views off alignment);
  - 3-D sample chunking of the column buffers across 2 (bf16) and 3 (f32) chunks;
  - the reference's padded goldens (tests/golden/tensors_pad.json) through the layer as an identity convolution."""
import json
import os

import numpy as np
import pytest

from test_gpu_conv_edges import offset_view
from test_gpu_conv_layer import DIRECT, MODES, ORACLE_MODE, WGMMA
from test_gpu_cuda_core_conv_edges import rounded

pytestmark = pytest.mark.gpu

F32 = np.float32
BF16_EXACT = 256          # every integer of magnitude <= 256 is a bf16 value
F32_EXACT = 2 ** 20       # far below 2^24: any f32 sum of such integers is exact
WG2 = ("wgmma_im2col_gemm_fwd", "wgmma_im2col_gemm_dx", "wgmma_im2col_gemm_dw")


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


# ------------------------------------------------------------------------------------------- exact-arithmetic helpers
def exact_regime(mag, bf16_out, what):
    """mag = sum|terms| per output (the oracle on absolute values, plus |beta.old| and |bias|): the largest partial sum
    any order of summation can form.  Asserts every output stays where integer arithmetic is exact."""
    mag = np.asarray(mag, np.float64)
    limit = BF16_EXACT if bf16_out else F32_EXACT
    assert float(mag.max(initial=0.0)) <= limit, ("out of the exact regime", what, float(mag.max()), limit)


def ints(rng, shape, density=1.0, hi=2):
    """integers in {-hi..hi} \\ {0} where a uniform draw falls below `density`, 0 elsewhere"""
    v = rng.integers(1, hi + 1, shape) * rng.choice([-1, 1], shape)
    return np.where(rng.uniform(0, 1, shape) < density, v, 0).astype(F32)


def densities(counts, target=12.0):
    """densities of the operands x, w, g such that each product's expected number of non-zero terms (count.d_a.d_b
    for its pair of operands) is at most `target`: the three GEMMs sum K (x.w), Cout.prod(k) (g.w) and N.L (g.x)
    terms, the last into dW that is also checked in bf16"""
    d = {"x": 1.0, "w": 1.0, "g": 1.0}
    for (a, b), cnt in sorted(counts.items(), key=lambda kv: -kv[1]):
        p = d[a] * d[b] * cnt
        if p > target:
            s = np.sqrt(target / p)
            d[a] *= s
            d[b] *= s
    return d


def equal(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got != want
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist(), got[bad][:4].tolist(),
                           want[bad][:4].tolist())


def padded_shape(xs, pad):
    return tuple(xs[:2]) + tuple(s + 2 * p for s, p in zip(xs[2:], pad))


def oracle_fwd(O, x, w, b, pad, mode, fill, stride, dil):
    om = ORACLE_MODE[mode]
    xp = O.pad_mode_forward(x.astype(np.float64), pad, om, fill)
    xpa = O.pad_mode_forward(np.abs(x).astype(np.float64), pad, om, abs(fill))
    bb = b.astype(np.float64).reshape((1, -1) + (1,) * len(pad))
    y = O.conv_forward(xp, w.astype(np.float64), stride, dil).astype(np.float64) + bb
    mag = O.conv_forward(xpa, np.abs(w).astype(np.float64), stride, dil).astype(np.float64) + np.abs(bb)
    return y, mag, xp, xpa


def oracle_dx_full(O, xs, g, w, pad, stride, dil):
    """(interior slice of the padded input's gradient, |terms| of the whole padded gradient)"""
    padded = padded_shape(xs, pad)
    gp = O.conv_backward_input(np.zeros(padded), g.astype(np.float64), w.astype(np.float64), stride, dil)
    gpa = O.conv_backward_input(np.zeros(padded), np.abs(g).astype(np.float64), np.abs(w).astype(np.float64), stride, dil)
    return O.pad_mode_backward(gp, np.zeros(xs), pad), gpa


ENGINES = {   # name: (data type, conv_engine, the kernels each call must take when the wgmma engine applies)
    "wgmma": ("bf16", "auto", WGMMA),
    "direct_bf16": ("bf16", "direct", DIRECT),
    "f32": ("f32", "auto", DIRECT),
}


def exact_case(nk, dev, O, xs, cout, k, pad, mode, stride, dil, *, engine="wgmma", kernels=None, seed=0, fill=None,
               target=12.0):
    """the forward (with bias), dX (beta 0 and 1), dW + db into f32 and bf16 (beta 0 and 1) of the layer on integer
    operands, each EQUAL to the float64 oracle; returns the results {name: array} so engines can be compared"""
    from neuronika_b200 import ops
    bf = ENGINES[engine][0] == "bf16"
    dt = nk.BF16 if bf else nk.F32
    kernels = kernels or ENGINES[engine][2]
    rng = np.random.default_rng(seed)
    n, cin = xs[:2]
    nsp = len(k)
    ksz = int(np.prod(k))
    if fill is None:
        fill = -1.0 if mode == "constant" else 0.0
    mode_c = "constant" if mode == "zero" else mode
    out_sp = [(s + 2 * p - d * (kk - 1) - 1) // st + 1 for s, p, d, kk, st in zip(xs[2:], pad, dil, k, stride)]
    L = int(np.prod(out_sp))
    d = densities({("x", "w"): cin * ksz, ("g", "w"): cout * ksz, ("g", "x"): n * L}, target)
    x = ints(rng, xs, d["x"])
    w = ints(rng, (cout, cin) + tuple(k), d["w"])
    b = ints(rng, (cout,))
    X, W, B = dev.from_ndarray(x, dt), dev.from_ndarray(w, dt), dev.from_ndarray(b, dt)
    res = {}
    if ENGINES[engine][1] != "auto":
        dev.conv_engine(ENGINES[engine][1])
    try:
        want, mag, xp, xpa = oracle_fwd(O, x, w, b, pad, mode, fill, stride, dil)
        exact_regime(mag, bf, "y")
        if bf and kernels[0].startswith("direct"):    # the composed path stores the convolution before the bias add
            exact_regime(mag, True, "y before the bias")
        y = ops.conv_layer_nd(X, W, pad, mode_c, fill, stride, dil, bias=B)
        assert dev.last_conv_kernel == kernels[0], (dev.last_conv_kernel, kernels)
        res["y"] = y.as_ndarray()
        equal(res["y"], want, ("y", engine))

        g = ints(rng, want.shape, d["g"])
        G = dev.from_ndarray(g, dt)
        gx, gpa = oracle_dx_full(O, xs, g, w, pad, stride, dil)
        dx0 = ints(rng, xs)
        for beta in (0.0, 1.0):
            exact_regime(gpa.max() + beta * 2, bf, ("dx", beta))
            DX = dev.from_ndarray(dx0, dt)
            ops.conv_layer_nd_bwd_input(DX, G, W, pad, mode_c, stride, dil, beta=beta)
            assert dev.last_conv_kernel == kernels[1], (dev.last_conv_kernel, kernels)
            res["dx", beta] = DX.as_ndarray()
            equal(res["dx", beta], beta * dx0 + gx, ("dx", beta, engine))

        g64 = g.astype(np.float64)
        gw = O.conv_backward_kernel(np.zeros(w.shape), g64, xp, stride, dil)
        gw_mag = O.conv_backward_kernel(np.zeros(w.shape), np.abs(g64), xpa, stride, dil)
        axes = tuple(i for i in range(g.ndim) if i != 1)
        gb, gb_mag = g64.sum(axis=axes), np.abs(g64).sum(axis=axes)
        for dwt in (nk.F32, nk.BF16):
            dbf = dwt == nk.BF16
            dw0, db0 = ints(rng, w.shape), ints(rng, (cout,))
            for beta in (0.0, 1.0):
                exact_regime(gw_mag + beta * 2, dbf, ("dw", dbf, beta))
                exact_regime(gb_mag + beta * 2, dbf, ("db", dbf, beta))
                DW, DB = dev.from_ndarray(dw0, dwt), dev.from_ndarray(db0, dwt)
                ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, mode_c, fill, stride, dil, beta=beta, dbias=DB)
                assert dev.last_conv_kernel == kernels[2], (dev.last_conv_kernel, kernels)
                res["dw", dbf, beta] = DW.as_ndarray()
                equal(res["dw", dbf, beta], beta * dw0 + gw, ("dw", dbf, beta, engine))
                equal(DB.as_ndarray(), beta * db0 + gb, ("db", dbf, beta, engine))
    finally:
        dev.conv_engine("auto")
    return res


# ------------------------------------------------------------------------------------------- the padding map
# name: (x shape, cout, kernel, padding, stride, dilation, modes)
ALL = tuple(MODES)
NO_REFLECT = ("zero", "constant", "replicative")
PAD_EDGES = {
    # reflective pad = len - 1: the first and last padded coordinates mirror onto the far ends of x
    "1d_pad_len_minus_1": ((2, 16, 5), 8, (3,), (4,), (1,), (1,), ALL),
    "3d_pad_len_minus_1": ((2, 2, 3, 4, 5), 8, (3, 2, 3), (2, 3, 4), (1, 1, 1), (1, 1, 1), ALL),
    # replicative pad > len (reflective cannot pad this far)
    "1d_pad_beyond_len": ((2, 8, 3), 8, (2,), (5,), (1,), (1,), NO_REFLECT),
    "3d_pad_beyond_len": ((2, 2, 2, 3, 2), 8, (2, 2, 3), (3, 4, 3), (1, 1, 1), (1, 1, 1), NO_REFLECT),
    # len = 1: every padded coordinate is the one element (or the fill)
    "1d_len_1": ((3, 16, 1), 8, (3,), (3,), (1,), (1,), NO_REFLECT),
    "3d_len_1": ((2, 2, 1, 1, 1), 8, (2, 2, 3), (1, 2, 3), (1, 1, 1), (1, 1, 1), NO_REFLECT),
    # the kernel spans more than the unpadded input
    "1d_kernel_wider_than_input": ((2, 4, 4), 8, (7,), (3,), (1,), (1,), ALL),
    "3d_kernel_wider_than_input": ((2, 2, 2, 3, 4), 8, (3, 4, 6), (1, 2, 3), (1, 1, 1), (1, 1, 1), ALL),
    # an output extent of 1 (L = 1: one output per row of Lp = 8, seven zero pad columns)
    "1d_output_extent_1": ((3, 4, 5), 8, (7,), (1,), (1,), (1,), ALL),
    "3d_output_extent_1": ((2, 2, 3, 2, 4), 8, (3, 4, 2), (1, 1, 0), (2, 1, 3), (1, 1, 3), ALL),
    # every tap reads padding: padded length 19, taps 13 apart from p in 0..5, the interior is 6..12
    "1d_taps_only_in_padding": ((2, 8, 7), 8, (2,), (6,), (1,), (13,), ALL),
    "3d_taps_only_in_padding": ((2, 4, 2, 3, 7), 8, (1, 2, 2), (1, 1, 6), (1, 1, 1), (1, 2, 13), ALL),
}
PAD_EDGE_CASES = [(name, mode) for name, c in PAD_EDGES.items() for mode in c[6]]


@pytest.mark.parametrize("name,mode", PAD_EDGE_CASES)
def test_padding_map_edges(nk, dev, O, name, mode):
    """each case exact on the tensor cores, under conv_engine("direct") and in f32 on the CUDA cores, so the three
    engines agree bit for bit"""
    xs, cout, k, pad, s, d, _ = PAD_EDGES[name]
    seed = sum(xs) + len(mode)
    res = {e: exact_case(nk, dev, O, xs, cout, k, pad, mode, s, d, engine=e, seed=seed) for e in ENGINES}
    for key in res["wgmma"]:
        equal(res["wgmma"][key], res["direct_bf16"][key], ("engines", key))
        equal(res["wgmma"][key], res["f32"][key], ("f32", key))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["1d_taps_only_in_padding", "3d_taps_only_in_padding"])
def test_taps_only_in_padding(nk, dev, O, name, mode):
    """no tap reaches the interior: y = fill.sum(w) + b in the constant modes, and dX is exactly beta.dx0 in every mode
    (the gradient of the padding is dropped, pad/mod.rs:157-182)"""
    from neuronika_b200 import ops
    xs, cout, k, pad, s, d, _ = PAD_EDGES[name]
    rng = np.random.default_rng(7)
    x, w, b = ints(rng, xs), ints(rng, (cout, xs[1]) + k, 0.5), ints(rng, (cout,))
    fill = {"zero": 0.0, "constant": 1.0}.get(mode, 0.0)
    mode_c = "constant" if mode == "zero" else mode
    X, W, B = (dev.from_ndarray(a, nk.BF16) for a in (x, w, b))
    y = ops.conv_layer_nd(X, W, pad, mode_c, fill, s, d, bias=B)
    assert dev.last_conv_kernel == WGMMA[0]
    want, mag, _, _ = oracle_fwd(O, x, w, b, pad, mode, fill, s, d)
    exact_regime(mag, True, "y")
    equal(y.as_ndarray(), want, "y")
    if mode in ("zero", "constant"):
        per_o = fill * w.reshape(cout, -1).astype(np.float64).sum(1) + b
        equal(y.as_ndarray(), np.broadcast_to(per_o.reshape((1, cout) + (1,) * len(k)), want.shape), "fill.sum(w) + b")
    g = ints(rng, want.shape)
    dx0 = ints(rng, xs)
    for beta in (0.0, 1.0):
        DX = dev.from_ndarray(dx0, nk.BF16)
        ops.conv_layer_nd_bwd_input(DX, dev.from_ndarray(g, nk.BF16), W, pad, mode_c, s, d, beta=beta)
        assert dev.last_conv_kernel == WGMMA[1]
        equal(DX.as_ndarray(), beta * dx0, ("dx", beta))


# ------------------------------------------------------------------------------------------- the gather branches
def gather_branches(xs, k, pad, mode, stride, dil):
    """which branch of im2col_nd_kernel each (sample, k, vector of 8 outputs) takes -- the kernel's conditions restated
    over the padded-to-3 geometry: 'fill_row', 'run_even', 'run_odd', 'run_last' (a run that ends on x's last element),
    'border', 'elementwise'"""
    nsp = len(k)
    one = [1] * (3 - nsp)
    inn, kk, ss, dd = one + list(xs[2:]), one + list(k), one + list(stride), one + list(dil)
    pp = [0] * (3 - nsp) + list(pad)
    out = [(i + 2 * p - d * (q - 1) - 1) // s + 1 for i, p, d, q, s in zip(inn, pp, dd, kk, ss)]
    L, Lp = int(np.prod(out)), -(-int(np.prod(out)) // 8) * 8
    x_elems = int(np.prod(xs))

    def src(u, length, p):
        if p <= u < length + p:
            return u - p
        if mode == "reflective":
            return (2 * p - u if u < p else 2 * (length + p - 1) - u) - p
        if mode == "replicative":
            return 0 if u < p else length - 1
        return -1

    seen = set()
    isz = int(np.prod(inn))
    for ns in range(xs[0]):
        for c in range(xs[1]):
            plane = (ns * xs[1] + c) * isz
            for i0 in range(kk[0]):
                for i1 in range(kk[1]):
                    for i2 in range(kk[2]):
                        for l0 in range(0, Lp, 8):
                            q, r = l0 % out[2], l0 // out[2]
                            if not (ss[2] == 1 and q + 8 <= out[2] and l0 + 8 <= L):
                                seen.add("elementwise")
                                continue
                            r0 = src((r // out[1]) * ss[0] + i0 * dd[0], inn[0], pp[0])
                            r1 = src((r % out[1]) * ss[1] + i1 * dd[1], inn[1], pp[1])
                            u2 = q + i2 * dd[2] - pp[2]
                            if r0 < 0 or r1 < 0:
                                seen.add("fill_row")
                            elif u2 >= 0 and u2 + 8 <= inn[2]:
                                off = plane + (r0 * inn[1] + r1) * inn[2] + u2
                                seen.add("run_odd" if off & 1 else "run_even")
                                if off + 8 == x_elems:
                                    seen.add("run_last")
                            else:
                                seen.add("border")
    return seen


# name: (x shape, kernel, padding, mode, stride, dilation, fill, the branches it must take)
GATHER = {
    # constant 3-D padding puts whole source rows outside x; interior runs at both parities, border runs
    "3d_constant_rows_in_padding": ((2, 3, 3, 4, 21), (2, 3, 3), (1, 2, 1), "constant", (1, 1, 1), (1, 1, 1), 0.75,
                                    {"fill_row", "run_even", "run_odd", "border"}),
    # unpadded 1-D: every vector but the tail is an interior run; odd x extent and odd Cin: the run of the last sample's
    # last channel at tap 1 ends on x's last element at an odd element offset (the fifth word's guarded load)
    "1d_run_ends_on_last_element_odd": ((1, 9, 25), (2,), (0,), "zero", (1,), (1,), 0.0,
                                        {"run_even", "run_odd", "run_last"}),
    "1d_run_ends_on_last_element_even": ((2, 8, 25), (2,), (0,), "zero", (1,), (1,), 0.0,
                                         {"run_even", "run_odd", "run_last"}),
    # reflective border runs along the last axis, dilated taps (d2 = 2) on the run path (an odd x extent: both parities)
    "1d_border_runs_dilated": ((2, 8, 41), (3,), (5,), "reflective", (1,), (2,), 0.0,
                               {"run_even", "run_odd", "border"}),
    # last-axis stride 2: element-wise only
    "1d_stride_2": ((2, 8, 37), (3,), (2,), "replicative", (2,), (1,), 0.0, {"elementwise"}),
    "3d_stride_2_dilation_2": ((2, 2, 4, 5, 19), (2, 2, 3), (1, 1, 2), "reflective", (1, 2, 2), (2, 1, 2), 0.0,
                               {"elementwise"}),
    # o2 = 5: every vector wraps an output row (o2 % 8 != 0), L % 8 != 0
    "3d_wrapping_vectors": ((2, 2, 3, 4, 5), (2, 2, 3), (1, 1, 1), "replicative", (1, 1, 1), (1, 1, 1), 0.0,
                            {"elementwise"}),
    # o2 = 13: runs and wrapping vectors in the same rows
    "3d_runs_and_wraps": ((2, 2, 3, 3, 11), (1, 2, 3), (0, 1, 2), "constant", (1, 1, 1), (1, 1, 1), 0.5,
                          {"fill_row", "run_even", "run_odd", "border", "elementwise"}),
    # L = 43: the L tail is gathered element by element; fills that bf16 cannot represent
    "1d_tail_fill_0.1": ((2, 8, 41), (3,), (2,), "constant", (1,), (1,), 0.1,
                         {"run_even", "run_odd", "border", "elementwise"}),
    "3d_fill_minus_third": ((2, 2, 3, 3, 17), (2, 2, 3), (1, 1, 1), "constant", (1, 1, 1), (1, 1, 1), -1.0 / 3.0,
                            {"fill_row", "run_even", "run_odd", "border", "elementwise"}),
}


def test_gather_cases_take_every_branch():
    seen = set()
    for name, (xs, k, pad, mode, s, d, _, want) in GATHER.items():
        got = gather_branches(xs, k, pad, mode, s, d)
        assert want <= got, (name, sorted(got))
        assert xs[1] * int(np.prod(k)) > 8, (name, "K = 8 or less runs on the CUDA cores")
        seen |= got
    assert seen == {"fill_row", "run_even", "run_odd", "run_last", "border", "elementwise"}


@pytest.mark.parametrize("name", list(GATHER))
def test_gather_branches_one_hot(nk, dev, O, name):
    """w[o] = 1 at one (c, tap) per output channel, every (c, tap) once: y[:, o] is the strided window of the padded
    input at that tap, compared bit for bit with ops.pad_nd (nk_padnd_fwd) of the same device operand, sliced -- the
    fill bits included"""
    from neuronika_b200 import ops
    xs, k, pad, mode, s, d, fill, _ = GATHER[name]
    rng = np.random.default_rng(len(name))
    n, cin = xs[:2]
    nsp = len(k)
    taps = [np.unravel_index(t, k) for t in range(int(np.prod(k)))]
    pairs = [(c, t) for c in range(cin) for t in taps]
    cout = max(8, -(-len(pairs) // 8) * 8)
    w = np.zeros((cout, cin) + tuple(k), F32)
    for o in range(cout):
        c, t = pairs[o % len(pairs)]
        w[(o, c) + tuple(t)] = 1.0
    x = rounded(O, rng.uniform(-4, 4, xs), True)
    X, W = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16)
    mode_c = "constant" if mode == "zero" else mode
    y = ops.conv_layer_nd(X, W, pad, mode_c, fill, s, d)
    assert dev.last_conv_kernel == WGMMA[0]
    xp = ops.pad_nd(X, pad, mode_c, fill).as_ndarray()
    got = y.as_ndarray()
    out_sp = got.shape[2:]
    for o in range(cout):
        c, t = pairs[o % len(pairs)]
        sl = tuple(slice(ti * di, ti * di + si * (oi - 1) + 1, si) for ti, di, si, oi in zip(t, d, s, out_sp))
        want = xp[(slice(None), c) + sl]
        assert np.array_equal(got[:, o], want), (name, o, c, t)
        nz = want != 0
        assert np.array_equal(got[:, o][nz].view(np.uint32), want[nz].view(np.uint32)), (name, o)
    if mode == "constant":
        want_fill = O.bf16_round(np.asarray([fill], F32))[0]
        border = np.ones(xp.shape[2:], bool)
        border[tuple(slice(p, p + e) for p, e in zip(pad, xs[2:]))] = False
        assert np.all(xp[:, :, border].view(np.uint32) == np.asarray(want_fill, F32).view(np.uint32)), "pad_nd fill"
    assert nsp == len(pad)


# ------------------------------------------------------------------------------------------- GEMM tile boundaries
COUTS = (8, 9, 120, 128, 136, 256, 264)
KS = (9, 15, 16, 17, 63, 64, 65, 128, 129, 200)
LS = (1, 7, 8, 9, 63, 64, 65, 128, 129, 256, 257)
# K = Cin . prod(k): (Cin, kernel) per K, 1-D and 3-D
K_1D = {9: (3, (3,)), 15: (5, (3,)), 16: (8, (2,)), 17: (17, (1,)), 63: (21, (3,)), 64: (16, (4,)), 65: (13, (5,)),
        128: (32, (4,)), 129: (43, (3,)), 200: (40, (5,))}
K_3D = {9: (1, (3, 1, 3)), 15: (5, (1, 1, 3)), 16: (2, (2, 2, 2)), 17: (17, (1, 1, 1)), 63: (7, (3, 3, 1)),
        64: (8, (2, 2, 2)), 65: (13, (1, 5, 1)), 128: (16, (2, 2, 2)), 129: (43, (1, 3, 1)), 200: (8, (5, 1, 5))}
# L = prod(output extents): 3-D extents per L (o2 % 8 != 0 for most of them)
L_3D = {1: (1, 1, 1), 7: (1, 1, 7), 8: (1, 2, 4), 9: (1, 3, 3), 63: (3, 3, 7), 64: (4, 4, 4), 65: (1, 5, 13),
        128: (2, 8, 8), 129: (3, 1, 43), 256: (4, 8, 8), 257: (1, 1, 257), 300: (3, 10, 10)}
# (nsp, Cout, K, L): every value of each axis at least once in 1-D and in 3-D, plus L = 300 / 1001 (> 256, % 8 != 0)
SWEEP = [
    (1, 8, 9, 1), (1, 9, 15, 7), (1, 120, 16, 8), (1, 128, 17, 9), (1, 136, 63, 63), (1, 256, 64, 64),
    (1, 264, 65, 65), (1, 128, 128, 128), (1, 8, 129, 129), (1, 136, 200, 256), (1, 264, 9, 257), (1, 120, 64, 1001),
    (3, 8, 200, 1), (3, 9, 129, 7), (3, 120, 128, 8), (3, 128, 65, 9), (3, 136, 64, 63), (3, 256, 63, 64),
    (3, 264, 17, 65), (3, 128, 16, 128), (3, 8, 15, 129), (3, 136, 9, 256), (3, 264, 64, 257), (3, 256, 128, 300),
]


def sweep_shape(nsp, K, L):
    """(x shape without N, kernel, padding, mode): input extents that give output extents L (1-D) / L_3D[L] with
    padding 1 where the input can take it"""
    cin, k = (K_1D if nsp == 1 else K_3D)[K]
    outs = (L,) if nsp == 1 else L_3D[L]
    sp, pad = [], []
    for o, kk in zip(outs, k):
        p = 1 if o + kk - 1 - 2 >= 2 else 0
        sp.append(o + kk - 1 - 2 * p)
        pad.append(p)
    return (cin,) + tuple(sp), k, tuple(pad)


def test_sweep_covers_every_value():
    for nsp in (1, 3):
        rows = [r for r in SWEEP if r[0] == nsp]
        assert {r[1] for r in rows} == set(COUTS), nsp
        assert {r[2] for r in rows} == set(KS), nsp
        assert set(LS) <= {r[3] for r in rows} and any(r[3] > 256 and r[3] % 8 for r in rows), nsp
    for nsp, cout, K, L in SWEEP:
        inner, k, pad = sweep_shape(nsp, K, L)
        outs = [s + 2 * p - kk + 1 for s, p, kk in zip(inner[1:], pad, k)]
        assert inner[0] * int(np.prod(k)) == K and int(np.prod(outs)) == L and min(inner[1:]) >= 1, (nsp, K, L)


@pytest.mark.parametrize("nsp,cout,K,L", SWEEP, ids=[f"{n}d-cout{c}-K{k}-L{l}" for n, c, k, l in SWEEP])
def test_tile_boundaries(nk, dev, O, nsp, cout, K, L):
    """integer operands, every result equal to the oracle; dX on the tensor cores only where Cout % 8 == 0"""
    inner, k, pad = sweep_shape(nsp, K, L)
    modes = ("replicative", "reflective", "zero", "constant")
    mode = modes[(cout + K + L) % 4]
    if mode == "reflective" and any(p >= s for p, s in zip(pad, inner[1:])):
        mode = "replicative"
    kernels = WGMMA if cout % 8 == 0 else (WGMMA[0], DIRECT[1], WGMMA[2])
    exact_case(nk, dev, O, (2,) + inner, cout, k, pad, mode, (1,) * nsp, (1,) * nsp, kernels=kernels,
               seed=cout * 7 + K * 3 + L)


# ------------------------------------------------------------------------------------------- applicability rules
@pytest.mark.parametrize("case", ["K8_direct", "K9_wgmma", "cout7", "cout12"])
def test_fallback_boundaries(nk, dev, O, case):
    """the fallback's results equal the oracle exactly, as the engine's do: K = Cin.prod(k) = 8 (Kp < 16) runs on the
    CUDA cores, K = 9 on wgmma; Cout 7 sends the forward and dX to the CUDA cores, Cout 12 only dX"""
    xs, cout, k, kernels = {
        "K8_direct": ((2, 4, 2, 3, 9), 16, (1, 1, 2), DIRECT),
        "K9_wgmma": ((2, 1, 4, 5, 9), 16, (1, 3, 3), WGMMA),
        "cout7": ((2, 4, 23), 7, (3,), (DIRECT[0], DIRECT[1], WGMMA[2])),
        "cout12": ((2, 2, 3, 4, 11), 12, (2, 2, 3), (WGMMA[0], DIRECT[1], WGMMA[2])),
    }[case]
    nsp = len(k)
    exact_case(nk, dev, O, xs, cout, k, (1,) * nsp, "reflective", (1,) * nsp, (1,) * nsp, kernels=kernels,
               seed=len(case))


@pytest.mark.parametrize("view", ["x_off1", "x_off2", "g_off1", "out_off1"])
def test_views_off_alignment(nk, dev, O, view):
    """x one element (2 bytes) off 4-byte alignment: the forward and dW go to the CUDA cores; two elements off: they stay
    on wgmma, the odd-offset runs reading through load_run8's funnel shift; g one element off: copied into padded rows
    (L = 240, a multiple of 8, so only the alignment forces the copy); out= one element off: the forward goes to the CUDA
    cores.  Every result equal to the oracle."""
    from neuronika_b200 import ops
    xs, cout, k, pad, mode = (2, 8, 3, 4, 16), 16, (1, 2, 3), (0, 1, 1), "replicative"
    s = d = (1, 1, 1)
    rng = np.random.default_rng(11)
    x, w, b = ints(rng, xs, 0.5), ints(rng, (cout, xs[1]) + k, 0.5), ints(rng, (cout,))
    want, mag, xp, xpa = oracle_fwd(O, x, w, b, pad, mode, 0.0, s, d)
    exact_regime(mag, True, "y")
    g = ints(rng, want.shape, 0.5)
    assert want.shape[2:] == (3, 5, 16) and int(np.prod(want.shape[2:])) % 8 == 0
    x_off = {"x_off1": 1, "x_off2": 2}.get(view, 0)
    X = offset_view(dev, x, nk.BF16, x_off)
    W, B = dev.from_ndarray(w, nk.BF16), dev.from_ndarray(b, nk.BF16)
    G = offset_view(dev, g, nk.BF16, 1 if view == "g_off1" else 0)
    fwd_dw = DIRECT if view == "x_off1" else WGMMA
    out = offset_view(dev, np.zeros(want.shape, F32), nk.BF16, 1) if view == "out_off1" else None
    y = ops.conv_layer_nd(X, W, pad, mode, 0.0, s, d, bias=B, out=out)
    assert dev.last_conv_kernel == (DIRECT[0] if view == "out_off1" else fwd_dw[0])
    equal(y.as_ndarray(), want, "y")
    gx, gpa = oracle_dx_full(O, xs, g, w, pad, s, d)
    exact_regime(gpa, True, "dx")
    DX = dev.zeros(xs, nk.BF16)
    ops.conv_layer_nd_bwd_input(DX, G, W, pad, mode, s, d, beta=0.0)
    assert dev.last_conv_kernel == WGMMA[1]
    equal(DX.as_ndarray(), gx, "dx")
    gw = O.conv_backward_kernel(np.zeros(w.shape), g.astype(np.float64), xp, s, d)
    gw_mag = O.conv_backward_kernel(np.zeros(w.shape), np.abs(g).astype(np.float64), xpa, s, d)
    exact_regime(gw_mag, False, "dw")
    DW = dev.zeros(w.shape, nk.F32)
    ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, mode, 0.0, s, d, beta=0.0)
    assert dev.last_conv_kernel == fwd_dw[2]
    equal(DW.as_ndarray(), gw, "dw")


# ------------------------------------------------------------------------------------------- 3-D sample chunking
def chunk_samples(Lp, Kp, elem_bytes, n):
    """samples per column-buffer chunk (nk_conv_gemm.cu chunk_samples): floor(4 GiB / (Lp.Kp.elem_bytes)), at most N"""
    return max(1, min(n, (4 << 30) // (Lp * Kp * elem_bytes)))


def test_3d_sample_chunking(nk, dev, O):
    """(N, 4, 12, 16, 16), k 3^3, replicative pad 1: L = Lp = 12.16.16 = 3072 and Kp = ceil8(4.27) = 112 per sample,
    so a 4 GiB chunk holds chunk_samples(3072, 112, 2) = 6241 samples of bf16 columns (forward, dW) and
    chunk_samples(3072, 112, 4) = 3120 of f32 column gradients (dX).  N = 6500 runs the forward and dW in 2 chunks and
    dX in 3, each with a partial last chunk.  x repeats a pool of 61 distinct integer samples (61 divides no chunk
    size); g is zero except on the samples on both sides of every chunk boundary (and the first and last), so dX must
    be exact there and exactly 0 everywhere else, dW must be the exact sum over those samples (a wrong sample offset in
    im2col, the gradient rows or col2im cannot hide), and the forward is exact on those samples.  The launch count of
    each call exceeds a one-chunk call's by the extra chunks."""
    import torch
    from neuronika_b200 import ops

    def in_use():
        free, whole = torch.cuda.mem_get_info()
        return whole - free

    used0 = in_use()
    cin, sp, cout, k, pad, mode = 4, (12, 16, 16), 8, (3, 3, 3), (1, 1, 1), "replicative"
    L, Kp = int(np.prod(sp)), -(-cin * 27 // 8) * 8
    N, period = 6500, 61
    c16, c32 = chunk_samples(L, Kp, 2, N), chunk_samples(L, Kp, 4, N)
    assert (c16, c32) == (6241, 3120) and -(-N // c16) == 2 and -(-N // c32) == 3
    hot = sorted({0, c32 - 1, c32, 2 * c32 - 1, 2 * c32, c16 - 1, c16, N - 1})
    rng = np.random.default_rng(66)
    xpool = ints(rng, (period, cin) + sp, 0.5, hi=1)
    w = ints(rng, (cout, cin) + k, 0.9, hi=1)
    b = ints(rng, (cout,))
    ghot = ints(rng, (len(hot), cout) + sp, 1.0, hi=1)
    W, B = dev.from_ndarray(w, nk.BF16), dev.from_ndarray(b, nk.BF16)
    per_x = cin * L
    X = dev.zeros((N, cin) + sp, nk.BF16)
    X.slice_flat(0, xpool.shape).copy_from(xpool)
    done = period
    while done < N:
        cnt = min(done, N - done)
        nk._lib.check(ops.lib.nk_d2d(dev.ctx, X.slice_flat(done * per_x, (cnt * per_x,)).ptr, X.ptr, cnt * per_x * 2),
                      dev.ctx)
        done += cnt
    G = dev.zeros((N, cout) + sp, nk.BF16)
    for j, s in enumerate(hot):
        G.slice_flat(s * cout * L, (cout,) + sp).copy_from(ghot[j])
    sub = lambda a, lo, hi: a.slice_flat(lo * (a.size // a.shape[0]), (hi - lo,) + a.shape[1:])

    def launches(fn):
        before = dev.launches
        fn()
        return dev.launches - before

    # forward: 2 chunks; 2 launches per chunk (im2col, batched GEMM)
    Y, Y16 = dev.zeros((N, cout) + sp, nk.BF16), dev.zeros((16, cout) + sp, nk.BF16)
    extra = launches(lambda: ops.conv_layer_nd(X, W, pad, mode, 0.0, bias=B, out=Y)) - \
        launches(lambda: ops.conv_layer_nd(sub(X, 0, 16), W, pad, mode, 0.0, bias=B, out=Y16))
    assert dev.last_conv_kernel == WGMMA[0]
    assert extra == 1 * 2
    for s in hot:
        want, mag, _, _ = oracle_fwd(O, xpool[s % period][None], w, b, pad, mode, 0.0, (1,) * 3, (1,) * 3)
        exact_regime(mag, True, ("y", s))
        equal(sub(Y, s, s + 1).as_ndarray(), want, ("y", s))
    del Y, Y16

    # dX: 3 chunks; 2 launches per chunk (batched GEMM, col2im).  The buffer starts at 1, so a chunk never written shows.
    DX, DX16 = dev.full((N, cin) + sp, 1.0, nk.BF16), dev.zeros((16, cin) + sp, nk.BF16)
    extra = launches(lambda: ops.conv_layer_nd_bwd_input(DX, G, W, pad, mode, beta=0.0)) - \
        launches(lambda: ops.conv_layer_nd_bwd_input(DX16, sub(G, 0, 16), W, pad, mode, beta=0.0))
    assert dev.last_conv_kernel == WGMMA[1]
    assert extra == 2 * 2
    dx = DX.as_ndarray()
    for j, s in enumerate(hot):
        gx, gpa = oracle_dx_full(O, (1, cin) + sp, ghot[j][None], w, pad, (1,) * 3, (1,) * 3)
        exact_regime(gpa, True, ("dx", s))
        equal(dx[s:s + 1], gx, ("dx", s))
    cold = np.ones(N, bool)
    cold[hot] = False
    assert not np.any(dx[cold]), ("dx of samples whose g is zero", np.flatnonzero(np.any(dx != 0, axis=(1, 2, 3, 4)) & cold)[:8])
    del DX, DX16, dx

    # dW (f32): 2 chunks; 2 launches per chunk (im2col, batched GEMM); the exact sum over the samples with a g
    DW, DW16 = dev.zeros(w.shape, nk.F32), dev.zeros(w.shape, nk.F32)
    extra = launches(lambda: ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, mode, 0.0, beta=0.0)) - \
        launches(lambda: ops.conv_layer_nd_bwd_kernel(DW16, sub(G, 0, 16), sub(X, 0, 16), pad, mode, 0.0, beta=0.0))
    assert dev.last_conv_kernel == WGMMA[2]
    assert extra == 1 * 2
    xh = np.stack([xpool[s % period] for s in hot]).astype(np.float64)
    xp = O.pad_mode_forward(xh, pad, mode)
    gw = O.conv_backward_kernel(np.zeros(w.shape), ghot.astype(np.float64), xp, (1,) * 3, (1,) * 3)
    gw_mag = O.conv_backward_kernel(np.zeros(w.shape), np.abs(ghot).astype(np.float64), np.abs(xp), (1,) * 3, (1,) * 3)
    exact_regime(gw_mag, False, "dw")
    equal(DW.as_ndarray(), gw, "dw")
    # the library's memory pool keeps what it has reserved, so its growth over the test bounds the test's peak from below
    print(f"device memory reserved by the 3-D chunking test: {(in_use() - used0) / 2 ** 30:.2f} GiB")


# ------------------------------------------------------------------------------------------- the 2-D entry points
# the same drivers through ops.conv2d*: (Cout, Cin, kernel, output extents, stride, dilation); unit steps take
# im2col_plane_kernel, the strided / dilated rows im2col_kernel
CONV2D = [
    (8, 1, (3, 3), (1, 1), (1, 1), (1, 1)), (9, 5, (1, 3), (1, 7), (1, 1), (1, 1)),
    (120, 8, (2, 1), (2, 4), (1, 1), (1, 1)), (128, 17, (1, 1), (3, 3), (1, 1), (1, 1)),
    (136, 7, (3, 3), (7, 9), (1, 1), (1, 1)), (256, 16, (2, 2), (8, 8), (1, 1), (1, 1)),
    (264, 13, (5, 1), (5, 13), (1, 1), (1, 1)), (128, 32, (2, 2), (8, 16), (1, 1), (1, 1)),
    (8, 43, (3, 1), (3, 43), (1, 1), (1, 1)), (136, 8, (5, 5), (16, 16), (1, 1), (1, 1)),
    (264, 3, (3, 3), (1, 257), (1, 1), (1, 1)),
    (64, 8, (3, 3), (6, 11), (2, 1), (1, 2)),        # im2col_kernel: strided rows, dilated columns
    (24, 5, (2, 3), (9, 7), (1, 2), (2, 1)),         # im2col_kernel: the element-wise path of a strided last axis
]


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("row", CONV2D, ids=[f"cout{r[0]}-K{r[1] * r[2][0] * r[2][1]}-L{r[3][0] * r[3][1]}"
                                             for r in CONV2D])
def test_conv2d_entry_points_exact(nk, dev, O, row, relu):
    """forward (with bias, with and without ReLU), dX (beta 0 and 1) and dW + db (f32, bf16) through the 2-D entry
    points on integer operands: every result equal to the oracle"""
    from neuronika_b200 import ops
    cout, cin, k, out, s, d = row
    xs = (2, cin) + tuple((o - 1) * st + di * (kk - 1) + 1 for o, st, di, kk in zip(out, s, d, k))
    K, L = cin * k[0] * k[1], out[0] * out[1]
    rng = np.random.default_rng(cout + K + L)
    dens = densities({("x", "w"): K, ("g", "w"): cout * k[0] * k[1], ("g", "x"): 2 * L})
    x, w, b = ints(rng, xs, dens["x"]), ints(rng, (cout, cin) + k, dens["w"]), ints(rng, (cout,))
    X, W, B = (dev.from_ndarray(a, nk.BF16) for a in (x, w, b))
    x64, w64 = x.astype(np.float64), w.astype(np.float64)
    conv = O.conv_forward(x64, w64, s, d).astype(np.float64)
    exact_regime(O.conv_forward(np.abs(x64), np.abs(w64), s, d) + 2, True, "y")
    want = conv + b[None, :, None, None]
    if relu:
        want = np.maximum(want, 0)
    y = ops.conv2d(X, W, s, d, bias=B, relu=relu)
    assert dev.last_conv_kernel == WG2[0]
    equal(y.as_ndarray(), want, "y")
    g = ints(rng, conv.shape, dens["g"])
    G = dev.from_ndarray(g, nk.BF16)
    gx = O.conv_backward_input(np.zeros(xs), g.astype(np.float64), w64, s, d)
    gxa = O.conv_backward_input(np.zeros(xs), np.abs(g).astype(np.float64), np.abs(w64), s, d)
    dx0 = ints(rng, xs)
    dx_kernel = WG2[1] if cout % 8 == 0 else "direct_bwd_input"
    for beta in (0.0, 1.0):
        exact_regime(gxa + 2 * beta, True, ("dx", beta))
        DX = dev.from_ndarray(dx0, nk.BF16)
        ops.conv2d_bwd_input(DX, G, W, s, d, beta=beta)
        assert dev.last_conv_kernel == dx_kernel
        equal(DX.as_ndarray(), beta * dx0 + gx, ("dx", beta))
    gw = O.conv_backward_kernel(np.zeros(w.shape), g.astype(np.float64), x64, s, d)
    gwa = O.conv_backward_kernel(np.zeros(w.shape), np.abs(g).astype(np.float64), np.abs(x64), s, d)
    gb = g.astype(np.float64).sum((0, 2, 3))
    for dwt in (nk.F32, nk.BF16):
        dbf = dwt == nk.BF16
        exact_regime(gwa + 2, dbf, ("dw", dbf))
        exact_regime(np.abs(g).sum((0, 2, 3)) + 2, dbf, ("db", dbf))
        dw0, db0 = ints(rng, w.shape), ints(rng, (cout, 1, 1))
        for beta in (0.0, 1.0):
            DW, DB = dev.from_ndarray(dw0, dwt), dev.from_ndarray(db0, dwt)
            ops.conv2d_bwd_kernel(DW, G, X, s, d, beta=beta, dbias=DB)
            assert dev.last_conv_kernel == WG2[2]
            equal(DW.as_ndarray(), beta * dw0 + gw, ("dw", dbf, beta))
            equal(DB.as_ndarray().ravel(), beta * db0.ravel() + gb, ("db", dbf, beta))


# ------------------------------------------------------------------------------------------- the reference's goldens
GOLDENS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tensors_pad.json")))
GOLDEN_CASES = [(mode, name) for mode, cases in GOLDENS.items() for name in cases]


@pytest.mark.parametrize("tap", ["k1", "first", "last"])
@pytest.mark.parametrize("mode,name", GOLDEN_CASES)
def test_reference_pad_goldens_through_the_layer(nk, dev, O, mode, name, tap):
    """each golden's `Array::range` input on 16 channels (channel c times +1 or -1), through the layer as an identity
    convolution (w[o, c] = delta(o, c)) on the tensor cores: with k = 1 the output is the golden itself; with k = 3 on
    every padded axis and the one-hot tap at the first or the last kernel position, it is the golden's window shifted by
    that tap.  2-D goldens run as 3-D layers with a leading extent-1 axis and pad 0 on it.  Every value exactly."""
    from neuronika_b200 import ops
    c = GOLDENS[mode][name]
    start, stop, step = c["base_range"]
    base = np.arange(start, stop, step).reshape(c["base_shape"])
    golden = np.asarray(c["expected"], np.float64)
    pad = list(c["padding"])
    if base.ndim == 2:
        base, golden, pad = base[None], golden[None], [0] + pad
    nsp = base.ndim
    fill = c.get("fill", 0.0)
    sign = np.where(np.arange(16) % 3 == 1, -1.0, 1.0)
    x = (sign.reshape((1, 16) + (1,) * nsp) * base[None, None]).astype(F32)
    inner = tuple(slice(p, p + e) for p, e in zip(pad, base.shape))
    border = np.ones(golden.shape, bool)
    border[inner] = False
    # the padded input of channel c: the golden times sign_c, except that the fill does not change sign
    want_padded = sign.reshape((16,) + (1,) * nsp) * golden[None]
    if mode in ("constant", "zero"):
        want_padded[:, border] = golden[border]
    k = [1] * nsp if tap == "k1" else [1 if p == 0 and e == 1 else 3 for p, e in zip(pad, base.shape)]
    t = [0 if tap in ("k1", "first") else kk - 1 for kk in k]
    w = np.zeros((16, 16) + tuple(k), F32)
    for o in range(16):
        w[(o, o) + tuple(t)] = 1.0
    X, W = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16)
    y = ops.conv_layer_nd(X, W, tuple(pad), "constant" if mode == "zero" else mode, fill)
    assert dev.last_conv_kernel == WGMMA[0]
    out = y.as_ndarray()[0]
    win = tuple(slice(ti, ti + e - kk + 1) for ti, e, kk in zip(t, golden.shape, k))
    equal(out, want_padded[(slice(None),) + win], (mode, name, tap))
