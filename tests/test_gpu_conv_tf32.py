"""f32 convolution on the tensor cores (Device.f32_conv, csrc/nk_conv_tf32.cu): the 2-D entry points, the 1-D / 3-D
convolution layers and the un-padded 1-D / 3-D convolutions, in TF32 and 3xTF32 mode.

Exact regime (the method of tests/test_gpu_conv_nd_edges.py): small-integer operands are TF32 values (their lo parts
are 0), every product is exact and every f32 partial sum an integer below 2^24, so both modes must EQUAL the float64
oracle -- over the padding map, stride / dilation, the tile edges (Cout, K around the 32-wide k-block, L % 4 != 0),
views off 16-byte alignment, sample chunks, beta accumulation, bf16 dW / dbias and the fused bias + ReLU forward.

Rounding bounds on random operands (tests/tf32_oracle.py models the operand rounding exactly, tests/tf32_conv_oracle.py
the convolution): tf32 against float64 on the rounded operands within (R + 2) 2^-22 of the magnitudes, tf32x3 against
float64 on the unrounded operands within (3R + 6) 2^-22, R the reduction length: K (+ the bias) forward, Cout plus the
f32 sum of the col2im taps for dX, N.L plus the split partials for dW."""
import numpy as np
import pytest

import tf32_conv_oracle as C
from tf32_oracle import tf32_round
from test_gpu_conv_nd_edges import PAD_EDGES, densities, equal, exact_case, exact_regime, ints

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0
MODES = ["tf32", "tf32x3"]


def names(mode, nd):
    mid = "_im2col_nd_" if nd else "_im2col_"
    return tuple(f"{mode}{mid}{p}" for p in ("fwd", "dx", "dw"))


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.f32_conv("ieee")
    d.synchronize()


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


@pytest.fixture(autouse=True)
def ieee_after(dev):
    yield
    dev.f32_conv("ieee")
    dev.f32_matmul("ieee")
    dev.conv_engine("auto")


class Guarded:
    """a device copy of `data` at element `off` of a larger buffer whose every other element holds CANARY"""

    def __init__(self, dev, nk, data, off=0, tail=37):
        data = np.asarray(data, F32)
        self.off, self.n = off, data.size
        host = np.full(off + data.size + tail, CANARY, F32)
        host[off:off + data.size] = data.ravel()
        self.buf = dev.from_ndarray(host, nk.F32)
        self.view = self.buf.slice_flat(off, data.shape)

    def read(self):
        flat = self.buf.as_ndarray()
        assert np.all(flat[:self.off] == CANARY) and np.all(flat[self.off + self.n:] == CANARY), "canary overwritten"
        return self.view.as_ndarray()


# ------------------------------------------------------------------------------------------- exact: the layers
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,pmode", [(n, m) for n, c in PAD_EDGES.items() for m in c[6]])
def test_layer_padding_map_exact(nk, dev, O, mode, name, pmode):
    """every padding mode in 1-D and 3-D at its limits (exact_case: forward with bias, dX beta 0 / 1, dW + dbias into
    f32 and bf16, beta 0 / 1), equal to the oracle"""
    xs, cout, k, pad, s, d, _ = PAD_EDGES[name]
    dev.f32_conv(mode)
    exact_case(nk, dev, O, xs, cout, k, pad, pmode, s, d, engine="f32", kernels=names(mode, True),
               seed=sum(xs) + len(pmode))


# (x shape, Cout, kernel, padding, padding mode, stride, dilation): the tile edges of the three products -- Cout 1 / 127 /
# 128 / 129 (forward and dW rows), K = Cin.prod(k) 1 / 31 / 32 / 33 / 100 around the k-block (forward, and dX's rows),
# L around 64 / 128 / 256 with L % 4 != 0 -- plus strides and dilations
TILES = [
    ((2, 1, 65), 1, (1,), (0,), "zero", (1,), (1,)),                  # K 1, L 65, Cout 1
    ((2, 31, 127), 127, (1,), (0,), "zero", (1,), (1,)),              # K 31, L 127
    ((2, 16, 129), 128, (2,), (1,), "replicative", (1,), (1,)),       # K 32, L 130
    ((3, 11, 255), 129, (3,), (1,), "reflective", (1,), (1,)),        # K 33, L 255
    ((2, 20, 257), 64, (5,), (2,), "constant", (1,), (1,)),           # K 100, L 257
    ((2, 4, 3, 5, 7), 129, (2, 2, 2), (1, 0, 1), "replicative", (1, 1, 1), (1, 1, 1)),   # K 32, L 4.4.8
    ((2, 3, 5, 6, 9), 33, (1, 3, 3), (0, 1, 2), "constant", (1, 1, 2), (1, 2, 1)),      # K 27, strided / dilated
    ((2, 5, 7, 9, 11), 8, (3, 2, 3), (1, 1, 1), "reflective", (2, 3, 2), (1, 1, 2)),    # K 90, both
    ((2, 8, 61), 40, (3,), (2,), "zero", (3,), (2,)),                 # stride 3, dilation 2
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", TILES, ids=[f"{len(c[2])}d-cout{c[1]}-K{c[0][1] * int(np.prod(c[2]))}" for c in TILES])
def test_layer_tiles_strides_exact(nk, dev, O, mode, case):
    xs, cout, k, pad, pmode, s, d = case
    dev.f32_conv(mode)
    exact_case(nk, dev, O, xs, cout, k, pad, pmode, s, d, engine="f32", kernels=names(mode, True), seed=cout + xs[1])


# ------------------------------------------------------------------------------------------- exact: the plain entry points
def plain_exact(nk, dev, O, mode, xs, cout, k, s, d, *, x_off=0, g_off=0, out_off=0, relu=False, seed=0):
    """the 2-D entry points (forward with bias and ReLU) or nk_convnd_* (1-D / 3-D, no bias): forward, dX (beta 0 / 1)
    and dW (f32 and bf16, beta 0 / 1; + dbias in 2-D) on integer operands equal to the oracle, with x, g and out at
    element offsets x_off / g_off / out_off of canary-guarded buffers"""
    from neuronika_b200 import ops
    nsp = len(k)
    two = nsp == 2
    rng = np.random.default_rng(seed)
    n, cin = xs[:2]
    out_sp = tuple((sz - dd * (kk - 1) - 1) // st + 1 for sz, kk, st, dd in zip(xs[2:], k, s, d))
    K, L = cin * int(np.prod(k)), int(np.prod(out_sp))
    dens = densities({("x", "w"): K, ("g", "w"): cout * int(np.prod(k)), ("g", "x"): n * L})
    x, w = ints(rng, xs, dens["x"]), ints(rng, (cout, cin) + tuple(k), dens["w"])
    b = ints(rng, (cout,)) if two else None
    want = C.forward(x, w, b, (0,) * nsp, "zero", 0.0, s, d)
    exact_regime(C.forward(np.abs(x), np.abs(w), None if b is None else np.abs(b), (0,) * nsp, "zero", 0.0, s, d), False,
                 "y")
    if relu:
        want = np.maximum(want, 0.0)
    X = Guarded(dev, nk, x, x_off)
    W = dev.from_ndarray(w, nk.F32)
    Y = Guarded(dev, nk, np.zeros(want.shape, F32), out_off)
    if two:
        ops.conv2d(X.view, W, s, d, bias=dev.from_ndarray(b.reshape(cout, 1, 1), nk.F32), relu=relu, out=Y.view)
    else:
        ops.convnd(X.view, W, s, d, out=Y.view)
    kern = names(mode, not two)
    assert dev.last_conv_kernel == kern[0], (dev.last_conv_kernel, kern)
    equal(Y.read(), want, "y")

    g = ints(rng, want.shape, dens["g"])
    G = Guarded(dev, nk, g, g_off)
    gx = C.backward_input(xs, g, w, (0,) * nsp, s, d)
    exact_regime(C.backward_input(xs, np.abs(g), np.abs(w), (0,) * nsp, s, d) + 2, False, "dx")
    dx0 = ints(rng, xs)
    for beta in (0.0, 1.0):
        DX = Guarded(dev, nk, dx0, out_off)
        (ops.conv2d_bwd_input if two else ops.convnd_bwd_input)(DX.view, G.view, W, s, d, beta=beta)
        assert dev.last_conv_kernel == kern[1], (dev.last_conv_kernel, kern)
        equal(DX.read(), beta * dx0 + gx, ("dx", beta))

    gw = C.backward_kernel(g, x, w.shape, (0,) * nsp, "zero", 0.0, s, d)
    gw_mag = C.backward_kernel(np.abs(g), np.abs(x), w.shape, (0,) * nsp, "zero", 0.0, s, d)
    gb = g.astype(np.float64).sum(axis=tuple(i for i in range(g.ndim) if i != 1))
    for dwt in (nk.F32, nk.BF16):
        dbf = dwt == nk.BF16
        exact_regime(gw_mag + 2, dbf, ("dw", dbf))
        dw0, db0 = ints(rng, w.shape), ints(rng, (cout, 1, 1))
        for beta in (0.0, 1.0):
            DW = dev.from_ndarray(dw0, dwt)
            if two:
                DB = dev.from_ndarray(db0, dwt)
                ops.conv2d_bwd_kernel(DW, G.view, X.view, s, d, beta=beta, dbias=DB)
                equal(DB.as_ndarray().ravel(), beta * db0.ravel() + gb, ("db", dbf, beta))
            else:
                ops.convnd_bwd_kernel(DW, G.view, X.view, s, d, beta=beta)
            assert dev.last_conv_kernel == kern[2], (dev.last_conv_kernel, kern)
            equal(DW.as_ndarray(), beta * dw0 + gw, ("dw", dbf, beta))


PLAIN = [   # (x shape, Cout, kernel, stride, dilation)
    ((2, 3, 10, 12), 64, (3, 3), (1, 1), (1, 1)),          # a stem: K 27, L 80
    ((2, 8, 13, 11), 129, (2, 2), (2, 1), (1, 2)),         # K 32, strided rows, dilated columns
    ((3, 11, 9, 9), 1, (1, 3), (1, 1), (1, 1)),            # K 33, Cout 1, L 63
    ((2, 5, 66), 127, (7,), (1,), (1,)),                   # 1-D K 35, L 60
    ((2, 4, 5, 6, 7), 128, (3, 2, 3), (1, 2, 1), (1, 1, 2)),   # 3-D K 72
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("case", PLAIN, ids=[f"{len(c[2])}d-cout{c[1]}" for c in PLAIN])
def test_plain_entry_points_exact(nk, dev, O, mode, relu, case):
    xs, cout, k, s, d = case
    if relu and len(k) != 2:
        pytest.skip("the fused ReLU is a 2-D forward option")
    dev.f32_conv(mode)
    plain_exact(nk, dev, O, mode, xs, cout, k, s, d, relu=relu, seed=cout + len(k))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("offs", [(1, 0, 0), (0, 1, 0), (0, 0, 1), (3, 2, 1)], ids=["x", "g", "out", "all"])
def test_views_off_alignment_exact(nk, dev, O, mode, offs):
    """x, g and out one to three f32 elements off 16-byte alignment: the gathers and packs read any address"""
    dev.f32_conv(mode)
    plain_exact(nk, dev, O, mode, (2, 6, 9, 14), 24, (3, 3), (1, 1), (1, 1), x_off=offs[0], g_off=offs[1],
                out_off=offs[2], relu=True, seed=5)
    plain_exact(nk, dev, O, mode, (2, 6, 5, 6, 7), 12, (2, 3, 2), (1, 1, 1), (1, 1, 1), x_off=offs[0], g_off=offs[1],
                out_off=offs[2], seed=6)


def test_sample_chunks_exact(nk, dev, O):
    """(N, 16, 4103) k 8 -> L 4096, K 128, Cout 8: a 4 GiB chunk of forward columns holds 2048 samples in TF32 mode
    (L.ceil4(K).4 = 2 MiB each), of dX temporaries 1927 (+ K.L.4 column gradients) and of dW operands 1927
    ((Cout + K).L.4); in 3xTF32 mode a third of that.  N = 2100 spans two chunks in each product (six or more in
    3xTF32).  x repeats a pool of 61 integer samples; g is zero except on the samples on both sides of every possible
    chunk boundary, so dX is exact there and 0 elsewhere, dW is the exact sum over those samples and the forward is
    checked on them."""
    from neuronika_b200 import ops
    n, cin, length, cout, k = 2100, 16, 4103, 8, 8
    rng = np.random.default_rng(21)
    pool = ints(rng, (61, cin, length), 0.05)
    x = pool[np.arange(n) % 61]
    w = ints(rng, (cout, cin, k), 0.5)
    bounds = set()
    for per in (2048, 1927, 682, 1724, 642):
        for b in range(per, n, per):
            bounds |= {b - 1, b}
    hot = sorted(bounds | {0, n - 1})
    X, W = dev.from_ndarray(x, nk.F32), dev.from_ndarray(w, nk.F32)
    g = np.zeros((n, cout, length - k + 1), F32)
    g[hot] = ints(rng, (len(hot), cout, length - k + 1), 0.05)
    G = dev.from_ndarray(g, nk.F32)
    xh, gh = x[hot], g[hot]
    yw = C.forward(xh, w, None, (0,), "zero", 0.0, (1,), (1,))
    gx = C.backward_input(xh.shape, gh, w, (0,), (1,), (1,))
    gw = C.backward_kernel(gh, xh, w.shape, (0,), "zero", 0.0, (1,), (1,))
    exact_regime(C.backward_kernel(np.abs(gh), np.abs(xh), w.shape, (0,), "zero", 0.0, (1,), (1,)), False, "dw")
    for mode in MODES:
        dev.f32_conv(mode)
        y = ops.convnd(X, W, (1,), (1,))
        assert dev.last_conv_kernel == names(mode, True)[0]
        equal(y.as_ndarray()[hot], yw, (mode, "y"))
        del y
        DX = dev.zeros(x.shape, nk.F32)
        ops.convnd_bwd_input(DX, G, W, (1,), (1,), beta=0.0)
        dx = DX.as_ndarray()
        del DX
        cold = np.ones(n, bool)
        cold[hot] = False
        assert not np.any(dx[cold]), mode
        equal(dx[hot], gx, (mode, "dx"))
        DW = dev.zeros(w.shape, nk.F32)
        ops.convnd_bwd_kernel(DW, G, X, (1,), (1,), beta=0.0)
        equal(DW.as_ndarray(), gw, (mode, "dw"))


def test_dw_beyond_two_million_output_positions_exact(nk, dev):
    """a 1-D layer with L = 2,200,000 output positions (N 1, Cin 1, Cout 2, k 3, zero pad 1): dW packs G with L on the
    pack's reduction axis, more than 65535 tiles of 32, so the pack steps through its k tiles.  Sparse integer operands,
    forward, dX and dW equal to the oracle in both modes."""
    from neuronika_b200 import ops
    n, cin, cout, length = 1, 1, 2, 2_200_000
    rng = np.random.default_rng(31)
    x = ints(rng, (n, cin, length), 0.01)
    w = ints(rng, (cout, cin, 3))
    g = ints(rng, (n, cout, length), 0.01)
    yw = C.forward(x, w, None, (1,), "zero", 0.0, (1,), (1,))
    gx = C.backward_input(x.shape, g, w, (1,), (1,), (1,))
    gw = C.backward_kernel(g, x, w.shape, (1,), "zero", 0.0, (1,), (1,))
    exact_regime(C.backward_kernel(np.abs(g), np.abs(x), w.shape, (1,), "zero", 0.0, (1,), (1,)), False, "dw")
    X, W, G = dev.from_ndarray(x, nk.F32), dev.from_ndarray(w, nk.F32), dev.from_ndarray(g, nk.F32)
    for mode in MODES:
        dev.f32_conv(mode)
        y = ops.conv_layer_nd(X, W, (1,), "constant", 0.0)
        assert dev.last_conv_kernel == names(mode, True)[0]
        equal(y.as_ndarray(), yw, (mode, "y"))
        DX = dev.zeros(x.shape, nk.F32)
        ops.conv_layer_nd_bwd_input(DX, G, W, (1,), "constant", beta=0.0)
        equal(DX.as_ndarray(), gx, (mode, "dx"))
        DW = dev.zeros(w.shape, nk.F32)
        ops.conv_layer_nd_bwd_kernel(DW, G, X, (1,), "constant", 0.0, beta=0.0)
        assert dev.last_conv_kernel == names(mode, True)[2]
        equal(DW.as_ndarray(), gw, (mode, "dw"))


# ------------------------------------------------------------------------------------------- rounding bounds
def rel(mode, R):
    return (R + 2) * 2.0 ** -22 if mode == "tf32" else (3 * R + 6) * 2.0 ** -22


def near(got, want, tol, what):
    err = np.abs(np.asarray(got, np.float64) - want)
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), float((err - tol).max()), np.argwhere(bad)[:3].tolist())


BOUND_CASES = [   # (x shape, Cout, kernel, padding, padding mode, stride, dilation, fill)
    ((4, 32, 300), 136, (5,), (2,), "reflective", (2,), (1,), 0.0),
    ((4, 16, 20, 20), 40, (3, 3), (0, 0), "zero", (1, 1), (1, 1), 0.0),
    ((2, 4, 8, 9, 10), 24, (3, 3, 3), (1, 1, 1), "constant", (1, 1, 1), (1, 2, 1), 0.1),
    ((2, 6, 7, 8, 9), 33, (3, 2, 3), (1, 1, 1), "replicative", (2, 1, 1), (1, 1, 1), 0.0),
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", BOUND_CASES, ids=[f"{len(c[2])}d-{c[4]}" for c in BOUND_CASES])
def test_rounding_bounds(nk, dev, mode, case):
    """random operands: forward (+ bias), dX with beta = 1 and dW with beta = 1 within the bounds of the module
    docstring, every output canary-guarded; then the same calls again give the same bits"""
    from neuronika_b200 import ops
    xs, cout, k, pad, pmode, s, d, fill = case
    nsp = len(k)
    rng = np.random.default_rng(cout)
    x = rng.standard_normal(xs).astype(F32)
    w = (rng.standard_normal((cout, xs[1]) + k) * 0.2).astype(F32)
    b = rng.standard_normal(cout).astype(F32)
    rx, rw = (tf32_round(v) if mode == "tf32" else v for v in (x, w))
    rfill = float(tf32_round(np.float32(fill))) if mode == "tf32" else float(np.float32(fill))
    want = C.forward(rx, rw, b, pad, pmode, rfill, s, d)
    mag = C.forward(np.abs(x), np.abs(w), np.abs(b), pad, pmode, abs(fill), s, d)
    K, ksz = xs[1] * int(np.prod(k)), int(np.prod(k))
    dev.f32_conv(mode)
    X, W = dev.from_ndarray(x, nk.F32), dev.from_ndarray(w, nk.F32)
    Y = Guarded(dev, nk, np.zeros(want.shape, F32), 1)
    if nsp == 2:
        ops.conv2d(X, W, s, d, bias=dev.from_ndarray(b.reshape(cout, 1, 1), nk.F32), out=Y.view)
    else:
        ops.conv_layer_nd(X, W, pad, "constant" if pmode == "zero" else pmode, fill, s, d,
                          bias=dev.from_ndarray(b, nk.F32), out=Y.view)
    kern = names(mode, nsp != 2)
    assert dev.last_conv_kernel == kern[0]
    y1 = Y.read()
    near(y1, want, rel(mode, K + 1) * mag + 1e-30, (mode, "y"))

    g = rng.standard_normal(want.shape).astype(F32)
    rg = tf32_round(g) if mode == "tf32" else g
    dx0 = rng.standard_normal(xs).astype(F32)
    dw0 = rng.standard_normal(w.shape).astype(F32)
    G = dev.from_ndarray(g, nk.F32)

    def backward():
        DX, DW = Guarded(dev, nk, dx0, 2), Guarded(dev, nk, dw0, 3)
        if nsp == 2:
            ops.conv2d_bwd_input(DX.view, G, W, s, d, beta=1.0)
            assert dev.last_conv_kernel == kern[1]
            ops.conv2d_bwd_kernel(DW.view, G, X, s, d, beta=1.0)
        else:
            mc = "constant" if pmode == "zero" else pmode
            ops.conv_layer_nd_bwd_input(DX.view, G, W, pad, mc, s, d, beta=1.0)
            assert dev.last_conv_kernel == kern[1]
            ops.conv_layer_nd_bwd_kernel(DW.view, G, X, pad, mc, fill, s, d, beta=1.0)
        assert dev.last_conv_kernel == kern[2]
        return DX.read(), DW.read()

    dx, dw = backward()
    gx = C.backward_input(xs, rg, rw, pad, s, d) + dx0
    gx_mag = C.backward_input(xs, np.abs(g), np.abs(w), pad, s, d)
    near(dx, gx, rel(mode, cout + ksz) * gx_mag + 2.0 ** -22 * np.abs(dx0) + 1e-30, (mode, "dx"))
    gw = C.backward_kernel(rg, rx, w.shape, pad, pmode, rfill, s, d) + dw0
    gw_mag = C.backward_kernel(np.abs(g), np.abs(x), w.shape, pad, pmode, abs(fill), s, d)
    R = xs[0] * int(np.prod(want.shape[2:])) + 140     # + the split partials (at most one per SM)
    near(dw, gw, rel(mode, R) * gw_mag + 2.0 ** -22 * np.abs(dw0) + 1e-30, (mode, "dw"))
    dx2, dw2 = backward()
    assert np.array_equal(dx.view(np.uint32), dx2.view(np.uint32)) and np.array_equal(dw.view(np.uint32),
                                                                                      dw2.view(np.uint32)), mode


def test_tf32x3_is_closer_than_tf32(nk, dev):
    """a stem-like 2-D forward: 3xTF32's error against float64 at least 100x below TF32's"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(4)
    x = rng.standard_normal((8, 3, 34, 34)).astype(F32)
    w = rng.standard_normal((64, 3, 3, 3)).astype(F32)
    want = C.forward(x, w, None, (0, 0), "zero", 0.0, (1, 1), (1, 1))
    X, W = dev.from_ndarray(x, nk.F32), dev.from_ndarray(w, nk.F32)
    err = {}
    for mode in MODES:
        dev.f32_conv(mode)
        err[mode] = float(np.abs(ops.conv2d(X, W).as_ndarray() - want).max())
    assert err["tf32x3"] * 100 < err["tf32"], err


# ------------------------------------------------------------------------------------------- unchanged behaviour
def direct_calls(nk, dev, groups=1, seed=3):
    """forward, dX and dW of a 2-D and a 3-D f32 convolution: (results, kernel names)"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    out, kerns = [], []
    x = rng.standard_normal((2, 4, 9, 10)).astype(F32)
    w = rng.standard_normal((8, 4 // groups, 3, 3)).astype(F32)
    X, W = dev.from_ndarray(x, nk.F32), dev.from_ndarray(w, nk.F32)
    y = ops.conv2d(X, W, groups=groups)
    kerns.append(dev.last_conv_kernel)
    G = dev.from_ndarray(rng.standard_normal(y.shape).astype(F32), nk.F32)
    DX, DW = dev.zeros(x.shape, nk.F32), dev.zeros(w.shape, nk.F32)
    ops.conv2d_bwd_input(DX, G, W, groups=groups)
    kerns.append(dev.last_conv_kernel)
    ops.conv2d_bwd_kernel(DW, G, X, groups=groups)
    kerns.append(dev.last_conv_kernel)
    out += [y.as_ndarray(), DX.as_ndarray(), DW.as_ndarray()]
    x3 = rng.standard_normal((2, 4, 5, 6, 7)).astype(F32)
    w3 = rng.standard_normal((6, 4 // groups, 2, 2, 3)).astype(F32)
    X3, W3 = dev.from_ndarray(x3, nk.F32), dev.from_ndarray(w3, nk.F32)
    y3 = ops.convnd(X3, W3, (1, 1, 1), (1, 1, 1), groups=groups)
    kerns.append(dev.last_conv_kernel)
    G3 = dev.from_ndarray(rng.standard_normal(y3.shape).astype(F32), nk.F32)
    DX3, DW3 = dev.zeros(x3.shape, nk.F32), dev.zeros(w3.shape, nk.F32)
    ops.convnd_bwd_input(DX3, G3, W3, (1, 1, 1), (1, 1, 1), groups=groups)
    kerns.append(dev.last_conv_kernel)
    ops.convnd_bwd_kernel(DW3, G3, X3, (1, 1, 1), (1, 1, 1), groups=groups)
    kerns.append(dev.last_conv_kernel)
    out += [y3.as_ndarray(), DX3.as_ndarray(), DW3.as_ndarray()]
    return out, kerns


DIRECT_NAMES = ["direct_fwd", "direct_bwd_input", "direct_bwd_kernel", "direct_nd_fwd", "direct_nd_dx", "direct_nd_dw"]


def same_bits(a, b):
    return all(np.array_equal(u.view(np.uint32), v.view(np.uint32)) for u, v in zip(a, b))


def test_ieee_mode_and_the_round_trip_keep_the_direct_kernels(nk, dev):
    fresh = nk.Device(0)
    ref, kerns = direct_calls(nk, fresh)
    assert kerns == DIRECT_NAMES
    dev.f32_conv("ieee")
    got, kerns = direct_calls(nk, dev)
    assert kerns == DIRECT_NAMES and same_bits(got, ref)
    dev.f32_conv("tf32")
    _, kerns = direct_calls(nk, dev)
    assert kerns == ["tf32_im2col_fwd", "tf32_im2col_dx", "tf32_im2col_dw"] + list(names("tf32", True))
    dev.f32_conv("ieee")
    got, kerns = direct_calls(nk, dev)
    assert kerns == DIRECT_NAMES and same_bits(got, ref)


@pytest.mark.parametrize("mode", MODES)
def test_grouped_direct_engine_and_f32_matmul_stay_on_the_cuda_cores(nk, dev, mode):
    fresh = nk.Device(0)
    ref_g, _ = direct_calls(nk, fresh, groups=2)
    ref, _ = direct_calls(nk, fresh)
    dev.f32_conv(mode)
    got, kerns = direct_calls(nk, dev, groups=2)
    assert kerns == DIRECT_NAMES and same_bits(got, ref_g)
    dev.conv_engine("direct")
    got, kerns = direct_calls(nk, dev)
    assert kerns == DIRECT_NAMES and same_bits(got, ref)
    dev.conv_engine("auto")
    dev.f32_conv("ieee")
    dev.f32_matmul(mode)
    got, kerns = direct_calls(nk, dev)
    assert kerns == DIRECT_NAMES and same_bits(got, ref)


def test_bad_modes_are_rejected(nk, dev):
    from neuronika_b200 import _lib as L
    for bad in ("TF32", "fp32", "", None):
        with pytest.raises(ValueError):
            dev.f32_conv(bad)
    assert L.lib.nk_conv_f32_config(dev.ctx, 3) == -1
    assert L.lib.nk_conv_f32_config(dev.ctx, -1) == -1
    assert "bad mode" in L.lib.nk_last_error(dev.ctx).decode()
    _, kerns = direct_calls(nk, dev)
    assert kerns == DIRECT_NAMES


# ------------------------------------------------------------------------------------------- graph level
def make_layer(nk, dev, nsp, rng):
    if nsp == 1:
        return nk.nn.Conv1d(dev, 8, 16, 5, padding=2, padding_mode=nk.nn.ReplicativePad(), stride=2, rng=rng), (6, 8, 64), \
            ((2,), "replicative", 0.0, (2,), (1,))
    if nsp == 2:
        return nk.nn.Conv2d(dev, 3, 32, (3, 3), rng=rng), (8, 3, 18, 18), ((0, 0), "zero", 0.0, (1, 1), (1, 1))
    return nk.nn.Conv3d(dev, 4, 12, (3, 3, 3), padding=(1, 1, 1), padding_mode=nk.nn.ReflectivePad(), rng=rng), \
        (2, 4, 6, 7, 8), ((1, 1, 1), "reflective", 0.0, (1, 1, 1), (1, 1, 1))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("nsp", [1, 2, 3])
def test_layer_training_step_against_float64(nk, dev, nsp, mode):
    """f32 Conv1d / Conv2d / Conv3d -> mse against a target -> backward -> SGD: the loss, the parameters' gradients and
    the updated parameters against float64 on the unrounded operands, within the TF32 rounding of each operand
    (2^-10 of each product for tf32) plus the bounds above; g = 2 (y - t) / numel carries y's error"""
    rng = np.random.default_rng(nsp)
    layer, xs, (pad, pmode, fill, s, d) = make_layer(nk, dev, nsp, rng)
    w, b = layer.weight.data().astype(np.float64), layer.bias.data().astype(np.float64).ravel()
    x = rng.standard_normal(xs).astype(F32)
    y64 = C.forward(x, w, b, pad, pmode, fill, s, d)
    t = rng.standard_normal(y64.shape).astype(F32)
    lr = 0.5
    opt = nk.optim.StochasticGD.new(lr)
    for p in layer.parameters():
        opt.register(p)
    dev.f32_conv(mode)
    opt.zero_grad()
    loss = layer.forward(nk.from_ndarray(dev, x)).mse_loss(nk.from_ndarray(dev, t))
    loss.forward()
    loss.backward(1.0)
    assert dev.last_conv_kernel == names(mode, nsp != 2)[2]
    opt.step()
    K = xs[1] * int(np.prod(w.shape[2:]))
    ext = 2.0 ** -10 if mode == "tf32" else 0.0
    ymag = C.forward(np.abs(x), np.abs(w), np.abs(b), pad, pmode, abs(fill), s, d)
    ytol = (ext + rel(mode, K + 1)) * ymag
    g64 = 2.0 * (y64 - t) / y64.size
    gtol = 2.0 * ytol / y64.size + 2.0 ** -23 * np.abs(g64)
    lo = float(np.mean((y64 - t) ** 2))
    assert abs(loss.item() - lo) <= float(np.mean(2.0 * np.abs(y64 - t) * ytol + ytol ** 2)) + 1e-6 * lo
    gw = C.backward_kernel(g64, x, w.shape, pad, pmode, fill, s, d)
    R = xs[0] * int(np.prod(y64.shape[2:])) + 140
    gw_tol = (ext + rel(mode, R)) * C.backward_kernel(np.abs(g64) + gtol, np.abs(x), w.shape, pad, pmode, abs(fill), s, d) \
        + C.backward_kernel(gtol, np.abs(x), w.shape, pad, pmode, abs(fill), s, d)
    near(layer.weight.grad(), gw, gw_tol + 1e-30, (nsp, mode, "dW"))
    axes = tuple(i for i in range(g64.ndim) if i != 1)
    gb = g64.sum(axis=axes)
    gb_tol = gtol.sum(axis=axes) + (g64.size // g64.shape[1]) * 2.0 ** -22 * np.abs(g64).sum(axis=axes)
    near(layer.bias.grad().ravel(), gb, gb_tol + 1e-30, (nsp, mode, "db"))
    near(layer.weight.data(), w - lr * gw, lr * gw_tol + 2.0 ** -23 * np.abs(w), (nsp, mode, "W"))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("nsp", [1, 2, 3])
def test_captured_step_replays_the_eager_step(nk, dev, nsp, mode):
    """the same training step eager and captured in one mode give the same weight bits (everything this engine
    computes); switching the mode after the capture does not change what the replay computes"""
    rng = np.random.default_rng(10 + nsp)
    layer, xs, _ = make_layer(nk, dev, nsp, rng)
    params = layer.parameters()
    init = [p.data().copy() for p in params]
    opt = nk.optim.StochasticGD.new(0.1)
    for p in params:
        opt.register(p)
    X = nk.from_ndarray(dev, rng.standard_normal(xs).astype(F32))
    y0 = layer.forward(X)
    T = nk.from_ndarray(dev, rng.standard_normal(y0.data().shape).astype(F32))
    kernels = []

    def step():
        opt.zero_grad()
        loss = layer.forward(X).relu().mse_loss(T)
        loss.forward()
        loss.backward(1.0)
        kernels.append(dev.last_conv_kernel)
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    dev.f32_conv(mode)
    step()                     # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [p.data().copy() for p in params]
    assert kernels[-1] == names(mode, nsp != 2)[2]
    assert any(np.any(e != i) for e, i in zip(eager, init))
    reset()
    with dev.capture(256 << 20) as cap:
        step()
    dev.f32_conv("tf32x3" if mode == "tf32" else "ieee")
    for _ in range(2):
        reset()
        cap.graph.launch()
        dev.synchronize()
        w, b = params[0].data(), params[1].data()
        assert np.array_equal(w.view(np.uint32), eager[0].view(np.uint32)), (nsp, mode)
        # The bias gradient is not this engine's: nk_unbroadcast_acc sums g over (N, L) with chansum_kernel, whose
        # blocks each add a partial sum into the f32 result with atomicAdd.  The order of those adds is whatever order
        # the blocks finish in, so two runs of the same step -- eager or replayed -- may differ in the last bit of db.
        assert np.all(np.abs(b - eager[1]) <= 2.0 ** -22 * np.abs(eager[1]) + 1e-9), (nsp, mode)
    cap.graph.close()
