"""The 1-D / 3-D convolution layers on the GPU: the layer entry points nk_conv_layer_nd_* (ops.conv_layer_nd*), the
one-node graph op (variable.conv_layer) and nn.Conv1d / nn.Conv3d.

Parity: against the oracle in float64 on the stored operands -- pad_mode_forward -> conv_forward -> + bias, and for dX
the gradient of the padded input sliced to its interior (pad_mode_backward, the reference's rule for every mode) -- with
the elementwise bound of tests/test_gpu_cuda_core_conv_edges.py: (taps + 4).2^-24.sum|terms| plus 2^-8.|want| for a bf16
output (2^-7 when accumulated into).  Every call's kernel is pinned: the tensor-core engine ("wgmma_im2col_nd_*") for
bf16 shapes it takes, the CUDA-core kernels ("direct_nd_*") for f32, K = Cin.prod(k) < 9, Cout < 8 (forward and dX) and
under conv_engine("direct")."""
import numpy as np
import pytest

from test_gpu_cuda_core_conv_edges import U, rounded

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = ["zero", "constant", "reflective", "replicative"]
ORACLE_MODE = {"zero": "constant", "constant": "constant", "reflective": "reflective", "replicative": "replicative"}
WGMMA = ("wgmma_im2col_nd_fwd", "wgmma_im2col_nd_dx", "wgmma_im2col_nd_dw")
DIRECT = ("direct_nd_fwd", "direct_nd_dx", "direct_nd_dw")


def check(got, want, mag, terms, bf16_out, accumulated, what, extra=0.0):
    """|got - want| <= terms.2^-24.mag (+ 2^-8 / 2^-7 of |want| for a bf16 output) + extra: the bound of
    test_gpu_cuda_core_conv_edges.check, plus one rounding of an intermediate that the CUDA-core path stores in bf16 as
    the composed graph does (the convolution before the bias add, the padded input's gradient before its interior
    slice)"""
    want = np.asarray(want, np.float64)
    rel = (2.0 ** -7 if accumulated else 2.0 ** -8) if bf16_out else 0.0
    tol = terms * U * mag + rel * np.abs(want) + extra
    err = np.abs(np.asarray(got, np.float64) - want)
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), np.unravel_index(int(np.argmax(err - tol)), err.shape),
                           float(err.max()))


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


def fill_value(mode):
    return 0.75 if mode == "constant" else 0.0


def oracle_layer(O, x64, w64, b64, pad, mode, stride, dil):
    """(y, |y| terms, padded x, padded |x|) in float64 of conv(pad(x)) + b"""
    om, v = ORACLE_MODE[mode], fill_value(mode)
    xp = O.pad_mode_forward(x64, pad, om, v)
    xpa = O.pad_mode_forward(np.abs(x64), pad, om, abs(v))
    bb = b64.reshape((1, -1) + (1,) * len(pad))
    y = O.conv_forward(xp, w64, stride, dil).astype(np.float64) + bb
    mag = O.conv_forward(xpa, np.abs(w64), stride, dil).astype(np.float64) + np.abs(bb)
    return y, mag, xp, xpa


def oracle_dx(O, xs, g64, w64, pad, stride, dil):
    """the interior slice of the padded input's gradient, and the same on absolute values"""
    padded = xs[:2] + tuple(s + 2 * p for s, p in zip(xs[2:], pad))
    out = []
    for gg, ww in ((g64, w64), (np.abs(g64), np.abs(w64))):
        gp = O.conv_backward_input(np.zeros(padded), gg, ww, stride, dil)
        out.append(O.pad_mode_backward(gp, np.zeros(xs), pad))
    return out


def layer_case(nk, dev, O, xs, cout, k, pad, mode, stride, dil, dtype, kernels, seed=0):
    """the forward, dX (beta 0 and 1) and dW + db into f32 and bf16 (beta 0 and 1) through the layer entry points against
    the oracle; each call's kernel is pinned to `kernels`.  Returns {name: (got, mag, taps, extra)} of y, dX and dW (f32,
    beta 0)"""
    from neuronika_b200 import ops
    bf = dtype == "bf16"
    dt = nk.BF16 if bf else nk.F32
    rng = np.random.default_rng(seed)
    n, cin = xs[:2]
    x = rounded(O, rng.uniform(-1, 1, xs), bf)
    wt = rounded(O, rng.uniform(-0.5, 0.5, (cout, cin) + tuple(k)), bf)
    b = rounded(O, rng.uniform(-0.5, 0.5, (cout,)), bf)
    x64, w64, b64 = x.astype(np.float64), wt.astype(np.float64), b.astype(np.float64)
    X, W, B = dev.from_ndarray(x, dt), dev.from_ndarray(wt, dt), dev.from_ndarray(b, dt)
    out = {}
    value = fill_value(mode)
    mode_c = "constant" if mode == "zero" else mode

    want, mag, xp, xpa = oracle_layer(O, x64, w64, b64, pad, mode, stride, dil)
    y = ops.conv_layer_nd(X, W, pad, mode_c, value, stride, dil, bias=B)
    assert dev.last_conv_kernel == kernels[0], dev.last_conv_kernel
    taps = cin * int(np.prod(k))
    got = y.as_ndarray()
    twice = bf and kernels[0].startswith("direct")      # bf16 convolution, then the bias add
    extra = 2.0 ** -8 * np.abs(want - b64.reshape((1, -1) + (1,) * len(pad))) if twice else 0.0
    check(got, want, mag, taps + 4, bf, False, "y", extra)
    out["y"] = (got, mag, taps + 4, extra)

    g = rounded(O, rng.uniform(-1, 1, want.shape), bf)
    g64 = g.astype(np.float64)
    G = dev.from_ndarray(g, dt)
    gx, gx_mag = oracle_dx(O, xs, g64, w64, pad, stride, dil)
    dx0 = rounded(O, rng.uniform(-1, 1, xs), bf)
    taps = cout * int(np.prod(k))
    extra = 2.0 ** -8 * np.abs(gx) if bf and kernels[1].startswith("direct") else 0.0   # the padded gradient in bf16
    for beta in (0.0, 1.0):
        DX = dev.from_ndarray(dx0, dt)
        ops.conv_layer_nd_bwd_input(DX, G, W, pad, mode_c, stride, dil, beta=beta)
        assert dev.last_conv_kernel == kernels[1], dev.last_conv_kernel
        got = DX.as_ndarray()
        check(got, beta * dx0 + gx, gx_mag + np.abs(beta * dx0), taps + 4, bf, beta != 0, ("dx", beta), extra)
        if beta == 0:
            out["dx"] = (got, gx_mag, taps + 4, extra)

    nl = n * int(np.prod(want.shape[2:]))
    gw = O.conv_backward_kernel(np.zeros(wt.shape), g64, xp, stride, dil)
    gw_mag = O.conv_backward_kernel(np.zeros(wt.shape), np.abs(g64), xpa, stride, dil)
    axes = tuple(i for i in range(g.ndim) if i != 1)
    gb, gb_mag = g64.sum(axis=axes), np.abs(g64).sum(axis=axes)
    for dwt in (nk.F32, nk.BF16):
        dbf = dwt == nk.BF16
        dw0 = rounded(O, rng.uniform(-1, 1, wt.shape), dbf)
        db0 = rounded(O, rng.uniform(-1, 1, (cout,)), dbf)
        for beta in (0.0, 1.0):
            DW, DB = dev.from_ndarray(dw0, dwt), dev.from_ndarray(db0, dwt)
            ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, mode_c, value, stride, dil, beta=beta, dbias=DB)
            assert dev.last_conv_kernel == kernels[2], dev.last_conv_kernel
            got = DW.as_ndarray()
            check(got, beta * dw0 + gw, gw_mag + np.abs(beta * dw0), nl + 4, dbf, beta != 0, ("dw", dbf, beta))
            check(DB.as_ndarray(), beta * db0 + gb, gb_mag + np.abs(beta * db0), nl + 4, dbf, beta != 0, ("db", dbf, beta))
            if beta == 0 and not dbf:
                out["dw"] = (got, gw_mag, nl + 4, 0.0)
    return out


# name: (x shape, cout, kernel, padding, stride, dilation)
SHAPES = {
    # L = 37 + 2.2 - 2 = 39 outputs: L % 8 != 0 (the gradient rows are copied to a pitch of 40)
    "1d": ((3, 16, 37), 16, (3,), (2,), (1,), (1,)),
    "1d_stride_dilation": ((2, 8, 41), 16, (4,), (5,), (2,), (3,)),
    "3d": ((2, 4, 6, 7, 9), 8, (3, 2, 3), (1, 2, 2), (1, 1, 1), (1, 1, 1)),
    "3d_unequal_stride_dilation": ((2, 3, 9, 8, 11), 16, (2, 3, 2), (1, 2, 3), (2, 1, 3), (2, 1, 1)),
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_layer_tensor_cores(nk, dev, O, shape, mode):
    xs, cout, k, pad, s, d = SHAPES[shape]
    layer_case(nk, dev, O, xs, cout, k, pad, mode, s, d, "bf16", WGMMA, seed=len(shape) + len(mode))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", ["1d_stride_dilation", "3d_unequal_stride_dilation"])
def test_layer_f32_runs_on_cuda_cores(nk, dev, O, shape, mode):
    xs, cout, k, pad, s, d = SHAPES[shape]
    layer_case(nk, dev, O, xs, cout, k, pad, mode, s, d, "f32", DIRECT, seed=len(shape) + len(mode))


def test_layer_outside_the_engine(nk, dev, O):
    """Cout < 8: forward and dX on the CUDA cores (dW stays on the tensor cores, as in 2-D); K = 2.3 = 6 < 9: all three"""
    layer_case(nk, dev, O, (2, 4, 23), 4, (3,), (1,), "reflective", (1,), (1,), "bf16",
               ("direct_nd_fwd", "direct_nd_dx", "wgmma_im2col_nd_dw"), seed=1)
    layer_case(nk, dev, O, (2, 2, 5, 6, 7), 8, (1, 3, 1), (0, 1, 0), "replicative", (1, 1, 1), (1, 1, 1), "bf16",
               DIRECT, seed=2)


@pytest.mark.parametrize("shape", ["1d", "3d_unequal_stride_dilation"])
def test_engines_agree(nk, dev, O, shape):
    """the bf16 layer under conv_engine("direct") and on the tensor cores: each within the bound of the oracle, and of
    each other"""
    xs, cout, k, pad, s, d = SHAPES[shape]
    tc = layer_case(nk, dev, O, xs, cout, k, pad, "replicative", s, d, "bf16", WGMMA, seed=9)
    dev.conv_engine("direct")
    try:
        cc = layer_case(nk, dev, O, xs, cout, k, pad, "replicative", s, d, "bf16", DIRECT, seed=9)
    finally:
        dev.conv_engine("auto")
    for name in ("y", "dx", "dw"):
        got, mag, taps, _ = tc[name]
        bf16_out = name != "dw"
        check(got, cc[name][0], mag, 2 * taps, bf16_out, bf16_out, ("engines", name), cc[name][3])


def test_sample_chunks(nk, dev, O):
    """N = 600 samples of 16384 positions and K = 8.31 = 248: the 4 GB column buffer holds 528 samples (bf16; 264 for
    the f32 dX columns), so every product runs over two or three chunks with a partial last one.  Sample i is the first
    sample scaled by 2^-(i % 4) (exact in bf16), so its forward and dX are the first sample's scaled, and dW and db are
    the first sample's times the sum of the scales."""
    from neuronika_b200 import ops
    n, cin, length, cout, k, pad = 600, 8, 16384, 8, (31,), (15,)
    rng = np.random.default_rng(4)
    scale = 2.0 ** -(np.arange(n) % 4)
    x1 = rounded(O, rng.uniform(-1, 1, (1, cin, length)), True)
    wt = rounded(O, rng.uniform(-0.5, 0.5, (cout, cin) + k), True)
    x = (x1 * scale[:, None, None]).astype(F32)
    X, W = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(wt, nk.BF16)
    b0 = np.zeros(cout, np.float64)
    y1, mag1, xp1, xpa1 = oracle_layer(O, x1.astype(np.float64), wt.astype(np.float64), b0, pad, "replicative", (1,), (1,))
    y = ops.conv_layer_nd(X, W, pad, "replicative", 0.0, (1,), (1,))
    assert dev.last_conv_kernel == WGMMA[0]
    sc = scale[:, None, None]
    check(y.as_ndarray(), y1 * sc, mag1 * sc, cin * 31 + 4, True, False, "y")
    del y
    g1 = rounded(O, rng.uniform(-1, 1, y1.shape), True)
    G = dev.from_ndarray((g1 * sc).astype(F32), nk.BF16)
    gx, gx_mag = oracle_dx(O, x1.shape, g1.astype(np.float64), wt.astype(np.float64), pad, (1,), (1,))
    DX = dev.zeros(x.shape, nk.BF16)
    ops.conv_layer_nd_bwd_input(DX, G, W, pad, "replicative", beta=0.0)
    assert dev.last_conv_kernel == WGMMA[1]
    check(DX.as_ndarray(), gx * sc, gx_mag * sc, cout * 31 + 4, True, False, "dx")
    del DX
    # dW of sample i = scale_i^2 . dW of the first sample (x and g both scaled); db: scale_i . db of the first
    gw1 = O.conv_backward_kernel(np.zeros(wt.shape), g1.astype(np.float64), xp1, (1,), (1,))
    gw1_mag = O.conv_backward_kernel(np.zeros(wt.shape), np.abs(g1.astype(np.float64)), xpa1, (1,), (1,))
    s2 = float((scale ** 2).sum())
    DW, DB = dev.zeros(wt.shape, nk.F32), dev.zeros((cout,), nk.F32)
    ops.conv_layer_nd_bwd_kernel(DW, G, X, pad, "replicative", beta=0.0, dbias=DB)
    assert dev.last_conv_kernel == WGMMA[2]
    check(DW.as_ndarray(), gw1 * s2, gw1_mag * s2, n * length + 4, False, False, "dw")
    gb1 = g1.astype(np.float64).sum(axis=(0, 2))
    check(DB.as_ndarray(), gb1 * scale.sum(), np.abs(g1).astype(np.float64).sum(axis=(0, 2)) * scale.sum(),
          n * length + 4, False, False, "db")


@pytest.mark.parametrize("nsp", [1, 3])
def test_empty_batch(nk, dev, O, nsp):
    """N = 0 with NULL data: the forward and dX do nothing; dW and db become beta times their old values"""
    from neuronika_b200 import ops, _lib as L
    lib = ops.lib
    cin, cout = 16, 8
    sp, k = [7, 6, 5][:nsp], [3, 2, 2][:nsp]
    one, pad = [1] * nsp, [1] * nsp
    geom = [nsp, 0, cin, L.shape_arr(sp), cout, L.shape_arr(k), L.shape_arr(one), L.shape_arr(one), L.shape_arr(pad),
            L.NK_PAD_REFLECTIVE]
    nk._lib.check(lib.nk_conv_layer_nd_fwd(dev.ctx, None, None, None, None, *geom, 0.0, nk.BF16), dev.ctx)
    nk._lib.check(lib.nk_conv_layer_nd_bwd_input(dev.ctx, None, None, None, *geom, nk.BF16, 1.0), dev.ctx)
    rng = np.random.default_rng(nsp)
    for beta in (0.0, 0.5, 1.0):
        dw0 = rounded(O, rng.uniform(-1, 1, (cout, cin) + tuple(k)), False)
        db0 = rounded(O, rng.uniform(-1, 1, (cout,)), False)
        DW, DB = dev.from_ndarray(dw0, nk.F32), dev.from_ndarray(db0, nk.F32)
        nk._lib.check(lib.nk_conv_layer_nd_bwd_kernel(dev.ctx, DW.ptr, nk.F32, DB.ptr, None, None, *geom, 0.0, nk.BF16,
                                                      beta), dev.ctx)
        assert np.array_equal(DW.as_ndarray(), beta * dw0) and np.array_equal(DB.as_ndarray(), beta * db0), beta


def test_argument_errors(nk, dev):
    from neuronika_b200 import ops
    x = dev.zeros((2, 4, 5), nk.BF16)
    w = dev.zeros((8, 4, 3), nk.BF16)
    with pytest.raises(nk.NkError, match="reflective padding 5 must be smaller than the dimension 5"):
        ops.conv_layer_nd(x, w, (5,), "reflective")
    with pytest.raises(nk.NkError, match="kernel size can't be greater than actual input size"):
        ops.conv_layer_nd(x, dev.zeros((8, 4, 8), nk.BF16), (1,), "constant")
    x2 = dev.zeros((2, 4, 5, 5), nk.BF16)
    with pytest.raises(nk.NkError, match="1 or 3 sample dimensions"):
        ops.conv_layer_nd(x2, dev.zeros((8, 4, 3, 3), nk.BF16), (1, 1), "constant")


# ------------------------------------------------------------------------------------------- graph node and layers
def composed(V, x, w, b, pad, mode, stride, dil):
    xp = x.pad(pad, fill_value(mode), mode=mode) if any(pad) else x
    return w.convolution(xp, stride, dil, 1) + b


@pytest.mark.parametrize("nsp", [1, 3])
@pytest.mark.parametrize("mode", MODES)
def test_f32_node_is_bit_equal_to_the_composed_graph(nk, dev, O, nsp, mode):
    """f32: one conv_layer node and pad -> convolution -> + bias make the same bits, forward and every gradient.  Two
    samples: the CUDA-core dW kernel adds per-chunk partial sums of the batch with f32 atomics, which commute for two
    chunks only."""
    from neuronika_b200 import variable as V
    rng = np.random.default_rng(nsp * 7 + len(mode))
    xs, k, pad, s, d = ((2, 5, 19), (3,), (2,), (2,), (1,)) if nsp == 1 else \
        ((2, 3, 6, 5, 7), (2, 3, 2), (1, 2, 1), (1, 2, 1), (2, 1, 1))
    cout = 6
    arrays = [rng.uniform(-1, 1, xs), rng.uniform(-0.5, 0.5, (cout, xs[1]) + k), rng.uniform(-0.5, 0.5, (cout,) + (1,) * nsp)]
    results = []
    for one_node in (True, False):
        x, w, b = (nk.from_ndarray(dev, a.astype(F32), nk.F32).requires_grad() for a in arrays)
        if one_node:
            y = V.conv_layer(x, w, b, pad, mode, fill_value(mode), s, d)
        else:
            y = composed(V, x, w, b, pad, mode, s, d)
        target = nk.from_ndarray(dev, np.zeros(y.shape, F32), nk.F32)
        loss = y.mse_loss(target)
        loss.forward()
        loss.backward(1.0)
        results.append([y.data(), x.grad(), w.grad(), b.grad()])
        if one_node:
            assert dev.last_conv_kernel == "direct_nd_dw"
    for name, a, c in zip(("y", "dx", "dw", "db"), *results):
        assert np.array_equal(a.view(np.uint32), c.view(np.uint32)), name


@pytest.mark.parametrize("grad_dtype", ["f32", "bf16"])
def test_node_gradients_and_accumulation(nk, dev, O, grad_dtype):
    """a bf16 Conv3d node with f32 or bf16 gradients: within the bound of the oracle; the input as a Var gets nothing
    and costs no dX; a second backward() doubles every gradient"""
    from neuronika_b200 import variable as V
    gdt = nk.F32 if grad_dtype == "f32" else nk.BF16
    rng = np.random.default_rng(3)
    xs, cout, k, pad, s, d = SHAPES["3d_unequal_stride_dilation"]
    xa = rounded(O, rng.uniform(-1, 1, xs), True)
    wa = rounded(O, rng.uniform(-0.5, 0.5, (cout, xs[1]) + k), True)
    ba = rounded(O, rng.uniform(-0.5, 0.5, (cout, 1, 1, 1)), True)
    for x_diff in (True, False):
        x = nk.from_ndarray(dev, xa, nk.BF16)
        if x_diff:
            x = x.requires_grad(gdt)
        w = nk.from_ndarray(dev, wa, nk.BF16).requires_grad(gdt)
        b = nk.from_ndarray(dev, ba, nk.BF16).requires_grad(gdt)
        y = V.conv_layer(x, w, b, pad, "reflective", 0.0, s, d)
        y.forward()
        assert dev.last_conv_kernel == WGMMA[0]
        y.backward(1.0)
        assert dev.last_conv_kernel == WGMMA[2]
        want, mag, xp, xpa = oracle_layer(O, xa.astype(np.float64), wa.astype(np.float64), ba.ravel().astype(np.float64),
                                          pad, "reflective", s, d)
        check(y.data(), want, mag, xs[1] * int(np.prod(k)) + 4, True, False, "y")
        g = np.ones(want.shape)
        bf = gdt == nk.BF16
        gw = O.conv_backward_kernel(np.zeros(wa.shape), g, xp, s, d)
        gw_mag = O.conv_backward_kernel(np.zeros(wa.shape), g, xpa, s, d)
        nl = int(np.prod(want.shape)) // cout
        first = [w.grad(), b.grad()]
        check(first[0], gw, gw_mag, nl + 4, bf, False, "dw")
        check(first[1].ravel(), np.full(cout, nl), np.full(cout, nl), nl + 4, bf, False, "db")
        if x_diff:
            gx, gx_mag = oracle_dx(O, xs, g, wa.astype(np.float64), pad, s, d)
            first.append(x.grad())
            # dX is produced in the data type (bf16) and then added into the gradient
            check(first[2], gx, gx_mag, cout * int(np.prod(k)) + 4, True, False, "dx")
        y.backward(1.0)
        again = [w.grad(), b.grad()] + ([x.grad()] if x_diff else [])
        for a, c in zip(first, again):
            tol = (2.0 ** -7 if bf else 2.0 ** -22) * np.abs(2 * a) + 1e-6 * np.abs(a).max()
            assert np.all(np.abs(c - 2 * a) <= tol)
        if not x_diff:
            assert type(x) is nk.Var


def test_layers_hold_the_reference_parameters(nk, dev):
    rng = np.random.default_rng(0)
    c1 = nk.nn.Conv1d(dev, 4, 8, 3, padding=1, padding_mode=nk.nn.ReflectivePad(), rng=rng)
    c3 = nk.nn.Conv3d(dev, 2, 8, (3, 1, 2), padding=(1, 0, 1), padding_mode=nk.nn.ReplicativePad(), rng=rng)
    assert [p.shape for p in c1.parameters()] == [(8, 4, 3), (8, 1)]
    assert [p.shape for p in c3.parameters()] == [(8, 2, 3, 1, 2), (8, 1, 1, 1)]
    for layer, fan_in in ((c1, 12), (c3, 12)):
        k = np.sqrt(1.0 / fan_in)
        for p in layer.parameters():
            assert np.abs(p.data()).max() <= k
    y = c3.forward(nk.from_ndarray(dev, np.ones((1, 2, 4, 4, 4), F32)))
    assert y.shape == (1, 8, 4, 4, 5) and y.history_len() == 1


def test_conv2d_reflective_padding_routes_through_pad(nk, dev, O):
    """nn.Conv2d with the new padding modes pads with them (f32: the composed graph's exact values)"""
    rng = np.random.default_rng(5)
    conv = nk.nn.Conv2d(dev, 2, 4, (3, 3), padding=(1, 2), padding_mode=nk.nn.ReflectivePad(), rng=rng)
    xa = rng.uniform(-1, 1, (2, 2, 6, 7)).astype(F32)
    y = conv.forward(nk.from_ndarray(dev, xa))
    y.forward()
    xp = O.pad_mode_forward(xa, (1, 2), "reflective")
    want = O.conv_forward(xp, conv.weight.data(), (1, 1), (1, 1)) + conv.bias.data()[None]
    assert np.allclose(y.data(), want, rtol=1e-5, atol=1e-5)


def test_captured_training_step_matches_eager(nk, dev):
    """Conv1d -> ReLU -> Conv1d -> flatten -> Linear -> mse, zero_grad -> forward -> backward -> SGD captured once and
    replayed from the same parameters as an eager step: the same parameters afterwards"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(8)
    n, cin, length = 16, 8, 64
    c1 = nk.nn.Conv1d(dev, cin, 16, 5, padding=2, padding_mode=nk.nn.ReplicativePad(), dtype=nk.BF16,
                      grad_dtype=nk.F32, rng=rng)
    c2 = nk.nn.Conv1d(dev, 16, 16, 3, padding=1, stride=2, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    head = nk.nn.Linear(dev, 16 * 32, 10, nk.BF16, grad_dtype=nk.F32, rng=rng)
    params = c1.parameters() + c2.parameters() + head.parameters()
    init = [p.data().copy() for p in params]
    opt = optim.StochasticGD.new(0.05)
    for p in params:
        opt.register(p)
    x = nk.from_ndarray(dev, rng.standard_normal((n, cin, length)).astype(F32), nk.BF16)
    tgt = nk.from_ndarray(dev, rng.standard_normal((n, 10)).astype(F32), nk.BF16)
    kernels = []

    def step():
        opt.zero_grad()
        loss = head.forward(c2.forward(c1.forward(x).relu()).flatten()).mse_loss(tgt)
        loss.forward()
        kernels.append(dev.last_conv_kernel)
        loss.backward(1.0)
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    step()                     # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [p.data().copy() for p in params]
    assert kernels[-1] == WGMMA[0]
    assert any(np.any(e != i) for e, i in zip(eager, init))
    reset()
    with dev.capture(256 << 20) as cap:
        step()
    reset()
    cap.graph.launch()
    dev.synchronize()
    for i, (p, e) in enumerate(zip(params, eager)):
        got = p.data()
        assert np.all(np.abs(got - e) <= 2.0 ** -7 * np.abs(e) + 1e-6), i
    cap.graph.close()
