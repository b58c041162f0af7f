"""The CUDA-core convolution engines at their edges: the direct 2-D kernels (nk_conv_direct.cu) and the 1-D / 3-D gather
kernels (nk_conv_nd.cu).  Covered: f32 and bf16 data, groups 1, 2 and depthwise, unequal strides and dilations, stride >
kernel (input rows and columns that no tap reads), grid-stride lengths past the sm_count.16.256 outputs of one pass, the
batch chunking of dW (several samples per block with a partial last chunk), dW into the other dtype, an empty batch, the
2-D case of the N-d engine against conv2d, and the argument errors.

Every case runs the forward (2-D: plain and with bias + ReLU), dX with beta 0 and 1, and dW into f32 and bf16 with beta 0
and 1 (2-D: with the bias gradient), against the oracle in float64 on the stored operands, and pins the kernel each call
takes.  The bound is elementwise, (taps + 4).2^-24.sum|terms| per output, where sum|terms| is the same operation on
absolute values plus |beta.old| (and |bias|); for dW and the bias gradient taps is the number of summed products (f32
atomics, per-block order).  bf16 outputs add 2^-8.|want|, or 2^-7.|want| when accumulated into.  dX elements that no tap
reaches are exactly beta.dx0."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24
DIRECT = ("direct_fwd", "direct_bwd_input", "direct_bwd_kernel")
ND = ("direct_nd_fwd", "direct_nd_dx", "direct_nd_dw")


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


def rounded(O, v, bf16):
    v = np.asarray(v, F32)
    return O.bf16_round(v) if bf16 else v


def check(got, want, mag, terms, bf16_out, accumulated, what):
    """|got - want| <= terms.2^-24.mag (+ 2^-8 / 2^-7 of |want| for a bf16 output)"""
    want = np.asarray(want, np.float64)
    rel = (2.0 ** -7 if accumulated else 2.0 ** -8) if bf16_out else 0.0
    tol = terms * U * mag + rel * np.abs(want)
    err = np.abs(np.asarray(got, np.float64) - want)
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), np.unravel_index(int(np.argmax(err - tol)), err.shape),
                           float(err.max()))


def tap_reached(n_in, k, s, d, n_out):
    """which input positions of one axis some (output, tap) pair reads"""
    hit = np.zeros(n_in, bool)
    for i in range(k):
        hit[i * d + s * np.arange(n_out)] = True
    return hit


def dw_chunking(sm, n, weights):
    """samples per block of the dW kernels (nk_conv_direct.cu / nk_conv_nd.cu): (per block, blocks along the batch)"""
    want_y = min(-(-(4 * sm) // weights), n, 65535)
    per = -(-n // max(1, want_y))
    return per, -(-n // per)


@pytest.fixture
def direct_engine(dev):
    dev.conv_engine("direct")
    yield
    dev.conv_engine("auto")


def conv_case(nk, dev, O, xs, cout, k, stride, dil, groups, dtype, *, nd=False, seed=0):
    """the whole protocol on one shape; nd: through the N-d entry points (no bias), else conv2d.  Returns
    {name: (got, mag, taps)} of the forward, dX (beta 0) and dW (f32, beta 0), for comparisons between engines."""
    from neuronika_b200 import ops
    kernels = ND if nd else DIRECT
    bf = dtype == "bf16"
    dt = nk.BF16 if bf else nk.F32
    rng = np.random.default_rng(seed)
    n, cin = xs[:2]
    sp = xs[2:]
    cin_g, cout_g = cin // groups, cout // groups
    x = rounded(O, rng.uniform(-1, 1, xs), bf)
    wt = rounded(O, rng.uniform(-0.5, 0.5, (cout, cin_g) + tuple(k)), bf)
    b = rounded(O, rng.uniform(-0.5, 0.5, (cout,)), bf)
    x64, w64 = x.astype(np.float64), wt.astype(np.float64)
    X, W, B = dev.from_ndarray(x, dt), dev.from_ndarray(wt, dt), dev.from_ndarray(b, dt)
    out = {}

    # forward (2-D: also with the bias + ReLU epilogue)
    taps = cin_g * int(np.prod(k))
    want = O.conv_forward(x64, w64, stride, dil, groups).astype(np.float64)
    mag = O.conv_forward(np.abs(x64), np.abs(w64), stride, dil, groups).astype(np.float64)
    y = ops.convnd(X, W, stride, dil, groups) if nd else ops.conv2d(X, W, stride, dil, groups)
    assert dev.last_conv_kernel == kernels[0], dev.last_conv_kernel
    got = y.as_ndarray()
    check(got, want, mag, taps + 4, bf, False, "y")
    out["y"] = (got, mag, taps + 4)
    if not nd:
        yb = ops.conv2d(X, W, stride, dil, groups, bias=B, relu=True)
        assert dev.last_conv_kernel == kernels[0]
        bb = b.astype(np.float64)[None, :, None, None]
        check(yb.as_ndarray(), np.maximum(want + bb, 0), mag + np.abs(bb), taps + 4, bf, False, "y + bias, relu")

    # dX, beta 0 and 1; elements that no tap reaches keep exactly beta.dx0
    g = rounded(O, rng.uniform(-1, 1, want.shape), bf)
    g64 = g.astype(np.float64)
    G = dev.from_ndarray(g, dt)
    gx = O.conv_backward_input(np.zeros(xs), g64, w64, stride, dil, groups)
    gx_mag = O.conv_backward_input(np.zeros(xs), np.abs(g64), np.abs(w64), stride, dil, groups)
    reach = np.ones(sp, bool)
    for ax, (ni, ki, si, di, no) in enumerate(zip(sp, k, stride, dil, want.shape[2:])):
        shape = [1] * len(sp)
        shape[ax] = ni
        reach = reach & tap_reached(ni, ki, si, di, no).reshape(shape)
    dx0 = rounded(O, rng.uniform(-1, 1, xs), bf)
    taps = cout_g * int(np.prod(k))
    for beta in (0.0, 1.0):
        DX = dev.from_ndarray(dx0, dt)
        if nd:
            ops.convnd_bwd_input(DX, G, W, stride, dil, groups, beta=beta)
        else:
            ops.conv2d_bwd_input(DX, G, W, stride, dil, groups, beta=beta)
        assert dev.last_conv_kernel == kernels[1], dev.last_conv_kernel
        got = DX.as_ndarray()
        check(got, beta * dx0 + gx, gx_mag + np.abs(beta * dx0), taps + 4, bf, beta != 0, ("dx", beta))
        assert np.array_equal(got[:, :, ~reach], (beta * dx0)[:, :, ~reach]), ("untouched dx", beta)
        if beta == 0:
            out["dx"] = (got, gx_mag, taps + 4)

    # dW into f32 and bf16, beta 0 and 1 (2-D: with the bias gradient)
    nl = n * int(np.prod(want.shape[2:]))
    gw = O.conv_backward_kernel(np.zeros(wt.shape), g64, x64, stride, dil, groups)
    gw_mag = O.conv_backward_kernel(np.zeros(wt.shape), np.abs(g64), np.abs(x64), stride, dil, groups)
    gb = g64.sum(axis=tuple(i for i in range(g.ndim) if i != 1))
    gb_mag = np.abs(g64).sum(axis=tuple(i for i in range(g.ndim) if i != 1))
    for dwt in (nk.F32, nk.BF16):
        dbf = dwt == nk.BF16
        dw0 = rounded(O, rng.uniform(-1, 1, wt.shape), dbf)
        db0 = rounded(O, rng.uniform(-1, 1, (cout, 1, 1)), dbf)
        for beta in (0.0, 1.0):
            DW, DB = dev.from_ndarray(dw0, dwt), dev.from_ndarray(db0, dwt)
            if nd:
                ops.convnd_bwd_kernel(DW, G, X, stride, dil, groups, beta=beta)
            else:
                ops.conv2d_bwd_kernel(DW, G, X, stride, dil, groups, beta=beta, dbias=DB)
            assert dev.last_conv_kernel == kernels[2], dev.last_conv_kernel
            got = DW.as_ndarray()
            check(got, beta * dw0 + gw, gw_mag + np.abs(beta * dw0), nl + 4, dbf, beta != 0, ("dw", dbf, beta))
            if beta == 0 and not dbf:
                out["dw"] = (got, gw_mag, nl + 4)
            if not nd:
                db = db0.ravel().astype(np.float64)
                check(DB.as_ndarray().ravel(), beta * db + gb, gb_mag + np.abs(beta * db), nl + 4, dbf, beta != 0,
                      ("db", dbf, beta))
    return out


# ------------------------------------------------------------------------------------------- direct 2-D
DIRECT_CASES = {
    # name: (x shape, cout, kernel, stride, dilation, groups, dtype)
    "f32_unequal_stride_dilation": ((2, 3, 11, 13), 4, (3, 2), (2, 1), (1, 2), 1, "f32"),
    "f32_stride_gt_kernel": ((2, 3, 14, 17), 5, (2, 2), (3, 3), (1, 1), 1, "f32"),
    "f32_groups2": ((2, 4, 9, 10), 6, (3, 3), (1, 2), (2, 1), 2, "f32"),
    "f32_depthwise": ((2, 5, 12, 11), 10, (3, 3), (1, 2), (2, 1), 5, "f32"),
    "bf16_unequal_stride_dilation": ((2, 3, 11, 13), 8, (3, 2), (2, 1), (1, 2), 1, "bf16"),
    "bf16_groups2": ((2, 4, 9, 10), 6, (3, 3), (2, 1), (1, 1), 2, "bf16"),
    "bf16_depthwise_stride_gt_kernel": ((2, 6, 14, 17), 6, (2, 2), (3, 3), (1, 1), 6, "bf16"),
}


@pytest.mark.parametrize("name", list(DIRECT_CASES))
def test_direct_2d(nk, dev, O, direct_engine, name):
    """bf16 runs with the direct engine forced (it would take the im2col engine at groups = 1)"""
    xs, cout, k, s, d, groups, dtype = DIRECT_CASES[name]
    conv_case(nk, dev, O, xs, cout, k, s, d, groups, dtype, seed=len(name))


def grid_stride_side(sm, n, c, k):
    """a square side at which both n.c.Ho.Wo and n.c.H.W exceed the sm_count.16.256 outputs of one grid pass by 20 %"""
    cap = sm * 16 * 256
    return int(np.ceil(np.sqrt(1.2 * cap / (n * c)))) + k - 1


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_direct_2d_grid_stride(nk, dev, O, direct_engine, dtype):
    """the forward and dX past one pass of their capped grids"""
    n, c, k = 2, 4, 3
    side = grid_stride_side(dev.sm_count, n, c, k)
    assert n * c * (side - k + 1) ** 2 > dev.sm_count * 16 * 256
    conv_case(nk, dev, O, (n, c, side, side), c, (k, k), (1, 1), (1, 1), 1, dtype, seed=side)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_direct_2d_dw_batch_chunks(nk, dev, O, direct_engine, dtype):
    """4 weights and n = 1001: every dW block sums several samples and the last block fewer"""
    n = 1001
    per, blocks = dw_chunking(dev.sm_count, n, 1 * 1 * 2 * 2)
    assert per > 1 and n % per != 0, (per, blocks)
    conv_case(nk, dev, O, (n, 1, 6, 5), 1, (2, 2), (1, 2), (1, 1), 1, dtype, seed=n)


@pytest.mark.parametrize("dwt", ["f32", "bf16"])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_direct_2d_empty_batch(nk, dev, O, dtype, dwt):
    """n = 0 through the C ABI: the forward and dX do nothing; dW and the bias gradient become beta.dW0 / beta.db0 (0 for
    beta = 0), with g and x given or NULL, and the im2col engine is not entered"""
    from neuronika_b200 import ops
    lib = ops.lib
    dt = nk.BF16 if dtype == "bf16" else nk.F32
    wdt = nk.BF16 if dwt == "bf16" else nk.F32
    cin, h, w, cout, kh, kw = 4, 7, 6, 8, 3, 2
    geom = [cin, h, w, cout, kh, kw, 1, 1, 1, 1, 1]
    rng = np.random.default_rng(3)
    dummy = dev.zeros((16,), dt)          # a valid pointer to data that must not be read
    nk._lib.check(lib.nk_conv2d_fwd(dev.ctx, None, None, None, None, 0, 0, *geom, dt), dev.ctx)
    nk._lib.check(lib.nk_conv2d_bwd_input(dev.ctx, None, None, None, 0, *geom, dt, 1.0), dev.ctx)
    for beta in (0.0, 0.5, 1.0):
        for ptr in (dummy.ptr, None):
            dw0 = rounded(O, rng.uniform(-1, 1, (cout, cin, kh, kw)), wdt == nk.BF16)
            db0 = rounded(O, rng.uniform(-1, 1, (cout, 1, 1)), wdt == nk.BF16)
            DW, DB = dev.from_ndarray(dw0, wdt), dev.from_ndarray(db0, wdt)
            nk._lib.check(lib.nk_conv2d_bwd_kernel(dev.ctx, DW.ptr, wdt, DB.ptr, ptr, ptr, 0, *geom, dt, beta),
                          dev.ctx)
            assert np.array_equal(DW.as_ndarray(), beta * dw0), ("dW of an empty batch", beta, ptr is None)
            assert np.array_equal(DB.as_ndarray(), beta * db0), ("dbias of an empty batch", beta, ptr is None)
            assert dev.last_conv_kernel == "direct_bwd_kernel"


# ------------------------------------------------------------------------------------------- N-d
ND_CASES = {
    # name: (x shape, cout, kernel, stride, dilation, groups, dtype)
    "1d_f32_groups2": ((3, 4, 29), 6, (4,), (3,), (2,), 2, "f32"),
    "1d_bf16_stride_gt_kernel": ((3, 3, 31), 5, (2,), (3,), (1,), 1, "bf16"),
    "3d_f32_groups2": ((2, 4, 7, 8, 9), 4, (2, 3, 2), (1, 2, 3), (2, 1, 1), 2, "f32"),
    "3d_bf16_depthwise": ((2, 3, 6, 7, 8), 3, (3, 2, 2), (2, 1, 1), (1, 2, 1), 3, "bf16"),
    "3d_f32_stride_gt_kernel": ((2, 2, 9, 7, 10), 3, (2, 1, 2), (3, 2, 3), (1, 1, 2), 1, "f32"),
}


@pytest.mark.parametrize("name", list(ND_CASES))
def test_nd(nk, dev, O, name):
    xs, cout, k, s, d, groups, dtype = ND_CASES[name]
    conv_case(nk, dev, O, xs, cout, k, s, d, groups, dtype, nd=True, seed=len(name))


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_nd_grid_stride(nk, dev, O, dtype):
    """1-D forward and dX past one pass of their capped grids"""
    n, c, k = 4, 8, 5
    cap = dev.sm_count * 16 * 256
    length = int(np.ceil(1.2 * cap / (n * c))) + k - 1
    conv_case(nk, dev, O, (n, c, length), c, (k,), (1,), (1,), 1, dtype, nd=True, seed=length)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_nd_dw_batch_chunks(nk, dev, O, dtype):
    """4 weights and n = 1001: every dW block sums several samples and the last block fewer"""
    n = 1001
    per, blocks = dw_chunking(dev.sm_count, n, 2 * 1 * 2)
    assert per > 1 and n % per != 0, (per, blocks)
    conv_case(nk, dev, O, (n, 1, 9), 2, (2,), (2,), (3,), 1, dtype, nd=True, seed=n)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_nd_two_sample_dims_match_conv2d(nk, dev, O, direct_engine, dtype):
    """nsp = 2 through the N-d engine agrees with conv2d on the direct engine, and both with the oracle, within the bound"""
    case = ((2, 4, 9, 11), 6, (3, 2), (2, 1), (1, 2), 2, dtype)
    nd = conv_case(nk, dev, O, *case, nd=True, seed=5)
    d2 = conv_case(nk, dev, O, *case, seed=5)
    for name in ("y", "dx", "dw"):
        got, mag, taps = nd[name]
        bf16_out = dtype == "bf16" and name != "dw"
        check(got, d2[name][0], mag, 2 * taps, bf16_out, bf16_out, ("nd vs 2d", name))


@pytest.mark.parametrize("dwt", ["f32", "bf16"])
@pytest.mark.parametrize("nsp", [1, 3])
def test_nd_empty_batch(nk, dev, O, nsp, dwt):
    """n = 0 with NULL data: the forward and dX do nothing, dW becomes beta.dW0"""
    from neuronika_b200 import ops, _lib as L
    lib = ops.lib
    wdt = nk.BF16 if dwt == "bf16" else nk.F32
    cin, cout = 4, 2
    sp, k = [7, 6, 5][:nsp], [3, 2, 2][:nsp]
    one = [1] * nsp
    geom = [cin, L.shape_arr(sp), cout, L.shape_arr(k), L.shape_arr(one), L.shape_arr(one), 1, nk.F32]
    nk._lib.check(lib.nk_convnd_fwd(dev.ctx, None, None, None, nsp, 0, *geom), dev.ctx)
    nk._lib.check(lib.nk_convnd_bwd_input(dev.ctx, None, None, None, nsp, 0, *geom, 1.0), dev.ctx)
    rng = np.random.default_rng(nsp)
    for beta in (0.0, 0.5, 1.0):
        dw0 = rounded(O, rng.uniform(-1, 1, (cout, cin) + tuple(k)), wdt == nk.BF16)
        DW = dev.from_ndarray(dw0, wdt)
        nk._lib.check(lib.nk_convnd_bwd_kernel(dev.ctx, DW.ptr, wdt, None, None, nsp, 0, *geom, beta), dev.ctx)
        assert dev.last_conv_kernel == "direct_nd_dw"
        assert np.array_equal(DW.as_ndarray(), beta * dw0), beta


@pytest.mark.parametrize("entry", ["fwd", "dx", "dw"])
def test_nd_argument_errors(nk, dev, entry):
    """a dilated kernel longer than the input, and channel counts that groups does not divide, are errors on every entry"""
    from neuronika_b200 import ops, _lib as L
    lib = ops.lib

    def call(cin, in_sp, cout, k, dil, groups):
        args = [cin, L.shape_arr(in_sp), cout, L.shape_arr(k), L.shape_arr([1] * len(k)), L.shape_arr(dil), groups,
                nk.F32]
        if entry == "fwd":
            rc = lib.nk_convnd_fwd(dev.ctx, None, None, None, len(k), 2, *args)
        elif entry == "dx":
            rc = lib.nk_convnd_bwd_input(dev.ctx, None, None, None, len(k), 2, *args, 1.0)
        else:
            rc = lib.nk_convnd_bwd_kernel(dev.ctx, None, nk.F32, None, None, len(k), 2, *args, 1.0)
        nk._lib.check(rc, dev.ctx)

    with pytest.raises(nk.NkError, match="kernel size can't be greater than actual input size"):
        call(2, [5], 2, [3], [3], 1)
    with pytest.raises(nk.NkError, match="kernel size can't be greater than actual input size"):
        call(2, [9, 4, 9], 2, [2, 3, 2], [1, 2, 1], 1)
    with pytest.raises(nk.NkError, match="In channels 3 is not divisible by groups 2"):
        call(3, [9], 4, [2], [1], 2)
    with pytest.raises(nk.NkError, match="Out channels 3 is not divisible by groups 2"):
        call(4, [9], 3, [2], [1], 2)
