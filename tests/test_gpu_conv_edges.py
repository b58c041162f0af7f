"""The im2col + batched wgmma convolution engine (bf16, groups = 1) at its edges: unequal strides and dilations, output
sizes that are not multiples of 8, strides that leave input rows and columns without a tap, the boundaries where a case
moves to the CUDA-core kernels, the shared-memory limit of the unit-step im2col, and the sample chunking of the column
buffers at config 5's layer.

Every case runs the forward (plain, and with bias + ReLU), dX with beta 0 and 1, dW into f32 and bf16 with beta 0 and 1,
and the bias gradient, against the oracle on the same bf16-rounded operands in float64, and pins the kernel each call
takes.  Tolerances: f32 outputs 2e-3.rms + 1e-6, bf16 outputs + 2^-8.|want|, accumulated into (beta = 1) + 2^-7.|want|,
with rms taken over what the call adds.  dX elements that no tap reaches are bit exact: 0 with beta 0, dx0 with beta 1."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32


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


def rms(x):
    return float(np.sqrt((np.asarray(x, np.float64) ** 2).mean())) + 1e-12


def check(got, want, fresh, bf16_out, accumulated, what):
    """|got - want| <= 2e-3.rms(fresh) + 1e-6 (+ 2^-8 / 2^-7 of |want| for bf16 outputs)"""
    want = np.asarray(want, np.float64)
    rel = (2.0 ** -7 if accumulated else 2.0 ** -8) if bf16_out else 0.0
    tol = 2e-3 * rms(fresh) + rel * np.abs(want) + 1e-6
    err = np.abs(np.asarray(got, np.float64) - want)
    assert np.all(err <= tol), (what, float(err.max()), np.unravel_index(int(np.argmax(err - tol)), err.shape))


def tap_reached(n_in, k, s, d, n_out):
    """which input positions of one axis some (output, tap) pair reads"""
    hit = np.zeros(n_in, bool)
    for i in range(k):
        hit[i * d + s * np.arange(n_out)] = True
    return hit


def offset_view(dev, data, dtype, off):
    """a device copy of `data` starting `off` elements into a larger buffer (off = 1: 2 bytes off 16-byte alignment)"""
    if off == 0:
        return dev.from_ndarray(data, dtype)
    buf = dev.zeros((data.size + off,), dtype)
    v = buf.slice_flat(off, data.shape)
    v.copy_from(data)
    return v


def conv_case(nk, dev, O, xs, cout, k, stride, dil, kernels, *, x_off=0, g_off=0, seed=0):
    """kernels = (forward, dX, dW) kernel names this case must take"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    n, cin, h, w = xs
    x = O.bf16_round(rng.uniform(-1, 1, xs).astype(F32))
    wt = O.bf16_round(rng.uniform(-0.3, 0.3, (cout, cin) + tuple(k)).astype(F32))
    b = O.bf16_round(rng.uniform(-0.5, 0.5, (cout,)).astype(F32))
    x64, w64 = x.astype(np.float64), wt.astype(np.float64)
    X, W, B = offset_view(dev, x, nk.BF16, x_off), dev.from_ndarray(wt, nk.BF16), dev.from_ndarray(b, nk.BF16)

    # forward, plain and with the bias + ReLU epilogue
    want = O.conv_forward(x64, w64, stride, dil).astype(np.float64)
    y = ops.conv2d(X, W, stride, dil)
    assert dev.last_conv_kernel == kernels[0], (dev.last_conv_kernel, kernels)
    check(y.as_ndarray(), want, want, True, False, "y")
    yb = ops.conv2d(X, W, stride, dil, bias=B, relu=True)
    assert dev.last_conv_kernel == kernels[0]
    wb = np.maximum(want + b[None, :, None, None], 0)
    check(yb.as_ndarray(), wb, want, True, False, "y + bias, relu")

    # dX: beta 0 and 1; elements no tap reaches keep exactly beta * dx0
    g = O.bf16_round(rng.uniform(-1, 1, want.shape).astype(F32))
    G = offset_view(dev, g, nk.BF16, g_off)
    gx = np.zeros(xs, np.float64)
    O.conv_backward_input(gx, g.astype(np.float64), w64, stride, dil)
    reach = tap_reached(h, k[0], stride[0], dil[0], want.shape[2])[:, None] & \
        tap_reached(w, k[1], stride[1], dil[1], want.shape[3])[None, :]
    dx0 = O.bf16_round(rng.uniform(-1, 1, xs).astype(F32))
    for beta in (0.0, 1.0):
        DX = dev.from_ndarray(dx0, nk.BF16)
        ops.conv2d_bwd_input(DX, G, W, stride, dil, beta=beta)
        assert dev.last_conv_kernel == kernels[1], (dev.last_conv_kernel, kernels)
        got = DX.as_ndarray()
        check(got, beta * dx0 + gx, gx, True, beta != 0, ("dx", beta))
        assert np.array_equal(got[:, :, ~reach], (beta * dx0)[:, :, ~reach]), ("untouched dx", beta)

    # dW into f32 and bf16, beta 0 and 1, with the bias gradient
    gw = np.zeros(wt.shape, np.float64)
    O.conv_backward_kernel(gw, g.astype(np.float64), x64, stride, dil)
    gb = g.astype(np.float64).sum((0, 2, 3))
    gb_l1 = np.abs(g.astype(np.float64)).sum((0, 2, 3))
    for dwt in (nk.F32, nk.BF16):
        bf = dwt == nk.BF16
        dw0 = rng.uniform(-1, 1, wt.shape).astype(F32)
        db0 = rng.uniform(-1, 1, (cout, 1, 1)).astype(F32)
        if bf:
            dw0, db0 = O.bf16_round(dw0), O.bf16_round(db0)
        for beta in (0.0, 1.0):
            DW, DB = dev.from_ndarray(dw0, dwt), dev.from_ndarray(db0, dwt)
            ops.conv2d_bwd_kernel(DW, G, X, stride, dil, beta=beta, dbias=DB)
            assert dev.last_conv_kernel == kernels[2], (dev.last_conv_kernel, kernels)
            check(DW.as_ndarray(), beta * dw0 + gw, gw, bf, beta != 0, ("dw", bf, beta))
            wantb = beta * db0.ravel() + gb
            rel = (2.0 ** -7 if beta else 2.0 ** -8) if bf else 0.0
            errb = np.abs(DB.as_ndarray().ravel().astype(np.float64) - wantb)
            assert np.all(errb <= 1e-5 * gb_l1 + rel * np.abs(wantb) + 1e-6), ("db", bf, beta, float(errb.max()))


WG = ("wgmma_im2col_gemm_fwd", "wgmma_im2col_gemm_dx", "wgmma_im2col_gemm_dw")
DIRECT = ("direct_fwd", "direct_bwd_input", "direct_bwd_kernel")


# ------------------------------------------------------------------------------------------- strides and dilations
@pytest.mark.parametrize("xs,cout,k,stride,dil", [
    ((2, 8, 13, 21), 16, (3, 3), (2, 1), (1, 1)),    # sh > 1, sw = 1: the vector im2col path, odd source offsets
    ((2, 8, 15, 20), 16, (3, 3), (1, 2), (2, 1)),    # unequal stride and dilation
    ((2, 8, 14, 17), 16, (2, 2), (3, 3), (1, 1)),    # stride > kernel: rows / columns of dX without a tap
    ((2, 8, 18, 18), 24, (3, 3), (2, 2), (1, 1)),    # the last input row / column is read by no window; L = 64
    ((3, 16, 19, 23), 32, (3, 3), (2, 2), (1, 1)),   # strided, Ho*Wo = 99
    ((2, 8, 16, 19), 16, (2, 3), (1, 3), (3, 1)),    # dh != dw and sh != sw together, Ho*Wo = 65
])
def test_strides_and_dilations(nk, dev, O, xs, cout, k, stride, dil):
    conv_case(nk, dev, O, xs, cout, k, stride, dil, WG, seed=sum(xs) + cout)


# ------------------------------------------------------------------------------------------- engine boundaries
@pytest.mark.parametrize("cout,kernels", [
    (7, ("direct_fwd", "direct_bwd_input", WG[2])),     # cout < 8: the forward and dX fall back
    (8, WG),
    (12, (WG[0], "direct_bwd_input", WG[2])),           # cout % 8 != 0: dX falls back, the forward does not
])
def test_output_channel_boundaries(nk, dev, O, cout, kernels):
    conv_case(nk, dev, O, (2, 6, 11, 14), cout, (3, 3), (1, 1), (1, 1), kernels, seed=cout)


@pytest.mark.parametrize("cin,k,kernels", [
    (2, (2, 2), DIRECT),      # K = 8: Kp < 16, every direction on the CUDA-core kernels
    (1, (3, 3), WG),          # K = 9
    (5, (1, 3), WG),          # K = 15
    (17, (1, 1), WG),         # K = 17
])
def test_reduction_length_boundaries(nk, dev, O, cin, k, kernels):
    conv_case(nk, dev, O, (2, cin, 12, 13), 16, k, (1, 1), (1, 1), kernels, seed=cin * 10 + k[1])


def test_gradient_view_off_alignment(nk, dev, O):
    """a g one element off 16-byte alignment is copied into padded rows even though Ho*Wo = 64 is a multiple of 8"""
    conv_case(nk, dev, O, (2, 8, 10, 10), 16, (3, 3), (1, 1), (1, 1), WG, g_off=1, seed=31)


def test_input_view_off_alignment(nk, dev, O):
    """an x that 4-byte loads cannot read sends the forward and dW to the CUDA-core kernels (dX does not read x)"""
    conv_case(nk, dev, O, (2, 8, 10, 10), 16, (3, 3), (1, 1), (1, 1), (DIRECT[0], WG[1], DIRECT[2]), x_off=1, seed=32)


@pytest.mark.parametrize("h,w", [(8, 3071), (79, 311)])
def test_unit_step_planes_at_the_shared_memory_limit(nk, dev, O, h, w):
    """(h*w + 8) * 2 bytes of staged plane: 49152 (exactly the 48 KB limit, im2col_plane_kernel) and 49154 (im2col_kernel)"""
    conv_case(nk, dev, O, (1, 2, h, w), 8, (3, 3), (1, 1), (1, 1), WG, seed=h)


# ------------------------------------------------------------------------------------------- sample chunking
def test_sample_chunking_at_config5_layer(nk, dev, O):
    """conv 32 -> 64, k3, on (N, 32, 34, 34): the 4 GiB column buffers hold 7281 samples of bf16 columns (forward, dW) and
    3640 of f32 column gradients (dX), so N = 8192 runs the forward and dW in 2 chunks and dX in 3, and config 5's
    N = 4096 runs dX in 2.  Checked: y and dx on both sides of every chunk boundary against the oracle; dW against the
    oracle on 4 samples and as the sum of two single-chunk halves; the launch count of every chunked call.
    Samples repeat with period 61 (copied on the device), which no chunk size divides."""
    import torch
    from neuronika_b200 import ops

    def in_use():
        free, whole = torch.cuda.mem_get_info()
        return whole - free

    used0 = in_use()
    cin, hh, ww_, cout = 32, 34, 34, 64
    ho, wo = hh - 2, ww_ - 2
    period = 61
    rng = np.random.default_rng(55)
    xp = O.bf16_round(rng.uniform(-1, 1, (period, cin, hh, ww_)).astype(F32))
    gp = O.bf16_round(rng.uniform(-1, 1, (period, cout, ho, wo)).astype(F32))
    wt = O.bf16_round(rng.uniform(-0.06, 0.06, (cout, cin, 3, 3)).astype(F32))
    b = O.bf16_round(rng.uniform(-0.5, 0.5, (cout,)).astype(F32))
    W, B = dev.from_ndarray(wt, nk.BF16), dev.from_ndarray(b, nk.BF16)

    def tiled(pool, n):
        """(n, ...) device tensor whose sample s is pool[s % period]: one upload, then doubling device copies"""
        arr = dev.zeros((n,) + pool.shape[1:], nk.BF16)
        per = arr.size // n
        arr.slice_flat(0, pool.shape).copy_from(pool)
        done = period
        while done < n:
            cnt = min(done, n - done)
            nk._lib.check(ops.lib.nk_d2d(dev.ctx, arr.slice_flat(done * per, (cnt * per,)).ptr, arr.ptr, cnt * per * 2),
                          dev.ctx)
            done += cnt
        return arr

    N = 8192
    X, G = tiled(xp, N), tiled(gp, N)
    sub = lambda a, lo, hi: a.slice_flat(lo * (a.size // a.shape[0]), (hi - lo,) + a.shape[1:])
    w64 = wt.astype(np.float64)

    def launches(fn):
        before = dev.launches
        fn()
        return dev.launches - before

    # forward: 2 chunks (7281 + 911); 2 launches per chunk (im2col, batched GEMM)
    Y = dev.zeros((N, cout, ho, wo), nk.BF16)
    Y16 = dev.zeros((16, cout, ho, wo), nk.BF16)
    extra = launches(lambda: ops.conv2d(X, W, bias=B, out=Y)) - launches(lambda: ops.conv2d(sub(X, 0, 16), W, bias=B, out=Y16))
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_fwd"
    assert extra == 1 * 2
    for s in (0, 3639, 3640, 7279, 7280, 7281, 8191):
        want = O.conv_forward(xp[s % period][None].astype(np.float64), w64, (1, 1), (1, 1)).astype(np.float64) \
            + b[None, :, None, None]
        check(sub(Y, s, s + 1).as_ndarray(), want, want, True, False, ("y", s))
    del Y, Y16

    # dX: 3 chunks (3640 + 3640 + 912) at N = 8192, 2 (3640 + 456) at config 5's N = 4096; 2 launches per chunk (batched
    # GEMM, col2im).  The buffer starts non-zero, so a chunk that is never written shows.
    def dx_want(s):
        gx = np.zeros((1, cin, hh, ww_), np.float64)
        O.conv_backward_input(gx, gp[s % period][None].astype(np.float64), w64, (1, 1), (1, 1))
        return gx

    DX = dev.full((N, cin, hh, ww_), 1.0, nk.BF16)
    DX16 = dev.zeros((16, cin, hh, ww_), nk.BF16)
    base = launches(lambda: ops.conv2d_bwd_input(DX16, sub(G, 0, 16), W, beta=0.0))
    extra = launches(lambda: ops.conv2d_bwd_input(DX, G, W, beta=0.0)) - base
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
    assert extra == 2 * 2
    for s in (0, 3639, 3640, 7279, 7280, 8191):
        gx = dx_want(s)
        check(sub(DX, s, s + 1).as_ndarray(), gx, gx, True, False, ("dx", s))
    DX.fill_(1.0)
    extra = launches(lambda: ops.conv2d_bwd_input(sub(DX, 0, 4096), sub(G, 0, 4096), W, beta=0.0)) - base
    assert extra == 1 * 2
    for s in (0, 3639, 3640, 4095):
        gx = dx_want(s)
        check(sub(DX, s, s + 1).as_ndarray(), gx, gx, True, False, ("dx, N = 4096", s))
    assert np.array_equal(sub(DX, 4096, 4097).as_ndarray(), np.ones((1, cin, hh, ww_), F32))
    del DX, DX16

    # dW: 2 chunks (7281 + 911); 2 launches per chunk (im2col, batched GEMM)
    dw_all, dw16 = dev.zeros(wt.shape, nk.F32), dev.zeros(wt.shape, nk.F32)
    extra = launches(lambda: ops.conv2d_bwd_kernel(dw_all, G, X, beta=0.0)) - \
        launches(lambda: ops.conv2d_bwd_kernel(dw16, sub(G, 0, 16), sub(X, 0, 16), beta=0.0))
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dw"
    assert extra == 1 * 2
    parts = []
    for lo, hi in ((0, 4), (0, N // 2), (N // 2, N)):
        d = dev.zeros(wt.shape, nk.F32)
        ops.conv2d_bwd_kernel(d, sub(G, lo, hi), sub(X, lo, hi), beta=0.0)
        parts.append(d.as_ndarray().astype(np.float64))
    gw = np.zeros(wt.shape, np.float64)
    O.conv_backward_kernel(gw, gp[:4].astype(np.float64), xp[:4].astype(np.float64), (1, 1), (1, 1))
    check(parts[0], gw, gw, False, False, "dw, 4 samples")
    total = parts[1] + parts[2]
    got = dw_all.as_ndarray().astype(np.float64)
    assert np.all(np.abs(got - total) <= 1e-4 * np.abs(total) + 1e-3 * float(np.abs(total).mean()))   # f32 atomics
    # the library's memory pool keeps what it has reserved, so its growth over the test bounds the test's peak from below
    print(f"device memory reserved by the chunking test: {(in_use() - used0) / 2 ** 30:.2f} GiB")
