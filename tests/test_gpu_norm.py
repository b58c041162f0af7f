"""Batch norm and layer norm on the H100 (csrc/nk_norm.cu) against the float64 oracle of tests/norm_oracle.py: every
dtype pairing of x, g, dx, dw and db; the (N, C) row layout, short and odd planes, a base one element off alignment and
config 5's map; 2^25 elements per channel and a bf16 input of more than 2^31 elements; a constant channel and
x = 1000 + U(-1, 1); layer-norm rows on both sides of the warp / CTA threshold and
more rows than one pass of the row kernels' grid; launch counts; bitwise repeatability;
the modules against torch's CUDA autograd; a captured Conv2d -> BatchNorm2d -> ReLU -> MaxPool2d -> Linear SGD step.

Bounds: an f32 y within 2e-5 (1 + |y64|); a bf16 y equal to y64 rounded to bf16 or one of its two neighbours, or, where
(x - mean) * rstd * w and b cancel, within the f32 bound plus one bf16 step of y64 (the f32 value it is rounded from
carries the f32 error, which near zero spans many bf16 steps); a gradient within 1e-4 max|grad64|, plus its own bf16
rounding, at most 2^-8 |value|, when it is stored in bf16."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import norm_oracle as O

pytestmark = pytest.mark.gpu

F32N = np.float32
DT = ("f32", "bf16")


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


def dt(nk, name):
    return nk.BF16 if name == "bf16" else nk.F32


def rnd(a, name):
    a = np.asarray(a, F32N)
    return O.bf16_round(a) if name == "bf16" else a


def put(nk, dev, a, name, offset=0):
    """a device copy of `a` in dtype `name`; offset > 0 places it that many elements after a 16-byte aligned base"""
    if offset == 0:
        return dev.from_ndarray(np.ascontiguousarray(a, F32N), dt(nk, name))
    base = dev.zeros((a.size + offset,), dt(nk, name))
    view = base.slice_flat(offset, a.shape)
    view.copy_from(np.ascontiguousarray(a, F32N))
    return view


def check_y(got, want, name, extra=0.0):
    want = np.asarray(want, np.float64)
    if name == "f32":
        err = np.abs(got.astype(np.float64) - want)
        bound = 2e-5 * (1 + np.abs(want)) + extra
        assert np.all(err <= bound), float(np.max(err - bound))
        return
    # bf16: y64 rounded to bf16, or a neighbour (in the order of the bf16 values)
    def order(a):
        u = (np.ascontiguousarray(a, F32N).view(np.uint32) >> 16).astype(np.int64)
        return np.where(u & 0x8000, -(u & 0x7FFF), u)
    d = np.abs(order(got) - order(O.bf16_round(want.astype(F32N))))
    near = np.abs(got.astype(np.float64) - want) <= 2e-5 * (1 + np.abs(want)) + 2.0 ** -8 * np.abs(want) + extra
    assert np.all((d <= 1) | near), int(np.max(np.where(near, 0, d)))


def check_grad(got, want, name, what=""):
    want = np.asarray(want, np.float64)
    bound = 1e-4 * max(float(np.max(np.abs(want), initial=0.0)), 1e-30)
    if name == "bf16":
        bound = bound + 2.0 ** -8 * np.abs(want)
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= bound), (what, float(np.max(err - bound)))


# ---- batch norm entry points against the oracle
def bn_case(nk, dev, shape, xd="f32", gd="f32", dxd="f32", dwd="f32", dbd="f32", training=True, affine=True,
            track=True, beta=0.0, offset=0, seed=0, x=None, extra=0.0):
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    c = shape[1]
    x = rnd(rng.standard_normal(shape) * 2 + 0.5 if x is None else x, xd)
    g = rnd(rng.standard_normal(shape), gd)
    w = rnd(rng.uniform(0.5, 1.5, c), xd) if affine else None
    b = rnd(rng.standard_normal(c), xd) if affine else None
    rm0, rv0 = (rng.standard_normal(c).astype(F32N), rng.uniform(0.5, 2, c).astype(F32N)) if track else (None, None)
    X = put(nk, dev, x, xd, offset)
    W, B = (put(nk, dev, w, xd), put(nk, dev, b, xd)) if affine else (None, None)
    RM, RV = (dev.from_ndarray(rm0), dev.from_ndarray(rv0)) if track else (None, None)
    before = dev.launches
    Y, SM, SR = ops.batch_norm(X, W, B, RM, RV, training, 0.1, 1e-5)
    fwd_launches = dev.launches - before
    y, mean, rstd, rm, rv, batch = O.bn_forward(x, w, b, rm0, rv0, training, 0.1, 1e-5)
    check_y(Y.as_ndarray(), y, xd, extra)
    np.testing.assert_allclose(SM.as_ndarray(), mean, rtol=2e-6, atol=2e-6 * (1 + np.abs(mean)).max())
    np.testing.assert_allclose(SR.as_ndarray(), rstd, rtol=1e-5)
    if track:
        np.testing.assert_allclose(RM.as_ndarray(), rm, rtol=2e-6, atol=1e-6)
        np.testing.assert_allclose(RV.as_ndarray(), rv, rtol=1e-5, atol=1e-6)
    init = {k: rng.standard_normal(s).astype(F32N) for k, s in (("dx", shape), ("dw", (c,)), ("db", (c,)))}
    DX = put(nk, dev, rnd(init["dx"], dxd), dxd)
    DW, DB = (put(nk, dev, rnd(init["dw"], dwd), dwd), put(nk, dev, rnd(init["db"], dbd), dbd)) if affine else (None, None)
    G = put(nk, dev, g, gd)
    before = dev.launches
    ops.batch_norm_bwd(G, X, SM, SR, W, DX, DW, DB, batch, beta)
    bwd_launches = dev.launches - before
    # the kernel's own saved statistics feed the oracle's backward, as they feed the kernels
    dx, dw, db = O.bn_backward(g, x, SM.as_ndarray().astype(np.float64), SR.as_ndarray().astype(np.float64), w, batch)
    check_grad(DX.as_ndarray(), beta * rnd(init["dx"], dxd) + dx, dxd, "dx")
    if affine:
        check_grad(DW.as_ndarray(), beta * rnd(init["dw"], dwd) + dw, dwd, "dw")
        check_grad(DB.as_ndarray(), beta * rnd(init["db"], dbd) + db, dbd, "db")
    return fwd_launches, bwd_launches


PAIRS = [(a, b, c, d, e) for a in DT for b in DT for c in DT for d in DT for e in DT]


@pytest.mark.parametrize("pair", PAIRS, ids=["-".join(p) for p in PAIRS])
def test_batch_norm_every_dtype_pairing(nk, dev, pair):
    xd, gd, dxd, dwd, dbd = pair
    bn_case(nk, dev, (6, 5, 24), xd, gd, dxd, dwd, dbd, beta=0.5, seed=len(PAIRS))
    bn_case(nk, dev, (33, 16), xd, gd, dxd, dwd, dbd, seed=1)


SHAPES = [(40, 13), (24, 16), (9, 4, 1), (9, 4, 3), (9, 4, 7), (5, 6, 7, 7), (3, 4, 2, 4, 8), (64, 32, 32, 32)]


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
def test_batch_norm_layouts_and_alignment(nk, dev, shape, offset):
    for training, track in ((True, True), (False, True), (False, False)):
        f, b = bn_case(nk, dev, shape, "bf16", "bf16", "f32", "f32", "f32", training, track=track, offset=offset,
                       seed=offset)
        assert f == (3 if training or not track else 1)
        assert b == 3
    bn_case(nk, dev, shape, "f32", "f32", "bf16", "bf16", "f32", affine=False, offset=offset, seed=2)


def test_batch_norm_launches_without_dx(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(4)
    X = dev.from_ndarray(rng.standard_normal((8, 3, 16)).astype(F32N))
    W = dev.from_ndarray(np.ones(3, F32N))
    Y, SM, SR = ops.batch_norm(X, W, None, None, None, True)
    DW, DB, DX = dev.zeros((3,), nk.F32), dev.zeros((3,), nk.F32), dev.zeros((8, 3, 16), nk.F32)
    for dx, batch, want in ((None, True, 2), (DX, False, 1), (None, False, 2)):
        before = dev.launches
        ops.batch_norm_bwd(X, X, SM, SR, W, dx, DW if dx is None else None, DB if dx is None else None, batch)
        assert dev.launches - before == want


def test_batch_norm_large_channel_counts(nk, dev):
    """2^25 elements per channel, f32: statistics, y and the gradients against torch in float64"""
    from neuronika_b200 import ops
    shape = (8192, 2, 64, 64)
    gen = torch.Generator(device="cuda").manual_seed(3)
    xt = torch.randn(shape, generator=gen, device="cuda") * 2 + 3
    gt = torch.randn(shape, generator=gen, device="cuda")
    torch.cuda.synchronize()
    X = nk.CuArray(dev, shape, nk.F32, ptr=xt.data_ptr(), owner=xt)
    G = nk.CuArray(dev, shape, nk.F32, ptr=gt.data_ptr(), owner=gt)
    RM, RV = dev.zeros((2,), nk.F32), dev.full((2,), 1.0, nk.F32)
    Y, SM, SR = ops.batch_norm(X, None, None, RM, RV, True, 0.5)
    DX, DW, DB = dev.zeros(shape, nk.F32), dev.zeros((2,), nk.F32), dev.zeros((2,), nk.F32)
    ones = dev.from_ndarray(np.ones(2, F32N))
    ops.batch_norm_bwd(G, X, SM, SR, ones, DX, DW, DB, True)
    dev.synchronize()
    x64 = xt.double()
    var, mean = torch.var_mean(x64, dim=(0, 2, 3), unbiased=False)
    m = shape[0] * 64 * 64
    np.testing.assert_allclose(SM.as_ndarray(), mean.cpu().numpy(), rtol=1e-6)
    np.testing.assert_allclose(SR.as_ndarray(), (1 / torch.sqrt(var + 1e-5)).cpu().numpy(), rtol=1e-6)
    np.testing.assert_allclose(RV.as_ndarray(), (0.5 + 0.5 * var * m / (m - 1)).cpu().numpy(), rtol=1e-6)
    rstd = 1 / torch.sqrt(var + 1e-5)
    xhat = (x64 - mean[None, :, None, None]) * rstd[None, :, None, None]
    del x64
    yd = torch.from_numpy(Y.as_ndarray()).cuda().double()
    assert float(((yd - xhat).abs() - 2e-5 * (1 + xhat.abs())).max()) <= 0
    del yd
    g64 = gt.double()
    sg, sgx = g64.sum(dim=(0, 2, 3)), (g64 * xhat).sum(dim=(0, 2, 3))
    check_grad(DB.as_ndarray(), sg.cpu().numpy(), "f32", "db")
    check_grad(DW.as_ndarray(), sgx.cpu().numpy(), "f32", "dw")
    dx = rstd[None, :, None, None] * (g64 - (sg / m)[None, :, None, None] - xhat * (sgx / m)[None, :, None, None])
    got = torch.from_numpy(DX.as_ndarray()).cuda().double()
    assert float((got - dx).abs().max()) <= 1e-4 * float(dx.abs().max())


def test_batch_norm_more_than_2_to_the_31_elements(nk, dev):
    """a bf16 (8193, 2, 512, 256) input, 2^31 + 2^18 elements: the statistics against float64 sums, y on the last
    planes (offsets past 2^31 elements)"""
    from neuronika_b200 import ops
    shape = (8193, 2, 512, 256)
    assert np.prod(shape) > 2 ** 31
    gen = torch.Generator(device="cuda").manual_seed(5)
    xt = torch.randn(shape, generator=gen, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    X = nk.CuArray(dev, shape, nk.BF16, ptr=xt.data_ptr(), owner=xt)
    Y, SM, SR = ops.batch_norm(X, None, None, None, None, True)
    dev.synchronize()
    s1 = torch.zeros(2, dtype=torch.float64, device="cuda")
    for i in range(0, shape[0], 1024):
        s1 += xt[i:i + 1024].double().sum(dim=(0, 2, 3))
    m = shape[0] * 512 * 256
    mean = s1 / m
    s2 = torch.zeros(2, dtype=torch.float64, device="cuda")
    for i in range(0, shape[0], 1024):
        s2 += ((xt[i:i + 1024].double() - mean[None, :, None, None]) ** 2).sum(dim=(0, 2, 3))
    rstd = 1 / torch.sqrt(s2 / m + 1e-5)
    np.testing.assert_allclose(SM.as_ndarray(), mean.cpu().numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(SR.as_ndarray(), rstd.cpu().numpy(), rtol=1e-5)
    tail = xt[-2:].float().cpu().numpy()
    want = (tail - SM.as_ndarray()[None, :, None, None].astype(np.float64)) * SR.as_ndarray()[None, :, None, None]
    plane = 2 * 512 * 256
    got = Y.slice_flat((shape[0] - 2) * plane, (2, 2, 512, 256)).as_ndarray()
    check_y(got, want, "bf16")
    del xt


def test_batch_norm_hard_inputs(nk, dev):
    """a constant channel (var = 0: y = b exactly) and x = 1000 + U(-1, 1)"""
    rng = np.random.default_rng(9)
    x = rng.standard_normal((16, 3, 40)).astype(F32N)
    x[:, 1] = 2.5
    bn_case(nk, dev, x.shape, x=x, seed=9)
    x = (1000 + rng.uniform(-1, 1, (64, 4, 50))).astype(F32N)
    # save_mean is f32: its rounding, up to ulp(1000)/2 = 2^-15, reaches y as w * rstd * 2^-15 (rstd ~ 1.7, w <= 1.5)
    bn_case(nk, dev, x.shape, x=x, seed=10, extra=1.5 * 1.8 * 2.0 ** -15)


def test_batch_norm_bitwise_repeatable(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(12)
    shape = (256, 8, 28, 28)
    X = dev.from_ndarray(rng.standard_normal(shape).astype(F32N), nk.BF16)
    G = dev.from_ndarray(rng.standard_normal(shape).astype(F32N), nk.BF16)
    W, B = dev.from_ndarray(np.ones(8, F32N), nk.BF16), dev.from_ndarray(np.zeros(8, F32N), nk.BF16)
    outs = []
    for _ in range(2):
        RM, RV = dev.zeros((8,), nk.F32), dev.full((8,), 1.0, nk.F32)
        Y, SM, SR = ops.batch_norm(X, W, B, RM, RV, True)
        DX, DW, DB = dev.zeros(shape, nk.F32), dev.zeros((8,), nk.F32), dev.zeros((8,), nk.F32)
        ops.batch_norm_bwd(G, X, SM, SR, W, DX, DW, DB, True)
        outs.append([a.as_ndarray().view(np.uint8).copy() for a in (Y, SM, SR, RM, RV, DX, DW, DB)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_batch_norm_empty_batch_and_one_value(nk, dev):
    from neuronika_b200 import ops
    RM, RV = dev.from_ndarray(np.array([0.5, -1.0], F32N)), dev.from_ndarray(np.array([2.0, 3.0], F32N))
    before = dev.launches
    ops.batch_norm(dev.zeros((0, 2, 5), nk.F32), None, None, RM, RV, True)
    assert dev.launches == before
    np.testing.assert_array_equal(RM.as_ndarray(), [0.5, -1.0])
    with pytest.raises(nk.NkError, match="Expected more than 1 value per channel when training"):
        ops.batch_norm(dev.zeros((1, 2), nk.F32), None, None, RM, RV, True)
    Y, _, _ = ops.batch_norm(dev.from_ndarray(np.array([[1.0, 2.0]], F32N)), None, None, RM, RV, False)
    np.testing.assert_allclose(Y.as_ndarray(), [[0.5 / np.sqrt(2 + 1e-5), 3.0 / np.sqrt(3 + 1e-5)]], rtol=1e-6)


# ---- layer norm
def ln_case(nk, dev, shape, cols, xd="f32", gd="f32", dxd="f32", dwd="f32", dbd="f32", affine=True, bias=True,
            beta=0.0, seed=0, offset=0):
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ns = (cols,)
    x = rnd(rng.standard_normal(shape) * 2 + 1, xd)
    g = rnd(rng.standard_normal(shape), gd)
    w = rnd(rng.uniform(0.5, 1.5, ns), xd) if affine else None
    b = rnd(rng.standard_normal(ns), xd) if affine and bias else None
    X = put(nk, dev, x, xd, offset)
    W = put(nk, dev, w, xd) if w is not None else None
    B = put(nk, dev, b, xd) if b is not None else None
    before = dev.launches
    Y, SM, SR = ops.layer_norm(X, cols, W, B)
    assert dev.launches - before == (1 if x.size else 0)
    y, mean, rstd = O.ln_forward(x, ns, w, b)
    check_y(Y.as_ndarray(), y, xd)
    d0 = rng.standard_normal(shape).astype(F32N)
    DX = put(nk, dev, rnd(d0, dxd), dxd)
    DW = dev.zeros(ns, dt(nk, dwd)) if w is not None else None
    DB = dev.zeros(ns, dt(nk, dbd)) if b is not None else None
    before = dev.launches
    ops.layer_norm_bwd(put(nk, dev, g, gd), X, cols, SM, SR, W, DX, DW, DB, beta, 0.0, 0.0)
    assert dev.launches - before <= 2
    dx, dw, db = O.ln_backward(g, x, ns, SM.as_ndarray().astype(np.float64), SR.as_ndarray().astype(np.float64), w)
    check_grad(DX.as_ndarray(), beta * rnd(d0, dxd) + dx, dxd, "dx")
    if w is not None:
        check_grad(DW.as_ndarray(), dw, dwd, "dw")
    if b is not None:
        check_grad(DB.as_ndarray(), db, dbd, "db")


@pytest.mark.parametrize("pair", PAIRS, ids=["-".join(p) for p in PAIRS])
def test_layer_norm_every_dtype_pairing(nk, dev, pair):
    ln_case(nk, dev, (37, 64), 64, *pair, beta=0.5, seed=3)
    ln_case(nk, dev, (5, 4096), 4096, *pair, seed=4)


COLS = [1, 7, 8, 1023, 1024, 4096, 65536, 2 ** 20]


def ln_case_device(nk, dev, rows, cols, xd, seed, block=1024):
    """ln_case for inputs too large for a host oracle: data made on the device, every output a torch tensor, and the
    float64 reference computed on the device one block of rows at a time, with ln_case's bounds (dx, dw, db in f32)"""
    from neuronika_b200 import ops
    tdt = torch.bfloat16 if xd == "bf16" else torch.float32
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn((rows, cols), generator=gen, device="cuda") * 2 + 1).to(tdt)
    g = torch.randn((rows, cols), generator=gen, device="cuda")
    w = (torch.rand(cols, generator=gen, device="cuda") + 0.5).to(tdt)
    b = torch.randn(cols, generator=gen, device="cuda").to(tdt)
    y = torch.empty((rows, cols), device="cuda", dtype=tdt)
    dx = torch.empty((rows, cols), device="cuda")
    sm, sr, dw, db = (torch.empty(n, device="cuda") for n in (rows, rows, cols, cols))
    torch.cuda.synchronize()
    wrap = lambda t: nk.CuArray(dev, tuple(t.shape), nk.BF16 if t.dtype == torch.bfloat16 else nk.F32,
                                ptr=t.data_ptr(), owner=t)
    X, G, W, B, Y, DX, SM, SR, DW, DB = (wrap(t) for t in (x, g, w, b, y, dx, sm, sr, dw, db))
    ops.layer_norm(X, cols, W, B, out=Y, save_mean=SM, save_rstd=SR)
    ops.layer_norm_bwd(G, X, cols, SM, SR, W, DX, DW, DB)
    dev.synchronize()
    w64, b64 = w.double(), b.double()
    dw64 = torch.zeros(cols, dtype=torch.float64, device="cuda")
    db64 = torch.zeros(cols, dtype=torch.float64, device="cuda")
    dx_err, dx_max = 0.0, 0.0
    for r0 in range(0, rows, block):
        xb, gb = x[r0:r0 + block].double(), g[r0:r0 + block].double()
        mean = xb.mean(dim=1, keepdim=True)
        want = (xb - mean) / torch.sqrt(((xb - mean) ** 2).mean(dim=1, keepdim=True) + 1e-5) * w64 + b64
        got = y[r0:r0 + block]
        if xd == "f32":
            assert bool(((got.double() - want).abs() <= 2e-5 * (1 + want.abs())).all()), r0
        else:   # as check_y: y64 rounded to bf16 or a neighbour, or the f32 bound plus one bf16 step
            order = lambda t: (lambda u: torch.where(u < 0, -(u & 0x7FFF), u))(t.view(torch.int16).long())
            d = (order(got) - order(want.float().bfloat16())).abs()
            near = (got.double() - want).abs() <= 2e-5 * (1 + want.abs()) + 2.0 ** -8 * want.abs()
            assert bool(((d <= 1) | near).all()), r0
        # the backward from the kernel's saved statistics, as they feed the kernels
        xhat = (xb - sm[r0:r0 + block, None].double()) * sr[r0:r0 + block, None].double()
        gw = gb * w64
        want = sr[r0:r0 + block, None].double() * (gw - gw.mean(dim=1, keepdim=True)
                                                   - xhat * (gw * xhat).mean(dim=1, keepdim=True))
        dx_err = max(dx_err, float((dx[r0:r0 + block].double() - want).abs().max()))
        dx_max = max(dx_max, float(want.abs().max()))
        dw64 += (gb * xhat).sum(dim=0)
        db64 += gb.sum(dim=0)
        del xb, gb, want, got, xhat, gw
    assert dx_err <= 1e-4 * dx_max, (dx_err, dx_max)
    for got, want in ((dw, dw64), (db, db64)):
        assert float((got.double() - want).abs().max()) <= 1e-4 * float(want.abs().max())
    del x, g, y, dx


@pytest.mark.parametrize("rows", [1, 3, 8192])
@pytest.mark.parametrize("cols", COLS)
def test_layer_norm_rows_and_columns(nk, dev, rows, cols):
    if rows * cols > 2 ** 31:
        pytest.skip("%d x %d is 2^33 elements: x, g, y and dx alone take 128 GB in f32 and 64 GB in bf16, more than "
                    "this 80 GB card holds beside a float64 reference" % (rows, cols))
    if rows * cols > 2 ** 24:   # the float64 reference on the device
        ln_case_device(nk, dev, rows, cols, "bf16", seed=cols)
        ln_case_device(nk, dev, rows, cols, "f32", seed=cols + 1)
        torch.cuda.empty_cache()
        return
    ln_case(nk, dev, (rows, cols), cols, "bf16", "f32", "f32", "f32", "f32", seed=cols)
    ln_case(nk, dev, (rows, cols), cols, "f32", "f32", "f32", "f32", "f32", seed=cols, offset=1 if cols > 1 else 0)


@pytest.mark.parametrize("cols", [256, 1024, 8192])
def test_layer_norm_more_rows_than_one_grid_pass(nk, dev, cols):
    """more rows than the row kernels' grid covers in one pass (16 CTAs per SM; 8 rows per CTA on the warp path, one on
    the CTA path), so each thread group loops over several rows, the CTA path's barriers included: 256 and 1024
    columns take the warp path in bf16, 8192 the CTA path"""
    rows_per_pass = 16 * dev.sm_count * (8 if cols * 2 <= 4096 else 1)
    rows = 2 * rows_per_pass + 37
    ln_case_device(nk, dev, rows, cols, "bf16", seed=cols + 2)
    ln_case_device(nk, dev, rows, cols, "f32", seed=cols + 3)
    torch.cuda.empty_cache()


def test_layer_norm_multi_dim_and_lstm_output(nk, dev):
    rng = np.random.default_rng(21)
    x = rng.standard_normal((4, 3, 5, 6)).astype(F32N)
    w = rng.standard_normal((3, 5, 6)).astype(F32N)
    X = nk.from_ndarray(dev, x).requires_grad()
    Wv = nk.from_ndarray(dev, w).requires_grad()
    Y = X.layer_norm((3, 5, 6), Wv)
    loss = Y.sum()
    loss.forward()
    loss.backward(1.0)
    xt, wt = torch.tensor(x, requires_grad=True), torch.tensor(w, requires_grad=True)
    yt = F.layer_norm(xt, (3, 5, 6), wt)
    yt.sum().backward()
    np.testing.assert_allclose(Y.data(), yt.detach().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(X.grad(), xt.grad.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(Wv.grad(), wt.grad.numpy(), rtol=1e-4, atol=1e-5)
    # (H,) over an LSTM's (T, N, H) output
    lstm = nk.nn.LSTM(dev, 6, 16, rng=rng)
    ln = nk.nn.LayerNorm(dev, 16)
    xs = nk.from_ndarray(dev, rng.standard_normal((5, 3, 6)).astype(F32N))
    out = lstm.forward((nk.zeros(dev, (3, 16)), nk.zeros(dev, (3, 16))), xs)[0]
    z = ln.forward(out)
    z.forward()
    np.testing.assert_allclose(z.data(), F.layer_norm(torch.tensor(out.data()), (16,)).numpy(), rtol=1e-5, atol=1e-5)
    with pytest.raises(nk.NkError, match=r"Given normalized_shape=\[5\], expected input with shape \[\*, 5\]"):
        X.layer_norm(5)


def test_layer_norm_bitwise_repeatable(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(13)
    for cols in (768, 4096):
        X = dev.from_ndarray(rng.standard_normal((512, cols)).astype(F32N), nk.BF16)
        W, B = dev.from_ndarray(np.ones(cols, F32N), nk.BF16), dev.from_ndarray(np.zeros(cols, F32N), nk.BF16)
        outs = []
        for _ in range(2):
            Y, SM, SR = ops.layer_norm(X, cols, W, B)
            DX, DW, DB = dev.zeros((512, cols), nk.F32), dev.zeros((cols,), nk.F32), dev.zeros((cols,), nk.F32)
            ops.layer_norm_bwd(X, X, cols, SM, SR, W, DX, DW, DB)
            outs.append([a.as_ndarray().view(np.uint8).copy() for a in (Y, SM, SR, DX, DW, DB)])
        for a, b in zip(*outs):
            assert np.array_equal(a, b)


# ---- modules against torch's CUDA autograd
MODULES = [("BatchNorm1d", (16, 6)), ("BatchNorm1d", (8, 6, 10)), ("BatchNorm2d", (4, 6, 7, 9)),
           ("BatchNorm3d", (2, 6, 3, 4, 5))]


@pytest.mark.parametrize("affine,track", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("m", range(len(MODULES)))
def test_batch_norm_modules_against_torch(nk, dev, m, affine, track):
    name, shape = MODULES[m]
    rng = np.random.default_rng(m)
    layer = getattr(nk.nn, name)(dev, 6, momentum=0.2, affine=affine, track_running_stats=track)
    ref = getattr(torch.nn, name)(6, momentum=0.2, affine=affine, track_running_stats=track).cuda()
    assert len(layer.parameters()) == (2 if affine else 0)
    for step in range(3):
        if step == 2:
            layer.eval()
            ref.eval()
        x = rng.standard_normal(shape).astype(F32N) + step
        g = rng.standard_normal(shape).astype(F32N)
        X = nk.from_ndarray(dev, x).requires_grad()
        Y = layer.forward(X)
        loss = (Y * nk.from_ndarray(dev, g)).sum()
        loss.forward()
        loss.backward(1.0)
        xt = torch.tensor(x, device="cuda", requires_grad=True)
        if affine:
            ref.weight.grad = ref.bias.grad = None
        ref(xt).backward(torch.tensor(g, device="cuda"))
        np.testing.assert_allclose(Y.data(), ref(xt.detach()).detach().cpu().numpy() if step == 2 else
                                   F.batch_norm(torch.tensor(x, device="cuda"), None, None, ref.weight, ref.bias, True
                                                ).detach().cpu().numpy(), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(X.grad(), xt.grad.cpu().numpy(), rtol=1e-4, atol=1e-4)
        if affine:
            np.testing.assert_allclose(layer.weight.grad(), ref.weight.grad.cpu().numpy(), rtol=1e-4, atol=1e-4)
            np.testing.assert_allclose(layer.bias.grad(), ref.bias.grad.cpu().numpy(), rtol=1e-4, atol=1e-4)
        if track:
            np.testing.assert_allclose(layer.running_mean.data(), ref.running_mean.cpu().numpy(), rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(layer.running_var.data(), ref.running_var.cpu().numpy(), rtol=1e-5, atol=1e-6)
        for p in layer.parameters():
            p.zero_grad()
    with pytest.raises(ValueError, match="expected"):
        layer.forward(nk.zeros(dev, (2, 6, 3, 4, 5, 6)))


def test_layer_norm_module_options(nk, dev):
    rng = np.random.default_rng(31)
    for affine, bias in ((True, True), (True, False), (False, True)):
        layer = nk.nn.LayerNorm(dev, (4, 8), eps=1e-3, elementwise_affine=affine, bias=bias)
        ref = torch.nn.LayerNorm((4, 8), eps=1e-3, elementwise_affine=affine, bias=bias).cuda()
        assert len(layer.parameters()) == len(list(ref.parameters()))
        x = rng.standard_normal((3, 4, 8)).astype(F32N)
        X = nk.from_ndarray(dev, x).requires_grad()
        Y = layer.forward(X)
        loss = Y.sum()
        loss.forward()
        loss.backward(1.0)
        xt = torch.tensor(x, device="cuda", requires_grad=True)
        ref(xt).sum().backward()
        np.testing.assert_allclose(X.grad(), xt.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)
        for p, q in zip(layer.parameters(), ref.parameters()):
            np.testing.assert_allclose(p.grad(), q.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)


def test_captured_training_step_with_batch_norm(nk, dev):
    """Conv2d -> BatchNorm2d -> ReLU -> MaxPool2d(2) -> flatten -> Linear -> mse, SGD, f32 IEEE convolutions, captured
    once and replayed 5 times: every replay advances the running statistics, and both they and the parameters follow
    torch's 5 steps"""
    rng = np.random.default_rng(17)
    N, Cin, H, C = 8, 3, 12, 6
    conv = nk.nn.Conv2d(dev, Cin, C, (3, 3), padding=(1, 1), rng=rng)
    bn = nk.nn.BatchNorm2d(dev, C)
    fc = nk.nn.Linear(dev, C * (H // 2) ** 2, 4, rng=rng)
    pool = nk.nn.MaxPool2d(2)
    params = conv.parameters() + bn.parameters() + fc.parameters()
    init = [p.data().copy() for p in params]
    x = rng.standard_normal((N, Cin, H, H)).astype(F32N)
    t = rng.standard_normal((N, 4)).astype(F32N)
    X, T = nk.from_ndarray(dev, x), nk.from_ndarray(dev, t)
    lr = 0.05
    opt = nk.optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)
    dev.f32_conv("ieee")

    def step():
        opt.zero_grad()
        h = pool.forward(bn.forward(conv.forward(X)).relu()).flatten()
        loss = fc.forward(h).mse_loss(T)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    step()                          # warm-up: first-use allocations cannot be captured
    for p, v in zip(params, init):
        p.set_data(v)
    bn.running_mean.set_data(np.zeros(C, F32N))
    bn.running_var.set_data(np.ones(C, F32N))
    dev.synchronize()
    with dev.capture(256 << 20) as cap:
        step()
    # torch, the same model and steps
    w1, b1, g1, be1, wf, bf = [torch.tensor(v.reshape(v.shape), requires_grad=True) for v in init]
    rm, rv = torch.zeros(C), torch.ones(C)
    for r in range(5):
        cap.graph.launch()
        dev.synchronize()
        h = F.conv2d(torch.from_numpy(x), w1, padding=1) + b1
        h = F.max_pool2d(F.relu(F.batch_norm(h, rm, rv, g1, be1, True, 0.1, 1e-5)), 2).flatten(1)
        loss = F.mse_loss(h @ wf.T + bf, torch.from_numpy(t))
        for p in (w1, b1, g1, be1, wf, bf):
            p.grad = None
        loss.backward()
        with torch.no_grad():
            for p in (w1, b1, g1, be1, wf, bf):
                p -= lr * p.grad
        np.testing.assert_allclose(bn.running_mean.data(), rm.numpy(), rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(bn.running_var.data(), rv.numpy(), rtol=1e-4, atol=1e-5)
        for p, q in zip(params, (w1, b1, g1, be1, wf, bf)):
            np.testing.assert_allclose(p.data(), q.detach().numpy().reshape(p.data().shape), rtol=1e-4, atol=1e-5)
