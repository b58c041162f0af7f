"""Max, average and adaptive average pooling on the GPU (csrc/nk_pool.cu): every ABI entry point bit-equal to the numpy
oracle of tests/pool_oracle.py (which restates the kernels' summation orders) for f32 and bf16 data, all four (dx, g)
dtype pairs and beta 0 / 1, over 1, 2 and 3 sample dims; last-axis extents at and around the 16-byte vector widths,
bases off 16-byte alignment, empty batches, both sides of the small / large window threshold and an input of more than
2^31 elements; repeated calls bitwise equal; the Var ops and nn modules against torch's CPU autograd; a captured training
step with pooling layers against its eager step and torch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pool_oracle as P

pytestmark = pytest.mark.gpu

F32N = np.float32


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


def put(nk, dev, a, dtype, offset=0):
    """a device copy of `a` in `dtype`; offset > 0 places it that many elements after a 16-byte aligned allocation"""
    if offset == 0:
        return dev.from_ndarray(a, dt(nk, dtype))
    base = dev.zeros((a.size + offset,), dt(nk, dtype))
    view = base.slice_flat(offset, a.shape)
    view.copy_from(a)
    return view


def same(got, want, what):
    """bitwise equal, NaN payloads aside"""
    got, want = np.asarray(got, F32N), np.asarray(want, F32N)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    bad = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    assert not bad.any(), (what, np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])


def data(rng, shape, dtype, special=False):
    x = rng.standard_normal(shape).astype(F32N)
    if special and x.size > 8:
        flat = x.reshape(-1)
        flat[rng.choice(x.size, x.size // 11, replace=False)] = np.inf
        flat[rng.choice(x.size, x.size // 13, replace=False)] = -np.inf
        flat[rng.choice(x.size, x.size // 17, replace=False)] = np.nan
        flat[rng.choice(x.size, x.size // 5, replace=False)] = 1.0           # ties
    return P.round_to(x, dtype)


# name: (kind, sample shape, kernel, stride, padding, dilation, ceil_mode, include_pad / output_size)
CASES = {
    "max1d_k3s2p1": ("max", (37,), (3,), (2,), (1,), (1,), False, None),
    "max1d_dil_ceil": ("max", (29,), (3,), (2,), (1,), (3,), True, None),
    "max2d_k2": ("max", (12, 18), (2, 2), (2, 2), (0, 0), (1, 1), False, None),
    "max2d_k3s2p1_ceil": ("max", (15, 33), (3, 3), (2, 2), (1, 1), (1, 1), True, None),
    "max2d_gaps": ("max", (11, 13), (2, 3), (3, 4), (1, 1), (1, 1), False, None),
    "max3d_k2": ("max", (6, 8, 18), (2, 2, 2), (2, 2, 2), (0, 0, 0), (1, 1, 1), False, None),
    "max3d_mixed": ("max", (5, 7, 9), (3, 2, 3), (1, 2, 2), (1, 1, 1), (1, 2, 1), True, None),
    "max2d_large": ("max", (20, 21), (6, 6), (3, 4), (3, 2), (1, 1), True, None),
    "avg1d_k3s2p1": ("avg", (37,), (3,), (2,), (1,), None, True, True),
    "avg2d_k2": ("avg", (12, 18), (2, 2), (2, 2), (0, 0), None, False, True),
    "avg2d_nopad": ("avg", (15, 33), (3, 3), (2, 2), (1, 1), None, True, False),
    "avg3d_k2": ("avg", (6, 8, 18), (2, 2, 2), (2, 2, 2), (0, 0, 0), None, False, True),
    "avg3d_k3": ("avg", (7, 6, 9), (3, 3, 3), (2, 1, 2), (1, 1, 0), None, True, False),
    "avg2d_large": ("avg", (20, 21), (8, 5), (4, 3), (4, 2), None, False, True),
    "adaptive1d": ("adaptive", (23,), None, None, None, None, False, (7,)),
    "adaptive1d_up": ("adaptive", (5,), None, None, None, None, False, (9,)),
    "adaptive2d": ("adaptive", (13, 10), None, None, None, None, False, (4, 3)),
    "adaptive2d_global": ("adaptive", (7, 7), None, None, None, None, False, (1, 1)),
    "adaptive2d_global_32": ("adaptive", (32, 32), None, None, None, None, False, (1, 1)),
    "adaptive3d": ("adaptive", (6, 5, 9), None, None, None, None, False, (4, 2, 3)),
    "adaptive3d_global": ("adaptive", (4, 6, 5), None, None, None, None, False, (1, 1, 1)),
}


def geometry(case):
    kind, sp, k, s, p, d, ceil, extra = CASES[case]
    if kind == "adaptive":
        return P.Geometry(kind, sp, output_size=extra)
    return P.Geometry(kind, sp, k, s, p, d, ceil, include_pad=bool(extra))


def run_fwd(nk, dev, case, X, geo, with_idx=True):
    """forward through the ABI; returns (y, idx or None)"""
    from neuronika_b200 import ops
    kind, sp, k, s, p, d, ceil, extra = CASES[case]
    if kind == "max":
        idx = dev.zeros(X.shape[:2] + geo.out_sp, nk.F32) if with_idx else None
        y = ops.max_pool_nd(X, k, s, p, d, ceil, idx=idx)
        return y, idx
    if kind == "avg":
        return ops.avg_pool_nd(X, k, s, p, ceil, extra), None
    return ops.adaptive_avg_pool_nd(X, extra), None


def run_bwd(nk, dev, case, DX, G, IDX, beta):
    from neuronika_b200 import ops
    kind, sp, k, s, p, d, ceil, extra = CASES[case]
    if kind == "max":
        return ops.max_pool_nd_bwd(DX, G, IDX, k, s, p, d, beta=beta)
    if kind == "avg":
        return ops.avg_pool_nd_bwd(DX, G, k, s, p, extra, beta=beta)
    return ops.adaptive_avg_pool_nd_bwd(DX, G, beta=beta, nsp=len(sp))


def host_idx(idx):
    return idx.as_ndarray().view(np.int32)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_forward_equals_the_oracle(nk, dev, case, dtype):
    rng = np.random.default_rng(sum(map(ord, case)))
    geo = geometry(case)
    x = data(rng, (2, 3) + geo.in_sp, dtype, special=CASES[case][0] == "max")
    y, idx = run_fwd(nk, dev, case, put(nk, dev, x, dtype), geo)
    want, want_idx, _ = P.forward(x, geo, dtype)
    same(y.as_ndarray(), want, (case, dtype))
    if idx is not None:
        assert np.array_equal(host_idx(idx), want_idx), case
        y2, _ = run_fwd(nk, dev, case, put(nk, dev, x, dtype), geo, with_idx=False)   # idx NULL: same values
        same(y2.as_ndarray(), want, (case, dtype, "no idx"))


@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("dx_dtype,g_dtype", [("f32", "f32"), ("bf16", "bf16"), ("f32", "bf16"), ("bf16", "f32")])
@pytest.mark.parametrize("case", sorted(CASES))
def test_backward_equals_the_oracle(nk, dev, case, dx_dtype, g_dtype, beta):
    rng = np.random.default_rng(7 + sum(map(ord, case)))
    geo = geometry(case)
    x = data(rng, (2, 3) + geo.in_sp, "bf16")
    _, want_idx, _ = P.forward(x, geo, "bf16")
    g = P.round_to(rng.standard_normal((2, 3) + geo.out_sp).astype(F32N), g_dtype)
    dx0 = P.round_to(rng.standard_normal(x.shape).astype(F32N), dx_dtype)
    IDX = None
    if CASES[case][0] == "max":
        _, IDX = run_fwd(nk, dev, case, put(nk, dev, x, "bf16"), geo)
    DX = put(nk, dev, dx0 if beta else np.full(x.shape, np.nan, F32N), dx_dtype)   # beta 0 never reads dx
    run_bwd(nk, dev, case, DX, put(nk, dev, g, g_dtype), IDX, beta)
    want = P.backward(g, geo, want_idx, dx0, beta, dx_dtype)
    same(DX.as_ndarray(), want, (case, dx_dtype, g_dtype, beta))


# last-axis extents at and around the vector widths (8 bf16 / 4 f32 outputs per thread) for the two specialised
# last-axis shapes and the generic path, with the bases 0 and 1..3 elements past 16-byte alignment
EDGE = [("max", (2,), (2,), (0,)), ("max", (3,), (2,), (1,)), ("avg", (3,), (2,), (1,)), ("max", (3,), (1,), (1,)),
        ("avg", (2,), (2,), (0,)), ("avg", (4,), (3,), (2,))]


@pytest.mark.parametrize("offset", [0, 1, 3])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("edge", range(len(EDGE)))
def test_vector_width_edges_and_misaligned_bases(nk, dev, edge, dtype, offset):
    from neuronika_b200 import ops
    kind, k, s, p = EDGE[edge]
    rng = np.random.default_rng(edge * 10 + offset)
    for out2 in (1, 3, 4, 5, 7, 8, 9, 16, 17, 33):
        L = (out2 - 1) * s[0] + k[0] - 2 * p[0]
        if L < 1:
            continue
        sp = (3, L)
        k2, s2, p2 = (2,) + k, (1,) + s, (0,) + p
        geo = P.Geometry(kind, sp, k2, s2, p2, (1, 1), False)
        assert geo.out_sp[1] == out2
        x = data(rng, (2, 2) + sp, dtype)
        X = put(nk, dev, x, dtype, offset)
        g = P.round_to(rng.standard_normal((2, 2) + geo.out_sp).astype(F32N), dtype)
        dx0 = P.round_to(rng.standard_normal(x.shape).astype(F32N), dtype)
        DX = put(nk, dev, dx0, dtype, offset)
        G = put(nk, dev, g, dtype, offset)
        want, want_idx, _ = P.forward(x, geo, dtype)
        if kind == "max":
            idx_base = dev.zeros((int(np.prod(want.shape)) + offset,), nk.F32)
            IDX = idx_base.slice_flat(offset, want.shape)
            y = ops.max_pool_nd(X, k2, s2, p2, (1, 1), idx=IDX)
            assert np.array_equal(host_idx(IDX), want_idx), (edge, out2)
            ops.max_pool_nd_bwd(DX, G, IDX, k2, s2, p2, (1, 1), beta=1.0)
        else:
            y = ops.avg_pool_nd(X, k2, s2, p2)
            ops.avg_pool_nd_bwd(DX, G, k2, s2, p2, beta=1.0)
        same(y.as_ndarray(), want, (edge, dtype, offset, out2))
        same(DX.as_ndarray(), P.backward(g, geo, want_idx, dx0, 1.0, dtype), (edge, dtype, offset, out2, "dx"))


@pytest.mark.parametrize("kernel", [(5, 6), (6, 6), (4, 8), (4, 7)])
def test_both_sides_of_the_large_window_threshold(nk, dev, kernel):
    """windows of 30, 36, 32 and 28 elements: below 32 one thread per output, from 32 on one warp"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(sum(kernel))
    for kind in ("max", "avg"):
        geo = P.Geometry(kind, (19, 23), kernel, (2, 3), (kernel[0] // 2, 1), (1, 1), True)
        assert geo.large == (kernel[0] * kernel[1] >= 32)
        for dtype in ("f32", "bf16"):
            x = data(rng, (3, 2, 19, 23), dtype, special=kind == "max")
            X = put(nk, dev, x, dtype)
            want, want_idx, _ = P.forward(x, geo, dtype)
            if kind == "max":
                IDX = dev.zeros(want.shape, nk.F32)
                y = ops.max_pool_nd(X, kernel, (2, 3), (kernel[0] // 2, 1), (1, 1), True, idx=IDX)
                assert np.array_equal(host_idx(IDX), want_idx)
            else:
                y = ops.avg_pool_nd(X, kernel, (2, 3), (kernel[0] // 2, 1), True)
            same(y.as_ndarray(), want, (kernel, kind, dtype))
    for o, L in (((2, 3), (12, 21)), ((1, 1), (5, 6)), ((1, 1), (6, 6))):   # adaptive: ceil(L/O) products 24, 30, 36
        geo = P.Geometry("adaptive", L, output_size=o)
        x = data(rng, (2, 3) + L, "f32")
        same(ops.adaptive_avg_pool_nd(put(nk, dev, x, "f32"), o).as_ndarray(), P.forward(x, geo, "f32")[0], (o, L))


def test_empty_batch_and_rejected_arguments(nk, dev):
    from neuronika_b200 import ops
    X = dev.zeros((0, 3, 8, 8), nk.F32)
    before = dev.launches
    y = ops.max_pool_nd(X, (2, 2), idx=dev.zeros((1,), nk.F32))
    ops.avg_pool_nd(X, (2, 2))
    ops.adaptive_avg_pool_nd(X, (1, 1))
    ops.avg_pool_nd_bwd(X, dev.zeros((0, 3, 4, 4), nk.F32), (2, 2))
    assert y.shape == (0, 3, 4, 4) and dev.launches == before
    X = dev.zeros((1, 1, 8, 8), nk.F32)
    bad = [lambda: ops.max_pool_nd(X, (3, 3), padding=(2, 0)),        # p > k/2
           lambda: ops.max_pool_nd(X, (0, 2)),                        # k < 1
           lambda: ops.avg_pool_nd(X, (9, 2)),                        # O < 1
           lambda: ops.max_pool_nd(X, (2, 2), out=dev.zeros((1, 1, 5, 4)), out_sp=(5, 4))]   # O is neither extent
    for call in bad:
        with pytest.raises(nk.NkError, match="NK_ERR_INVALID_ARG"):
            call()
    assert dev.launches == before


def test_repeated_calls_are_bitwise_equal(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(3)
    x = data(rng, (4, 8, 33, 35), "bf16")
    X = put(nk, dev, x, "bf16")
    g = rng.standard_normal((4, 8, 17, 18)).astype(F32N)
    outs = []
    for _ in range(2):
        IDX = dev.zeros((4, 8, 17, 18), nk.F32)
        y = ops.max_pool_nd(X, (3, 3), (2, 2), (1, 1), ceil_mode=True, idx=IDX)
        DX = dev.zeros(x.shape, nk.F32)
        ops.max_pool_nd_bwd(DX, put(nk, dev, g, "f32"), IDX, (3, 3), (2, 2), (1, 1), beta=0.0)
        ga = ops.adaptive_avg_pool_nd(X, (1, 1))
        DA = dev.zeros(x.shape, nk.BF16)
        ops.adaptive_avg_pool_nd_bwd(DA, put(nk, dev, g[:, :, :1, :1], "f32"), beta=0.0)
        outs.append([a.as_ndarray().view(np.uint32) for a in (y, IDX, DX, ga, DA)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_more_than_2_to_the_31_elements(nk, dev):
    """a bf16 (1, 32769, 256, 256) input: 2^31 + 2^16 elements, max pool 2x2 forward and backward; the last planes,
    whose offsets pass 2^31 elements, checked against the oracle"""
    from neuronika_b200 import ops
    shape = (1, 32769, 256, 256)
    assert np.prod(shape) > 2 ** 31
    torch.cuda.synchronize()
    gen = torch.Generator(device="cuda").manual_seed(5)
    xt = torch.randn(shape, generator=gen, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    X = nk.CuArray(dev, shape, nk.BF16, ptr=xt.data_ptr(), owner=xt)
    oshape = (1, 32769, 128, 128)
    IDX = dev.zeros(oshape, nk.F32)
    y = ops.max_pool_nd(X, (2, 2), idx=IDX)
    G = dev.full(oshape, 0.5, nk.BF16)
    DX = dev.zeros(shape, nk.BF16)
    ops.max_pool_nd_bwd(DX, G, IDX, (2, 2), beta=0.0)
    dev.synchronize()
    tail = 3
    x = xt[0, -tail:].float().cpu().numpy()[None]
    geo = P.Geometry("max", (256, 256), (2, 2))
    want, want_idx, _ = P.forward(x, geo, "bf16")
    plane = 128 * 128
    first = (32769 - tail) * plane
    same(y.slice_flat(first, (1, tail, 128, 128)).as_ndarray(), want, "y")
    assert np.array_equal(host_idx(IDX.slice_flat(first, (1, tail, 128, 128))), want_idx)
    dx = DX.slice_flat((32769 - tail) * 256 * 256, (1, tail, 256, 256)).as_ndarray()
    same(dx, P.backward(np.full(want.shape, 0.5, F32N), geo, want_idx, None, 0.0, "bf16"), "dx")
    del xt


# ---- graph level: Var ops and nn modules against torch's CPU autograd
def _torch(fn, x, g):
    xt = torch.from_numpy(x.copy()).requires_grad_(True)
    yt = fn(xt)
    yt.backward(torch.from_numpy(g))
    return yt.detach().numpy(), xt.grad.numpy()


MODULES = [
    ("MaxPool1d", (3,), dict(stride=2, padding=1), lambda t: F.max_pool1d(t, 3, 2, 1), (2, 4, 19)),
    ("MaxPool2d", (2,), {}, lambda t: F.max_pool2d(t, 2), (2, 4, 10, 12)),
    ("MaxPool2d", ((3, 2),), dict(stride=(2, 1), padding=(1, 0), dilation=(1, 2), ceil_mode=True),
     lambda t: F.max_pool2d(t, (3, 2), (2, 1), (1, 0), (1, 2), True), (2, 3, 11, 9)),
    ("MaxPool3d", (2,), dict(stride=2), lambda t: F.max_pool3d(t, 2, 2), (1, 3, 6, 8, 10)),
    ("AvgPool1d", (4,), dict(stride=3, padding=2, ceil_mode=True), lambda t: F.avg_pool1d(t, 4, 3, 2, True), (2, 3, 20)),
    ("AvgPool2d", (3,), dict(stride=2, padding=1, count_include_pad=False),
     lambda t: F.avg_pool2d(t, 3, 2, 1, False, False), (2, 3, 9, 11)),
    ("AvgPool3d", (2,), {}, lambda t: F.avg_pool3d(t, 2), (1, 2, 6, 6, 8)),
    ("AdaptiveAvgPool1d", (5,), {}, lambda t: F.adaptive_avg_pool1d(t, 5), (2, 3, 17)),
    ("AdaptiveAvgPool2d", (1,), {}, lambda t: F.adaptive_avg_pool2d(t, 1), (2, 6, 7, 7)),
    ("AdaptiveAvgPool2d", ((3, 4),), {}, lambda t: F.adaptive_avg_pool2d(t, (3, 4)), (2, 3, 8, 9)),
    ("AdaptiveAvgPool3d", (2,), {}, lambda t: F.adaptive_avg_pool3d(t, 2), (1, 2, 5, 6, 7)),
]


@pytest.mark.parametrize("m", range(len(MODULES)))
def test_modules_against_torch_autograd(nk, dev, m):
    name, args, kw, fn, shape = MODULES[m]
    rng = np.random.default_rng(m)
    x = rng.standard_normal(shape).astype(F32N)
    layer = getattr(nk.nn, name)(*args, **kw)
    assert layer.parameters() == []
    X = nk.from_ndarray(dev, x).requires_grad()
    Y = layer.forward(X)
    Y.forward()
    yt, _ = _torch(fn, x, np.zeros(Y.shape, F32N))
    g = rng.standard_normal(yt.shape).astype(F32N)
    loss = (Y * nk.from_ndarray(dev, g)).sum()
    loss.forward()
    loss.backward(1.0)
    yt, gt = _torch(fn, x, g)
    exact = name.startswith("Max")
    tol = 0.0 if exact else 1e-6
    np.testing.assert_allclose(Y.data(), yt, rtol=tol, atol=tol)
    np.testing.assert_allclose(X.grad(), gt, rtol=tol, atol=tol)


def test_var_ops_broadcast_ints_and_need_no_index_for_constants(nk, dev):
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 3, 9, 8)).astype(F32N)
    v = nk.from_ndarray(dev, x)
    y = v.max_pool(3, stride=2, padding=1, ceil_mode=True)
    assert not isinstance(y, nk.VarDiff)
    y.forward()
    np.testing.assert_array_equal(y.data(), F.max_pool2d(torch.from_numpy(x), 3, 2, 1, ceil_mode=True).numpy())
    a = v.avg_pool((2, 3), padding=(1, 1), count_include_pad=False)
    a.forward()
    np.testing.assert_allclose(a.data(), F.avg_pool2d(torch.from_numpy(x), (2, 3), padding=(1, 1),
                                                      count_include_pad=False).numpy(), rtol=1e-6, atol=1e-6)
    with pytest.raises(nk.NkError, match="at most half the kernel size"):
        v.max_pool(2, padding=2)
    with pytest.raises(nk.NkError, match="Invalid kernel_size"):
        v.avg_pool((2, 2, 2))


def test_captured_training_step_with_pooling(nk, dev):
    """Conv2d -> ReLU -> MaxPool2d(2) -> Conv2d -> ReLU -> AdaptiveAvgPool2d(1) -> flatten -> Linear -> mse, SGD, f32
    IEEE convolutions: the replays equal the eager step (the biases up to their gradients' atomic sums) and torch"""
    rng = np.random.default_rng(11)
    N, Cin, H = 4, 3, 16
    c1 = nk.nn.Conv2d(dev, Cin, 8, (3, 3), padding=(1, 1), rng=rng)
    c2 = nk.nn.Conv2d(dev, 8, 16, (3, 3), padding=(1, 1), rng=rng)
    fc = nk.nn.Linear(dev, 16, 5, rng=rng)
    pool, gap = nk.nn.MaxPool2d(2), nk.nn.AdaptiveAvgPool2d(1)
    params = c1.parameters() + c2.parameters() + fc.parameters()
    init = [p.data().copy() for p in params]
    x = rng.standard_normal((N, Cin, H, H)).astype(F32N)
    t = rng.standard_normal((N, 5)).astype(F32N)
    X, T = nk.from_ndarray(dev, x), nk.from_ndarray(dev, t)
    lr = 0.05
    opt = nk.optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)
    dev.f32_conv("ieee")

    def step():
        opt.zero_grad()
        h = gap.forward(c2.forward(pool.forward(c1.forward(X).relu())).relu()).flatten()
        loss = fc.forward(h).mse_loss(T)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    step()                          # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [p.data().copy() for p in params]
    reset()
    with dev.capture(256 << 20) as cap:
        step()
    for _ in range(3):
        reset()
        cap.graph.launch()
        dev.synchronize()
        for i, (p, e) in enumerate(zip(params, eager)):
            got = p.data()
            if i % 2 == 0:          # weights
                assert np.array_equal(got.view(np.uint32), e.view(np.uint32)), i
            else:                   # biases: their gradients are summed with atomics (nk_unbroadcast_acc)
                assert np.all(np.abs(got - e) <= 2.0 ** -21 * np.abs(e) + 1e-8), i
    # torch CPU, the same step
    tp = [torch.from_numpy(v.copy()).requires_grad_(True) for v in init]
    w1, b1, w2, b2, wf, bf = tp
    h = F.max_pool2d(F.relu(F.conv2d(torch.from_numpy(x), w1, padding=1) + b1), 2)
    h = F.adaptive_avg_pool2d(F.relu(F.conv2d(h, w2, padding=1) + b2), 1).flatten(1)
    loss = F.mse_loss(h @ wf.T + bf, torch.from_numpy(t))
    loss.backward()
    for v, e in zip(tp, eager):
        want = (v - lr * v.grad).detach().numpy().reshape(e.shape)
        np.testing.assert_allclose(e, want, rtol=1e-4, atol=1e-5)
