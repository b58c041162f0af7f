"""Operator-level parity on the H100: every C-ABI entry point against the oracle on the same
seeded inputs.  Tolerances (SURVEY.md 8-d):
  f32 path            : |dev - oracle| <= 1e-5 * (1 + |oracle|) * sqrt(K)/4 (accumulation order)
  indexing/shape ops  : bit exact
  reference goldens   : the reference's own 4.88e-4 abs
  bf16 operands       : tier 1 -- oracle on the SAME bf16-rounded operands, f32 accumulate:
                        rel 2e-3 of the output rms for f32 outputs, + one bf16 rounding (2^-8 rel)
                        for bf16 outputs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
F16_EPS = 4.88e-4


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


def rnd(rng, shape, lo=-1.0, hi=1.0):
    return rng.uniform(lo, hi, size=shape).astype(F32)


def close_f32(got, want, k=1):
    tol = 1e-5 * (1 + np.abs(want)) * max(1.0, np.sqrt(k) / 4)
    return bool(np.all(np.abs(got - want) <= tol))


# ------------------------------------------------------------------------------- plumbing
def test_roundtrip_and_fill(nk, dev):
    rng = np.random.default_rng(0)
    a = rnd(rng, (7, 13))
    d = dev.from_ndarray(a)
    assert np.array_equal(d.as_ndarray(), a)                      # bit exact
    b = dev.from_ndarray(a, nk.BF16)
    from oracle import bf16_round
    assert np.array_equal(b.as_ndarray(), bf16_round(a))          # RNE rounding on the host
    assert np.array_equal(dev.zeros((3, 5)).as_ndarray(), np.zeros((3, 5), F32))   # CuArray::zeroed
    assert np.array_equal(dev.full((4, 4), 2.5, nk.BF16).as_ndarray(), np.full((4, 4), 2.5, F32))
    assert np.array_equal(b.astype(nk.F32).as_ndarray(), bf16_round(a))
    assert np.array_equal(d.astype(nk.BF16).as_ndarray(), bf16_round(a))           # device RNE == host RNE


def test_errors_are_reported_not_fatal(nk, dev):
    from neuronika_b200 import ops
    a, b = dev.zeros((3, 4)), dev.zeros((5, 6))
    with pytest.raises(ValueError):
        ops.mm(a, b)
    with pytest.raises(ValueError, match="incompatible shape"):
        ops.add(dev.zeros((2, 3)), dev.zeros((4, 3)))
    x, w = dev.zeros((1, 3, 2, 2)), dev.zeros((2, 3, 3, 3))
    with pytest.raises(nk.NkError, match="kernel size can't be greater"):
        ops.conv2d(x, w, out=dev.zeros((1, 2, 1, 1)))
    with pytest.raises(nk.NkError, match="not divisible by groups"):
        ops.conv2d(dev.zeros((1, 3, 5, 5)), dev.zeros((8, 2, 2, 2)), groups=2, out=dev.zeros((1, 8, 4, 4)))
    # the context is still usable afterwards
    assert np.array_equal(ops.relu(dev.from_ndarray(np.array([-1.0, 2.0], F32))).as_ndarray(), [0, 2])


# ------------------------------------------------------------------------------- matmul f32
def test_mm_reference_goldens(nk, dev, tensor_goldens):
    """matrix_matrix_mul/test.rs:138-185 through the C ABI, including the accumulate-on-second-
    backward protocol."""
    from neuronika_b200 import ops
    g = tensor_goldens["matrix_matrix_mul"]["backward"][0]["tensors"]
    T = lambda e: np.asarray(e["values"], F32).reshape(e["shape"])
    a = np.linspace(1, 9, 9, dtype=F32).reshape(3, 3)
    b = np.linspace(10, 18, 9, dtype=F32).reshape(3, 3)
    da_, db_, dg = dev.from_ndarray(a), dev.from_ndarray(b), dev.from_ndarray(np.ones((3, 3), F32))
    assert np.array_equal(ops.mm(da_, dev.zeros((3, 3))).as_ndarray(), np.zeros((3, 3)))   # :27-40
    gA, gB = dev.zeros((3, 3)), dev.zeros((3, 3))
    for k in (0, 2):
        ops.gemm(dg, db_, gA, trans_b=True, beta=1.0)            # dA += G.B^T
        ops.gemm(da_, dg, gB, trans_a=True, beta=1.0)            # dB += A^T.G
        assert np.allclose(gA.as_ndarray(), T(g[k]), atol=F16_EPS)
        assert np.allclose(gB.as_ndarray(), T(g[k + 1]), atol=F16_EPS)


def test_mm_t_reference_goldens(nk, dev, tensor_goldens):
    from neuronika_b200 import ops
    T = lambda e: np.asarray(e["values"], F32).reshape(e["shape"])
    f = tensor_goldens["matrix_matrix_mul_t"]["forward"][0]["tensors"]
    y = ops.mm_t(dev.from_ndarray(T(f[0])), dev.from_ndarray(T(f[1])))
    assert np.allclose(y.as_ndarray(), T(f[2]), atol=F16_EPS)
    b = tensor_goldens["matrix_matrix_mul_t"]["backward"][0]["tensors"]
    x, w, g = (dev.from_ndarray(T(b[i])) for i in (2, 3, 4))
    dx, dw = dev.zeros((3, 3)), dev.zeros((2, 3))
    for k in (6, 8):
        ops.gemm(g, w, dx, beta=1.0)                              # dX += G.W
        ops.gemm(g, x, dw, trans_a=True, beta=1.0)                # dW += G^T.X
        assert np.allclose(dx.as_ndarray(), T(b[k]), atol=F16_EPS)
        assert np.allclose(dw.as_ndarray(), T(b[k + 1]), atol=F16_EPS)


@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (37, 53, 29), (1, 1, 1), (10, 300, 2048), (65, 64, 17)])
def test_gemm_f32_all_forms(nk, dev, O, ta, tb, M, N, K):
    """config 1 (Var::mm 128x128.128x128) and ragged shapes, all four operand layouts, f32 engine."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    a = rnd(rng, (K, M) if ta else (M, K))
    b = rnd(rng, (N, K) if tb else (K, N))
    c0 = rnd(rng, (M, N))
    dc = dev.from_ndarray(c0)
    ops.gemm(dev.from_ndarray(a), dev.from_ndarray(b), dc, trans_a=bool(ta), trans_b=bool(tb), alpha=0.5, beta=1.0)
    want = 0.5 * ((a.T if ta else a).astype(np.float64) @ (b.T if tb else b).astype(np.float64)) + c0
    assert close_f32(dc.as_ndarray(), want.astype(F32), K)
    assert dev.last_gemm_kernel.startswith("simt")


def test_config1_mm_fwd_bwd(nk, dev, O):
    """BASELINE config 1: Var::mm 128x128 . 128x128 fwd+bwd (root = sum => G = 1)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(0)
    a, b = rnd(rng, (128, 128)), rnd(rng, (128, 128))
    g = np.ones((128, 128), F32)
    da, db, dg = dev.from_ndarray(a), dev.from_ndarray(b), dev.from_ndarray(g)
    c = ops.mm(da, db)
    gA, gB = dev.zeros((128, 128)), dev.zeros((128, 128))
    ops.gemm(dg, db, gA, trans_b=True, beta=1.0)
    ops.gemm(da, dg, gB, trans_a=True, beta=1.0)
    wa, wb = np.zeros_like(a), np.zeros_like(b)
    O.mm_backward(a, b, g, wa, wb)
    assert close_f32(c.as_ndarray(), O.mm_forward(a, b), 128)
    assert close_f32(gA.as_ndarray(), wa, 128) and close_f32(gB.as_ndarray(), wb, 128)


# ------------------------------------------------------------------------------- matmul bf16 (wgmma)
def _bf16_case(nk, dev, O, form, M, N, K, cdt, beta=0.0, bias=False, relu=False, engine="wgmma"):
    from neuronika_b200 import ops
    ta, tb = form[0] == "T", form[1] == "T"
    rng = np.random.default_rng(hash((form, M, N, K)) % (2 ** 31))
    a = O.bf16_round(rnd(rng, (K, M) if ta else (M, K)))
    b = O.bf16_round(rnd(rng, (N, K) if tb else (K, N)))
    c0 = O.bf16_round(rnd(rng, (M, N)))
    bv = O.bf16_round(rnd(rng, (N,))) if bias else None
    dev.gemm_engine(engine)
    try:
        dc = dev.from_ndarray(c0, cdt)
        ops.gemm(dev.from_ndarray(a, nk.BF16), dev.from_ndarray(b, nk.BF16), dc, trans_a=ta, trans_b=tb, beta=beta,
                 bias=dev.from_ndarray(bv, cdt) if bias else None, relu=relu)
        got = dc.as_ndarray()
        kern = dev.last_gemm_kernel
    finally:
        dev.gemm_engine("auto")
    want = (a.T if ta else a).astype(np.float64) @ (b.T if tb else b).astype(np.float64) + beta * c0
    if bias:
        want = want + bv[None, :]
    if relu:
        want = np.maximum(want, 0)
    scale = max(1e-6, float(np.sqrt((want ** 2).mean())))
    tol = 2e-3 * scale + (2.0 ** -8) * np.abs(want) * (1.0 if cdt == nk.BF16 else 0.0) + 1e-6
    err = np.abs(got - want)
    assert np.all(err <= tol), (form, M, N, K, kern, float(err.max()), scale)
    return kern


@pytest.mark.parametrize("form", ["NT", "NN", "TN", "TT"])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 512), (384, 128, 192), (128, 64, 128)])
def test_gemm_tcgen05_forms(nk, dev, O, form, M, N, K):
    kern = _bf16_case(nk, dev, O, form, M, N, K, nk.F32)
    assert kern.startswith("wgmma_" + form.lower())


@pytest.mark.parametrize("form,M,N,K", [("NT", 200, 72, 136), ("NN", 200, 72, 136), ("TN", 200, 72, 136),
                                        ("NT", 130, 300, 1000), ("TN", 1000, 520, 264), ("NN", 77, 1000, 72),
                                        ("NT", 1000, 10, 4096), ("NT", 64, 24, 64), ("NT", 1, 8, 8)])
def test_gemm_tcgen05_ragged(nk, dev, O, form, M, N, K):
    """tails in M, N and K are handled by TMA zero fill + predicated stores"""
    _bf16_case(nk, dev, O, form, M, N, K, nk.F32)
    _bf16_case(nk, dev, O, form, M, N, K, nk.BF16, beta=1.0)


def test_gemm_tcgen05_epilogues(nk, dev, O):
    _bf16_case(nk, dev, O, "NT", 256, 256, 256, nk.BF16, bias=True, relu=True)       # Linear fwd fused
    _bf16_case(nk, dev, O, "NT", 256, 256, 256, nk.F32, bias=True)
    _bf16_case(nk, dev, O, "TN", 256, 256, 512, nk.F32, beta=1.0)                     # dW += G^T.X
    _bf16_case(nk, dev, O, "NN", 256, 384, 256, nk.BF16, beta=1.0)                    # dX += G.W


def test_gemm_bf16_fallback_when_not_tma_addressable(nk, dev, O):
    """(N,10) logits: leading dimension 10 elements = 20 bytes -> SIMT engine, same numerics contract"""
    from neuronika_b200 import ops
    kern = _bf16_case(nk, dev, O, "NN", 512, 256, 10, nk.BF16, engine="auto")         # dH = G3.W3, lda = 10
    assert kern.startswith("simt")
    kern = _bf16_case(nk, dev, O, "TN", 10, 256, 2048, nk.F32, beta=1.0, engine="auto")   # dW3 = G3^T.H2, split-K
    assert kern.startswith("simt")
    with pytest.raises(nk.NkError, match="not TMA-addressable"):
        _bf16_case(nk, dev, O, "NN", 512, 256, 10, nk.BF16, engine="wgmma")


def test_linear_4096_fwd_bwd_properties(nk, dev, O):
    """config 2 at full size (Linear 4096->4096, batch 4096, bf16): size-independent checks --
    a 64-row slab against the oracle, and linearity of the backward pass in G."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(2)
    n = 4096
    k = 1.0 / np.sqrt(n)
    x = O.bf16_round(rnd(rng, (n, n)))
    w = O.bf16_round(rnd(rng, (n, n), -k, k))
    bias = O.bf16_round(rnd(rng, (n,), -k, k))
    g = O.bf16_round(rnd(rng, (n, n)) / n)
    dx_, dw_, db_, dg = (dev.from_ndarray(v, nk.BF16) for v in (x, w, bias, g))
    y = ops.mm_t(dx_, dw_, bias=db_)
    assert dev.last_gemm_kernel.startswith("wgmma_nt")
    rows = slice(1000, 1064)
    want = x[rows].astype(np.float64) @ w.T.astype(np.float64) + bias
    got = y.as_ndarray()[rows]
    assert np.all(np.abs(got - want) <= 2e-3 * np.sqrt((want ** 2).mean()) + 2.0 ** -8 * np.abs(want))
    gx, gw = dev.zeros((n, n), nk.BF16), dev.zeros((n, n), nk.F32)
    ops.gemm(dg, dw_, gx, beta=0.0)                       # dX = G.W
    ops.gemm(dg, dx_, gw, trans_a=True, beta=0.0)         # dW = G^T.X
    want_dx = g[rows].astype(np.float64) @ w.astype(np.float64)
    assert np.all(np.abs(gx.as_ndarray()[rows] - want_dx) <= 2e-3 * np.sqrt((want_dx ** 2).mean()) + 2.0 ** -8 * np.abs(want_dx))
    want_dw = g[:, rows].T.astype(np.float64) @ x.astype(np.float64)
    assert np.all(np.abs(gw.as_ndarray()[rows] - want_dw) <= 2e-3 * np.sqrt((want_dw ** 2).mean()))
    # accumulate protocol: second backward doubles dW (beta = 1)
    gw2 = dev.from_ndarray(gw.as_ndarray())
    ops.gemm(dg, dx_, gw2, trans_a=True, beta=1.0)
    assert np.allclose(gw2.as_ndarray(), 2 * gw.as_ndarray(), rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------- elementwise family
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_add_broadcast_and_unbroadcast(nk, dev, O, dt):
    from neuronika_b200 import ops
    D = nk.F32 if dt == "f32" else nk.BF16
    r = (lambda v: v) if dt == "f32" else O.bf16_round
    rng = np.random.default_rng(3)
    cases = [((64, 40), (40,)), ((6, 5, 7, 9), (5, 1, 1)), ((33, 17), (33, 17)), ((1, 3), (2, 2, 3)),
             ((4, 1, 5), (3, 1)), ((8, 16), ())]
    for ls, rs in cases:
        l, rr = r(rnd(rng, ls)), r(rnd(rng, rs))
        got = ops.add(dev.from_ndarray(l, D), dev.from_ndarray(rr, D)).as_ndarray()
        assert np.array_equal(got, r(O.add_forward(l, rr))), (ls, rs)
    # un-broadcast (bias gradients): column sums, channel sums, generic
    for gs, ds in [((256, 40), (40,)), ((6, 5, 7, 9), (5, 1, 1)), ((12, 7), (12, 1)), ((5, 3, 4), (3, 1)),
                   ((4, 6), (4, 6)), ((3, 4, 5), (1, 1, 1))]:
        g = r(rnd(rng, gs))
        d0 = r(rnd(rng, ds))
        dst = dev.from_ndarray(d0, nk.F32)
        ops.unbroadcast_acc(dst, dev.from_ndarray(g, D), beta=1.0)
        want = d0 + O.unbroadcast(g, ds)
        assert np.allclose(dst.as_ndarray(), want, rtol=1e-5, atol=1e-4), (gs, ds)
    # reference golden: addition/test.rs:109-124
    d = dev.zeros((3,))
    ops.unbroadcast_acc(d, dev.full((3, 3), 1.0), beta=1.0)
    assert np.array_equal(d.as_ndarray(), [3, 3, 3])
    ops.unbroadcast_acc(d, dev.full((3, 3), 1.0), beta=1.0)
    assert np.array_equal(d.as_ndarray(), [6, 6, 6])


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n", [1, 7, 4096, 100003])
def test_relu(nk, dev, O, dt, n):
    from neuronika_b200 import ops
    D = nk.F32 if dt == "f32" else nk.BF16
    r = (lambda v: v) if dt == "f32" else O.bf16_round
    rng = np.random.default_rng(n)
    x, g, d0 = r(rnd(rng, (n,))), r(rnd(rng, (n,))), r(rnd(rng, (n,)))
    x[::5] = 0.0
    dx_ = dev.from_ndarray(x, D)
    assert np.array_equal(ops.relu(dx_).as_ndarray(), O.relu_forward(x))                  # bit exact
    acc = dev.from_ndarray(d0, D)
    ops.relu_bwd(acc, dx_, dev.from_ndarray(g, D), beta=1.0)
    want = d0.copy()
    O.relu_backward(x, g, want)
    assert np.array_equal(acc.as_ndarray(), r(want))
    acc0 = dev.from_ndarray(d0, D)
    ops.relu_bwd(acc0, dx_, dev.from_ndarray(g, D), beta=0.0)
    assert np.array_equal(acc0.as_ndarray(), np.where(x > 0, g, 0))


def test_relu_goldens(nk, dev, tensor_goldens):
    from neuronika_b200 import ops
    T = lambda e: np.asarray(e["values"], F32).reshape(e["shape"])
    f = tensor_goldens["relu"]["forward"][0]["tensors"]
    assert np.array_equal(ops.relu(dev.from_ndarray(T(f[0]))).as_ndarray(), T(f[1]))
    b = tensor_goldens["relu"]["backward"][0]["tensors"]
    dx = dev.zeros((3,))
    for k in (4, 5):
        ops.relu_bwd(dx, dev.from_ndarray(T(b[1])), dev.from_ndarray(T(b[2])), beta=1.0)
        assert np.array_equal(dx.as_ndarray(), T(b[k]))


@pytest.mark.parametrize("log", [False, True])
@pytest.mark.parametrize("shape,axis", [((8192, 10), 1), ((3, 3), 0), ((3, 3), 1), ((5, 100, 7), 1), ((4, 6, 300), 2)])
def test_softmax_family(nk, dev, O, log, shape, axis):
    from neuronika_b200 import ops
    rng = np.random.default_rng(5)
    x, g, d0 = rnd(rng, shape, -4, 4), rnd(rng, shape), rnd(rng, shape)
    fwd = O.log_softmax_forward if log else O.softmax_forward
    bwd = O.log_softmax_backward if log else O.softmax_backward
    y = ops.softmax(dev.from_ndarray(x), axis, log=log)
    want_y = fwd(x, axis)
    assert np.allclose(y.as_ndarray(), want_y, rtol=2e-6, atol=2e-6)
    dx = dev.from_ndarray(d0)
    ops.softmax_bwd(dx, dev.from_ndarray(want_y), dev.from_ndarray(g), axis, beta=1.0, log=log)
    want = d0.copy()
    bwd(want_y, g, want, axis)
    assert np.allclose(dx.as_ndarray(), want, rtol=1e-5, atol=1e-5)


def test_softmax_goldens(nk, dev, tensor_goldens):
    from neuronika_b200 import ops
    T = lambda e: np.asarray(e["values"], F32).reshape(e["shape"])
    for node, log in (("softmax", False), ("logsoftmax", True)):
        for which, axis in (("rows", 0), ("columns", 1)):
            f = tensor_goldens[node][f"forward_{which}"][0]["tensors"]
            y = ops.softmax(dev.from_ndarray(T(f[0])), axis, log=log)
            assert np.allclose(y.as_ndarray(), T(f[1]), atol=F16_EPS)
            b = tensor_goldens[node][f"backward_{which}"][0]["tensors"]
            yy = ops.softmax(dev.from_ndarray(T(b[1])), axis, log=log)
            dx = dev.zeros((3, 3))
            ops.softmax_bwd(dx, yy, dev.from_ndarray(T(b[2])), axis, beta=1.0, log=log)
            assert np.allclose(dx.as_ndarray(), T(b[4]), atol=1e-3)
            ops.softmax_bwd(dx, yy, dev.from_ndarray(T(b[2])), axis, beta=1.0, log=log)
            assert np.allclose(dx.as_ndarray(), T(b[5]), atol=2e-3)


def test_losses_and_reductions(nk, dev, O, tensor_goldens):
    from neuronika_b200 import ops
    T = lambda e: np.asarray(e["values"], F32).reshape(e["shape"])
    one = dev.full((), 1.0)
    for red in ("mean", "sum"):
        blk = tensor_goldens["squared_error"][red][0]
        t, x = T(blk["tensors"][0]), T(blk["tensors"][1])
        dx_, dt_ = dev.from_ndarray(x), dev.from_ndarray(t)
        assert abs(float(ops.mse(dx_, dt_, mean=red == "mean").as_ndarray()) - blk["scalars"][0]) <= F16_EPS
        d = dev.zeros((3, 3))
        for k in (3, 4):
            ops.mse_bwd(d, dx_, dt_, one, mean=red == "mean", beta=1.0)
            assert np.allclose(d.as_ndarray(), T(blk["tensors"][k]), atol=F16_EPS)
        nb = tensor_goldens["nll"][red][0]
        target, logits = T(nb["tensors"][0]), T(nb["tensors"][1])
        logp = ops.softmax(dev.from_ndarray(logits), 1, log=True)
        dt2 = dev.from_ndarray(target)
        assert abs(float(ops.nll(logp, dt2, mean=red == "mean").as_ndarray()) - nb["scalars"][0]) <= F16_EPS
        dl = dev.zeros((3, 5))
        ops.nll_bwd(dl, dt2, one, mean=red == "mean", beta=1.0)
        assert np.allclose(dl.as_ndarray(), T(nb["tensors"][3]), atol=F16_EPS)
    rng = np.random.default_rng(6)
    x, t = rnd(rng, (8192, 10)), rnd(rng, (8192, 10))
    got = float(ops.mse(dev.from_ndarray(x), dev.from_ndarray(t)).as_ndarray())
    assert abs(got - float(O.mse_forward(x, t))) <= 1e-6 * abs(got) + 1e-7
    s = float(ops.reduce_sum(dev.from_ndarray(x)).as_ndarray())
    assert abs(s - float(O.sum_forward(x))) <= 1e-6 * abs(s) + 1e-4
    m = float(ops.reduce_sum(dev.from_ndarray(x), mean=True).as_ndarray())
    assert abs(m - float(O.mean_forward(x))) <= 1e-6
    d = dev.zeros((10, 10))
    ops.reduce_sum_bwd(d, one, mean=True, beta=1.0)
    ops.reduce_sum_bwd(d, one, mean=True, beta=1.0)
    assert np.allclose(d.as_ndarray(), 0.02, atol=1e-7)          # mean/test.rs:141


def test_pad_bit_exact(nk, dev, O):
    from neuronika_b200 import ops
    base = np.arange(25, dtype=F32).reshape(1, 1, 5, 5)
    want = O.pad_forward(base, (1, 2), 8.0)                       # pad/constant/test.rs:5-32
    assert np.array_equal(ops.pad2d(dev.from_ndarray(base), (1, 2), 8.0).as_ndarray(), want)
    rng = np.random.default_rng(7)
    x = rnd(rng, (3, 4, 9, 11))
    for D, r in ((nk.F32, lambda v: v), (nk.BF16, O.bf16_round)):
        xr = r(x)
        y = ops.pad2d(dev.from_ndarray(xr, D), (2, 1), 0.0)
        assert np.array_equal(y.as_ndarray(), O.pad_forward(xr, (2, 1), 0.0))
        g = r(rnd(rng, y.shape))
        d0 = r(rnd(rng, x.shape))
        dx = dev.from_ndarray(d0, D)
        ops.pad2d_bwd(dx, dev.from_ndarray(g, D), (2, 1), beta=1.0)
        want = d0.copy()
        O.pad_backward(g, want, (2, 1))
        assert np.array_equal(dx.as_ndarray(), r(want))


def test_multi_sgd_step(nk, dev, O):
    """nk_multi_sgd_step on one tensor, lr from an nk_optim_hyper block"""
    import ctypes as C
    from neuronika_b200 import _lib as L
    from neuronika_b200.device import CuArray
    rng = np.random.default_rng(8)
    hyper = CuArray(dev, (C.sizeof(L.OptimHyper) // 4,), nk.F32)
    L.check(L.lib.nk_optim_hyper_set(dev.ctx, hyper.ptr, C.byref(L.OptimHyper(lr=0.01))), dev.ctx)

    def one(a):
        return None if a is None else (C.c_void_p * 1)(a.ptr.value)
    for kw in ({}, {"l2": 0.01}, {"momentum": 0.9}, {"momentum": 0.9, "dampening": 0.1, "nesterov": True, "l2": 0.001}):
        w, g = rnd(rng, (1000,)), rnd(rng, (1000,))
        dw_, dg_ = dev.from_ndarray(w), dev.from_ndarray(g)
        buf = dev.zeros((1000,)) if "momentum" in kw else None
        ww, gg, bb = w.copy(), g.copy(), None
        for _ in range(3):
            L.check(L.lib.nk_multi_sgd_step(dev.ctx, 1, one(dw_), one(dg_), dw_.dtype, dg_.dtype, one(buf), None,
                                            (C.c_int64 * 1)(1000), hyper.ptr, kw.get("l2", 0.0),
                                            kw.get("momentum", 0.0), kw.get("dampening", 0.0),
                                            int(kw.get("nesterov", False)), 1.0, 1), dev.ctx)
            bb = O.sgd_step(ww, gg, 0.01, buf=bb, **kw)
        assert np.allclose(dw_.as_ndarray(), ww, rtol=1e-6, atol=1e-7), kw
        assert np.allclose(dg_.as_ndarray(), gg, rtol=1e-6, atol=1e-7), kw   # reference mutates grad (+= penalty)


# ------------------------------------------------------------------------------- convolution
CONV2D = ["conv2d", "conv2d_strided", "conv2d_dilated", "grouped_conv2d"]


@pytest.mark.parametrize("name", CONV2D)
def test_conv2d_reference_goldens(nk, dev, conv_goldens, name):
    """convolution/test.rs 2-D cases through the C ABI: exact integer goldens."""
    from neuronika_b200 import ops
    c = conv_goldens[name]
    x = np.arange(c["input_arange"], dtype=F32).reshape(c["input_shape"])
    w = np.full(c["kernel_shape"], 1.0, F32)
    dx_, dw_ = dev.from_ndarray(x), dev.from_ndarray(w)
    y = ops.conv2d(dx_, dw_, c["stride"], c["dilation"], c["groups"])
    assert np.array_equal(y.as_ndarray().ravel(), np.asarray(c["output"], F32))
    g = dev.full(y.shape, 1.0)
    gx, gw = dev.zeros(x.shape), dev.zeros(w.shape)
    for rep in (1, 2):                                            # accumulate on the second backward
        ops.conv2d_bwd_input(gx, g, dw_, c["stride"], c["dilation"], c["groups"], beta=1.0)
        ops.conv2d_bwd_kernel(gw, g, dx_, c["stride"], c["dilation"], c["groups"], beta=1.0)
        assert np.array_equal(gx.as_ndarray().ravel(), rep * np.asarray(c["input_grad"], F32))
        assert np.array_equal(gw.as_ndarray().ravel(), rep * np.asarray(c["kernel_grad"], F32))


@pytest.mark.parametrize("stride,dil,groups", [((1, 1), (1, 1), 1), ((2, 1), (1, 2), 1), ((1, 2), (2, 1), 2)])
def test_conv2d_random_f32(nk, dev, O, stride, dil, groups):
    """non-uniform kernels/gradients: pins the dX layout the reference's own tests cannot see"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(9)
    x, w = rnd(rng, (3, 4, 13, 11)), rnd(rng, (6, 4 // groups, 3, 2))
    y = ops.conv2d(dev.from_ndarray(x), dev.from_ndarray(w), stride, dil, groups)
    want = O.conv_forward(x, w, stride, dil, groups)
    assert close_f32(y.as_ndarray(), want, 24)
    g = rnd(rng, want.shape)
    bias = rnd(rng, (6,))
    yb = ops.conv2d(dev.from_ndarray(x), dev.from_ndarray(w), stride, dil, groups, bias=dev.from_ndarray(bias), relu=True)
    assert close_f32(yb.as_ndarray(), np.maximum(want + bias[None, :, None, None], 0), 24)
    gx, gw, gb = dev.zeros(x.shape), dev.zeros(w.shape), dev.zeros((6, 1, 1))
    ops.conv2d_bwd_input(gx, dev.from_ndarray(g), dev.from_ndarray(w), stride, dil, groups, beta=1.0)
    ops.conv2d_bwd_kernel(gw, dev.from_ndarray(g), dev.from_ndarray(x), stride, dil, groups, beta=1.0, dbias=gb)
    wx, ww = np.zeros_like(x), np.zeros_like(w)
    O.conv_backward_input(wx, g, w, stride, dil, groups)
    O.conv_backward_kernel(ww, g, x, stride, dil, groups)
    assert close_f32(gx.as_ndarray(), wx, 64) and close_f32(gw.as_ndarray(), ww, 400)
    assert np.allclose(gb.as_ndarray().ravel(), g.sum((0, 2, 3)), rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("shape,k", [((2, 3, 20, 24), (3, 3)), ((5, 3, 13, 16), (3, 3)), ((3, 1, 9, 40), (3, 3)),
                                     ((2, 3, 10, 224), (3, 3)), ((1, 2, 7, 8), (3, 3)), ((2, 4, 9, 32), (2, 5)),
                                     ((2, 4, 6, 24), (2, 1)), ((3, 3, 30, 64), (3, 9)), ((300, 3, 8, 16), (3, 3))])
def test_conv2d_toeplitz_forward(nk, dev, O, shape, k):
    """thin inputs (Cin*kh <= 9, Cout = 64): partial 8-pixel groups, every tap width up to 9, widths up to 224 pixels,
    more tiles than SMs; the output is written into a slice of a larger buffer whose canaries must survive"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(sum(shape) + k[1])
    x = O.bf16_round(rnd(rng, shape, -1, 1))
    w = O.bf16_round(rnd(rng, (64, shape[1]) + k, -0.3, 0.3))
    b = O.bf16_round(rnd(rng, (64,), -0.2, 0.2))
    dx_, dw_, db_ = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16), dev.from_ndarray(b, nk.BF16)
    ho, wo = shape[2] - k[0] + 1, shape[3] - k[1] + 1
    # canaries around the output: the aligned-span copy-out must not write a byte outside y
    big = dev.full((shape[0] * 64 * ho * wo + 64,), 7.0, nk.BF16)
    y = big.slice_flat(32, (shape[0], 64, ho, wo))
    ops.conv2d(dx_, dw_, out=y)
    # every case runs on the tensor cores except (2, 4, 6, 24) with a 2x1 kernel: K = Cin*kh*kw = 8 is below the
    # im2col engine's minimum of 9, so it runs on the CUDA cores
    small_k = (shape, k) == ((2, 4, 6, 24), (2, 1))
    assert dev.last_conv_kernel == ("direct_fwd" if small_k else "wgmma_im2col_gemm_fwd")
    want = O.conv_forward(x, w, (1, 1), (1, 1)).astype(np.float64)
    scale = float(np.sqrt((want ** 2).mean())) + 1e-9
    got = big.as_ndarray()
    assert np.all(got[:32] == 7.0) and np.all(got[-32:] == 7.0)
    err = np.abs(y.as_ndarray() - want)
    assert np.all(err <= 2e-3 * scale + 2.0 ** -8 * np.abs(want)), float(err.max())
    yb = ops.conv2d(dx_, dw_, bias=db_, relu=True)
    wb = np.maximum(want + b[None, :, None, None], 0)
    assert np.all(np.abs(yb.as_ndarray() - wb) <= 2e-3 * scale + 2.0 ** -8 * np.abs(wb))


@pytest.mark.parametrize("shape,cout,k", [((2, 3, 20, 24), 64, (3, 3)), ((1, 3, 224, 224), 64, (3, 3)),
                                          ((3, 8, 17, 40), 32, (3, 3)), ((2, 5, 9, 72), 100, (2, 4)),
                                          ((2, 32, 12, 32), 64, (3, 3)), ((1, 1, 6, 8), 1, (1, 1))])
def test_conv2d_tensor_core_forward(nk, dev, O, shape, cout, k):
    """bf16 stride-1 convolution on the tensor-core engine vs the oracle on the same bf16-rounded
    operands (f32 accumulate); bias + ReLU fused in the epilogue; ragged widths (Wo not a multiple of 64)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(11)
    x = O.bf16_round(rnd(rng, shape, 0, 1))
    w = O.bf16_round(rnd(rng, (cout, shape[1]) + k, -0.3, 0.3))
    b = O.bf16_round(rnd(rng, (cout,), -0.2, 0.2))
    dx_, dw_, db_ = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16), dev.from_ndarray(b, nk.BF16)
    y = ops.conv2d(dx_, dw_)
    # every case runs on the tensor cores except the 1x1 convolution of one channel into one (K = 1, Cout = 1)
    one_by_one = cout == 1
    assert dev.last_conv_kernel == ("direct_fwd" if one_by_one else "wgmma_im2col_gemm_fwd")
    want = O.conv_forward(x, w, (1, 1), (1, 1)).astype(np.float64)
    scale = float(np.sqrt((want ** 2).mean())) + 1e-9
    err = np.abs(y.as_ndarray() - want)
    assert np.all(err <= 2e-3 * scale + 2.0 ** -8 * np.abs(want)), float(err.max())
    yb = ops.conv2d(dx_, dw_, bias=db_, relu=True)
    wb = np.maximum(want + b[None, :, None, None], 0)
    assert np.all(np.abs(yb.as_ndarray() - wb) <= 2e-3 * scale + 2.0 ** -8 * np.abs(wb))
    # the direct engine gives the same numbers up to bf16 rounding of the output
    dev.conv_engine("direct")
    try:
        yd = ops.conv2d(dx_, dw_)
        assert dev.last_conv_kernel == "direct_fwd"
    finally:
        dev.conv_engine("auto")
    assert np.all(np.abs(yd.as_ndarray() - y.as_ndarray()) <= 2e-3 * scale + 2.0 ** -7 * np.abs(want))


@pytest.mark.parametrize("shape,cout,k", [((2, 3, 20, 24), 64, (3, 3)), ((1, 3, 224, 224), 64, (3, 3)),
                                          ((3, 8, 17, 40), 32, (3, 3)), ((2, 5, 9, 72), 100, (2, 3)),
                                          ((2, 32, 12, 32), 64, (3, 3)), ((2, 4, 6, 16), 8, (4, 1))])
def test_conv2d_tensor_core_backward_kernel(nk, dev, O, shape, cout, k):
    """dW (+ dbias) on the tensor-core engine: accumulate-into-grad protocol (beta = 1)"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(12)
    x = O.bf16_round(rnd(rng, shape, 0, 1))
    ho, wo = shape[2] - k[0] + 1, shape[3] - k[1] + 1
    g = O.bf16_round(rnd(rng, (shape[0], cout, ho, wo)))
    w0 = rnd(rng, (cout, shape[1]) + k)
    b0 = rnd(rng, (cout, 1, 1))
    dw = dev.from_ndarray(w0, nk.F32)
    db = dev.from_ndarray(b0, nk.F32)
    ops.conv2d_bwd_kernel(dw, dev.from_ndarray(g, nk.BF16), dev.from_ndarray(x, nk.BF16), beta=1.0, dbias=db)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dw"
    want = np.zeros_like(w0, dtype=np.float32)
    O.conv_backward_kernel(want, g, x, (1, 1), (1, 1))
    scale = float(np.sqrt((want.astype(np.float64) ** 2).mean())) + 1e-9
    assert np.all(np.abs(dw.as_ndarray() - (w0 + want)) <= 2e-3 * scale + 1e-5), float(np.abs(dw.as_ndarray() - (w0 + want)).max())
    wb = g.astype(np.float64).sum((0, 2, 3)).reshape(cout, 1, 1)
    assert np.all(np.abs(db.as_ndarray() - (b0 + wb)) <= 2e-3 * (np.abs(wb).max() + 1) + 1e-4)
    # overwrite mode (beta = 0) and bf16 gradient storage
    dwb = dev.from_ndarray(w0, nk.BF16)
    ops.conv2d_bwd_kernel(dwb, dev.from_ndarray(g, nk.BF16), dev.from_ndarray(x, nk.BF16), beta=0.0)
    assert np.all(np.abs(dwb.as_ndarray() - want) <= 2e-3 * scale + 2.0 ** -8 * np.abs(want) + 1e-5)


@pytest.mark.parametrize("shape,cout", [((2, 3, 20, 24), 64), ((1, 3, 224, 224), 64), ((3, 1, 9, 40), 32),
                                        ((2, 2, 70, 16), 16), ((2, 3, 130, 256), 64)])
def test_conv2d_tensor_core_backward_input(nk, dev, O, shape, cout):
    """dX on the tensor-core engine (3x3, Cin <= 3); random (non-uniform) kernels and gradients pin the layout the
    reference's all-ones tests cannot see; beta = 1 accumulates into an existing gradient."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(13)
    w = O.bf16_round(rnd(rng, (cout, shape[1], 3, 3), -0.3, 0.3))
    g = O.bf16_round(rnd(rng, (shape[0], cout, shape[2] - 2, shape[3] - 2)))
    d0 = O.bf16_round(rnd(rng, shape))
    want = np.zeros(shape, F32)
    O.conv_backward_input(want, g, w, (1, 1), (1, 1))
    want = want.astype(np.float64)
    scale = float(np.sqrt((want ** 2).mean())) + 1e-9
    dx = dev.zeros(shape, nk.BF16)
    ops.conv2d_bwd_input(dx, dev.from_ndarray(g, nk.BF16), dev.from_ndarray(w, nk.BF16), beta=0.0)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
    err = np.abs(dx.as_ndarray() - want)
    assert np.all(err <= 2e-3 * scale + 2.0 ** -8 * np.abs(want)), float(err.max())
    dx1 = dev.from_ndarray(d0, nk.BF16)
    ops.conv2d_bwd_input(dx1, dev.from_ndarray(g, nk.BF16), dev.from_ndarray(w, nk.BF16), beta=1.0)
    want1 = want + d0
    assert np.all(np.abs(dx1.as_ndarray() - want1) <= 2e-3 * scale + 2.0 ** -7 * np.abs(want1))


@pytest.mark.parametrize("shape,cout", [((2, 3, 20, 24), 64), ((1, 3, 224, 224), 64), ((3, 1, 9, 40), 32),
                                        ((2, 2, 70, 16), 16), ((2, 3, 130, 256), 64), ((5, 3, 120, 64), 128),
                                        ((1, 3, 113, 24), 16)])
def test_conv2d_tensor_core_backward_kernel_then_input(nk, dev, O, shape, cout):
    """ConvolutionBackward's two calls on one output gradient, in the graph's order: dW (+ dbias), then dX, on the tensor
    cores.  Accumulate with beta = 1, overwrite with beta = 0; results agree with the oracle and with the CUDA-core
    engine."""
    import os
    from neuronika_b200 import ops
    rng = np.random.default_rng(14)
    x = O.bf16_round(rnd(rng, shape, 0, 1))
    w = O.bf16_round(rnd(rng, (cout, shape[1], 3, 3), -0.3, 0.3))
    g = O.bf16_round(rnd(rng, (shape[0], cout, shape[2] - 2, shape[3] - 2)))
    w0 = rnd(rng, w.shape)
    b0 = rnd(rng, (cout, 1, 1))
    d0 = O.bf16_round(rnd(rng, shape))
    want_dx = np.zeros(shape, F32)
    O.conv_backward_input(want_dx, g, w, (1, 1), (1, 1))
    want_dw = np.zeros_like(w0)
    O.conv_backward_kernel(want_dw, g, x, (1, 1), (1, 1))
    want_db = g.astype(np.float64).sum((0, 2, 3)).reshape(cout, 1, 1)
    sx = float(np.sqrt((want_dx.astype(np.float64) ** 2).mean())) + 1e-9
    sw = float(np.sqrt((want_dw.astype(np.float64) ** 2).mean())) + 1e-9
    G, X, Wd = dev.from_ndarray(g, nk.BF16), dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16)

    def backward(dx, dw, beta, dbias=None):
        ops.conv2d_bwd_kernel(dw, G, X, beta=beta, dbias=dbias)
        ops.conv2d_bwd_input(dx, G, Wd, beta=beta)

    dx, dw, db = dev.from_ndarray(d0, nk.BF16), dev.from_ndarray(w0, nk.F32), dev.from_ndarray(b0, nk.F32)
    backward(dx, dw, 1.0, dbias=db)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
    assert np.all(np.abs(dx.as_ndarray() - (want_dx + d0)) <= 2e-3 * sx + 2.0 ** -7 * np.abs(want_dx + d0))
    assert np.all(np.abs(dw.as_ndarray() - (w0 + want_dw)) <= 2e-3 * sw + 1e-5)
    assert np.all(np.abs(db.as_ndarray() - (b0 + want_db)) <= 2e-3 * (np.abs(want_db).max() + 1) + 1e-4)

    dx2, dw2 = dev.from_ndarray(d0, nk.BF16), dev.from_ndarray(w0, nk.F32)   # overwrite mode, no dbias
    backward(dx2, dw2, 0.0)
    assert np.all(np.abs(dx2.as_ndarray() - want_dx) <= 2e-3 * sx + 2.0 ** -8 * np.abs(want_dx))
    assert np.all(np.abs(dw2.as_ndarray() - want_dw) <= 2e-3 * sw + 1e-5)

    dev.conv_engine("direct")                  # an independent implementation: the same numbers to rounding
    try:
        dx3, dw3 = dev.from_ndarray(d0, nk.BF16), dev.from_ndarray(w0, nk.F32)
        backward(dx3, dw3, 0.0)
        assert dev.last_conv_kernel == "direct_bwd_input"
    finally:
        dev.conv_engine("auto")
    # each within the oracle bounds above, so within twice those of each other
    assert np.all(np.abs(dx3.as_ndarray() - dx2.as_ndarray()) <= 4e-3 * sx + 2.0 ** -7 * np.abs(want_dx))
    assert np.all(np.abs(dw3.as_ndarray() - dw2.as_ndarray()) <= 4e-3 * sw + 2e-5)


@pytest.mark.parametrize("form,M,N,K,cdt,beta,bias,relu", [
    ("NN", 70, 1027, 10, "bf16", 0.0, False, False),     # dH = G.W of a 10-wide layer: ragged N, scalar tail path
    ("NN", 8192, 4096, 10, "bf16", 1.0, False, False),   # config 4 at size, accumulating
    ("NN", 129, 1024, 13, "f32", 0.0, True, True),       # vector path with the bias / ReLU epilogue
    ("TN", 10, 1027, 515, "f32", 1.0, False, False),     # dW = G^T.H of a 10-wide layer: ragged N and K
    ("TN", 10, 4096, 8192, "f32", 0.0, False, False),    # config 4 at size
    ("TN", 12, 512, 4096, "bf16", 0.0, False, False)])
def test_gemm_skinny_kernels(nk, dev, O, form, M, N, K, cdt, beta, bias, relu):
    """the two memory-bound kernels behind the 10-wide output layer of config 4 (operands TMA cannot address)"""
    kern = _bf16_case(nk, dev, O, form, M, N, K, nk.BF16 if cdt == "bf16" else nk.F32, beta=beta, bias=bias, relu=relu,
                      engine="auto")
    assert kern == ("simt_small_k" if form == "NN" else "simt_small_m"), kern
