"""Parity of the SURVEY.md 8-f rows on the H100, through the C ABI, against the oracle on the same seeded inputs:
the rest of the elementwise / broadcast / shape family (operator level, graph level with double backward, reference
goldens), mv / vm / vv, 1-d / 3-d convolution (the reference's own golden cases), Adam / AMSGrad / RMSProp / Adagrad.
Tolerances: shape ops (transpose, pad) bit exact; f32 maths 1e-5 relative (+1e-6 abs; device expf / logf / tanhf differ
from numpy's by a few ulp); bf16 storage: oracle on the same bf16-rounded inputs, one output rounding (2^-8)."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS = 4.88e-4
HERE = os.path.dirname(os.path.abspath(__file__))


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


@pytest.fixture(scope="module")
def G():
    with open(os.path.join(HERE, "golden", "tensors_next.json")) as fh:
        return json.load(fh)


def T(e):
    return np.asarray(e["values"], F32).reshape(e["shape"])


def close(got, want, rtol=1e-5, atol=1e-6):
    return bool(np.all(np.abs(got - want) <= atol + rtol * np.abs(want)))


def close_bf16(got, want):
    return bool(np.all(np.abs(got - want) <= 2.0 ** -7 * np.abs(want) + 1e-6))


UNARY = [("neg", 0), ("exp", 0), ("ln", 0), ("sqrt", 0), ("sigmoid", 0), ("tanh", 0), ("softplus", 0),
         ("leaky_relu", 0), ("powi", 3), ("powi", -2), ("powi", 0)]


# ------------------------------------------------------------------------------------------- operator level
@pytest.mark.parametrize("op,ip", UNARY)
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n", [1, 1000, 100003])
def test_unary_ops(nk, dev, O, op, ip, dt, n):
    from neuronika_b200 import ops
    rng = np.random.default_rng(n + ip + 10)
    lo = 0.25 if op in ("ln", "sqrt") or (op == "powi" and ip < 0) else -2.0
    x = rng.uniform(lo, 2.0, n).astype(F32)
    g = rng.standard_normal(n).astype(F32)
    d0 = rng.standard_normal(n).astype(F32)
    D = nk.BF16 if dt == "bf16" else nk.F32
    if dt == "bf16":
        x, g, d0 = O.bf16_round(x), O.bf16_round(g), O.bf16_round(d0)
    y = ops.unary(op, dev.from_ndarray(x, D), ip)
    yo = O.unary_forward(op, x, ip)
    cmp = close_bf16 if dt == "bf16" else close
    assert cmp(y.as_ndarray(), yo), "forward"
    # the Backward node reads the OUTPUT the device stored (exp, sqrt, sigmoid, tanh): hand the oracle the same values
    saved_o = y.as_ndarray() if op in O.UNARY_SAVES_OUTPUT else x
    saved = y if op in O.UNARY_SAVES_OUTPUT else dev.from_ndarray(x, D)
    for beta in (0.0, 1.0):
        dx = dev.from_ndarray(d0, D)
        ops.unary_bwd(op, dx, None if op == "neg" else saved, dev.from_ndarray(g, D), ip, beta=beta)
        want = (d0 if beta else np.zeros_like(d0)).copy()
        O.unary_backward(op, g, saved_o, want, ip)
        got = dx.as_ndarray()
        if dt == "bf16":
            assert np.all(np.abs(got - want) <= 2.0 ** -7 * np.abs(want) + 2.0 ** -7 * np.abs(d0) + 1e-5), ("backward", beta)
        else:
            assert close(got, want, rtol=2e-5, atol=2e-6), ("backward", beta)


@pytest.mark.parametrize("op", ["sub", "mul", "div"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("ls,rs", [((5, 7), (5, 7)), ((1024, 256), (1024, 256)), ((4, 1, 6), (3, 6)), ((6,), (2, 3, 6)),
                                   ((3, 1), (1, 4)), ((8, 16, 5, 5), (16, 1, 1)), ((512, 300), (300,))])
def test_binary_ops(nk, dev, O, op, dt, ls, rs):
    from neuronika_b200 import ops
    rng = np.random.default_rng(len(ls) * 100 + len(rs) + sum(ls))
    l = rng.uniform(0.5, 2, ls).astype(F32)
    r = rng.uniform(0.5, 2, rs).astype(F32)
    D = nk.BF16 if dt == "bf16" else nk.F32
    if dt == "bf16":
        l, r = O.bf16_round(l), O.bf16_round(r)
    dl_, dr_ = dev.from_ndarray(l, D), dev.from_ndarray(r, D)
    y = ops.binary(op, dl_, dr_)
    yo = O.binary_forward(op, l, r)
    assert (close_bf16 if dt == "bf16" else close)(y.as_ndarray(), yo)
    g = rng.standard_normal(yo.shape).astype(F32)
    if dt == "bf16":
        g = O.bf16_round(g)
    dg = dev.from_ndarray(g, D)
    for side, shape in ((0, ls), (1, rs)):
        for beta in (0.0, 1.0):
            d0 = rng.standard_normal(shape).astype(F32)
            dst = dev.from_ndarray(d0, nk.F32)               # f32 gradient whatever the operand type
            ops.binary_bwd(op, side, dst, dg, dl_, dr_, beta=beta)
            want = (d0 if beta else np.zeros_like(d0)).copy()
            O.binary_backward(op, g, l, r, want if side == 0 else None, want if side == 1 else None)
            k = yo.size // max(1, int(np.prod(shape)))
            tol = 1e-5 * (1 + np.abs(want)) * max(1.0, np.sqrt(k)) * (4.0 if dt == "bf16" else 1.0)
            assert np.all(np.abs(dst.as_ndarray() - want) <= tol), (side, beta)


def test_transpose_bit_exact(nk, dev, O):
    from neuronika_b200 import ops
    rng = np.random.default_rng(5)
    for shape in ((3, 3), (4, 3), (1, 7), (257, 129), (1000, 33), (5,), (2, 3, 4), (2, 3, 4, 5)):
        x = rng.standard_normal(shape).astype(F32)
        for D, xx in ((nk.F32, x), (nk.BF16, O.bf16_round(x))):
            y = ops.transpose(dev.from_ndarray(xx, D))
            assert np.array_equal(y.as_ndarray(), O.transpose_forward(xx)), shape
        d0 = rng.standard_normal(shape).astype(F32)
        g = rng.standard_normal(tuple(reversed(shape))).astype(F32)
        dx = dev.from_ndarray(d0)
        ops.transpose(dev.from_ndarray(g), out=dx, beta=1.0)          # dX += G^T
        assert np.array_equal(dx.as_ndarray(), d0 + g.T), shape


@pytest.mark.parametrize("mode", ["constant", "reflective", "replicative"])
def test_pad_modes_bit_exact(nk, dev, O, mode):
    from neuronika_b200 import ops
    rng = np.random.default_rng(9)
    for shape, pad in (((2, 3, 7), (2,)), ((2, 2, 4, 5), (1, 3)), ((1, 2, 3, 4, 5), (2, 1, 3)), ((3, 2, 6, 6), (0, 2)),
                       ((2, 3, 30, 34), (1, 1))):
        x = rng.standard_normal(shape).astype(F32)
        for D, xx in ((nk.F32, x), (nk.BF16, O.bf16_round(x))):
            y = ops.pad_nd(dev.from_ndarray(xx, D), pad, mode, 1.5)
            assert np.array_equal(y.as_ndarray(), O.pad_mode_forward(xx, pad, mode, 1.5)), (shape, pad)
        g = rng.standard_normal(y.shape).astype(F32)
        d0 = rng.standard_normal(shape).astype(F32)
        dx = dev.from_ndarray(d0)
        ops.pad_nd_bwd(dx, dev.from_ndarray(g), pad, beta=1.0)
        want = d0.copy()
        O.pad_mode_backward(g, want, pad)
        assert np.array_equal(dx.as_ndarray(), want)
    if mode == "reflective":
        with pytest.raises(nk.NkError, match="smaller than the dimension"):
            ops.pad_nd(dev.zeros((1, 1, 3, 3)), (3, 1), mode)


@pytest.mark.parametrize("rows,cols", [(3, 3), (5, 7), (1000, 37), (64, 4096), (4096, 250)])
def test_gemv_outer_dot(nk, dev, O, rows, cols):
    from neuronika_b200 import ops
    rng = np.random.default_rng(rows + cols)
    a = rng.standard_normal((rows, cols)).astype(F32)
    v = rng.standard_normal(cols).astype(F32)
    u = rng.standard_normal(rows).astype(F32)
    A, Vv, U = dev.from_ndarray(a), dev.from_ndarray(v), dev.from_ndarray(u)
    tol = lambda w, k: 1e-5 * (1 + np.abs(w)) * max(1.0, np.sqrt(k))
    y = ops.gemv(A, Vv)
    assert np.all(np.abs(y.as_ndarray() - O.mv_forward(a, v)) <= tol(O.mv_forward(a, v), cols))
    yt = ops.gemv(A, U, trans=True)
    assert np.all(np.abs(yt.as_ndarray() - O.vm_forward(u, a)) <= tol(O.vm_forward(u, a), rows))
    y0 = rng.standard_normal(cols).astype(F32)
    yy = dev.from_ndarray(y0)
    ops.gemv(A, U, yy, trans=True, beta=1.0)                            # dv += A^T.g
    assert np.all(np.abs(yy.as_ndarray() - (y0 + a.T @ u)) <= tol(y0 + a.T @ u, rows))
    a0 = rng.standard_normal((rows, cols)).astype(F32)
    AA = dev.from_ndarray(a0)
    ops.outer_acc(AA, U, Vv, beta=1.0)
    assert close(AA.as_ndarray(), a0 + np.outer(u, v), rtol=1e-6, atol=1e-6)
    s = ops.dot(Vv, Vv)
    assert abs(float(s.as_ndarray()) - float(np.dot(v.astype(np.float64), v))) <= 1e-5 * cols
    d0 = rng.standard_normal(cols).astype(F32)
    dd = dev.from_ndarray(d0)
    ops.scale_acc(dd, Vv, dev.from_ndarray(np.array(2.5, F32)), beta=1.0)
    assert close(dd.as_ndarray(), d0 + 2.5 * v, rtol=1e-6, atol=1e-6)
    # bf16 storage
    ab, vb = O.bf16_round(a), O.bf16_round(v)
    yb = ops.gemv(dev.from_ndarray(ab, nk.BF16), dev.from_ndarray(vb, nk.BF16))
    wantb = ab.astype(np.float64) @ vb.astype(np.float64)
    assert np.all(np.abs(yb.as_ndarray() - wantb) <= 2.0 ** -7 * np.abs(wantb) + 1e-3 * np.sqrt(cols))


CONV_ND = ["conv1d", "conv1d_strided", "conv1d_dilated", "grouped_conv1d", "conv3d", "conv3d_strided", "conv3d_dilated",
           "grouped_conv3d"]


def test_convnd_reference_goldens(nk, dev, conv_goldens):
    """convolution/test.rs 1-d and 3-d cases (plain / strided / dilated / grouped) through nk_convnd_*, incl. the
    accumulate-on-second-backward protocol"""
    from neuronika_b200 import ops
    ran = 0
    for name, c in conv_goldens.items():
        if name == "im2col" or len(c["input_shape"]) == 4:
            continue
        ran += 1
        x = np.arange(c["input_arange"], dtype=F32).reshape(c["input_shape"])
        w = np.full(c["kernel_shape"], c["kernel_fill"], F32)
        X, W = dev.from_ndarray(x), dev.from_ndarray(w)
        y = ops.convnd(X, W, c["stride"], c["dilation"], c["groups"])
        want = np.asarray(c["output"], F32).reshape(y.shape)
        assert np.allclose(y.as_ndarray(), want, atol=EPS, rtol=1e-6), name
        g = dev.full(y.shape, c["grad_fill"])
        dx, dw = dev.zeros(x.shape), dev.zeros(w.shape)
        for rep in (1, 2):
            ops.convnd_bwd_input(dx, g, W, c["stride"], c["dilation"], c["groups"], beta=1.0)
            ops.convnd_bwd_kernel(dw, g, X, c["stride"], c["dilation"], c["groups"], beta=1.0)
            assert np.allclose(dx.as_ndarray(), rep * np.asarray(c["input_grad"], F32).reshape(x.shape), atol=EPS, rtol=1e-6), name
            assert np.allclose(dw.as_ndarray(), rep * np.asarray(c["kernel_grad"], F32).reshape(w.shape), rtol=1e-5), name
    assert ran >= 8


@pytest.mark.parametrize("xs,ws,stride,dil,groups", [((3, 4, 29), (6, 4, 5), (2,), (1,), 1), ((2, 6, 40), (4, 3, 3), (1,), (3,), 2),
                                                     ((2, 3, 9, 10, 11), (4, 3, 2, 3, 2), (1, 2, 1), (2, 1, 2), 1),
                                                     ((1, 4, 6, 7, 8), (6, 2, 3, 3, 3), (1, 1, 1), (1, 1, 1), 2)])
def test_convnd_random(nk, dev, O, xs, ws, stride, dil, groups):
    from neuronika_b200 import ops
    rng = np.random.default_rng(sum(xs))
    x = rng.standard_normal(xs).astype(F32)
    w = rng.standard_normal(ws).astype(F32)
    X, W = dev.from_ndarray(x), dev.from_ndarray(w)
    y = ops.convnd(X, W, stride, dil, groups)
    yo = O.conv_forward(x, w, stride, dil, groups)
    K = int(np.prod(ws[1:]))
    assert np.all(np.abs(y.as_ndarray() - yo) <= 1e-5 * (1 + np.abs(yo)) * np.sqrt(K))
    g = rng.standard_normal(yo.shape).astype(F32)
    dx0, dw0 = rng.standard_normal(xs).astype(F32), rng.standard_normal(ws).astype(F32)
    dx, dw = dev.from_ndarray(dx0), dev.from_ndarray(dw0)
    ops.convnd_bwd_input(dx, dev.from_ndarray(g), W, stride, dil, groups, beta=1.0)
    ops.convnd_bwd_kernel(dw, dev.from_ndarray(g), X, stride, dil, groups, beta=1.0)
    wx, ww = dx0.copy(), dw0.copy()
    O.conv_backward_input(wx, g, w, stride, dil, groups)
    O.conv_backward_kernel(ww, g, x, stride, dil, groups)
    assert np.all(np.abs(dx.as_ndarray() - wx) <= 1e-5 * (1 + np.abs(wx)) * np.sqrt(K * ws[0]))
    L = int(np.prod(yo.shape[2:])) * xs[0]
    assert np.all(np.abs(dw.as_ndarray() - ww) <= 2e-5 * (1 + np.abs(ww)) * np.sqrt(L))


# ------------------------------------------------------------------------------------------- reference goldens on device
def test_unary_goldens_on_device(nk, dev, G):
    from neuronika_b200 import ops
    for file, op, ip in [("negation", "neg", 0), ("sqrt", "sqrt", 0), ("sigmoid", "sigmoid", 0), ("tanh", "tanh", 0),
                         ("softplus", "softplus", 0), ("leaky_relu", "leaky_relu", 0), ("power", "powi", 3)]:
        t = G[file]["forward"][0]["tensors"]
        assert np.allclose(ops.unary(op, dev.from_ndarray(T(t[0])), ip).as_ndarray(), T(t[1]), atol=EPS, rtol=1e-4), file
        if file == "negation":
            continue
        b = G[file]["backward"][0]["tensors"]
        x = dev.from_ndarray(T(b[1]))
        saved = ops.unary(op, x, ip) if op in ("sigmoid", "tanh") else x
        dx = dev.zeros(T(b[1]).shape)
        for k in (4, 5):                                               # first backward, accumulated second backward
            ops.unary_bwd(op, dx, saved, dev.from_ndarray(T(b[2])), ip, beta=1.0)
            assert np.allclose(dx.as_ndarray(), T(b[k]), atol=2 * EPS, rtol=1e-4), (file, k)


# ------------------------------------------------------------------------------------------- graph level
def test_graph_elementwise_chain_matches_oracle(nk, dev, O):
    """z = ((a * b - c) / d).exp().sigmoid() ... with broadcasting operands; forward, backward, second backward"""
    rng = np.random.default_rng(21)
    a = rng.uniform(0.5, 1.5, (6, 5)).astype(F32)
    b = rng.uniform(0.5, 1.5, (5,)).astype(F32)
    c = rng.uniform(0.5, 1.5, (6, 1)).astype(F32)
    d = rng.uniform(1.0, 2.0, (6, 5)).astype(F32)
    A, B, C, D = (nk.from_ndarray(dev, v).requires_grad() for v in (a, b, c, d))
    root = (((A * B - C) / D).tanh().pow(2).softplus() + (-A).exp().sqrt().ln().sigmoid().leaky_relu()).sum()
    root.forward()
    # oracle
    m = O.binary_forward("mul", a, b)
    s = O.binary_forward("sub", m, c)
    q = O.binary_forward("div", s, d)
    t = O.unary_forward("tanh", q)
    p = O.unary_forward("powi", t, 2)
    sp = O.unary_forward("softplus", p)
    na = O.unary_forward("neg", a)
    e = O.unary_forward("exp", na)
    sq = O.unary_forward("sqrt", e)
    ln = O.unary_forward("ln", sq)
    sg = O.unary_forward("sigmoid", ln)
    lr = O.unary_forward("leaky_relu", sg)
    tot = sp + lr
    assert abs(root.item() - float(tot.sum(dtype=np.float64))) <= 1e-5 * tot.size
    # backward by the oracle, following the reference's protocol: backward(seed) fills the ROOT gradient and every
    # node accumulates into its operands' gradients -- intermediates included, nothing zeroes them between passes
    # (vardiff.rs:125-141) -- so a second backward() is NOT twice the first on a deep graph
    Z = lambda v: np.zeros_like(v)
    dsp, dlr, dp, dt, dq, ds, dm = Z(sp), Z(lr), Z(p), Z(t), Z(q), Z(s), Z(m)
    dsg, dln, dsq, de, dna = Z(sg), Z(ln), Z(sq), Z(e), Z(na)
    da, db, dc, dd = Z(a), Z(b), Z(c), Z(d)

    dtot_acc = Z(tot)
    for rep in (1, 2):
        # the scalar root's gradient is filled with the seed; SumBackward then ACCUMULATES it into d(tot)
        dtot_acc += 1.0
        dtot_saved = dtot_acc.copy()
        # run the pass with d(tot) holding its accumulated value
        def run():
            O.add_backward(dtot_saved, dsp, dlr)
            O.unary_backward("leaky_relu", dlr, sg, dsg)
            O.unary_backward("sigmoid", dsg, sg, dln)
            O.unary_backward("ln", dln, sq, dsq)
            O.unary_backward("sqrt", dsq, sq, de)
            O.unary_backward("exp", de, e, dna)
            O.unary_backward("neg", dna, None, da)
            O.unary_backward("softplus", dsp, p, dp)
            O.unary_backward("powi", dp, t, dt, 2)
            O.unary_backward("tanh", dt, t, dq)
            O.binary_backward("div", dq, s, d, ds, dd)
            O.binary_backward("sub", ds, m, c, dm, dc)
            O.binary_backward("mul", dm, a, b, da, db)
        run()
        root.backward(1.0)
        for var, want in ((A, da), (B, db), (C, dc), (D, dd)):
            assert close(var.grad(), want, rtol=1e-4, atol=1e-5), rep


def test_graph_transpose_pad_mv_vm_vv(nk, dev, O):
    rng = np.random.default_rng(22)
    a = rng.standard_normal((4, 3)).astype(F32)
    v = rng.standard_normal(4).astype(F32)
    u = rng.standard_normal(3).astype(F32)
    A, Vv, U = (nk.from_ndarray(dev, t).requires_grad() for t in (a, v, u))
    # s = < A^T.v , u > + < u.A^T, v >  -> touches t(), mv, vm, vv
    At = A.t()
    root = At.mv(Vv).vv(U) + U.vm(At).vv(Vv)
    root.forward()
    want = float((a.T @ v) @ u + (u @ a.T) @ v)
    assert abs(root.item() - want) <= 1e-5 * (1 + abs(want))
    root.backward(1.0)
    assert close(A.grad(), 2 * np.outer(v, u), rtol=1e-5, atol=1e-6)
    assert close(Vv.grad(), 2 * (a @ u), rtol=1e-5, atol=1e-5)
    assert close(U.grad(), 2 * (a.T @ v), rtol=1e-5, atol=1e-5)
    # padding modes through the graph (backward = interior slice, pad/mod.rs:157-182)
    x = rng.standard_normal((2, 3, 5, 6)).astype(F32)
    for mode in ("reflective", "replicative", "constant"):
        X = nk.from_ndarray(dev, x).requires_grad()
        y = X.pad((2, 1), 0.5, mode=mode)
        y.forward()
        assert np.array_equal(y.data(), O.pad_mode_forward(x, (2, 1), mode, 0.5))
        s = y.sum()
        s.forward()
        s.backward(2.0)
        assert np.array_equal(X.grad(), np.full(x.shape, 2.0, F32))
    x1 = rng.standard_normal((2, 3, 9)).astype(F32)
    X1 = nk.from_ndarray(dev, x1).requires_grad()
    y1 = X1.pad((3,), mode="reflective")
    y1.forward()
    assert np.array_equal(y1.data(), O.pad_mode_forward(x1, (3,), "reflective"))


def test_graph_conv1d_conv3d(nk, dev, O):
    rng = np.random.default_rng(23)
    for xs, ws, stride, dil, groups in (((2, 4, 20), (6, 2, 3), (2,), (1,), 2), ((1, 2, 6, 7, 8), (3, 2, 2, 3, 2), (1, 1, 2), (1, 1, 1), 1)):
        x, w = rng.standard_normal(xs).astype(F32), rng.standard_normal(ws).astype(F32)
        X, W = nk.from_ndarray(dev, x).requires_grad(), nk.from_ndarray(dev, w).requires_grad()
        y = W.convolution(X, stride, dil, groups)
        root = y.sum()
        root.forward()
        yo = O.conv_forward(x, w, stride, dil, groups)
        assert close(y.data(), yo, rtol=1e-4, atol=1e-4)
        root.backward(1.0)
        g = np.ones_like(yo)
        dx, dw = np.zeros_like(x), np.zeros_like(w)
        O.conv_backward_input(dx, g, w, stride, dil, groups)
        O.conv_backward_kernel(dw, g, x, stride, dil, groups)
        assert close(X.grad(), dx, rtol=1e-4, atol=1e-4) and close(W.grad(), dw, rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------- optimizers
def _params(nk, dev, rng, dtype_name):
    w = rng.standard_normal((37, 19)).astype(F32)
    g = [rng.standard_normal((37, 19)).astype(F32) for _ in range(3)]
    return w, g


@pytest.mark.parametrize("kind", ["adam", "amsgrad", "adagrad", "rmsprop", "rmsprop_c", "rmsprop_m", "rmsprop_cm"])
@pytest.mark.parametrize("penalty", ["none", "l2", "l1", "elastic"])
def test_adam_family_matches_oracle(nk, dev, O, kind, penalty):
    from neuronika_b200 import optim
    rng = np.random.default_rng(31)
    w, grads = _params(nk, dev, rng, "f32")
    pen = {"none": (None, 0.0, 0.0), "l2": (optim.L2(0.01), 0.0, 0.01), "l1": (optim.L1(0.02), 0.02, 0.0),
           "elastic": (optim.ElasticNet(0.02, 0.01), 0.02, 0.01)}[penalty]
    P = nk.from_ndarray(dev, w).requires_grad()
    if kind in ("adam", "amsgrad"):
        opt = (optim.AMSGrad if kind == "amsgrad" else optim.Adam).new(1e-2, 0.9, 0.999, pen[0], 1e-8)
    elif kind == "adagrad":
        opt = optim.Adagrad.new(1e-2, 0.1, pen[0], 1e-10)
    else:
        opt = optim.RMSProp.new(1e-2, pen[0], 0.99, 0.9 if "m" in kind.split("_")[-1] and kind != "rmsprop" else None,
                                kind in ("rmsprop_c", "rmsprop_cm"), 1e-8)
    opt.register(P)
    wo = w.copy()
    m, v, vmax = np.zeros_like(w), np.zeros_like(w), np.zeros_like(w)
    sq, ga, buf, gs = np.zeros_like(w), np.zeros_like(w), np.zeros_like(w), np.zeros_like(w)
    for t, g in enumerate(grads, 1):
        opt.zero_grad()
        P.grad_array().copy_from(g)
        opt.step()
        go = g.copy()
        if kind == "adam":
            O.adam_step(wo, go, m, v, t, 1e-2, 0.9, 0.999, 1e-8, pen[1], pen[2])
        elif kind == "amsgrad":
            O.adam_step(wo, go, m, v, t, 1e-2, 0.9, 0.999, 1e-8, pen[1], pen[2], max_exp_avg_sq=vmax)
        elif kind == "adagrad":
            O.adagrad_step(wo, go, gs, t, 1e-2, 0.1, 1e-10, pen[1], pen[2])
        else:
            O.rmsprop_step(wo, go, sq, 1e-2, 0.99, 1e-8, momentum=0.9 if kind in ("rmsprop_m", "rmsprop_cm") else None,
                           centered=kind in ("rmsprop_c", "rmsprop_cm"), grad_avg=ga, buffer=buf, l1=pen[1], l2=pen[2])
        assert close(P.data(), wo, rtol=2e-5, atol=2e-6), (kind, penalty, t)
        assert close(P.grad(), go, rtol=1e-6, atol=1e-7)               # the penalty is added INTO the gradient


def test_adam_bf16_parameter_with_master_weights(nk, dev, O):
    from neuronika_b200 import optim
    rng = np.random.default_rng(32)
    w = O.bf16_round(rng.standard_normal(1000).astype(F32))
    P = nk.from_ndarray(dev, w, nk.BF16).requires_grad(nk.F32)
    opt = optim.Adam.new(1e-3, master_weights=True)
    opt.register(P)
    wo, m, v = w.copy(), np.zeros_like(w), np.zeros_like(w)
    for t in range(1, 4):
        g = rng.standard_normal(1000).astype(F32)
        opt.zero_grad()
        P.grad_array().copy_from(g)
        opt.step()
        O.adam_step(wo, g.copy(), m, v, t, 1e-3, 0.9, 0.999, 1e-8)
        assert np.all(np.abs(P.data() - wo) <= 2.0 ** -8 * np.abs(wo) + 1e-6)


# ------------------------------------------------------------------------------------------- round-1 advisor findings
def test_mixed_gradient_dtype_through_every_backward_node(nk, dev, O):
    """a bf16 leaf with an f32 gradient (requires_grad(F32)) feeding relu / softmax / pad / loss directly: the
    gradient buffer is f32, so the backward kernel must not write bf16 into it"""
    rng = np.random.default_rng(41)
    x = O.bf16_round(rng.standard_normal((6, 10)).astype(F32))
    t = O.bf16_round(rng.standard_normal((6, 10)).astype(F32))
    for fn, ofwd, obwd in (
        (lambda X: X.relu(), lambda v: O.relu_forward(v), lambda v, y, g, d: O.relu_backward(v, g, d)),
        (lambda X: X.softmax(1), lambda v: O.softmax_forward(v, 1), lambda v, y, g, d: O.softmax_backward(y, g, d, 1)),
        (lambda X: X.log_softmax(1), lambda v: O.log_softmax_forward(v, 1), lambda v, y, g, d: O.log_softmax_backward(y, g, d, 1)),
        (lambda X: X.tanh(), lambda v: O.unary_forward("tanh", v), lambda v, y, g, d: O.unary_backward("tanh", g, y, d)),
    ):
        X = nk.from_ndarray(dev, x, nk.BF16).requires_grad(nk.F32)
        root = fn(X).sum()
        root.forward()
        root.backward(1.0)
        y = O.bf16_round(ofwd(x))
        want = np.zeros_like(x)
        obwd(x, y, np.ones_like(x), want)
        got = X.grad()
        assert got.dtype == np.float32 and got.shape == x.shape
        assert np.all(np.abs(got - want) <= 2.0 ** -6 * np.abs(want) + 5e-2), fn
    X = nk.from_ndarray(dev, x, nk.BF16).requires_grad(nk.F32)
    loss = X.mse_loss(nk.from_ndarray(dev, t, nk.BF16))
    loss.forward()
    loss.backward(1.0)
    want = np.zeros_like(x)
    O.mse_backward(x, t, np.float32(1.0), want, "mean")
    assert np.all(np.abs(X.grad() - want) <= 2.0 ** -7 * np.abs(want) + 1e-5)
    xi = O.bf16_round(rng.standard_normal((2, 3, 5, 5)).astype(F32))
    XI = nk.from_ndarray(dev, xi, nk.BF16).requires_grad(nk.F32)
    r = XI.pad((1, 2)).sum()
    r.forward()
    r.backward(3.0)
    assert np.array_equal(XI.grad(), np.full(xi.shape, 3.0, F32))
    # conv input: bf16 data, f32 gradient
    w = O.bf16_round(rng.uniform(-0.3, 0.3, (4, 3, 3, 3)).astype(F32))
    XI = nk.from_ndarray(dev, xi, nk.BF16).requires_grad(nk.F32)
    W = nk.from_ndarray(dev, w, nk.BF16).requires_grad(nk.F32)
    r = W.convolution(XI, (1, 1), (1, 1), 1).sum()
    r.forward()
    r.backward(1.0)
    dx, dw = np.zeros_like(xi), np.zeros_like(w)
    O.conv_backward_input(dx, np.ones((2, 4, 3, 3), F32), w, (1, 1), (1, 1))
    O.conv_backward_kernel(dw, np.ones((2, 4, 3, 3), F32), xi, (1, 1), (1, 1))
    assert np.all(np.abs(XI.grad() - dx) <= 2.0 ** -7 * np.abs(dx) + 1e-3)
    assert np.all(np.abs(W.grad() - dw) <= 1e-3 * (1 + np.abs(dw)))


def test_leaf_plus_constant_keeps_the_leaf_gradient(nk, dev):
    """`y = leaf + c`: the peephole must not alias the leaf's gradient to y's (hooks sit on the leaf, the gradient
    accumulates over backward() calls and outlives the graph)"""
    fired = []
    leaf = nk.from_ndarray(dev, np.ones((4, 4), F32)).requires_grad()
    leaf.set_grad_hook(lambda b, e: fired.append((b, e)))
    c = nk.from_ndarray(dev, np.full((4, 4), 2.0, F32))
    y = leaf + c
    y.forward()
    y.backward(1.0)
    assert fired == [(0, 16)]
    assert np.array_equal(leaf.grad(), np.ones((4, 4), F32))
    y.backward(1.0)                                                    # accumulates, like the reference
    assert np.array_equal(leaf.grad(), np.full((4, 4), 2.0, F32))
    del y
    y2 = leaf + c                                                      # a second graph: the gradient is still the leaf's
    y2.forward()
    y2.backward(0.5)
    assert np.array_equal(leaf.grad(), np.full((4, 4), 2.5, F32))


def test_nll_target_dtype(nk, dev, O):
    """class ids above 256 are not representable in bf16: an f32 target is accepted with bf16 inputs, a bf16 target
    with more than 256 classes is rejected"""
    rng = np.random.default_rng(43)
    n, c = 64, 1000
    logits = rng.standard_normal((n, c)).astype(F32)
    logp = O.bf16_round(O.log_softmax_forward(logits, 1))
    target = rng.integers(0, c, n).astype(F32)
    X = nk.from_ndarray(dev, logp, nk.BF16).requires_grad(nk.F32)
    loss = X.nll_loss(nk.from_ndarray(dev, target, nk.F32))
    loss.forward()
    assert abs(loss.item() - float(O.nll_forward(logp, target, "mean"))) <= 1e-4
    loss.backward(1.0)
    want = np.zeros_like(logp)
    O.nll_backward(target, np.float32(1.0), want, "mean")
    assert np.allclose(X.grad(), want, atol=1e-7)
    with pytest.raises(nk.NkError, match="bf16 target"):
        X.nll_loss(nk.from_ndarray(dev, target, nk.BF16))


# ------------------------------------------------------------------------------------------- whole-step capture
def test_captured_step_replays_like_eager_steps(nk, dev, O):
    """Device.capture records zero_grad -> build -> forward -> backward -> SGD once; replaying it k times must leave the
    parameters where k eager steps leave them (same kernels on the same data; the bias-gradient column sums use f32
    atomics, so equality is to rounding, not bit for bit)"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(51)
    sizes = [64, 256, 128, 10]
    x = O.bf16_round(rng.uniform(-1, 1, (512, sizes[0])).astype(F32))
    t = np.eye(10, dtype=F32)[rng.integers(0, 10, 512)]
    init = []
    for i, o in zip(sizes[:-1], sizes[1:]):
        k = 1.0 / np.sqrt(i)
        init += [rng.uniform(-k, k, (o, i)).astype(F32), rng.uniform(-k, k, (o,)).astype(F32)]

    def build():
        params = [nk.from_ndarray(dev, v, nk.BF16).requires_grad(nk.F32) for v in init]
        opt = optim.StochasticGD.new(0.05, optim.L2(1e-4), momentum=0.9, master_weights=True)
        for p in params:
            opt.register(p)
        X, Tt = nk.from_ndarray(dev, x, nk.BF16), nk.from_ndarray(dev, t, nk.BF16)
        live = {}

        def step():
            opt.zero_grad()
            h = X
            for li in range(3):
                h = h.mm_t(params[2 * li]) + params[2 * li + 1]
                h = h.relu() if li < 2 else h.softmax(1)
            loss = h.mse_loss(Tt)
            loss.forward()
            loss.backward(1.0)
            opt.step()
            live["loss"] = loss
        return params, step, live

    pa, step_a, live_a = build()
    pb, step_b, live_b = build()
    K = 4
    for _ in range(2 + K):
        step_a()
    loss_a = live_a["loss"].item()
    for _ in range(2):
        step_b()                                   # eager warm-up (first-use allocations cannot be captured)
    dev.synchronize()
    before = dev.launches
    with dev.capture(256 << 20) as cap:
        step_b()
    assert dev.launches - before > 0               # the kernels were recorded ...
    g = cap.graph
    assert g.kernel_count >= 15 and 0 < g.arena_used <= 256 << 20
    w_mid = pb[0].data().copy()
    dev.synchronize()
    assert np.array_equal(pb[0].data(), w_mid)     # ... not executed
    for _ in range(K):
        g.launch()
    dev.synchronize()
    loss_b = live_b["loss"].item()                 # the recorded root lives at a fixed arena address
    assert abs(loss_a - loss_b) <= 1e-5 * (1 + abs(loss_a))
    for a, b in zip(pa, pb):
        wa, wb = a.data(), b.data()
        assert np.all(np.abs(wa - wb) <= 2.0 ** -7 * np.abs(wa) + 1e-6)
    # an eager step after the replays continues from the same state
    step_a()
    step_b()
    assert abs(live_a["loss"].item() - live_b["loss"].item()) <= 1e-5
    g.close()


def test_capture_rejects_what_cannot_be_captured(nk, dev):
    a = nk.from_ndarray(dev, np.ones((4, 4), F32))
    with pytest.raises(nk.NkError):
        with dev.capture(1 << 20):
            a.data()                               # a synchronous device-to-host copy inside a capture
    # the context is usable afterwards
    assert np.array_equal(a.data(), np.ones((4, 4), F32))
    big = nk.from_ndarray(dev, np.ones((64, 64), F32))
    with pytest.raises(nk.NkError, match="arena exhausted"):
        with dev.capture(1 << 12):                 # 4 KB arena, 16 KB result
            b = (big + big)
            b.forward()
    r = big + big                                 # and the context still works
    r.forward()
    assert np.array_equal(r.data(), np.full((64, 64), 2.0, F32))


def test_fusion_level_2_relu_backward_in_the_gemm_epilogue(nk, dev, O):
    """level 2 applies a layer's ReLU backward in the epilogue of the dX GEMM above it: same gradients as level 1 (bit
    for bit: the mask is applied before the one bf16 rounding in both), and a second backward() on such a tape fails"""
    rng = np.random.default_rng(61)
    sizes = [128, 512, 256, 10]
    x = O.bf16_round(rng.uniform(-1, 1, (256, sizes[0])).astype(F32))
    t = np.eye(10, dtype=F32)[rng.integers(0, 10, 256)]
    init = []
    for i, o in zip(sizes[:-1], sizes[1:]):
        k = 1.0 / np.sqrt(i)
        init += [rng.uniform(-k, k, (o, i)).astype(F32), rng.uniform(-k, k, (o,)).astype(F32)]
    grads = {}
    try:
        for level in (1, 2, 3):     # 3 = 2 + the hidden layers' bias gradients summed in the dX GEMM epilogue
            nk.set_fusion(level)
            params = [nk.from_ndarray(dev, v, nk.BF16).requires_grad(nk.F32) for v in init]
            X, Tt = nk.from_ndarray(dev, x, nk.BF16).requires_grad(), nk.from_ndarray(dev, t, nk.BF16)
            h = X
            for li in range(3):
                h = h.mm_t(params[2 * li]) + params[2 * li + 1]
                h = h.relu() if li < 2 else h.softmax(1)
            loss = h.mse_loss(Tt)
            del h
            loss.forward()
            before = dev.launches
            loss.backward(1.0)
            launched = dev.launches - before
            grads[level] = ([p.grad().copy() for p in params] + [X.grad().copy()], launched, loss.item())
            if level >= 2:
                with pytest.raises(nk.NkError, match="ONE backward pass"):
                    loss.backward(1.0)
    finally:
        nk.set_fusion(1)
    # the 4096-wide layer's ReLU backward is gone; the one below the 10-wide layer stays a separate launch (its dX
    # GEMM runs on the skinny CUDA-core kernel, whose result then goes through nk_relu_bwd)
    assert grads[2][1] <= grads[1][1] - 1
    assert grads[3][1] <= grads[2][1] - 2          # two column-sum passes (colsum + finalize each) less
    assert grads[1][2] == grads[2][2] == grads[3][2]
    for i, (a, b) in enumerate(list(zip(grads[1][0], grads[2][0])) + list(zip(grads[1][0], grads[3][0]))):
        i = i % len(grads[1][0])
        # bias gradients (column sums) and the 10-row dW of the output layer (gemm_small_m_kernel) are accumulated with
        # f32 atomics, whose order varies from launch to launch: equal to rounding.  Everything else is bit equal.
        if a.ndim == 1 or a.shape[0] <= 16:
            assert np.allclose(a, b, rtol=1e-4, atol=1e-7), i
        else:
            assert np.array_equal(a, b), i
    # and against the oracle (bf16 operands, f32 accumulate)
    wo = [O.bf16_round(v) for v in init]
    h1 = O.bf16_round(O.relu_forward(O.linear_forward(x, wo[0], wo[1])))
    h2 = O.bf16_round(O.relu_forward(O.linear_forward(h1, wo[2], wo[3])))
    z3 = O.bf16_round(O.linear_forward(h2, wo[4], wo[5]))
    y = O.bf16_round(O.softmax_forward(z3, 1))
    dy = np.zeros_like(y)
    O.mse_backward(y, t, np.float32(1.0), dy, "mean")
    dz3 = np.zeros_like(z3)
    O.softmax_backward(y, O.bf16_round(dy), dz3, 1)
    dz3 = O.bf16_round(dz3)
    dw3 = dz3.T @ h2
    assert np.all(np.abs(grads[2][0][4] - dw3) <= 2e-2 * np.abs(dw3).max())


def test_conv_backward_with_a_uniform_output_gradient(nk, dev, O):
    """backward(seed) on a convolution's own output: the graph fills the root gradient and runs the convolution's two
    backward calls on it -- the same launches and results as that sequence made by hand"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(71)
    x = O.bf16_round(rng.uniform(0, 1, (3, 3, 20, 24)).astype(F32))
    w = O.bf16_round(rng.uniform(-0.3, 0.3, (64, 3, 3, 3)).astype(F32))
    X, W = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16)
    seed = 0.37
    sb = float(O.bf16_round(np.array([seed], F32))[0])
    g = np.full((3, 64, 18, 22), sb, F32)
    dx2, dw2, db2 = dev.zeros(x.shape, nk.BF16), dev.zeros(w.shape, nk.F32), dev.zeros((64, 1, 1), nk.F32)
    before = dev.launches
    G = dev.full(g.shape, seed, nk.BF16)
    ops.conv2d_bwd_kernel(dw2, G, X, beta=0.0, dbias=db2)
    ops.conv2d_bwd_input(dx2, G, W, beta=0.0)
    sequence_launches = dev.launches - before
    assert np.array_equal(G.as_ndarray(), g)
    wx, ww = np.zeros_like(x), np.zeros_like(w)
    O.conv_backward_input(wx, g, w, (1, 1), (1, 1))
    O.conv_backward_kernel(ww, g, x, (1, 1), (1, 1))
    assert np.all(np.abs(dx2.as_ndarray() - wx) <= 2.0 ** -7 * np.abs(wx) + 1e-3)
    assert np.all(np.abs(dw2.as_ndarray() - ww) <= 1e-3 * (1 + np.abs(ww)))
    # through the graph: y = conv(x) + b
    Xv = nk.from_ndarray(dev, x, nk.BF16).requires_grad()
    Wv = nk.from_ndarray(dev, w, nk.BF16).requires_grad(nk.F32)
    Bv = nk.from_ndarray(dev, np.zeros((64, 1, 1), F32), nk.BF16).requires_grad(nk.F32)
    y = Wv.convolution(Xv, (1, 1), (1, 1), 1) + Bv
    y.forward()
    before = dev.launches
    y.backward(seed)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
    assert dev.launches - before == sequence_launches
    assert np.array_equal(Xv.grad(), dx2.as_ndarray())                          # same G, same kernels
    assert np.allclose(Wv.grad(), dw2.as_ndarray(), rtol=1e-5, atol=1e-4)       # f32 atomics across CTAs
    assert np.allclose(Bv.grad().ravel(), db2.as_ndarray().ravel(), rtol=1e-5)
    assert np.array_equal(y.grad(), g)
    # the f32 / direct-engine path materialises the fill and gives the oracle's numbers
    Xf, Wf = nk.from_ndarray(dev, x).requires_grad(), nk.from_ndarray(dev, w).requires_grad()
    yf = Wf.convolution(Xf, (1, 1), (1, 1), 1)
    yf.forward()
    yf.backward(seed)
    gf = np.full((3, 64, 18, 22), seed, F32)
    wx, ww = np.zeros_like(x), np.zeros_like(w)
    O.conv_backward_input(wx, gf, w, (1, 1), (1, 1))
    O.conv_backward_kernel(ww, gf, x, (1, 1), (1, 1))
    assert close(Xf.grad(), wx, rtol=1e-4, atol=1e-4) and close(Wf.grad(), ww, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("xs,cout,k,stride,dil", [((4, 32, 10, 18), 64, (3, 3), (1, 1), (1, 1)),
                                                  ((8, 32, 34, 34), 64, (3, 3), (1, 1), (1, 1)),
                                                  ((2, 3, 34, 34), 32, (3, 3), (1, 1), (1, 1)),
                                                  ((2, 16, 17, 33), 24, (3, 3), (2, 2), (1, 1)),
                                                  ((2, 8, 12, 20), 16, (3, 3), (1, 1), (2, 2)),
                                                  ((3, 20, 9, 12), 136, (2, 5), (1, 1), (1, 1))])
def test_conv2d_im2col_gemm_engine(nk, dev, O, xs, cout, k, stride, dil):
    """every bf16, groups = 1 convolution with Ho*Wo % 8 == 0 runs as im2col + batched wgmma GEMM
    (forward with bias + ReLU in the epilogue, dX through col2im, dW as a split reduction over the samples): config 5's
    32 -> 64 layer, strides, dilations, Cout not a multiple of 128, K not a multiple of 8"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(sum(xs) + cout)
    x = O.bf16_round(rng.uniform(-1, 1, xs).astype(F32))
    w = O.bf16_round(rng.uniform(-0.2, 0.2, (cout, xs[1]) + k).astype(F32))
    b = O.bf16_round(rng.uniform(-0.2, 0.2, (cout,)).astype(F32))
    X, W, B = dev.from_ndarray(x, nk.BF16), dev.from_ndarray(w, nk.BF16), dev.from_ndarray(b, nk.BF16)
    y = ops.conv2d(X, W, stride, dil)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_fwd"
    want = O.conv_forward(x, w, stride, dil).astype(np.float64)
    scale = float(np.sqrt((want ** 2).mean())) + 1e-9
    assert np.all(np.abs(y.as_ndarray() - want) <= 2e-3 * scale + 2.0 ** -8 * np.abs(want))
    yb = ops.conv2d(X, W, stride, dil, bias=B, relu=True)
    wb = np.maximum(want + b[None, :, None, None], 0)
    assert np.all(np.abs(yb.as_ndarray() - wb) <= 2e-3 * scale + 2.0 ** -8 * np.abs(wb))
    g = O.bf16_round(rng.uniform(-1, 1, want.shape).astype(F32))
    G = dev.from_ndarray(g, nk.BF16)
    dx0 = O.bf16_round(rng.uniform(-1, 1, xs).astype(F32))
    dw0 = rng.uniform(-1, 1, w.shape).astype(F32)
    for beta in (0.0, 1.0):
        dx, dw, db = dev.from_ndarray(dx0, nk.BF16), dev.from_ndarray(dw0, nk.F32), dev.zeros((cout, 1, 1), nk.F32)
        ops.conv2d_bwd_input(dx, G, W, stride, dil, beta=beta)
        assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
        ops.conv2d_bwd_kernel(dw, G, X, stride, dil, beta=beta, dbias=db)
        assert dev.last_conv_kernel == "wgmma_im2col_gemm_dw"
        wx = (dx0 if beta else np.zeros_like(x)).astype(np.float64)
        ww = (dw0 if beta else np.zeros_like(w)).copy()
        gx = np.zeros_like(x)
        O.conv_backward_input(gx, g, w, stride, dil)
        O.conv_backward_kernel(ww, g, x, stride, dil)
        wx = wx + gx
        sx = float(np.sqrt((gx.astype(np.float64) ** 2).mean())) + 1e-9
        # dX: the column gradients stay in f32 through col2im, so each element is rounded to bf16 once
        assert np.all(np.abs(dx.as_ndarray() - wx) <= 2e-3 * sx + (2.0 ** -7 if beta else 2.0 ** -8) * np.abs(wx) + 1e-6), beta
        sw_ = float(np.sqrt(((ww - (dw0 if beta else 0)) ** 2).mean())) + 1e-9
        assert np.all(np.abs(dw.as_ndarray() - ww) <= 2e-3 * sw_ + 1e-5 * np.abs(ww)), beta
        assert np.allclose(db.as_ndarray().ravel(), g.astype(np.float64).sum((0, 2, 3)), rtol=1e-4, atol=1e-3)


def test_small_convnet_runs_on_tensor_cores(nk, dev, O):
    """config 5's shape of network (Conv2d 3->32 p1, Conv2d 32->64 p1, Linear) at a small batch: every convolution kernel
    of forward and backward is a wgmma one, and the step matches the oracle"""
    rng = np.random.default_rng(81)
    n = 16
    x = O.bf16_round(rng.uniform(0, 1, (n, 3, 32, 32)).astype(F32))
    w1 = O.bf16_round(rng.uniform(-0.2, 0.2, (32, 3, 3, 3)).astype(F32))
    w2 = O.bf16_round(rng.uniform(-0.06, 0.06, (64, 32, 3, 3)).astype(F32))
    X = nk.from_ndarray(dev, x, nk.BF16)
    W1 = nk.from_ndarray(dev, w1, nk.BF16).requires_grad(nk.F32)
    W2 = nk.from_ndarray(dev, w2, nk.BF16).requires_grad(nk.F32)
    seen = []
    h1 = W1.convolution(X.pad((1, 1)), (1, 1), (1, 1), 1).relu()
    h2 = W2.convolution(h1.pad((1, 1)), (1, 1), (1, 1), 1).relu()
    loss = h2.mean()
    loss.forward()
    seen.append(dev.last_conv_kernel)
    loss.backward(1.0)
    seen.append(dev.last_conv_kernel)
    assert all(s.startswith("wgmma") for s in seen), seen
    # oracle
    xp = O.pad_forward(x, (1, 1))
    a1 = O.conv_forward(xp, w1, (1, 1), (1, 1))
    h1o = O.bf16_round(O.relu_forward(O.bf16_round(a1)))
    a2 = O.conv_forward(O.pad_forward(h1o, (1, 1)), w2, (1, 1), (1, 1))
    h2o = O.relu_forward(O.bf16_round(a2))
    assert abs(loss.item() - float(h2o.mean(dtype=np.float64))) <= 2e-3 * float(np.abs(h2o).mean()) + 1e-6
    g2 = O.bf16_round(np.full(h2o.shape, 1.0 / h2o.size, F32)) * (O.bf16_round(a2) > 0)
    dw2 = np.zeros_like(w2)
    O.conv_backward_kernel(dw2, g2.astype(F32), O.pad_forward(h1o, (1, 1)), (1, 1), (1, 1))
    got = W2.grad()
    assert np.all(np.abs(got - dw2) <= 2e-2 * np.abs(dw2).max())
