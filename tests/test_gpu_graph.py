"""Graph-level parity on the H100: Var / VarDiff / nn / optim through the C++ graph + C ABI against the
oracle.  Mirrors the reference's graph tests (neuronika-variable/src/test.rs) and optimizer tests
(neuronika-optim/src/sgd/test.rs) for the in-scope operators."""
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
    return nk.Device(0)


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


def rnd(rng, shape, lo=-1.0, hi=1.0):
    return rng.uniform(lo, hi, size=shape).astype(F32)


def test_history_and_laziness(nk, dev):
    """test.rs:748-806: every op adds exactly one node; nothing is computed before forward()."""
    a = nk.from_ndarray(dev, np.ones((3, 4), F32))
    b = nk.from_ndarray(dev, np.ones((4, 5), F32)).requires_grad()
    c = a.mm(b)
    assert isinstance(c, nk.VarDiff) and c.history_len() == 1 and c.backward_history_len() == 1
    assert np.array_equal(c.data(), np.zeros((3, 5), F32))            # zero-filled until forward()
    c.forward()
    assert np.array_equal(c.data(), np.full((3, 5), 4, F32))
    d = a.mm_t(nk.from_ndarray(dev, np.ones((2, 4), F32)))
    assert type(d) is nk.Var and d.history_len() == 1                   # Var x Var stays Var
    e = c.relu().softmax(1)
    assert e.history_len() == 3 and e.backward_history_len() == 3
    with pytest.raises(nk.NkError, match="forgot to call .forward"):
        e.backward(1.0)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_zeros_after_the_pool_reuses_memory(nk, dev, dtype):
    """nk.zeros() (a leaf) is zero-filled even when the memory pool hands it a block that held other data: the LSTM /
    GRU tests take their initial states from it."""
    dt = nk.F32 if dtype == "f32" else nk.BF16
    shape = (257, 129)
    for _ in range(4):
        junk = dev.full(shape, 3.5, dt)
        dev.synchronize()
        del junk
        z = nk.zeros(dev, shape, dt)
        assert np.array_equal(z.data(), np.zeros(shape, F32))


def test_accumulate_protocol_and_zero_grad(nk, dev, O):
    """second backward() doubles leaf gradients (matrix_matrix_mul/test.rs:138-185), zero_grad clears"""
    rng = np.random.default_rng(0)
    a, b = rnd(rng, (5, 7)), rnd(rng, (7, 3))
    va = nk.from_ndarray(dev, a).requires_grad()
    vb = nk.from_ndarray(dev, b).requires_grad()
    loss = va.mm(vb).sum()
    loss.forward()
    loss.backward(1.0)
    wa, wb = np.zeros_like(a), np.zeros_like(b)
    O.mm_backward(a, b, np.ones((5, 3), F32), wa, wb)
    assert np.allclose(va.grad(), wa, atol=1e-5) and np.allclose(vb.grad(), wb, atol=1e-5)
    assert abs(loss.item() - float((a @ b).sum())) < 1e-4
    loss.backward(1.0)
    # leaves accumulate; the intermediate grad was re-seeded through sum's backward (+=) as in the reference
    assert np.allclose(va.grad(), 3 * wa, atol=1e-4)                    # 1x + (2x: intermediate grad also accumulated)
    va.zero_grad()
    assert np.array_equal(va.grad(), np.zeros_like(a))


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("fusion", [True, False])
def test_linear_layer_matches_oracle(nk, dev, O, dtype, fusion):
    D = nk.F32 if dtype == "f32" else nk.BF16
    r = (lambda v: v) if dtype == "f32" else O.bf16_round
    rng = np.random.default_rng(1)
    nk.set_fusion(fusion)
    try:
        lin = nk.nn.Linear(dev, 64, 48, dtype=D, grad_dtype=nk.F32, rng=rng)
        x = r(rnd(rng, (32, 64)))
        t = r(rnd(rng, (32, 48)))
        w, b = lin.weight.data(), lin.bias.data()
        vx = nk.from_ndarray(dev, x, D).requires_grad()
        y = lin.forward(vx)
        loss = y.mse_loss(nk.from_ndarray(dev, t, D))
        loss.forward()
        loss.backward(1.0)
        yo = r(O.linear_forward(x, w, b))
        g = np.zeros_like(yo)
        O.mse_backward(yo, t, F32(1.0), g, "mean")
        g = r(g)
        dx, dw, db = np.zeros_like(x), np.zeros_like(w), np.zeros_like(b)
        O.linear_backward(x, w, g, dx, dw, db)
        def close(got, want):
            # f32: accumulation-order noise only.  bf16: every stored activation / gradient is rounded to 8
            # bits of mantissa (twice on the unfused path), so the error scales with the operand magnitude
            rms = float(np.sqrt((want.astype(np.float64) ** 2).mean())) + 1e-12
            if dtype == "f32":
                return bool(np.all(np.abs(got - want) <= 1e-4 * np.abs(want) + 1e-5 * rms))
            return bool(np.all(np.abs(got - want) <= 2e-2 * np.abs(want) + 1e-2 * rms))

        assert close(y.data(), yo)
        assert abs(loss.item() - float(O.mse_forward(yo, t))) <= 1e-5 + 1e-3 * abs(loss.item())
        assert close(lin.weight.grad(), dw)
        assert close(lin.bias.grad(), db)
        assert close(vx.grad(), r(dx))
    finally:
        nk.set_fusion(True)


def test_fusion_is_invisible(nk, dev):
    """identical bits with and without the peephole (bias epilogue, gradient aliasing)"""
    outs = []
    for fusion in (True, False):
        nk.set_fusion(fusion)
        rng = np.random.default_rng(2)
        l1 = nk.nn.Linear(dev, 40, 24, rng=rng)
        l2 = nk.nn.Linear(dev, 24, 8, rng=rng)
        x = nk.from_ndarray(dev, rnd(rng, (16, 40)))
        t = nk.from_ndarray(dev, rnd(rng, (16, 8)))
        loss = l2.forward(l1.forward(x).relu()).softmax(1).mse_loss(t)
        loss.forward()
        loss.backward(1.0)
        outs.append([loss.data()] + [p.grad() for p in l1.parameters() + l2.parameters()])
    nk.set_fusion(True)
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("final", ["softmax", "log_softmax"])
def test_mlp_training_step_f32(nk, dev, O, final):
    """config 4 in miniature (64-128-128-10, batch 256), f32: loss, grads and SGD-updated weights"""
    rng = np.random.default_rng(3)
    sizes = [64, 128, 128, 10]
    layers = [nk.nn.Linear(dev, a, b, rng=rng) for a, b in zip(sizes[:-1], sizes[1:])]
    params = [(l.weight.data().copy(), l.bias.data().copy()) for l in layers]
    x = rnd(rng, (256, 64))
    t = np.eye(10, dtype=F32)[np.argmax(x[:, :10], 1)]
    opt = nk.optim.StochasticGD.new(0.05, nk.optim.L2(0.001))
    for l in layers:
        for p in l.parameters():
            opt.register(p)
    losses = []
    for step in range(3):
        opt.zero_grad()
        h = nk.from_ndarray(dev, x)
        for i, l in enumerate(layers):
            h = l.forward(h)
            h = h.relu() if i < 2 else (h.softmax(1) if final == "softmax" else h.log_softmax(1))
        loss = h.mse_loss(nk.from_ndarray(dev, t))
        loss.forward()
        loss.backward(1.0)
        opt.step()
        lo, _ = O.mlp_step(x, t, params, 0.05, 0.001, final=final)
        losses.append(loss.item())
        assert abs(loss.item() - float(lo)) <= 1e-5 * (1 + abs(float(lo)))
    for l, (w, b) in zip(layers, params):
        assert np.allclose(l.weight.data(), w, rtol=1e-4, atol=1e-6)
        assert np.allclose(l.bias.data(), b, rtol=1e-4, atol=1e-6)
    assert losses[-1] < losses[0]


def test_mlp_training_step_bf16_master_weights(nk, dev, O):
    """bf16 activations/weights, f32 gradients + f32 master weights: tracks the f32 oracle step closely"""
    rng = np.random.default_rng(4)
    sizes = [64, 128, 10]
    layers = [nk.nn.Linear(dev, a, b, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng) for a, b in zip(sizes[:-1], sizes[1:])]
    params = [(l.weight.data().copy(), l.bias.data().copy()) for l in layers]   # bf16-representable values
    x = O.bf16_round(rnd(rng, (128, 64)))
    t = np.eye(10, dtype=F32)[np.argmax(x[:, :10], 1)]
    opt = nk.optim.StochasticGD.new(0.1, None, master_weights=True)
    for l in layers:
        for p in l.parameters():
            opt.register(p)
    first = last = None
    for step in range(5):
        opt.zero_grad()
        h = nk.from_ndarray(dev, x, nk.BF16)
        h = layers[0].forward(h).relu()
        p = layers[1].forward(h).softmax(1)
        loss = p.mse_loss(nk.from_ndarray(dev, t, nk.BF16))
        loss.forward()
        loss.backward(1.0)
        opt.step()
        lo, _ = O.mlp_step(x, t, params, 0.1, 0.0)
        assert abs(loss.item() - float(lo)) <= 2e-2 * abs(float(lo)) + 1e-4
        first = first if first is not None else loss.item()
        last = loss.item()
    assert last < first


def test_sgd_loss_decreases_like_reference_test(nk, dev):
    """neuronika-optim/src/sgd/test.rs:64-134 pattern with in-scope ops: loss = mse(x.mm(y), z)"""
    rng = np.random.default_rng(5)
    for kw in ({}, {"momentum": 0.9}, {"momentum": 0.9, "dampening": 0.1, "nesterov": True}):
        x = nk.from_ndarray(dev, rng.random((3, 3), dtype=F32)).requires_grad()
        y = nk.from_ndarray(dev, rng.random((3, 3), dtype=F32)).requires_grad()
        z = nk.from_ndarray(dev, rng.random((3, 3), dtype=F32))
        loss = x.mm(y).mse_loss(z, nk.Reduction.Sum)
        opt = nk.optim.StochasticGD.new(0.01, nk.optim.L2(0.0), kw.get("momentum"), kw.get("dampening"),
                                        kw.get("nesterov", False))
        opt.register(x)
        opt.register(y)
        loss.forward()
        first = loss.item()
        for _ in range(10):
            loss.forward()
            loss.backward(1.0)
            opt.step()
            opt.zero_grad()
        loss.forward()
        assert loss.item() < first
    with pytest.raises(AssertionError, match="Dampening and Nesterov"):       # sgd/test.rs:18-28
        nk.optim.StochasticGD.new(0.01, None, None, 0.1, False)


@pytest.mark.parametrize("padding", [(0, 0), (1, 1), (2, 1)])
def test_conv2d_layer_matches_oracle(nk, dev, O, padding):
    rng = np.random.default_rng(6)
    conv = nk.nn.Conv2d(dev, 3, 8, (3, 3), padding=padding, rng=rng)
    x = rnd(rng, (4, 3, 12, 10), 0, 1)
    w, b = conv.weight.data(), conv.bias.data()
    vx = nk.from_ndarray(dev, x).requires_grad()
    y = conv.forward(vx)
    loss = y.relu().mean()
    loss.forward()
    loss.backward(1.0)
    yo = O.conv2d_layer_forward(x, w, b, padding)
    assert np.allclose(y.data(), yo, rtol=1e-5, atol=1e-5)
    g = np.where(yo > 0, F32(1.0) / yo.size, 0).astype(F32)
    dx, dw, db = np.zeros_like(x), np.zeros_like(w), np.zeros_like(b)
    O.conv2d_layer_backward(x, w, g, dx, dw, db, padding)
    assert np.allclose(conv.weight.grad(), dw, rtol=1e-4, atol=1e-6)
    assert np.allclose(conv.bias.grad(), db, rtol=1e-4, atol=1e-6)
    assert np.allclose(vx.grad(), dx, rtol=1e-4, atol=1e-7)


def test_small_convnet_step(nk, dev, O):
    """config 5 in miniature: Conv2d(3->8,p1) ReLU Conv2d(8->16,p1) ReLU flatten Linear -> MSE, one SGD step"""
    rng = np.random.default_rng(7)
    c1 = nk.nn.Conv2d(dev, 3, 8, (3, 3), padding=(1, 1), rng=rng)
    c2 = nk.nn.Conv2d(dev, 8, 16, (3, 3), padding=(1, 1), rng=rng)
    fc = nk.nn.Linear(dev, 16 * 8 * 8, 10, rng=rng)
    P = [(m.weight.data().copy(), m.bias.data().copy()) for m in (c1, c2, fc)]
    x = rnd(rng, (16, 3, 8, 8), 0, 1)
    t = np.eye(10, dtype=F32)[rng.integers(0, 10, 16)]
    h = c2.forward(c1.forward(nk.from_ndarray(dev, x)).relu()).relu().flatten()
    loss = fc.forward(h).mse_loss(nk.from_ndarray(dev, t))
    loss.forward()
    loss.backward(1.0)
    # oracle
    z1 = O.conv2d_layer_forward(x, *P[0], (1, 1)); a1 = O.relu_forward(z1)
    z2 = O.conv2d_layer_forward(a1, *P[1], (1, 1)); a2 = O.relu_forward(z2)
    f = a2.reshape(16, -1)
    yo = O.linear_forward(f, *P[2])
    assert abs(loss.item() - float(O.mse_forward(yo, t))) <= 1e-5
    g = np.zeros_like(yo); O.mse_backward(yo, t, F32(1), g, "mean")
    df, dwf, dbf = np.zeros_like(f), np.zeros_like(P[2][0]), np.zeros_like(P[2][1])
    O.linear_backward(f, P[2][0], g, df, dwf, dbf)
    dz2 = np.zeros_like(z2); O.relu_backward(z2, df.reshape(z2.shape), dz2)
    da1, dw2, db2 = np.zeros_like(a1), np.zeros_like(P[1][0]), np.zeros_like(P[1][1])
    O.conv2d_layer_backward(a1, P[1][0], dz2, da1, dw2, db2, (1, 1))
    dz1 = np.zeros_like(z1); O.relu_backward(z1, da1, dz1)
    dw1, db1 = np.zeros_like(P[0][0]), np.zeros_like(P[0][1])
    O.conv2d_layer_backward(x, P[0][0], dz1, None, dw1, db1, (1, 1))
    for got, want in ((fc.weight.grad(), dwf), (fc.bias.grad(), dbf), (c2.weight.grad(), dw2), (c2.bias.grad(), db2),
                      (c1.weight.grad(), dw1), (c1.bias.grad(), db1)):
        assert np.allclose(got, want, rtol=2e-4, atol=1e-6)


def test_no_grad_with_grad(nk, dev):
    """gradient.rs:68-78: no_grad() drops node gradients, with_grad() brings back zeros"""
    a = nk.from_ndarray(dev, np.ones((2, 3), F32)).requires_grad()
    y = a.relu()
    z = y.sum()
    z.forward()
    z.backward(1.0)
    assert np.array_equal(y.grad(), np.ones((2, 3), F32))
    z.no_grad()
    with pytest.raises(nk.NkError, match="de-allocated gradient"):
        y.grad()
    z.with_grad()
    assert np.array_equal(y.grad(), np.zeros((2, 3), F32))
    z.forward()
    z.backward(1.0)
    assert np.array_equal(y.grad(), np.ones((2, 3), F32))
    assert np.array_equal(a.grad(), 2 * np.ones((2, 3), F32))           # the leaf kept accumulating


def test_gradient_hooks_deliver_row_blocks(nk, dev, O):
    """Gradient-ready hooks (data-parallel overlap): every element range is reported exactly once, the weight of a
    Linear arrives in `row_chunks` row blocks computed by separate GEMMs, and the gradients are bit-identical to the
    un-hooked run (same arithmetic per element)."""
    rng = np.random.default_rng(11)
    B, I, Oo = 256, 192, 512
    x = rnd(rng, (B, I))
    t = rnd(rng, (B, Oo))
    w0, b0 = rnd(rng, (Oo, I), -0.1, 0.1), rnd(rng, (Oo,), -0.1, 0.1)
    runs = []
    for chunks in (0, 1, 4):
        lin = nk.nn.Linear(dev, I, Oo, dtype=nk.BF16, grad_dtype=nk.F32, rng=np.random.default_rng(0))
        lin.weight.set_data(w0)
        lin.bias.set_data(b0)
        seen = {"w": [], "b": []}
        if chunks:
            lin.weight.set_grad_hook(lambda b, e: seen["w"].append((b, e)), row_chunks=chunks)
            lin.bias.set_grad_hook(lambda b, e: seen["b"].append((b, e)))
        loss = lin.forward(nk.from_ndarray(dev, x, nk.BF16)).relu().mse_loss(nk.from_ndarray(dev, t, nk.BF16))
        loss.forward()
        loss.backward(1.0)
        runs.append((lin.weight.grad().copy(), lin.bias.grad().copy()))
        if chunks:
            assert seen["b"] == [(0, Oo)]
            rc = Oo // chunks
            assert seen["w"] == [(c * rc * I, (c + 1) * rc * I) for c in range(chunks)]
    for gw, gb in runs[1:]:
        assert np.array_equal(gw, runs[0][0]) and np.array_equal(gb, runs[0][1])
    assert np.abs(runs[0][0]).max() > 0
