"""`mae`, `bce`, `bce_with_logits`, `kldiv` and `dropout` on the GPU: the entry points of csrc/nk_criteria.cu and
csrc/nk_dropout.cu, the graph nodes, capture and a small training loop, against tests/criteria_oracle.py.

Backward passes and dropout are elementwise f32 maths, so they are compared bit for bit (bf16 results after one
round-to-nearest-even), except where a transcendental enters (bce_with_logits' backward: CUDA's expf against numpy's,
a few ulps).  Forward losses are fixed-order sums: compared with the oracle's float64 sum to a relative 1e-5, and
with themselves bit for bit.  bf16 operands are rounded once on the host and the oracle runs on the rounded values."""
import zlib

import numpy as np
import pytest

import criteria_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
NAMES = ["mae", "bce", "bce_with_logits", "kldiv"]
EXACT_BWD = {"mae", "bce", "kldiv"}


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


def bf16_round(x):
    from oracle import bf16_round as r
    return r(np.asarray(x, F32))


def held(x, dt):
    x = np.asarray(x, F32)
    return bf16_round(x) if dt == "bf16" else x


def D(nk, dt):
    return nk.BF16 if dt == "bf16" else nk.F32


def bits_equal(got, want, what=""):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (what, f"{bad.size} of {got.size} differ", bad[0], got.ravel()[bad[0]], want.ravel()[bad[0]])


def operands(name, shape, rng):
    """x and t in each criterion's domain"""
    if name == "mae":
        return rng.standard_normal(shape).astype(F32), rng.standard_normal(shape).astype(F32)
    if name == "bce":
        return rng.uniform(0.01, 0.99, shape).astype(F32), rng.uniform(0, 1, shape).astype(F32)
    if name == "bce_with_logits":
        return (4 * rng.standard_normal(shape)).astype(F32), rng.uniform(0, 1, shape).astype(F32)
    t = rng.uniform(0, 1, shape).astype(F32)
    t[rng.uniform(0, 1, shape) < 0.1] = 0
    return np.log(rng.uniform(0.01, 1, shape)).astype(F32), t


def check_bwd(name, got, want, gdt, gscale=1.0):
    """bit for bit, or for bce_with_logits a few ulps of the result plus a few ulps of sigmoid(x) ~ 1 times the seed
    (`gscale` = |g| [/ n]): expf may round 1 + e^-x the other way"""
    if name in EXACT_BWD:
        bits_equal(got, held(want, gdt), name)
    else:
        ulp = 2.0 ** -7 if gdt == "bf16" else 2.0 ** -21
        assert np.all(np.abs(got - want) <= ulp * np.abs(want) + 2.0 ** -21 * gscale), name


# ------------------------------------------------------------------------------------------------ criteria, ops level
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dt,gdt", [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32")])
@pytest.mark.parametrize("mean", [True, False])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_criterion_ops_random(nk, dev, name, dt, gdt, mean, beta):
    from neuronika_b200 import ops
    rng = np.random.default_rng(zlib.crc32(repr((name, dt, gdt, mean, beta)).encode()))
    shape = (37, 129)
    x, t = (held(v, dt) for v in operands(name, shape, rng))
    xd, td = dev.from_ndarray(x, D(nk, dt)), dev.from_ndarray(t, D(nk, dt))
    loss = ops.criterion(name, xd, td, mean).as_ndarray()
    want = O.forward(name, x, t, mean)
    assert np.isclose(loss, want, rtol=1e-5, atol=1e-6), (name, loss, want)
    g = F32(rng.uniform(0.5, 2.0))
    dx0 = held(rng.standard_normal(shape), gdt)
    dx = dev.from_ndarray(dx0, D(nk, gdt))
    ops.criterion_bwd(name, dx, xd, td, dev.from_ndarray(np.array(g, F32)), mean, beta)
    expect = O.backward(name, x, t, g, mean)
    if beta:
        expect = (dx0 + expect).astype(F32)
    check_bwd(name, dx.as_ndarray(), expect, gdt, g / (O.divisor(name, shape) if mean else 1))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("off", [0, 1])
def test_criterion_lengths_and_alignment(nk, dev, name, off):
    """lengths around the 8-element vector, the grid-stride step and past one wave; starts 16-byte aligned (vector
    body) or one element in (scalar path)"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(5 + off)
    wave = dev.sm_count * 8 * 256 * 8
    for n in (1, 7, 8, 9, 4095, 4097, 8191, 8193, wave + 13):
        x, t = operands(name, (n,), rng)
        xb = dev.from_ndarray(np.concatenate([np.zeros(off, F32), x, np.zeros(8, F32)]))
        tb = dev.from_ndarray(np.concatenate([np.zeros(off, F32), t, np.zeros(8, F32)]))
        xd, td = xb.slice_flat(off, (n,)), tb.slice_flat(off, (n,))
        loss = ops.criterion(name, xd, td, False).as_ndarray()
        assert np.isclose(loss, O.forward(name, x, t, False), rtol=1e-5, atol=1e-6), (name, n, off)
        canary = np.full(n + off + 8, -7.0, F32)
        db = dev.from_ndarray(canary)
        ops.criterion_bwd(name, db.slice_flat(off, (n,)), xd, td, dev.from_ndarray(np.array(1.0, F32)), False, 0.0)
        out = db.as_ndarray()
        assert np.all(out[:off] == -7.0) and np.all(out[off + n:] == -7.0), (name, n, off)
        check_bwd(name, out[off:off + n], O.backward(name, x, t, 1.0, False), "f32")


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_criterion_forward_is_bitwise_repeatable(nk, dev, name, dt):
    from neuronika_b200 import ops
    rng = np.random.default_rng(8)
    x, t = operands(name, (1 << 22,), rng)
    xd, td = dev.from_ndarray(x, D(nk, dt)), dev.from_ndarray(t, D(nk, dt))
    a = ops.criterion(name, xd, td, True).as_ndarray()
    b = ops.criterion(name, xd, td, True).as_ndarray()
    assert a.view(np.uint32) == b.view(np.uint32)


def test_bce_clamps_and_kldiv_zero_targets(nk, dev):
    from neuronika_b200 import ops
    x = np.array([0.0, 1.0, 0.0, 1.0, 0.5], F32)
    t = np.array([1.0, 0.0, 0.0, 1.0, 0.5], F32)
    xd, td = dev.from_ndarray(x), dev.from_ndarray(t)
    assert np.isclose(ops.criterion("bce", xd, td, False).as_ndarray(), O.forward("bce", x, t, False), rtol=1e-6)
    dx = dev.zeros((5,))
    ops.criterion_bwd("bce", dx, xd, td, dev.from_ndarray(np.array(1.0, F32)), False, 0.0)
    bits_equal(dx.as_ndarray(), O.backward("bce", x, t, 1.0, False))
    assert dx.as_ndarray()[0] == -8388608.0 and dx.as_ndarray()[1] == 8388608.0
    t = np.array([[0.0, 0.0, 1.0], [0.0, 0.5, 0.5]], F32)
    lx = np.log(np.array([[0.2, 0.3, 0.5], [0.1, 0.6, 0.3]], F32))
    loss = ops.criterion("kldiv", dev.from_ndarray(lx), dev.from_ndarray(t), True).as_ndarray()
    assert np.isfinite(loss) and np.isclose(loss, O.forward("kldiv", lx, t, True), rtol=1e-6)


# ------------------------------------------------------------------------------------------------ criteria, graph
def golden_cases():
    import json
    import os
    import test_oracle_criteria as T
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tensors_criteria.json")) as fh:
        return T.reference_cases(json.load(fh))


@pytest.mark.parametrize("case", range(8))
def test_goldens_through_vardiff(nk, dev, case):
    """the reference's goldens through Var/VarDiff; a second backward() on the same tape doubles the gradient"""
    name, x, t, mean, loss, grad = golden_cases()[case]
    xv = nk.from_ndarray(dev, x).requires_grad()
    tv = nk.from_ndarray(dev, t)
    red = nk.Reduction.Mean if mean else nk.Reduction.Sum
    out = getattr(xv, name)(tv, red)
    assert out.history_len() == 1 and out.backward_history_len() == 1
    out.forward()
    assert abs(out.item() - loss) <= 1e-4 * max(1.0, abs(loss)), (name, out.item(), loss)
    out.backward(1.0)
    g1 = xv.grad()
    assert np.all(np.abs(g1 - grad) <= 1e-4 * np.maximum(1.0, np.abs(grad))), (name, g1, grad)
    check_bwd(name, g1, O.backward(name, x, t, 1.0, mean), "f32", 1.0 / (O.divisor(name, x.shape) if mean else 1))
    out.backward(1.0)
    bits_equal(xv.grad(), (g1 + g1).astype(F32), name + " second backward")
    # a Var input records a forward node and no backward node
    v = getattr(nk.from_ndarray(dev, x), name)(tv, red)
    assert not isinstance(v, nk.VarDiff)
    v.forward()
    assert v.item() == out.item()


@pytest.mark.parametrize("name", NAMES)
def test_graph_bf16_data_f32_gradient(nk, dev, name):
    rng = np.random.default_rng(11)
    x, t = (bf16_round(v) for v in operands(name, (24, 40), rng))
    xv = nk.from_ndarray(dev, x, nk.BF16).requires_grad(nk.F32)
    loss = getattr(xv, name)(nk.from_ndarray(dev, t, nk.BF16))
    loss.forward()
    loss.backward(2.0)
    assert xv.grad_dtype == nk.F32
    check_bwd(name, xv.grad(), O.backward(name, x, t, 2.0, True), "f32", 2.0 / O.divisor(name, x.shape))
    assert np.isclose(loss.item(), O.forward(name, x, t, True), rtol=1e-5, atol=1e-6)


def test_graph_criterion_errors(nk, dev):
    a = nk.from_ndarray(dev, np.zeros((3, 4), F32)).requires_grad()
    with pytest.raises(nk.NkError, match="shapes differ"):
        a.bce(nk.from_ndarray(dev, np.zeros((4, 3), F32)))
    with pytest.raises(nk.NkError, match="element types"):
        a.mae(nk.from_ndarray(dev, np.zeros((3, 4), F32), nk.BF16))
    with pytest.raises(nk.NkError, match="not be differentiable"):
        a.kldiv(a)


# ------------------------------------------------------------------------------------------------ dropout, ops level
def mask_array(dev, n):
    return dev.zeros(((n + 31) // 32,))


def mask_words(m):
    return m.as_ndarray().view(np.uint32)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("off", [0, 1])
def test_dropout_mask_and_values_match_the_oracle(nk, dev, dt, off):
    """mask bit for bit for (seed, call id) at lengths that are not multiples of 4 or 32, y bit for bit; the call id
    advances by one per drawing forward"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(2)
    seed, p = 0x5EED0000ABCD + off, 0.3
    dev.manual_seed(seed)
    assert dev.rng_state() == (seed, 0)
    call = 0
    for n in (1, 3, 5, 31, 33, 127, 129, 1000, 4099, dev.sm_count * 8 * 256 * 4 + 37):
        x = held(rng.standard_normal(n) + 0.1, dt)
        xb = dev.from_ndarray(np.concatenate([np.zeros(off, F32), x, np.zeros(4, F32)]), D(nk, dt))
        y = dev.zeros((n + off + 4,), D(nk, dt))
        m = mask_array(dev, n)
        ops.dropout(xb.slice_flat(off, (n,)), p, m, out=y.slice_flat(off, (n,)))
        keep = O.dropout_keep(seed, call, n, p)
        assert np.array_equal(mask_words(m), O.pack_mask(keep)), (n, off)
        yh = y.as_ndarray()
        bits_equal(yh[off:off + n], held(O.dropout_forward(x, keep, p), dt), f"y n={n}")
        assert np.all(yh[:off] == 0) and np.all(yh[off + n:] == 0)
        call += 1
        assert dev.rng_state() == (seed, call)


@pytest.mark.parametrize("dt,gdt", [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32")])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_dropout_backward_given_the_mask(nk, dev, dt, gdt, beta):
    from neuronika_b200 import ops
    rng = np.random.default_rng(4)
    for n in (1, 9, 1000, 70001):
        p = 0.4
        keep = rng.uniform(0, 1, n) < 0.6
        m = dev.from_ndarray(O.pack_mask(keep).view(F32))
        g = held(rng.standard_normal(n), dt)
        dx0 = held(rng.standard_normal(n), gdt)
        dx = dev.from_ndarray(dx0, D(nk, gdt))
        ops.dropout_bwd(dx, m, dev.from_ndarray(g, D(nk, dt)), p, beta)
        want = O.dropout_backward(g, keep, p)
        if beta:
            want = (dx0 + want).astype(F32)
        bits_equal(dx.as_ndarray(), held(want, gdt), f"n={n}")
        # p = 0 and a NULL mask: the identity; p = 1: nothing
        for pp, mm, w in ((0.0, m, g), (0.4, None, g), (1.0, m, np.zeros(n, F32))):
            dx = dev.from_ndarray(dx0, D(nk, gdt))
            ops.dropout_bwd(dx, mm, dev.from_ndarray(g, D(nk, dt)), pp, beta)
            bits_equal(dx.as_ndarray(), held((dx0 + w) if beta else w, gdt), f"p={pp}")


def test_dropout_p0_p1_draw_nothing(nk, dev):
    from neuronika_b200 import ops
    dev.manual_seed(1)
    x = dev.from_ndarray(np.arange(1, 100, dtype=F32))
    bits_equal(ops.dropout(x, 0.0).as_ndarray(), np.arange(1, 100, dtype=F32))
    bits_equal(ops.dropout(x, 1.0).as_ndarray(), np.zeros(99, F32))
    assert dev.rng_state() == (1, 0)
    with pytest.raises(nk.NkError, match="Wrong probability"):
        ops.dropout(x, 1.5, mask_array(dev, 99))


def test_dropout_past_2_31_elements_bf16(nk, dev):
    """one bf16 dropout over 2^31 + 4099 elements: keep rate within 6 sigma, and spot elements (around 2^31 and at the
    end) against the oracle"""
    import torch
    from neuronika_b200 import ops
    n, p, seed = (1 << 31) + 4099, 0.25, 77
    xt = torch.full((n,), 1.5, dtype=torch.bfloat16, device="cuda")
    yt = torch.empty_like(xt)
    mt = torch.zeros(((n + 31) // 32,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    wrap = lambda t, d: nk.CuArray(dev, (t.numel(),), d, ptr=t.data_ptr(), owner=t)
    dev.manual_seed(seed)
    ops.dropout(wrap(xt, nk.BF16), p, wrap(mt, nk.F32), out=wrap(yt, nk.BF16))
    dev.synchronize()
    kept = int(torch.count_nonzero(yt).item())
    q = float(O.keep_prob(p))
    assert abs(kept - n * q) <= 6 * np.sqrt(n * q * (1 - q)), kept
    idx = np.concatenate([np.arange(5), (1 << 31) - 3 + np.arange(8), n - 7 + np.arange(7)]).astype(np.int64)
    keep = O.dropout_keep(seed, 0, n, p, elements=idx)
    words = mt[torch.tensor(idx // 32, device="cuda")].cpu().numpy().view(np.uint32)
    assert np.array_equal(((words >> (idx % 32).astype(np.uint32)) & 1).astype(bool), keep)
    ys = yt[torch.tensor(idx, device="cuda")].float().cpu().numpy()
    bits_equal(ys, np.where(keep, bf16_round(np.float32(1.5) / O.keep_prob(p)), 0).astype(F32))
    del xt, yt, mt
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ dropout, graph
def test_graph_dropout_paths(nk, dev):
    """train draws (y = x/q or 0, a new mask per forward), eval copies, p = 0 copies, p = 1 zeros; the backward applies
    what the forward did even after the status changed"""
    dev.manual_seed(5)
    n = 300
    x = np.linspace(1, 2, n, dtype=F32)
    xv = nk.from_ndarray(dev, x).requires_grad()
    st = nk.Status()
    y = xv.dropout(0.5, st)
    assert y.history_len() == 1 and y.backward_history_len() == 1
    y.forward()
    k0 = O.dropout_keep(5, 0, n, 0.5)
    bits_equal(y.data(), O.dropout_forward(x, k0, 0.5))
    st.eval()                      # the backward still applies the forward's mask
    y.backward(1.0)
    bits_equal(xv.grad(), O.dropout_backward(np.ones(n, F32), k0, 0.5))
    y.forward()                    # eval: a copy, no draw
    bits_equal(y.data(), x)
    assert dev.rng_state() == (5, 1)
    xv.zero_grad()
    y.backward(1.0)
    bits_equal(xv.grad(), np.ones(n, F32))
    st.train()
    y.forward()
    y.forward()                    # two forwards, two different masks
    k2 = O.dropout_keep(5, 2, n, 0.5)
    assert not np.array_equal(O.dropout_keep(5, 1, n, 0.5), k2)
    bits_equal(y.data(), O.dropout_forward(x, k2, 0.5))
    for p, want in ((0.0, x), (1.0, np.zeros(n, F32))):
        z = xv.dropout(p, st)
        z.forward()
        bits_equal(z.data(), want)
    assert dev.rng_state() == (5, 3)
    m = nk.nn.Dropout(0.5)
    m.eval()
    z = m.forward(xv)
    z.forward()
    bits_equal(z.data(), x)
    assert m.status.get() is False


def test_graph_dropout_rejects_bad_p(nk, dev):
    xv = nk.from_ndarray(dev, np.ones(8, F32)).requires_grad()
    before = xv.history_len()
    for p in (-0.5, 1.5, float("nan")):
        with pytest.raises(nk.NkError, match="Wrong probability received"):
            xv.dropout(p, nk.Status())
    assert xv.history_len() == before
    with pytest.raises(ValueError, match="Wrong probability"):
        nk.nn.Dropout(2.0)


def test_captured_dropout_draws_a_new_mask_per_replay(nk, dev):
    """seed s, one eager step, capture, two replays; reseed s, three eager steps: the three masks match pairwise, bit for
    bit, the two replays differ, and each equals the oracle's mask for its call id"""
    n, p, s = 5000, 0.5, 0xC0FFEE
    x = nk.from_ndarray(dev, np.ones(n, F32))
    st = nk.Status()
    y = x.dropout(p, st)

    def mask():
        return y.data() != 0

    dev.manual_seed(s)
    y.forward()
    first = [mask()]
    with dev.capture(64 << 20) as cap:
        y.forward()
    for _ in range(2):
        cap.graph.launch()
        dev.synchronize()
        first.append(mask())
    assert dev.rng_state() == (s, 3)
    dev.manual_seed(s)
    again = []
    for _ in range(3):
        y.forward()
        again.append(mask())
    for k in range(3):
        assert np.array_equal(first[k], again[k]), k
        assert np.array_equal(first[k], O.dropout_keep(s, k, n, p)), k
    assert not np.array_equal(first[1], first[2])
    with dev.capture(1 << 20) as cap2:
        y.forward()
        with pytest.raises(nk.NkError, match="cannot be captured"):
            dev.manual_seed(1)
    cap.graph.close()
    cap2.graph.close()


def test_captured_mlp_with_dropout_and_bce_with_logits_matches_torch(nk, dev):
    """Linear(8 -> 16) -> ReLU -> dropout(0.5) -> Linear(16 -> 1) -> bce_with_logits, SGD: one eager step, then the step
    captured and replayed three times; against torch CPU autograd on the same weights fed the oracle's masks"""
    import torch
    from neuronika_b200 import optim
    rng = np.random.default_rng(17)
    nb, lr, seed = 64, 0.5, 2024
    l1 = nk.nn.Linear(dev, 8, 16, rng=rng)
    l2 = nk.nn.Linear(dev, 16, 1, rng=rng)
    drop = nk.nn.Dropout(0.5)
    params = l1.parameters() + l2.parameters()
    init = [p.data().copy() for p in params]
    opt = optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)
    xh = rng.standard_normal((nb, 8)).astype(F32)
    th = (rng.uniform(0, 1, (nb, 1)) < 0.5).astype(F32)
    x, t = nk.from_ndarray(dev, xh), nk.from_ndarray(dev, th)
    losses = []

    def step():
        opt.zero_grad()
        loss = l2.forward(drop.forward(l1.forward(x).relu())).bce_with_logits(t)
        loss.forward()
        loss.backward(1.0)
        opt.step()
        losses.append(loss)

    dev.manual_seed(seed)
    step()
    with dev.capture(64 << 20) as cap:
        step()
    replays = []
    for _ in range(3):
        cap.graph.launch()
        replays.append(losses[-1].item())
    assert cap.graph.kernel_count > 0
    got = [p.data() for p in params]

    w = [torch.tensor(v, requires_grad=True) for v in init]
    xt, tt = torch.tensor(xh), torch.tensor(th)
    want_losses = []
    for call in range(4):
        keep = torch.tensor(O.dropout_keep(seed, call, nb * 16, 0.5).reshape(nb, 16))
        h = torch.relu(xt @ w[0].T + w[1])
        d = torch.where(keep, h / torch.tensor(O.keep_prob(0.5)), torch.zeros(()))
        z = d @ w[2].T + w[3]
        loss = torch.nn.functional.binary_cross_entropy_with_logits(z, tt)
        for v in w:
            v.grad = None
        loss.backward()
        want_losses.append(loss.item())
        with torch.no_grad():
            for v in w:
                v -= lr * v.grad
    for a, b in zip(got, w):
        np.testing.assert_allclose(a, b.detach().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(replays, want_losses[1:], rtol=1e-4, atol=1e-5)
    cap.graph.close()
