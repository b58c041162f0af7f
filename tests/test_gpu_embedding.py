"""Embedding on the GPU (csrc/nk_embedding.cu): nk_embedding_fwd / nk_embedding_bwd bit-equal to the numpy oracle of
tests/embedding_oracle.py (which restates the backward's summation order) for every (w, g, dw) dtype combination and
both id dtypes; row lengths around the 16-byte access widths with misaligned bases; v on each side of the radix sort's
pass boundaries; n = 0 and 1 and more positions than one grid pass; uniform, Zipf, all-distinct and all-equal ids;
invalid ids, padding_idx and beta 0 / 0.5 / 1; an output over 2^31 elements.  Also: repeated calls bitwise equal,
launch counts, argument errors, nn.Embedding and a tied embedding / head weight against torch CUDA, a second backward,
and a captured language-model step (Embedding -> LSTM -> reshape -> Linear -> log_softmax -> nll, SGD) against torch
and replayed bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import embedding_oracle as E

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


def bf16r(a):
    import neuronika_b200._lib as L
    return L.bf16_bits_to_f32(L.f32_to_bf16_bits(np.asarray(a, F32N)))


def rnd(name, a):
    return bf16r(a) if name == "bf16" else np.asarray(a, F32N)


def put(nk, dev, a, dtype, offset=0):
    """a device copy of `a` in `dtype`; offset > 0 places it that many elements after a 16-byte aligned allocation"""
    if offset == 0:
        return dev.from_ndarray(a, dt(nk, dtype))
    base = dev.zeros((a.size + offset,), dt(nk, dtype))
    view = base.slice_flat(offset, a.shape)
    view.copy_from(a)
    view._base = base
    return view


def same(got, want, what=""):
    got, want = np.asarray(got, F32N), np.asarray(want, F32N)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (what, np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])


def make_ids(kind, rng, n, v, invalid=False):
    if kind == "uniform":
        ids = rng.integers(0, v, n).astype(F32N)
    elif kind == "zipf":
        ids = np.minimum(rng.zipf(1.3, n) - 1, v - 1).astype(F32N)
    elif kind == "equal":
        ids = np.full(n, (v - 1) // 2, F32N)
    else:
        ids = rng.permutation(v)[:n].astype(F32N)
    if invalid and n > 8:
        ids = ids + F32N(0.25) * (ids < v - 1)          # truncated to the same row
        ids[rng.choice(n, n // 9, replace=False)] = rng.choice(np.array([-1, -0.5, v, v + 0.5, np.nan, np.inf],
                                                                        F32N), n // 9)
    return ids


def run_bwd(nk, dev, ids, g, dw0, v, e, wdt, gdt, idt, pad=-1, beta=0.0, offset=0):
    I = put(nk, dev, ids, idt)
    G = put(nk, dev, g, gdt, offset)
    DW = put(nk, dev, dw0, wdt, offset)
    nk.ops.embedding_bwd(DW, I, G, padding_idx=None if pad < 0 else pad, beta=beta)
    want = E.backward(dw0, ids, rnd(gdt, g), padding_idx=pad, beta=beta,
                      round_out=bf16r if wdt == "bf16" else None)
    return DW.as_ndarray(), want


# ---------------------------------------------------------------------------------------------- bit for bit
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("e", [1, 7, 8, 9, 650, 768, 4096])
@pytest.mark.parametrize("idt", ["f32", "bf16"])
@pytest.mark.parametrize("wdt", ["f32", "bf16"])
def test_forward_bits(nk, dev, wdt, idt, e, offset):
    rng = np.random.default_rng(e * 7 + offset)
    v, n = 200, 300
    w = rnd(wdt, rng.standard_normal((v, e)))
    ids = make_ids("uniform", rng, n, v, invalid=True)
    if idt == "bf16":
        ids = bf16r(ids)
    W = put(nk, dev, w, wdt, offset)
    Y = put(nk, dev, np.zeros((n, e), F32N), wdt, offset)
    nk.ops.embedding(W, put(nk, dev, ids, idt), out=Y)
    same(Y.as_ndarray(), E.forward(w, ids))


@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("e", [1, 7, 8, 9, 650, 768, 4096])
@pytest.mark.parametrize("idt", ["f32", "bf16"])
@pytest.mark.parametrize("pair", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
def test_backward_bits(nk, dev, pair, idt, e, offset, beta):
    wdt, gdt = pair
    rng = np.random.default_rng(e * 13 + offset)
    v, n = 200, 700 if e < 4096 else 150
    ids = make_ids("zipf", rng, n, v, invalid=True)
    if idt == "bf16":
        ids = bf16r(ids)
    g = rnd(gdt, rng.standard_normal((n, e)))
    dw0 = rnd(wdt, rng.standard_normal((v, e)))
    got, want = run_bwd(nk, dev, ids, g, dw0, v, e, wdt, gdt, idt, pad=3 if e % 2 else -1, beta=beta, offset=offset)
    same(got, want)


@pytest.mark.parametrize("v", [255, 256, 257, 65535, 65536, 65537, 1 << 24])
def test_radix_pass_boundaries(nk, dev, v):
    rng = np.random.default_rng(v % 1000)
    n, e = 5000, 3
    ids = make_ids("uniform", rng, n, v)
    ids[:40] = v - 1
    ids[40:80] = 0
    g = rng.standard_normal((n, e)).astype(F32N)
    got, want = run_bwd(nk, dev, ids, g, np.ones((v, e), F32N), v, e, "f32", "f32", "f32", beta=0.0)
    same(got, want)
    w = rng.standard_normal((v, e)).astype(F32N) if v <= 65537 else np.zeros((v, e), F32N) + F32N(2.5)
    y = nk.ops.embedding(dev.from_ndarray(w), dev.from_ndarray(ids))
    same(y.as_ndarray(), E.forward(w, ids))


@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("n", [0, 1])
def test_zero_and_one_position(nk, dev, n, beta):
    rng = np.random.default_rng(n)
    v, e = 40, 9
    ids = np.array([5.0], F32N)[:n]
    g = rng.standard_normal((max(n, 1), e)).astype(F32N)[:n]
    dw0 = rng.standard_normal((v, e)).astype(F32N)
    I = dev.from_ndarray(ids if n else np.zeros(1, F32N)).slice_flat(0, (n,))
    G = dev.from_ndarray(g if n else np.zeros((1, e), F32N)).slice_flat(0, (n, e))
    DW = dev.from_ndarray(dw0)
    before = dev.launches
    nk.ops.embedding_bwd(DW, I, G, beta=beta)
    assert dev.launches - before == (0 if (n == 0 and beta == 1.0) else (1 if n == 0 else 4 + (beta != 1.0)))
    same(DW.as_ndarray(), E.backward(dw0, ids, g, beta=beta))
    W = dev.from_ndarray(dw0)
    Y = dev.zeros((1, e), nk.F32).slice_flat(0, (n, e))
    before = dev.launches
    nk.ops.embedding(W, I, out=Y)
    assert dev.launches - before == n
    if n:
        same(Y.as_ndarray(), E.forward(dw0, ids))


@pytest.mark.parametrize("kind", ["uniform", "zipf", "distinct", "equal"])
def test_id_distributions(nk, dev, kind):
    """2^20 positions; all-equal ids put one row over 32768 slots"""
    rng = np.random.default_rng(11)
    n, e = 1 << 20, 8
    v = n if kind == "distinct" else 50000
    ids = make_ids(kind, rng, n, v)
    g = rng.standard_normal((n, e)).astype(F32N)
    got, want = run_bwd(nk, dev, ids, g, np.zeros((v, e), F32N), v, e, "f32", "f32", "f32", beta=0.0)
    same(got, want)


def test_more_positions_than_one_grid_pass(nk, dev):
    rng = np.random.default_rng(12)
    n, v, e = 9_000_000, 1000, 1
    ids = make_ids("uniform", rng, n, v)
    g = rng.integers(-8, 9, (n, e)).astype(F32N)
    got, want = run_bwd(nk, dev, ids, g, np.zeros((v, e), F32N), v, e, "f32", "f32", "f32", beta=0.0)
    same(got, want)
    w = rng.standard_normal((v, e)).astype(F32N)
    same(nk.ops.embedding(dev.from_ndarray(w), dev.from_ndarray(ids)).as_ndarray(), E.forward(w, ids))


def test_output_over_2_31_elements(nk, dev):
    rng = np.random.default_rng(13)
    v, e = 64, 4096
    n = (1 << 19) + 100                                 # n * e = 2^31 + 409600
    w = bf16r(rng.standard_normal((v, e)))
    ids = make_ids("uniform", rng, n, v, invalid=True)
    Y = nk.ops.embedding(dev.from_ndarray(w, nk.BF16), dev.from_ndarray(ids))
    for p0 in (0, (1 << 19) - 7, n - 50):
        rows = Y.slice_flat(p0 * e, (min(50, n - p0), e)).as_ndarray()
        same(rows, E.forward(w, ids[p0:p0 + rows.shape[0]]), p0)
    del Y


# ---------------------------------------------------------------------------------------------- behaviour
def test_repeated_calls_are_bitwise_equal(nk, dev):
    rng = np.random.default_rng(14)
    n, v, e = 50000, 10000, 768
    ids = make_ids("zipf", rng, n, v)
    I, G = dev.from_ndarray(ids), dev.from_ndarray(rng.standard_normal((n, e)).astype(F32N))
    outs = []
    for _ in range(2):
        DW = dev.zeros((v, e), nk.F32)
        nk.ops.embedding_bwd(DW, I, G, beta=0.0)
        outs.append(DW.as_ndarray())
    same(outs[0], outs[1])


@pytest.mark.parametrize("v, beta, n, want", [(200, 0.0, 700, 5), (200, 1.0, 20, 4), (200, 1.0, 700, 5),
                                              (65536, 1.0, 700, 11), (1 << 24, 0.0, 100, 14)])
def test_launch_counts(nk, dev, v, beta, n, want):
    e = 4
    I = dev.from_ndarray(np.zeros(n, F32N))
    G = dev.zeros((n, e), nk.F32)
    DW = dev.zeros((v, e), nk.F32)
    before = dev.launches
    nk.ops.embedding_bwd(DW, I, G, beta=beta)
    assert dev.launches - before == want
    before = dev.launches
    nk.ops.embedding(DW, I)
    assert dev.launches - before == 1


def test_argument_errors(nk, dev):
    G = dev.zeros((4, 3), nk.F32)
    with pytest.raises(nk.NkError, match="bf16 id table"):
        nk.ops.embedding(dev.zeros((257, 3), nk.F32), dev.zeros((4,), nk.BF16))
    with pytest.raises(nk.NkError, match="2\\^24"):
        nk.ops.embedding_bwd(dev.zeros(((1 << 24) + 1, 1), nk.F32), dev.zeros((4,), nk.F32), dev.zeros((4, 1)))
    with pytest.raises(nk.NkError, match="padding_idx"):
        nk.ops.embedding_bwd(dev.zeros((10, 3), nk.F32), dev.zeros((4,), nk.F32), G, padding_idx=10)


# ---------------------------------------------------------------------------------------------- modules
def test_nn_embedding_against_torch(nk, dev):
    rng = np.random.default_rng(15)
    v, e = 300, 24
    emb = nk.nn.Embedding(dev, v, e, padding_idx=-2, rng=rng)
    w0 = emb.weight.data().copy()
    assert not w0[v - 2].any() and emb.padding_idx == v - 2
    ids = rng.integers(0, v, (5, 7)).astype(F32N)
    ids[0, :3] = v - 2
    y = emb.forward(nk.from_ndarray(dev, ids))
    assert y.shape == (5, 7, e)
    loss = (y * y).sum()
    loss.forward()
    loss.backward(1.0)
    tw = torch.tensor(w0, device="cuda", requires_grad=True)
    ty = F.embedding(torch.tensor(ids.astype(np.int64), device="cuda"), tw, padding_idx=-2)
    (ty * ty).sum().backward()
    same(y.data(), ty.detach().cpu().numpy())
    np.testing.assert_allclose(emb.weight.grad(), tw.grad.cpu().numpy(), rtol=1e-5, atol=1e-5)
    assert not emb.weight.grad()[v - 2].any()
    # backward() from the embedding's own output, twice: the second pass accumulates into the leaf gradient
    y2 = emb.forward(nk.from_ndarray(dev, ids))
    y2.forward()
    emb.weight.zero_grad()
    y2.backward(1.0)
    g1 = emb.weight.grad().copy()
    counts = np.bincount(ids.reshape(-1).astype(np.int64), minlength=v).astype(F32N)
    counts[v - 2] = 0
    same(g1, np.repeat(counts[:, None], e, 1))
    y2.backward(1.0)
    same(emb.weight.grad(), 2 * g1)
    with pytest.raises(ValueError):
        nk.nn.Embedding(dev, v, e, padding_idx=v)


def test_tied_embedding_and_head_weight(nk, dev):
    rng = np.random.default_rng(16)
    v, e, n = 120, 16, 40
    w = rng.standard_normal((v, e)).astype(F32N) * F32N(0.3)
    ids = rng.integers(0, v, n).astype(F32N)
    t = rng.integers(0, v, n).astype(F32N)
    W = nk.from_ndarray(dev, w).requires_grad()
    h = nk.variable.embedding(nk.from_ndarray(dev, ids), W)
    loss = h.mm_t(W).log_softmax(1).nll_loss(nk.from_ndarray(dev, t))
    loss.forward()
    loss.backward(1.0)
    tw = torch.tensor(w, device="cuda", requires_grad=True)
    tl = F.nll_loss(F.log_softmax(F.embedding(torch.tensor(ids.astype(np.int64), device="cuda"), tw) @ tw.T, 1),
                    torch.tensor(t.astype(np.int64), device="cuda"))
    tl.backward()
    np.testing.assert_allclose(loss.item(), tl.item(), rtol=1e-5)
    np.testing.assert_allclose(W.grad(), tw.grad.cpu().numpy(), rtol=1e-4, atol=1e-6)


def test_reshape_shares_the_gradient(nk, dev):
    rng = np.random.default_rng(18)
    x = rng.standard_normal((3, 4, 5)).astype(F32N)
    X = nk.from_ndarray(dev, x).requires_grad()
    y = X.reshape(-1, 5)
    assert y.shape == (12, 5)
    loss = (y * y).sum()
    loss.forward()
    loss.backward(1.0)
    np.testing.assert_allclose(X.grad(), 2 * x, rtol=1e-6)
    with pytest.raises(RuntimeError, match=r"shape '\[7, -1\]' is invalid for input of size 60"):
        X.reshape(7, -1)
    with pytest.raises(RuntimeError, match="only one dimension can be inferred"):
        X.reshape(-1, -1)


def test_captured_language_model_step(nk, dev):
    """Embedding -> LSTM -> reshape(T*N, H) -> Linear -> log_softmax -> nll, SGD in f32: the first eager step against
    torch CUDA, then one step captured and replayed 5 times, equal to 5 eager steps bit for bit"""
    rng = np.random.default_rng(19)
    V, E_, H, T, N = 500, 32, 32, 7, 8
    emb = nk.nn.Embedding(dev, V, E_, rng=rng)
    lstm = nk.nn.LSTM(dev, E_, H, rng=rng)
    head = nk.nn.Linear(dev, H, V, rng=rng)
    params = emb.parameters() + lstm.parameters() + head.parameters()
    init = [p.data().copy() for p in params]
    ids = rng.integers(0, V, (T, N)).astype(F32N)
    tgt = rng.integers(0, V, T * N).astype(F32N)
    I, TG = nk.from_ndarray(dev, ids), nk.from_ndarray(dev, tgt)
    c0, h0 = nk.zeros(dev, (N, H)), nk.zeros(dev, (N, H))
    lr = 0.5
    opt = nk.optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)

    def step():
        opt.zero_grad()
        out, _ = lstm.forward((c0, h0), emb.forward(I))
        loss = head.forward(out.reshape(T * N, H)).log_softmax(1).nll_loss(TG)
        loss.forward()
        loss.backward(1.0)
        opt.step()

    eager = []
    for _ in range(5):
        step()
        eager.append([p.data().copy() for p in params])
    # torch CUDA, one step from the same weights
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    tl = torch.nn.LSTM(E_, H).cuda()
    with torch.no_grad():
        for q, v in zip((tl.weight_ih_l0, tl.weight_hh_l0, tl.bias_ih_l0, tl.bias_hh_l0), init[1:5]):
            q.copy_(torch.from_numpy(v))
    tw = [torch.tensor(init[0], device="cuda", requires_grad=True), tl.weight_ih_l0, tl.weight_hh_l0, tl.bias_ih_l0,
          tl.bias_hh_l0] + [torch.tensor(v, device="cuda", requires_grad=True) for v in init[5:]]
    x = F.embedding(torch.tensor(ids.astype(np.int64), device="cuda"), tw[0])
    o, _ = tl(x)
    loss = F.nll_loss(F.log_softmax(o.reshape(T * N, H) @ tw[5].T + tw[6], 1),
                      torch.tensor(tgt.astype(np.int64), device="cuda"))
    loss.backward()
    for got, p0, q in zip(eager[0], init, tw):
        np.testing.assert_allclose(got, (torch.tensor(p0, device="cuda") - lr * q.grad).cpu().numpy(), rtol=1e-4,
                                   atol=2e-5)
    # replay
    for p, v in zip(params, init):
        p.set_data(v)
    dev.synchronize()
    with dev.capture(256 << 20) as cap:
        step()
    for r in range(5):
        cap.graph.launch()
        dev.synchronize()
        for p, want in zip(params, eager[r]):
            same(p.data(), want, r)
