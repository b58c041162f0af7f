"""Cross-entropy on the GPU (csrc/nk_cross_entropy.cu) against the float64 oracle of tests/cross_entropy_oracle.py on
the same rounded inputs: the loss within 1e-5 relative; every dx element within 2e-6*B (f32 dx) or 2^-8*B (bf16 dx) of
beta*dx0 + the oracle's gradient, B = |g|*max(w)*s the largest value a gradient element can take (B + |beta|*max|dx0|
when beta != 0, the largest value the accumulated result can take).  Every (x, dx) dtype
pair and both target dtypes; C around the vector width and the warp / CTA row threshold with misaligned bases; rows
split over CTAs; spatial inputs; N = 0 and 1; weights, label smoothing, ignore_index, invalid ids; beta 0 / 0.5 / 1;
n*c > 2^31; repeated calls bitwise equal in every layout; the f32 composition log_softmax -> nll_loss; the bf16 precision
at the language-model shape; a captured Linear -> cross_entropy -> SGD step with targets changed between replays."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cross_entropy_oracle as O

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
    a = np.asarray(a, F32N)
    if offset == 0:
        return dev.from_ndarray(a, dt(nk, dtype))
    base = dev.zeros((a.size + offset,), dt(nk, dtype))
    view = base.slice_flat(offset, a.shape)
    view.copy_from(a)
    view._base = base
    return view


def make_targets(rng, shape, c, tdt, ignore_index=-100, ignore_frac=0.0, invalid=False):
    t = rng.integers(0, c, shape).astype(F32N)
    if ignore_frac:
        t = np.where(rng.random(shape) < ignore_frac, F32N(ignore_index), t)
    if invalid and t.size > 8:
        flat = t.reshape(-1)
        pick = rng.choice(flat.size, max(1, flat.size // 9), replace=False)
        flat[pick] = rng.choice(np.array([-1, -0.5, c, c + 0.5, np.nan, np.inf], F32N), pick.size)
        if tdt == "f32":
            flat += F32N(0.25) * (flat < c - 1) * (flat >= 0)          # truncated to the same class
    return rnd(tdt, t)


def run(nk, dev, x, t, xdt, ddt, tdt, w=None, mean=True, ig=-100, eps=0.0, beta=0.0, g=1.0, off=0, seed=0):
    """forward + backward on the device; checks against the oracle; returns (loss, dx) as host arrays"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    X, T = put(nk, dev, x, xdt, off), put(nk, dev, t, tdt, off)
    W = put(nk, dev, w, "f32") if w is not None else None
    loss, lse, denom = ops.cross_entropy(X, T, W, mean, ig, eps)
    want_loss, _, want_den = O.forward(x, t, w, mean, ig, eps)
    got = float(loss.as_ndarray())
    if np.isnan(want_loss):
        assert np.isnan(got)
    elif np.isinf(want_loss):
        assert got == want_loss
    else:
        assert abs(got - want_loss) <= 1e-5 * abs(want_loss) + 1e-30, (got, want_loss)
    assert float(denom.as_ndarray()) == pytest.approx(want_den, rel=1e-6)
    scale = (1.0 / want_den if want_den else 0.0) if mean else 1.0
    B = O.grad_bound(g, w, scale)
    d0 = rnd(ddt, rng.uniform(-1, 1, x.shape) * max(B, 1e-30))
    DX = put(nk, dev, d0, ddt, off)
    G = dev.from_ndarray(np.array(g, F32N))
    ops.cross_entropy_bwd(DX, X, T, lse, denom, G, W, mean, ig, eps, beta)
    dx = DX.as_ndarray()
    want = beta * d0.astype(np.float64) + O.backward(x, t, g, w, mean, ig, eps)
    # rounding dx to its type is relative to |beta*dx0 + grad| <= |beta|*max|dx0| + B
    tol = (2e-6 if ddt == "f32" else 2.0 ** -8) * (B + abs(beta) * float(np.abs(d0).max(initial=0.0)))
    err = np.abs(dx - want)
    assert err.max(initial=0.0) <= tol, (err.max(), tol, np.unravel_index(err.argmax(), err.shape))
    return got, dx


DTYPES = [(x, d, t) for x in ("f32", "bf16") for d in ("f32", "bf16") for t in ("f32", "bf16")]


@pytest.mark.parametrize("xdt,ddt,tdt", DTYPES)
@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
def test_dtype_pairs_weights_smoothing_ignore(nk, dev, xdt, ddt, tdt, beta):
    rng = np.random.default_rng(1)
    n, c = 300, 200
    x = rnd(xdt, rng.standard_normal((n, c)) * 2)
    t = make_targets(rng, (n,), c, tdt, 3, 0.2, invalid=True)
    w = rng.uniform(0.25, 2.0, c).astype(F32N)
    for mean in (True, False):
        run(nk, dev, x, t, xdt, ddt, tdt, w, mean, 3, 0.1, beta, g=0.75)
        run(nk, dev, x, t, xdt, ddt, tdt, None, mean, 3, 0.0, beta, g=1.5)


# warp rows up to 4096 bytes (1024 f32 / 2048 bf16 classes), CTA rows above; C around the 8-element vector width
CLASSES = {"f32": [1, 2, 7, 8, 9, 1023, 1024, 1025, 1032], "bf16": [1, 2, 7, 8, 9, 2047, 2048, 2049, 2056, 3000]}


@pytest.mark.parametrize("xdt", ["f32", "bf16"])
@pytest.mark.parametrize("off", [0, 1, 3])
def test_class_counts_layouts_and_alignment(nk, dev, xdt, off):
    rng = np.random.default_rng(2 + off)
    for c in CLASSES[xdt]:
        for n in (1, 37):
            x = rnd(xdt, rng.standard_normal((n, c)) * 3)
            t = make_targets(rng, (n,), c, "f32", 0, 0.1)
            run(nk, dev, x, t, xdt, "f32", "f32", None, True, 0, 0.0, 0.5, off=off)
            run(nk, dev, x, t, xdt, xdt, "f32", rng.uniform(0.5, 1.5, c).astype(F32N), False, 0, 0.2, 0.0, off=off)


@pytest.mark.parametrize("xdt,ddt", [("bf16", "f32"), ("bf16", "bf16"), ("f32", "f32")])
def test_rows_split_over_ctas(nk, dev, xdt, ddt):
    rng = np.random.default_rng(4)
    for n, c in ((16, 262144), (3, 70001)):
        x = rnd(xdt, rng.standard_normal((n, c)) * 2)
        t = make_targets(rng, (n,), c, "f32", 5, 0.0)
        t[1] = 5                                                         # one ignored row
        run(nk, dev, x, t, xdt, ddt, "f32", None, True, 5, 0.0, 0.0)
        run(nk, dev, x, t, xdt, ddt, "f32", rng.uniform(0.5, 1.5, c).astype(F32N), True, 5, 0.1, 1.0)


@pytest.mark.parametrize("shape", [(100000, 5, 3), (70, 4, 64, 64), (6, 19, 4096), (50, 7, 1)],
                         ids=lambda s: "x".join(map(str, s)))
def test_spatial(nk, dev, shape):
    """S = 3, 4096 and 1 (an (N, C, 1) input), with more positions than one grid pass (8 CTAs of 256 per SM)"""
    rng = np.random.default_rng(5)
    n, c = shape[:2]
    for xdt, ddt in (("f32", "f32"), ("bf16", "f32"), ("bf16", "bf16")):
        x = rnd(xdt, rng.standard_normal(shape) * 2)
        t = make_targets(rng, (n,) + shape[2:], c, "f32", 1, 0.1, invalid=True)
        run(nk, dev, x, t, xdt, ddt, "f32", rng.uniform(0.5, 2, c).astype(F32N), True, 1, 0.1, 0.5)
        run(nk, dev, x, t, xdt, ddt, "bf16", None, False, 1, 0.0, 0.0)


def masked(rng, shape, xdt):
    """logits with -inf (masked) classes: class 0 and the last class of every position, the first 8 classes of a few
    positions (a thread's whole first vector or group), and about 10 % of the rest"""
    x = rng.standard_normal(shape) * 2
    x[:, 0] = -np.inf
    x[:, -1] = -np.inf
    x[1::5, :8] = -np.inf
    x[rng.random(shape) < 0.1] = -np.inf
    xm = np.moveaxis(x, 1, -1)                      # a view with the classes last
    xm[~np.isfinite(xm).any(axis=-1), shape[1] // 2] = 0.5   # every position keeps one finite logit
    return rnd(xdt, x)


def finite_targets(rng, x):
    """per position a class whose logit is finite (so the loss stays finite), one ignored (-100) position in 7"""
    xp, n, c, s = O.positions(x)
    t = np.array([rng.choice(np.flatnonzero(np.isfinite(r))) for r in xp], F32N)
    t[::7] = -100
    return t.reshape((n, s)).reshape((n,) + x.shape[2:])


# one case per layout: warp rows (odd C: scalar heads and tails), CTA rows, split rows, spatial positions
MASKED = [((37, 10), "f32"), ((37, 13), "bf16"), ((20, 1031), "f32"), ((20, 3001), "bf16"), ((16, 65537), "bf16"),
          ((9, 10, 33), "f32")]


@pytest.mark.parametrize("shape,xdt", MASKED, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else v)
@pytest.mark.parametrize("off", [0, 1])
def test_minus_inf_logits(nk, dev, shape, xdt, off):
    """masked (-inf) logits, also where they fill a thread's first vector or group: the loss and dx against the oracle
    and against torch CPU; with label smoothing the loss is +inf, as torch's, and dx stays finite"""
    rng = np.random.default_rng(13 + off)
    x = masked(rng, shape, xdt)
    t = finite_targets(rng, x)
    for ddt in ("f32", xdt):
        loss, dx = run(nk, dev, x, t, xdt, ddt, "f32", None, True, -100, 0.0, 0.0, off=off)
        xt = torch.tensor(x.astype(np.float64), requires_grad=True)
        lt = F.cross_entropy(xt, torch.tensor(t.astype(np.int64)), ignore_index=-100)
        lt.backward()
        assert np.isfinite(loss) and loss == pytest.approx(lt.item(), rel=1e-5)
        np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=0, atol=(2e-6 if ddt == "f32" else 2 ** -8) * O.grad_bound(
            1.0, None, 1.0 / np.sum(t != -100)))
        w = rng.uniform(0.5, 1.5, shape[1]).astype(F32N)
        loss, dx = run(nk, dev, x, t, xdt, ddt, "f32", w, False, -100, 0.1, 0.5, off=off)
        assert loss == np.inf and np.isfinite(dx).all()


def test_layout_thresholds(nk, dev):
    """both sides of each layout bound: rows longer than 4096 bytes take a warp each from 4096 rows on, a CTA each below;
    rows are split over CTAs when there are fewer than 2 per SM and at least 65536 classes"""
    rng = np.random.default_rng(14)
    sms = dev.sm_count
    for n, c in ((4095, 2049), (4096, 2049), (2 * sms - 1, 65536), (2 * sms, 65536), (16, 65535), (16, 65536),
                 (1, 65536)):
        x = rnd("bf16", rng.standard_normal((n, c)) * 2)
        t = make_targets(rng, (n,), c, "f32", 7, 0.05)
        run(nk, dev, x, t, "bf16", "f32", "f32", None, True, 7, 0.0, 0.0)
        run(nk, dev, x, t, "bf16", "bf16", "f32", rng.uniform(0.5, 1.5, c).astype(F32N), False, 7, 0.1, 1.0)


def test_empty_and_single(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(6)
    for shape in ((0, 5), (0, 3, 4)):
        X = dev.zeros(shape)
        T = dev.zeros((0,) + shape[2:])
        loss, lse, denom = ops.cross_entropy(X, T, mean=True)
        assert np.isnan(float(loss.as_ndarray())) and float(denom.as_ndarray()) == 0.0
        loss, lse, denom = ops.cross_entropy(X, T, mean=False)
        assert float(loss.as_ndarray()) == 0.0
        ops.cross_entropy_bwd(X, X, T, lse, denom, dev.from_ndarray(np.ones((), F32N)), beta=0.0)
    x = rng.standard_normal((1, 11)).astype(F32N)
    run(nk, dev, x, np.array([4], F32N), "f32", "f32", "f32", None, True)
    run(nk, dev, x, np.array([4], F32N), "f32", "f32", "f32", None, True, ig=4, beta=0.5)   # all ignored: NaN, dx = beta*dx


def test_bf16_more_than_2_31_elements(nk, dev):
    """(65600, 32768) bf16 logits, n*c > 2^31: the loss against torch's float64 lse per chunk of rows, and the gradient
    of the last rows (beyond element 2^31) against the oracle"""
    from neuronika_b200 import ops
    n, c = 65600, 32768
    assert n * c > 2 ** 31
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, c, device="cuda", generator=gen).to(torch.bfloat16)
    t = torch.randint(0, c, (n,), device="cuda", generator=gen).float()
    t[::7] = 0.0
    dx = torch.empty(n, c, device="cuda", dtype=torch.bfloat16)
    wrap = lambda a, d: nk.CuArray(dev, tuple(a.shape), d, ptr=a.data_ptr(), owner=a)
    torch.cuda.synchronize()
    loss, lse, denom = ops.cross_entropy(wrap(x, nk.BF16), wrap(t, nk.F32), ignore_index=0)
    ops.cross_entropy_bwd(wrap(dx, nk.BF16), wrap(x, nk.BF16), wrap(t, nk.F32), lse, denom,
                          dev.from_ndarray(np.ones((), F32N)), ignore_index=0, beta=0.0)
    dev.synchronize()
    keep = t != 0
    total = 0.0
    for r in range(0, n, 4096):
        xs = x[r:r + 4096].double()
        ll = torch.logsumexp(xs, 1) - xs.gather(1, t[r:r + 4096].long()[:, None])[:, 0]
        total += float(ll[keep[r:r + 4096]].sum())
    want = total / float(keep.sum())
    assert abs(float(loss.as_ndarray()) - want) <= 1e-5 * abs(want)
    rows = slice(n - 40, n)
    xr = x[rows].float().cpu().numpy()
    tr = t[rows].cpu().numpy()
    scale = 1.0 / float(keep.sum())
    ref = O.backward(xr, tr, 1.0, None, False, 0) * scale
    got = dx[rows].float().cpu().numpy()
    assert np.abs(got - ref).max() <= 2.0 ** -8 * scale


def test_repeated_calls_bitwise_equal(nk, dev):
    from neuronika_b200 import ops
    rng = np.random.default_rng(8)
    for shape, xdt in (((500, 100), "f32"), ((300, 5000), "bf16"), ((16, 262144), "bf16"), ((40, 19, 512), "f32")):
        n, c = shape[:2]
        x = rnd(xdt, rng.standard_normal(shape))
        t = make_targets(rng, (n,) + shape[2:], c, "f32", 2, 0.1)
        X, T = put(nk, dev, x, xdt), put(nk, dev, t, "f32")
        W = dev.from_ndarray(rng.uniform(0.5, 1.5, c).astype(F32N))
        G = dev.from_ndarray(np.array(0.5, F32N))
        outs = []
        for _ in range(3):
            loss, lse, denom = ops.cross_entropy(X, T, W, True, 2, 0.1)
            DX = dev.zeros(shape, nk.F32)
            ops.cross_entropy_bwd(DX, X, T, lse, denom, G, W, True, 2, 0.1, 0.0)
            outs.append((loss.as_ndarray(), lse.as_ndarray(), DX.as_ndarray()))
        for o in outs[1:]:
            for a, b in zip(o, outs[0]):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), shape


def test_matches_log_softmax_nll_composition(nk, dev):
    rng = np.random.default_rng(9)
    for n, c in ((256, 10), (64, 3000)):
        x = rng.standard_normal((n, c)).astype(F32N) * 2
        t = rng.integers(0, c, n).astype(F32N)
        T = nk.from_ndarray(dev, t)
        xa = nk.from_ndarray(dev, x).requires_grad()
        la = xa.cross_entropy(T)
        la.forward()
        la.backward(1.0)
        xb = nk.from_ndarray(dev, x).requires_grad()
        lb = xb.log_softmax(1).nll_loss(T)
        lb.forward()
        lb.backward(1.0)
        assert la.item() == pytest.approx(lb.item(), rel=1e-5)
        np.testing.assert_allclose(xa.grad(), xb.grad(), rtol=0, atol=1e-5 * np.abs(xb.grad()).max())


def test_bf16_language_model_shape_precision(nk, dev):
    """(8960, 10000) bf16 logits, bf16 dx: every off-target gradient element within 2^-7 relative of the float64 oracle
    on the same bf16 logits"""
    rng = np.random.default_rng(10)
    n, c = 8960, 10000
    x = bf16r(rng.standard_normal((n, c)).astype(F32N))
    t = rng.integers(0, c, n).astype(F32N)
    from neuronika_b200 import ops
    X, T = put(nk, dev, x, "bf16"), put(nk, dev, t, "f32")
    loss, lse, denom = ops.cross_entropy(X, T)
    DX = dev.zeros((n, c), nk.BF16)
    ops.cross_entropy_bwd(DX, X, T, lse, denom, dev.from_ndarray(np.ones((), F32N)), beta=0.0)
    got = DX.as_ndarray()
    want = O.backward(x, t, 1.0, None, True)
    off = np.ones((n, c), bool)
    off[np.arange(n), t.astype(np.int64)] = False
    rel = np.abs(got[off] - want[off]) / np.abs(want[off])
    assert rel.max() <= 2.0 ** -7, rel.max()
    assert float(loss.as_ndarray()) == pytest.approx(O.forward(x, t)[0], rel=1e-5)


def test_captured_linear_cross_entropy_sgd_step(nk, dev):
    """Linear -> cross_entropy(ignore_index=0) -> SGD in f32: the first eager step against torch CPU autograd; then the
    step captured and replayed 4 times with the targets rewritten in place before each replay (so the ignored count
    changes), bit for bit equal to 4 eager steps on the same targets, each replay's loss equal to the oracle's"""
    rng = np.random.default_rng(11)
    N, I, C = 96, 48, 37
    head = nk.nn.Linear(dev, I, C, rng=rng)
    params = head.parameters()
    init = [p.data().copy() for p in params]
    x = rng.standard_normal((N, I)).astype(F32N)
    targets = [rng.integers(0, C, N).astype(F32N) for _ in range(4)]
    for k, tg in enumerate(targets):
        tg[: 10 * (k + 1)] = 0.0                                         # 10, 20, 30, 40 ignored positions (and more)
    X, TG = nk.from_ndarray(dev, x), nk.from_ndarray(dev, targets[0])
    lr = 0.3
    opt = nk.optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)
    holder = {}

    def step():
        opt.zero_grad()
        loss = head.forward(X).cross_entropy(TG, ignore_index=0, label_smoothing=0.05)
        loss.forward()
        loss.backward(1.0)
        opt.step()
        holder["loss"] = loss

    eager, losses = [], []
    for tg in targets:
        TG.set_data(tg)
        step()
        losses.append(holder["loss"].item())
        eager.append([p.data().copy() for p in params])
    # torch CPU autograd, first step
    tw = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in init]
    lt = F.cross_entropy(torch.tensor(x, dtype=torch.float64) @ tw[0].T + tw[1],
                         torch.tensor(targets[0].astype(np.int64)), ignore_index=0, label_smoothing=0.05)
    lt.backward()
    assert losses[0] == pytest.approx(lt.item(), rel=1e-5)
    for got, p0, q in zip(eager[0], init, tw):
        np.testing.assert_allclose(got, p0 - lr * q.grad.numpy(), rtol=1e-5, atol=1e-6)
    # replays
    for p, v in zip(params, init):
        p.set_data(v)
    dev.synchronize()
    with dev.capture(64 << 20) as cap:
        step()
    loss = holder["loss"]
    for r, tg in enumerate(targets):
        before = [p.data().astype(np.float64) for p in params]
        TG.set_data(tg)
        cap.graph.launch()
        dev.synchronize()
        for p, want in zip(params, eager[r]):
            assert np.array_equal(p.data().view(np.uint32), want.view(np.uint32)), r
        want_loss = O.forward(x.astype(np.float64) @ before[0].T + before[1], tg, None, True, 0, 0.05)[0]
        assert loss.item() == pytest.approx(want_loss, rel=1e-5), r
        assert loss.item() == losses[r]
    cap.graph.close()
