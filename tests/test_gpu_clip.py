"""Gradient clipping on the GPU (csrc/nk_optim_multi.cu nk_grad_norm / nk_grad_scale_by_norm / nk_grad_clamp, the
optim.get_total_norm / clip_grads_with_norm_ / clip_grad_norm_ / clip_grad_value_ entry points) against the float64
oracle of tests/clip_oracle.py: the total within a bound derived from the summation depth, and, given the device's own
total, the scaled and clamped gradients to the bit; across dtype groups, the 64-tensors-per-launch boundary, every
n % 4, empty tensors, misaligned bases and a bf16 gradient of more than 2^31 elements; NaN and infinity; repeatability;
launch counts; the data-parallel grad_scale identity; error_if_nonfinite; torch CUDA; and a captured language-model
step that clips on some replays and not on others, to the bits of the same steps run eagerly."""
import numpy as np
import pytest

import clip_oracle as O

pytestmark = pytest.mark.gpu

NORMS = [1.0, 2.0, 3.0, 0.5, float("inf")]
SIZES = [0, 1, 2, 3, 4, 5, 6, 7, 4096, 8191, 8193, 70001, 0, 262147]
# f32 rounding depth of one partial: a thread folds up to kNormChunk / kThreads = 16 elements in order, then 5 butterfly
# levels and 8 warp partials; each term carries one rounding (v = k*g) plus its own (v*v or powf, <= 2 ulp); the double
# merge and the root add less than one more.  The p-th root scales a relative error of the sum by 1/p.
DEPTH = 16 + 5 + 8 + 3 + 1
U = 2.0 ** -24


def _bound(p):
    """relative bound of the device total; the max of p = inf is exact"""
    return 0.0 if np.isinf(p) else DEPTH * U * max(1.0, 1.0 / p)


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    return nk.Device(0)


def _dt(nk, name):
    return nk.BF16 if name == "bf16" else nk.F32


def _params(nk, dev, sizes, gdts, rng, scale=1.0):
    """differentiable leaves with random gradients; returns (params, host gradients as the device holds them)"""
    ps, hs = [], []
    for n, gd in zip(sizes, gdts):
        p = nk.zeros(dev, (n,), nk.F32).requires_grad(_dt(nk, gd))
        g = (rng.standard_normal(n) * scale).astype(np.float32)
        if n:
            p.grad_array().copy_from(g)
        ps.append(p)
        hs.append(O.bf16(g) if gd == "bf16" else g)
    return ps, hs


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    assert np.array_equal(nan, np.isnan(b)), (np.flatnonzero(nan != np.isnan(b))[:5])
    bad = np.flatnonzero(a[~nan].view(np.uint32) != b[~nan].view(np.uint32))
    assert bad.size == 0, (bad[:5], a[~nan][bad[:5]], b[~nan][bad[:5]])


def _check_total(got, want, p):
    if not np.isfinite(want):
        assert (np.isnan(got) and np.isnan(want)) or got == want, (got, want)
    else:
        assert abs(got - want) <= _bound(p) * want + 1e-37, (got, want, abs(got - want) / max(want, 1e-37))


MIXES = {"f32": lambda i: "f32", "bf16": lambda i: "bf16", "mixed": lambda i: "bf16" if i % 3 == 1 else "f32"}


@pytest.mark.parametrize("mix", sorted(MIXES))
@pytest.mark.parametrize("p", NORMS, ids=str)
def test_norm_scale_and_clamp_against_the_oracle(nk, dev, p, mix):
    from neuronika_b200 import optim
    rng = np.random.default_rng(NORMS.index(p) * 10 + len(mix))
    gdts = [MIXES[mix](i) for i in range(len(SIZES))]
    ps, hs = _params(nk, dev, SIZES, gdts, rng)
    k = 0.5
    total = optim.get_total_norm(ps, p, grad_scale=k)
    t = float(total.as_ndarray())
    _check_total(t, O.total_norm(hs, p, k), p)
    for max_norm in (0.3 * t, 3.0 * t):
        optim.clip_grads_with_norm_(ps, max_norm, total)
        c = O.coefficient(t, max_norm)
        hs = [O.scale(h, c, gd) for h, gd in zip(hs, gdts)]
        for q, h in zip(ps, hs):
            _same(q.grad(), h)
    optim.clip_grad_value_(ps, 0.2, grad_scale=k)
    for q, h, gd in zip(ps, hs, gdts):
        _same(q.grad(), O.clamp(h, 0.2, k, gd))


@pytest.mark.parametrize("gd", ["f32", "bf16"])
def test_many_tensors_several_launches_per_group(nk, dev, gd):
    """200 tensors: 4 launches per pass for one dtype; mixed, the groups in order of first appearance"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(5)
    sizes = [int(s) for s in rng.integers(0, 3000, 200)]
    gdts = [gd if i % 7 else ("bf16" if gd == "f32" else "f32") for i in range(200)]
    ps, hs = _params(nk, dev, sizes, gdts, rng)
    before = dev.launches
    total = optim.clip_grad_norm_(ps, 1.0)
    groups = sum(-(-sum(1 for d in gdts if d == x) // 64) for x in set(gdts))
    assert dev.launches - before == 2 * groups + 1
    t = float(total.as_ndarray())
    _check_total(t, O.total_norm(hs, 2.0), 2.0)
    c = O.coefficient(t, 1.0)
    for q, h, d in zip(ps, hs, gdts):
        _same(q.grad(), O.scale(h, c, d))


@pytest.mark.parametrize("gd", ["f32", "bf16"])
def test_misaligned_views_into_one_bucket(nk, dev, gd):
    """gradients at odd element offsets of one bucket take the element path; each n % 4 and an empty view"""
    from neuronika_b200 import optim
    rng = np.random.default_rng(6)
    sizes = [5, 4, 0, 4099, 3, 9000, 2, 1]
    bucket = dev.zeros((sum(sizes) + 2 * len(sizes) + 1,), _dt(nk, gd))
    ps, hs, off = [], [], 1
    for n in sizes:
        view = bucket.slice_flat(off, (n,))
        p = nk.zeros(dev, (n,), nk.F32).requires_grad(_dt(nk, gd), grad_array=view)
        g = rng.standard_normal(n).astype(np.float32)
        if n:
            view.copy_from(g)
        ps.append(p)
        hs.append(O.bf16(g) if gd == "bf16" else g)
        off += n + (1 if n % 2 else 2)       # the next view starts at an odd element again
    for p_ in NORMS:
        t = float(optim.get_total_norm(ps, p_).as_ndarray())
        _check_total(t, O.total_norm(hs, p_), p_)
    t = float(optim.clip_grad_norm_(ps, 0.5).as_ndarray())
    c = O.coefficient(t, 0.5)
    for q, h in zip(ps, hs):
        _same(q.grad(), O.scale(h, c, gd))
    optim.clip_grad_value_(ps, 0.01)
    for q, h in zip(ps, hs):
        _same(q.grad(), O.clamp(O.scale(h, c, gd), 0.01, 1.0, gd))


def test_bf16_gradient_beyond_2_31_elements(nk, dev):
    """64-bit element offsets: a value planted past element 2^31 enters the norm and is scaled"""
    from neuronika_b200 import optim
    n = (1 << 31) + 1029
    p = nk.zeros(dev, (n,), nk.BF16).requires_grad()
    g = p.grad_array()
    g.fill_(0.5)
    tail = g.slice_flat(n - 5, (5,))
    tail.copy_from(np.array([0.5, 0.5, 1024.0, 0.5, -8.0], np.float32))
    want = np.sqrt((n - 2) * 0.25 + 1024.0 ** 2 + 64.0)
    total = optim.clip_grad_norm_(p, 1.0)
    t = float(total.as_ndarray())
    assert abs(t - want) <= _bound(2.0) * want, (t, want)
    c = O.coefficient(t, 1.0)
    _same(tail.as_ndarray(), O.scale(np.array([0.5, 0.5, 1024.0, 0.5, -8.0], np.float32), c, "bf16"))
    _same(g.slice_flat(0, (3,)).as_ndarray(), O.scale(np.full(3, 0.5, np.float32), c, "bf16"))
    assert float(optim.get_total_norm(p, float("inf")).as_ndarray()) == float(O.bf16(np.float32([1024.0 * c]))[0])
    del p, g, tail


@pytest.mark.parametrize("what", ["nan", "inf", "nan_and_inf"])
@pytest.mark.parametrize("gd", ["f32", "bf16"])
def test_nan_and_inf_gradients(nk, dev, what, gd):
    from neuronika_b200 import optim
    rng = np.random.default_rng(7)
    sizes = [33, 9000, 4, 1]
    ps, hs = _params(nk, dev, sizes, [gd] * 4, rng)
    if "nan" in what:
        hs[1][8191] = np.nan
    if "inf" in what:
        hs[2][1] = -np.inf
        hs[0][0] = np.inf
    for q, h in zip(ps, hs):
        q.grad_array().copy_from(h)
    for p_ in NORMS:
        t = float(optim.get_total_norm(ps, p_).as_ndarray())
        _check_total(t, O.total_norm(hs, p_), p_)
        assert np.isnan(t) if "nan" in what else t == np.inf
    t = float(optim.clip_grad_norm_(ps, 1.0).as_ndarray())
    c = O.coefficient(t, 1.0)
    for q, h in zip(ps, hs):
        _same(q.grad(), O.scale(h, c, gd))
    with pytest.raises(RuntimeError, match="is non-finite, so it cannot be clipped"):
        optim.clip_grad_norm_(ps, 1.0, error_if_nonfinite=True)


def test_no_clip_leaves_every_bit_and_repeats_bitwise(nk, dev):
    from neuronika_b200 import optim
    rng = np.random.default_rng(8)
    ps, hs = _params(nk, dev, SIZES, [MIXES["mixed"](i) for i in range(len(SIZES))], rng)
    bits = [q.grad().copy() for q in ps]
    totals = [optim.clip_grad_norm_(ps, 1e30).as_ndarray() for _ in range(3)]
    assert len({t.tobytes() for t in totals}) == 1
    for q, b in zip(ps, bits):
        _same(q.grad(), b)
    for p_ in NORMS:
        assert len({optim.get_total_norm(ps, p_).as_ndarray().tobytes() for _ in range(3)}) == 1


def test_launch_counts_from_the_profiler(nk, dev):
    """norm: one launch per (dtype, 64 tensors) group plus one finish; scale and clamp: one per group; with c == 1 the
    scale kernel still runs (it reads the total) and writes nothing"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from neuronika_b200 import optim
    rng = np.random.default_rng(9)
    gdts = ["f32"] * 70 + ["bf16"] * 3
    ps, _ = _params(nk, dev, [100] * 73, gdts, rng)
    dev.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        optim.clip_grad_norm_(ps, 0.01)
        optim.clip_grad_value_(ps, 0.001)
        dev.synchronize()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    count = lambda s: sum(s in n for n in names)
    assert count("nk_grad_norm_kernel") == 3 and count("nk_grad_norm_finish_kernel") == 1, names
    assert count("nk_grad_pointwise_kernel<0") == 3 and count("nk_grad_pointwise_kernel<1") == 3, names


def test_empty_lists(nk, dev):
    from neuronika_b200 import ops, optim
    out = dev.full((), 7.0)
    ops.grad_norm([], out=out)
    assert float(out.as_ndarray()) == 0.0
    optim.clip_grad_value_([], 1.0)
    optim.clip_grads_with_norm_([], 1.0, out)
    with pytest.raises(ValueError):
        optim.get_total_norm([])
    p = nk.zeros(dev, (4,), nk.F32).requires_grad()
    with pytest.raises(nk.NkError, match="norm_type"):
        optim.get_total_norm(p, 0.0)


def test_power_of_two_grad_scale_identity(nk, dev):
    """clip + SGD on world*G with grad_scale = 1/world gives the weights of the unscaled run, bit for bit"""
    from neuronika_b200 import optim
    world = 4
    rng = np.random.default_rng(10)
    sizes = [300, 4097, 5]
    ws = [rng.standard_normal(n).astype(np.float32) for n in sizes]
    gs = [rng.standard_normal(n).astype(np.float32) for n in sizes]
    runs = []
    for k in (1, world):
        ps = [nk.from_ndarray(dev, w).requires_grad() for w in ws]
        opt = optim.StochasticGD.new(0.1, momentum=0.9, dampening=0.0, grad_scale=1.0 / k)
        for q in ps:
            opt.register(q)
        for step in range(3):
            for q, g in zip(ps, gs):
                q.grad_array().copy_from(g * np.float32(k) * np.float32(1 + step))
            optim.clip_grad_norm_(ps, 2.0, grad_scale=1.0 / k)
            optim.clip_grad_value_(ps, 0.05, grad_scale=1.0 / k)
            opt.step()
        runs.append([q.data() for q in ps])
    for a, b in zip(*runs):
        _same(a, b)


def test_error_if_nonfinite_refused_inside_a_capture(nk, dev):
    from neuronika_b200 import optim
    ps, _ = _params(nk, dev, [10, 20], ["f32", "f32"], np.random.default_rng(11))
    assert np.isfinite(optim.clip_grad_norm_(ps, 1.0, error_if_nonfinite=True).as_ndarray())
    optim.clip_grad_norm_(ps, 1.0)
    with pytest.raises(nk.NkError, match="error_if_nonfinite"):
        with dev.capture(1 << 20):
            optim.clip_grad_norm_(ps, 1.0, error_if_nonfinite=True)


@pytest.mark.parametrize("p", NORMS, ids=str)
def test_against_torch_cuda(nk, dev, p):
    import torch
    from neuronika_b200 import optim
    rng = np.random.default_rng(12)
    sizes = [1000, 3, 65536, 0, 777] if not np.isinf(p) else [1000, 3, 65536, 777]
    ps, hs = _params(nk, dev, sizes, ["f32"] * len(sizes), rng)
    tp = [torch.nn.Parameter(torch.zeros(len(h), device="cuda")) for h in hs]
    for q, h in zip(tp, hs):
        q.grad = torch.from_numpy(h).cuda()
    t_total = float(torch.nn.utils.clip_grad_norm_(tp, 0.5, norm_type=p, foreach=True))
    total = float(optim.clip_grad_norm_(ps, 0.5, norm_type=p).as_ndarray())
    assert abs(total - t_total) <= 1e-5 * t_total
    for q, t in zip(ps, tp):
        np.testing.assert_allclose(q.grad(), t.grad.cpu().numpy(), rtol=2e-5, atol=1e-30)


# ------------------------------------------------------------------------------------------ captured LM step
def _lm(nk, dev, seed, V=1000, E=64, T=8, N=16):
    from neuronika_b200 import optim
    rng = np.random.default_rng(seed)
    emb = nk.nn.Embedding(dev, V, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    lstm = nk.nn.LSTM(dev, E, E, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    head = nk.nn.Linear(dev, E, V, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    params = emb.parameters() + lstm.parameters() + head.parameters()
    ids = nk.zeros(dev, (T, N), nk.F32)
    tgt = nk.zeros(dev, (T * N,), nk.F32)
    c0, h0 = nk.zeros(dev, (N, E), nk.BF16), nk.zeros(dev, (N, E), nk.BF16)
    opt = optim.StochasticGD.new(0.5)
    for q in params:
        opt.register(q)

    def loss():
        out, _ = lstm.forward((c0, h0), emb.forward(ids))
        return head.forward(out.reshape(T * N, E)).cross_entropy(tgt)
    return dict(params=params, ids=ids, tgt=tgt, loss=loss, opt=opt)


def _batch(rng, V, T, N, sparse):
    """token ids, and targets: every position (a small mean gradient) or one position, the rest ignored (a large one)"""
    ids = rng.integers(0, V, (T, N)).astype(np.float32)
    tgt = rng.integers(0, V, T * N).astype(np.float32)
    if sparse:
        tgt[1:] = -100
    return ids, tgt


def test_captured_lm_step_with_clipping_replays_the_eager_steps(nk, dev):
    from neuronika_b200 import optim
    V, T, N = 1000, 8, 16
    eager, capt = _lm(nk, dev, 0), _lm(nk, dev, 0)
    rng = np.random.default_rng(1)
    probe = []
    for sparse in (False, True):        # totals of both kinds of batch: max_norm between them
        ids, tgt = _batch(rng, V, T, N, sparse)
        eager["ids"].set_data(ids)
        eager["tgt"].set_data(tgt)
        loss = eager["loss"]()
        loss.forward()
        loss.backward(1.0)
        probe.append(float(optim.get_total_norm(eager["params"]).as_ndarray()))
        eager["opt"].zero_grad()
    assert probe[0] < probe[1], probe
    max_norm = float(np.sqrt(probe[0] * probe[1]))

    def step(m):
        m["opt"].zero_grad()
        loss = m["loss"]()
        loss.forward()
        loss.backward(1.0)
        total = optim.clip_grad_norm_(m["params"], max_norm)
        m["opt"].step()
        return total

    def feed(sparse):
        ids, tgt = _batch(rng, V, T, N, sparse)
        for m in (eager, capt):
            m["ids"].set_data(ids)
            m["tgt"].set_data(tgt)

    for sparse in (False, True):         # warm-up, eagerly, on both
        feed(sparse)
        step(eager)
        step(capt)
    dev.synchronize()
    with dev.capture(256 << 20) as cap:
        total_c = step(capt)
    clipped = []
    for r in range(8):
        feed(r % 3 == 1)
        total_e = float(step(eager).as_ndarray())
        cap.graph.launch()
        assert float(total_c.as_ndarray()) == total_e, r
        clipped.append(total_e > max_norm)
        for a, b in zip(eager["params"], capt["params"]):
            _same(a.data(), b.data())
    assert any(clipped) and not all(clipped), clipped
    cap.graph.close()
