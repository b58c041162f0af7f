"""f32 models on the tensor cores (Device.f32_matmul) at the graph level: an SGD step of an f32 MLP in TF32 and 3xTF32
mode against the float64 oracle, an f32 nn.LSTM in TF32 mode against the float64 sequence oracle, and a captured 3xTF32
training step that replays bit for bit.

Tolerances, from the per-GEMM bounds of tests/test_gpu_gemm_tf32.py: TF32 rounds both operands of every product to
2^-11, so one GEMM is within ~2^-10 of |A|.|B| (+ accumulation).  A weight gradient dW = dZ^T.X of the MLP below
depends on at most six chained GEMMs (three forward, three backward), so it is checked against rel (|dZ|^T.|X|) with
rel = 2^-7, where |dZ| is the magnitude the backward GEMMs see: the softmax backward's magnitude p (|dp| + sum |dp| p)
(it cancels, and is computed in f32) carried down through |W| and the ReLU masks in float64, and |X| likewise the
magnitude |X_below|.|W|^T + |b| of each activation, so that cancellation in dZ or dW does not count against the kernel (db: rel sum |dZ|).  A ReLU mask is
discontinuous: a pre-activation within `flip` of its magnitude (|X|.|W|^T + |b|) of zero -- its forward error after
two GEMMs: 2^-9 in TF32, 2^-18 in 3xTF32 -- may land on the other side, and then its whole term is the error.  Those terms are added to the bound at full size and carried down like |dZ|.  3xTF32 is within ~3 2^-22 of each product plus f32 accumulation: rel = 2^-16.  The LSTM's
TF32 operands (including every h_t fed back into the recurrent GEMM) are rounded 8x finer than the bf16 storage that the
bf16 tolerances of tests/test_gpu_rnn_seq.py cover, so those tolerances hold for TF32."""
import numpy as np
import pytest

import rnn_seq_oracle as S
from test_gpu_rnn import UB, held, k_e, leaf, near

pytestmark = pytest.mark.gpu
F32 = np.float32
SIZES = [1024, 1024, 1024, 10]
BATCH = 512
LR = 0.05


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.f32_matmul("ieee")
    d.synchronize()


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


@pytest.fixture(autouse=True)
def ieee_after(dev):
    yield
    dev.f32_matmul("ieee")


def make_mlp(nk, dev, seed):
    rng = np.random.default_rng(seed)
    layers = [nk.nn.Linear(dev, a, b, rng=rng) for a, b in zip(SIZES[:-1], SIZES[1:])]
    x = rng.uniform(-1, 1, (BATCH, SIZES[0])).astype(F32)
    t = np.eye(SIZES[-1], dtype=F32)[rng.integers(0, SIZES[-1], BATCH)]
    return layers, x, t


def forward_loss(nk, dev, layers, x, t):
    h = nk.from_ndarray(dev, x)
    for i, l in enumerate(layers):
        h = l.forward(h)
        h = h.relu() if i < len(layers) - 1 else h.softmax(1)
    return h.mse_loss(nk.from_ndarray(dev, t))


def magnitudes(x, t, params, rel, flip_margin):
    """float64 forward and backward of the MLP in magnitudes: for each layer the bounds of dW and db,
    rel (|dZ|^T.|X|, sum |dZ|) + (F^T.|X|, sum F), where |dZ| is carried down as |dZ| |W| through the ReLU masks and F
    collects the terms of mask elements that may flip (|z| <= flip_margin (|X|.|W|^T + |b|)), carried down the same way"""
    acts, pre, amb, amag = [x], [], [], [np.abs(x)]   # amag: |X| carried up as |X|.|W|^T + |b| through the masks
    for i, (w, b) in enumerate(params):
        z = acts[-1] @ w.T + b
        zmag = amag[-1] @ np.abs(w).T + np.abs(b)
        pre.append(z)
        amb.append(np.abs(z) <= flip_margin * zmag)
        amag.append(zmag * ((z > 0) | amb[-1]))
        if i < len(params) - 1:
            acts.append(np.maximum(z, 0.0))
        else:
            e = np.exp(z - z.max(1, keepdims=True))
            acts.append(e / e.sum(1, keepdims=True))
    p = acts[-1]
    dp = 2.0 * (p - t) / p.size
    # the softmax backward p (dp - sum dp p) cancels; its f32 rounding scales with p (|dp| + sum |dp| p)
    dz = p * (np.abs(dp) + (np.abs(dp) * p).sum(1, keepdims=True))
    flip = np.zeros_like(dz)
    out = [None] * len(params)
    for i in reversed(range(len(params))):
        out[i] = (rel * dz.T @ amag[i] + flip.T @ amag[i], rel * dz.sum(0) + flip.sum(0))
        if i:
            up, up_flip = dz @ np.abs(params[i][0]), flip @ np.abs(params[i][0])
            live = (pre[i - 1] > 0) | amb[i - 1]
            dz, flip = up * live, up_flip * live + up * amb[i - 1]
    return out


@pytest.mark.parametrize("mode,rel,flip", [("tf32", 2.0 ** -7, 2.0 ** -9), ("tf32x3", 2.0 ** -16, 2.0 ** -18)])
def test_mlp_sgd_step_against_float64_oracle(nk, dev, O, mode, rel, flip):
    layers, x, t = make_mlp(nk, dev, 1)
    params64 = [(l.weight.data().astype(np.float64), l.bias.data().astype(np.float64)) for l in layers]
    bounds = magnitudes(x.astype(np.float64), t.astype(np.float64), params64, rel, flip)
    opt = nk.optim.StochasticGD.new(LR)
    for l in layers:
        for p in l.parameters():
            opt.register(p)
    dev.f32_matmul(mode)
    opt.zero_grad()
    loss = forward_loss(nk, dev, layers, x, t)
    loss.forward()
    assert dev.last_gemm_kernel == f"{mode}_nt_128x64"       # the 1024 -> 10 head
    loss.backward(1.0)
    kern_bwd = dev.last_gemm_kernel
    opt.step()
    lo, grads = O.mlp_step(x.astype(np.float64), t.astype(np.float64), params64, LR, 0.0)
    assert kern_bwd.startswith(f"{mode}_"), kern_bwd
    assert abs(loss.item() - float(lo)) <= rel * abs(float(lo)), (loss.item(), float(lo))
    for i, (l, (dw, db), (w, b), (tw, tb)) in enumerate(zip(layers, grads, params64, bounds)):
        near(l.weight.grad(), dw, tw + 1e-30, (mode, i, "dW"))
        near(l.bias.grad(), db, tb + 1e-30, (mode, i, "db"))
        # the SGD update: w - lr dW, rounded to f32
        near(l.weight.data(), w, LR * tw + 2.0 ** -24 * np.abs(w), (mode, i, "W"))
        near(l.bias.data(), b, LR * tb + 2.0 ** -24 * np.abs(b), (mode, i, "b"))


def test_lstm_in_tf32_against_the_oracle(nk, dev):
    T, n, n_in, hidden = 5, 6, 40, 24
    rng = np.random.default_rng(17)
    layer = nk.nn.LSTM(dev, n_in, hidden, nk.F32, rng=np.random.default_rng(3))
    W = [getattr(layer, name).data() for name in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    xs = held(rng.standard_normal((T, n, n_in)), "f32")
    h0 = held(rng.standard_normal((n, hidden)) * 0.5, "f32")
    c0 = held(rng.standard_normal((n, hidden)) * 0.5, "f32")
    tgt = held(rng.standard_normal((T, n, hidden)) * 0.5, "f32")
    X, H0, C0 = leaf(nk, dev, xs, "f32", True), leaf(nk, dev, h0, "f32", True), leaf(nk, dev, c0, "f32", True)
    dev.f32_matmul("tf32")
    out, _ = layer.forward((C0, H0), X)
    loss = out.mse_loss(nk.from_ndarray(dev, tgt), nk.Reduction.Sum)
    loss.forward()
    assert dev.last_gemm_kernel.startswith("tf32_"), dev.last_gemm_kernel
    loss.backward(1.0)
    assert dev.last_gemm_kernel.startswith("tf32_"), dev.last_gemm_kernel
    w_out, _ = S.lstm_seq_forward(xs, c0, h0, *W)
    near(out.data(), w_out, 2 * UB * T * (1 + np.abs(w_out)), "output")
    g, mag = S.lstm_seq_backward(xs, c0, h0, *W, 2.0 * (w_out - tgt), None)
    for k, name in (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh")):
        m = np.asarray(mag[k], np.float64)
        near(getattr(layer, name).grad(), g[k], k_e("bf16") * (2 * T + 2) * (m + m.mean()) + 1e-9, name)
    for v, k in ((X, "x"), (H0, "h"), (C0, "c")):
        m = np.asarray(mag[k], np.float64)
        near(v.grad(), g[k], k_e("bf16") * (2 * T + 2) * (m + m.mean()) + 1e-9, "d" + k)


def test_captured_tf32x3_step_replays_the_eager_step(nk, dev):
    layers, x, t = make_mlp(nk, dev, 2)
    params = [p for l in layers for p in l.parameters()]
    init = [p.data().copy() for p in params]
    opt = nk.optim.StochasticGD.new(LR)
    for p in params:
        opt.register(p)
    X, Tt = nk.from_ndarray(dev, x), nk.from_ndarray(dev, t)
    kernels = []

    def step():
        opt.zero_grad()
        h = X
        for i, l in enumerate(layers):
            h = l.forward(h)
            h = h.relu() if i < len(layers) - 1 else h.softmax(1)
        loss = h.mse_loss(Tt)
        loss.forward()
        kernels.append(dev.last_gemm_kernel)
        loss.backward(1.0)
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    dev.f32_matmul("tf32x3")
    step()                     # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [p.data().copy() for p in params]
    assert kernels[-1] == "tf32x3_nt_128x64"
    assert any(np.any(e != i) for e, i in zip(eager, init))
    reset()
    with dev.capture(1 << 30) as cap:
        step()
    dev.f32_matmul("ieee")     # the captured step keeps the mode it was captured with
    for _ in range(2):
        reset()
        cap.graph.launch()
        dev.synchronize()
        for i, (p, e) in enumerate(zip(params, eager)):
            assert np.array_equal(p.data().view(np.uint32), e.view(np.uint32)), i
    cap.graph.close()
