"""BASELINE.json's full sizes through the public graph API, checked with properties that do not need the oracle to run the
whole problem: slabs of the outputs against the oracle, linearity over the batch, checksums of the bias gradient, and --
config 4 -- the complete training step against the oracle's restatement (numpy/OpenBLAS finishes it in seconds).
bf16 operands: the oracle consumes the same bf16-rounded values; tolerances are stated at each assertion."""
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
    d = nk.Device(0)
    yield d
    d.synchronize()


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


def test_config3_conv2d_full_size_properties(nk, dev, O):
    """nn::Conv2d 3->64 k3 on 224x224, batch 256, bf16: forward + backward(seed) through the graph (the path bench.py runs:
    conv + bias peephole forward, seeded backward, both on the wgmma im2col engine).  Checked: samples 0 and 255 of y and dx
    against the oracle; dW and db against the oracle on a 4-sample problem plus LINEARITY over the batch (the gradient of
    the whole batch equals the sum of the gradients of its two halves, which run through the same kernels)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(3)
    n, cin, h, w, cout = 256, 3, 224, 224, 64
    k = 1.0 / np.sqrt(27.0)
    x = O.bf16_round(rng.uniform(0, 1, (n, cin, h, w)).astype(F32))
    wt = O.bf16_round(rng.uniform(-k, k, (cout, cin, 3, 3)).astype(F32))
    b = O.bf16_round(rng.uniform(-k, k, (cout, 1, 1)).astype(F32))
    seed = 1.0 / 1024                                     # exact in bf16
    X = nk.from_ndarray(dev, x, nk.BF16).requires_grad()
    W = nk.from_ndarray(dev, wt, nk.BF16).requires_grad(nk.F32)
    B = nk.from_ndarray(dev, b, nk.BF16).requires_grad(nk.F32)
    y = W.convolution(X, (1, 1), (1, 1), 1) + B
    y.forward()
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_fwd"
    y.backward(seed)
    assert dev.last_conv_kernel == "wgmma_im2col_gemm_dx"
    yv = y.data()
    dx, dw, db = X.grad(), W.grad(), B.grad()
    for s in (0, n - 1):
        want = O.conv_forward(x[s:s + 1], wt, (1, 1), (1, 1)).astype(np.float64) + b[None]
        scale = float(np.sqrt((want ** 2).mean()))
        assert np.all(np.abs(yv[s:s + 1] - want) <= 2e-3 * scale + 2.0 ** -8 * np.abs(want)), s      # bf16 output
        g1 = np.full((1, cout, h - 2, w - 2), seed, F32)
        wx = np.zeros((1, cin, h, w), F32)
        O.conv_backward_input(wx, g1, wt, (1, 1), (1, 1))
        assert np.all(np.abs(dx[s:s + 1] - wx) <= 2.0 ** -7 * np.abs(wx) + 1e-6), s                  # bf16 output
    # db: every output pixel contributes the seed
    assert np.allclose(db.ravel(), seed * n * (h - 2) * (w - 2), rtol=1e-5)
    # dW against the oracle on the first 4 samples, then linearity over the batch halves
    g4 = np.full((4, cout, h - 2, w - 2), seed, F32)
    ww = np.zeros_like(wt)
    O.conv_backward_kernel(ww, g4, x[:4], (1, 1), (1, 1))
    parts = []
    for lo, hi in ((0, 4), (0, n // 2), (n // 2, n)):
        d_w = dev.zeros(wt.shape, nk.F32)
        xs = dev.from_ndarray(x[lo:hi], nk.BF16)
        ops.conv2d_bwd_kernel(d_w, dev.full((hi - lo, cout, h - 2, w - 2), seed, nk.BF16), xs, beta=0.0)
        parts.append(d_w.as_ndarray().astype(np.float64))
    assert np.all(np.abs(parts[0] - ww) <= 2e-3 * float(np.sqrt((ww.astype(np.float64) ** 2).mean())) + 1e-5 * np.abs(ww))
    total = parts[1] + parts[2]
    assert np.all(np.abs(dw - total) <= 1e-4 * np.abs(total) + 1e-3 * float(np.abs(total).mean()))  # f32 atomics across CTAs


def test_config4_mlp_step_full_size_matches_oracle(nk, dev, O):
    """MLP 1024-4096-4096-10 + ReLU / Softmax, MSE, batch 8192, one SGD step (lr 0.01) in bf16 through the graph with every
    peephole on (bias / ReLU epilogues, ReLU backward in the dX GEMM, skinny kernels for the 10-wide layer): loss, all six
    gradients and the updated weights against the oracle's restatement of the same step on the same bf16-rounded values."""
    rng = np.random.default_rng(4)
    sizes, bsz = [1024, 4096, 4096, 10], 8192
    x = O.bf16_round(rng.uniform(-1, 1, (bsz, sizes[0])).astype(F32))
    t = np.eye(10, dtype=F32)[np.argmax(x[:, :10], 1)]
    init = []
    for i, o in zip(sizes[:-1], sizes[1:]):
        kk = 1.0 / np.sqrt(i)
        init.append((O.bf16_round(rng.uniform(-kk, kk, (o, i)).astype(F32)), O.bf16_round(rng.uniform(-kk, kk, (o,)).astype(F32))))
    nk.set_fusion(2)
    try:
        params = []
        for wv, bv in init:
            params += [nk.from_ndarray(dev, wv, nk.BF16).requires_grad(nk.F32), nk.from_ndarray(dev, bv, nk.BF16).requires_grad(nk.F32)]
        opt = nk.optim.StochasticGD.new(0.01, nk.optim.L2(0.0))
        for p in params:
            opt.register(p)
        X, Tt = nk.from_ndarray(dev, x, nk.BF16), nk.from_ndarray(dev, t, nk.BF16)
        hcur = X
        for li in range(3):
            hcur = hcur.mm_t(params[2 * li]) + params[2 * li + 1]
            hcur = hcur.relu() if li < 2 else hcur.softmax(1)
        loss = hcur.mse_loss(Tt)
        del hcur
        loss.forward()
        loss.backward(1.0)
        got_loss = loss.item()
        got_grads = [p.grad().copy() for p in params]
        opt.step()
        got_w = [p.data().copy() for p in params]
    finally:
        nk.set_fusion(1)
    # oracle: same step, activations rounded to bf16 where the device stores them in bf16
    ws = [(wv.copy(), bv.copy()) for wv, bv in init]
    acts, pre, hcur = [x], [], x
    for li, (wv, bv) in enumerate(ws):
        z = O.linear_forward(hcur, wv, bv)
        if li < 2:
            hcur = O.bf16_round(O.relu_forward(z))            # relu(z) is stored in bf16; z itself is never stored
            pre.append(hcur)
        else:
            z = O.bf16_round(z)
            hcur = O.bf16_round(O.softmax_forward(z, 1))
        acts.append(hcur)
    pr = acts[-1]
    want_loss = float(O.mse_forward(pr, t, "mean"))
    assert abs(got_loss - want_loss) <= 2e-3 * abs(want_loss)
    dp = np.zeros_like(pr)
    O.mse_backward(pr, t, F32(1.0), dp, "mean")
    dz = np.zeros_like(pr)
    O.softmax_backward(pr, O.bf16_round(dp), dz, 1)
    dz = O.bf16_round(dz)
    want_grads = [None] * 6
    for li in reversed(range(3)):
        wv, bv = ws[li]
        dw, dbv = np.zeros_like(wv), np.zeros_like(bv)
        dh = np.zeros_like(acts[li]) if li > 0 else None
        O.linear_backward(acts[li], wv, dz, dh, dw, dbv)
        want_grads[2 * li], want_grads[2 * li + 1] = dw, dbv
        if li > 0:
            dzn = np.zeros_like(dh)
            O.relu_backward(pre[li - 1], dh, dzn)             # mask with y = relu(z) > 0  <=>  z > 0
            dz = O.bf16_round(dzn)
    for i, (g, want) in enumerate(zip(got_grads, want_grads)):
        rms = float(np.sqrt((want.astype(np.float64) ** 2).mean())) + 1e-30
        # f32 gradients of bf16 GEMM operands.  The intermediate gradients are rounded to bf16 on both sides and the ReLU masks
        # come from pre-activations summed in a different order, so single elements may differ by a rounding step or by one
        # sample's contribution: the bound is on the whole tensor (Frobenius, 1 %), on all but 1e-4 of the elements (10 % of
        # rms + 2 % of the value) and on the worst element (1 rms)
        err = np.abs(g.astype(np.float64) - want)
        fro = float(np.sqrt((err ** 2).sum()) / (np.sqrt((want.astype(np.float64) ** 2).sum()) + 1e-30))
        outl = float((err > 0.1 * rms + 2e-2 * np.abs(want)).mean())
        print(f"config 4 gradient {i}: rms {rms:.3e} max err {err.max():.3e} frobenius {fro:.3e} outliers {outl:.2e}")
        assert fro <= 1e-2, (i, fro)
        assert outl <= 1e-4, (i, outl, float(err.max()), rms)
        assert float(err.max()) <= rms, (i, float(err.max()), rms)
        # checksum of the whole tensor: the two sums agree to 0.2 % of the tensor's L1 norm
        assert abs(float(g.astype(np.float64).sum()) - float(want.astype(np.float64).sum())) <= \
            2e-3 * float(np.abs(want.astype(np.float64)).sum()) + 1e-6, i
    for i, (wnew, (w0, g)) in enumerate(zip(got_w, [(v, want_grads[j]) for j, v in enumerate([a for pair in init for a in pair])])):
        want_w = O.bf16_round(w0 - F32(0.01) * g)
        assert np.all(np.abs(wnew - want_w) <= 2.0 ** -7 * np.abs(want_w) + 1e-6), i
