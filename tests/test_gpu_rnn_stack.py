"""Stacked and bidirectional LSTM / GRU on the GPU: nk_gemm_strided_batched, the two-direction step kernels of
csrc/nk_rnn.cu (nk_lstm_bidir_fwd_step, nk_gru_bidir_fwd_step, nk_lstm_bidir_bwd_step, nk_gru_bidir_bwd_step), the layer
node (variable.lstm_layer / gru_layer) and nn.LSTM / nn.GRU(num_layers, bidirectional, dropout).

Operators: every operand sits in a canary-filled buffer, the two directions' operands a (sometimes negative) distance
apart and the output-like ones with row stride 2H, as the layer lays them out; everything outside the operands must come
back bit for bit.  Base offsets 0 and 1 element select the vector and the scalar bodies.  Tolerances as in
test_gpu_rnn_seq.py.  Layers: against the float64 oracle of tests/rnn_stack_oracle.py on the same (bf16-rounded) values,
with the bound k_e * (2T + 2) * (mag + mean(mag)) of test_gpu_rnn_seq.py, times the number of layers (a lower layer's
gradient carries the rounding of the layers above it).
"""
import ctypes as C

import numpy as np
import pytest

import criteria_oracle as CO
import rnn_oracle as R
import rnn_stack_oracle as K
from test_gpu_rnn import CANARY, D, F32, UB, gates_like, held, k_e, near, pw_tol
from test_gpu_rnn_seq import step_tol, tile

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


class Placed:
    """matrices mats[b] (rows, cols) at element base + b*stride, rows ld apart, of one canary-filled device buffer"""

    def __init__(self, nk, dev, mats, dt, base, stride, ld):
        mats = np.asarray(mats, F32)
        self.dt, self.stride = dt, stride
        rows, cols = mats.shape[1:]
        self.idx = [base + b * stride + np.arange(rows)[:, None] * ld + np.arange(cols)[None, :]
                    for b in range(mats.shape[0])]
        assert min(int(i.min()) for i in self.idx) >= 0
        self.host = np.full(max(int(i.max()) for i in self.idx) + 24, CANARY, F32)
        for b, ix in enumerate(self.idx):
            self.host[ix] = mats[b]
        self.buf = dev.from_ndarray(self.host, D(nk, dt))
        self.ptr = self.buf.ptr.value + base * self.buf.itemsize

    def read(self):
        flat = self.buf.as_ndarray().ravel()
        outside = np.ones(flat.size, bool)
        for ix in self.idx:
            outside[ix.ravel()] = False
        bad = np.flatnonzero(flat[outside].view(np.uint32) != self.host[outside].view(np.uint32))
        assert bad.size == 0, f"{bad.size} elements outside the operands were written"
        return np.stack([flat[ix] for ix in self.idx])


def ck(nk, dev, rc):
    nk._lib.check(rc, dev.ctx)


# ------------------------------------------------------------------------------------------------ strided-batched GEMM
# (M, N, K, pad): pad 8 keeps leading dimensions and strides on 16 bytes (one wgmma launch for bf16), pad 1 / base 1
# element leaves them off TMA's alignment (one GEMM per product)
SHAPES = [(70, 104, 64, 8, 0), (5, 13, 7, 1, 1)]   # N = 104: three full 32-column chunks and a tail of 8


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("form", ["NT", "NN"])
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("bias", [None, "f32", "bf16"])
def test_strided_batched_gemm(nk, dev, dt, form, shape, batch, beta, bias):
    """bias: none, or a per-product column bias of either element type (the vector loads of a full 32-column chunk and
    the scalar tail)"""
    from neuronika_b200 import ops
    M, N, Kd, pad, base = shape
    rng = np.random.default_rng([M, batch, int(beta), len(bias or ""), len(form), len(dt)])
    a = held(rng.standard_normal((batch, M, Kd)), dt)
    b = held(rng.standard_normal((batch, N, Kd) if form == "NT" else (batch, Kd, N)), dt)
    c0 = rng.standard_normal((batch, M, N)).astype(F32)
    bv = held(rng.standard_normal((batch, 1, N)), bias or "f32")
    lda, ldb, ldc = Kd + pad, b.shape[2] + pad, N + pad
    A = Placed(nk, dev, a, dt, base, M * lda + pad, lda)
    B = Placed(nk, dev, b, dt, base, b.shape[1] * ldb + 2 * pad, ldb)
    Cm = Placed(nk, dev, c0, "f32", base, M * ldc + 3 * pad, ldc)
    Bias = Placed(nk, dev, bv, bias or "f32", base, N + pad, N)
    before = dev.launches
    view = lambda p, t: nk.CuArray(dev, (1,), D(nk, t), ptr=p.ptr, owner=p.buf)
    ops.gemm_strided_batched(view(A, dt), view(B, dt), view(Cm, "f32"), M, N, Kd, batch, lda, ldb, ldc, A.stride,
                             B.stride, Cm.stride, trans_b=form == "NT", alpha=0.5, beta=beta,
                             bias=view(Bias, bias) if bias else None, bias_stride=Bias.stride)
    dev.synchronize()
    if dt == "bf16" and pad == 8:
        assert dev.launches - before == 1 and dev.last_gemm_kernel == "wgmma_batched"
    bt = b if form == "NN" else np.transpose(b, (0, 2, 1))
    A64, B64 = a.astype(np.float64), bt.astype(np.float64)
    want = 0.5 * A64 @ B64 + beta * c0 + (bv if bias else 0.0)
    scale = 0.5 * np.abs(A64) @ np.abs(B64) + beta * np.abs(c0) + (np.abs(bv) if bias else 0.0)
    near(Cm.read(), want, 1e-5 * scale + 1e-6, f"C {form} {shape} batch={batch}")
    assert np.array_equal(A.read(), a) and np.array_equal(B.read(), b) and np.array_equal(Bias.read(), bv)


def test_strided_batched_gemm_argument_errors(nk, dev):
    from neuronika_b200 import ops
    x = dev.zeros((64,), nk.BF16)
    with pytest.raises(nk.NkError, match="negative dimension"):
        ops.gemm_strided_batched(x, x, dev.zeros((64,)), 2, 2, 2, -1, 2, 2, 2, 4, 4, 4)
    ops.gemm_strided_batched(x, x, dev.zeros((64,)), 2, 2, 2, 0, 2, 2, 2, 4, 4, 4)   # an empty batch does nothing


# ------------------------------------------------------------------------------------------------ step kernels
STEP_SIZES = [(3, 16), (5, 7), (33, 64)]


def out_like(nk, dev, mats, dt, off, n, h):
    """(2, n, h) at the layer output's positions of a middle step of T = 2: direction 0 in row 1, direction 1 in row 0,
    columns [h, 2h) -- a negative direction distance, row stride 2h"""
    return Placed(nk, dev, mats, dt, off + n * 2 * h, -n * 2 * h + h, 2 * h)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n,h", STEP_SIZES)
@pytest.mark.parametrize("off", [0, 1])
def test_lstm_bidir_fwd_step(nk, dev, dt, n, h, off):
    rng = np.random.default_rng([n, h, off, 1])
    gates = np.stack([gates_like(rng, n, 4, h) for _ in range(2)])
    c0 = held(rng.standard_normal((2, n, h)), dt)
    nan = np.full((2, n, h), np.nan, F32)
    G = Placed(nk, dev, gates, "f32", off, n * 4 * h + 8, 4 * h)
    CP = Placed(nk, dev, c0, dt, off, n * h + 8, h)
    CO_ = Placed(nk, dev, nan, dt, off, n * h + 16, h)
    Y, HN = out_like(nk, dev, nan, dt, off, n, h), Placed(nk, dev, nan, dt, off, n * h, h)
    ck(nk, dev, nk._lib.lib.nk_lstm_bidir_fwd_step(dev.ctx, Y.ptr, Y.stride, 2 * h, HN.ptr, CO_.ptr, CO_.stride, G.ptr,
                                                   G.stride, CP.ptr, CP.stride, n, h, D(nk, dt)))
    want = [R.lstm_pointwise(gates[d], c0[d]) for d in range(2)]
    wc, wh = np.stack([w[0] for w in want]), np.stack([w[1] for w in want])
    near(CO_.read(), wc, pw_tol(wc, dt), "c'")
    near(Y.read(), wh, pw_tol(wh, dt), "y")
    near(HN.read(), wh, pw_tol(wh, dt), "h_next")
    assert np.array_equal(G.read(), gates) and np.array_equal(CP.read(), c0)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n,h", STEP_SIZES)
@pytest.mark.parametrize("off", [0, 1])
def test_gru_bidir_fwd_step(nk, dev, dt, n, h, off):
    rng = np.random.default_rng([n, h, off, 2])
    ig = np.stack([gates_like(rng, n, 3, h) for _ in range(2)])
    hg = np.stack([gates_like(rng, n, 3, h) for _ in range(2)])
    h0 = held(rng.standard_normal((2, n, h)), dt)
    nan = np.full((2, n, h), np.nan, F32)
    gds = n * 3 * h + 8
    IG, HG = Placed(nk, dev, ig, "f32", off, gds, 3 * h), Placed(nk, dev, hg, "f32", off, gds, 3 * h)
    HP = Placed(nk, dev, h0, dt, off, n * h + 8, h)
    Y, HN = out_like(nk, dev, nan, dt, off, n, h), Placed(nk, dev, nan, dt, off, n * h, h)
    ck(nk, dev, nk._lib.lib.nk_gru_bidir_fwd_step(dev.ctx, Y.ptr, Y.stride, 2 * h, HN.ptr, IG.ptr, HG.ptr, gds, HP.ptr,
                                                  HP.stride, n, h, D(nk, dt)))
    wh = np.stack([R.gru_pointwise(ig[d], hg[d], h0[d]) for d in range(2)])
    near(Y.read(), wh, pw_tol(wh, dt), "y")
    near(HN.read(), wh, pw_tol(wh, dt), "h_next")
    assert np.array_equal(HP.read(), h0)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n,h", STEP_SIZES)
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("use_out,use_rec", [(True, True), (False, True), (True, False)])
def test_lstm_bidir_bwd_step(nk, dev, dt, n, h, off, use_out, use_rec):
    rng = np.random.default_rng([n, h, off, 3, use_out, use_rec])
    gates = np.stack([gates_like(rng, n, 4, h) for _ in range(2)])
    c0 = held(rng.standard_normal((2, n, h)), dt)
    dh = held(rng.standard_normal((2, n, h)), dt)
    dr, d0 = rng.standard_normal((2, 2, n, h)).astype(F32)
    gds = n * 4 * h + 8
    G = Placed(nk, dev, gates, "f32", off, gds, 4 * h)
    DG = Placed(nk, dev, np.full((2, n, 4 * h), np.nan, F32), dt, off, gds, 4 * h)
    CP = Placed(nk, dev, c0, dt, off, n * h + 8, h)
    DH, DR, DC = out_like(nk, dev, dh, dt, off, n, h), Placed(nk, dev, dr, "f32", off, n * h, h), \
        Placed(nk, dev, d0, "f32", off, n * h, h)
    ck(nk, dev, nk._lib.lib.nk_lstm_bidir_bwd_step(dev.ctx, DG.ptr, D(nk, dt), gds, DC.ptr, G.ptr, CP.ptr, CP.stride,
                                                   DH.ptr if use_out else None, DH.stride, 2 * h,
                                                   DR.ptr if use_rec else None, n, h, D(nk, dt)))
    for d, (g, c) in enumerate(zip(DG.read(), DC.read())):
        wg, wdc = R.lstm_pointwise_backward(gates[d], c0[d], use_out * dh[d] + use_rec * dr[d], d0[d])
        scale = (1 + np.abs(d0[d]) + use_out * np.abs(dh[d]) + use_rec * np.abs(dr[d])) * (1 + np.abs(c0[d]))
        near(g, wg, step_tol(wg, tile(scale, 4), dt), f"dgates {d}")
        near(c, wdc, step_tol(wdc, scale, "f32"), f"dc {d}")
    assert np.array_equal(DH.read(), dh) and np.array_equal(DR.read(), dr) and np.array_equal(CP.read(), c0)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("n,h", STEP_SIZES)
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("use_out", [True, False])
def test_gru_bidir_bwd_step(nk, dev, dt, n, h, off, use_out):
    rng = np.random.default_rng([n, h, off, 4, use_out])
    ig = np.stack([gates_like(rng, n, 3, h) for _ in range(2)])
    hg = np.stack([gates_like(rng, n, 3, h) for _ in range(2)])
    h0 = held(rng.standard_normal((2, n, h)), dt)
    dh = held(rng.standard_normal((2, n, h)), dt)
    dr = rng.standard_normal((2, n, h)).astype(F32)
    gds = n * 3 * h + 8
    IG, HG = Placed(nk, dev, ig, "f32", off, gds, 3 * h), Placed(nk, dev, hg, "f32", off, gds, 3 * h)
    nan = np.full((2, n, 3 * h), np.nan, F32)
    DI, DHG = Placed(nk, dev, nan, dt, off, gds, 3 * h), Placed(nk, dev, nan, dt, off, gds, 3 * h)
    HP, DH = out_like(nk, dev, h0, dt, off, n, h), out_like(nk, dev, dh, dt, off, n, h)   # h_prev read from the output
    DR = Placed(nk, dev, dr, "f32", off, n * h, h)
    ck(nk, dev, nk._lib.lib.nk_gru_bidir_bwd_step(dev.ctx, DI.ptr, DHG.ptr, D(nk, dt), gds, DR.ptr, IG.ptr, HG.ptr, HP.ptr,
                                                  HP.stride, 2 * h, DH.ptr if use_out else None, DH.stride, 2 * h, n, h,
                                                  D(nk, dt)))
    di, dhg, zdh = DI.read(), DHG.read(), DR.read()
    for d in range(2):
        wi, whg, wz = R.gru_pointwise_backward(ig[d], hg[d], h0[d], use_out * dh[d] + dr[d])
        scale = (1 + use_out * np.abs(dh[d]) + np.abs(dr[d])) * (1 + np.abs(h0[d]))
        near(di[d], wi, step_tol(wi, tile(scale, 3), dt), f"digates {d}")
        near(dhg[d], whg, step_tol(whg, tile(scale, 3), dt), f"dhgates {d}")
        near(zdh[d], wz, step_tol(wz, scale, "f32"), f"dh_rec {d}")
    assert np.array_equal(HP.read(), h0) and np.array_equal(DH.read(), dh)


# ------------------------------------------------------------------------------------------------ layers
NAMES = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")
KEYS = ("w_ih", "w_hh", "b_ih", "b_hh")


def make_module(nk, dev, kind, n_in, hidden, dt, layers, dirs, seed, dropout=0.0):
    cls = nk.nn.LSTM if kind == "lstm" else nk.nn.GRU
    # a one-layer, one-direction module takes the stacked form (and its (1, N, H) states) when given a dropout, which
    # one layer never applies
    if layers == 1 and dirs == 1 and dropout == 0.0:
        dropout = 0.5
    return cls(dev, n_in, hidden, D(nk, dt), grad_dtype=nk.F32 if dt == "bf16" else None,
               rng=np.random.default_rng(seed), num_layers=layers, bidirectional=dirs == 2, dropout=dropout)


def module_params(m):
    return [tuple(getattr(m, f"{name}_l{k}").data().astype(np.float64) for name in NAMES) for k in range(m.num_layers)]


def fwd_tol(want, dt, T, layers):
    return (2 * UB if dt == "bf16" else 1e-4) * T * layers * (1 + np.abs(want))


def grad_tol(mag, dt, T, layers):
    mag = np.asarray(mag, np.float64)
    return k_e(dt) * (2 * T + 2) * layers * (mag + mag.mean()) + 1e-9


def leaf(nk, dev, a, dt):
    return nk.from_ndarray(dev, a, D(nk, dt)).requires_grad(nk.F32 if dt == "bf16" else None)


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("layers", [1, 2, 3])
@pytest.mark.parametrize("dirs", [1, 2])
@pytest.mark.parametrize("T,n,n_in,hidden", [(3, 4, 10, 16), (2, 3, 5, 7)])
def test_layers_against_oracle(nk, dev, kind, dt, layers, dirs, T, n, n_in, hidden):
    """output, h_n, c_n and every gradient; hidden = 7 takes the scalar bodies and the one-GEMM-per-product path"""
    lstm = kind == "lstm"
    rng = np.random.default_rng([layers, dirs, T, hidden, len(kind), len(dt)])
    m = make_module(nk, dev, kind, n_in, hidden, dt, layers, dirs, 5)
    m.eval()
    params = module_params(m)
    LD = layers * dirs
    xs = held(rng.standard_normal((T, n, n_in)), dt)
    h0, c0 = (held(rng.standard_normal((LD, n, hidden)) * 0.5, dt) for _ in range(2))
    tgt = held(rng.standard_normal((T, n, dirs * hidden)) * 0.5, dt)
    tgt_h, tgt_c = (held(rng.standard_normal((LD, n, hidden)) * 0.5, dt) for _ in range(2))
    X, H0, C0 = leaf(nk, dev, xs, dt), leaf(nk, dev, h0, dt), leaf(nk, dev, c0, dt)
    res = m.forward((C0, H0), X) if lstm else m.forward(H0, X)
    y, hn = res[0], res[1]
    assert y.shape == (T, n, dirs * hidden) and hn.shape == (LD, n, hidden)
    loss = y.mse_loss(nk.from_ndarray(dev, tgt, D(nk, dt)), nk.Reduction.Sum) + \
        hn.mse_loss(nk.from_ndarray(dev, tgt_h, D(nk, dt)), nk.Reduction.Sum)
    if lstm:
        loss = loss + res[2].mse_loss(nk.from_ndarray(dev, tgt_c, D(nk, dt)), nk.Reduction.Sum)
    loss.forward()
    loss.backward(1.0)

    w_y, w_hn, w_cn, _ = K.stack_forward(lstm, xs, c0 if lstm else None, h0, params)
    near(y.data(), w_y, fwd_tol(w_y, dt, T, layers), "output")
    near(hn.data(), w_hn, fwd_tol(w_hn, dt, T, layers), "h_n")
    if lstm:
        near(res[2].data(), w_cn, fwd_tol(w_cn, dt, T, layers), "c_n")
    g, mag = K.stack_backward(lstm, xs, c0 if lstm else None, h0, params, 2.0 * (w_y - tgt), 2.0 * (w_hn - tgt_h),
                              2.0 * (w_cn - tgt_c) if lstm else None)
    for k in range(layers):
        for key, name in zip(KEYS, NAMES):
            near(getattr(m, f"{name}_l{k}").grad(), g[f"{key}{k}"], grad_tol(mag[f"{key}{k}"], dt, T, layers),
                 f"{name}_l{k}")
    near(X.grad(), g["x"], grad_tol(mag["x"], dt, T, layers), "dx")
    near(H0.grad(), g["h"], grad_tol(mag["h"], dt, T, layers), "dh0")
    if lstm:
        near(C0.grad(), g["c"], grad_tol(mag["c"], dt, T, layers), "dc0")


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_directions_match_one_direction_layers(nk, dev, kind, dt):
    """the forward half of a bidirectional layer is a one-direction layer with direction 0's parameters; the reverse
    half is a one-direction layer with direction 1's parameters on the time-reversed input (outputs, last states and
    every parameter gradient)"""
    import neuronika_b200.variable as V
    lstm = kind == "lstm"
    T, n, n_in, hidden = 5, 8, 24, 32
    rng = np.random.default_rng(31 + len(kind) + len(dt))
    G = (4 if lstm else 3) * hidden
    k = 1.0 / np.sqrt(hidden)
    w = [held(rng.uniform(-k, k, s), dt) for s in ((2, G, n_in), (2, G, hidden), (2, G), (2, G))]
    xs = held(rng.standard_normal((T, n, n_in)), dt)
    h0, c0 = (held(rng.standard_normal((2, n, hidden)) * 0.5, dt) for _ in range(2))
    tgt = held(rng.standard_normal((T, n, 2 * hidden)) * 0.5, dt)

    def run(x, sl, target):
        P = [leaf(nk, dev, p[sl], dt) for p in w]
        X = nk.from_ndarray(dev, x, D(nk, dt))
        Hs, Cs = (nk.from_ndarray(dev, s[sl], D(nk, dt)) for s in (h0, c0))
        out = V.lstm_layer(X, Cs, Hs, *P) if lstm else V.gru_layer(X, Hs, *P)
        loss = out[0].mse_loss(nk.from_ndarray(dev, target, D(nk, dt)), nk.Reduction.Sum)
        loss.forward()
        loss.backward(1.0)
        return [o.data() for o in out], [p.grad() for p in P]

    both, g2 = run(xs, slice(0, 2), tgt)
    fwd, g0 = run(xs, slice(0, 1), np.ascontiguousarray(tgt[..., :hidden]))
    rev, g1 = run(np.ascontiguousarray(xs[::-1]), slice(1, 2), np.ascontiguousarray(tgt[::-1, :, hidden:]))
    tol = lambda a: fwd_tol(a, dt, T, 1)
    near(both[0][..., :hidden], fwd[0], tol(fwd[0]), "forward half")
    near(both[0][..., hidden:], rev[0][::-1], tol(rev[0]), "reverse half")
    for i in range(1, len(both)):
        near(both[i][0], fwd[i][0], tol(fwd[i][0]), f"last state {i} direction 0")
        near(both[i][1], rev[i][0], tol(rev[i][0]), f"last state {i} direction 1")
    for a, b0, b1, name in zip(g2, g0, g1, NAMES):
        for d, b in ((0, b0[0]), (1, b1[0])):
            scale = np.abs(b) + np.abs(b).mean()
            near(a[d], b, k_e(dt) * (2 * T + 2) * scale + 1e-9, f"{name} direction {d}")


def test_stacked_module_layout(nk, dev):
    """torch's state shapes and parameter shapes; parameters listed layer by layer; the defaults keep the cell's form"""
    m = nk.nn.LSTM(dev, 6, 5, num_layers=3, bidirectional=True, rng=np.random.default_rng(1))
    shapes = [p.shape for p in m.parameters()]
    assert shapes == [(2, 20, 6), (2, 20, 5), (2, 20), (2, 20)] + [(2, 20, 10), (2, 20, 5), (2, 20), (2, 20)] * 2
    g = nk.nn.GRU(dev, 6, 5, num_layers=2, rng=np.random.default_rng(1))
    assert [p.shape for p in g.parameters()] == [(1, 15, 6), (1, 15, 5), (1, 15), (1, 15), (1, 15, 5), (1, 15, 5),
                                                 (1, 15), (1, 15)]
    plain = nk.nn.LSTM(dev, 6, 5, rng=np.random.default_rng(1))
    cell = nk.nn.LSTMCell(dev, 6, 5, rng=np.random.default_rng(1))
    assert sorted(vars(plain)) == sorted(vars(cell))
    for p, q in zip(plain.parameters(), cell.parameters()):
        assert np.array_equal(p.data(), q.data())
    x = nk.from_ndarray(dev, np.ones((4, 3, 6), F32))
    zeros = nk.from_ndarray(dev, np.zeros((6, 3, 5), F32))
    y, h_n, c_n = m.forward((zeros, zeros), x)
    assert y.shape == (4, 3, 10) and h_n.shape == (6, 3, 5) and c_n.shape == (6, 3, 5)


def test_dropout_between_layers_in_training_mode(nk, dev):
    """training mode: layer 0's output is masked by the Philox draw of dropout call 0 (criteria_oracle's restatement)
    before layer 1 reads it; eval mode: no mask"""
    T, n, n_in, hidden, p, seed = 3, 4, 8, 16, 0.4, 0xD00D
    m = make_module(nk, dev, "gru", n_in, hidden, "f32", 2, 2, 9, dropout=p)
    params = module_params(m)
    rng = np.random.default_rng(3)
    xs = rng.standard_normal((T, n, n_in)).astype(F32)
    h0 = (rng.standard_normal((4, n, hidden)) * 0.5).astype(F32)
    X, H0 = nk.from_ndarray(dev, xs), nk.from_ndarray(dev, h0)
    dev.manual_seed(seed)
    y, _ = m.forward(H0, X)
    y.forward()
    y0, _, _ = K.layer_forward(False, xs, None, h0[:2], params[0])
    keep = CO.dropout_keep(seed, 0, y0.size, p)
    y0m = CO.dropout_forward(y0.astype(F32), keep, p)
    want, _, _ = K.layer_forward(False, y0m, None, h0[2:], params[1])
    near(y.data(), want, fwd_tol(want, "f32", T, 2), "output after the masked layer 0")
    m.eval()
    y.forward()
    plain, _, _, _ = K.stack_forward(False, xs, None, h0, params)
    near(y.data(), plain, fwd_tol(plain, "f32", T, 2), "eval mode")


def test_captured_stacked_bidirectional_step_matches_eager(nk, dev):
    """zero_grad -> 2-layer bidirectional LSTM (dropout, eval mode) + mse -> backward -> SGD, captured once and replayed
    from the same parameters as an eager step: same output and weight gradients bit for bit, bias gradients (f32
    atomics) to rounding"""
    from neuronika_b200 import optim
    n, n_in, hidden, T = 32, 64, 64, 6
    rng = np.random.default_rng(22)
    m = make_module(nk, dev, "lstm", n_in, hidden, "bf16", 2, 2, 8, dropout=0.3)
    m.eval()
    params = m.parameters()
    init = [p.data().copy() for p in params]
    opt = optim.StochasticGD.new(0.01)
    for p in params:
        opt.register(p)
    x = nk.from_ndarray(dev, rng.standard_normal((T, n, n_in)).astype(F32), nk.BF16)
    tgt = nk.from_ndarray(dev, rng.standard_normal((T, n, 2 * hidden)).astype(F32), nk.BF16)
    zeros = nk.from_ndarray(dev, np.zeros((4, n, hidden), F32), nk.BF16)
    live = {}

    def step():
        opt.zero_grad()
        out = m.forward((zeros, zeros), x)[0]
        loss = out.mse_loss(tgt)
        loss.forward()
        loss.backward(1.0)
        live["out"] = out
        live["grads"] = [p.grad_array() for p in params]
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    step()                     # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [live["out"].data()] + [g.as_ndarray().copy() for g in live["grads"]]
    eager_w = [p.data().copy() for p in params]
    reset()
    with dev.capture(512 << 20) as cap:
        step()
    reset()
    cap.graph.launch()
    dev.synchronize()
    replay = [live["out"].data()] + [g.as_ndarray() for g in live["grads"]]
    names = ["output"] + [f"{nm}_l{k}" for k in range(2) for nm in NAMES]
    for name, a, b in zip(names, eager, replay):
        if "bias" in name:
            assert np.all(np.abs(a - b) <= 1e-6 * np.abs(a) + 1e-7), name
        else:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name
    assert np.abs(eager[1]).max() > 0
    for p, w in zip(params, eager_w):
        assert np.all(np.abs(p.data() - w) <= UB * np.abs(w) + 1e-7)
    cap.graph.close()
