"""LSTM / GRU sequence layers on the GPU: the two backward step kernels of csrc/nk_rnn.cu (nk_lstm_seq_bwd_step,
nk_gru_seq_bwd_step), the one-node-per-sequence graph ops (variable.lstm / variable.gru) and the nn.LSTM / nn.GRU layers.

Operator level: as tests/test_gpu_rnn.py -- the float64 oracle (tests/rnn_seq_oracle.py) on the same inputs, operands
as views into canary-filled buffers at offset 0 (vector body) or 1 element (scalar body).  The hidden-state gradient of a
step is the sum of two sources, so the bound of a gate gradient scales with |dh_out| + |dh_rec| + |dc| (and with
1 + |state|, which the forget / update gate gradients carry): 3e-6 of that scale for the f32 maths, plus one bf16
rounding of the value for a bf16 output.

Layer level: the whole sequence against the float64 oracle on the same (bf16-rounded) parameters and inputs.  The oracle
returns with every gradient the same sums over absolute values, `mag`; a device gradient is within
k_e * (2T + 2) * (mag + mean(mag)) of the oracle's, k_e as in test_gpu_rnn.py (3e-5 for f32, 2^-8 + 3e-5 for bf16: one
rounding of the gate gradients per term), the factor 2T + 2 for the roundings of the T hidden states that every later
step and every gradient reads.
"""
import numpy as np
import pytest

import rnn_seq_oracle as S
from test_gpu_rnn import D, F32, UB, Guarded, gates_like, held, k_e, leaf, make_cell, near, wave_rows

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


# ------------------------------------------------------------------------------------------------ operator level
HS = [1, 7, 64, 1000, 1024]
NS = [1, 3, 257]
SOURCES = [(True, True), (True, False), (False, True), (False, False)]   # (dh_out given, dh_rec given)


def step_tol(want, scale, dt):
    want = np.abs(np.asarray(want, np.float64))
    return 3e-6 * scale + (UB * want if dt == "bf16" else 0.0)


def tile(a, k):
    return np.concatenate([a] * k, axis=1)


def check_lstm_step(nk, dev, dt, n, h, off, gates, sources=SOURCES):
    from neuronika_b200 import ops
    rng = np.random.default_rng(h * 13 + n + off)
    c0 = held(rng.standard_normal((n, h)), dt)
    dh = held(rng.standard_normal((n, h)), dt)
    dr = rng.standard_normal((n, h)).astype(F32)
    d0 = rng.standard_normal((n, h)).astype(F32)
    G, C0 = Guarded(nk, dev, gates, "f32", off), Guarded(nk, dev, c0, dt, off)
    DH, DR = Guarded(nk, dev, dh, dt, off), Guarded(nk, dev, dr, "f32", off)
    for use_out, use_rec in sources:
        DG = Guarded(nk, dev, np.full((n, 4 * h), np.nan, F32), dt, off)
        DC = Guarded(nk, dev, d0, "f32", off)
        ops.lstm_seq_bwd_step(DG.view, DC.view, G.view, C0.view, DH.view if use_out else None, DR.view if use_rec else None)
        wg, wdc = S.lstm_seq_bwd_step(gates, c0, d0, dh if use_out else None, dr if use_rec else None)
        scale = (1 + np.abs(d0) + use_out * np.abs(dh) + use_rec * np.abs(dr)) * (1 + np.abs(c0))
        what = f"out={use_out} rec={use_rec}"
        near(DG.read(), wg, step_tol(wg, tile(scale, 4), dt), "dgates " + what)
        near(DC.read(), wdc, step_tol(wdc, scale, "f32"), "dc " + what)
    assert np.array_equal(G.read(), gates) and np.array_equal(C0.read(), c0)
    assert np.array_equal(DH.read(), dh) and np.array_equal(DR.read(), dr)


def check_gru_step(nk, dev, dt, n, h, off, ig, hg, sources=SOURCES):
    from neuronika_b200 import ops
    rng = np.random.default_rng(h * 17 + n + off)
    h0 = held(rng.standard_normal((n, h)), dt)
    dh = held(rng.standard_normal((n, h)), dt)
    dr = rng.standard_normal((n, h)).astype(F32)
    IG, HG, H0 = Guarded(nk, dev, ig, "f32", off), Guarded(nk, dev, hg, "f32", off), Guarded(nk, dev, h0, dt, off)
    DH = Guarded(nk, dev, dh, dt, off)
    for use_out, use_rec in sources:
        DI = Guarded(nk, dev, np.full((n, 3 * h), np.nan, F32), dt, off)
        DHG = Guarded(nk, dev, np.full((n, 3 * h), np.nan, F32), dt, off)
        DR = Guarded(nk, dev, dr, "f32", off)
        ops.gru_seq_bwd_step(DI.view, DHG.view, DR.view if use_rec else None, IG.view, HG.view, H0.view,
                             DH.view if use_out else None)
        wi, whg, wz = S.gru_seq_bwd_step(ig, hg, h0, dh if use_out else None, dr if use_rec else None)
        scale = (1 + use_out * np.abs(dh) + use_rec * np.abs(dr)) * (1 + np.abs(h0))
        what = f"out={use_out} rec={use_rec}"
        near(DI.read(), wi, step_tol(wi, tile(scale, 3), dt), "digates " + what)
        near(DHG.read(), whg, step_tol(whg, tile(scale, 3), dt), "dhgates " + what)
        if use_rec:
            near(DR.read(), wz, step_tol(wz, scale, "f32"), "dh_rec " + what)   # NULL: nothing carried, nothing written
    assert np.array_equal(IG.read(), ig) and np.array_equal(HG.read(), hg) and np.array_equal(H0.read(), h0)
    assert np.array_equal(DH.read(), dh)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", HS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("off", [0, 1])
def test_lstm_seq_bwd_step(nk, dev, dt, h, n, off):
    check_lstm_step(nk, dev, dt, n, h, off, gates_like(np.random.default_rng(h + n), n, 4, h))


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", HS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("off", [0, 1])
def test_gru_seq_bwd_step(nk, dev, dt, h, n, off):
    rng = np.random.default_rng(h + n + 1)
    check_gru_step(nk, dev, dt, n, h, off, gates_like(rng, n, 3, h), gates_like(rng, n, 3, h))


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", [1000, 1024])
def test_steps_past_one_wave(nk, dev, dt, h):
    """more vector units than one grid wave: the grid-stride loop covers the rest"""
    n = wave_rows(dev, h, dt)
    rng = np.random.default_rng(6)
    check_lstm_step(nk, dev, dt, n, h, 0, gates_like(rng, n, 4, h), sources=[(True, True)])
    check_gru_step(nk, dev, dt, n, h, 0, gates_like(rng, n, 3, h), gates_like(rng, n, 3, h), sources=[(True, True)])


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_steps_with_saturated_gates(nk, dev, dt):
    """+-30 and +-inf pre-activations: gates at 0 / 1 / +-1, finite gradients that match the oracle, no NaN"""
    from neuronika_b200 import ops
    n, h = 4, 16
    vals = np.array([30.0, -30.0, np.inf, -np.inf], F32)
    rng = np.random.default_rng(10)
    check_lstm_step(nk, dev, dt, n, h, 0, rng.choice(vals, (n, 4 * h)).astype(F32))
    ig, hg = rng.choice(vals, (n, 3 * h)).astype(F32), rng.choice(vals[:2], (n, 3 * h)).astype(F32)
    h0 = dev.from_ndarray(held(rng.standard_normal((n, h)), dt), D(nk, dt))
    ones, rec = dev.from_ndarray(np.ones((n, h), F32), D(nk, dt)), dev.from_ndarray(np.ones((n, h), F32))
    di, dhg = dev.zeros((n, 3 * h), D(nk, dt)), dev.zeros((n, 3 * h), D(nk, dt))
    ops.gru_seq_bwd_step(di, dhg, rec, dev.from_ndarray(ig), dev.from_ndarray(hg), h0, ones)
    assert np.isfinite(di.as_ndarray()).all() and np.isfinite(dhg.as_ndarray()).all()
    assert np.isfinite(rec.as_ndarray()).all()


# ------------------------------------------------------------------------------------------------ layer level
def make_layer(nk, dev, kind, n_in, hidden, dt, seed):
    cls = nk.nn.LSTM if kind == "lstm" else nk.nn.GRU
    return cls(dev, n_in, hidden, D(nk, dt), grad_dtype=nk.F32 if dt == "bf16" else None, rng=np.random.default_rng(seed))


NAMES = (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh"))


def grad_tol(mag, dt, T):
    mag = np.asarray(mag, np.float64)
    return k_e(dt) * (2 * T + 2) * (mag + mag.mean()) + 1e-9


def run_layer_against_oracle(nk, dev, kind, dt, T, n, n_in, hidden, state_diff, input_diff, through):
    rng = np.random.default_rng([len(kind), len(dt), T, n, int(state_diff), int(input_diff), len(through)])
    layer = make_layer(nk, dev, kind, n_in, hidden, dt, 3)
    W = [getattr(layer, name).data() for _, name in NAMES]
    xs_h = held(rng.standard_normal((T, n, n_in)), dt)
    h0 = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    c0 = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    tgt = held(rng.standard_normal((T, n, hidden)) * 0.5, dt)
    tgt_c = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    X = leaf(nk, dev, xs_h, dt, input_diff)
    H0, C0 = leaf(nk, dev, h0, dt, state_diff), leaf(nk, dev, c0, dt, state_diff)
    if kind == "lstm":
        out, c_last = layer.forward((C0, H0), X)
    else:
        out, c_last = layer.forward(H0, X), None
    assert out.shape == (T, n, hidden) and (c_last is None or c_last.shape == (n, hidden))
    assert isinstance(out, nk.VarDiff)   # the parameters are differentiable
    loss = None
    if through != "cell":
        loss = out.mse_loss(nk.from_ndarray(dev, tgt, D(nk, dt)), nk.Reduction.Sum)
    if through != "output":
        lc = c_last.mse_loss(nk.from_ndarray(dev, tgt_c, D(nk, dt)), nk.Reduction.Sum)
        loss = lc if loss is None else loss + lc
    loss.forward()
    loss.backward(1.0)

    if kind == "lstm":
        w_out, w_cs = S.lstm_seq_forward(xs_h, c0, h0, *W)
    else:
        w_out, w_cs = S.gru_seq_forward(xs_h, h0, *W), None
    fwd = (2 * UB if dt == "bf16" else 1e-4) * T
    near(out.data(), w_out, fwd * (1 + np.abs(w_out)), "output")
    if kind == "lstm":
        near(c_last.data(), w_cs[-1], fwd * (1 + np.abs(w_cs[-1])), "c_T")
    d_out = 2.0 * (w_out - tgt) if through != "cell" else None
    d_c = 2.0 * (w_cs[-1] - tgt_c) if through != "output" else None
    if kind == "lstm":
        g, mag = S.lstm_seq_backward(xs_h, c0, h0, *W, d_out, d_c)
    else:
        g, mag = S.gru_seq_backward(xs_h, h0, *W, d_out)
    for k, name in NAMES:
        near(getattr(layer, name).grad(), g[k], grad_tol(mag[k], dt, T), name)
    if input_diff:
        near(X.grad(), g["x"], grad_tol(mag["x"], dt, T), "dx")
    if state_diff:
        near(H0.grad(), g["h"], grad_tol(mag["h"], dt, T), "dh0")
        if kind == "lstm":
            near(C0.grad(), g["c"], grad_tol(mag["c"], dt, T), "dc0")


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("T", [1, 2, 5])
@pytest.mark.parametrize("state_diff,input_diff", [(False, False), (True, False), (False, True), (True, True)])
def test_layers_against_oracle(nk, dev, kind, dt, T, state_diff, input_diff):
    run_layer_against_oracle(nk, dev, kind, dt, T, 6, 40, 24, state_diff, input_diff,
                             "both" if kind == "lstm" else "output")


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("through", ["output", "cell"])
def test_lstm_gradient_through_one_result_only(nk, dev, dt, through):
    """`cell`: nothing writes the output's gradient, every step's dh_out is NULL; `output`: the running dc starts at zero"""
    run_layer_against_oracle(nk, dev, "lstm", dt, 3, 6, 40, 24, True, True, through)


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("T", [2, 5])
def test_time_slices_that_are_not_16_byte_aligned(nk, dev, kind, dt, T):
    """N*H = 21 is odd: the slices output[t], C[t] (and the GRU's f32 gates) start off a 16-byte boundary, so the gate
    kernels take their scalar body and the GEMMs whatever engine accepts such operands"""
    run_layer_against_oracle(nk, dev, kind, dt, T, 3, 5, 7, True, True, "both" if kind == "lstm" else "output")


# ------------------------------------------------------------------------------------------------ sequence vs unrolled cells
def with_same_type_grads(nk, dev, layer, dt):
    """the layer's parameters again as leaves whose gradients have the data's element type"""
    for _, name in NAMES:
        setattr(layer, name, nk.from_ndarray(dev, getattr(layer, name).data(), D(nk, dt)).requires_grad())
    return layer


def unrolled(nk, cell, kind, xs, state):
    """T cell steps; returns (stacked hidden states (T, N, H), last cell state or None)"""
    hs = []
    for x in xs:
        state = cell.forward(state, x)
        hs.append(state[1] if kind == "lstm" else state)
    return hs[0].stack(hs[1:], 0), (state[0] if kind == "lstm" else None)


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_sequence_matches_unrolled_cells_with_fewer_launches(nk, dev, kind, dt):
    from neuronika_b200 import ops
    T, n, n_in, hidden = 4, 64, 128, 64
    rng = np.random.default_rng(12)
    xs_h = held(rng.standard_normal((T, n, n_in)), dt)
    h_h = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    c_h = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    res = {}
    for mode in ("sequence", "unrolled"):
        # the same seed: the layer and the cell hold the same weights; leaf gradients of the data's element type, so no
        # mixed-type accumulation pass enters the launch count
        layer = with_same_type_grads(nk, dev, (make_layer if mode == "sequence" else make_cell)(nk, dev, kind, n_in, hidden, dt, 6), dt)
        h, c = (nk.from_ndarray(dev, a, D(nk, dt)).requires_grad() for a in (h_h, c_h))
        if mode == "sequence":
            x = nk.from_ndarray(dev, xs_h, D(nk, dt)).requires_grad()
            out = layer.forward((c, h), x) if kind == "lstm" else layer.forward(h, x)
            out = out[0] if kind == "lstm" else out
            xg = lambda: x.grad()
        else:
            xs = [nk.from_ndarray(dev, a, D(nk, dt)).requires_grad() for a in xs_h]
            out, _ = unrolled(nk, layer, kind, xs, (c, h) if kind == "lstm" else h)
            xg = lambda: np.stack([v.grad() for v in xs])
        dev.synchronize()
        l0 = dev.launches
        out.forward()
        l1 = dev.launches
        out.backward(1.0)
        l2 = dev.launches
        grads = [p.grad() for p in layer.parameters()] + [xg(), h.grad()] + ([c.grad()] if kind == "lstm" else [])
        res[mode] = (out.data(), grads, l1 - l0, l2 - l1)
    (ys, gs, fs, bs), (yu, gu, fu, bu) = res["sequence"], res["unrolled"]
    # the same arithmetic per step but for the element type of the carried state gradient (f32 in the sequence node,
    # the data's in the unrolled graph) and the order of the sums over T
    kb = 0.04 if dt == "bf16" else 1e-5
    assert np.max(np.abs(ys - yu)) <= kb * (1 + np.max(np.abs(yu))), "output"
    for a, b in zip(gs, gu):
        assert np.max(np.abs(a - b)) <= kb * (1 + np.max(np.abs(b))) * 4, a.shape
    G = (4 if kind == "lstm" else 3) * hidden
    dev.synchronize()
    u0 = dev.launches
    ops.unbroadcast_acc(dev.zeros((G,), D(nk, dt)), dev.zeros((T * n, G), D(nk, dt)), beta=0.0)
    u1 = dev.launches
    ops.unbroadcast_acc(dev.zeros((n, hidden), D(nk, dt)), dev.zeros((n, hidden), nk.F32), beta=0.0)
    ub, ua = u1 - u0, dev.launches - u1
    assert fs == 1 + 2 * T, fs      # X.W_ih^T, then per step h.W_hh^T and the gate kernel
    assert fs < fu, (fs, fu)
    assert bs < bu, (bs, bu)
    if dt == "bf16":   # one launch per GEMM on the tensor-core engine (the CUDA-core engine may add a split-K reduction)
        # the deferred fill of the root gradient; per step the step kernel and dh_rec = dG_t.W_hh; dW_hh (steps 1.. and
        # step 0), dW_ih, dX; the two bias column sums; the f32 state gradients converted into dhidden (and dcell_state)
        states = 2 if kind == "lstm" else 1
        assert bs == 1 + 2 * T + 2 + 1 + 1 + 2 * ub + states * ua, (bs, ub, ua)


# ------------------------------------------------------------------------------------------------ f32 state gradient
@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_bf16_state_gradients_no_further_from_the_oracle_than_unrolled_cells(nk, dev, kind):
    """T = 32 in bf16: the unrolled graph rounds the state gradient to bf16 at every step, the sequence node carries it in
    f32 and rounds once; its dhidden / dcell_state are at least as close to the float64 oracle"""
    T, n, n_in, hidden = 32, 16, 32, 64
    rng = np.random.default_rng(31)
    xs_h = held(rng.standard_normal((T, n, n_in)), "bf16")
    h_h = held(rng.standard_normal((n, hidden)) * 0.5, "bf16")
    c_h = held(rng.standard_normal((n, hidden)) * 0.5, "bf16")
    tgt = held(rng.standard_normal((n, hidden)), "bf16")
    err = {}
    for mode in ("sequence", "unrolled"):
        layer = (make_layer if mode == "sequence" else make_cell)(nk, dev, kind, n_in, hidden, "bf16", 5)
        W = [getattr(layer, name).data() for _, name in NAMES]
        # bf16 state gradients: the unrolled chain's own element type, and one rounding at the end for the sequence node
        h, c = (nk.from_ndarray(dev, a, nk.BF16).requires_grad() for a in (h_h, c_h))
        if mode == "sequence":
            x = nk.from_ndarray(dev, xs_h, nk.BF16)
            out = layer.forward((c, h), x) if kind == "lstm" else layer.forward(h, x)
            hs = out[0] if kind == "lstm" else out
            # the last step's hidden state, as the unrolled loss sees it: gradient only into output[T-1]
            last = hs.chunks((1, n, hidden))[T - 1]
            loss = last.mse_loss(nk.from_ndarray(dev, tgt.reshape(1, n, hidden), nk.BF16), nk.Reduction.Sum)
        else:
            state = (c, h) if kind == "lstm" else h
            for a in xs_h:
                state = layer.forward(state, nk.from_ndarray(dev, a, nk.BF16))
            loss = (state[1] if kind == "lstm" else state).mse_loss(nk.from_ndarray(dev, tgt, nk.BF16), nk.Reduction.Sum)
        loss.forward()
        loss.backward(1.0)
        if kind == "lstm":
            w_out, _ = S.lstm_seq_forward(xs_h, c_h, h_h, *W)
        else:
            w_out = S.gru_seq_forward(xs_h, h_h, *W)
        d_out = np.zeros_like(w_out)
        d_out[-1] = 2.0 * (w_out[-1] - tgt)
        if kind == "lstm":
            g, _ = S.lstm_seq_backward(xs_h, c_h, h_h, *W, d_out, None)
        else:
            g, _ = S.gru_seq_backward(xs_h, h_h, *W, d_out)
        err[mode] = [float(np.sqrt(np.mean((h.grad() - g["h"]) ** 2)) / np.sqrt(np.mean(g["h"] ** 2)))]
        if kind == "lstm":
            err[mode].append(float(np.sqrt(np.mean((c.grad() - g["c"]) ** 2)) / np.sqrt(np.mean(g["c"] ** 2))))
    for s, u in zip(err["sequence"], err["unrolled"]):
        assert s <= u * 1.05 + 1e-12, err    # rms relative error; 5 % for two chains of roundings that happen to tie


# ------------------------------------------------------------------------------------------------ tape protocol
@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_second_backward_doubles_leaf_gradients(nk, dev, kind):
    T, n, n_in, hidden = 3, 5, 16, 8
    rng = np.random.default_rng(2)
    layer = make_layer(nk, dev, kind, n_in, hidden, "f32", 4)
    x = leaf(nk, dev, rng.standard_normal((T, n, n_in)).astype(F32), "f32", True)
    h0 = leaf(nk, dev, rng.standard_normal((n, hidden)).astype(F32), "f32", True)
    c0 = leaf(nk, dev, rng.standard_normal((n, hidden)).astype(F32), "f32", True)
    out = layer.forward((c0, h0), x)[0] if kind == "lstm" else layer.forward(h0, x)
    out.forward()
    out.backward(1.0)
    leaves = layer.parameters() + [x, h0] + ([c0] if kind == "lstm" else [])
    first = [v.grad().copy() for v in leaves]
    out.backward(1.0)
    for v, g in zip(leaves, first):
        assert np.all(np.abs(v.grad() - 2 * g) <= 1e-6 * np.abs(g) + 1e-7), v.shape


def test_no_differentiable_operand_gives_plain_vars(nk, dev):
    T, n, n_in, hidden = 2, 3, 8, 8
    z = lambda *s: nk.from_ndarray(dev, np.zeros(s, F32))
    y, c = nk.variable.lstm(z(T, n, n_in), z(n, hidden), z(n, hidden), z(4 * hidden, n_in), z(4 * hidden, hidden),
                            z(4 * hidden), z(4 * hidden))
    assert type(y) is nk.Var and type(c) is nk.Var and y.history_len() == 1 and c.history_len() == 1
    y.forward()
    assert y.shape == (T, n, hidden) and not y.data().any()
    g = nk.variable.gru(z(T, n, n_in), z(n, hidden), z(3 * hidden, n_in), z(3 * hidden, hidden), z(3 * hidden),
                        z(3 * hidden))
    assert type(g) is nk.Var and g.history_len() == 1


def test_layer_and_cell_from_one_seed_hold_the_same_weights(nk, dev):
    for kind in ("lstm", "gru"):
        a, b = make_layer(nk, dev, kind, 12, 8, "bf16", 11), make_cell(nk, dev, kind, 12, 8, "bf16", 11)
        assert len(a.parameters()) == 4
        for p, q in zip(a.parameters(), b.parameters()):
            assert p.shape == q.shape and p.grad_dtype == q.grad_dtype and np.array_equal(p.data(), q.data())


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_captured_sequence_step_matches_eager(nk, dev, kind):
    """zero_grad -> sequence layer + mse over every step's hidden state -> backward -> SGD, captured once and replayed
    from the same parameters as an eager step: same output and weight gradients bit for bit, bias gradients (f32
    atomics) to rounding"""
    from neuronika_b200 import optim
    n, n_in, hidden, T = 32, 64, 64, 8
    rng = np.random.default_rng(21)
    layer = make_layer(nk, dev, kind, n_in, hidden, "bf16", 7)
    params = layer.parameters()
    init = [p.data().copy() for p in params]
    opt = optim.StochasticGD.new(0.01)
    for p in params:
        opt.register(p)
    x = nk.from_ndarray(dev, rng.standard_normal((T, n, n_in)).astype(F32), nk.BF16)
    tgt = nk.from_ndarray(dev, rng.standard_normal((T, n, hidden)).astype(F32), nk.BF16)
    zeros = nk.from_ndarray(dev, np.zeros((n, hidden), F32), nk.BF16)
    live = {}

    def step():
        opt.zero_grad()
        out = layer.forward((zeros, zeros), x)[0] if kind == "lstm" else layer.forward(zeros, x)
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
    with dev.capture(256 << 20) as cap:
        step()
    reset()
    cap.graph.launch()
    dev.synchronize()
    replay = [live["out"].data()] + [g.as_ndarray() for g in live["grads"]]
    for name, a, b in zip(["output", "weight_ih", "weight_hh", "bias_ih", "bias_hh"], eager, replay):
        if "bias" in name:
            assert np.all(np.abs(a - b) <= 1e-6 * np.abs(a) + 1e-7), name
        else:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name
    assert np.abs(eager[1]).max() > 0
    for p, w in zip(params, eager_w):
        assert np.all(np.abs(p.data() - w) <= UB * np.abs(w) + 1e-7)
    cap.graph.close()


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_hooks_and_reduce_scatter_plan_report_once_per_backward(nk, dev, kind):
    """one node writes each weight gradient: its hook fires once per backward(), after the last GEMM into it, and a
    weight with a reduce-scatter plan (world = 2 on one GPU; the slot buffers are never written) is computed locally and
    reported as not pushed once, with the gradient it has without a plan, bit for bit"""
    T, n, n_in, hidden = 4, 8, 256, 256
    G = (4 if kind == "lstm" else 3) * hidden
    rng = np.random.default_rng(17)
    x_h = rng.standard_normal((T, n, n_in)).astype(F32)
    grads, slots = [], []
    seen = {"hook_ih": [], "hook_hh": [], "rs_ih": [], "rs_hh": []}
    for planned in (False, True):
        layer = make_layer(nk, dev, kind, n_in, hidden, "bf16", 13)
        if planned:
            for key, w in (("ih", layer.weight_ih), ("hh", layer.weight_hh)):
                bufs = [dev.zeros((int(np.prod(w.shape)),), nk.F32) for _ in range(2)]
                slots.append(bufs)
                w.set_grad_hook(lambda b, e, key=key: seen["hook_" + key].append((b, e)))
                w.set_grad_rs(2, 0, [b.ptr.value for b in bufs], lambda pushed, key=key: seen["rs_" + key].append(pushed))
        zero = nk.zeros(dev, (n, hidden), nk.BF16)
        x = nk.from_ndarray(dev, x_h, nk.BF16)
        out = layer.forward((zero, zero), x)[0] if kind == "lstm" else layer.forward(zero, x)
        loss = out.sum()
        loss.forward()
        for k in (1, 2):
            loss.backward(1.0)
            if planned:
                assert seen["hook_ih"] == [(0, G * n_in)] * k and seen["hook_hh"] == [(0, G * hidden)] * k, seen
                assert seen["rs_ih"] == [0] * k and seen["rs_hh"] == [0] * k, seen
        grads.append([layer.weight_ih.grad(), layer.weight_hh.grad()])
        if planned:
            for w in (layer.weight_ih, layer.weight_hh):
                w.set_grad_rs(0, 0, None, None)
                w.set_grad_hook(None)
    for a, b in zip(*grads):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for bufs in slots:
        for b in bufs:
            assert not b.as_ndarray().any()


# ------------------------------------------------------------------------------------------------ errors
def test_shape_rank_type_and_device_errors(nk, dev):
    """host-side checks: every message names the argument; nothing is launched"""
    V = nk.variable
    z = lambda *s, dt=None: nk.from_ndarray(dev, np.zeros(s, F32), dt if dt is not None else nk.F32)
    T, n, n_in, hidden = 2, 3, 8, 4
    x, h = z(T, n, n_in), z(n, hidden)
    lw = [z(4 * hidden, n_in), z(4 * hidden, hidden), z(4 * hidden), z(4 * hidden)]
    gw = [z(3 * hidden, n_in), z(3 * hidden, hidden), z(3 * hidden), z(3 * hidden)]
    dev.synchronize()
    before = dev.launches
    with pytest.raises(nk.NkError, match=r"lstm: input must be \(seq_len, batch, input_size\), got \(3, 8\)"):
        V.lstm(z(n, n_in), h, h, *lw)
    with pytest.raises(nk.NkError, match=r"gru: input must be \(seq_len, batch, input_size\), got \(2, 3, 8, 1\)"):
        V.gru(z(T, n, n_in, 1), h, *gw)
    with pytest.raises(nk.NkError, match=r"lstm: hidden must be \(batch = 3, hidden_size\), got \(2, 4\)"):
        V.lstm(x, h, z(2, hidden), *lw)
    with pytest.raises(nk.NkError, match=r"lstm: cell_state must be \(3, 4\), got \(3, 5\)"):
        V.lstm(x, z(n, 5), h, *lw)
    with pytest.raises(nk.NkError, match=r"lstm: weight_ih must be \(16, 9\), got \(16, 8\)"):
        V.lstm(z(T, n, 9), h, h, *lw)
    with pytest.raises(nk.NkError, match=r"gru: weight_hh must be \(12, 4\), got \(16, 4\)"):
        V.gru(x, h, gw[0], lw[1], gw[2], gw[3])
    with pytest.raises(nk.NkError, match=r"gru: bias_ih must be \(12,\), got \(16,\)"):
        V.gru(x, h, gw[0], gw[1], lw[2], gw[3])
    with pytest.raises(nk.NkError, match=r"gru: bias_hh must be \(12,\), got \(16,\)"):
        V.gru(x, h, gw[0], gw[1], gw[2], lw[3])
    with pytest.raises(nk.NkError, match="lstm: cell_state has another element type than the input"):
        V.lstm(x, z(n, hidden, dt=nk.BF16), h, *lw)
    with pytest.raises(nk.NkError, match="gru: weight_ih has another element type than the input"):
        V.gru(x, h, z(3 * hidden, n_in, dt=nk.BF16), *gw[1:])
    with pytest.raises(nk.NkError, match=r"gru: input needs at least one time step, got \(0, 3, 8\)"):
        V.gru(z(0, n, n_in), h, *gw)
    other = nk.Device(0)      # a second context on the same GPU is another device to the graph
    with pytest.raises(nk.NkError, match="lstm: hidden lives on another device than the input"):
        V.lstm(x, h, nk.from_ndarray(other, np.zeros((n, hidden), F32)), *lw)
    dev.synchronize()
    assert dev.launches == before
