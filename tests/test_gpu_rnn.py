"""LSTM / GRU cells and `chunks` on the GPU: the six entry points of csrc/nk_rnn.cu, the fused graph nodes and the
nn.LSTMCell / nn.GRUCell layers.

Operator level: every entry point against the float64 oracle (tests/rnn_oracle.py) on the same f32 / bf16 inputs, at H
around the 4- and 8-wide vector bodies, N around the row count and past one grid wave (8 CTAs x 256 threads per SM).
Operands are views into canary-filled buffers, at offset 0 (16-byte aligned: vector body) or 1 element (scalar body);
every element outside an output view must keep its canary bit for bit, and outputs written with beta = 0 start as NaN.
Bounds: an f32 result is within 2e-6 * (1 + |want|) of the float64 value (expf / tanhf are a few ulp; the values are
products of at most five O(1) factors); a bf16 output adds one rounding, 2^-8 * |want|.

Layer level: against torch CPU float64 on the same bf16-rounded parameters and inputs.  Multi-step checks go one step at
a time: step t of the oracle is fed the states and the output gradients the device stored, so the bound of each step is
that of one step.  A product sum_k a_k b_k (GEMM, column sums) is within k_e * S of the float64 value, S = sum_k |a_k b_k|
computed by the oracle: k_e = 3e-5 for f32 cells (SIMT GEMM, f32 gate gradients, and the f32 gates the step recomputes
its activations from), 2^-8 + 3e-5 for bf16 cells (the gate gradient is stored in bf16 for the tensor-core GEMMs: one
rounding per term).
"""
import numpy as np
import pytest

import rnn_oracle as R

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0
UB = 2.0 ** -8
VEC = {"f32": 4, "bf16": 8}


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


class Guarded:
    """`data` (float32 values the storage type holds) at element `off` of a canary-filled device buffer"""

    def __init__(self, nk, dev, data, dt, off=0, tail=24):
        data = np.asarray(data, F32)
        self.shape, self.n, self.off = data.shape, data.size, off
        host = np.full(off + self.n + tail, CANARY, F32)
        host[off:off + self.n] = data.ravel()
        self.buf = dev.from_ndarray(host, D(nk, dt))
        self.view = self.buf.slice_flat(off, self.shape)
        assert (self.view.ptr.value % 16 == 0) == (off == 0)

    def read(self):
        flat = self.buf.as_ndarray().ravel()
        outside = np.concatenate([flat[:self.off], flat[self.off + self.n:]])
        bad = np.flatnonzero(outside.view(np.uint32) != F32(CANARY).view(np.uint32))
        assert bad.size == 0, f"{bad.size} elements outside the view were written"
        return flat[self.off:self.off + self.n].reshape(self.shape)


def near(got, want, tol, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - want)
    bad = np.flatnonzero(~(err <= tol))
    assert bad.size == 0, (what, f"{bad.size} of {got.size} outside", float(got.ravel()[bad[0]]),
                           float(want.ravel()[bad[0]]), float(np.broadcast_to(tol, got.shape).ravel()[bad[0]]))


def pw_tol(want, dt):
    want = np.abs(np.asarray(want, np.float64))
    return 2e-6 * (1 + want) + (UB * want if dt == "bf16" else 0.0)


def wave_rows(dev, hidden, dt):
    """rows that put one more row than a full grid wave of vector units on the device"""
    return dev.sm_count * 8 * 256 * VEC[dt] // hidden + 1


# ------------------------------------------------------------------------------------------------ operator level
HS = [1, 7, 8, 9, 1000, 1024]
NS = [1, 3, 257]


def gates_like(rng, n, g, h):
    return (rng.standard_normal((n, g * h)) * 2).astype(F32)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", HS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("off", [0, 1])
def test_lstm_cell_ops(nk, dev, dt, h, n, off):
    from neuronika_b200 import ops
    rng = np.random.default_rng(h * 7 + n + off)
    gates = gates_like(rng, n, 4, h)
    c0 = held(rng.standard_normal((n, h)), dt)
    G = Guarded(nk, dev, gates, "f32", off)
    C0 = Guarded(nk, dev, c0, dt, off)
    CO = Guarded(nk, dev, np.full((n, h), np.nan, F32), dt, off)
    HO = Guarded(nk, dev, np.full((n, h), np.nan, F32), dt, off)
    ops.lstm_cell(G.view, C0.view, CO.view, HO.view)
    wc, wh = R.lstm_pointwise(gates, c0)
    near(CO.read(), wc, pw_tol(wc, dt), "c'")
    near(HO.read(), wh, pw_tol(wh, dt), "h'")
    assert np.array_equal(G.read(), gates) and np.array_equal(C0.read(), c0)
    # backward: (beta 0, both output gradients), (beta 1, dh NULL), (dc NULL, dc_prev NULL)
    dh = held(rng.standard_normal((n, h)), dt)
    dc = held(rng.standard_normal((n, h)), dt)
    d0 = held(rng.standard_normal((n, h)), dt)
    for mode in ("beta0", "beta1_no_dh", "no_dc_no_dcprev"):
        use_dh, use_dc = mode != "beta1_no_dh", mode != "no_dc_no_dcprev"
        beta = 1.0 if mode == "beta1_no_dh" else 0.0
        DH, DC = Guarded(nk, dev, dh, dt, off), Guarded(nk, dev, dc, dt, off)
        DG = Guarded(nk, dev, np.full((n, 4 * h), np.nan, F32), dt, off)
        DP = None if mode == "no_dc_no_dcprev" else Guarded(nk, dev, d0 if beta else np.full((n, h), np.nan, F32), dt, off)
        ops.lstm_cell_bwd(DG.view, G.view, C0.view, DH.view if use_dh else None, DC.view if use_dc else None,
                          DP.view if DP else None, beta_dc=beta)
        wg, wdc = R.lstm_pointwise_backward(gates, c0, dh if use_dh else None, dc if use_dc else None)
        near(DG.read(), wg, pw_tol(wg, dt), f"dgates {mode}")
        if DP:
            want = wdc + beta * d0
            near(DP.read(), want, pw_tol(want, dt) + 2e-6 * beta * np.abs(d0), f"dc_prev {mode}")
        DH.read(), DC.read()


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", HS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("off", [0, 1])
def test_gru_cell_ops(nk, dev, dt, h, n, off):
    from neuronika_b200 import ops
    rng = np.random.default_rng(h * 11 + n + off)
    ig, hg = gates_like(rng, n, 3, h), gates_like(rng, n, 3, h)
    h0 = held(rng.standard_normal((n, h)), dt)
    IG, HG, H0 = Guarded(nk, dev, ig, "f32", off), Guarded(nk, dev, hg, "f32", off), Guarded(nk, dev, h0, dt, off)
    HO = Guarded(nk, dev, np.full((n, h), np.nan, F32), dt, off)
    ops.gru_cell(IG.view, HG.view, H0.view, HO.view)
    wh = R.gru_pointwise(ig, hg, h0)
    near(HO.read(), wh, pw_tol(wh, dt) + 2e-6 * np.abs(h0), "h'")
    dh = held(rng.standard_normal((n, h)), dt)
    d0 = held(rng.standard_normal((n, h)), dt)
    for beta, with_prev in ((0.0, True), (1.0, True), (0.0, False)):
        DH = Guarded(nk, dev, dh, dt, off)
        DI = Guarded(nk, dev, np.full((n, 3 * h), np.nan, F32), dt, off)
        DHG = Guarded(nk, dev, np.full((n, 3 * h), np.nan, F32), dt, off)
        DP = Guarded(nk, dev, d0 if beta else np.full((n, h), np.nan, F32), dt, off) if with_prev else None
        ops.gru_cell_bwd(DI.view, DHG.view, IG.view, HG.view, H0.view, DH.view, DP.view if DP else None, beta_dh=beta)
        wi, whg, wp = R.gru_pointwise_backward(ig, hg, h0, dh)
        # dz carries (h - nn): its magnitude bound includes |h|
        t_extra = 2e-6 * np.abs(np.concatenate([h0, h0, h0], 1) * np.concatenate([dh, dh, dh], 1))
        near(DI.read(), wi, pw_tol(wi, dt) + t_extra, f"digates beta={beta}")
        near(DHG.read(), whg, pw_tol(whg, dt) + t_extra, f"dhgates beta={beta}")
        if DP:
            want = wp + beta * d0
            near(DP.read(), want, pw_tol(want, dt) + 2e-6 * beta * np.abs(d0), f"dh_prev beta={beta}")
        DH.read()


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("h", [1000, 1024])
def test_cells_past_one_wave(nk, dev, dt, h):
    """more vector units than one grid wave: the grid-stride loop covers the rest"""
    from neuronika_b200 import ops
    n = wave_rows(dev, h, dt)
    rng = np.random.default_rng(5)
    gates = gates_like(rng, n, 4, h)
    c0 = held(rng.standard_normal((n, h)), dt)
    g, c = dev.from_ndarray(gates), dev.from_ndarray(c0, D(nk, dt))
    co, ho = ops.lstm_cell(g, c)
    wc, wh = R.lstm_pointwise(gates, c0)
    near(co.as_ndarray(), wc, pw_tol(wc, dt), "c'")
    near(ho.as_ndarray(), wh, pw_tol(wh, dt), "h'")
    dh = held(rng.standard_normal((n, h)), dt)
    dg = dev.zeros((n, 4 * h), D(nk, dt))
    dcp = dev.zeros((n, h), D(nk, dt))
    ops.lstm_cell_bwd(dg, g, c, dev.from_ndarray(dh, D(nk, dt)), None, dcp, beta_dc=0.0)
    wg, wdc = R.lstm_pointwise_backward(gates, c0, dh, None)
    near(dg.as_ndarray(), wg, pw_tol(wg, dt), "dgates")
    near(dcp.as_ndarray(), wdc, pw_tol(wdc, dt), "dc_prev")
    ig, hg = gates_like(rng, n, 3, h), gates_like(rng, n, 3, h)
    hp = ops.gru_cell(dev.from_ndarray(ig), dev.from_ndarray(hg), c)
    wh = R.gru_pointwise(ig, hg, c0)
    near(hp.as_ndarray(), wh, pw_tol(wh, dt) + 2e-6 * np.abs(c0), "gru h'")


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_saturated_gates(nk, dev, dt):
    """+-30 and +-inf pre-activations: gates at 0 / 1 / +-1, finite values and gradients, no NaN"""
    from neuronika_b200 import ops
    n, h = 4, 16
    vals = np.array([30.0, -30.0, np.inf, -np.inf], F32)
    rng = np.random.default_rng(9)
    gates = rng.choice(vals, (n, 4 * h)).astype(F32)
    c0 = held(rng.standard_normal((n, h)), dt)
    g, c = dev.from_ndarray(gates), dev.from_ndarray(c0, D(nk, dt))
    co, ho = ops.lstm_cell(g, c)
    wc, wh = R.lstm_pointwise(gates, c0)
    near(co.as_ndarray(), wc, pw_tol(wc, dt), "c'")
    near(ho.as_ndarray(), wh, pw_tol(wh, dt), "h'")
    ones = dev.from_ndarray(np.ones((n, h), F32), D(nk, dt))
    dg, dcp = dev.zeros((n, 4 * h), D(nk, dt)), dev.zeros((n, h), D(nk, dt))
    ops.lstm_cell_bwd(dg, g, c, ones, ones, dcp, beta_dc=0.0)
    wg, wdc = R.lstm_pointwise_backward(gates, c0, np.ones((n, h)), np.ones((n, h)))
    near(dg.as_ndarray(), wg, pw_tol(wg, dt), "dgates")
    near(dcp.as_ndarray(), wdc, pw_tol(wdc, dt), "dc_prev")
    ig, hg = rng.choice(vals, (n, 3 * h)).astype(F32), rng.choice(vals[:2], (n, 3 * h)).astype(F32)
    hp = ops.gru_cell(dev.from_ndarray(ig), dev.from_ndarray(hg), c)
    assert np.isfinite(hp.as_ndarray()).all()
    di, dhg = dev.zeros((n, 3 * h), D(nk, dt)), dev.zeros((n, 3 * h), D(nk, dt))
    ops.gru_cell_bwd(di, dhg, dev.from_ndarray(ig), dev.from_ndarray(hg), c, ones, dcp, beta_dh=0.0)
    assert np.isfinite(di.as_ndarray()).all() and np.isfinite(dhg.as_ndarray()).all()


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("shape,chunk", [((3, 3), (1, 3)), ((5, 7), (2, 3)), ((4, 6, 10), (2, 3, 5)),
                                         ((257, 4096), (257, 1024))])
@pytest.mark.parametrize("off", [0, 1])
def test_chunk_ops_bit_exact(nk, dev, dt, shape, chunk, off):
    from neuronika_b200 import ops
    rng = np.random.default_rng(len(shape) + off)
    x = held(rng.standard_normal(shape), dt)
    X = Guarded(nk, dev, x, dt, off)
    blocks = R.chunks(x, chunk)
    for i, want in enumerate(blocks):
        Y = Guarded(nk, dev, np.full(chunk, np.nan, F32), dt, off)
        ops.chunk(X.view, chunk, i, out=Y.view)
        got = Y.read()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"block {i}"
    d0 = held(rng.standard_normal(shape), dt)
    for i in (0, len(blocks) - 1):
        g = held(rng.standard_normal(chunk), dt)
        for beta in (0.0, 1.0):
            DX = Guarded(nk, dev, d0, dt, off)
            G = Guarded(nk, dev, g, dt, off)
            ops.chunk_bwd(DX.view, G.view, i, beta=beta)
            want = d0.copy()
            sl = R.chunk_slices(shape, chunk, i)
            want[sl] = held((beta * d0[sl].astype(F32) + g).astype(F32), dt)
            assert np.array_equal(DX.read().view(np.uint32), want.view(np.uint32)), f"bwd block {i} beta {beta}"


# ------------------------------------------------------------------------------------------------ layer level
def make_cell(nk, dev, kind, n_in, hidden, dt, seed):
    cls = nk.nn.LSTMCell if kind == "lstm" else nk.nn.GRUCell
    grad_dt = nk.F32 if dt == "bf16" else None
    return cls(dev, n_in, hidden, D(nk, dt), grad_dtype=grad_dt, rng=np.random.default_rng(seed))


def leaf(nk, dev, a, dt, diff):
    v = nk.from_ndarray(dev, a, D(nk, dt))
    return v.requires_grad(nk.F32 if dt == "bf16" else None) if diff else v


def k_e(dt):
    return UB + 3e-5 if dt == "bf16" else 3e-5


def unroll(cell, xs, state):
    """T steps; returns the per-step outputs ((c, h) for the LSTM, h for the GRU)"""
    outs = []
    for x in xs:
        state = cell.forward(state, x)
        outs.append(state)
    return outs


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("T", [1, 5])
@pytest.mark.parametrize("state_diff,input_diff", [(False, False), (True, False), (False, True), (True, True)])
def test_cell_layers_against_torch(nk, dev, kind, dt, T, state_diff, input_diff):
    import torch
    n, n_in, hidden = 6, 40, 24
    rng = np.random.default_rng([len(kind), len(dt), T, int(state_diff), int(input_diff)])
    cell = make_cell(nk, dev, kind, n_in, hidden, dt, 3)
    P = {k: getattr(cell, k).data() for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
    xs_h = [held(rng.standard_normal((n, n_in)), dt) for _ in range(T)]
    h0 = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    c0 = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    tgt = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    xs = [leaf(nk, dev, x, dt, input_diff) for x in xs_h]
    H0, C0 = leaf(nk, dev, h0, dt, state_diff), leaf(nk, dev, c0, dt, state_diff)
    outs = unroll(cell, xs, (C0, H0) if kind == "lstm" else H0)
    hT = outs[-1][1] if kind == "lstm" else outs[-1]
    loss = hT.mse_loss(nk.from_ndarray(dev, tgt, D(nk, dt)))
    loss.forward()
    loss.backward(1.0)
    ke, kf = k_e(dt), (UB if dt == "bf16" else 0.0)

    # forward, one step at a time from the states the device stored
    hs = [h0] + [(o[1] if kind == "lstm" else o).data() for o in outs]
    cs = [c0] + [o[0].data() for o in outs] if kind == "lstm" else None
    W = [P["weight_ih"], P["weight_hh"], P["bias_ih"], P["bias_hh"]]
    for t in range(T):
        if kind == "lstm":
            g = R.lstm_gates(xs_h[t], hs[t], *W)
            S = np.abs(xs_h[t]) @ np.abs(W[0]).T + np.abs(hs[t]) @ np.abs(W[1]).T + np.abs(W[2]) + np.abs(W[3])
            S = S.reshape(n, 4, hidden).max(1)
            wc, wh = R.lstm_pointwise(g, cs[t])
            # a gate error e moves c' and h' by at most e (the derivatives of sigmoid / tanh are <= 1, |c| enters once)
            tc = 1e-5 * S * (1 + np.abs(cs[t])) + 2e-6 * (1 + np.abs(wc)) + kf * np.abs(wc)
            near(cs[t + 1], wc, tc, f"c[{t + 1}]")
            near(hs[t + 1], wh, 1e-5 * S * (1 + np.abs(cs[t])) + 2e-6 + kf * np.abs(wh), f"h[{t + 1}]")
        else:
            ig, hg = R.gru_gates(xs_h[t], hs[t], *W)
            S = np.abs(xs_h[t]) @ np.abs(W[0]).T + np.abs(hs[t]) @ np.abs(W[1]).T + np.abs(W[2]) + np.abs(W[3])
            S = S.reshape(n, 3, hidden).max(1)
            wh = R.gru_pointwise(ig, hg, hs[t])
            near(hs[t + 1], wh, 1e-5 * S * (2 + np.abs(hs[t])) + 2e-6 * (1 + np.abs(wh)) + kf * np.abs(wh), f"h[{t + 1}]")

    # the last step against torch float64 end to end: h_T, and the loss gradient seed
    hT64 = hs[-1].astype(np.float64)
    dhT = 2.0 * (hT.data().astype(np.float64) - tgt) / tgt.size
    # backward, one step at a time from the output gradients the device stored
    dh = [None] * (T + 1)
    dc = [None] * (T + 1)
    for t in range(1, T + 1):
        o = outs[t - 1]
        dh[t] = (o[1] if kind == "lstm" else o).grad().astype(np.float64)
        if kind == "lstm":
            dc[t] = o[0].grad().astype(np.float64) if t < T else None
    near(dh[T], dhT, 2e-6 * np.abs(dhT) + kf * np.abs(dhT) + 1e-9, "dh_T (mse)")
    def dc_tol(t):
        # dc_prev = f * (dc + dh*o*(1 - tanh^2 c')): pointwise in f32 from gates within 3e-5 * S of the float64 ones
        g = R.lstm_gates(xs_h[t - 1], hs[t - 1], *W)
        S = np.abs(xs_h[t - 1]) @ np.abs(W[0]).T + np.abs(hs[t - 1]) @ np.abs(W[1]).T + 1
        S = S.reshape(n, 4, hidden).max(1)
        _, want = R.lstm_pointwise_backward(g, cs[t - 1], dh[t], dc[t])
        mag = (0 if dc[t] is None else np.abs(dc[t])) + np.abs(dh[t])
        return (2e-6 + 3e-5 * S * (1 + np.abs(cs[t - 1]))) * mag + kf * np.abs(want) + 1e-9

    acc = {k: 0.0 for k in ("w_ih", "w_hh", "b_ih", "b_hh")}
    tolw = {k: 0.0 for k in acc}
    Wa = [np.abs(w) for w in W]
    for t in range(T, 0, -1):
        x, hp = xs_h[t - 1], hs[t - 1]
        if kind == "lstm":
            g = R.lstm_gates(x, hp, *W)
            dg, dcp = R.lstm_pointwise_backward(g, cs[t - 1], dh[t], dc[t])
            dgi = dgh = dg
        else:
            ig, hg = R.gru_gates(x, hp, *W)
            dgi, dgh, dhp = R.gru_pointwise_backward(ig, hg, hp, dh[t])
        acc["w_ih"] = acc["w_ih"] + dgi.T @ x
        acc["w_hh"] = acc["w_hh"] + dgh.T @ hp
        acc["b_ih"] = acc["b_ih"] + dgi.sum(0)
        acc["b_hh"] = acc["b_hh"] + dgh.sum(0)
        tolw["w_ih"] = tolw["w_ih"] + np.abs(dgi).T @ np.abs(x)
        tolw["w_hh"] = tolw["w_hh"] + np.abs(dgh).T @ np.abs(hp)
        tolw["b_ih"] = tolw["b_ih"] + np.abs(dgi).sum(0)
        tolw["b_hh"] = tolw["b_hh"] + np.abs(dgh).sum(0)
        # the gradients of the step's inputs
        want_h = dgh @ W[1] + (dhp if kind == "gru" else 0.0)
        tol_h = ke * (np.abs(dgh) @ Wa[1] + (np.abs(dhp) if kind == "gru" else 0.0)) + kf * np.abs(want_h) + 1e-9
        if t > 1:
            o = outs[t - 2]
            near((o[1] if kind == "lstm" else o).grad(), want_h, tol_h, f"dh[{t - 1}]")
            if kind == "lstm":
                near(o[0].grad(), dcp, dc_tol(t), f"dc[{t - 1}]")
        else:
            if state_diff:
                near(H0.grad(), want_h, tol_h, "dh0")
                if kind == "lstm":
                    near(C0.grad(), dcp, dc_tol(t), "dc0")
        if input_diff:
            want_x = dgi @ W[0]
            near(xs[t - 1].grad(), want_x, ke * (np.abs(dgi) @ Wa[0]) + 1e-9, f"dx[{t - 1}]")
    for k, name in (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh")):
        near(getattr(cell, name).grad(), acc[k], ke * tolw[k] + 1e-9, name)

    # and the whole unrolled sequence against torch.nn.*Cell in float64 (same parameters, same inputs): the composition
    # of T rounded steps stays close to the exact one
    tc_ = (torch.nn.LSTMCell if kind == "lstm" else torch.nn.GRUCell)(n_in, hidden).double()
    with torch.no_grad():
        for p, k in zip((tc_.weight_ih, tc_.weight_hh, tc_.bias_ih, tc_.bias_hh), ("weight_ih", "weight_hh", "bias_ih", "bias_hh")):
            p.copy_(torch.from_numpy(P[k].astype(np.float64)))
    th, tcs = torch.from_numpy(h0.astype(np.float64)), torch.from_numpy(c0.astype(np.float64))
    for x in xs_h:
        if kind == "lstm":
            th, tcs = tc_(torch.from_numpy(x.astype(np.float64)), (th, tcs))
        else:
            th = tc_(torch.from_numpy(x.astype(np.float64)), th)
    bound = (0.05 if dt == "bf16" else 1e-4) * T
    assert np.max(np.abs(hT64 - th.detach().numpy())) <= bound


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_second_backward_doubles_leaf_gradients(nk, dev, kind):
    """backward() twice from the cell's own output re-seeds that output and adds every leaf gradient again; the gates
    the forward stored are read by both passes"""
    n, n_in, hidden = 5, 16, 8
    rng = np.random.default_rng(2)
    cell = make_cell(nk, dev, kind, n_in, hidden, "f32", 4)
    x = leaf(nk, dev, rng.standard_normal((n, n_in)).astype(F32), "f32", True)
    h0 = leaf(nk, dev, rng.standard_normal((n, hidden)).astype(F32), "f32", True)
    c0 = leaf(nk, dev, rng.standard_normal((n, hidden)).astype(F32), "f32", True)
    out = cell.forward((c0, h0), x)[1] if kind == "lstm" else cell.forward(h0, x)
    out.forward()
    out.backward(1.0)
    leaves = cell.parameters() + [x, h0] + ([c0] if kind == "lstm" else [])
    first = [v.grad().copy() for v in leaves]
    out.backward(1.0)
    for v, g in zip(leaves, first):
        got = v.grad()
        assert np.all(np.abs(got - 2 * g) <= 1e-6 * np.abs(g) + 1e-7), v.shape


def test_shape_and_type_errors(nk, dev):
    cell = make_cell(nk, dev, "lstm", 8, 4, "f32", 1)
    x = nk.from_ndarray(dev, np.zeros((3, 8), F32))
    h = nk.from_ndarray(dev, np.zeros((3, 4), F32))
    with pytest.raises(nk.NkError, match=r"lstm_cell: input must be \(batch, input_size\)"):
        cell.forward((h, h), nk.from_ndarray(dev, np.zeros((3, 8, 1), F32)))
    with pytest.raises(nk.NkError, match=r"lstm_cell: cell_state must be \(3, 4\), got \(3, 5\)"):
        cell.forward((nk.from_ndarray(dev, np.zeros((3, 5), F32)), h), x)
    with pytest.raises(nk.NkError, match=r"lstm_cell: hidden must be \(batch = 3, hidden_size\)"):
        cell.forward((h, nk.from_ndarray(dev, np.zeros((2, 4), F32))), x)
    with pytest.raises(nk.NkError, match=r"lstm_cell: weight_ih must be \(16, 9\), got \(16, 8\)"):
        cell.forward((h, h), nk.from_ndarray(dev, np.zeros((3, 9), F32)))
    with pytest.raises(nk.NkError, match="lstm_cell: cell_state has another element type than the input"):
        cell.forward((nk.from_ndarray(dev, np.zeros((3, 4), F32), nk.BF16), h), x)
    g = make_cell(nk, dev, "gru", 8, 4, "f32", 1)
    with pytest.raises(nk.NkError, match=r"gru_cell: bias_hh must be \(12,\), got \(16,\)"):
        nk.variable.gru_cell(x, h, g.weight_ih, g.weight_hh, g.bias_ih, cell.bias_hh)
    with pytest.raises(nk.NkError, match="gru_cell: input has another element type|gru_cell: hidden has another"):
        g.forward(h, nk.from_ndarray(dev, np.zeros((3, 8), F32), nk.BF16))
    with pytest.raises(nk.NkError, match=r"chunks: chunk dimension 1 \(5\) must be in \[1, 4\]"):
        h.chunks((1, 5))


# ------------------------------------------------------------------------------------------------ fused vs composed
def composed_lstm(nk, cell, state, x, n, hidden):
    """the cell written as the reference writes it, with the intended gate assignment"""
    c, h = state
    gates = x.mm_t(cell.weight_ih) + cell.bias_ih + h.mm_t(cell.weight_hh) + cell.bias_hh
    i, f, g, o = gates.chunks((n, hidden))
    c2 = f.sigmoid() * c + i.sigmoid() * g.tanh()
    return c2, o.sigmoid() * c2.tanh()


def composed_gru(nk, cell, h, x, n, hidden):
    ig = x.mm_t(cell.weight_ih) + cell.bias_ih
    hg = h.mm_t(cell.weight_hh) + cell.bias_hh
    ir, iz, i_n = ig.chunks((n, hidden))
    hr, hz, hn = hg.chunks((n, hidden))
    r, z = (hr + ir).sigmoid(), (hz + iz).sigmoid()
    nn = (i_n + hn * r).tanh()
    return (h - nn) * z + nn


@pytest.mark.parametrize("kind", ["lstm", "gru"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_fused_matches_composed_with_fewer_launches(nk, dev, kind, dt):
    from neuronika_b200 import ops
    n, n_in, hidden = 64, 128, 64
    rng = np.random.default_rng(8)
    x_h = held(rng.standard_normal((n, n_in)), dt)
    h_h = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    c_h = held(rng.standard_normal((n, hidden)) * 0.5, dt)
    res = {}
    for mode in ("fused", "composed"):
        cell = make_cell(nk, dev, kind, n_in, hidden, dt, 6)
        # leaf gradients of the data's element type: no mixed-type accumulation pass in the launch count
        x, h, c = (nk.from_ndarray(dev, a, D(nk, dt)).requires_grad() for a in (x_h, h_h, c_h))
        if mode == "fused":
            out = cell.forward((c, h), x)[1] if kind == "lstm" else cell.forward(h, x)
        else:
            out = composed_lstm(nk, cell, (c, h), x, n, hidden)[1] if kind == "lstm" else composed_gru(nk, cell, h, x, n, hidden)
        dev.synchronize()
        l0 = dev.launches
        out.forward()
        l1 = dev.launches
        out.backward(1.0)
        l2 = dev.launches
        res[mode] = (out.data(), [p.grad() for p in cell.parameters()] + [x.grad(), h.grad()] +
                     ([c.grad()] if kind == "lstm" else []), l1 - l0, l2 - l1)
    (yf, gf, ff, bf), (yc, gc, fc, bc) = res["fused"], res["composed"]
    # the composed graph rounds its gate pre-activations and every intermediate to the element type; the fused cell
    # keeps them in f32: the two agree to those roundings (the bf16 bound is ~4 roundings of O(1) values)
    kb = 0.04 if dt == "bf16" else 1e-5
    assert np.max(np.abs(yf - yc)) <= kb * (1 + np.max(np.abs(yc))), "h'"
    for a, b in zip(gf, gc):
        assert np.max(np.abs(a - b)) <= kb * (1 + np.max(np.abs(b))) * 4, a.shape
    # launches: forward = two GEMMs + the gate kernel; backward = the deferred fill of the root gradient, the gate
    # kernel, four GEMMs (dW_ih, dW_hh, dx, dh) and the two bias column sums
    G = (4 if kind == "lstm" else 3) * hidden
    g = dev.zeros((n, G), D(nk, dt))
    db = dev.zeros((G,), nk.F32 if dt == "bf16" else D(nk, dt))
    dev.synchronize()
    u0 = dev.launches
    ops.unbroadcast_acc(db, g, beta=0.0)
    ub = dev.launches - u0
    assert ff == 3, ff
    assert bf == 1 + 1 + 4 + 2 * ub, (bf, ub)
    assert ff < fc and bf < bc, (ff, fc, bf, bc)


# ------------------------------------------------------------------------------------------------ capture, hooks
@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_captured_sequence_step_matches_eager(nk, dev, kind):
    """zero_grad -> T = 8 cell steps + Linear head + mse -> backward -> SGD, captured once and replayed from the same
    parameters as an eager step: same outputs and weight gradients bit for bit, bias gradients (f32 atomics) to rounding"""
    from neuronika_b200 import optim
    n, n_in, hidden, T = 32, 64, 64, 8
    rng = np.random.default_rng(21)
    cell = make_cell(nk, dev, kind, n_in, hidden, "bf16", 7)
    head = nk.nn.Linear(dev, hidden, 16, nk.BF16, grad_dtype=nk.F32, rng=np.random.default_rng(8))
    params = cell.parameters() + head.parameters()
    init = [p.data().copy() for p in params]
    opt = optim.StochasticGD.new(0.01)
    for p in params:
        opt.register(p)
    xs = [nk.from_ndarray(dev, rng.standard_normal((n, n_in)).astype(F32), nk.BF16) for _ in range(T)]
    tgt = nk.from_ndarray(dev, rng.standard_normal((n, 16)).astype(F32), nk.BF16)
    zeros = nk.from_ndarray(dev, np.zeros((n, hidden), F32), nk.BF16)
    live = {}

    def step():
        opt.zero_grad()
        state = (zeros, zeros) if kind == "lstm" else zeros
        for x in xs:
            state = cell.forward(state, x)
        h = state[1] if kind == "lstm" else state
        y = head.forward(h)
        loss = y.mse_loss(tgt)
        loss.forward()
        loss.backward(1.0)
        live["h"], live["y"] = h, y
        live["grads"] = [p.grad_array() for p in params]
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    step()                     # warm-up: first-use allocations cannot be captured
    reset()
    step()
    dev.synchronize()
    eager = [live["h"].data(), live["y"].data()] + [g.as_ndarray().copy() for g in live["grads"]]
    eager_w = [p.data().copy() for p in params]
    reset()
    with dev.capture(256 << 20) as cap:
        step()
    reset()
    cap.graph.launch()
    dev.synchronize()
    replay = [live["h"].data(), live["y"].data()] + [g.as_ndarray() for g in live["grads"]]
    names = ["h", "y", "weight_ih", "weight_hh", "bias_ih", "bias_hh", "head.weight", "head.bias"]
    for name, a, b in zip(names, eager, replay):
        if "bias" in name:
            assert np.all(np.abs(a - b) <= 1e-6 * np.abs(a) + 1e-7), name
        else:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name
    for p, w in zip(params, eager_w):
        assert np.all(np.abs(p.data() - w) <= UB * np.abs(w) + 1e-7)
    cap.graph.close()


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_grad_hooks_fire_once_per_backward(nk, dev, kind):
    n, n_in, hidden, T = 4, 8, 8, 3
    cell = make_cell(nk, dev, kind, n_in, hidden, "bf16", 9)
    seen = {"ih": [], "hh": []}
    cell.weight_ih.set_grad_hook(lambda b, e: seen["ih"].append((b, e)))
    cell.weight_hh.set_grad_hook(lambda b, e: seen["hh"].append((b, e)))
    rng = np.random.default_rng(3)
    state = (nk.zeros(dev, (n, hidden), nk.BF16),) * 2 if kind == "lstm" else nk.zeros(dev, (n, hidden), nk.BF16)
    for _ in range(T):
        state = cell.forward(state, nk.from_ndarray(dev, rng.standard_normal((n, n_in)).astype(F32), nk.BF16))
    loss = (state[1] if kind == "lstm" else state).sum()
    loss.forward()
    for k in (1, 2):
        loss.backward(1.0)
        assert seen["ih"] == [(0, 4 * hidden * n_in if kind == "lstm" else 3 * hidden * n_in)] * k
        assert seen["hh"] == [(0, (4 if kind == "lstm" else 3) * hidden * hidden)] * k


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_reduce_scatter_plan_reported_once_per_backward(nk, dev, kind):
    """data-parallel contract of the cell weights: a weight with a reduce-scatter plan (set_grad_rs) is computed locally by
    the cell's backward and reported as not pushed, cb(0), exactly ONCE per backward() -- by the last of the T nodes that
    accumulate into it -- and the gradient is the one computed without a plan, bit for bit.  The plan is world = 2 on one
    GPU; its slot buffers are never written."""
    n, n_in, hidden, T = 8, 256, 256, 4
    rng = np.random.default_rng(17)
    xs_h = [rng.standard_normal((n, n_in)).astype(F32) for _ in range(T)]
    grads, calls, slots = [], {"weight_ih": [], "weight_hh": []}, []
    for planned in (False, True):
        cell = make_cell(nk, dev, kind, n_in, hidden, "bf16", 13)
        if planned:
            for name in calls:
                w = getattr(cell, name)
                numel = int(np.prod(w.shape))
                bufs = [dev.zeros((numel,), nk.F32) for _ in range(2)]
                slots.append(bufs)
                w.set_grad_rs(2, 0, [b.ptr.value for b in bufs], lambda pushed, name=name: calls[name].append(pushed))
        zero = nk.zeros(dev, (n, hidden), nk.BF16)
        state = (zero, zero) if kind == "lstm" else zero
        for x in xs_h:
            state = cell.forward(state, nk.from_ndarray(dev, x, nk.BF16))
        loss = (state[1] if kind == "lstm" else state).sum()
        loss.forward()
        for k in (1, 2):
            loss.backward(1.0)
            if planned:
                assert calls["weight_ih"] == [0] * k and calls["weight_hh"] == [0] * k, calls
        grads.append([cell.weight_ih.grad(), cell.weight_hh.grad()])
        if planned:
            for name in calls:
                getattr(cell, name).set_grad_rs(0, 0, None, None)
    for a, b in zip(*grads):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for bufs in slots:
        for b in bufs:
            assert not b.as_ndarray().any()
