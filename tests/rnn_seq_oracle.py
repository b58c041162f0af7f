"""numpy oracle of the LSTM / GRU sequence layers (test infrastructure, like tests/rnn_oracle.py): one layer, one
direction, time-major, as a loop over the step functions of rnn_oracle, in float64.  Also the maths of the two backward
step kernels (nk_lstm_seq_bwd_step / nk_gru_seq_bwd_step).  tests/test_oracle_rnn_seq.py pins it against torch.nn.LSTM /
torch.nn.GRU CPU autograd in float64.

Every backward returns, beside the gradients, a dict `mag` of the same keys: the same sums taken over absolute values
(sum_k |a_k b_k| of every product), the scale a rounding error of the device is proportional to.
"""
from __future__ import annotations

import numpy as np

import rnn_oracle as R

_f = R._f


# --------------------------------------------------------------------------- the step kernels
def lstm_seq_bwd_step(gates, c_prev, dc, dh_out, dh_rec):
    """(dgates, new dc) of one time step: dh = dh_out + dh_rec (None = zero), dc the running cell-state gradient"""
    return R.lstm_pointwise_backward(gates, c_prev, _sum(dh_out, dh_rec, np.shape(c_prev)), dc)


def gru_seq_bwd_step(ig, hg, h_prev, dh_out, dh_rec):
    """(digates, dhgates, z*dh) of one time step: dh = dh_out + dh_rec (None = zero)"""
    return R.gru_pointwise_backward(ig, hg, h_prev, _sum(dh_out, dh_rec, np.shape(h_prev)))


def _sum(a, b, shape):
    return (np.zeros(shape) if a is None else _f(a)) + (np.zeros(shape) if b is None else _f(b))


# --------------------------------------------------------------------------- LSTM
def lstm_seq_forward(xs, c0, h0, w_ih, w_hh, b_ih, b_hh):
    """(output (T, N, H), cell states (T, N, H)); the last cell state is cs[-1]"""
    c, h = _f(c0), _f(h0)
    out, cs = [], []
    for x in xs:
        c, h = R.lstm_forward(x, c, h, w_ih, w_hh, b_ih, b_hh)
        out.append(h)
        cs.append(c)
    return np.stack(out), np.stack(cs)


def lstm_seq_backward(xs, c0, h0, w_ih, w_hh, b_ih, b_hh, d_out, d_c_last):
    """(gradients, mag): dicts x (T, N, I), c, h, w_ih, w_hh, b_ih, b_hh for output gradients d_out (T, N, H) and
    d_c_last (N, H); None = zero"""
    T = len(xs)
    out, cs = lstm_seq_forward(xs, c0, h0, w_ih, w_hh, b_ih, b_hh)
    hp = [_f(h0)] + list(out[:-1])
    cp = [_f(c0)] + list(cs[:-1])
    W_ih, W_hh = _f(w_ih), _f(w_hh)
    dc = np.zeros_like(cp[0]) if d_c_last is None else _f(d_c_last)
    dh_rec, m_rec, m_dc = None, np.zeros_like(cp[0]), np.abs(dc)
    g = {k: 0.0 for k in ("w_ih", "w_hh", "b_ih", "b_hh")}
    m = dict(g)
    dx, mx = [None] * T, [None] * T
    for t in range(T - 1, -1, -1):
        gates = R.lstm_gates(xs[t], hp[t], w_ih, w_hh, b_ih, b_hh)
        dy = None if d_out is None else d_out[t]
        dg, dc = lstm_seq_bwd_step(gates, cp[t], dc, dy, dh_rec)
        # the magnitude of dg: the same step with every source replaced by its magnitude bounds it only loosely; the
        # gradient's own absolute value is the scale of its rounding
        ag = np.abs(dg)
        g["w_ih"] = g["w_ih"] + dg.T @ _f(xs[t])
        g["w_hh"] = g["w_hh"] + dg.T @ hp[t]
        g["b_ih"] = g["b_ih"] + dg.sum(0)
        g["b_hh"] = g["b_hh"] + dg.sum(0)
        m["w_ih"] = m["w_ih"] + ag.T @ np.abs(_f(xs[t]))
        m["w_hh"] = m["w_hh"] + ag.T @ np.abs(hp[t])
        m["b_ih"] = m["b_ih"] + ag.sum(0)
        m["b_hh"] = m["b_hh"] + ag.sum(0)
        dx[t], mx[t] = dg @ W_ih, ag @ np.abs(W_ih)
        dh_rec, m_rec, m_dc = dg @ W_hh, ag @ np.abs(W_hh), np.abs(dc)
    g.update(x=np.stack(dx), h=dh_rec, c=dc)
    m.update(x=np.stack(mx), h=m_rec, c=m_dc)
    return g, m


# --------------------------------------------------------------------------- GRU
def gru_seq_forward(xs, h0, w_ih, w_hh, b_ih, b_hh):
    h = _f(h0)
    out = []
    for x in xs:
        h = R.gru_forward(x, h, w_ih, w_hh, b_ih, b_hh)
        out.append(h)
    return np.stack(out)


def gru_seq_backward(xs, h0, w_ih, w_hh, b_ih, b_hh, d_out):
    """(gradients, mag): dicts x (T, N, I), h, w_ih, w_hh, b_ih, b_hh for the output gradient d_out (T, N, H)"""
    T = len(xs)
    out = gru_seq_forward(xs, h0, w_ih, w_hh, b_ih, b_hh)
    hp = [_f(h0)] + list(out[:-1])
    W_ih, W_hh = _f(w_ih), _f(w_hh)
    dh_rec, m_rec = None, np.zeros_like(hp[0])
    g = {k: 0.0 for k in ("w_ih", "w_hh", "b_ih", "b_hh")}
    m = dict(g)
    dx, mx = [None] * T, [None] * T
    for t in range(T - 1, -1, -1):
        ig, hg = R.gru_gates(xs[t], hp[t], w_ih, w_hh, b_ih, b_hh)
        dy = None if d_out is None else d_out[t]
        di, dhg, zdh = gru_seq_bwd_step(ig, hg, hp[t], dy, dh_rec)
        ai, ah = np.abs(di), np.abs(dhg)
        g["w_ih"] = g["w_ih"] + di.T @ _f(xs[t])
        g["w_hh"] = g["w_hh"] + dhg.T @ hp[t]
        g["b_ih"] = g["b_ih"] + di.sum(0)
        g["b_hh"] = g["b_hh"] + dhg.sum(0)
        m["w_ih"] = m["w_ih"] + ai.T @ np.abs(_f(xs[t]))
        m["w_hh"] = m["w_hh"] + ah.T @ np.abs(hp[t])
        m["b_ih"] = m["b_ih"] + ai.sum(0)
        m["b_hh"] = m["b_hh"] + ah.sum(0)
        dx[t], mx[t] = di @ W_ih, ai @ np.abs(W_ih)
        dh_rec, m_rec = zdh + dhg @ W_hh, np.abs(zdh) + ah @ np.abs(W_hh)
    g.update(x=np.stack(dx), h=dh_rec)
    m.update(x=np.stack(mx), h=m_rec)
    return g, m
