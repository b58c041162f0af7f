"""numpy oracle of stacked and bidirectional LSTM / GRU layers (test infrastructure, like tests/rnn_seq_oracle.py), in
float64.  A direction is the sequence oracle of rnn_seq_oracle: the reverse one runs it on the time-reversed input and
reverses its output back.  Layer k > 0 reads layer k-1's output (no dropout).  tests/test_oracle_rnn_stack.py pins it
against torch.nn.LSTM / torch.nn.GRU(num_layers, bidirectional) CPU autograd in float64.

Parameters are given per layer as (w_ih, w_hh, b_ih, b_hh), each stacked over the D directions: (D, G, I_k), (D, G, H),
(D, G), (D, G).  States are torch-shaped, (L*D, N, H).  Every backward returns, beside the gradients, a dict `mag` of the
same keys: the same sums over absolute values (see rnn_seq_oracle), the scale of a device's rounding error.
"""
from __future__ import annotations

import numpy as np

import rnn_seq_oracle as S

_f = S._f


def _dirs(params):
    return np.shape(params[0][0])[0]


# --------------------------------------------------------------------------- one layer
def layer_forward(lstm, xs, c0, h0, w):
    """(output (T, N, D*H), h_n (D, N, H), c_n (D, N, H) or None) of one layer; c0 is ignored for the GRU"""
    outs, hn, cn = [], [], []
    for d in range(np.shape(h0)[0]):
        xin = _f(xs)[::-1] if d else _f(xs)
        wd = [_f(p)[d] for p in w]
        if lstm:
            out, cs = S.lstm_seq_forward(xin, c0[d], h0[d], *wd)
            cn.append(cs[-1])
        else:
            out = S.gru_seq_forward(xin, h0[d], *wd)
        hn.append(out[-1])
        outs.append(out[::-1] if d else out)
    return np.concatenate(outs, axis=-1), np.stack(hn), (np.stack(cn) if lstm else None)


def layer_backward(lstm, xs, c0, h0, w, d_y, d_hn, d_cn):
    """(gradients, mag) of one layer: dicts x, h, c (LSTM), w_ih, w_hh, b_ih, b_hh (stacked over directions) for the
    output gradients d_y (T, N, D*H), d_hn and d_cn (D, N, H); None = zero"""
    T, H = np.shape(xs)[0], np.shape(h0)[-1]
    gs, ms = [], []
    for d in range(np.shape(h0)[0]):
        xin = _f(xs)[::-1] if d else _f(xs)
        wd = [_f(p)[d] for p in w]
        dy = np.zeros((T,) + np.shape(h0)[1:]) if d_y is None else np.array(_f(d_y)[..., d * H:(d + 1) * H])
        if d:
            dy = dy[::-1].copy()
        if d_hn is not None:   # h_n of the direction is its output at its last step
            dy[-1] += _f(d_hn)[d]
        if lstm:
            g, m = S.lstm_seq_backward(xin, c0[d], h0[d], *wd, dy, None if d_cn is None else _f(d_cn)[d])
        else:
            g, m = S.gru_seq_backward(xin, h0[d], *wd, dy)
        if d:
            g["x"], m["x"] = g["x"][::-1], m["x"][::-1]
        gs.append(g)
        ms.append(m)
    keys = ("w_ih", "w_hh", "b_ih", "b_hh", "h") + (("c",) if lstm else ())
    g = {k: np.stack([x[k] for x in gs]) for k in keys}
    m = {k: np.stack([x[k] for x in ms]) for k in keys}
    g["x"], m["x"] = sum(x["x"] for x in gs), sum(x["x"] for x in ms)
    return g, m


# --------------------------------------------------------------------------- the stack
def stack_forward(lstm, xs, c0, h0, params):
    """(output (T, N, D*H) of the last layer, h_n (L*D, N, H), c_n (L*D, N, H) or None, every layer's output)"""
    D = _dirs(params)
    x, hn, cn, ys = _f(xs), [], [], []
    for k, w in enumerate(params):
        y, h, c = layer_forward(lstm, x, None if c0 is None else _f(c0)[k * D:(k + 1) * D], _f(h0)[k * D:(k + 1) * D], w)
        hn.append(h)
        cn.append(c)
        ys.append(y)
        x = y
    return x, np.concatenate(hn), (np.concatenate(cn) if lstm else None), ys


def stack_backward(lstm, xs, c0, h0, params, d_y, d_hn, d_cn):
    """(gradients, mags): dicts with x (T, N, I), h and c (L*D, N, H), and per layer k w_ih{k}, w_hh{k}, b_ih{k},
    b_hh{k}, for gradients d_y of the last layer's output, d_hn and d_cn (L*D, N, H); None = zero.  The mag of a layer
    covers its own products only."""
    D, L = _dirs(params), len(params)
    _, _, _, ys = stack_forward(lstm, xs, c0, h0, params)
    ins = [_f(xs)] + ys[:-1]
    g, m = {}, {}
    hs, ms_h, cs, ms_c = [None] * L, [None] * L, [None] * L, [None] * L
    dy = d_y
    for k in range(L - 1, -1, -1):
        sl = slice(k * D, (k + 1) * D)
        gk, mk = layer_backward(lstm, ins[k], None if c0 is None else _f(c0)[sl], _f(h0)[sl], params[k], dy,
                                None if d_hn is None else _f(d_hn)[sl], None if d_cn is None else _f(d_cn)[sl])
        for name in ("w_ih", "w_hh", "b_ih", "b_hh"):
            g[f"{name}{k}"], m[f"{name}{k}"] = gk[name], mk[name]
        hs[k], ms_h[k] = gk["h"], mk["h"]
        if lstm:
            cs[k], ms_c[k] = gk["c"], mk["c"]
        dy = gk["x"]
        g["x"], m["x"] = gk["x"], mk["x"]
    g["h"], m["h"] = np.concatenate(hs), np.concatenate(ms_h)
    if lstm:
        g["c"], m["c"] = np.concatenate(cs), np.concatenate(ms_c)
    return g, m
