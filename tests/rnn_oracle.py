"""numpy oracle of the recurrent cells and of `chunks` (test infrastructure, like oracle/): neuronika-nn's LSTMCell and
GRUCell (neuronika-nn/src/lib.rs:450-626) with the intended LSTM gate assignment (SURVEY.md 8-c defect 7: i, f, o =
sigmoid, g = tanh, the layout of torch.nn.LSTMCell) and the Chunk node (neuronika-variable/src/node/chunk/mod.rs).

Inputs are f32 (as the device holds them); the maths runs in float64 (the f32 -> f64 shadow of oracle/), so the oracle
is the exact value the kernels approximate.  tests/test_oracle_rnn.py pins it against torch CPU autograd in float64 and
against the reference's own chunk test vectors (tests/golden/tensors_rnn.json).
"""
from __future__ import annotations

import numpy as np

F64 = np.float64


def _f(a):
    return np.asarray(a, F64)


def sigmoid(x):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-_f(x)))


# --------------------------------------------------------------------------- LSTM
def lstm_gates(x, h, w_ih, w_hh, b_ih, b_hh):
    """gates = x.W_ih^T + b_ih + h.W_hh^T + b_hh, (N, 4H), chunks [i | f | g | o]"""
    return _f(x) @ _f(w_ih).T + _f(b_ih) + _f(h) @ _f(w_hh).T + _f(b_hh)


def lstm_pointwise(gates, c):
    """(c', h') from the pre-activations"""
    gi, gf, gg, go = np.split(_f(gates), 4, axis=1)
    i, f, g, o = sigmoid(gi), sigmoid(gf), np.tanh(gg), sigmoid(go)
    c2 = f * _f(c) + i * g
    return c2, o * np.tanh(c2)


def lstm_pointwise_backward(gates, c, dh, dc):
    """(dgates, dc_prev) for output gradients dh, dc (None = zero)"""
    gi, gf, gg, go = np.split(_f(gates), 4, axis=1)
    i, f, g, o = sigmoid(gi), sigmoid(gf), np.tanh(gg), sigmoid(go)
    c = _f(c)
    tc = np.tanh(f * c + i * g)
    dh = np.zeros_like(c) if dh is None else _f(dh)
    dct = (np.zeros_like(c) if dc is None else _f(dc)) + dh * o * (1 - tc * tc)
    dgates = np.concatenate([dct * g * i * (1 - i), dct * c * f * (1 - f), dct * i * (1 - g * g),
                             dh * tc * o * (1 - o)], axis=1)
    return dgates, f * dct


def lstm_forward(x, c, h, w_ih, w_hh, b_ih, b_hh):
    """one step: (c', h')"""
    return lstm_pointwise(lstm_gates(x, h, w_ih, w_hh, b_ih, b_hh), c)


def lstm_backward(x, c, h, w_ih, w_hh, b_ih, b_hh, dh, dc):
    """every gradient of one step: dict x, c, h, w_ih, w_hh, b_ih, b_hh"""
    gates = lstm_gates(x, h, w_ih, w_hh, b_ih, b_hh)
    dg, dcp = lstm_pointwise_backward(gates, c, dh, dc)
    return {"x": dg @ _f(w_ih), "h": dg @ _f(w_hh), "c": dcp, "w_ih": dg.T @ _f(x), "w_hh": dg.T @ _f(h),
            "b_ih": dg.sum(0), "b_hh": dg.sum(0)}


# --------------------------------------------------------------------------- GRU
def gru_gates(x, h, w_ih, w_hh, b_ih, b_hh):
    """(igates, hgates), (N, 3H) each, chunks [r | z | n]"""
    return _f(x) @ _f(w_ih).T + _f(b_ih), _f(h) @ _f(w_hh).T + _f(b_hh)


def gru_pointwise(ig, hg, h):
    ir, iz, i_n = np.split(_f(ig), 3, axis=1)
    hr, hz, hn = np.split(_f(hg), 3, axis=1)
    r, z = sigmoid(ir + hr), sigmoid(iz + hz)
    nn = np.tanh(i_n + r * hn)
    return (_f(h) - nn) * z + nn


def gru_pointwise_backward(ig, hg, h, dh):
    """(digates, dhgates, pointwise part of dh_prev)"""
    ir, iz, i_n = np.split(_f(ig), 3, axis=1)
    hr, hz, hn = np.split(_f(hg), 3, axis=1)
    r, z = sigmoid(ir + hr), sigmoid(iz + hz)
    nn = np.tanh(i_n + r * hn)
    dh = _f(dh)
    dpn = dh * (1 - z) * (1 - nn * nn)
    dpz = dh * (_f(h) - nn) * z * (1 - z)
    dpr = dpn * hn * r * (1 - r)
    return (np.concatenate([dpr, dpz, dpn], axis=1), np.concatenate([dpr, dpz, dpn * r], axis=1), z * dh)


def gru_forward(x, h, w_ih, w_hh, b_ih, b_hh):
    ig, hg = gru_gates(x, h, w_ih, w_hh, b_ih, b_hh)
    return gru_pointwise(ig, hg, h)


def gru_backward(x, h, w_ih, w_hh, b_ih, b_hh, dh):
    ig, hg = gru_gates(x, h, w_ih, w_hh, b_ih, b_hh)
    di, dhg, dhp = gru_pointwise_backward(ig, hg, h, dh)
    return {"x": di @ _f(w_ih), "h": dhp + dhg @ _f(w_hh), "w_ih": di.T @ _f(x), "w_hh": dhg.T @ _f(h),
            "b_ih": di.sum(0), "b_hh": dhg.sum(0)}


# --------------------------------------------------------------------------- chunks
def _blocks(shape, chunk_shape):
    return [s // c for s, c in zip(shape, chunk_shape)]


def chunk_slices(shape, chunk_shape, index):
    """the slices of block `index` of exact_chunks(chunk_shape), row-major block order"""
    nb = _blocks(shape, chunk_shape)
    coords = np.unravel_index(index, nb)
    return tuple(slice(int(k) * c, (int(k) + 1) * c) for k, c in zip(coords, chunk_shape))


def chunks(x, chunk_shape):
    """every block (copies), as Var::chunks (var.rs:401-417)"""
    x = np.asarray(x)
    n = int(np.prod(_blocks(x.shape, chunk_shape)))
    return [x[chunk_slices(x.shape, chunk_shape, i)].copy() for i in range(n)]


def chunk_backward(dx, g, index):
    """dx[block] += g (ChunkBackward::backward, chunk/mod.rs)"""
    dx[chunk_slices(dx.shape, np.shape(g), index)] += g
    return dx
