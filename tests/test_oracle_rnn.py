"""The numpy oracle of the recurrent cells and of `chunks` (tests/rnn_oracle.py), pinned on the CPU:
  - LSTM / GRU values and every gradient (x, h, c, both weights, both biases) against torch.nn.LSTMCell / GRUCell CPU
    autograd in float64, at several shapes and with random output gradients on both LSTM outputs;
  - chunks forward / backward against the reference's own chunk test vectors (tests/golden/tensors_rnn.json)."""
import json
import os

import numpy as np
import pytest
import torch

import rnn_oracle as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tensors_rnn.json")
SHAPES = [(1, 1, 1), (3, 5, 7), (4, 9, 8), (2, 16, 33)]   # (N, I, H)


def params(rng, n, i, h, gates):
    k = 1.0 / np.sqrt(h)
    u = lambda *s: rng.uniform(-k, k, s).astype(np.float32)
    return (rng.standard_normal((n, i)).astype(np.float32), u(gates * h, i), u(gates * h, h), u(gates * h),
            u(gates * h))


def close(got, want, what):
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12, err_msg=what)


@pytest.mark.parametrize("n,i,h", SHAPES)
def test_lstm_oracle_matches_torch(n, i, h):
    rng = np.random.default_rng(n * 100 + h)
    x, w_ih, w_hh, b_ih, b_hh = params(rng, n, i, h, 4)
    h0 = rng.standard_normal((n, h)).astype(np.float32)
    c0 = rng.standard_normal((n, h)).astype(np.float32)
    dh, dc = rng.standard_normal((2, n, h))
    cell = torch.nn.LSTMCell(i, h).double()
    with torch.no_grad():
        for p, v in zip((cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh), (w_ih, w_hh, b_ih, b_hh)):
            p.copy_(torch.from_numpy(v.astype(np.float64)))
    tx, th, tc = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (x, h0, c0))
    h1, c1 = cell(tx, (th, tc))
    (h1 * torch.from_numpy(dh)).sum().add((c1 * torch.from_numpy(dc)).sum()).backward()
    c_o, h_o = R.lstm_forward(x, c0, h0, w_ih, w_hh, b_ih, b_hh)
    close(h_o, h1.detach().numpy(), "h'")
    close(c_o, c1.detach().numpy(), "c'")
    g = R.lstm_backward(x, c0, h0, w_ih, w_hh, b_ih, b_hh, dh, dc)
    for k, t in (("x", tx.grad), ("h", th.grad), ("c", tc.grad), ("w_ih", cell.weight_ih.grad),
                 ("w_hh", cell.weight_hh.grad), ("b_ih", cell.bias_ih.grad), ("b_hh", cell.bias_hh.grad)):
        close(g[k], t.numpy(), k)


def test_lstm_oracle_zero_output_gradients():
    """an output nobody used (None) is a zero gradient"""
    rng = np.random.default_rng(1)
    gates = rng.standard_normal((3, 20))
    c = rng.standard_normal((3, 5))
    dh = rng.standard_normal((3, 5))
    a = R.lstm_pointwise_backward(gates, c, dh, None)
    b = R.lstm_pointwise_backward(gates, c, dh, np.zeros((3, 5)))
    close(a[0], b[0], "dgates")
    close(a[1], b[1], "dc")
    z = R.lstm_pointwise_backward(gates, c, None, None)
    assert not z[0].any() and not z[1].any()


@pytest.mark.parametrize("n,i,h", SHAPES)
def test_gru_oracle_matches_torch(n, i, h):
    rng = np.random.default_rng(n * 100 + h + 7)
    x, w_ih, w_hh, b_ih, b_hh = params(rng, n, i, h, 3)
    h0 = rng.standard_normal((n, h)).astype(np.float32)
    dh = rng.standard_normal((n, h))
    cell = torch.nn.GRUCell(i, h).double()
    with torch.no_grad():
        for p, v in zip((cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh), (w_ih, w_hh, b_ih, b_hh)):
            p.copy_(torch.from_numpy(v.astype(np.float64)))
    tx, th = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (x, h0))
    h1 = cell(tx, th)
    (h1 * torch.from_numpy(dh)).sum().backward()
    close(R.gru_forward(x, h0, w_ih, w_hh, b_ih, b_hh), h1.detach().numpy(), "h'")
    g = R.gru_backward(x, h0, w_ih, w_hh, b_ih, b_hh, dh)
    for k, t in (("x", tx.grad), ("h", th.grad), ("w_ih", cell.weight_ih.grad), ("w_hh", cell.weight_hh.grad),
                 ("b_ih", cell.bias_ih.grad), ("b_hh", cell.bias_hh.grad)):
        close(g[k], t.numpy(), k)


def test_lstm_saturated_gates_are_finite():
    gates = np.array([[30.0, -30.0, np.inf, -np.inf, 30.0, np.inf, -np.inf, -30.0]])
    c = np.array([[0.5, -2.0]])
    c2, h2 = R.lstm_pointwise(gates, c)
    dg, dc = R.lstm_pointwise_backward(gates, c, np.ones((1, 2)), np.ones((1, 2)))
    assert np.isfinite(c2).all() and np.isfinite(h2).all() and np.isfinite(dg).all() and np.isfinite(dc).all()


@pytest.fixture(scope="module")
def goldens():
    with open(GOLDEN) as fh:
        return json.load(fh)["chunk"]


def test_chunk_forward_goldens(goldens):
    """chunk/test.rs forward base_case: the three (1, 3) blocks of linspace(-4, 4, 9).into_shape((3, 3))"""
    case = goldens["base_case"][0]
    ls = case["linspace"][0]
    x = np.linspace(ls["start"], ls["stop"], ls["num"]).reshape(ls["shape"]).astype(np.float32)
    assert len(case["tensors"]) == len(case["indices"]) == 3
    blocks = R.chunks(x, case["tensors"][0]["shape"])
    for idx, t in zip(case["indices"], case["tensors"]):
        np.testing.assert_array_equal(blocks[idx], np.array(t["values"], np.float32).reshape(t["shape"]))


def test_chunk_backward_goldens(goldens):
    """chunk/test.rs backward base_case: ones (1, 3) into block k of a (3, 3) zero gradient, twice (1 -> 2)"""
    case = goldens["base_case"][1]
    assert case["indices"] == [0, 1, 2] and len(case["tensors"]) == 6
    for j, idx in enumerate(case["indices"]):
        dx = np.zeros((3, 3), np.float32)
        for rep in range(2):
            R.chunk_backward(dx, np.ones((1, 3), np.float32), idx)
            t = case["tensors"][2 * j + rep]
            np.testing.assert_array_equal(dx, np.array(t["values"], np.float32).reshape(t["shape"]))


def test_chunks_drop_partial_blocks():
    """exact_chunks: (5, 7) in (2, 3) blocks -> 2 x 2 blocks, row-major order"""
    x = np.arange(35, dtype=np.float32).reshape(5, 7)
    b = R.chunks(x, (2, 3))
    assert len(b) == 4
    np.testing.assert_array_equal(b[1], x[0:2, 3:6])
    np.testing.assert_array_equal(b[2], x[2:4, 0:3])
