"""The numpy oracle of the LSTM / GRU sequence layers (tests/rnn_seq_oracle.py), pinned on the CPU against
torch.nn.LSTM / torch.nn.GRU (one layer, time-major) autograd in float64: every step's output, the last cell state and
every gradient (input, initial states, both weights, both biases), with gradients flowing in through `output`, through
the last cell state, and through both."""
import numpy as np
import pytest
import torch

import rnn_oracle as R
import rnn_seq_oracle as S

SHAPES = [(1, 1, 1), (3, 5, 7), (2, 16, 33)]   # (N, I, H)
TS = [1, 2, 7]


def params(rng, t, n, i, h, gates):
    k = 1.0 / np.sqrt(h)
    u = lambda *s: rng.uniform(-k, k, s).astype(np.float32)
    return (rng.standard_normal((t, n, i)).astype(np.float32), u(gates * h, i), u(gates * h, h), u(gates * h),
            u(gates * h))


def close(got, want, what):
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12, err_msg=what)


def torch_layer(cls, i, h, w):
    layer = cls(i, h).double()
    with torch.no_grad():
        for p, v in zip((layer.weight_ih_l0, layer.weight_hh_l0, layer.bias_ih_l0, layer.bias_hh_l0), w):
            p.copy_(torch.from_numpy(v.astype(np.float64)))
    return layer


@pytest.mark.parametrize("n,i,h", SHAPES)
@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("through", ["output", "cell", "both"])
def test_lstm_seq_oracle_matches_torch(n, i, h, t, through):
    rng = np.random.default_rng([n, h, t, len(through)])
    xs, *w = params(rng, t, n, i, h, 4)
    h0 = rng.standard_normal((n, h)).astype(np.float32)
    c0 = rng.standard_normal((n, h)).astype(np.float32)
    d_out = rng.standard_normal((t, n, h)) if through != "cell" else None
    d_c = rng.standard_normal((n, h)) if through != "output" else None
    layer = torch_layer(torch.nn.LSTM, i, h, w)
    tx, th, tc = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (xs, h0, c0))
    y, (hn, cn) = layer(tx, (th[None], tc[None]))
    loss = 0.0
    if d_out is not None:
        loss = loss + (y * torch.from_numpy(d_out)).sum()
    if d_c is not None:
        loss = loss + (cn[0] * torch.from_numpy(d_c)).sum()
    loss.backward()
    out, cs = S.lstm_seq_forward(xs, c0, h0, *w)
    close(out, y.detach().numpy(), "output")
    close(out[-1], hn[0].detach().numpy(), "h_T = output[T-1]")
    close(cs[-1], cn[0].detach().numpy(), "c_T")
    g, mag = S.lstm_seq_backward(xs, c0, h0, *w, d_out, d_c)
    for k, tg in (("x", tx.grad), ("h", th.grad), ("c", tc.grad), ("w_ih", layer.weight_ih_l0.grad),
                  ("w_hh", layer.weight_hh_l0.grad), ("b_ih", layer.bias_ih_l0.grad), ("b_hh", layer.bias_hh_l0.grad)):
        close(g[k], tg.numpy(), k)
        assert np.all(np.abs(g[k]) <= mag[k] * (1 + 1e-12) + 1e-300), k


@pytest.mark.parametrize("n,i,h", SHAPES)
@pytest.mark.parametrize("t", TS)
def test_gru_seq_oracle_matches_torch(n, i, h, t):
    rng = np.random.default_rng([n, h, t, 3])
    xs, *w = params(rng, t, n, i, h, 3)
    h0 = rng.standard_normal((n, h)).astype(np.float32)
    d_out = rng.standard_normal((t, n, h))
    layer = torch_layer(torch.nn.GRU, i, h, w)
    tx, th = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (xs, h0))
    y, hn = layer(tx, th[None])
    (y * torch.from_numpy(d_out)).sum().backward()
    out = S.gru_seq_forward(xs, h0, *w)
    close(out, y.detach().numpy(), "output")
    close(out[-1], hn[0].detach().numpy(), "h_T = output[T-1]")
    g, mag = S.gru_seq_backward(xs, h0, *w, d_out)
    for k, tg in (("x", tx.grad), ("h", th.grad), ("w_ih", layer.weight_ih_l0.grad), ("w_hh", layer.weight_hh_l0.grad),
                  ("b_ih", layer.bias_ih_l0.grad), ("b_hh", layer.bias_hh_l0.grad)):
        close(g[k], tg.numpy(), k)
        assert np.all(np.abs(g[k]) <= mag[k] * (1 + 1e-12) + 1e-300), k


def test_step_functions_add_their_two_sources():
    """dh = dh_out + dh_rec, None = zero: the step of the sum is the step of one source holding the sum"""
    rng = np.random.default_rng(4)
    n, h = 3, 5
    gates, c, dc = rng.standard_normal((n, 4 * h)), rng.standard_normal((n, h)), rng.standard_normal((n, h))
    a, b = rng.standard_normal((2, n, h))
    want = R.lstm_pointwise_backward(gates, c, a + b, dc)
    for got in (S.lstm_seq_bwd_step(gates, c, dc, a, b), S.lstm_seq_bwd_step(gates, c, dc, a + b, None),
                S.lstm_seq_bwd_step(gates, c, dc, None, a + b)):
        close(got[0], want[0], "dgates")
        close(got[1], want[1], "dc")
    z = S.lstm_seq_bwd_step(gates, c, np.zeros((n, h)), None, None)
    assert not z[0].any() and not z[1].any()
    ig, hg = rng.standard_normal((2, n, 3 * h))
    want = R.gru_pointwise_backward(ig, hg, c, a + b)
    for got in (S.gru_seq_bwd_step(ig, hg, c, a, b), S.gru_seq_bwd_step(ig, hg, c, None, a + b)):
        for x, y in zip(got, want):
            close(x, y, "gru step")
