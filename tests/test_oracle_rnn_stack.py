"""The numpy oracle of stacked and bidirectional LSTM / GRU layers (tests/rnn_stack_oracle.py), pinned on the CPU against
torch.nn.LSTM / torch.nn.GRU(num_layers in 1..3, bidirectional) autograd in float64: the output, h_n, c_n and every
gradient (input, initial states, every layer's weights and biases), with gradients flowing in through all three."""
import numpy as np
import pytest
import torch

import rnn_stack_oracle as K

NAMES = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


def make(rng, t, n, i, h, layers, dirs, gates):
    k = 1.0 / np.sqrt(h)
    u = lambda *s: rng.uniform(-k, k, s)
    params = []
    for layer in range(layers):
        isz = i if layer == 0 else dirs * h
        params.append((u(dirs, gates * h, isz), u(dirs, gates * h, h), u(dirs, gates * h), u(dirs, gates * h)))
    xs = rng.standard_normal((t, n, i))
    h0, c0 = rng.standard_normal((2, layers * dirs, n, h))
    return xs, h0, c0, params


def torch_module(cls, i, h, layers, dirs, params):
    m = cls(i, h, num_layers=layers, bidirectional=dirs == 2).double()
    with torch.no_grad():
        for k, w in enumerate(params):
            for d in range(dirs):
                for name, v in zip(NAMES, w):
                    getattr(m, f"{name}_l{k}" + ("_reverse" if d else "")).copy_(torch.from_numpy(v[d]))
    return m


def torch_grad(m, name, k, dirs):
    return np.stack([getattr(m, f"{name}_l{k}" + ("_reverse" if d else "")).grad.numpy() for d in range(dirs)])


def close(got, want, what):
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12, err_msg=what)


@pytest.mark.parametrize("lstm", [True, False])
@pytest.mark.parametrize("layers", [1, 2, 3])
@pytest.mark.parametrize("dirs", [1, 2])
@pytest.mark.parametrize("t,n,i,h", [(1, 2, 3, 4), (5, 3, 4, 5)])
def test_stack_oracle_matches_torch(lstm, layers, dirs, t, n, i, h):
    rng = np.random.default_rng([layers, dirs, t, int(lstm)])
    xs, h0, c0, params = make(rng, t, n, i, h, layers, dirs, 4 if lstm else 3)
    m = torch_module(torch.nn.LSTM if lstm else torch.nn.GRU, i, h, layers, dirs, params)
    tx, th, tc = (torch.tensor(v, requires_grad=True) for v in (xs, h0, c0))
    if lstm:
        y, (hn, cn) = m(tx, (th, tc))
    else:
        y, hn = m(tx, th)
    d_y, d_hn, d_cn = rng.standard_normal(y.shape), rng.standard_normal(hn.shape), rng.standard_normal(hn.shape)
    loss = (y * torch.from_numpy(d_y)).sum() + (hn * torch.from_numpy(d_hn)).sum()
    if lstm:
        loss = loss + (cn * torch.from_numpy(d_cn)).sum()
    loss.backward()
    out, o_hn, o_cn, _ = K.stack_forward(lstm, xs, c0 if lstm else None, h0, params)
    close(out, y.detach().numpy(), "output")
    close(o_hn, hn.detach().numpy(), "h_n")
    if lstm:
        close(o_cn, cn.detach().numpy(), "c_n")
    g, mag = K.stack_backward(lstm, xs, c0 if lstm else None, h0, params, d_y, d_hn, d_cn if lstm else None)
    want = {"x": tx.grad.numpy(), "h": th.grad.numpy()}
    if lstm:
        want["c"] = tc.grad.numpy()
    for k in range(layers):
        for key, name in zip(("w_ih", "w_hh", "b_ih", "b_hh"), NAMES):
            want[f"{key}{k}"] = torch_grad(m, name, k, dirs)
    assert set(want) == set(g)
    for key, w in want.items():
        close(g[key], w, key)
    # the magnitudes bound the gradients of the last layer's products (lower layers' mags cover their own products)
    top = layers - 1
    for key in (f"w_ih{top}", f"w_hh{top}", f"b_ih{top}", f"b_hh{top}"):
        assert np.all(np.abs(g[key]) <= mag[key] * (1 + 1e-12) + 1e-300), key


def test_reverse_direction_is_the_forward_oracle_on_reversed_time():
    """the reverse half of a bidirectional layer is a one-direction layer run on the time-reversed input"""
    rng = np.random.default_rng(7)
    xs, h0, c0, params = make(rng, 4, 2, 3, 5, 1, 2, 4)
    y, hn, cn, _ = K.stack_forward(True, xs, c0, h0, params)
    rev = tuple(p[1:] for p in params[0])
    y1, hn1, cn1, _ = K.stack_forward(True, xs[::-1], c0[1:], h0[1:], [rev])
    close(y[..., 5:], y1[::-1], "reverse half")
    close(hn[1], hn1[0], "reverse h_n")
    close(cn[1], cn1[0], "reverse c_n")
