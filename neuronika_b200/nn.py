"""Layers: the mirror of neuronika-nn's Linear, LSTMCell, GRUCell and Conv2d (neuronika-nn/src/lib.rs:406-626, 724-815),
and the sequence layers LSTM and GRU over them."""
from __future__ import annotations

import math

import numpy as np

from . import variable as V
from .device import F32, Device


def uniform(rng: np.random.Generator, shape, low: float, high: float) -> np.ndarray:
    """`init::uniform` (neuronika-nn/src/init.rs:177-183); seeded here, thread_rng in the reference."""
    return rng.uniform(low, high, size=shape).astype(np.float32)


class ZeroPad:
    """`Zero` padding mode (pad/zero/mod.rs:14-22)."""
    value = 0.0


class ConstantPad:
    """`Constant(value)` padding mode (pad/constant/mod.rs:14-39)."""

    def __init__(self, value: float):
        self.value = float(value)


class Linear:
    """y = x.A^T + b;  weight (out, in), bias (out,), both ~ U(-k, k), k = sqrt(1/in)
    (neuronika-nn/src/lib.rs:406-448)."""

    def __init__(self, device: Device, in_features: int, out_features: int, dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None):
        rng = rng or np.random.default_rng()
        k = math.sqrt(1.0 / in_features)
        self.weight = V.from_ndarray(device, uniform(rng, (out_features, in_features), -k, k), dtype).requires_grad(grad_dtype)
        self.bias = V.from_ndarray(device, uniform(rng, (out_features,), -k, k), dtype).requires_grad(grad_dtype)

    def forward(self, input: V.Var) -> V.VarDiff:
        """`input.mm_t(self.weight.clone()).into() + self.bias.clone()` (:441-447)"""
        return input.mm_t(self.weight) + self.bias

    def parameters(self):
        return [self.weight, self.bias]


class Conv2d:
    """2-D convolution layer: weight (Cout, Cin, kh, kw), bias (Cout, 1, 1) ~ U(-k, k),
    k = sqrt(1/(Cin*kh*kw)) (neuronika-nn/src/lib.rs:724-788).  The reference's `forward` is
    `todo!()` (:809-814); the documented intent (:789-808) is implemented:
    pad(input) -> weight.convolution(padded, stride, dilation, 1) + bias."""

    def __init__(self, device: Device, in_channels: int, out_channels: int, kernel_size, padding=(0, 0),
                 padding_mode=None, stride=(1, 1), dilation=(1, 1), dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None):
        rng = rng or np.random.default_rng()
        kh, kw = kernel_size
        k = math.sqrt(1.0 / (in_channels * kh * kw))
        self.padding, self.stride, self.dilation = tuple(padding), tuple(stride), tuple(dilation)
        self.padding_mode = padding_mode or ZeroPad()
        self.weight = V.from_ndarray(device, uniform(rng, (out_channels, in_channels, kh, kw), -k, k), dtype).requires_grad(grad_dtype)
        self.bias = V.from_ndarray(device, uniform(rng, (out_channels, 1, 1), -k, k), dtype).requires_grad(grad_dtype)

    def forward(self, input: V.Var) -> V.VarDiff:
        x = input.pad(self.padding, self.padding_mode.value) if any(self.padding) else input
        return self.weight.convolution(x, self.stride, self.dilation, 1) + self.bias

    def parameters(self):
        return [self.weight, self.bias]


class LSTMCell:
    """One LSTM step (neuronika-nn/src/lib.rs:450-540): weight_ih (4H, I), weight_hh (4H, H), bias_ih, bias_hh (4H,),
    all ~ U(-k, k), k = 1/sqrt(hidden_size) (:471-489).  Gate chunks [i | f | g | o] with i, f, o = sigmoid and
    g = tanh: the reference's names, and torch.nn.LSTMCell's layout (the reference applies tanh to the forget gate and
    sigmoid to the candidate, SURVEY.md 8-c defect 7).  The step is one fused graph node (variable.lstm_cell)."""

    def __init__(self, device: Device, input_size: int, hidden_size: int, dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None):
        rng = rng or np.random.default_rng()
        k = 1.0 / math.sqrt(hidden_size)
        g = 4 * hidden_size
        self.weight_ih = V.from_ndarray(device, uniform(rng, (g, input_size), -k, k), dtype).requires_grad(grad_dtype)
        self.weight_hh = V.from_ndarray(device, uniform(rng, (g, hidden_size), -k, k), dtype).requires_grad(grad_dtype)
        self.bias_ih = V.from_ndarray(device, uniform(rng, (g,), -k, k), dtype).requires_grad(grad_dtype)
        self.bias_hh = V.from_ndarray(device, uniform(rng, (g,), -k, k), dtype).requires_grad(grad_dtype)

    def forward(self, state, input: V.Var):
        """`state = (cell_state, hidden)`, both (batch, hidden_size); returns (new_cell_state, new_hidden) (:510-540)."""
        cell_state, hidden = state
        return V.lstm_cell(input, cell_state, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)

    def parameters(self):
        return [self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh]


class LSTM(LSTMCell):
    """The LSTMCell applied to a whole time-major sequence as one graph node (variable.lstm): same parameters and
    initialisation as the cell, so a layer built from the same `rng` seed holds the same weights.  One layer, one
    direction."""

    def forward(self, state, input: V.Var):
        """`state = (cell_state, hidden)`, both (batch, hidden_size); `input` (seq_len, batch, input_size).  Returns
        (output, cell_T): every step's hidden state (seq_len, batch, hidden_size), whose last slice is the last hidden
        state, and the last cell state."""
        cell_state, hidden = state
        return V.lstm(input, cell_state, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)


class Dropout:
    """Dropout with probability p and a status of its own: `train()` (the initial mode) draws a new mask on every
    forward() of the graph, `eval()` passes the input through.  The reference's docs name `nn::Dropout`; its crate
    defines only the op (var.rs:375-397)."""

    def __init__(self, p: float):
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"Wrong probability received: {p}.")
        self.p = float(p)
        self.status = V.Status(True)

    def forward(self, input: V.Var) -> V.Var:
        return input.dropout(self.p, self.status)

    def train(self) -> None:
        self.status.train()

    def eval(self) -> None:
        self.status.eval()

    def parameters(self):
        return []


class GRUCell:
    """One GRU step (neuronika-nn/src/lib.rs:543-626, = torch.nn.GRUCell): weight_ih (3H, I), weight_hh (3H, H),
    bias_ih, bias_hh (3H,), all ~ U(-k, k), k = 1/sqrt(hidden_size); gate chunks [r | z | n].  One fused graph node."""

    def __init__(self, device: Device, input_size: int, hidden_size: int, dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None):
        rng = rng or np.random.default_rng()
        k = 1.0 / math.sqrt(hidden_size)
        g = 3 * hidden_size
        self.weight_ih = V.from_ndarray(device, uniform(rng, (g, input_size), -k, k), dtype).requires_grad(grad_dtype)
        self.weight_hh = V.from_ndarray(device, uniform(rng, (g, hidden_size), -k, k), dtype).requires_grad(grad_dtype)
        self.bias_ih = V.from_ndarray(device, uniform(rng, (g,), -k, k), dtype).requires_grad(grad_dtype)
        self.bias_hh = V.from_ndarray(device, uniform(rng, (g,), -k, k), dtype).requires_grad(grad_dtype)

    def forward(self, hidden: V.Var, input: V.Var):
        """(:607-624) returns the new hidden state (batch, hidden_size)."""
        return V.gru_cell(input, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)

    def parameters(self):
        return [self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh]


class GRU(GRUCell):
    """The GRUCell applied to a whole time-major sequence as one graph node (variable.gru): same parameters and
    initialisation as the cell.  One layer, one direction."""

    def forward(self, hidden: V.Var, input: V.Var):
        """`hidden` (batch, hidden_size), `input` (seq_len, batch, input_size); returns every step's hidden state
        (seq_len, batch, hidden_size)."""
        return V.gru(input, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)
