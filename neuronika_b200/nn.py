"""Layers: the mirror of neuronika-nn's Linear, LSTMCell, GRUCell, Conv1d, Conv2d and Conv3d (neuronika-nn/src/lib.rs:
406-916), the sequence layers LSTM and GRU over them (stacked and bidirectional like torch.nn.LSTM / GRU), and torch's
max, average and adaptive average pooling layers, its batch and layer normalization layers and its embedding."""
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
    mode, value = "zero", 0.0


class ConstantPad:
    """`Constant(value)` padding mode (pad/constant/mod.rs:14-39)."""
    mode = "constant"

    def __init__(self, value: float):
        self.value = float(value)


class ReflectivePad:
    """`Reflective` padding mode (pad/reflective/mod.rs:14-31): the border mirrored without repeating the edge, like
    numpy's "reflect"; the padding must be smaller than the padded dimension."""
    mode, value = "reflective", 0.0


class ReplicativePad:
    """`Replicative` padding mode (pad/replicative/mod.rs:14-31): the edge element repeated, like numpy's "edge"."""
    mode, value = "replicative", 0.0


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


class Embedding:
    """torch.nn.Embedding: weight (num_embeddings, embedding_dim) ~ N(0, 1) (`init::normal`, neuronika-nn/src/init.rs:195),
    its padding_idx row zeroed; forward(ids) = weight[ids] with ids a non-differentiable Var of float ids (f32, or bf16
    for num_embeddings <= 256).  A negative padding_idx counts from num_embeddings; that row gets no gradient."""

    def __init__(self, device: Device, num_embeddings: int, embedding_dim: int, padding_idx=None, dtype=F32,
                 grad_dtype=None, rng: np.random.Generator | None = None):
        rng = rng or np.random.default_rng()
        if padding_idx is not None:
            if not -num_embeddings <= padding_idx < num_embeddings:
                raise ValueError("Padding_idx must be within num_embeddings")
            padding_idx = padding_idx % num_embeddings
        self.padding_idx = padding_idx
        w = rng.standard_normal((num_embeddings, embedding_dim)).astype(np.float32)
        if padding_idx is not None:
            w[padding_idx] = 0.0
        self.weight = V.from_ndarray(device, w, dtype).requires_grad(grad_dtype)

    def forward(self, ids: V.Var) -> V.VarDiff:
        return V.embedding(ids, self.weight, self.padding_idx)

    def parameters(self):
        return [self.weight]


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
        mode = getattr(self.padding_mode, "mode", "constant")
        if not any(self.padding):
            x = input
        elif mode in ("zero", "constant"):
            x = input.pad(self.padding, self.padding_mode.value)
        else:
            x = input.pad(self.padding, mode=mode)
        return self.weight.convolution(x, self.stride, self.dilation, 1) + self.bias

    def parameters(self):
        return [self.weight, self.bias]


class _ConvNd:
    """The 1-D / 3-D convolution layers (neuronika-nn/src/lib.rs:630-723, 817-916): weight (Cout, Cin, k...), bias
    (Cout, 1) / (Cout, 1, 1, 1), both ~ U(-k, k), k = sqrt(1/(Cin*prod(kernel))).  The reference's `forward` is
    `todo!()`; the documented intent, pad(input) -> weight.convolution(padded, stride, dilation, 1) + bias, runs as ONE
    graph node (variable.conv_layer): bf16 layers on the tensor cores with the padding applied inside the im2col gather,
    so neither the padded input nor its gradient is ever stored.  The input gradient follows the reference's pad
    backward: the interior slice of the padded input's gradient for every mode (torch folds the border gradient of
    reflect / replicate padding back instead)."""

    nsp = 0

    def __init__(self, device: Device, in_channels: int, out_channels: int, kernel_size, padding, padding_mode, stride,
                 dilation, dtype, grad_dtype, rng):
        rng = rng or np.random.default_rng()
        kernel = self._tuple(kernel_size, "kernel_size")
        self.padding = self._tuple(padding, "padding")
        self.stride = self._tuple(stride, "stride")
        self.dilation = self._tuple(dilation, "dilation")
        self.padding_mode = padding_mode or ZeroPad()
        k = math.sqrt(1.0 / (in_channels * math.prod(kernel)))
        self.weight = V.from_ndarray(device, uniform(rng, (out_channels, in_channels) + kernel, -k, k), dtype).requires_grad(grad_dtype)
        self.bias = V.from_ndarray(device, uniform(rng, (out_channels,) + (1,) * self.nsp, -k, k), dtype).requires_grad(grad_dtype)

    def _tuple(self, v, name):
        t = (int(v),) * self.nsp if np.isscalar(v) else tuple(int(x) for x in v)
        if len(t) != self.nsp:
            raise ValueError(f"{name} must have {self.nsp} entries, got {t}")
        return t

    def forward(self, input: V.Var) -> V.VarDiff:
        return V.conv_layer(input, self.weight, self.bias, self.padding, getattr(self.padding_mode, "mode", "constant"),
                            self.padding_mode.value, self.stride, self.dilation)

    def parameters(self):
        return [self.weight, self.bias]


class Conv1d(_ConvNd):
    """1-D convolution over (N, Cin, L): kernel_size, padding, stride and dilation as ints or 1-tuples."""
    nsp = 1

    def __init__(self, device: Device, in_channels: int, out_channels: int, kernel_size, padding=0, padding_mode=None,
                 stride=1, dilation=1, dtype=F32, grad_dtype=None, rng: np.random.Generator | None = None):
        super().__init__(device, in_channels, out_channels, kernel_size, padding, padding_mode, stride, dilation, dtype,
                         grad_dtype, rng)


class Conv3d(_ConvNd):
    """3-D convolution over (N, Cin, D, H, W): kernel_size, padding, stride and dilation as ints or 3-tuples."""
    nsp = 3

    def __init__(self, device: Device, in_channels: int, out_channels: int, kernel_size, padding=(0, 0, 0),
                 padding_mode=None, stride=(1, 1, 1), dilation=(1, 1, 1), dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None):
        super().__init__(device, in_channels, out_channels, kernel_size, padding, padding_mode, stride, dilation, dtype,
                         grad_dtype, rng)


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


class _Stacked:
    """`num_layers` layers of one or two directions, one graph node per layer (variable.lstm_layer / gru_layer).

    Layer k holds weight_ih_l{k} (D, G, I_k), weight_hh_l{k} (D, G, H), bias_ih_l{k} and bias_hh_l{k} (D, G), stacked
    over the D directions (index 1 = torch's `_reverse` parameters); I_0 = input_size and I_k = D*H above.  All are
    ~ U(-k, k), k = 1/sqrt(hidden_size), drawn from `rng` layer by layer, direction by direction, in the order weight_ih,
    weight_hh, bias_ih, bias_hh.  Torch weights port as `np.stack([w_l0, w_l0_reverse])` (or `w_l0[None]` for one
    direction): e.g. `weight_ih_l0 = np.stack([m.weight_ih_l0, m.weight_ih_l0_reverse])`.
    `dropout` > 0 applies Var.dropout to every layer's output but the last, while the module is in training mode
    (`train()`, the initial mode; `eval()` turns it off)."""

    num_layers, bidirectional, dropout = 1, False, 0.0
    _stacked = False   # the default configuration keeps the cell's parameters and results

    def _init_stacked(self, device, input_size, hidden_size, gates, dtype, grad_dtype, rng, num_layers, bidirectional,
                      dropout):
        if num_layers < 1:
            raise ValueError(f"num_layers must be at least 1, got {num_layers}")
        if not 0.0 <= dropout <= 1.0:
            raise ValueError(f"Wrong probability received: {dropout}.")
        self._stacked = True
        self.num_layers, self.bidirectional, self.dropout = int(num_layers), bool(bidirectional), float(dropout)
        self.hidden_size = int(hidden_size)
        self.status = V.Status(True)
        rng = rng or np.random.default_rng()
        k = 1.0 / math.sqrt(hidden_size)
        g, dirs = gates * hidden_size, 2 if bidirectional else 1
        for layer in range(self.num_layers):
            isz = input_size if layer == 0 else dirs * hidden_size
            drawn = [[], [], [], []]
            for _ in range(dirs):
                for i, shape in enumerate(((g, isz), (g, hidden_size), (g,), (g,))):
                    drawn[i].append(uniform(rng, shape, -k, k))
            for name, arrays in zip(self._names, drawn):
                setattr(self, f"{name}_l{layer}",
                        V.from_ndarray(device, np.stack(arrays), dtype).requires_grad(grad_dtype))

    _names = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")

    def _layer_params(self, layer):
        return [getattr(self, f"{name}_l{layer}") for name in self._names]

    def _run_stacked(self, layer_fn, states, input: V.Var):
        """`states`: the (num_layers*D, N, H) initial states, split per layer with one chunks node; returns (output,
        *last states), the last states of all layers joined with one cat node each."""
        dirs = 2 if self.bidirectional else 1
        if self.num_layers > 1:
            per_layer = [s.chunks((dirs,) + tuple(s.shape[1:])) for s in states]
        else:
            per_layer = [[s] for s in states]
        x, lasts = input, []
        for layer in range(self.num_layers):
            y, *last = layer_fn(x, [p[layer] for p in per_layer], self._layer_params(layer))
            if self.dropout > 0.0 and layer < self.num_layers - 1:
                y = y.dropout(self.dropout, self.status)
            x = y
            lasts.append(last)
        joined = [ls[0] if len(ls) == 1 else ls[0].cat(ls[1:], 0) for ls in zip(*lasts)]
        return (x, *joined)

    def _stacked_parameters(self):
        return [p for layer in range(self.num_layers) for p in self._layer_params(layer)]

    def train(self) -> None:
        """Dropout between the layers on (the initial mode)."""
        if self._stacked:
            self.status.train()

    def eval(self) -> None:
        """Dropout between the layers off."""
        if self._stacked:
            self.status.eval()


class LSTM(_Stacked, LSTMCell):
    """torch.nn.LSTM over a whole time-major sequence, one graph node per layer.

    With the defaults (one layer, one direction, no dropout) it is the LSTMCell applied to every step (variable.lstm):
    the cell's parameters weight_ih (4H, I), weight_hh, bias_ih, bias_hh and initialisation, so a layer built from the
    same `rng` seed holds the same weights.  With `num_layers` > 1 or `bidirectional` it holds the stacked parameters of
    `_Stacked` (weight_ih_l0 (D, 4H, I), ...) and takes and returns states shaped like torch's, (num_layers*D, N, H)."""

    def __init__(self, device: Device, input_size: int, hidden_size: int, dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None, num_layers: int = 1, bidirectional: bool = False,
                 dropout: float = 0.0):
        if num_layers == 1 and not bidirectional and dropout == 0.0:
            super().__init__(device, input_size, hidden_size, dtype, grad_dtype, rng)
        else:
            self._init_stacked(device, input_size, hidden_size, 4, dtype, grad_dtype, rng, num_layers, bidirectional,
                               dropout)

    def forward(self, state, input: V.Var):
        """`state = (cell_state, hidden)`; `input` (seq_len, batch, input_size).  With the defaults the states are
        (batch, hidden_size) and the result is (output, cell_T): every step's hidden state (seq_len, batch,
        hidden_size), whose last slice is the last hidden state, and the last cell state.  Otherwise the states are
        (num_layers*D, batch, hidden_size) and the result is (output, h_n, c_n) as torch.nn.LSTM returns it: output
        (seq_len, batch, D*hidden_size) of the last layer, and every layer's and direction's last states."""
        cell_state, hidden = state
        if not self._stacked:
            return V.lstm(input, cell_state, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)
        return self._run_stacked(lambda x, st, p: V.lstm_layer(x, st[0], st[1], *p), [cell_state, hidden], input)

    def parameters(self):
        return self._stacked_parameters() if self._stacked else super().parameters()


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


class _Pool:
    """The pooling layers: no parameters; `forward` is one graph node (Var.max_pool / avg_pool / adaptive_avg_pool)
    over an input with `nsp` sample dimensions after (N, C)."""

    nsp = 0

    def _check(self, input: V.Var) -> None:
        if len(input.shape) != self.nsp + 2:
            raise ValueError(f"{type(self).__name__} expects a {self.nsp + 2}-d (N, C, ...) input, got shape {input.shape}")

    def parameters(self):
        return []


class _MaxPoolNd(_Pool):
    def __init__(self, kernel_size, stride=None, padding=0, dilation=1, ceil_mode: bool = False):
        self.kernel_size, self.stride, self.padding = kernel_size, stride, padding
        self.dilation, self.ceil_mode = dilation, bool(ceil_mode)

    def forward(self, input: V.Var) -> V.Var:
        self._check(input)
        return input.max_pool(self.kernel_size, self.stride, self.padding, self.dilation, self.ceil_mode)


class _AvgPoolNd(_Pool):
    def __init__(self, kernel_size, stride=None, padding=0, ceil_mode: bool = False, count_include_pad: bool = True):
        self.kernel_size, self.stride, self.padding = kernel_size, stride, padding
        self.ceil_mode, self.count_include_pad = bool(ceil_mode), bool(count_include_pad)

    def forward(self, input: V.Var) -> V.Var:
        self._check(input)
        return input.avg_pool(self.kernel_size, self.stride, self.padding, self.ceil_mode, self.count_include_pad)


class _AdaptiveAvgPoolNd(_Pool):
    def __init__(self, output_size):
        self.output_size = output_size

    def forward(self, input: V.Var) -> V.Var:
        self._check(input)
        return input.adaptive_avg_pool(self.output_size)


class MaxPool1d(_MaxPoolNd):
    """torch.nn.MaxPool1d over (N, C, L)."""
    nsp = 1


class MaxPool2d(_MaxPoolNd):
    """torch.nn.MaxPool2d over (N, C, H, W)."""
    nsp = 2


class MaxPool3d(_MaxPoolNd):
    """torch.nn.MaxPool3d over (N, C, D, H, W)."""
    nsp = 3


class AvgPool1d(_AvgPoolNd):
    """torch.nn.AvgPool1d over (N, C, L)."""
    nsp = 1


class AvgPool2d(_AvgPoolNd):
    """torch.nn.AvgPool2d over (N, C, H, W)."""
    nsp = 2


class AvgPool3d(_AvgPoolNd):
    """torch.nn.AvgPool3d over (N, C, D, H, W)."""
    nsp = 3


class AdaptiveAvgPool1d(_AdaptiveAvgPoolNd):
    """torch.nn.AdaptiveAvgPool1d over (N, C, L)."""
    nsp = 1


class AdaptiveAvgPool2d(_AdaptiveAvgPoolNd):
    """torch.nn.AdaptiveAvgPool2d over (N, C, H, W); AdaptiveAvgPool2d(1) is global average pooling."""
    nsp = 2


class AdaptiveAvgPool3d(_AdaptiveAvgPoolNd):
    """torch.nn.AdaptiveAvgPool3d over (N, C, D, H, W)."""
    nsp = 3


class _BatchNorm:
    """torch's BatchNorm over (N, C, ...): weight = 1 and bias = 0 of the input's dtype when affine, f32 running_mean = 0
    and running_var = 1 when track_running_stats.  Each module owns a Status: `train()` (the initial mode) normalizes
    with the batch statistics and updates the running ones on every forward() of the graph, `eval()` normalizes with the
    running statistics (with the batch ones when not tracking).  `forward` is one graph node (Var.batch_norm)."""

    ranks: tuple = ()
    expected = ""

    def __init__(self, device: Device, num_features: int, eps: float = 1e-5, momentum: float | None = 0.1,
                 affine: bool = True, track_running_stats: bool = True, dtype=F32, grad_dtype=None):
        if momentum is None:
            raise ValueError("momentum=None (a cumulative moving average) is not supported")
        self.num_features, self.eps, self.momentum = int(num_features), float(eps), float(momentum)
        self.affine, self.track_running_stats = bool(affine), bool(track_running_stats)
        c = (self.num_features,)
        self.weight = self.bias = self.running_mean = self.running_var = None
        if self.affine:
            self.weight = V.from_ndarray(device, np.ones(c, np.float32), dtype).requires_grad(grad_dtype)
            self.bias = V.from_ndarray(device, np.zeros(c, np.float32), dtype).requires_grad(grad_dtype)
        if self.track_running_stats:
            self.running_mean = V.zeros(device, c)
            self.running_var = V.ones(device, c)
        self.status = V.Status(True)

    def forward(self, input: V.Var) -> V.Var:
        if len(input.shape) not in self.ranks:
            raise ValueError(f"expected {self.expected} input (got {len(input.shape)}D input)")
        return input.batch_norm(self.weight, self.bias, self.running_mean, self.running_var, self.status,
                                self.momentum, self.eps)

    def train(self) -> None:
        self.status.train()

    def eval(self) -> None:
        self.status.eval()

    def parameters(self):
        return [self.weight, self.bias] if self.affine else []


class BatchNorm1d(_BatchNorm):
    """torch.nn.BatchNorm1d over (N, C) or (N, C, L)."""
    ranks, expected = (2, 3), "2D or 3D"


class BatchNorm2d(_BatchNorm):
    """torch.nn.BatchNorm2d over (N, C, H, W)."""
    ranks, expected = (4,), "4D"


class BatchNorm3d(_BatchNorm):
    """torch.nn.BatchNorm3d over (N, C, D, H, W)."""
    ranks, expected = (5,), "5D"


class LayerNorm:
    """torch.nn.LayerNorm over the trailing dims `normalized_shape`: weight = 1 (when elementwise_affine) and bias = 0
    (when also `bias`) of that shape and the input's dtype.  `forward` is one graph node (Var.layer_norm)."""

    def __init__(self, device: Device, normalized_shape, eps: float = 1e-5, elementwise_affine: bool = True,
                 bias: bool = True, dtype=F32, grad_dtype=None):
        ns = (int(normalized_shape),) if np.isscalar(normalized_shape) else tuple(int(d) for d in normalized_shape)
        self.normalized_shape, self.eps, self.elementwise_affine = ns, float(eps), bool(elementwise_affine)
        self.weight = self.bias = None
        if self.elementwise_affine:
            self.weight = V.from_ndarray(device, np.ones(ns, np.float32), dtype).requires_grad(grad_dtype)
            if bias:
                self.bias = V.from_ndarray(device, np.zeros(ns, np.float32), dtype).requires_grad(grad_dtype)

    def forward(self, input: V.Var) -> V.Var:
        return input.layer_norm(self.normalized_shape, self.weight, self.bias, self.eps)

    def parameters(self):
        return [p for p in (self.weight, self.bias) if p is not None]


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


class GRU(_Stacked, GRUCell):
    """torch.nn.GRU over a whole time-major sequence, one graph node per layer.  With the defaults it is the GRUCell
    applied to every step (variable.gru), with the cell's parameters and initialisation; otherwise it holds the stacked
    parameters of `_Stacked` (weight_ih_l0 (D, 3H, I), ...)."""

    def __init__(self, device: Device, input_size: int, hidden_size: int, dtype=F32, grad_dtype=None,
                 rng: np.random.Generator | None = None, num_layers: int = 1, bidirectional: bool = False,
                 dropout: float = 0.0):
        if num_layers == 1 and not bidirectional and dropout == 0.0:
            super().__init__(device, input_size, hidden_size, dtype, grad_dtype, rng)
        else:
            self._init_stacked(device, input_size, hidden_size, 3, dtype, grad_dtype, rng, num_layers, bidirectional,
                               dropout)

    def forward(self, hidden: V.Var, input: V.Var):
        """`input` (seq_len, batch, input_size).  With the defaults `hidden` is (batch, hidden_size) and the result is
        every step's hidden state (seq_len, batch, hidden_size).  Otherwise `hidden` is (num_layers*D, batch,
        hidden_size) and the result is (output, h_n) as torch.nn.GRU returns it."""
        if not self._stacked:
            return V.gru(input, hidden, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)
        return self._run_stacked(lambda x, st, p: V.gru_layer(x, st[0], *p), [hidden], input)

    def parameters(self):
        return self._stacked_parameters() if self._stacked else super().parameters()
