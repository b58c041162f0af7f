"""Var / VarDiff: thin Python handles over the C++ graph (csrc/nk_graph.cpp, include/nk_graph.h).

Method names and semantics follow the reference's op surface (neuronika-variable/src/var.rs,
vardiff.rs): ops are lazy, `.forward()` recomputes the tape, `.backward(seed)` runs the backward
tape in reverse and every node accumulates into its operands' gradients."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .device import BF16, F32, CuArray, Device, as_shape, dtype_of

lib = L.lib
vp, i64, i32, f32 = C.c_void_p, C.c_int64, C.c_int, C.c_float
pvp = C.POINTER(vp)
pi64 = C.POINTER(C.c_int64)
pf32 = C.POINTER(C.c_float)

_G = {
    "nkg_last_error": (C.c_char_p, []),
    "nkg_leaf": (i32, [vp, i32, pi64, i32, pvp]),
    "nkg_leaf_external": (i32, [vp, i32, pi64, i32, vp, pvp]),
    "nkg_requires_grad": (i32, [vp, i32, vp, pvp]),
    "nkg_clone": (i32, [vp, pvp]),
    "nkg_release": (i32, [vp]),
    "nkg_is_diff": (i32, [vp]),
    "nkg_ndim": (i32, [vp]),
    "nkg_shape": (i32, [vp, pi64]),
    "nkg_dtype": (i32, [vp]),
    "nkg_grad_dtype": (i32, [vp]),
    "nkg_data_ptr": (vp, [vp]),
    "nkg_grad_ptr": (vp, [vp]),
    "nkg_history_len": (i32, [vp]),
    "nkg_backward_history_len": (i32, [vp]),
    "nkg_forward": (i32, [vp]),
    "nkg_backward": (i32, [vp, f32]),
    "nkg_zero_grad": (i32, [vp]),
    "nkg_no_grad": (i32, [vp]),
    "nkg_with_grad": (i32, [vp]),
    "nkg_set_fusion": (i32, [i32]),
    "nkg_mm": (i32, [vp, vp, pvp]),
    "nkg_mm_t": (i32, [vp, vp, pvp]),
    "nkg_add": (i32, [vp, vp, pvp]),
    "nkg_relu": (i32, [vp, pvp]),
    "nkg_softmax": (i32, [vp, i32, pvp]),
    "nkg_log_softmax": (i32, [vp, i32, pvp]),
    "nkg_sum": (i32, [vp, pvp]),
    "nkg_mean": (i32, [vp, pvp]),
    "nkg_mse_loss": (i32, [vp, vp, i32, pvp]),
    "nkg_nll_loss": (i32, [vp, vp, i32, pvp]),
    "nkg_pad": (i32, [vp, i64, i64, f32, pvp]),
    "nkg_convolution": (i32, [vp, vp, i64, i64, i64, i64, i64, pvp]),
    "nkg_flatten": (i32, [vp, pvp]),
    "nkg_sub": (i32, [vp, vp, pvp]),
    "nkg_mul": (i32, [vp, vp, pvp]),
    "nkg_div": (i32, [vp, vp, pvp]),
    "nkg_unary": (i32, [vp, i32, i32, pvp]),
    "nkg_neg": (i32, [vp, pvp]),
    "nkg_exp": (i32, [vp, pvp]),
    "nkg_ln": (i32, [vp, pvp]),
    "nkg_sqrt": (i32, [vp, pvp]),
    "nkg_sigmoid": (i32, [vp, pvp]),
    "nkg_tanh": (i32, [vp, pvp]),
    "nkg_softplus": (i32, [vp, pvp]),
    "nkg_leaky_relu": (i32, [vp, pvp]),
    "nkg_pow": (i32, [vp, i32, pvp]),
    "nkg_transpose": (i32, [vp, pvp]),
    "nkg_pad_mode": (i32, [vp, i32, pi64, i32, f32, pvp]),
    "nkg_mv": (i32, [vp, vp, pvp]),
    "nkg_vm": (i32, [vp, vp, pvp]),
    "nkg_vv": (i32, [vp, vp, pvp]),
    "nkg_convolution_nd": (i32, [vp, vp, i32, pi64, pi64, i64, pvp]),
    "nkg_conv_layer": (i32, [vp, vp, vp, i32, pi64, i32, f32, pi64, pi64, pvp]),
    "nkg_multi_sgd_step": (i32, [pvp, i32, pvp, pvp, vp, f32, f32, f32, i32, f32]),
    "nkg_multi_adam_step": (i32, [pvp, i32, pvp, pvp, pvp, pvp, vp, f32, f32, f32, f32, f32, f32]),
    "nkg_multi_rmsprop_step": (i32, [pvp, i32, pvp, pvp, pvp, pvp, vp, f32, f32, f32, f32, f32, f32]),
    "nkg_multi_adagrad_step": (i32, [pvp, i32, pvp, pvp, vp, f32, f32, f32, f32, f32]),
    "nkg_grad_norm": (i32, [pvp, i32, f32, f32, vp]),
    "nkg_clip_grads_with_norm": (i32, [pvp, i32, f32, vp]),
    "nkg_clip_grad_value": (i32, [pvp, i32, f32, f32]),
    "nkg_set_grad_hook": (i32, [vp, vp, vp, i32]),
    "nkg_set_grad_rs": (i32, [vp, i32, i32, pvp, vp, vp]),
    "nkg_chunks": (i32, [vp, i32, pi64, i32, pvp, C.POINTER(i32)]),
    "nkg_lstm_cell": (i32, [vp, vp, vp, vp, vp, vp, vp, pvp, pvp]),
    "nkg_gru_cell": (i32, [vp, vp, vp, vp, vp, vp, pvp]),
    "nkg_lstm": (i32, [vp, vp, vp, vp, vp, vp, vp, pvp, pvp]),
    "nkg_gru": (i32, [vp, vp, vp, vp, vp, vp, pvp]),
    "nkg_lstm_layer": (i32, [vp, vp, vp, vp, vp, vp, vp, pvp, pvp, pvp]),
    "nkg_gru_layer": (i32, [vp, vp, vp, vp, vp, vp, pvp, pvp]),
    "nkg_cat": (i32, [pvp, i32, i32, pvp]),
    "nkg_stack": (i32, [pvp, i32, i32, pvp]),
    "nkg_unsqueeze": (i32, [vp, i32, pvp]),
    "nkg_reshape": (i32, [vp, i32, pi64, pvp]),
    "nkg_embedding": (i32, [vp, vp, i64, pvp]),
    "nkg_cross_entropy": (i32, [vp, vp, vp, i32, i64, f32, pvp]),
    "nkg_mae": (i32, [vp, vp, i32, pvp]),
    "nkg_bce": (i32, [vp, vp, i32, pvp]),
    "nkg_bce_with_logits": (i32, [vp, vp, i32, pvp]),
    "nkg_kldiv": (i32, [vp, vp, i32, pvp]),
    "nkg_status_create": (i32, [i32, pvp]),
    "nkg_status_set": (i32, [vp, i32]),
    "nkg_status_get": (i32, [vp]),
    "nkg_status_release": (i32, [vp]),
    "nkg_dropout": (i32, [vp, C.c_double, vp, pvp]),
    "nkg_max_pool": (i32, [vp, i32, pi64, pi64, pi64, pi64, i32, pvp]),
    "nkg_avg_pool": (i32, [vp, i32, pi64, pi64, pi64, i32, i32, pvp]),
    "nkg_adaptive_avg_pool": (i32, [vp, i32, pi64, pvp]),
    "nkg_batch_norm": (i32, [vp, vp, vp, vp, vp, vp, f32, f32, pvp]),
    "nkg_layer_norm": (i32, [vp, i32, vp, vp, f32, pvp]),
}
for _n, (_r, _a) in _G.items():
    _f = getattr(lib, _n)
    _f.restype = _r
    _f.argtypes = _a


GRAD_HOOK = C.CFUNCTYPE(None, vp, i64, i64)
GRAD_RS_HOOK = C.CFUNCTYPE(None, vp, i32)


def graph_symbols():
    return sorted(_G)


def _ck(rc: int) -> None:
    if rc != 0:
        raise L.NkError(rc, lib.nkg_last_error().decode())


def set_fusion(level) -> None:
    """Host-side peephole fusion: False / 0 off, True / 1 (default) fusions that are invisible for any use of a tape,
    2 additionally fuses a layer's ReLU backward into the dX GEMM above it (exact for one backward() per tape, which
    is what a training loop does; a second backward() on such a tape raises); 3 additionally takes that layer's bias
    gradient in the same epilogue (nk_gemm_relu_bwd_colsum; correct, four launches fewer per MLP step, no measured gain,
    so nothing uses it by default)."""
    _ck(lib.nkg_set_fusion(int(level)))


class Reduction:
    """neuronika-variable/src/lib.rs:29-36"""
    Mean = 0
    Sum = 1


class Status:
    """The train / eval flag that dropout nodes share (the reference's `Rc<Cell<bool>>`): every node built with it reads
    it on each forward().  A captured step keeps the flag it was captured with."""

    def __init__(self, train: bool = True):
        h = vp()
        _ck(lib.nkg_status_create(int(bool(train)), C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                lib.nkg_status_release(self._h)
                self._h = None
        except Exception:
            pass

    def train(self) -> None:
        _ck(lib.nkg_status_set(self._h, 1))

    def eval(self) -> None:
        _ck(lib.nkg_status_set(self._h, 0))

    def get(self) -> bool:
        """True in training mode."""
        return bool(lib.nkg_status_get(self._h))


class Var:
    """A non-differentiable variable (var.rs:25-61) with data on the device."""

    def __init__(self, device: Device, handle):
        self.device = device
        self._h = vp(handle) if not isinstance(handle, vp) else handle

    def __del__(self):
        try:
            if self._h:
                lib.nkg_release(self._h)
                self._h = None
        except Exception:
            pass

    # ---- wrapping results
    def _wrap(self, out: vp):
        cls = VarDiff if lib.nkg_is_diff(out) else Var
        return cls(self.device, out)

    def _unary(self, fn, *args):
        out = vp()
        _ck(fn(self._h, *args, C.byref(out)))
        return self._wrap(out)

    def _binary(self, fn, other: "Var", *args):
        out = vp()
        _ck(fn(self._h, other._h, *args, C.byref(out)))
        return self._wrap(out)

    # ---- introspection
    @property
    def shape(self):
        n = lib.nkg_ndim(self._h)
        buf = (C.c_int64 * max(1, n))()
        _ck(lib.nkg_shape(self._h, buf))
        return tuple(int(buf[i]) for i in range(n))

    @property
    def dtype(self) -> int:
        return int(lib.nkg_dtype(self._h))

    def data(self) -> np.ndarray:
        """Copy of the data on the host (`Var::data`, var.rs:67-69).  Zeros before forward()."""
        return self.data_array().as_ndarray()

    def data_array(self) -> CuArray:
        ptr = lib.nkg_data_ptr(self._h)
        if not ptr:
            raise L.NkError(-1, lib.nkg_last_error().decode())
        return CuArray(self.device, self.shape, self.dtype, ptr=ptr, owner=self)

    def set_data(self, array: np.ndarray) -> None:
        """`*var.data_mut() = array` (var.rs:75-77)."""
        self.data_array().copy_from(array)

    def history_len(self) -> int:
        return int(lib.nkg_history_len(self._h))

    def clone(self) -> "Var":
        out = vp()
        _ck(lib.nkg_clone(self._h, C.byref(out)))
        return type(self)(self.device, out)

    # ---- differentiability
    def requires_grad(self, grad_dtype=None, grad_array: CuArray | None = None) -> "VarDiff":
        """`Var::requires_grad` (var.rs:104-107)."""
        out = vp()
        gd = -1 if grad_dtype is None else dtype_of(grad_dtype)
        _ck(lib.nkg_requires_grad(self._h, gd, grad_array.ptr if grad_array is not None else None, C.byref(out)))
        v = VarDiff(self.device, out)
        v._grad_owner = grad_array
        return v

    # ---- execution
    def forward(self) -> None:
        """var.rs:110-128"""
        _ck(lib.nkg_forward(self._h))

    # ---- operators (same names as the reference's methods / traits)
    def mm(self, other): return self._binary(lib.nkg_mm, other)                   # MatMatMul, core lib.rs:4-13
    def mm_t(self, other): return self._binary(lib.nkg_mm_t, other)               # MatMatMulT, core lib.rs:19-28
    def __add__(self, other): return self._binary(lib.nkg_add, other)
    def __sub__(self, other): return self._binary(lib.nkg_sub, other)             # subtraction/mod.rs
    def __mul__(self, other): return self._binary(lib.nkg_mul, other)             # multiplication/mod.rs
    def __truediv__(self, other): return self._binary(lib.nkg_div, other)         # division/mod.rs
    def __neg__(self): return self._unary(lib.nkg_neg)                            # negation/mod.rs
    def exp(self): return self._unary(lib.nkg_exp)
    def ln(self): return self._unary(lib.nkg_ln)
    def sqrt(self): return self._unary(lib.nkg_sqrt)
    def sigmoid(self): return self._unary(lib.nkg_sigmoid)
    def tanh(self): return self._unary(lib.nkg_tanh)
    def softplus(self): return self._unary(lib.nkg_softplus)
    def leaky_relu(self): return self._unary(lib.nkg_leaky_relu)
    def pow(self, exp: int): return self._unary(lib.nkg_pow, int(exp))            # power/mod.rs (`powi`)
    def t(self): return self._unary(lib.nkg_transpose)                            # transpose/mod.rs (reverses all axes)
    def mv(self, vector): return self._binary(lib.nkg_mv, vector)                 # MatVecMul, core lib.rs
    def vm(self, matrix): return self._binary(lib.nkg_vm, matrix)                 # VecMatMul
    def vv(self, other): return self._binary(lib.nkg_vv, other)                   # VecVecMul
    def relu(self): return self._unary(lib.nkg_relu)
    def softmax(self, axis: int): return self._unary(lib.nkg_softmax, int(axis))
    def log_softmax(self, axis: int): return self._unary(lib.nkg_log_softmax, int(axis))
    def sum(self): return self._unary(lib.nkg_sum)
    def mean(self): return self._unary(lib.nkg_mean)
    def mse_loss(self, target, reduction=Reduction.Mean): return self._binary(lib.nkg_mse_loss, target, int(reduction))
    def nll_loss(self, target, reduction=Reduction.Mean): return self._binary(lib.nkg_nll_loss, target, int(reduction))

    def cross_entropy(self, target, reduction=Reduction.Mean, weight=None, ignore_index: int = -100,
                      label_smoothing: float = 0.0):
        """torch's F.cross_entropy with class-index targets, as ONE node: the receiver holds the logits, (N, C) or
        (N, C, d1, ..., dk); `target` (N) or (N, d1, ..., dk) holds float class ids (f32, or bf16 for C <= 256) and is
        not differentiable; `weight` is None or an f32 (C,) Var.  Positions whose id equals `ignore_index`, or is not a
        class (NaN, < 0, >= C: torch raises there), are left out.  Mean divides by the summed weights of the other
        positions, as torch does (nll_loss's Mean divides by N); it is NaN when every position is ignored."""
        out = vp()
        _ck(lib.nkg_cross_entropy(self._h, target._h, weight._h if weight is not None else None, int(reduction),
                                  int(ignore_index), float(label_smoothing), C.byref(out)))
        return self._wrap(out)
    def mae(self, target, reduction=Reduction.Mean): return self._binary(lib.nkg_mae, target, int(reduction))
    def bce(self, target, reduction=Reduction.Mean): return self._binary(lib.nkg_bce, target, int(reduction))

    def bce_with_logits(self, target, reduction=Reduction.Mean):
        return self._binary(lib.nkg_bce_with_logits, target, int(reduction))

    def kldiv(self, target, reduction=Reduction.Mean):
        """KL divergence of `target` (probabilities) from the receiver (log-probabilities).  Mean divides by the
        leading (batch) dimension, like torch's reduction='batchmean', not by the element count."""
        return self._binary(lib.nkg_kldiv, target, int(reduction))

    def dropout(self, p: float, status: Status | None = None):
        """`dropout(p, status)` (var.rs:375-397): zeroes each element with probability p and scales the rest by 1/(1-p)
        while `status` is in training mode; a copy in eval mode.  Each forward() draws a new mask from the device's
        Philox generator (Device.manual_seed).  Without a status the node has its own, in training mode."""
        return self._unary(lib.nkg_dropout, float(p), (status or Status())._h)

    def flatten(self): return self._unary(lib.nkg_flatten)

    def _nsp_tuple(self, v, name):
        nsp = len(self.shape) - 2
        t = (int(v),) * nsp if np.isscalar(v) else tuple(int(x) for x in v)
        if len(t) != nsp or not 1 <= nsp <= 3:
            raise L.NkError(-1, f"Invalid {name} {list(t)} for a pool over {nsp} sample dimensions.")
        return t

    def max_pool(self, kernel_size, stride=None, padding=0, dilation=1, ceil_mode: bool = False):
        """torch's max_pool{1,2,3}d over the sample dims of a (N, C, ...) operand, as one node; ints broadcast to every
        sample dim and stride defaults to kernel_size.  The backward sends each output's gradient to its window's first
        maximum (the last NaN), through int32 indices the node keeps when the operand is differentiable."""
        k = self._nsp_tuple(kernel_size, "kernel_size")
        s = self._nsp_tuple(kernel_size if stride is None else stride, "stride")
        p, d = self._nsp_tuple(padding, "padding"), self._nsp_tuple(dilation, "dilation")
        return self._unary(lib.nkg_max_pool, len(k), *(L.shape_arr(t) for t in (k, s, p, d)), int(bool(ceil_mode)))

    def avg_pool(self, kernel_size, stride=None, padding=0, ceil_mode: bool = False, count_include_pad: bool = True):
        """torch's avg_pool{1,2,3}d over the sample dims of a (N, C, ...) operand, as one node."""
        k = self._nsp_tuple(kernel_size, "kernel_size")
        s = self._nsp_tuple(kernel_size if stride is None else stride, "stride")
        p = self._nsp_tuple(padding, "padding")
        return self._unary(lib.nkg_avg_pool, len(k), *(L.shape_arr(t) for t in (k, s, p)), int(bool(ceil_mode)),
                           int(bool(count_include_pad)))

    def adaptive_avg_pool(self, output_size):
        """torch's adaptive_avg_pool{1,2,3}d over the sample dims of a (N, C, ...) operand, as one node: window i of an
        axis is [floor(i*L/O), ceil((i+1)*L/O))."""
        o = self._nsp_tuple(output_size, "output_size")
        return self._unary(lib.nkg_adaptive_avg_pool, len(o), L.shape_arr(o))

    def batch_norm(self, weight=None, bias=None, running_mean=None, running_var=None, status: Status | None = None,
                   momentum: float = 0.1, eps: float = 1e-5):
        """torch's batch_norm over N and the sample dims of an (N, C, ...) operand, as one node.  weight / bias: (C,)
        of the operand's dtype or None; running_mean / running_var: f32 (C,) Vars (not differentiable) updated in place
        by every training forward, or both None.  `status` (a Status; training when None) is read on each forward():
        batch statistics in training mode or without running statistics, the running ones otherwise."""
        h = lambda v: v._h if v is not None else None
        return self._unary(lib.nkg_batch_norm, h(weight), h(bias), h(running_mean), h(running_var),
                           (status or Status())._h, float(momentum), float(eps))

    def layer_norm(self, normalized_shape, weight=None, bias=None, eps: float = 1e-5):
        """torch's layer_norm over the trailing dims `normalized_shape`, as one node; weight / bias have that shape and
        the operand's dtype, or are None."""
        ns = (int(normalized_shape),) if np.isscalar(normalized_shape) else tuple(int(d) for d in normalized_shape)
        shape = self.shape
        if not ns or len(ns) > len(shape) or shape[len(shape) - len(ns):] != ns:
            raise L.NkError(-1, f"Given normalized_shape={list(ns)}, expected input with shape [*, "
                                f"{', '.join(str(d) for d in ns)}], but got input of size{list(shape)}")
        h = lambda v: v._h if v is not None else None
        return self._unary(lib.nkg_layer_norm, len(ns), h(weight), h(bias), float(eps))

    def pad(self, padding, value: float = 0.0, mode: str = "constant"):
        """`pad(padding, mode)` (var.rs:726-737): Zero / Constant(value) / Reflective / Replicative over the 1..3
        sample dimensions of a (N, C, ...) operand."""
        padding = tuple(int(p) for p in padding)
        if len(padding) == 2 and _pad_mode(mode) == L.NK_PAD_CONSTANT:
            return self._unary(lib.nkg_pad, padding[0], padding[1], float(value))
        return self._unary(lib.nkg_pad_mode, len(padding), L.shape_arr(padding), _pad_mode(mode), float(value))

    def convolution(self, input, stride=(1, 1), dilation=(1, 1), groups: int = 1):
        """`kernel.convolution(input, stride, dilation, groups)` -- the receiver is the kernel
        (Convolution trait, core lib.rs:91-106; var.rs:704-716)."""
        nsp = len(self.shape) - 2
        if len(stride) != nsp:
            raise L.NkError(-1, f"Invalid stride {list(stride)} for {nsp}d conv.")
        if len(dilation) != nsp:
            raise L.NkError(-1, f"Invalid dilation {list(dilation)} for {nsp}d conv.")
        if nsp != 2:       # 1-d / 3-d operands (convolution/mod.rs is generic over the sample dimensions)
            return self._binary(lib.nkg_convolution_nd, input, nsp, L.shape_arr(stride), L.shape_arr(dilation),
                                int(groups))
        return self._binary(lib.nkg_convolution, input, int(stride[0]), int(stride[1]), int(dilation[0]),
                            int(dilation[1]), int(groups))

    def chunks(self, chunk_shape) -> list:
        """`chunks(chunk_size)` (var.rs:401-417): the blocks of ndarray's exact_chunks in row-major block order (trailing
        partial blocks dropped), one lazy node each; differentiable when the receiver is."""
        cs = tuple(int(c) for c in chunk_shape)
        count = C.c_int(0)
        _ck(lib.nkg_chunks(self._h, len(cs), L.shape_arr(cs), 0, None, C.byref(count)))
        outs = (vp * max(1, count.value))()
        _ck(lib.nkg_chunks(self._h, len(cs), L.shape_arr(cs), count.value, outs, C.byref(count)))
        return [self._wrap(vp(outs[i])) for i in range(count.value)]

    def cat(self, others, axis: int):
        """`cat(variables, axis)` (var.rs:564-587, vardiff.rs:627-641): the receiver and `others` side by side along
        `axis`, as ONE node; differentiable when any operand is, and only those operands receive gradients."""
        return _join(lib.nkg_cat, [self, *others], axis)

    def stack(self, others, axis: int):
        """`stack(variables, axis)` (var.rs:622-645, vardiff.rs:681-): the receiver and `others` (one shape) along a new
        axis, as ONE node."""
        return _join(lib.nkg_stack, [self, *others], axis)

    def unsqueeze(self, axis: int):
        """`unsqueeze(axis)` (var.rs:425-431): a new axis of length 1.  A view like flatten(): no kernel and no node
        (the reference records one)."""
        return self._unary(lib.nkg_unsqueeze, int(axis))

    def reshape(self, *shape):
        """torch's reshape of a contiguous tensor: the same elements under `shape` (ints or one tuple), at most one -1
        (inferred).  A view like flatten(): no kernel and no node, and the gradient is the operand's."""
        if len(shape) == 1 and isinstance(shape[0], (tuple, list)):
            shape = tuple(shape[0])
        shape = [int(s) for s in shape]
        size = int(np.prod(self.shape, dtype=np.int64))
        if shape.count(-1) > 1:
            raise RuntimeError("only one dimension can be inferred")
        if any(s < -1 for s in shape):
            raise RuntimeError(f"invalid shape dimension {min(shape)}")
        known = int(np.prod([s for s in shape if s != -1], dtype=np.int64))
        if -1 in shape:
            if known == 0 or size % known:
                raise RuntimeError(f"shape '{shape}' is invalid for input of size {size}")
            shape[shape.index(-1)] = size // known
        elif known != size:
            raise RuntimeError(f"shape '{shape}' is invalid for input of size {size}")
        return self._unary(lib.nkg_reshape, len(shape), L.shape_arr(shape))

    def item(self) -> float:
        return float(self.data().reshape(()))


class VarDiff(Var):
    """A differentiable variable (vardiff.rs:25-65)."""

    def __init__(self, device, handle):
        super().__init__(device, handle)
        self._grad_owner = None

    @property
    def grad_dtype(self) -> int:
        return int(lib.nkg_grad_dtype(self._h))

    def grad(self) -> np.ndarray:
        """`VarDiff::grad` (vardiff.rs:84-86)."""
        return self.grad_array().as_ndarray()

    def grad_array(self) -> CuArray:
        ptr = lib.nkg_grad_ptr(self._h)
        if not ptr:
            raise L.NkError(-1, "Trying to get a de-allocated gradient. Switch on the gradients first by "
                                "using `.with_grad()`")
        return CuArray(self.device, self.shape, self.grad_dtype, ptr=ptr, owner=self)

    def backward(self, seed: float) -> None:
        """vardiff.rs:125-141"""
        _ck(lib.nkg_backward(self._h, float(seed)))

    def zero_grad(self) -> None:
        _ck(lib.nkg_zero_grad(self._h))

    def no_grad(self) -> None:
        _ck(lib.nkg_no_grad(self._h))

    def with_grad(self) -> None:
        _ck(lib.nkg_with_grad(self._h))

    def backward_history_len(self) -> int:
        return int(lib.nkg_backward_history_len(self._h))

    def set_grad_hook(self, fn, row_chunks: int = 1) -> None:
        """Call `fn(begin, end)` from inside backward() as soon as elements [begin, end) of this leaf's gradient are
        final for the running pass (used to overlap the data-parallel all-reduce with the rest of backward).  With
        row_chunks > 1 a matmul backward that writes the gradient last delivers it in that many row blocks."""
        if fn is None:
            self._hook_ref = None
            _ck(lib.nkg_set_grad_hook(self._h, None, None, 1))
            return
        cb = GRAD_HOOK(lambda _user, b, e: fn(int(b), int(e)))
        self._hook_ref = cb  # keep the trampoline alive
        _ck(lib.nkg_set_grad_hook(self._h, C.cast(cb, vp), None, int(row_chunks)))


    def set_grad_rs(self, world: int, rank: int, slot_ptrs, fn) -> None:
        """Fused data-parallel exchange (nk_b200.h nk_gemm_rs): the matmul backward node that produces this leaf's
        gradient pushes row shard o of its product into `slot_ptrs[o]` (rank o's slot buffer, peer-mapped) and then
        calls `fn(pushed)`; pushed == 0 means the gradient was computed locally (caller falls back to all-reduce)."""
        if world <= 1:
            self._rs_ref = None
            _ck(lib.nkg_set_grad_rs(self._h, 0, 0, None, None, None))
            return
        arr = (vp * world)(*[int(p) for p in slot_ptrs])
        cb = GRAD_RS_HOOK(lambda _user, pushed: fn(int(pushed)))
        self._rs_ref = (cb, arr)
        _ck(lib.nkg_set_grad_rs(self._h, int(world), int(rank), arr, C.cast(cb, vp), None))


_PAD_MODES = {"constant": L.NK_PAD_CONSTANT, "zero": L.NK_PAD_CONSTANT, "reflective": L.NK_PAD_REFLECTIVE,
              "replicative": L.NK_PAD_REPLICATIVE}


def _pad_mode(mode: str) -> int:
    if mode not in _PAD_MODES:
        raise L.NkError(-1, f"unknown padding mode {mode!r}")
    return _PAD_MODES[mode]


# ---- the 1-d / 3-d convolution layer (one node; see include/nk_graph.h nkg_conv_layer)
def conv_layer(input: Var, weight: Var, bias: Var | None, padding, mode: str = "zero", value: float = 0.0, stride=None,
               dilation=None):
    """`conv(pad(input, padding, mode), weight, stride, dilation) + bias` as ONE node, for input (N, Cin, L) or
    (N, Cin, D, H, W): weight (Cout, Cin, k...), bias (Cout, 1) / (Cout, 1, 1, 1) or None.  `mode` is one of
    Var.pad's modes ("zero", "constant" with `value`, "reflective", "replicative").  The same results as those three
    nodes; the input gradient is the interior slice of the padded input's gradient for every mode, as in Var.pad."""
    nsp = len(input.shape) - 2
    padding = tuple(int(p) for p in padding)
    stride = tuple(int(s) for s in (stride or (1,) * nsp))
    dilation = tuple(int(d) for d in (dilation or (1,) * nsp))
    for name, t in (("padding", padding), ("stride", stride), ("dilation", dilation)):
        if len(t) != nsp:
            raise L.NkError(-1, f"Invalid {name} {list(t)} for {nsp}d conv.")
    out = vp()
    _ck(lib.nkg_conv_layer(input._h, weight._h, bias._h if bias is not None else None, nsp, L.shape_arr(padding),
                           _pad_mode(mode), float(value), L.shape_arr(stride), L.shape_arr(dilation), C.byref(out)))
    return input._wrap(out)


# ---- embedding (one node; see include/nk_graph.h nkg_embedding)
def embedding(ids: Var, weight: Var, padding_idx: int | None = None):
    """torch's F.embedding(ids, weight, padding_idx): weight (v, e), ids a non-differentiable Var of float ids (f32,
    or bf16 for v <= 256) of any shape; the result has shape ids.shape + (e,).  Invalid ids (NaN, < 0, >= v) give zero
    rows and no gradient; a negative padding_idx counts from v."""
    v = weight.shape[0] if len(weight.shape) == 2 else 0
    pad = -1
    if padding_idx is not None:
        pad = int(padding_idx)
        if pad < 0:
            pad += v
        if not 0 <= pad < v:
            raise ValueError("Padding_idx must be within num_embeddings")
    out = vp()
    _ck(lib.nkg_embedding(ids._h, weight._h, pad, C.byref(out)))
    return weight._wrap(out)


# ---- concatenation (neuronika-variable/src/lib.rs:258, 281)
def _join(fn, vars, axis):
    handles = (vp * len(vars))(*[v._h.value for v in vars])
    out = vp()
    _ck(fn(handles, len(vars), int(axis), C.byref(out)))
    return vars[0]._wrap(out)


def cat(lhs: Var, rhs: Var, axis: int):
    """`cat(lhs, rhs, axis)`: the two side by side along `axis`, any mix of Var and VarDiff."""
    return _join(lib.nkg_cat, [lhs, rhs], axis)


def stack(lhs: Var, rhs: Var, axis: int):
    """`stack(lhs, rhs, axis)`: the two (one shape) along a new axis, any mix of Var and VarDiff."""
    return _join(lib.nkg_stack, [lhs, rhs], axis)


# ---- recurrent cells (one fused node per step; see include/nk_graph.h)
def lstm_cell(input: Var, cell_state: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """One LSTM step, gate chunks [i | f | g | o] (torch.nn.LSTMCell): returns (new_cell_state, new_hidden)."""
    c, h = vp(), vp()
    _ck(lib.nkg_lstm_cell(input._h, cell_state._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h,
                          C.byref(c), C.byref(h)))
    return input._wrap(c), input._wrap(h)


def gru_cell(input: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """One GRU step, gate chunks [r | z | n] (torch.nn.GRUCell): returns the new hidden state."""
    h = vp()
    _ck(lib.nkg_gru_cell(input._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h, C.byref(h)))
    return input._wrap(h)


# ---- recurrent sequence layers (one node per sequence; see include/nk_graph.h)
def lstm(input: Var, cell_state: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """An LSTM over a whole time-major sequence, as ONE node: `input` (T, N, I), `cell_state` and `hidden` (N, H), the
    weights as `lstm_cell` takes them.  Returns (output, cell_T): `output` (T, N, H) holds every step's hidden state and
    `cell_T` (N, H) the last cell state.  The last hidden state is `output[T-1]`; it is not a third result."""
    y, c = vp(), vp()
    _ck(lib.nkg_lstm(input._h, cell_state._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h,
                     C.byref(y), C.byref(c)))
    return input._wrap(y), input._wrap(c)


def gru(input: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """A GRU over a whole time-major sequence, as ONE node: `input` (T, N, I), `hidden` (N, H), the weights as `gru_cell`
    takes them.  Returns `output` (T, N, H), every step's hidden state; the last one is `output[T-1]`."""
    y = vp()
    _ck(lib.nkg_gru(input._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h, C.byref(y)))
    return input._wrap(y)


def lstm_layer(input: Var, cell_state: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """One layer of torch.nn.LSTM with D = 1 or 2 directions (D = hidden.shape[0]), as ONE node: `input` (T, N, I),
    `cell_state` and `hidden` (D, N, H), the parameters stacked over the directions: weight_ih (D, 4H, I), weight_hh
    (D, 4H, H), biases (D, 4H).  Returns (output, h_n, c_n): `output` (T, N, D*H), the reverse direction in columns
    [H, 2H), and each direction's last hidden and cell state, (D, N, H)."""
    y, h, c = vp(), vp(), vp()
    _ck(lib.nkg_lstm_layer(input._h, cell_state._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h,
                           C.byref(y), C.byref(h), C.byref(c)))
    return input._wrap(y), input._wrap(h), input._wrap(c)


def gru_layer(input: Var, hidden: Var, weight_ih: Var, weight_hh: Var, bias_ih: Var, bias_hh: Var):
    """One layer of torch.nn.GRU with D = 1 or 2 directions, as ONE node; the operands as `lstm_layer` takes them (gates
    3H).  Returns (output, h_n): `output` (T, N, D*H) and each direction's last hidden state (D, N, H)."""
    y, h = vp(), vp()
    _ck(lib.nkg_gru_layer(input._h, hidden._h, weight_ih._h, weight_hh._h, bias_ih._h, bias_hh._h, C.byref(y),
                          C.byref(h)))
    return input._wrap(y), input._wrap(h)


# ---- constructors (neuronika-variable/src/lib.rs:51-240), on a device
def zeros(device: Device, shape, dtype=F32) -> Var:
    shape = as_shape(shape)
    out = vp()
    _ck(lib.nkg_leaf(device.ctx, len(shape), L.shape_arr(shape), dtype_of(dtype), C.byref(out)))
    return Var(device, out)


def full(device: Device, shape, value: float, dtype=F32) -> Var:
    v = zeros(device, shape, dtype)
    v.data_array().fill_(value)
    return v


def ones(device: Device, shape, dtype=F32) -> Var:
    return full(device, shape, 1.0, dtype)


def from_ndarray(device: Device, array: np.ndarray, dtype=F32) -> Var:
    v = zeros(device, np.shape(array), dtype)
    v.set_data(array)
    return v


def rand(device: Device, shape, dtype=F32, rng: np.random.Generator | None = None) -> Var:
    """U(0,1) like `neuronika::rand`; host-generated (the reference uses an unseeded thread_rng)."""
    rng = rng or np.random.default_rng()
    return from_ndarray(device, rng.random(as_shape(shape), dtype=np.float32), dtype)


def from_device_memory(device: Device, array: CuArray) -> Var:
    """Leaf over caller-owned device memory (parameter / gradient buckets)."""
    out = vp()
    _ck(lib.nkg_leaf_external(device.ctx, array.ndim, L.shape_arr(array.shape), array.dtype, array.ptr, C.byref(out)))
    v = Var(device, out)
    v._keep = array  # keep the storage alive as long as the handle
    return v
