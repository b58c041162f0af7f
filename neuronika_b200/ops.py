"""Functional wrappers: one Python function per C-ABI operator entry point (include/nk_b200.h).

Each takes/returns CuArray and launches asynchronously on the device's stream.  `beta`
selects the reference's accumulate protocol on backward ops (1 = `+=`, the reference
behaviour; 0 = overwrite a buffer known to be zero)."""
from __future__ import annotations

import numpy as np

from . import _lib as L
from .device import BF16, F32, CuArray, Device

lib = L.lib


def _ck(rc, dev: Device):
    L.check(rc, dev.ctx)


# ---------------------------------------------------------------- gemm
def gemm(a: CuArray, b: CuArray, c: CuArray, trans_a=False, trans_b=False, alpha=1.0, beta=0.0,
         bias: CuArray | None = None, relu=False) -> CuArray:
    """c = alpha*op(a).op(b) + beta*c (+bias, relu); shapes are the stored (row-major) shapes."""
    dev = a.device
    m, k = (a.shape[1], a.shape[0]) if trans_a else a.shape
    kb, n = (b.shape[1], b.shape[0]) if trans_b else b.shape
    if k != kb or tuple(c.shape) != (m, n):
        raise ValueError(f"gemm: shape mismatch op(a)=({m},{k}) op(b)=({kb},{n}) c={c.shape}")
    if a.dtype != b.dtype:
        raise ValueError("gemm: operand dtypes differ")
    _ck(lib.nk_gemm_bias_act(dev.ctx, int(trans_a), int(trans_b), m, n, k, float(alpha), a.ptr, a.shape[1],
                             b.ptr, b.shape[1], float(beta), c.ptr, n, a.dtype, c.dtype,
                             bias.ptr if bias is not None else None, bias.dtype if bias is not None else F32,
                             int(relu)), dev)
    return c


def gemm_strided_batched(a: CuArray, b: CuArray, c: CuArray, m: int, n: int, k: int, batch: int, lda: int, ldb: int,
                         ldc: int, stride_a: int, stride_b: int, stride_c: int, trans_a=False, trans_b=False, alpha=1.0,
                         beta=0.0, bias: CuArray | None = None, bias_stride: int = 0) -> CuArray:
    """`batch` products c_i = alpha*op(a_i).op(b_i) + beta*c_i + bias_i, where x_i starts stride_x elements after x_{i-1}
    (the arrays' first elements are the first product's) and bias_i (n elements) bias_stride after bias_{i-1}."""
    dev = a.device
    if a.dtype != b.dtype:
        raise ValueError("gemm_strided_batched: operand dtypes differ")
    _ck(lib.nk_gemm_strided_batched(dev.ctx, int(trans_a), int(trans_b), m, n, k, float(alpha), a.ptr, lda, stride_a,
                                    b.ptr, ldb, stride_b, float(beta), c.ptr, ldc, stride_c, batch, a.dtype, c.dtype,
                                    bias.ptr if bias is not None else None, bias_stride,
                                    bias.dtype if bias is not None else F32), dev)
    return c


def mm(a, b, out=None, out_dtype=None):
    out = out or CuArray(a.device, (a.shape[0], b.shape[1]), out_dtype if out_dtype is not None else a.dtype)
    return gemm(a, b, out)


def mm_t(x, w, out=None, out_dtype=None, bias=None, relu=False):
    out = out or CuArray(x.device, (x.shape[0], w.shape[0]), out_dtype if out_dtype is not None else x.dtype)
    return gemm(x, w, out, trans_b=True, bias=bias, relu=relu)


# ---------------------------------------------------------------- broadcast add
def cobroadcast(ls, rs):
    """utils.rs:97-125"""
    big, small = (ls, rs) if len(ls) >= len(rs) else (rs, ls)
    out = list(big)
    off = len(big) - len(small)
    for i, r in enumerate(small):
        l = out[off + i]
        if l != r:
            if l == 1:
                out[off + i] = r
            elif r != 1:
                raise ValueError("The two tensors have incompatible shape.")
    return tuple(out)


def add(l: CuArray, r: CuArray, out: CuArray | None = None) -> CuArray:
    dev = l.device
    shape = cobroadcast(l.shape, r.shape)
    out = out or CuArray(dev, shape, l.dtype)
    _ck(lib.nk_add_bcast_fwd(dev.ctx, out.ptr, l.ptr, r.ptr, l.dtype, len(shape), L.shape_arr(shape),
                             l.ndim, L.shape_arr(l.shape), r.ndim, L.shape_arr(r.shape)), dev)
    return out


def unbroadcast_acc(dst: CuArray, g: CuArray, beta=1.0) -> CuArray:
    dev = g.device
    _ck(lib.nk_unbroadcast_acc(dev.ctx, dst.ptr, dst.dtype, dst.ndim, L.shape_arr(dst.shape), g.ptr, g.dtype,
                               g.ndim, L.shape_arr(g.shape), float(beta)), dev)
    return dst


# ---------------------------------------------------------------- relu / softmax
def relu(x: CuArray, out=None) -> CuArray:
    out = out or CuArray(x.device, x.shape, x.dtype)
    _ck(lib.nk_relu_fwd(x.device.ctx, out.ptr, x.ptr, x.size, x.dtype), x.device)
    return out


def relu_bwd(dx: CuArray, x: CuArray, g: CuArray, beta=1.0) -> CuArray:
    _ck(lib.nk_relu_bwd(x.device.ctx, dx.ptr, x.ptr, g.ptr, x.size, x.dtype, float(beta)), x.device)
    return dx


def _lanes(shape, axis):
    outer = int(np.prod(shape[:axis])) if axis > 0 else 1
    inner = int(np.prod(shape[axis + 1:])) if axis + 1 < len(shape) else 1
    return outer, int(shape[axis]), inner


def softmax(x: CuArray, axis: int, out=None, log=False) -> CuArray:
    out = out or CuArray(x.device, x.shape, x.dtype)
    o, n, i = _lanes(x.shape, axis)
    fn = lib.nk_log_softmax_fwd if log else lib.nk_softmax_fwd
    _ck(fn(x.device.ctx, out.ptr, x.ptr, o, n, i, x.dtype), x.device)
    return out


def softmax_bwd(dx: CuArray, y: CuArray, g: CuArray, axis: int, beta=1.0, log=False) -> CuArray:
    o, n, i = _lanes(y.shape, axis)
    fn = lib.nk_log_softmax_bwd if log else lib.nk_softmax_bwd
    _ck(fn(y.device.ctx, dx.ptr, y.ptr, g.ptr, o, n, i, y.dtype, float(beta)), y.device)
    return dx


# ---------------------------------------------------------------- losses / reductions
def mse(x: CuArray, t: CuArray, mean=True, out=None) -> CuArray:
    out = out or CuArray(x.device, (), F32)
    _ck(lib.nk_mse_fwd(x.device.ctx, out.ptr, x.ptr, t.ptr, x.size, x.dtype, int(mean)), x.device)
    return out


def mse_bwd(dx, x, t, g: CuArray, mean=True, beta=1.0):
    _ck(lib.nk_mse_bwd(x.device.ctx, dx.ptr, x.ptr, t.ptr, g.ptr, x.size, x.dtype, int(mean), float(beta)), x.device)
    return dx


def nll(logp: CuArray, target: CuArray, mean=True, out=None) -> CuArray:
    out = out or CuArray(logp.device, (), F32)
    n, c = logp.shape
    _ck(lib.nk_nll_fwd(logp.device.ctx, out.ptr, logp.ptr, target.ptr, target.dtype, n, c, logp.dtype, int(mean)),
        logp.device)
    return out


def nll_bwd(dlogp, target, g, mean=True, beta=1.0):
    n, c = dlogp.shape
    _ck(lib.nk_nll_bwd(dlogp.device.ctx, dlogp.ptr, target.ptr, target.dtype, g.ptr, n, c, dlogp.dtype, int(mean),
                       float(beta)), dlogp.device)
    return dlogp


def _ce_dims(x: CuArray):
    s = 1
    for d in x.shape[2:]:
        s *= int(d)
    return x.shape[0], x.shape[1], s


def cross_entropy(x: CuArray, target: CuArray, weight: CuArray | None = None, mean=True, ignore_index=-100,
                  label_smoothing=0.0, out=None, lse=None, denom=None):
    """torch's F.cross_entropy with class-index targets (nk_cross_entropy_fwd): x (N, C, d1, ...), target (N, d1, ...)
    float class ids, weight f32 (C,) or None.  Returns (loss, lse, denom): the 0-d f32 loss, the per-position f32 lse
    (N*S) and the 0-d f32 denominator that cross_entropy_bwd reads."""
    n, c, s = _ce_dims(x)
    out = out or CuArray(x.device, (), F32)
    lse = lse or CuArray(x.device, (n * s,), F32)
    denom = denom or CuArray(x.device, (), F32)
    _ck(lib.nk_cross_entropy_fwd(x.device.ctx, out.ptr, lse.ptr, denom.ptr, x.ptr, x.dtype, target.ptr, target.dtype,
                                 weight.ptr if weight is not None else None, n, c, s, int(ignore_index),
                                 float(label_smoothing), int(mean)), x.device)
    return out, lse, denom


def cross_entropy_bwd(dx: CuArray, x: CuArray, target: CuArray, lse: CuArray, denom: CuArray, g: CuArray,
                      weight: CuArray | None = None, mean=True, ignore_index=-100, label_smoothing=0.0,
                      beta=1.0) -> CuArray:
    """dx = beta*dx + the cross-entropy gradient times the seed g (nk_cross_entropy_bwd), dx in its own element type"""
    n, c, s = _ce_dims(x)
    _ck(lib.nk_cross_entropy_bwd(x.device.ctx, dx.ptr, dx.dtype, x.ptr, x.dtype, target.ptr, target.dtype,
                                 weight.ptr if weight is not None else None, lse.ptr, denom.ptr, g.ptr, n, c, s,
                                 int(ignore_index), float(label_smoothing), int(mean), float(beta)), x.device)
    return dx


_CRITERIA = {"mae": (lib.nk_mae_fwd, lib.nk_mae_bwd), "bce": (lib.nk_bce_fwd, lib.nk_bce_bwd),
             "bce_with_logits": (lib.nk_bce_with_logits_fwd, lib.nk_bce_with_logits_bwd),
             "kldiv": (lib.nk_kldiv_fwd, lib.nk_kldiv_bwd)}


def criterion(name: str, x: CuArray, t: CuArray, mean=True, out=None) -> CuArray:
    """the loss of one of "mae", "bce", "bce_with_logits", "kldiv" into a 0-d f32 array (kldiv's mean: by x.shape[0])"""
    out = out or CuArray(x.device, (), F32)
    fwd = _CRITERIA[name][0]
    if name == "kldiv":
        _ck(fwd(x.device.ctx, out.ptr, x.ptr, t.ptr, x.size, x.shape[0] if x.shape else 1, x.dtype, int(mean)), x.device)
    else:
        _ck(fwd(x.device.ctx, out.ptr, x.ptr, t.ptr, x.size, x.dtype, int(mean)), x.device)
    return out


def criterion_bwd(name: str, dx: CuArray, x: CuArray, t: CuArray, g: CuArray, mean=True, beta=1.0) -> CuArray:
    """dx = beta*dx + dloss/dx * g, dx in its own element type"""
    bwd = _CRITERIA[name][1]
    if name == "kldiv":
        _ck(bwd(x.device.ctx, dx.ptr, dx.dtype, t.ptr, g.ptr, x.size, x.shape[0] if x.shape else 1, x.dtype, int(mean),
                float(beta)), x.device)
    else:
        _ck(bwd(x.device.ctx, dx.ptr, dx.dtype, x.ptr, t.ptr, g.ptr, x.size, x.dtype, int(mean), float(beta)), x.device)
    return dx


def dropout(x: CuArray, p: float, mask: CuArray | None = None, out=None) -> CuArray:
    """y = x*keep/(1-p) with a new mask from the device's generator; `mask` (ceil(n/32) 32-bit words, e.g. an f32 array
    of that many elements) receives the keep bits"""
    out = out or CuArray(x.device, x.shape, x.dtype)
    _ck(lib.nk_dropout_fwd(x.device.ctx, out.ptr, mask.ptr if mask is not None else None, x.ptr, x.size, x.dtype,
                           float(p)), x.device)
    return out


def dropout_bwd(dx: CuArray, mask: CuArray | None, g: CuArray, p: float, beta=1.0) -> CuArray:
    _ck(lib.nk_dropout_bwd(g.device.ctx, dx.ptr, dx.dtype, mask.ptr if mask is not None else None, g.ptr, g.size,
                           g.dtype, float(p), float(beta)), g.device)
    return dx


def reduce_sum(x: CuArray, mean=False, out=None) -> CuArray:
    out = out or CuArray(x.device, (), F32)
    _ck(lib.nk_sum_fwd(x.device.ctx, out.ptr, x.ptr, x.size, x.dtype, int(mean)), x.device)
    return out


def reduce_sum_bwd(dx: CuArray, g: CuArray, mean=False, beta=1.0):
    _ck(lib.nk_sum_bwd(dx.device.ctx, dx.ptr, g.ptr, dx.size, dx.dtype, int(mean), float(beta)), dx.device)
    return dx


# ---------------------------------------------------------------- pad / conv
def pad2d(x: CuArray, padding, value=0.0, out=None) -> CuArray:
    ph, pw = padding
    *lead, h, w = x.shape
    out = out or CuArray(x.device, tuple(lead) + (h + 2 * ph, w + 2 * pw), x.dtype)
    planes = int(np.prod(lead)) if lead else 1
    _ck(lib.nk_pad2d_fwd(x.device.ctx, out.ptr, x.ptr, planes, h, w, ph, pw, float(value), x.dtype), x.device)
    return out


def pad2d_bwd(dx: CuArray, g: CuArray, padding, beta=1.0):
    ph, pw = padding
    *lead, h, w = dx.shape
    planes = int(np.prod(lead)) if lead else 1
    _ck(lib.nk_pad2d_bwd(dx.device.ctx, dx.ptr, g.ptr, planes, h, w, ph, pw, dx.dtype, float(beta)), dx.device)
    return dx


def conv_out_shape(xs, ws, stride, dilation):
    """utils.rs:207-237"""
    out = [xs[0], ws[0]]
    for i, k, s, d in zip(xs[2:], ws[2:], stride, dilation):
        out.append((i - d * (k - 1) - 1) // s + 1)
    return tuple(out)


def _conv_args(x_shape, w_shape, stride, dilation, groups):
    n, cin, h, w = x_shape
    cout, _, kh, kw = w_shape
    return [n, cin, h, w, cout, kh, kw, stride[0], stride[1], dilation[0], dilation[1], groups]


def conv2d(x: CuArray, w: CuArray, stride=(1, 1), dilation=(1, 1), groups=1, bias=None, relu=False, out=None):
    dev = x.device
    if x.ndim != 4 or w.ndim != 4:
        raise ValueError(f"Invalid kernel shape {list(w.shape)} for 2d conv")
    out = out or CuArray(dev, conv_out_shape(x.shape, w.shape, stride, dilation), x.dtype)
    _ck(lib.nk_conv2d_fwd(dev.ctx, out.ptr, x.ptr, w.ptr, bias.ptr if bias is not None else None, int(relu),
                          *_conv_args(x.shape, w.shape, stride, dilation, groups), x.dtype), dev)
    return out


def conv2d_bwd_input(dx: CuArray, g: CuArray, w: CuArray, stride=(1, 1), dilation=(1, 1), groups=1, beta=1.0):
    dev = g.device
    _ck(lib.nk_conv2d_bwd_input(dev.ctx, dx.ptr, g.ptr, w.ptr,
                                *_conv_args(dx.shape, w.shape, stride, dilation, groups), g.dtype, float(beta)), dev)
    return dx


def conv2d_bwd_kernel(dw: CuArray, g: CuArray, x: CuArray, stride=(1, 1), dilation=(1, 1), groups=1, beta=1.0,
                      dbias: CuArray | None = None):
    dev = g.device
    _ck(lib.nk_conv2d_bwd_kernel(dev.ctx, dw.ptr, dw.dtype, dbias.ptr if dbias is not None else None, g.ptr, x.ptr,
                                 *_conv_args(x.shape, dw.shape, stride, dilation, groups), g.dtype, float(beta)), dev)
    return dw


# ---------------------------------------------------------------- 8-f: elementwise family
BIN = {"add": L.NK_BIN_ADD, "sub": L.NK_BIN_SUB, "mul": L.NK_BIN_MUL, "div": L.NK_BIN_DIV}
UN = {"neg": L.NK_UN_NEG, "exp": L.NK_UN_EXP, "ln": L.NK_UN_LN, "sqrt": L.NK_UN_SQRT, "sigmoid": L.NK_UN_SIGMOID,
      "tanh": L.NK_UN_TANH, "softplus": L.NK_UN_SOFTPLUS, "leaky_relu": L.NK_UN_LEAKY_RELU, "powi": L.NK_UN_POWI}
PAD = {"constant": L.NK_PAD_CONSTANT, "reflective": L.NK_PAD_REFLECTIVE, "replicative": L.NK_PAD_REPLICATIVE}


def binary(op: str, l: CuArray, r: CuArray, out: CuArray | None = None) -> CuArray:
    dev = l.device
    shape = cobroadcast(l.shape, r.shape)
    out = out or CuArray(dev, shape, l.dtype)
    _ck(lib.nk_binary_bcast_fwd(dev.ctx, BIN[op], out.ptr, l.ptr, r.ptr, l.dtype, len(shape), L.shape_arr(shape),
                                l.ndim, L.shape_arr(l.shape), r.ndim, L.shape_arr(r.shape)), dev)
    return out


def binary_bwd(op: str, side: int, dst: CuArray, g: CuArray, l: CuArray, r: CuArray, beta=1.0) -> CuArray:
    """dst (the gradient of operand `side`) = beta*dst + unbroadcast(factor(g, l, r))."""
    dev = g.device
    _ck(lib.nk_binary_bcast_bwd(dev.ctx, BIN[op], int(side), dst.ptr, dst.dtype, g.ptr, l.ptr, r.ptr, g.dtype,
                                l.ndim, L.shape_arr(l.shape), r.ndim, L.shape_arr(r.shape), float(beta)), dev)
    return dst


def unary(op: str, x: CuArray, iparam: int = 0, out: CuArray | None = None) -> CuArray:
    out = out or CuArray(x.device, x.shape, x.dtype)
    _ck(lib.nk_unary_fwd(x.device.ctx, UN[op], out.ptr, x.ptr, x.size, x.dtype, int(iparam)), x.device)
    return out


def unary_bwd(op: str, dx: CuArray, saved: CuArray | None, g: CuArray, iparam: int = 0, beta=1.0) -> CuArray:
    _ck(lib.nk_unary_bwd(g.device.ctx, UN[op], dx.ptr, saved.ptr if saved is not None else None, g.ptr, g.size,
                         g.dtype, int(iparam), float(beta)), g.device)
    return dx


def transpose(src: CuArray, out: CuArray | None = None, beta=0.0) -> CuArray:
    out = out or CuArray(src.device, tuple(reversed(src.shape)), src.dtype)
    _ck(lib.nk_transpose(src.device.ctx, out.ptr, out.dtype, src.ptr, src.dtype, src.ndim, L.shape_arr(src.shape),
                         float(beta)), src.device)
    return out


def pad_nd(x: CuArray, padding, mode="constant", value=0.0, out=None) -> CuArray:
    nsp = len(padding)
    lead, sp = x.shape[:x.ndim - nsp], x.shape[x.ndim - nsp:]
    out = out or CuArray(x.device, tuple(lead) + tuple(s + 2 * p for s, p in zip(sp, padding)), x.dtype)
    planes = int(np.prod(lead)) if lead else 1
    _ck(lib.nk_padnd_fwd(x.device.ctx, out.ptr, x.ptr, planes, nsp, L.shape_arr(sp), L.shape_arr(padding), PAD[mode],
                         float(value), x.dtype), x.device)
    return out


def pad_nd_bwd(dx: CuArray, g: CuArray, padding, beta=1.0) -> CuArray:
    nsp = len(padding)
    lead, sp = dx.shape[:dx.ndim - nsp], dx.shape[dx.ndim - nsp:]
    planes = int(np.prod(lead)) if lead else 1
    _ck(lib.nk_padnd_bwd(dx.device.ctx, dx.ptr, g.ptr, planes, nsp, L.shape_arr(sp), L.shape_arr(padding), dx.dtype,
                         float(beta)), dx.device)
    return dx


# ---------------------------------------------------------------- pooling over 1..3 sample dims (csrc/nk_pool.cu)
def pool_out_extent(length, k, stride, pad, dilation=1, ceil_mode=False) -> int:
    """torch's pooling output extent along one axis (the value nk_*_pool_nd_* check out_sp against)."""
    if stride < 1:
        return 0                            # nk_*_pool_nd_* reject the stride
    num = length + 2 * pad - dilation * (k - 1) - 1
    o = (num + (stride - 1 if ceil_mode else 0)) // stride + 1
    if ceil_mode and (o - 1) * stride >= length + pad:
        o -= 1
    return o


def _pool_geom(x_shape, out_sp, *per_axis):
    nsp = len(out_sp)
    planes = int(np.prod(x_shape[:len(x_shape) - nsp]))
    return [planes, nsp, L.shape_arr(x_shape[len(x_shape) - nsp:]), L.shape_arr(out_sp)] + [L.shape_arr(a) for a in per_axis]


def _pool_out(x: CuArray, k, stride, padding, dilation, ceil_mode):
    sp = x.shape[x.ndim - len(k):]
    return tuple(pool_out_extent(*a, ceil_mode) for a in zip(sp, k, stride, padding, dilation))


def max_pool_nd(x: CuArray, k, stride=None, padding=None, dilation=None, ceil_mode=False, out=None,
                idx: CuArray | None = None, out_sp=None) -> CuArray:
    """y = max pool of the last len(k) dims of x (nk_max_pool_nd_fwd); idx (int32 as F32-sized elements, y's shape) gets
    the winners' in-plane flat indices when given."""
    nsp = len(k)
    stride, padding, dilation = stride or k, padding or (0,) * nsp, dilation or (1,) * nsp
    out_sp = out_sp or _pool_out(x, k, stride, padding, dilation, ceil_mode)
    out = out or CuArray(x.device, x.shape[:x.ndim - nsp] + tuple(out_sp), x.dtype)
    _ck(lib.nk_max_pool_nd_fwd(x.device.ctx, out.ptr, _ptr(idx), x.ptr,
                               *_pool_geom(x.shape, out_sp, k, stride, padding, dilation), x.dtype), x.device)
    return out


def max_pool_nd_bwd(dx: CuArray, g: CuArray, idx: CuArray, k, stride=None, padding=None, dilation=None,
                    beta=1.0) -> CuArray:
    """dx = beta*dx + the gradient gathered through the saved indices (nk_max_pool_nd_bwd)."""
    nsp = len(k)
    stride, padding, dilation = stride or k, padding or (0,) * nsp, dilation or (1,) * nsp
    _ck(lib.nk_max_pool_nd_bwd(dx.device.ctx, dx.ptr, dx.dtype, g.ptr, g.dtype, idx.ptr,
                               *_pool_geom(dx.shape, g.shape[g.ndim - nsp:], k, stride, padding, dilation),
                               float(beta)), dx.device)
    return dx


def avg_pool_nd(x: CuArray, k, stride=None, padding=None, ceil_mode=False, count_include_pad=True, out=None,
                out_sp=None) -> CuArray:
    """y = average pool of the last len(k) dims of x (nk_avg_pool_nd_fwd)."""
    nsp = len(k)
    stride, padding = stride or k, padding or (0,) * nsp
    out_sp = out_sp or _pool_out(x, k, stride, padding, (1,) * nsp, ceil_mode)
    out = out or CuArray(x.device, x.shape[:x.ndim - nsp] + tuple(out_sp), x.dtype)
    _ck(lib.nk_avg_pool_nd_fwd(x.device.ctx, out.ptr, x.ptr, *_pool_geom(x.shape, out_sp, k, stride, padding),
                               int(bool(count_include_pad)), x.dtype), x.device)
    return out


def avg_pool_nd_bwd(dx: CuArray, g: CuArray, k, stride=None, padding=None, count_include_pad=True,
                    beta=1.0) -> CuArray:
    """dx = beta*dx + the average pool's input gradient (nk_avg_pool_nd_bwd)."""
    nsp = len(k)
    stride, padding = stride or k, padding or (0,) * nsp
    _ck(lib.nk_avg_pool_nd_bwd(dx.device.ctx, dx.ptr, dx.dtype, g.ptr, g.dtype,
                               *_pool_geom(dx.shape, g.shape[g.ndim - nsp:], k, stride, padding),
                               int(bool(count_include_pad)), float(beta)), dx.device)
    return dx


def adaptive_avg_pool_nd(x: CuArray, output_size, out=None) -> CuArray:
    """y = adaptive average pool of the last len(output_size) dims of x to output_size (nk_adaptive_avg_pool_nd_fwd)."""
    nsp = len(output_size)
    out = out or CuArray(x.device, x.shape[:x.ndim - nsp] + tuple(output_size), x.dtype)
    _ck(lib.nk_adaptive_avg_pool_nd_fwd(x.device.ctx, out.ptr, x.ptr, *_pool_geom(x.shape, output_size), x.dtype),
        x.device)
    return out


def adaptive_avg_pool_nd_bwd(dx: CuArray, g: CuArray, beta=1.0, nsp=None) -> CuArray:
    """dx = beta*dx + the adaptive average pool's input gradient (nk_adaptive_avg_pool_nd_bwd); nsp defaults to
    dx.ndim - 2."""
    nsp = nsp or dx.ndim - 2
    _ck(lib.nk_adaptive_avg_pool_nd_bwd(dx.device.ctx, dx.ptr, dx.dtype, g.ptr, g.dtype,
                                        *_pool_geom(dx.shape, g.shape[g.ndim - nsp:]), float(beta)), dx.device)
    return dx


# ---------------------------------------------------------------- batch norm / layer norm (csrc/nk_norm.cu)
def _bn_dims(shape):
    return int(shape[0]), int(shape[1]), int(np.prod(shape[2:], dtype=np.int64))


def batch_norm(x: CuArray, weight: CuArray | None = None, bias: CuArray | None = None,
               running_mean: CuArray | None = None, running_var: CuArray | None = None, training=True, momentum=0.1,
               eps=1e-5, out=None, save_mean: CuArray | None = None, save_rstd: CuArray | None = None):
    """y = batch norm of x (N, C, ...) over N and the sample dims (nk_batch_norm_fwd).  Returns (y, save_mean,
    save_rstd), the f32 (C,) statistics the backward takes; running_mean / running_var (f32) are updated in place when
    training."""
    n, c, s = _bn_dims(x.shape)
    out = out or CuArray(x.device, x.shape, x.dtype)
    save_mean = save_mean or CuArray(x.device, (c,), F32)
    save_rstd = save_rstd or CuArray(x.device, (c,), F32)
    _ck(lib.nk_batch_norm_fwd(x.device.ctx, out.ptr, x.ptr, x.dtype, n, c, s, _ptr(weight), _ptr(bias),
                              _ptr(running_mean), _ptr(running_var), save_mean.ptr, save_rstd.ptr, int(bool(training)),
                              float(momentum), float(eps)), x.device)
    return out, save_mean, save_rstd


def _grads(*pairs):
    """(ptr, dtype, beta) for each (array or None, beta)"""
    out = []
    for a, beta in pairs:
        out += [_ptr(a), a.dtype if a is not None else F32, float(beta)]
    return out


def batch_norm_bwd(g: CuArray, x: CuArray, save_mean: CuArray, save_rstd: CuArray, weight: CuArray | None = None,
                   dx: CuArray | None = None, dw: CuArray | None = None, db: CuArray | None = None, batch_stats=True,
                   beta=0.0, dw_beta=None, db_beta=None):
    """dx / dw / db = beta*d + the batch norm's gradients (nk_batch_norm_bwd); any of them may be None."""
    n, c, s = _bn_dims(x.shape)
    betas = (beta, beta if dw_beta is None else dw_beta, beta if db_beta is None else db_beta)
    _ck(lib.nk_batch_norm_bwd(x.device.ctx, *_grads((dx, betas[0]), (dw, betas[1]), (db, betas[2])), g.ptr, g.dtype,
                              x.ptr, x.dtype, n, c, s, _ptr(weight), save_mean.ptr, save_rstd.ptr,
                              int(bool(batch_stats))), x.device)
    return dx, dw, db


def layer_norm(x: CuArray, cols: int, weight: CuArray | None = None, bias: CuArray | None = None, eps=1e-5, out=None,
               save_mean: CuArray | None = None, save_rstd: CuArray | None = None):
    """y = layer norm of x's rows of `cols` elements (nk_layer_norm_fwd).  Returns (y, save_mean, save_rstd), the f32
    (rows,) statistics the backward takes."""
    rows = int(np.prod(x.shape, dtype=np.int64)) // cols
    out = out or CuArray(x.device, x.shape, x.dtype)
    save_mean = save_mean or CuArray(x.device, (rows,), F32)
    save_rstd = save_rstd or CuArray(x.device, (rows,), F32)
    _ck(lib.nk_layer_norm_fwd(x.device.ctx, out.ptr, x.ptr, x.dtype, rows, cols, _ptr(weight), _ptr(bias),
                              save_mean.ptr, save_rstd.ptr, float(eps)), x.device)
    return out, save_mean, save_rstd


def layer_norm_bwd(g: CuArray, x: CuArray, cols: int, save_mean: CuArray, save_rstd: CuArray,
                   weight: CuArray | None = None, dx: CuArray | None = None, dw: CuArray | None = None,
                   db: CuArray | None = None, beta=0.0, dw_beta=None, db_beta=None):
    """dx / dw / db = beta*d + the layer norm's gradients (nk_layer_norm_bwd); any of them may be None."""
    rows = int(np.prod(x.shape, dtype=np.int64)) // cols
    betas = (beta, beta if dw_beta is None else dw_beta, beta if db_beta is None else db_beta)
    _ck(lib.nk_layer_norm_bwd(x.device.ctx, *_grads((dx, betas[0]), (dw, betas[1]), (db, betas[2])), g.ptr, g.dtype,
                              x.ptr, x.dtype, rows, cols, _ptr(weight), save_mean.ptr, save_rstd.ptr), x.device)
    return dx, dw, db


def embedding(w: CuArray, ids: CuArray, out=None) -> CuArray:
    """y = w[ids] (nk_embedding_fwd): w (v, e); ids of any shape, f32 (or bf16 for v <= 256) ids; y ids.shape + (e,).
    Invalid ids give zero rows."""
    v, e = w.shape
    out = out or CuArray(w.device, tuple(ids.shape) + (e,), w.dtype)
    _ck(lib.nk_embedding_fwd(w.device.ctx, out.ptr, w.ptr, ids.ptr, ids.dtype, ids.size, v, e, w.dtype), w.device)
    return out


def embedding_bwd(dw: CuArray, ids: CuArray, g: CuArray, padding_idx=None, beta=1.0) -> CuArray:
    """dw = beta*dw + the embedding's weight gradient (nk_embedding_bwd); padding_idx None = -1 (none)."""
    v, e = dw.shape
    _ck(lib.nk_embedding_bwd(dw.device.ctx, dw.ptr, dw.dtype, ids.ptr, ids.dtype, g.ptr, g.dtype, ids.size, v, e,
                             -1 if padding_idx is None else int(padding_idx), float(beta)), dw.device)
    return dw


# ---------------------------------------------------------------- 8-f: mv / vm / vv
def gemv(a: CuArray, x: CuArray, y: CuArray | None = None, trans=False, beta=0.0) -> CuArray:
    rows, cols = a.shape
    y = y or CuArray(a.device, (cols if trans else rows,), a.dtype)
    _ck(lib.nk_gemv(a.device.ctx, int(trans), rows, cols, a.ptr, x.ptr, float(beta), y.ptr, a.dtype, y.dtype), a.device)
    return y


def outer_acc(a: CuArray, u: CuArray, v: CuArray, beta=1.0) -> CuArray:
    rows, cols = a.shape
    _ck(lib.nk_outer_acc(a.device.ctx, a.ptr, a.dtype, u.ptr, v.ptr, rows, cols, u.dtype, float(beta)), a.device)
    return a


def dot(a: CuArray, b: CuArray, out: CuArray | None = None) -> CuArray:
    out = out or CuArray(a.device, (), F32)
    _ck(lib.nk_dot(a.device.ctx, out.ptr, a.ptr, b.ptr, a.size, a.dtype), a.device)
    return out


def scale_acc(dst: CuArray, x: CuArray, scalar: CuArray, beta=1.0) -> CuArray:
    _ck(lib.nk_scale_acc(dst.device.ctx, dst.ptr, dst.dtype, x.ptr, x.dtype, scalar.ptr, x.size, float(beta)), dst.device)
    return dst


# ---------------------------------------------------------------- 8-f: 1-d / 3-d convolution
def _convnd_args(x_shape, w_shape, stride, dilation, groups):
    nsp = len(x_shape) - 2
    return [nsp, x_shape[0], x_shape[1], L.shape_arr(x_shape[2:]), w_shape[0], L.shape_arr(w_shape[2:]),
            L.shape_arr(stride), L.shape_arr(dilation), groups]


def convnd(x: CuArray, w: CuArray, stride, dilation, groups=1, out=None) -> CuArray:
    out = out or CuArray(x.device, conv_out_shape(x.shape, w.shape, stride, dilation), x.dtype)
    _ck(lib.nk_convnd_fwd(x.device.ctx, out.ptr, x.ptr, w.ptr, *_convnd_args(x.shape, w.shape, stride, dilation, groups),
                          x.dtype), x.device)
    return out


def convnd_bwd_input(dx: CuArray, g: CuArray, w: CuArray, stride, dilation, groups=1, beta=1.0) -> CuArray:
    _ck(lib.nk_convnd_bwd_input(g.device.ctx, dx.ptr, g.ptr, w.ptr,
                                *_convnd_args(dx.shape, w.shape, stride, dilation, groups), g.dtype, float(beta)), g.device)
    return dx


def convnd_bwd_kernel(dw: CuArray, g: CuArray, x: CuArray, stride, dilation, groups=1, beta=1.0) -> CuArray:
    _ck(lib.nk_convnd_bwd_kernel(g.device.ctx, dw.ptr, dw.dtype, g.ptr, x.ptr,
                                 *_convnd_args(x.shape, dw.shape, stride, dilation, groups), g.dtype, float(beta)), g.device)
    return dw


def _layer_args(x_shape, w_shape, stride, dilation, padding, mode):
    nsp = len(x_shape) - 2
    stride, dilation = stride or (1,) * nsp, dilation or (1,) * nsp
    return [nsp, x_shape[0], x_shape[1], L.shape_arr(x_shape[2:]), w_shape[0], L.shape_arr(w_shape[2:]),
            L.shape_arr(stride), L.shape_arr(dilation), L.shape_arr(padding), PAD[mode]]


def conv_layer_nd(x: CuArray, w: CuArray, padding, mode="constant", value=0.0, stride=None, dilation=None, bias=None,
                  out=None) -> CuArray:
    """y = conv(pad(x, padding, mode), w) + bias for 1-D / 3-D x (nk_conv_layer_nd_fwd); bias (Cout) or None."""
    stride, dilation = stride or (1,) * len(padding), dilation or (1,) * len(padding)
    padded = x.shape[:2] + tuple(s + 2 * p for s, p in zip(x.shape[2:], padding))
    out = out or CuArray(x.device, conv_out_shape(padded, w.shape, stride, dilation), x.dtype)
    _ck(lib.nk_conv_layer_nd_fwd(x.device.ctx, out.ptr, x.ptr, w.ptr, _ptr(bias),
                                 *_layer_args(x.shape, w.shape, stride, dilation, padding, mode), float(value), x.dtype),
        x.device)
    return out


def conv_layer_nd_bwd_input(dx: CuArray, g: CuArray, w: CuArray, padding, mode="constant", stride=None, dilation=None,
                            beta=1.0) -> CuArray:
    """dx = beta*dx + the interior slice of the padded input's gradient (nk_conv_layer_nd_bwd_input)."""
    _ck(lib.nk_conv_layer_nd_bwd_input(g.device.ctx, dx.ptr, g.ptr, w.ptr,
                                       *_layer_args(dx.shape, w.shape, stride, dilation, padding, mode), g.dtype,
                                       float(beta)), g.device)
    return dx


def conv_layer_nd_bwd_kernel(dw: CuArray, g: CuArray, x: CuArray, padding, mode="constant", value=0.0, stride=None,
                             dilation=None, beta=1.0, dbias: CuArray | None = None) -> CuArray:
    """dw = beta*dw + dW of the layer, and dbias likewise when given (nk_conv_layer_nd_bwd_kernel)."""
    _ck(lib.nk_conv_layer_nd_bwd_kernel(g.device.ctx, dw.ptr, dw.dtype, _ptr(dbias), g.ptr, x.ptr,
                                        *_layer_args(x.shape, dw.shape, stride, dilation, padding, mode), float(value),
                                        g.dtype, float(beta)), g.device)
    return dw


# ---------------------------------------------------------------- 8-f: recurrent cells and chunks (csrc/nk_rnn.cu)
def _ptr(a: CuArray | None):
    return a.ptr if a is not None else None


def lstm_cell(gates: CuArray, c_prev: CuArray, c_out: CuArray | None = None, h_out: CuArray | None = None):
    """c' = sigmoid(f)*c + sigmoid(i)*tanh(g), h' = sigmoid(o)*tanh(c') from the f32 (n, 4H) pre-activations
    [i | f | g | o].  Returns (c_out, h_out)."""
    n, hidden = c_prev.shape
    if gates.dtype != F32 or tuple(gates.shape) != (n, 4 * hidden):
        raise ValueError(f"lstm_cell: gates must be f32 ({n}, {4 * hidden}), got {gates}")
    c_out = c_out or CuArray(c_prev.device, (n, hidden), c_prev.dtype)
    h_out = h_out or CuArray(c_prev.device, (n, hidden), c_prev.dtype)
    _ck(lib.nk_lstm_cell_fwd(c_prev.device.ctx, c_out.ptr, h_out.ptr, gates.ptr, c_prev.ptr, n, hidden, c_prev.dtype),
        c_prev.device)
    return c_out, h_out


def lstm_cell_bwd(dgates: CuArray, gates: CuArray, c_prev: CuArray, dh_out: CuArray | None, dc_out: CuArray | None,
                  dc_prev: CuArray | None = None, beta_dc=1.0) -> CuArray:
    """dgates (overwritten, its own element type) and dc_prev = beta_dc*dc_prev + sigmoid(f)*dc_total.  dh_out / dc_out
    None = a zero gradient; dc_prev None = the cell state is not differentiable."""
    n, hidden = c_prev.shape
    _ck(lib.nk_lstm_cell_bwd(c_prev.device.ctx, dgates.ptr, dgates.dtype, _ptr(dc_prev), float(beta_dc), gates.ptr,
                             c_prev.ptr, _ptr(dh_out), _ptr(dc_out), n, hidden, c_prev.dtype), c_prev.device)
    return dgates


def gru_cell(igates: CuArray, hgates: CuArray, h_prev: CuArray, h_out: CuArray | None = None) -> CuArray:
    """h' = (h - nn)*z + nn from the f32 (n, 3H) pre-activations [r | z | n] of the input and of the hidden state."""
    n, hidden = h_prev.shape
    for g in (igates, hgates):
        if g.dtype != F32 or tuple(g.shape) != (n, 3 * hidden):
            raise ValueError(f"gru_cell: gates must be f32 ({n}, {3 * hidden}), got {g}")
    h_out = h_out or CuArray(h_prev.device, (n, hidden), h_prev.dtype)
    _ck(lib.nk_gru_cell_fwd(h_prev.device.ctx, h_out.ptr, igates.ptr, hgates.ptr, h_prev.ptr, n, hidden, h_prev.dtype),
        h_prev.device)
    return h_out


def gru_cell_bwd(digates: CuArray, dhgates: CuArray, igates: CuArray, hgates: CuArray, h_prev: CuArray, dh_out: CuArray,
                 dh_prev: CuArray | None = None, beta_dh=1.0):
    """digates, dhgates (overwritten) and the pointwise part of the hidden-state gradient dh_prev = beta_dh*dh_prev +
    z*dh_out.  Returns (digates, dhgates)."""
    n, hidden = h_prev.shape
    if digates.dtype != dhgates.dtype:
        raise ValueError("gru_cell_bwd: digates and dhgates must have one element type")
    _ck(lib.nk_gru_cell_bwd(h_prev.device.ctx, digates.ptr, dhgates.ptr, digates.dtype, _ptr(dh_prev), float(beta_dh),
                            igates.ptr, hgates.ptr, h_prev.ptr, dh_out.ptr, n, hidden, h_prev.dtype), h_prev.device)
    return digates, dhgates


def lstm_seq_bwd_step(dgates: CuArray, dc: CuArray, gates: CuArray, c_prev: CuArray, dh_out: CuArray | None,
                      dh_rec: CuArray | None) -> CuArray:
    """One backward time step of the LSTM sequence node: dgates (overwritten) from dh = dh_out + dh_rec (None = zero;
    dh_rec f32) and the running f32 cell-state gradient dc, which is replaced by sigmoid(f)*dc_total."""
    n, hidden = c_prev.shape
    if dc.dtype != F32 or (dh_rec is not None and dh_rec.dtype != F32):
        raise ValueError("lstm_seq_bwd_step: dc and dh_rec are f32")
    _ck(lib.nk_lstm_seq_bwd_step(c_prev.device.ctx, dgates.ptr, dgates.dtype, dc.ptr, gates.ptr, c_prev.ptr, _ptr(dh_out),
                                 _ptr(dh_rec), n, hidden, c_prev.dtype), c_prev.device)
    return dgates


def gru_seq_bwd_step(digates: CuArray, dhgates: CuArray, dh_rec: CuArray | None, igates: CuArray, hgates: CuArray,
                     h_prev: CuArray, dh_out: CuArray | None):
    """One backward time step of the GRU sequence node: digates, dhgates (overwritten) from dh = dh_out + dh_rec (None =
    zero); the f32 dh_rec is replaced by z*dh.  Returns (digates, dhgates)."""
    n, hidden = h_prev.shape
    if digates.dtype != dhgates.dtype:
        raise ValueError("gru_seq_bwd_step: digates and dhgates must have one element type")
    if dh_rec is not None and dh_rec.dtype != F32:
        raise ValueError("gru_seq_bwd_step: dh_rec is f32")
    _ck(lib.nk_gru_seq_bwd_step(h_prev.device.ctx, digates.ptr, dhgates.ptr, digates.dtype, _ptr(dh_rec), igates.ptr,
                                hgates.ptr, h_prev.ptr, _ptr(dh_out), n, hidden, h_prev.dtype), h_prev.device)
    return digates, dhgates


def chunk(x: CuArray, chunk_shape, index: int, out: CuArray | None = None) -> CuArray:
    """Block `index` of x's exact_chunks(chunk_shape) (row-major block order), bit exact."""
    cs = tuple(int(c) for c in chunk_shape)
    out = out or CuArray(x.device, cs, x.dtype)
    _ck(lib.nk_chunk_fwd(x.device.ctx, out.ptr, x.ptr, x.ndim, L.shape_arr(x.shape), L.shape_arr(cs), int(index),
                         x.dtype), x.device)
    return out


def chunk_bwd(dx: CuArray, g: CuArray, index: int, beta=1.0) -> CuArray:
    """dx[block index] = beta*dx[block] + g; the rest of dx is untouched."""
    _ck(lib.nk_chunk_bwd(dx.device.ctx, dx.ptr, dx.dtype, g.ptr, g.dtype, dx.ndim, L.shape_arr(dx.shape),
                         L.shape_arr(g.shape), int(index), float(beta)), dx.device)
    return dx


# ---------------------------------------------------------------- concatenation (csrc/nk_cat.cu)
def _cat_view(shape, axis):
    if not 0 <= axis < len(shape):
        raise ValueError(f"cat: axis {axis} out of range for shape {tuple(shape)}")
    return _lanes(shape, axis)


def cat(xs, axis: int, out: CuArray | None = None) -> CuArray:
    """The arrays side by side along `axis` (equal shapes on every other axis), bit exact; one launch per
    NK_CAT_OPS_PER_LAUNCH operands."""
    xs = list(xs)
    shape = list(xs[0].shape)
    outer, _, inner = _cat_view(shape, axis)
    lens = [int(x.shape[axis]) for x in xs]
    shape[axis] = sum(lens)
    out = out or CuArray(xs[0].device, tuple(shape), xs[0].dtype)
    ptrs = (L.vp * len(xs))(*[x.ptr.value for x in xs])
    _ck(lib.nk_cat_fwd(out.device.ctx, out.ptr, ptrs, (L.i64 * len(xs))(*lens), len(xs), outer, inner, out.dtype),
        out.device)
    return out


def cat_bwd(dxs, g: CuArray, axis: int, betas, lens=None):
    """dxs[i] = betas[i]*dxs[i] + (slice i of g along `axis`), each in its own element type; a None entry gets nothing
    (then `lens` gives every operand's length along `axis`)."""
    dxs = list(dxs)
    outer, _, inner = _cat_view(g.shape, axis)
    lens = [int(d.shape[axis]) for d in dxs] if lens is None else [int(v) for v in lens]
    n = len(dxs)
    ptrs = (L.vp * n)(*[_ptr(d).value if d is not None else None for d in dxs])
    dts = (L.i32 * n)(*[d.dtype if d is not None else F32 for d in dxs])
    _ck(lib.nk_cat_bwd(g.device.ctx, ptrs, dts, (L.f32 * n)(*[float(b) for b in betas]), g.ptr, g.dtype,
                       (L.i64 * n)(*lens), n, outer, inner), g.device)
    return dxs


# ---------------------------------------------------------------- gradient clipping (csrc/nk_optim_multi.cu)
def _grad_tables(grads):
    n = len(grads)
    return ((L.vp * n)(*[g.ptr.value for g in grads]), (L.i32 * n)(*[g.dtype for g in grads]),
            (L.i64 * n)(*[g.size for g in grads]))


def grad_norm(grads, norm_type=2.0, grad_scale=1.0, out: CuArray | None = None) -> CuArray:
    """out = the norm_type-norm of grad_scale * (every element of every array), one f32 on the device (0 for no arrays;
    then `out` gives the device)."""
    grads = list(grads)
    dev = out.device if out is not None else grads[0].device
    out = out if out is not None else CuArray(dev, (), F32)
    _ck(lib.nk_grad_norm(dev.ctx, len(grads), *_grad_tables(grads), float(norm_type), float(grad_scale), out.ptr), dev)
    return out


def grad_scale_by_norm(grads, total: CuArray, max_norm: float):
    """every array *= min(max_norm / (total + 1e-6), 1), torch's clip coefficient from the device scalar `total`"""
    grads = list(grads)
    _ck(lib.nk_grad_scale_by_norm(total.device.ctx, len(grads), *_grad_tables(grads), total.ptr, float(max_norm)),
        total.device)
    return grads


def grad_clamp(grads, clip_value: float, grad_scale=1.0):
    """every array = clamp(array, -b, b), b = clip_value / grad_scale in f32"""
    grads = list(grads)
    if not grads:
        return grads
    dev = grads[0].device
    _ck(lib.nk_grad_clamp(dev.ctx, len(grads), *_grad_tables(grads), float(clip_value), float(grad_scale)), dev)
    return grads
