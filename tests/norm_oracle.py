"""Batch norm and layer norm restated in numpy with torch's semantics (include/nk_b200.h nk_batch_norm_* /
nk_layer_norm_*).  Everything runs in float64 on the (possibly bf16-rounded) inputs: the float64 shadow that the
kernels' f32 / bf16 results are bounded against.  tests/test_oracle_norm.py pins this module to torch."""
from __future__ import annotations

import numpy as np


def _size(shape):
    return "torch.Size([%s])" % ", ".join(str(d) for d in shape)


def bn_forward(x, w=None, b=None, rm=None, rv=None, training=True, momentum=0.1, eps=1e-5):
    """-> (y, mean, rstd, rm', rv', batch): y and the statistics the forward normalized with (the batch's when
    `batch`, else the running ones), and the running statistics after the forward (None when not tracked)."""
    x = np.asarray(x, np.float64)
    n, c = x.shape[:2]
    xs = x.reshape(n, c, int(np.prod(x.shape[2:], dtype=np.int64)))
    m = n * xs.shape[2]
    batch = training or rm is None
    if batch and m == 1:
        raise ValueError("Expected more than 1 value per channel when training, got input size " + _size(x.shape))
    rm = None if rm is None else np.asarray(rm, np.float64).copy()
    rv = None if rv is None else np.asarray(rv, np.float64).copy()
    if m == 0 or n == 0:
        return x.copy(), np.zeros(c), np.ones(c), rm, rv, batch
    if batch:
        mean = xs.mean(axis=(0, 2))
        var = ((xs - mean[None, :, None]) ** 2).mean(axis=(0, 2))
        if training and rm is not None:
            rm = (1 - momentum) * rm + momentum * mean
            rv = (1 - momentum) * rv + momentum * var * m / (m - 1)
    else:
        mean, var = rm, rv
    rstd = 1.0 / np.sqrt(var + eps)
    wv = np.ones(c) if w is None else np.asarray(w, np.float64)
    bv = np.zeros(c) if b is None else np.asarray(b, np.float64)
    y = (xs - mean[None, :, None]) * (rstd * wv)[None, :, None] + bv[None, :, None]
    return y.reshape(x.shape), mean, rstd, rm, rv, batch


def bn_backward(g, x, mean, rstd, w=None, batch=True):
    """-> (dx, dw, db) of the batch norm that normalized x with (mean, rstd)"""
    x = np.asarray(x, np.float64)
    n, c = x.shape[:2]
    s = int(np.prod(x.shape[2:], dtype=np.int64))
    xs, gs = x.reshape(n, c, s), np.asarray(g, np.float64).reshape(n, c, s)
    m = n * xs.shape[2]
    xhat = (xs - mean[None, :, None]) * rstd[None, :, None]
    sg, sgx = gs.sum(axis=(0, 2)), (gs * xhat).sum(axis=(0, 2))
    k = rstd * (np.ones(c) if w is None else np.asarray(w, np.float64))
    if batch and m > 0:
        dx = k[None, :, None] * (gs - (sg / m)[None, :, None] - xhat * (sgx / m)[None, :, None])
    else:
        dx = k[None, :, None] * gs
    return dx.reshape(x.shape), sgx, sg


def ln_check(shape, normalized_shape):
    ns = tuple(normalized_shape)
    if not ns or len(ns) > len(shape) or tuple(shape[len(shape) - len(ns):]) != ns:
        raise ValueError("Given normalized_shape=%s, expected input with shape [*, %s], but got input of size%s"
                         % (list(ns), ", ".join(str(d) for d in ns), list(shape)))


def ln_forward(x, normalized_shape, w=None, b=None, eps=1e-5):
    """-> (y, mean, rstd): mean and rstd per row (the leading dims flattened)"""
    x = np.asarray(x, np.float64)
    ln_check(x.shape, normalized_shape)
    d = int(np.prod(normalized_shape))
    xr = x.reshape(x.size // d, d)
    mean = xr.mean(axis=1)
    rstd = 1.0 / np.sqrt(((xr - mean[:, None]) ** 2).mean(axis=1) + eps)
    y = (xr - mean[:, None]) * rstd[:, None]
    if w is not None:
        y = y * np.asarray(w, np.float64).reshape(1, d)
    if b is not None:
        y = y + np.asarray(b, np.float64).reshape(1, d)
    return y.reshape(x.shape), mean, rstd


def ln_backward(g, x, normalized_shape, mean, rstd, w=None):
    """-> (dx, dw, db); dw / db have normalized_shape"""
    x = np.asarray(x, np.float64)
    d = int(np.prod(normalized_shape))
    xr, gr = x.reshape(x.size // d, d), np.asarray(g, np.float64).reshape(x.size // d, d)
    xhat = (xr - mean[:, None]) * rstd[:, None]
    gw = gr * (1.0 if w is None else np.asarray(w, np.float64).reshape(1, d))
    dx = rstd[:, None] * (gw - gw.mean(axis=1, keepdims=True) - xhat * (gw * xhat).mean(axis=1, keepdims=True))
    ns = tuple(normalized_shape)
    return dx.reshape(x.shape), (gr * xhat).sum(axis=0).reshape(ns), gr.sum(axis=0).reshape(ns)


def bf16_round(a):
    """round float32 values to bfloat16 (nearest even), returned as float32"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).reshape(np.shape(a))
