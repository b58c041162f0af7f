"""Pins the pooling oracle (tests/pool_oracle.py) to torch's CPU max / avg / adaptive average pooling and their autograd:
max values and indices bit-equal, averages within (R + 1) * 2^-24 * sum|x| of float64 (R: the window's element count)
and exact on small-integer inputs, over overlapping and gapped strides, padding k/2, dilation, ceil_mode windows that are
clipped or dropped, count_include_pad, adaptive sizes that do not divide the input or exceed it, ties, infinities and
NaN."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pool_oracle as P

MAX = {1: F.max_pool1d, 2: F.max_pool2d, 3: F.max_pool3d}
AVG = {1: F.avg_pool1d, 2: F.avg_pool2d, 3: F.avg_pool3d}
ADAPTIVE = {1: F.adaptive_avg_pool1d, 2: F.adaptive_avg_pool2d, 3: F.adaptive_avg_pool3d}

# (input sample shape, kernel, stride, padding, dilation, ceil_mode)
MAX_CASES = [
    ((11,), (3,), (2,), (1,), (1,), False),               # overlap, p = k/2
    ((13,), (2,), (3,), (0,), (1,), False),               # gaps
    ((12,), (3,), (2,), (1,), (2,), True),                # dilation, ceil_mode
    ((9, 10), (3, 3), (2, 2), (1, 1), (1, 1), True),      # ceil_mode clips the last window
    ((8, 7), (2, 3), (1, 2), (1, 0), (1, 1), False),
    ((7, 9), (3, 2), (2, 2), (1, 1), (2, 1), True),
    ((5,), (2,), (2,), (1,), (1,), True),                 # ceil_mode drops the window that would start in the padding
    ((4, 6, 5), (2, 2, 2), (2, 2, 2), (0, 0, 0), (1, 1, 1), True),
    ((5, 6, 7), (3, 2, 3), (1, 2, 2), (1, 1, 0), (1, 2, 1), False),
    ((16, 16), (8, 5), (4, 3), (4, 2), (1, 1), False),    # a large window (40 elements)
]
AVG_CASES = [
    ((11,), (3,), (2,), (1,), False),
    ((13,), (2,), (3,), (0,), False),
    ((5,), (2,), (2,), (1,), True),
    ((9, 10), (3, 3), (2, 2), (1, 1), True),
    ((8, 7), (2, 3), (1, 2), (1, 0), False),
    ((4, 6, 5), (2, 2, 2), (2, 2, 2), (0, 0, 0), True),
    ((6, 7, 8), (3, 3, 3), (2, 2, 3), (1, 1, 1), True),   # 27 elements
    ((16, 16), (8, 5), (4, 3), (4, 2), True),             # 40 elements: the warp order
    ((12, 12, 12), (4, 4, 4), (4, 4, 4), (2, 0, 1), False),
]
ADAPTIVE_CASES = [((10,), (3,)), ((5,), (8,)), ((7, 9), (3, 4)), ((7, 7), (1, 1)), ((32, 32), (1, 1)),
                  ((4, 5, 6), (3, 2, 4)), ((6, 5, 4), (1, 1, 1)), ((3, 2), (5, 7))]


def _data(rng, shape, kind):
    if kind == "int":
        return rng.integers(-8, 9, shape).astype(np.float32)
    if kind == "ties":
        return rng.integers(0, 3, shape).astype(np.float32)
    x = rng.standard_normal(shape).astype(np.float32)
    if kind == "special":
        flat = x.reshape(-1)
        n = flat.size
        flat[rng.choice(n, max(1, n // 7), replace=False)] = np.inf
        flat[rng.choice(n, max(1, n // 7), replace=False)] = -np.inf
        flat[rng.choice(n, max(1, n // 9), replace=False)] = np.nan
    return x


def _torch_fwd_bwd(fn, x, g, *args, **kw):
    xt = torch.from_numpy(x.copy()).requires_grad_(True)
    out = fn(xt, *args, **kw)
    y = out[0] if isinstance(out, tuple) else out
    y.backward(torch.from_numpy(g))
    return out, xt.grad.numpy()


@pytest.mark.parametrize("kind", ["normal", "ties", "special"])
@pytest.mark.parametrize("case", range(len(MAX_CASES)))
def test_max_pool_matches_torch(case, kind):
    sp, k, s, p, d, ceil = MAX_CASES[case]
    rng = np.random.default_rng(case * 3 + len(kind))
    x = _data(rng, (2, 3) + sp, kind)
    geo = P.Geometry("max", sp, k, s, p, d, ceil)
    y, idx, _ = P.forward(x, geo)
    g = rng.integers(-4, 5, y.shape).astype(np.float32)
    (yt, it), dxt = _torch_fwd_bwd(MAX[len(sp)], x, g, k, s, p, d, ceil, return_indices=True)
    assert y.shape == tuple(yt.shape)
    np.testing.assert_array_equal(y.view(np.uint32), yt.detach().numpy().view(np.uint32))
    np.testing.assert_array_equal(idx, it.numpy())
    dx = P.backward(g, geo, idx)
    np.testing.assert_array_equal(dx, dxt)


def _bound(x, geo, y64):
    """(R + 1) * 2^-24 * sum|x| / divisor per output, R the window's element count"""
    _, _, abs64 = P.forward(np.abs(x), geo)
    r = np.array([len(w) for w in geo.windows], dtype=np.float64)
    return ((r + 1) * 2.0 ** -24 * abs64.reshape(-1, geo.n_out) * geo.div).reshape(y64.shape) / \
        geo.div.astype(np.float64).reshape((1,) * (y64.ndim - len(geo.out_sp)) + geo.out_sp) + 1e-30


def _check_average(geo, fn, args, kw, sp, kind, seed):
    rng = np.random.default_rng(seed)
    x = _data(rng, (2, 3) + sp, kind)
    y, _, y64 = P.forward(x, geo)
    g = (rng.integers(-4, 5, y.shape) if kind == "int" else rng.standard_normal(y.shape)).astype(np.float32)
    yt, dxt = _torch_fwd_bwd(fn, x, g, *args, **kw)
    yt = yt.detach().numpy()
    assert y.shape == yt.shape
    bound = _bound(x, geo, y64)
    assert np.all(np.abs(y - y64) <= bound)
    assert np.all(np.abs(yt - y64) <= bound)
    dx = P.backward(g, geo)
    if kind == "int":
        np.testing.assert_array_equal(y.astype(np.float64), y64.astype(np.float32).astype(np.float64))
    np.testing.assert_allclose(dx, dxt, rtol=1e-6, atol=1e-6 * float(np.abs(g).max()))


@pytest.mark.parametrize("kind", ["normal", "int"])
@pytest.mark.parametrize("include_pad", [True, False])
@pytest.mark.parametrize("case", range(len(AVG_CASES)))
def test_avg_pool_matches_torch(case, include_pad, kind):
    sp, k, s, p, ceil = AVG_CASES[case]
    geo = P.Geometry("avg", sp, k, s, p, None, ceil, include_pad=include_pad)
    _check_average(geo, AVG[len(sp)], (k, s, p, ceil, include_pad), {}, sp, kind, case)


@pytest.mark.parametrize("kind", ["normal", "int"])
@pytest.mark.parametrize("case", range(len(ADAPTIVE_CASES)))
def test_adaptive_avg_pool_matches_torch(case, kind):
    sp, o = ADAPTIVE_CASES[case]
    geo = P.Geometry("adaptive", sp, output_size=o)
    _check_average(geo, ADAPTIVE[len(sp)], (o,), {}, sp, kind, 100 + case)


def test_large_window_order_is_the_warp_tree():
    """a 7x7 global average has 49 elements: the lane chunks and the xor tree, not the row-major sum"""
    geo = P.Geometry("adaptive", (7, 7), output_size=(1, 1))
    assert geo.large
    x = np.zeros(49, dtype=np.float32)
    x[[0, 4, 8, 12]] = [1.0, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24]      # f32 chunks of 4: lanes 0, 1, 2, 3
    y, _, _ = P.forward(x.reshape(1, 1, 7, 7), geo, "f32")
    # row-major, each 1 + 2^-24 rounds back to 1; the tree adds lanes 1 and 3 first (2^-23), then lane 0 gets them
    assert float(y.reshape(())) == float(np.float32(1.0 + 2.0 ** -23) / np.float32(49))
    assert not P.Geometry("max", (9, 9), (5, 5), (1, 1), (2, 2), (1, 1)).large
    assert P.Geometry("max", (9, 9), (6, 6), (1, 1), (3, 3), (1, 1)).large


def test_beta_rounds_product_and_sum_separately():
    geo = P.Geometry("avg", (4,), (2,), (2,), (0,))
    g = np.array([[[3.0, 5.0]]], dtype=np.float32)
    dx = np.array([[[1.0, 2.0, 3.0, 4.0]]], dtype=np.float32)
    out = P.backward(g, geo, dx=dx, beta=0.5)
    np.testing.assert_array_equal(out, np.array([[[2.0, 2.5, 4.0, 4.5]]], dtype=np.float32))
