"""A numpy restatement of the pooling ops of csrc/nk_pool.cu (max, average, adaptive average over 1..3 sample dims),
forward and gather backward, in the kernels' f32 summation orders, with a float64 shadow of the averages.

Windows: along each axis output o of a max / avg pool starts at a = o*s - p and holds a + j*d, j < k (d = 1 for avg); the
adaptive pool's window i is [floor(i*L/O), ceil((i+1)*L/O)).  Only in-bounds positions are candidates.  A window of
LARGE_WINDOW or more elements (prod(k), or prod(ceil(L/O)) for the adaptive pool) is reduced by one warp:
its in-bounds elements in row-major order go to the 32 lanes in chunks of V (8 for bf16, 4 for f32; chunk c to lane
c % 32), each lane adds its chunks in order, and the lanes are combined by the xor-shuffle tree 16, 8, 4, 2, 1.  Smaller
windows are added in row-major order by one thread.  The average is the f32 sum divided once by the divisor."""
from __future__ import annotations

import itertools
import math

import numpy as np

LARGE_WINDOW = 32


def bf16_round(x: np.ndarray) -> np.ndarray:
    """float32 -> nearest bfloat16 (ties to even), as float32; NaN stays NaN"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    bits = x.view(np.uint32).astype(np.uint64)
    r = (((bits + ((bits >> 16) & 1) + 0x7FFF) >> 16) << 16).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(x), x, r).reshape(x.shape)


def round_to(x: np.ndarray, dtype: str) -> np.ndarray:
    return bf16_round(x) if dtype == "bf16" else np.asarray(x, dtype=np.float32)


def out_extent(L, k, s, p, d=1, ceil_mode=False):
    """torch's pooling output extent"""
    num = L + 2 * p - d * (k - 1) - 1
    o = (num + (s - 1 if ceil_mode else 0)) // s + 1
    if ceil_mode and (o - 1) * s >= L + p:
        o -= 1
    return o


class Geometry:
    """the windows of one pool: kind "max" / "avg" / "adaptive" over in_sp (nsp entries)"""

    def __init__(self, kind, in_sp, k=None, stride=None, padding=None, dilation=None, ceil_mode=False,
                 output_size=None, include_pad=True):
        nsp = len(in_sp)
        self.kind, self.in_sp = kind, tuple(in_sp)
        axes = []
        if kind == "adaptive":
            self.out_sp = tuple(output_size)
            vol = math.prod(-(-L // O) for L, O in zip(in_sp, output_size))
            for L, O in zip(in_sp, output_size):
                wins = []
                for o in range(O):
                    lo, hi = o * L // O, -(-(o + 1) * L // O)
                    wins.append((list(range(lo, hi)), hi - lo))
                axes.append(wins)
        else:
            stride = stride or k
            padding = padding or (0,) * nsp
            dilation = dilation or (1,) * nsp
            self.out_sp = tuple(out_extent(L, kk, s, p, d, ceil_mode)
                                for L, kk, s, p, d in zip(in_sp, k, stride, padding, dilation))
            vol = math.prod(k)
            for L, O, kk, s, p, d in zip(in_sp, self.out_sp, k, stride, padding, dilation):
                wins = []
                for o in range(O):
                    a = o * s - p
                    pos = [a + j * d for j in range(kk) if 0 <= a + j * d < L]
                    div = min(a + kk, L + p) - a if kind == "avg" and include_pad else len(pos)
                    wins.append((pos, div))
                axes.append(wins)
        self.large = vol >= LARGE_WINDOW
        # per output (row-major): the in-plane flat indices of its in-bounds window elements in row-major order
        strides = [math.prod(in_sp[i + 1:]) for i in range(nsp)]
        self.windows, divs = [], []
        for combo in itertools.product(*axes):
            pos = [sum(u * st for u, st in zip(us, strides)) for us in itertools.product(*(w[0] for w in combo))]
            self.windows.append(pos)
            divs.append(math.prod(w[1] for w in combo))
        self.div = np.array(divs, dtype=np.float32)
        self.n_in, self.n_out = math.prod(in_sp), len(self.windows)
        wmax = max([len(w) for w in self.windows] + [1])
        self.widx = np.full((self.n_out, wmax), -1, dtype=np.int64)
        for o, w in enumerate(self.windows):
            self.widx[o, :len(w)] = w
        # per input element: the outputs whose windows hold it, ascending
        cands = [[] for _ in range(self.n_in)]
        for o, w in enumerate(self.windows):
            for u in w:
                cands[u].append(o)
        cmax = max([len(c) for c in cands] + [1])
        self.cidx = np.full((self.n_in, cmax), -1, dtype=np.int64)
        for u, c in enumerate(cands):
            self.cidx[u, :len(c)] = c


def forward(x: np.ndarray, geo: Geometry, dtype: str = "f32"):
    """x (N, C, *in_sp) holding values of `dtype`.  Returns (y rounded to dtype, idx int32 or None, float64 shadow)."""
    lead = x.shape[:x.ndim - len(geo.in_sp)]
    xv = np.asarray(x, dtype=np.float32).reshape(-1, geo.n_in)
    mask = geo.widx >= 0
    vals = xv[:, geo.widx.clip(0)]                                     # (planes, n_out, wmax)
    shape = lead + geo.out_sp
    if geo.kind == "max":
        m = np.full(vals.shape[:2], -np.inf, dtype=np.float32)
        best = np.full(vals.shape[:2], -1, dtype=np.int64)
        with np.errstate(invalid="ignore"):
            for j in range(vals.shape[2]):
                v = vals[..., j]
                rep = mask[None, :, j] & ((best < 0) | (v > m) | np.isnan(v))
                m = np.where(rep, v, m)
                best = np.where(rep, geo.widx[None, :, j], best)
        return round_to(m, dtype).reshape(shape), best.astype(np.int32).reshape(shape), m.astype(np.float64).reshape(shape)
    if geo.large:
        V = 8 if dtype == "bf16" else 4
        lanes = np.zeros(vals.shape[:2] + (32,), dtype=np.float32)
        for q in range(vals.shape[2]):
            lane = (q // V) % 32
            lanes[..., lane] = np.where(mask[None, :, q], lanes[..., lane] + vals[..., q], lanes[..., lane])
        for off in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[..., np.arange(32) ^ off]
        acc = lanes[..., 0]
    else:
        acc = np.zeros(vals.shape[:2], dtype=np.float32)
        for j in range(vals.shape[2]):
            acc = np.where(mask[None, :, j], acc + vals[..., j], acc)
    y = acc / geo.div
    y64 = np.where(mask[None], vals.astype(np.float64), 0.0).sum(axis=2) / geo.div.astype(np.float64)
    return round_to(y, dtype).reshape(shape), None, y64.reshape(shape)


def backward(g: np.ndarray, geo: Geometry, idx: np.ndarray | None = None, dx: np.ndarray | None = None,
             beta: float = 0.0, dx_dtype: str = "f32"):
    """the gather backward: dx = beta*dx + sum over the outputs holding each element, ascending, in f32 (max: g[o] where
    idx[o] is the element; averages: g[o] / divisor), the product and the add rounded separately.  g (N, C, *out_sp)
    holding values of its dtype; returns dx (N, C, *in_sp) rounded to dx_dtype."""
    lead = g.shape[:g.ndim - len(geo.out_sp)]
    gv = np.asarray(g, dtype=np.float32).reshape(-1, geo.n_out)
    mask = geo.cidx >= 0
    c = geo.cidx.clip(0)
    contrib = gv[:, c]                                                 # (planes, n_in, cmax)
    valid = np.broadcast_to(mask[None], contrib.shape)
    if geo.kind == "max":
        iv = np.asarray(idx).reshape(-1, geo.n_out)[:, c]
        valid = valid & (iv == np.arange(geo.n_in)[None, :, None])
    else:
        contrib = contrib / geo.div[c][None]
    acc = np.zeros(contrib.shape[:2], dtype=np.float32)
    for j in range(contrib.shape[2]):
        acc = np.where(valid[..., j], acc + contrib[..., j], acc)
    if beta != 0.0:
        acc = np.float32(beta) * np.asarray(dx, dtype=np.float32).reshape(acc.shape) + acc
    return round_to(acc, dx_dtype).reshape(lead + geo.in_sp)
