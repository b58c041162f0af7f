"""numpy restatement of the embedding kernels (neuronika_b200/csrc/nk_embedding.cu, include/nk_b200.h nk_embedding_*).

Ids are floats: x is a valid id when 0 <= x < v (NaN, negatives and x >= v are not), and its id is trunc(x).  An
invalid id reads a zero row and adds no gradient; neither does padding_idx in the backward.

The backward's f32 summation order: the keys (the id, or v for an invalid or padding position) are sorted stably, so
each row's positions ascend; the sorted sequence is cut into slots of CHUNK entries; each row's run inside a slot is
summed sequentially from its first element; a row spanning several slots adds those runs' partials in slot order.
The sum is rounded once into dw's type as dw = beta*dw + sum, the product and the add rounded separately (beta = 0
does not read dw); rows without a valid position get beta*dw (zeros for beta = 0) unless beta == 1."""
from __future__ import annotations

import numpy as np

CHUNK = 32


def keys(ids, v: int, padding_idx: int = -1) -> np.ndarray:
    x = np.asarray(ids, dtype=np.float32).reshape(-1)
    with np.errstate(invalid="ignore"):
        valid = (x >= 0) & (x < np.float32(v))
    k = np.where(valid, np.trunc(np.where(valid, x, 0)), v).astype(np.int64)
    if padding_idx >= 0:
        k[k == padding_idx] = v
    return k


def forward(w: np.ndarray, ids) -> np.ndarray:
    """y = w[id] with zero rows for invalid ids; shape ids.shape + (e,), w's dtype (bit-exact copy)"""
    v, e = w.shape
    k = keys(ids, v)
    y = np.zeros((k.size, e), dtype=w.dtype)
    ok = k < v
    y[ok] = w[k[ok]]
    return y.reshape(tuple(np.shape(ids)) + (e,))


def row_sums(g: np.ndarray, ids, v: int, padding_idx: int = -1):
    """{row: f32 sum} in the kernel's order; g (n, e) as f32 values"""
    g = np.asarray(g, dtype=np.float32).reshape(-1, np.shape(g)[-1])
    k = keys(ids, v, padding_idx)
    order = np.argsort(k, kind="stable")
    sk = k[order]
    out = {}
    n = sk.size
    bounds = np.flatnonzero(np.diff(sk)) + 1
    starts = np.concatenate(([0], bounds)) if n else np.zeros(0, np.int64)
    ends = np.concatenate((bounds, [n])) if n else np.zeros(0, np.int64)
    for s, t in zip(starts, ends):
        r = int(sk[s])
        if r >= v:
            continue
        # the run's pieces, cut at the slot boundaries; np.cumsum adds strictly in order in f32 (np.sum would not)
        cuts = [s] + list(range((s // CHUNK + 1) * CHUNK, t, CHUNK)) + [t]
        rows = g[order[s:t]]
        first = cuts[1] - s
        parts = [np.cumsum(rows[:first], axis=0, dtype=np.float32)[-1]]
        full = (len(cuts) - 3) * CHUNK            # whole slots between the first and the last piece
        if full > 0:
            mid = rows[first:first + full].reshape(-1, CHUNK, rows.shape[1])
            parts.extend(np.cumsum(mid, axis=1, dtype=np.float32)[:, -1])
        if t > cuts[-2] and len(cuts) > 2:
            parts.append(np.cumsum(rows[cuts[-2] - s:], axis=0, dtype=np.float32)[-1])
        out[r] = np.cumsum(np.stack(parts), axis=0, dtype=np.float32)[-1]
    return out


def backward(dw: np.ndarray, ids, g: np.ndarray, padding_idx: int = -1, beta: float = 1.0,
             round_out=None) -> np.ndarray:
    """dw (v, e) f32 values after nk_embedding_bwd; round_out rounds f32 values into dw's type (None: f32)"""
    rnd = round_out or (lambda a: a.astype(np.float32))
    v, e = dw.shape
    sums = row_sums(g, ids, v, padding_idx)
    b = np.float32(beta)
    out = np.array(dw, dtype=np.float32, copy=True)
    rows = np.fromiter(sums, dtype=np.int64, count=len(sums))
    s = np.stack([sums[r] for r in rows]) if len(rows) else np.zeros((0, e), np.float32)
    if beta == 0.0:
        new = rnd(s)
        out[:] = 0.0
    else:
        new = rnd((b * out[rows]).astype(np.float32) + s)
        if beta != 1.0:
            out[:] = rnd((b * out).astype(np.float32))
    out[rows] = new
    return out
