"""numpy restatement of the criteria and of dropout (csrc/nk_criteria.cu, csrc/nk_dropout.cu; reference node/
absolute_error, bce, bce_with_logits, kldiv and dropout).

Per-element maths is float32 in the reference's operation order; a forward's sum is taken in float64 (the kernels sum
f32 partials into double, so the two agree to a few f32 ulps of the total, not bit for bit).  Backward results and
dropout are elementwise and exact: the device reproduces them bit for bit in f32 (bf16 results are these rounded once
to nearest even).

Dropout's generator is Philox4x32-10 (Salmon et al., SC'11): key = the 64-bit seed, counter = (e/4 as 64 bits, call id
as 64 bits), element e takes word e%4; keep iff (r >> 8) * 2^-24 < 1 - float32(p)."""
from __future__ import annotations

import numpy as np

F32 = np.float32
FLT_EPSILON = F32(np.finfo(np.float32).eps)   # f32::EPSILON, 2^-23

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr (N, 4) uint32, key (2,) uint32 -> (N, 4) uint32"""
    c = [np.asarray(ctr, np.uint32)[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0, k1 = np.uint32(k0 + _W0), np.uint32(k1 + _W1)
            p0, p1 = _M0 * c[0], _M1 * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1),
                 p0 & _LO]
    return np.stack(c, axis=1).astype(np.uint32)


def dropout_words(seed: int, call: int, elements):
    """the Philox word element e draws, for each e in `elements` (int64 array)"""
    e = np.asarray(elements, np.int64)
    g = (e // 4).astype(np.uint64)
    ctr = np.stack([g & _LO, g >> np.uint64(32), np.full_like(g, call & 0xFFFFFFFF),
                    np.full_like(g, (call >> 32) & 0xFFFFFFFF)], axis=1).astype(np.uint32)
    out = philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
    return out[np.arange(e.size), (e % 4).astype(np.int64)]


def keep_prob(p: float):
    return F32(1.0) - F32(p)


def dropout_keep(seed: int, call: int, n: int, p: float, elements=None):
    """keep flags of elements [0, n) (or of `elements`) for one dropout forward"""
    e = np.arange(n, dtype=np.int64) if elements is None else np.asarray(elements, np.int64)
    u = (dropout_words(seed, call, e) >> np.uint32(8)).astype(F32) * F32(2.0 ** -24)
    return u < keep_prob(p)


def pack_mask(keep):
    """bit e%32 of word e/32"""
    keep = np.asarray(keep, bool)
    words = (keep.size + 31) // 32
    bits = np.zeros(words * 32, np.uint64)
    bits[:keep.size] = keep
    return (bits.reshape(words, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)


def unpack_mask(words, n):
    w = np.asarray(words, np.uint32).astype(np.uint64)
    return ((w[:, None] >> np.arange(32, dtype=np.uint64)) & np.uint64(1)).astype(bool).ravel()[:n]


def dropout_forward(x, keep, p):
    """x * keep / q in f32 (x / q where kept)"""
    x = np.asarray(x, F32)
    q = keep_prob(p)
    return np.where(keep.reshape(x.shape), x / q, F32(0)).astype(F32)


def dropout_backward(g, keep, p):
    """the true gradient of dropout_forward: g * keep / q (SURVEY.md 8-c defect 8)"""
    g = np.asarray(g, F32)
    q = keep_prob(p)
    with np.errstate(divide="ignore", invalid="ignore"):   # p = 1 keeps nothing
        return np.where(keep.reshape(g.shape), g / q, F32(0)).astype(F32)


# ---------------------------------------------------------------- criteria: (forward term, backward before the mean)
def _clamp_log(v):
    return np.where(v < F32(-100), F32(-100), np.where(v > np.finfo(F32).max, np.finfo(F32).max, v)).astype(F32)


def terms(name, x, t):
    x, t = np.asarray(x, F32), np.asarray(t, F32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if name == "mae":
            return np.abs(x - t)
        if name == "bce":
            return (t - F32(1)) * _clamp_log(np.log(F32(1) - x)) - t * _clamp_log(np.log(x))
        if name == "bce_with_logits":
            m = np.maximum(-x, F32(0))
            return (F32(1) - t) * x + m + np.log(np.exp(-m) + np.exp(-x - m))
        if name == "kldiv":
            return np.where(t > 0, t * (np.log(np.where(t > 0, t, F32(1))) - x), F32(0)).astype(F32)
    raise KeyError(name)


def divisor(name, shape):
    return shape[0] if name == "kldiv" else int(np.prod(shape))


def forward(name, x, t, mean=True):
    """the loss: float64 sum of the float32 terms, [/ n (kldiv: / shape[0])], as float32"""
    s = terms(name, x, t).astype(np.float64).sum()
    if mean:
        s = s * (1.0 / divisor(name, np.shape(x)))
    return F32(s)


def backward(name, x, t, g=1.0, mean=True):
    """dloss/dx * g [/ n], float32, the reference's operation order"""
    x, t, g = np.asarray(x, F32), np.asarray(t, F32), F32(g)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if name == "mae":
            d = x - t
            v = np.where(d == 0, F32(0), np.where(np.isnan(d), d, np.copysign(F32(1), d)) * g)
        elif name == "bce":
            v = (x - t) / np.maximum((F32(1) - x) * x, FLT_EPSILON) * g
        elif name == "bce_with_logits":
            v = (F32(1) / (F32(1) + np.exp(-x)) - t) * g
        elif name == "kldiv":
            v = -t * g
        else:
            raise KeyError(name)
        v = v.astype(F32)
        if mean:
            v = (v / F32(divisor(name, x.shape))).astype(F32)
    return v
