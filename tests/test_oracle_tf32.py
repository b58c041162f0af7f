"""The host model of the TF32 / 3xTF32 GEMM modes (tests/tf32_oracle.py), pinned on the CPU against hand-made bit
patterns -- ties, negative values, rounding up into the next binade and to Inf, subnormals, Inf / NaN -- and, on random
data, the accuracy that makes 3xTF32 worth its cost: at least 2^8 closer to the float64 product than one TF32 pass."""
import numpy as np
import pytest

import tf32_oracle as T


def bits(v):
    return np.asarray(v, np.float32).view(np.uint32)


def f(u):
    return np.array([u], np.uint32).view(np.float32)


# (input bits, cvt.rna.tf32.f32 result bits)
ROUNDING = [
    (0x3F800000, 0x3F800000),   # 1.0: already TF32
    (0x3F800FFF, 0x3F800000),   # just below half a TF32 ulp: down
    (0x3F801000, 0x3F802000),   # exactly half: a tie, away from zero
    (0x3F801001, 0x3F802000),   # just above half: up
    (0x3F803000, 0x3F804000),   # a tie with an odd TF32 mantissa: away from zero (not to even)
    (0x3F805000, 0x3F806000),   # a tie with an even one: still away from zero
    (0xBF801000, 0xBF802000),   # negative tie: away from zero = more negative
    (0xBF800FFF, 0xBF800000),   # negative, below half: toward zero
    (0x3FFFF000, 0x40000000),   # 2 - 2^-11: the tie carries into the next binade (2.0)
    (0xBFFFFFFF, 0xC0000000),   # -(2 - 2^-23): up into the next binade, negative
    (0x7F7FF000, 0x7F800000),   # the tie above the largest TF32 value: Inf
    (0x7F7FE000, 0x7F7FE000),   # the largest TF32 value itself
    (0x00001000, 0x00002000),   # subnormal tie: away from zero, not flushed
    (0x00000FFF, 0x00000000),   # subnormal below half: to +0
    (0x80000FFF, 0x80000000),   # ... and to -0 keeping the sign
    (0x807FF000, 0x80800000),   # the largest subnormal's tie: up into the smallest normal
    (0x00000000, 0x00000000),
    (0x80000000, 0x80000000),
    (0x7F800000, 0x7F800000),   # +Inf
    (0xFF800000, 0xFF800000),   # -Inf
]


@pytest.mark.parametrize("src,want", ROUNDING)
def test_rounding_bit_patterns(src, want):
    got = bits(T.tf32_round(f(src)))[0]
    assert got == want, (hex(src), hex(got), hex(want))


def test_nan_passes_through():
    for u in (0x7FC00000, 0x7F800001, 0xFFC00123):
        out = T.tf32_round(f(u))
        assert np.isnan(out[0]) and bits(out)[0] == u
        hi, lo = T.tf32_split(f(u))
        assert np.isnan(hi[0]) and np.isnan(lo[0])


def test_low_13_bits_are_zero():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(4096).astype(np.float32) * np.float32(2.0) ** rng.integers(-140, 120, 4096)
    assert np.all((bits(T.tf32_round(x)) & 0x1FFF) == 0)


SPLITS = [
    # x, hi, lo
    (0x3F801FFF, 0x3F802000, 0xB4000000),   # 1 + 8191 * 2^-23: hi rounds up to 1 + 2^-10, lo = -2^-23
    (0x3F800FFF, 0x3F800000, 0x3A000000),   # 1 + 4095 * 2^-23: hi = 1, x - hi (12 bits) rounds to lo = 2^-11
    (0x3F800501, 0x3F800000, 0x39202000),   # 1 + 1281 * 2^-23: hi = 1, x - hi = 1281 * 2^-23 (11 bits) exact in TF32
    (0xBF801000, 0xBF802000, 0x3A000000),   # negative tie: hi = -(1 + 2^-10), lo = +2^-11
    (0x3F800000, 0x3F800000, 0x00000000),   # TF32 already: lo = 0
    (0x00001FFF, 0x00002000, 0x80000000),   # subnormal: x - hi = -2^-149 is below TF32's subnormal step: lo = -0
]


@pytest.mark.parametrize("x,hi,lo", SPLITS)
def test_split_bit_patterns(x, hi, lo):
    h, l = T.tf32_split(f(x))
    assert (bits(h)[0], bits(l)[0]) == (hi, lo), (hex(x), hex(bits(h)[0]), hex(bits(l)[0]))


def test_split_recovers_x_to_2_pow_minus_22():
    """x - hi is exact in f32 and has at most 13 significant bits; lo keeps 11 of them, so |x - hi - lo| <= 2^-22 |x|"""
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(1 << 16) * np.exp(rng.uniform(-20, 20, 1 << 16))).astype(np.float32)
    hi, lo = T.tf32_split(x)
    err = np.abs(x.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
    assert np.all(err <= 2.0 ** -22 * np.abs(x.astype(np.float64)))
    assert np.all(np.abs(lo.astype(np.float64)) <= 2.0 ** -11 * np.abs(x.astype(np.float64)))


@pytest.mark.parametrize("m,n,k", [(64, 48, 256), (33, 70, 1000)])
def test_three_passes_are_2_pow_8_closer(m, n, k):
    rng = np.random.default_rng(m + n + k)
    a = rng.uniform(-1, 1, (m, k)).astype(np.float32)
    b = rng.uniform(-1, 1, (k, n)).astype(np.float32)
    want = a.astype(np.float64) @ b.astype(np.float64)
    e1 = np.sqrt(np.mean((T.matmul_tf32(a, b) - want) ** 2))
    e3 = np.sqrt(np.mean((T.matmul_tf32x3(a, b) - want) ** 2))
    assert e3 * 2 ** 8 <= e1, (e1, e3)
