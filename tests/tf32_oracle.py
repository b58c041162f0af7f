"""Host model of the f32 tensor-core GEMM modes (nk_gemm_f32_config, csrc/nk_gemm_tf32.cu).

Every operand element is rounded to TF32 by the pack kernel with cvt.rna.tf32.f32: to nearest on the 10-bit mantissa,
ties away from zero, subnormals kept, Inf / NaN passed through, finite values past the largest TF32 value to Inf.  In
3xTF32 mode each element is split into hi = tf32(x) and lo = tf32(x - hi) and the product is
A_hi.B_hi + A_hi.B_lo + A_lo.B_hi.  The tensor cores multiply TF32 values exactly (11 x 11 significant bits fit in f32), so
everything the kernel does beyond this model is f32 accumulation."""
import numpy as np


def tf32_round(x):
    """cvt.rna.tf32.f32 on every element of a float32 array (returned as float32 with the low 13 bits zero)"""
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    special = (u & 0x7F800000) == 0x7F800000               # Inf / NaN: unchanged
    r = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)      # add half a TF32 ulp to the magnitude, truncate: ties away
    r = np.where(special, u.astype(np.uint32), r)
    return r.view(np.float32).reshape(x.shape)


def tf32_split(x):
    """(hi, lo) = (tf32(x), tf32(x - hi)), the difference taken in f32 as the pack kernel does"""
    x = np.asarray(x, np.float32)
    hi = tf32_round(x)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = tf32_round((x - hi).astype(np.float32))
    return hi, lo


def matmul_tf32(a, b):
    """float64 product of the TF32-rounded operands (op(A) M x K, op(B) K x N): what TF32 mode computes, up to f32
    accumulation"""
    return tf32_round(a).astype(np.float64) @ tf32_round(b).astype(np.float64)


def matmul_tf32x3(a, b):
    """float64 sum of the three TF32 products of 3xTF32 mode"""
    ah, al = (v.astype(np.float64) for v in tf32_split(a))
    bh, bl = (v.astype(np.float64) for v in tf32_split(b))
    return ah @ bh + ah @ bl + al @ bh
