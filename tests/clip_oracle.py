"""Float64 restatement of the gradient clipping of include/nk_b200.h (nk_grad_norm, nk_grad_scale_by_norm,
nk_grad_clamp), which is torch.nn.utils' get_total_norm / clip_grads_with_norm_ / clip_grad_value_ with a gradient
scale k: every element enters the norm as v = f32(k * g).  The total is computed directly in float64 (torch takes the
norm of the per-tensor norms, which is the same number before rounding); the coefficient, the scaling and the clamp are
evaluated in f32, one rounding per operation, as the device does."""
import numpy as np

F32 = np.float32


def bf16(x):
    """float32 -> nearest-even bfloat16, returned as float32; NaN stays NaN"""
    x = np.ascontiguousarray(x, dtype=F32)
    bits = x.view(np.uint32).astype(np.uint64)
    out = (((bits + ((bits >> 16) & 1) + 0x7FFF) >> 16) << 16).astype(np.uint32).view(F32).reshape(x.shape)
    return np.where(np.isnan(x), x, out)


def terms(grads, grad_scale=1.0):
    """|v| of every element of every gradient, v = f32(k * g), as one float64 vector"""
    k = F32(grad_scale)
    with np.errstate(over="ignore", invalid="ignore"):
        vs = [(np.asarray(g, F32).ravel() * k).astype(F32) for g in grads]
    return np.abs(np.concatenate(vs).astype(np.float64)) if vs else np.zeros(0)


def total_norm(grads, norm_type=2.0, grad_scale=1.0):
    """the total norm as a float64 (0 for no elements); NaN when any element is NaN, also for p = inf"""
    p = float(norm_type)
    if not p > 0:
        raise ValueError("norm_type must be > 0 or inf")
    a = terms(grads, grad_scale)
    if a.size == 0:
        return 0.0
    if np.isnan(a).any():
        return float("nan")
    with np.errstate(over="ignore", invalid="ignore"):
        if np.isinf(p):
            return float(a.max())
        if p == 2.0:
            return float(np.sqrt(np.sum(a * a)))
        if p == 1.0:
            return float(np.sum(a))
        return float(np.sum(a ** p) ** (1.0 / p))


def coefficient(total, max_norm):
    """torch's clip coefficient in f32: (1 / (total + 1e-6)) * max_norm (max_norm / x is x.reciprocal() * max_norm in
    torch), then 1 where it is > 1; a NaN total gives NaN"""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        c = (F32(1) / (F32(total) + F32(1e-6))) * F32(max_norm)
    return F32(1) if c > F32(1) else F32(c)


def scale(g, c, dtype="f32"):
    """g * c rounded once into the gradient's dtype"""
    with np.errstate(over="ignore", invalid="ignore"):
        out = (np.asarray(g, F32) * F32(c)).astype(F32)
    return bf16(out) if dtype == "bf16" else out


def clamp(g, clip_value, grad_scale=1.0, dtype="f32"):
    """torch's clamp_min(-b) then clamp_max(b), b = f32(clip_value / k); NaN elements stay NaN"""
    b = F32(F32(clip_value) / F32(grad_scale))
    g = np.asarray(g, F32)
    with np.errstate(invalid="ignore"):
        out = np.where(g < -b, -b, g)
        out = np.where(out > b, b, out).astype(F32)
    return bf16(out) if dtype == "bf16" else out
