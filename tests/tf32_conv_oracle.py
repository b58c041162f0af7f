"""Host model of the f32 convolution modes (Device.f32_conv, csrc/nk_conv_tf32.cu), in float64.

The convolution of x padded by `pad` (mode "zero" / "constant" with a fill value, "reflective", "replicative") as one
column matrix per sample, cols[n] (L x K) with k = (c, i0, i1, ..) and l the output position in row-major order -- the
im2col engine's own formulation -- so that the three products are plain matrix products:
  forward  y[n] = W (Cout x K) . cols[n]^T + b
  dX       the gradient of the padded input, sum over the taps of G[n]^T . W scattered back, then its interior slice
           (the reference's pad backward: the padding's gradient is dropped in every mode)
  dW       sum_n G[n] . cols[n]
What TF32 mode computes, up to f32 accumulation, is this model on the TF32-rounded x (fill value included), w and g
(tf32_oracle.tf32_round); 3xTF32 is within (3R + 4) 2^-22 of it on the unrounded operands.  Called on |x|, |w|, |g| and
|fill| it gives the magnitudes the rounding bounds scale with."""
import numpy as np

NP_PAD = {"zero": "constant", "constant": "constant", "reflective": "reflect", "replicative": "edge"}


def pad_input(x, pad, mode, fill=0.0):
    widths = [(0, 0), (0, 0)] + [(p, p) for p in pad]
    if NP_PAD[mode] == "constant":
        return np.pad(x, widths, constant_values=fill if mode == "constant" else 0.0)
    return np.pad(x, widths, mode=NP_PAD[mode])


def columns(xp, k, stride, dil):
    """(cols (N, L, K), output extents) of the padded input xp"""
    nsp = len(k)
    span = [(kk - 1) * d + 1 for kk, d in zip(k, dil)]
    v = np.lib.stride_tricks.sliding_window_view(xp, span, axis=tuple(range(2, 2 + nsp)))
    v = v[(slice(None), slice(None)) + tuple(slice(None, None, s) for s in stride) + tuple(slice(None, None, d) for d in dil)]
    out = v.shape[2:2 + nsp]
    perm = (0,) + tuple(range(2, 2 + nsp)) + (1,) + tuple(range(2 + nsp, 2 + 2 * nsp))
    return v.transpose(perm).reshape(xp.shape[0], int(np.prod(out)), -1), out


def forward(x, w, b, pad, mode, fill, stride, dil):
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    cols, out = columns(pad_input(x, pad, mode, fill), w.shape[2:], stride, dil)
    y = (cols @ w.reshape(w.shape[0], -1).T).transpose(0, 2, 1).reshape((x.shape[0], w.shape[0]) + out)
    if b is not None:
        y = y + np.asarray(b, np.float64).reshape((1, -1) + (1,) * len(pad))
    return y


def backward_input(x_shape, g, w, pad, stride, dil):
    g, w = np.asarray(g, np.float64), np.asarray(w, np.float64)
    n, cout = g.shape[:2]
    padded = tuple(x_shape[:2]) + tuple(s + 2 * p for s, p in zip(x_shape[2:], pad))
    idx, _ = columns(np.arange(int(np.prod(padded))).reshape(padded), w.shape[2:], stride, dil)
    dcols = g.reshape(n, cout, -1).transpose(0, 2, 1) @ w.reshape(cout, -1)
    gp = np.bincount(idx.ravel(), weights=dcols.ravel(), minlength=int(np.prod(padded))).reshape(padded)
    return gp[(slice(None), slice(None)) + tuple(slice(p, p + s) for p, s in zip(pad, x_shape[2:]))]


def backward_kernel(g, x, w_shape, pad, mode, fill, stride, dil):
    g, x = np.asarray(g, np.float64), np.asarray(x, np.float64)
    cols, _ = columns(pad_input(x, pad, mode, fill), w_shape[2:], stride, dil)
    return np.einsum("nol,nlk->ok", g.reshape(g.shape[0], g.shape[1], -1), cols).reshape(w_shape)
