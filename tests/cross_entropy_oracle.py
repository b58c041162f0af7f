"""Float64 restatement of the cross-entropy of include/nk_b200.h (nk_cross_entropy_fwd / nk_cross_entropy_bwd), which is
torch's F.cross_entropy with class-index targets except that an invalid id (NaN, < 0, >= C) is ignored instead of
raising.  x is (N, C) or (N, C, d1, ..., dk); the target (N) or (N, d1, ..., dk) holds float class ids."""
import numpy as np


def positions(x):
    """x as a (positions, classes) float64 matrix in the position order of the target, and (n, c, s)"""
    x = np.asarray(x, np.float64)
    n, c = x.shape[0], x.shape[1]
    s = int(np.prod(x.shape[2:], dtype=np.int64)) if x.ndim > 2 else 1
    return x.reshape(n, c, s).transpose(0, 2, 1).reshape(n * s, c), n, c, s


def classes(target, c, ignore_index=-100):
    """the class of each position, -1 where it is ignored"""
    t = np.asarray(target, np.float64).reshape(-1)
    with np.errstate(invalid="ignore"):
        valid = (t >= 0) & (t < c)
    k = np.where(valid, np.trunc(np.where(valid, t, 0)), -1).astype(np.int64)
    k[k == ignore_index] = -1
    return k


def _parts(x, target, weight, ignore_index):
    xp, n, c, s = positions(x)
    k = classes(target, c, ignore_index)
    w = np.ones(c) if weight is None else np.asarray(weight, np.float64)
    keep = k >= 0
    kk = np.where(keep, k, 0)
    if xp.shape[0]:
        m = xp.max(axis=1, keepdims=True)
        lse = (m + np.log(np.exp(xp - m).sum(axis=1, keepdims=True)))[:, 0]
    else:
        lse = np.zeros(0)
    wt = np.where(keep, w[kk], 0.0)
    return xp, (n, c, s), k, keep, kk, w, wt, lse


def forward(x, target, weight=None, mean=True, ignore_index=-100, label_smoothing=0.0):
    """(loss, lse per position with 0 where ignored, denominator = summed weights of the non-ignored positions)"""
    xp, (n, c, s), k, keep, kk, w, wt, lse = _parts(x, target, weight, ignore_index)
    eps = float(label_smoothing)
    xt = xp[np.arange(xp.shape[0]), kk] if xp.shape[0] else np.zeros(0)
    with np.errstate(invalid="ignore"):  # an ignored position whose class-0 logit is -inf gives 0 * inf, dropped below
        ell = (1 - eps) * wt * (lse - xt)
        if eps:  # without smoothing a -inf logit of another class adds nothing (0 * inf would be NaN)
            ell = ell + eps / c * ((lse[:, None] - xp) * w[None, :]).sum(axis=1)
    ell = np.where(keep, ell, 0.0)
    denom = float(wt.sum())
    total = float(ell.sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        loss = np.float64(total) / np.float64(denom) if mean else total
    return float(loss), np.where(keep, lse, 0.0), denom


def backward(x, target, g=1.0, weight=None, mean=True, ignore_index=-100, label_smoothing=0.0):
    """g * d loss / d x, in x's shape"""
    xp, (n, c, s), k, keep, kk, w, wt, lse = _parts(x, target, weight, ignore_index)
    eps = float(label_smoothing)
    p = np.exp(xp - lse[:, None]) if xp.shape[0] else xp
    onehot = np.zeros_like(xp)
    onehot[np.arange(xp.shape[0])[keep], kk[keep]] = 1.0
    d = (1 - eps) * wt[:, None] * (p - onehot) + eps / c * (w.sum() * p - w[None, :])
    denom = wt.sum()
    with np.errstate(invalid="ignore", divide="ignore"):
        scale = g / denom if mean else g
        d = np.where(keep[:, None], d * scale, 0.0)
    return d.reshape(n, s, c).transpose(0, 2, 1).reshape(np.shape(x))


def grad_bound(g, weight, scale):
    """B = |g| * max(w) * s: the largest magnitude any gradient element can take (s = 1 / denominator for Mean)"""
    wmax = 1.0 if weight is None else float(np.max(np.abs(weight)))
    return abs(g) * wmax * scale
