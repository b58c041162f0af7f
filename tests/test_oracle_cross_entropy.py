"""The float64 cross-entropy oracle (tests/cross_entropy_oracle.py) against torch CPU F.cross_entropy, forward and
autograd: (N, C) and (N, C, d1[, d2]) inputs, with and without class weights, label smoothing 0 / 0.1 / 1, Sum and
Mean, ignore_index on a valid class, C = 1, N = 0 and a fully ignored batch (NaN loss, zero gradient)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cross_entropy_oracle as O


def torch_ce(x, target, weight, mean, ignore_index, eps, g=1.0):
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    w = None if weight is None else torch.tensor(weight, dtype=torch.float64)
    loss = F.cross_entropy(xt, torch.tensor(target.astype(np.int64)), weight=w, ignore_index=ignore_index,
                           reduction="mean" if mean else "sum", label_smoothing=eps)
    (loss * g).backward()
    return loss.item(), xt.grad.numpy()


def make(rng, shape, c, ignore_index=None, ignore_frac=0.0):
    n, rest = shape[0], shape[2:]
    x = rng.standard_normal(shape) * 2
    t = rng.integers(0, c, (n,) + tuple(rest))
    if ignore_index is not None and ignore_frac:
        t = np.where(rng.random(t.shape) < ignore_frac, ignore_index, t)
    return x, t


SHAPES = [(9, 7), (6, 5, 4), (3, 4, 5, 3), (13, 1)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("mean", [True, False], ids=["mean", "sum"])
def test_oracle_matches_torch(shape, weighted, eps, mean):
    rng = np.random.default_rng(hash((shape, weighted, eps, mean)) % (1 << 32))
    c = shape[1]
    x, t = make(rng, shape, c)
    w = rng.uniform(0.2, 2.0, c) if weighted else None
    want_loss, want_grad = torch_ce(x, t, w, mean, -100, eps, g=0.75)
    loss, lse, denom = O.forward(x, t.astype(np.float32), w, mean, -100, eps)
    np.testing.assert_allclose(loss, want_loss, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(O.backward(x, t.astype(np.float32), 0.75, w, mean, -100, eps), want_grad, rtol=1e-10,
                               atol=1e-12)


@pytest.mark.parametrize("ignore_index", [0, 2, -100])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("shape", [(40, 6), (5, 6, 7)], ids=lambda s: "x".join(map(str, s)))
def test_ignore_index(ignore_index, weighted, eps, shape):
    """ignored positions add nothing to the loss, the Mean denominator or the gradient; ignore_index may be a valid
    class"""
    rng = np.random.default_rng(7 + abs(ignore_index))
    x, t = make(rng, shape, shape[1], ignore_index, 0.3)
    w = rng.uniform(0.2, 2.0, shape[1]) if weighted else None
    for mean in (True, False):
        want_loss, want_grad = torch_ce(x, t, w, mean, ignore_index, eps)
        loss, lse, denom = O.forward(x, t.astype(np.float32), w, mean, ignore_index, eps)
        np.testing.assert_allclose(loss, want_loss, rtol=1e-12)
        np.testing.assert_allclose(O.backward(x, t.astype(np.float32), 1.0, w, mean, ignore_index, eps), want_grad,
                                   rtol=1e-10, atol=1e-13)
        tf = t.reshape(-1)
        kept = tf != ignore_index
        assert denom == pytest.approx((w[tf[kept]] if weighted else np.ones(kept.sum())).sum())


def test_empty_batch():
    x = np.zeros((0, 5))
    t = np.zeros((0,), np.int64)
    for mean in (True, False):
        want_loss, want_grad = torch_ce(x, t, None, mean, -100, 0.0)
        loss, lse, denom = O.forward(x, t.astype(np.float32), None, mean)
        assert (np.isnan(loss) and np.isnan(want_loss)) if mean else loss == want_loss == 0.0
        assert lse.shape == (0,) and denom == 0.0
        assert O.backward(x, t.astype(np.float32), 1.0, None, mean).shape == want_grad.shape == (0, 5)


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
def test_all_ignored_is_nan_with_zero_gradient(eps, weighted):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((6, 4, 3))
    t = np.full((6, 3), 1)
    w = rng.uniform(0.5, 1.5, 4) if weighted else None
    want_loss, want_grad = torch_ce(x, t, w, True, 1, eps)
    loss, _, denom = O.forward(x, t.astype(np.float32), w, True, 1, eps)
    assert np.isnan(want_loss) and np.isnan(loss) and denom == 0.0
    got = O.backward(x, t.astype(np.float32), 1.0, w, True, 1, eps)
    assert not np.any(got) and not np.any(want_grad)
    want_loss, _ = torch_ce(x, t, w, False, 1, eps)
    assert O.forward(x, t.astype(np.float32), w, False, 1, eps)[0] == want_loss == 0.0


def test_invalid_ids_are_ignored_and_fractions_truncate():
    """torch raises on an out-of-range id; the oracle (and the kernels) ignore it.  The result equals torch's with those
    positions given ignore_index, and a fractional id selects trunc(id)."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((8, 5))
    ids = np.array([0.5, 4.75, -1, 5, np.nan, 2, -0.5, np.inf], np.float32)
    t = np.array([0, 4, -100, -100, -100, 2, -100, -100])
    for mean in (True, False):
        want_loss, want_grad = torch_ce(x, t, None, mean, -100, 0.1)
        np.testing.assert_allclose(O.forward(x, ids, None, mean, -100, 0.1)[0], want_loss, rtol=1e-12)
        np.testing.assert_allclose(O.backward(x, ids, 1.0, None, mean, -100, 0.1), want_grad, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_minus_inf_logits(eps):
    """masked (-inf) logits of other classes: a finite loss without smoothing, +inf with it (each -inf class adds
    eps/C * inf), and a finite gradient with 0 at the masked classes either way"""
    rng = np.random.default_rng(12)
    x = rng.standard_normal((7, 10, 3))
    x[:, 0] = -np.inf
    x[:, 9, 1] = -np.inf
    x[2, :8] = -np.inf
    t = rng.integers(1, 9, (7, 3))
    t[2] = 8
    for mean in (True, False):
        want_loss, want_grad = torch_ce(x, t, None, mean, -100, eps)
        loss = O.forward(x, t.astype(np.float32), None, mean, -100, eps)[0]
        assert np.isfinite(loss) == (eps == 0) and loss == pytest.approx(want_loss, rel=1e-12)
        got = O.backward(x, t.astype(np.float32), 1.0, None, mean, -100, eps)
        np.testing.assert_allclose(got, want_grad, rtol=1e-10, atol=1e-14)
