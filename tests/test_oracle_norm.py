"""Pins tests/norm_oracle.py to torch's CPU F.batch_norm / F.layer_norm and their autograd, in float64: every module
option, momentum 0 and 1, the running statistics after three forwards (with the M/(M-1) correction), eval with one value
per channel, the one-value training error, empty batches and layer norm's shape-mismatch message."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import norm_oracle as O


def close(a, b, tol=1e-10):
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=tol, atol=tol)


def torch_bn(x, w, b, rm, rv, training, momentum, eps, g):
    t = lambda a, grad=False: None if a is None else torch.tensor(a, dtype=torch.float64, requires_grad=grad)
    xt, wt, bt = t(x, True), t(w, w is not None), t(b, b is not None)
    rmt, rvt = t(rm), t(rv)
    # nn.BatchNorm*d passes training=True whenever it tracks no running statistics
    y = F.batch_norm(xt, rmt, rvt, wt, bt, training or rm is None, momentum, eps)
    y.backward(torch.tensor(g))
    grad = lambda a: None if a is None else a.grad.numpy()
    return (y.detach().numpy(), grad(xt), grad(wt), grad(bt), None if rmt is None else rmt.numpy(),
            None if rvt is None else rvt.numpy())


BN_CASES = [  # shape, affine, track, training, momentum
    ((6, 5), True, True, True, 0.1),
    ((4, 3, 7), True, True, True, 0.0),
    ((4, 3, 7), False, True, True, 1.0),
    ((3, 4, 5, 6), True, False, True, 0.1),
    ((3, 4, 5, 6), True, False, False, 0.1),     # no running stats: batch statistics in eval too
    ((2, 3, 4, 3, 5), True, True, False, 0.1),
    ((5, 2, 1), False, False, True, 0.3),
]


@pytest.mark.parametrize("case", range(len(BN_CASES)))
def test_batch_norm_matches_torch(case):
    shape, affine, track, training, momentum = BN_CASES[case]
    rng = np.random.default_rng(case)
    c = shape[1]
    x = rng.standard_normal(shape) * 3 + 1
    g = rng.standard_normal(shape)
    w, b = (rng.standard_normal(c), rng.standard_normal(c)) if affine else (None, None)
    rm, rv = (rng.standard_normal(c), rng.uniform(0.5, 2, c)) if track else (None, None)
    y, mean, rstd, rm2, rv2, batch = O.bn_forward(x, w, b, rm, rv, training, momentum, 1e-5)
    dx, dw, db = O.bn_backward(g, x, mean, rstd, w, batch)
    ty, tdx, tdw, tdb, trm, trv = torch_bn(x, w, b, rm, rv, training, momentum, 1e-5, g)
    close(y, ty)
    close(dx, tdx)
    if affine:
        close(dw, tdw)
        close(db, tdb)
    if track:
        close(rm2, trm)
        close(rv2, trv)


def test_running_stats_after_three_forwards():
    rng = np.random.default_rng(3)
    rm, rv = np.zeros(4), np.ones(4)
    trm, trv = torch.zeros(4, dtype=torch.float64), torch.ones(4, dtype=torch.float64)
    for step in range(3):
        x = rng.standard_normal((3, 4, 2)) * (step + 1) + step   # M = 6: the unbiased correction is 6/5
        _, _, _, rm, rv, _ = O.bn_forward(x, rm=rm, rv=rv, training=True, momentum=0.25)
        F.batch_norm(torch.tensor(x), trm, trv, training=True, momentum=0.25)
    close(rm, trm.numpy())
    close(rv, trv.numpy())


def test_eval_with_one_value_per_channel_and_the_training_error():
    x = np.array([[1.0, -2.0, 3.0]])
    rm, rv = np.array([0.5, 0.0, -1.0]), np.array([2.0, 1.0, 0.5])
    y, *_ = O.bn_forward(x, rm=rm, rv=rv, training=False)
    close(y, F.batch_norm(torch.tensor(x), torch.tensor(rm), torch.tensor(rv), training=False).numpy())
    with pytest.raises(ValueError) as want:
        F.batch_norm(torch.tensor(x), torch.tensor(rm), torch.tensor(rv), training=True)
    with pytest.raises(ValueError) as got:
        O.bn_forward(x, rm=rm, rv=rv, training=True)
    assert str(got.value) == str(want.value)


def test_empty_batch_leaves_running_stats():
    x = np.zeros((0, 3, 4))
    rm, rv = np.array([0.5, 0.0, -1.0]), np.array([2.0, 1.0, 0.5])
    trm, trv = torch.tensor(rm), torch.tensor(rv)
    ty = F.batch_norm(torch.tensor(x), trm, trv, training=True)
    y, _, _, rm2, rv2, _ = O.bn_forward(x, rm=rm, rv=rv, training=True)
    assert y.shape == tuple(ty.shape) == (0, 3, 4)
    close(rm2, trm.numpy())
    close(rv2, trv.numpy())
    close(rm2, rm)


LN_CASES = [  # shape, normalized_shape, affine, bias
    ((4, 7), (7,), True, True),
    ((3, 5, 8), (8,), True, False),
    ((2, 3, 4, 5), (3, 4, 5), True, True),
    ((6, 9), (9,), False, False),
    ((0, 5), (5,), True, True),
    ((2, 1), (1,), True, True),
]


@pytest.mark.parametrize("case", range(len(LN_CASES)))
def test_layer_norm_matches_torch(case):
    shape, ns, affine, bias = LN_CASES[case]
    rng = np.random.default_rng(10 + case)
    x, g = rng.standard_normal(shape) * 2 - 1, rng.standard_normal(shape)
    w = rng.standard_normal(ns) if affine else None
    b = rng.standard_normal(ns) if affine and bias else None
    y, mean, rstd = O.ln_forward(x, ns, w, b, 1e-5)
    dx, dw, db = O.ln_backward(g, x, ns, mean, rstd, w)
    t = lambda a: None if a is None else torch.tensor(a, requires_grad=True)
    xt, wt, bt = t(x), t(w), t(b)
    yt = F.layer_norm(xt, ns, wt, bt, 1e-5)
    yt.backward(torch.tensor(g))
    close(y, yt.detach().numpy())
    close(dx, xt.grad.numpy())
    if w is not None:
        close(dw, wt.grad.numpy())
    if b is not None:
        close(db, bt.grad.numpy())


def test_layer_norm_mismatch_message():
    x = np.zeros((2, 3, 4))
    with pytest.raises(RuntimeError) as want:
        F.layer_norm(torch.tensor(x), (3,))
    with pytest.raises(ValueError) as got:
        O.ln_forward(x, (3,))
    assert str(got.value) == str(want.value)
