"""The embedding oracle (tests/embedding_oracle.py) against torch's CPU F.embedding and its autograd: the forward exact;
the weight gradient exact where the gradient values are small integers (every order gives the same sum), and within
an f32 reordering bound otherwise, for uniform, Zipf and all-equal ids (rows split over many slots included), invalid
ids, padding_idx (negative form included) and beta."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import embedding_oracle as E


def torch_grad(v, e, ids, g, padding_idx=None):
    """torch's weight gradient, with the invalid ids' positions dropped (torch rejects them)"""
    k = E.keys(ids, v)
    ok = k < v
    w = torch.zeros(v, e, dtype=torch.float64, requires_grad=True)
    y = F.embedding(torch.from_numpy(k[ok]), w, padding_idx=padding_idx)
    y.backward(torch.from_numpy(np.asarray(g, np.float64).reshape(-1, e)[ok]))
    return w.grad.numpy()


def reorder_bound(v, e, ids, g):
    """|f32 sum in any order - exact sum| <= (count - 1) * 2^-24 * sum |g| per row, doubled for the slot partials"""
    k = E.keys(ids, v)
    absg = np.abs(np.asarray(g, np.float64).reshape(-1, e))
    cnt = np.bincount(k[k < v], minlength=v)[:v]
    s = np.zeros((v, e))
    np.add.at(s, k[k < v], absg[k < v])
    return 2 * np.maximum(cnt - 1, 0)[:, None] * 2.0 ** -24 * s + 1e-30


def ids_of(kind, rng, n, v):
    if kind == "uniform":
        return rng.integers(0, v, n).astype(np.float32)
    if kind == "zipf":
        return np.minimum(rng.zipf(1.2, n) - 1, v - 1).astype(np.float32)
    if kind == "equal":
        return np.full(n, v // 2, np.float32)
    return rng.permutation(v)[:n].astype(np.float32)   # distinct


def test_forward_is_torch_embedding():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((50, 7)).astype(np.float32)
    ids = rng.integers(0, 50, (3, 4, 5)).astype(np.float32) + np.float32(0.75)   # truncated to the row
    want = F.embedding(torch.from_numpy(np.trunc(ids).astype(np.int64)), torch.from_numpy(w)).numpy()
    got = E.forward(w, ids)
    assert got.shape == (3, 4, 5, 7)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_invalid_ids_read_zero_rows():
    w = np.arange(12, dtype=np.float32).reshape(4, 3) + 1
    ids = np.array([0, -1, 4, np.nan, 3.999, -0.5, np.inf, 2], np.float32)
    y = E.forward(w, ids)
    assert np.array_equal(y[[0, 4, 7]], w[[0, 3, 2]])
    assert not y[[1, 2, 3, 5, 6]].any()
    assert list(E.keys(ids, 4)) == [0, 4, 4, 4, 3, 4, 4, 2]


@pytest.mark.parametrize("kind", ["uniform", "zipf", "equal", "distinct"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 5000])
def test_small_integer_gradients_are_exact(kind, n):
    rng = np.random.default_rng(n)
    v, e = (max(n, 7) if kind == "distinct" else 300), 5
    ids = ids_of(kind, rng, n, v)
    g = rng.integers(-8, 9, (n, e)).astype(np.float32)
    got = E.backward(np.zeros((v, e), np.float32), ids, g, beta=0.0)
    assert np.array_equal(got, torch_grad(v, e, ids, g))


@pytest.mark.parametrize("kind", ["uniform", "zipf", "equal"])
def test_real_gradients_within_the_reordering_bound(kind):
    rng = np.random.default_rng(3)
    v, e, n = 1000, 9, 20000            # the equal row spans 625 slots
    ids = ids_of(kind, rng, n, v)
    g = rng.standard_normal((n, e)).astype(np.float32)
    got = E.backward(np.zeros((v, e), np.float32), ids, g, beta=0.0)
    want = torch_grad(v, e, ids, g)
    assert np.all(np.abs(got - want) <= reorder_bound(v, e, ids, g))


def test_slot_order_of_a_split_row():
    """one row over 3 slots, starting mid-slot: (piece sums in order) added in slot order"""
    v, e = 4, 1
    ids = np.array([0] * 10 + [1] * 70, np.float32)
    g = np.random.default_rng(1).standard_normal((80, e)).astype(np.float32)
    pieces = [g[10:32], g[32:64], g[64:80]]
    want = None
    for p in pieces:
        s = p[0].copy()
        for x in p[1:]:
            s = (s + x).astype(np.float32)
        want = s if want is None else (want + s).astype(np.float32)
    assert np.array_equal(E.row_sums(g, ids, v)[1], want)


@pytest.mark.parametrize("padding_idx", [0, 5, -1, -7])
def test_padding_idx_and_invalid_ids_add_nothing(padding_idx):
    rng = np.random.default_rng(4)
    v, e, n = 7, 4, 300
    ids = rng.integers(-2, v + 2, n).astype(np.float32)
    ids[::17] = np.nan
    g = rng.integers(-4, 5, (n, e)).astype(np.float32)
    pad = padding_idx % v
    got = E.backward(np.zeros((v, e), np.float32), ids, g, padding_idx=pad, beta=0.0)
    assert np.array_equal(got, torch_grad(v, e, ids, g, padding_idx=padding_idx))
    assert not got[pad].any()


@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
def test_beta(beta):
    rng = np.random.default_rng(5)
    v, e, n = 50, 3, 40                 # most rows receive nothing
    ids = rng.integers(0, v, n).astype(np.float32)
    g = rng.integers(-4, 5, (n, e)).astype(np.float32)
    dw0 = rng.integers(-4, 5, (v, e)).astype(np.float32)
    dw0[0, 0] = np.nan                  # beta = 0 never reads dw
    ids[ids == 0] = 1
    got = E.backward(dw0, ids, g, beta=beta)
    want = torch_grad(v, e, ids, g) + (beta * dw0 if beta else 0.0)
    assert np.array_equal(got, want, equal_nan=True)
