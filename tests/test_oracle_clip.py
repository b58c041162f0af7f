"""The clipping oracle (tests/clip_oracle.py) against torch CPU's get_total_norm, clip_grads_with_norm_,
clip_grad_norm_ and clip_grad_value_ on f32 gradients: the total within the rounding of torch's norm of per-tensor
norms, and the scaled and clamped gradients to the bit, NaN and infinity included."""
import numpy as np
import pytest
import torch
from torch.nn.utils import clip_grad_norm_, clip_grad_value_, clip_grads_with_norm_, get_total_norm

import clip_oracle as O

NORMS = [1.0, 2.0, 3.0, 0.5, float("inf")]


def _grads(seed, sizes=(7, 0, 130, 1, 4096, 0, 33), scale=1.0):
    rng = np.random.default_rng(seed)
    return [(rng.standard_normal(n) * scale).astype(np.float32) for n in sizes]


def _params(grads):
    ps = []
    for g in grads:
        p = torch.nn.Parameter(torch.zeros(g.shape))
        p.grad = torch.from_numpy(g.copy())
        ps.append(p)
    return ps


def _same(a, b):
    """bitwise equal, any NaN equal to any NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape
    nan = np.isnan(a)
    assert np.array_equal(nan, np.isnan(b))
    assert np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


def _close(got, want, rtol=2e-6):
    if np.isnan(want) or np.isinf(want):
        assert (np.isnan(got) and np.isnan(want)) or got == want, (got, want)
    else:
        assert abs(got - want) <= rtol * abs(want) + 1e-30, (got, want)


def _special(seed):
    gs = _grads(seed)
    gs[2][5] = np.nan
    gs[4][17] = np.inf
    gs[6][0] = -np.inf
    return gs


CASES = {
    "normal": lambda: _grads(0),
    "tiny": lambda: _grads(1, scale=1e-10),      # |v|^p stays a normal f32 for every p here (overflow of the
    "huge": lambda: _grads(2, scale=1e10),       # f32 terms is where torch's f32 path overflows too)
    "nan": lambda: [g if i != 2 else np.where(np.arange(g.size) == 5, np.nan, g).astype(np.float32)
                    for i, g in enumerate(_grads(3))],
    "pos_inf": lambda: [g if i != 4 else np.where(np.arange(g.size) == 17, np.inf, g).astype(np.float32)
                        for i, g in enumerate(_grads(4))],
    "neg_inf": lambda: [g if i != 6 else np.where(np.arange(g.size) == 0, -np.inf, g).astype(np.float32)
                        for i, g in enumerate(_grads(5))],
    "nan_and_inf": lambda: _special(6),
    "all_empty": lambda: [np.zeros(0, np.float32)] * 3,
}


@pytest.mark.parametrize("p", NORMS, ids=str)
@pytest.mark.parametrize("case", sorted(CASES))
def test_total_norm(case, p):
    grads = CASES[case]()
    if np.isinf(p):   # torch has no inf-norm of an empty tensor; here an empty tensor adds nothing, as for other p
        with pytest.raises(RuntimeError, match="empty tensor"):
            get_total_norm([torch.from_numpy(g) for g in grads], p)
        _close(O.total_norm(grads, p), O.total_norm([g for g in grads if g.size], p), rtol=0.0)
        grads = [g for g in grads if g.size]
    want = float(get_total_norm([torch.from_numpy(g) for g in grads], p))
    _close(O.total_norm(grads, p), want, rtol=2e-6 if p != 0.5 else 2e-5)


def test_empty_list_has_norm_zero():
    assert float(get_total_norm([], 2.0)) == 0.0 and O.total_norm([], 2.0) == 0.0
    assert float(clip_grad_norm_([], 1.0)) == 0.0


@pytest.mark.parametrize("bad", [0.0, -1.0, float("-inf"), float("nan")])
def test_rejected_norm_types(bad):
    with pytest.raises(ValueError):
        O.total_norm(_grads(0), bad)


@pytest.mark.parametrize("p", NORMS, ids=str)
@pytest.mark.parametrize("where", ["below", "at", "above", "zero"])
def test_clip_grad_norm_scaling_is_bit_exact(p, where):
    grads = _grads(7)
    total = O.total_norm(grads, p)
    max_norm = {"below": 0.25 * total, "at": total, "above": 4.0 * total, "zero": 0.0}[where]
    ps = _params([g for g in grads if g.size] if np.isinf(p) else grads)
    t_total = clip_grad_norm_(ps, max_norm, norm_type=p)
    _close(O.total_norm(grads, p), float(t_total), rtol=2e-6 if p != 0.5 else 2e-5)
    c = O.coefficient(float(t_total), max_norm)
    assert (c == 1.0) == (where == "above")
    for g, q in zip([g for g in grads if g.size] if np.isinf(p) else grads, ps):
        _same(q.grad.numpy(), O.scale(g, c))


@pytest.mark.parametrize("case", ["nan", "pos_inf", "neg_inf", "nan_and_inf", "huge", "tiny"])
def test_clip_grads_with_norm_special_totals(case):
    grads = CASES[case]()
    for total in (O.total_norm(grads), 1.5, 0.0):
        ps = _params(grads)
        clip_grads_with_norm_(ps, 1.0, torch.tensor(total, dtype=torch.float32))
        c = O.coefficient(total, 1.0)
        for g, q in zip(grads, ps):
            _same(q.grad.numpy(), O.scale(g, c))


def test_nonfinite_totals_give_torch_coefficients():
    assert np.isnan(O.coefficient(float("nan"), 1.0))
    assert O.coefficient(float("inf"), 1.0) == 0.0
    _same(O.scale(np.array([1.0, np.inf, -2.0], np.float32), O.coefficient(float("inf"), 1.0)),
          np.array([0.0, np.nan, -0.0], np.float32))


@pytest.mark.parametrize("clip_value", [0.5, 0.0, -0.3, 1e-30, 3.0])
@pytest.mark.parametrize("case", ["normal", "nan_and_inf"])
def test_clip_grad_value_is_bit_exact(case, clip_value):
    grads = CASES[case]()
    ps = _params(grads)
    clip_grad_value_(ps, clip_value)
    for g, q in zip(grads, ps):
        _same(q.grad.numpy(), O.clamp(g, clip_value))


@pytest.mark.parametrize("k", [0.5, 0.25, 0.125])
def test_grad_scale_of_a_power_of_two_world(k):
    """clipping world*G with k = 1/world gives world * (the clipped G), bit for bit"""
    grads = _grads(9)
    world = F = 1.0 / k
    summed = [(g * np.float32(F)).astype(np.float32) for g in grads]
    total = O.total_norm(summed, 2.0, k)
    assert total == O.total_norm(grads, 2.0)
    c = O.coefficient(total, 0.3)
    for g, s in zip(grads, summed):
        _same(O.scale(s, c), (O.scale(g, c) * np.float32(world)).astype(np.float32))
    for g, s in zip(grads, summed):
        _same(O.clamp(s, 0.3, k), (O.clamp(g, 0.3) * np.float32(world)).astype(np.float32))
