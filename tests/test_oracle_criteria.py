"""CPU checks of tests/criteria_oracle.py: the reference's own goldens (tests/golden/tensors_criteria.json), torch's CPU
losses, the Random123 known-answer vectors of Philox4x32-10 and the keep rate of the dropout masks."""
import json
import os

import numpy as np
import pytest

import criteria_oracle as O

F32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tensors_criteria.json")


@pytest.fixture(scope="module")
def goldens():
    with open(GOLDEN) as fh:
        return json.load(fh)


def build(a):
    """an array entry of the fixture as float32"""
    if a["kind"] == "linspace":
        v = np.linspace(a["start"], a["stop"], a["num"], dtype=F32)
        return v.reshape(a["shape"]) if a["shape"] else v
    if a["kind"] in ("from_shape_vec", "new_input", "new_backward_input"):
        return np.asarray(a["values"], F32).reshape(a["shape"])
    if a["kind"] == "zeros":
        return np.zeros(a["shape"], F32)
    if a["kind"] == "ones":
        return np.ones(a["shape"], F32)
    return np.full(a["shape"], a["value"], F32)


def similar(got, want):
    """the reference's are_similar / assert_almost_equals: |got - want| <= 1e-4, relative for large values"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.all(np.abs(got - want) <= 1e-4 * np.maximum(1.0, np.abs(want))), (got, want)


def reference_cases(goldens):
    """(name, x, t, mean, expected loss, expected gradient for seed 1) of every criterion golden"""
    out = []
    for ref, name in (("absolute_error", "mae"), ("bce", "bce")):
        c = goldens[ref]
        for red in ("mean", "sum"):
            f, b = c[f"base_case_{red}"], c[f"base_case_{red}@{84 if red == 'mean' else (101 if ref == 'absolute_error' else 107)}"]
            x, t = build(f["arrays"][0]), build(f["arrays"][1])
            assert np.array_equal(build(b["arrays"][0]), x) and np.array_equal(build(b["arrays"][1]), t)
            grad = build(b["arrays"][2])
            if b["arrays"][2]["kind"] == "from_elem":
                grad = np.full(x.shape, b["arrays"][2]["value"], F32)
            out.append((name, x, t, red == "mean", f["arr0"][-1], grad))
    for red in ("mean", "sum"):
        c = goldens["bce_with_logits"][red]
        t, x = build(c["arrays"][0]), build(c["arrays"][1])
        out.append(("bce_with_logits", x, t, red == "mean", c["arr0"][0], np.asarray(c["vecs"][0], F32).reshape(x.shape)))
        c = goldens["kldiv"][red]
        t = build(c["arrays"][0])
        x = np.log(np.asarray(c["vecs"][0], F32)).reshape(t.shape)
        out.append(("kldiv", x, t, red == "mean", c["arr0"][0], np.asarray(c["vecs"][1], F32).reshape(t.shape)))
    return out


def test_goldens_transcribed(goldens):
    assert set(goldens) == {"dropout", "absolute_error", "bce", "bce_with_logits", "kldiv"}
    vals = {(n, m): (loss, g) for n, _, _, m, loss, g in reference_cases(goldens)}
    assert vals[("mae", True)][0] == 9.0 and vals[("mae", False)][0] == 81.0
    assert vals[("bce", True)][0] == 23.12971 and vals[("bce", False)][0] == 208.16739
    assert vals[("bce", True)][1].ravel()[0] == F32(-932067.56)
    assert vals[("bce_with_logits", True)][0] == 8.0 and vals[("bce_with_logits", False)][0] == 72.0001
    assert vals[("kldiv", True)][0] == 0.153 and vals[("kldiv", False)][0] == 0.306


def test_oracle_reproduces_the_reference_goldens(goldens):
    for name, x, t, mean, loss, grad in reference_cases(goldens):
        similar(O.forward(name, x, t, mean), loss)
        similar(O.backward(name, x, t, 1.0, mean), grad)
    # the mae backward goldens: -1/9 everywhere (Mean) and -1 (Sum)
    mae = [c for c in reference_cases(goldens) if c[0] == "mae"]
    assert np.all(mae[0][5] == F32(-1.0 / 9.0)) or np.allclose(mae[0][5], -1.0 / 9.0)
    assert np.all(mae[1][5] == -1.0)


def test_bce_clamps_and_epsilon():
    """ln clamped at -100 (a finite loss at x in {0, 1}) and the backward's max(., f32::EPSILON): (0 - 1)/2^-23"""
    x = np.array([0.0, 1.0, 0.0, 1.0], F32)
    t = np.array([1.0, 0.0, 0.0, 1.0], F32)
    assert O.forward("bce", x, t, mean=False) == F32(200.0)
    assert np.array_equal(O.backward("bce", x, t, 1.0, mean=False), np.array([-8388608.0, 8388608.0, 0.0, 0.0], F32))


def test_kldiv_zero_target_is_finite():
    """SURVEY.md 8-c defect 9: the reference's t*(ln t - x)*[t > 0] is NaN at t = 0; here the term is 0"""
    t = np.array([[0.0, 1.0]], F32)
    x = np.log(np.array([[0.5, 0.5]], F32))
    assert np.isfinite(O.forward("kldiv", x, t)) and O.forward("kldiv", x, t) == F32(np.log(2.0))


@pytest.mark.parametrize("mean", [True, False])
def test_oracle_matches_torch(mean):
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(3)
    shape = (16, 33)
    red = "mean" if mean else "sum"
    x, t = rng.standard_normal(shape).astype(F32), rng.standard_normal(shape).astype(F32)
    p = rng.uniform(0.02, 0.98, shape).astype(F32)
    tp = rng.uniform(0, 1, shape).astype(F32)
    logits = (3 * rng.standard_normal(shape)).astype(F32)
    dist = rng.uniform(0.01, 1, shape).astype(F32)
    dist[:, :3] = 0   # zero targets
    dist /= dist.sum(axis=1, keepdims=True)
    logq = np.log(rng.dirichlet(np.ones(shape[1]), size=shape[0]).astype(F32) + F32(1e-6)).astype(F32)

    def check(name, xi, ti, fn):
        xt = torch.tensor(xi, requires_grad=True)
        loss = fn(xt, torch.tensor(ti))
        loss.backward()
        assert np.isclose(O.forward(name, xi, ti, mean), loss.item(), rtol=2e-6, atol=1e-6), name
        np.testing.assert_allclose(O.backward(name, xi, ti, 1.0, mean), xt.grad.numpy(), rtol=2e-6, atol=1e-7,
                                   err_msg=name)

    check("mae", x, t, lambda a, b: F.l1_loss(a, b, reduction=red))
    check("bce", p, tp, lambda a, b: F.binary_cross_entropy(a, b, reduction=red))
    check("bce_with_logits", logits, tp, lambda a, b: F.binary_cross_entropy_with_logits(a, b, reduction=red))
    check("kldiv", logq, dist, lambda a, b: F.kl_div(a, b, reduction="batchmean" if mean else "sum"))


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10"""
    kats = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
            ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
            ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
             (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kats:
        got = O.philox4x32_10(np.array([ctr], np.uint32), key)[0]
        assert tuple(int(v) for v in got) == want


def test_dropout_counter_layout():
    """element e takes word e%4 of the block at counter (e/4, call): the words of elements past 2^34 use the high
    counter word, and the call id enters words 2-3"""
    seed, call = 0x0123456789ABCDEF, (7 << 32) + 5
    e = np.array([0, 1, 2, 3, (1 << 34) + 6], np.int64)
    blk = O.philox4x32_10(np.array([[0, 0, 5, 7]], np.uint32), (0x89ABCDEF, 0x01234567))[0]
    assert np.array_equal(O.dropout_words(seed, call, e[:4]), blk)
    hi = O.philox4x32_10(np.array([[1, 1, 5, 7]], np.uint32), (0x89ABCDEF, 0x01234567))[0]
    assert O.dropout_words(seed, call, e[4:])[0] == hi[2]


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_dropout_keep_rate_is_binomial(p):
    n = 1 << 20
    for seed, call in ((1, 0), (2**63 + 12345, 3), (99, 2**40)):
        k = int(O.dropout_keep(seed, call, n, p).sum())
        q = float(O.keep_prob(p))
        assert abs(k - n * q) <= 6 * np.sqrt(n * q * (1 - q)), (seed, call, k)
    assert not np.array_equal(O.dropout_keep(1, 0, 4096, p), O.dropout_keep(1, 1, 4096, p))


def test_dropout_goldens(goldens):
    """dropout/test.rs: p = 0 is the identity, p = 1 zeros, p = 0.5 bounded by 2*linspace(1, 9); bad p are rejected"""
    d = goldens["dropout"]
    x = build(d["base_case"]["arrays"][0])
    bound = build(d["base_case"]["arrays"][3])
    assert d["base_case"]["probabilities"] == [0.5]
    for call in range(16):
        y = O.dropout_forward(x, O.dropout_keep(7, call, x.size, 0.5), 0.5)
        assert np.all(y <= bound) and set(np.unique(y / x)) <= {0.0, 2.0}
    assert np.array_equal(O.dropout_forward(x, np.ones(x.size, bool), d["zero_probability"]["probabilities"][0]),
                          build(d["zero_probability"]["arrays"][3]))
    assert not O.dropout_keep(7, 0, x.size, d["one_probability"]["probabilities"][0]).any()
    g = build(d["one_probability@133"]["arrays"][0])
    assert np.array_equal(O.dropout_backward(g, np.zeros(g.size, bool), 1.0), np.zeros_like(g))
    assert [d["too_low_probability"]["probabilities"][0], d["too_high_probability"]["probabilities"][0]] == [-0.5, 1.5]
    keep = O.dropout_keep(3, 1, 1000, 0.25)
    assert np.array_equal(O.unpack_mask(O.pack_mask(keep), 1000), keep)
