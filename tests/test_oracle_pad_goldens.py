"""The oracle's padding against the reference's own padded arrays (tests/golden/tensors_pad.json, transcribed from
node/pad/{reflective,replicative,constant,zero}/test.rs by make_goldens_pad.py): pad_mode_forward of each `Array::range`
input reproduces the golden bit for bit, in float32 as the reference computes it and in float64."""
import json
import os

import numpy as np
import pytest

import oracle as O

GOLDENS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tensors_pad.json")))
CASES = [(mode, name) for mode, cases in GOLDENS.items() for name in cases]


def golden_case(mode, name):
    """(base, padding, oracle mode, fill, expected) of one golden"""
    c = GOLDENS[mode][name]
    start, stop, step = c["base_range"]
    base = np.arange(start, stop, step).reshape(c["base_shape"])
    om = "constant" if mode == "zero" else mode
    return base, tuple(c["padding"]), om, c.get("fill", 0.0), np.asarray(c["expected"], np.float64)


def test_every_golden_is_transcribed():
    assert sorted(CASES) == sorted([(m, f"test_{d}d") for m in ("reflective", "replicative") for d in (1, 2, 3)]
                                   + [("constant", "test"), ("zero", "test")])
    for mode, name in CASES:
        c = GOLDENS[mode][name]
        assert np.asarray(c["expected"]).shape == tuple(c["padded_shape"]), (mode, name)
        assert c["padded_shape"] == [s + 2 * p for s, p in zip(c["base_shape"], c["padding"])], (mode, name)
    assert GOLDENS["constant"]["test"]["fill"] == 8.0


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("mode,name", CASES)
def test_pad_mode_forward_reproduces_the_golden(mode, name, dtype):
    base, pad, om, fill, want = golden_case(mode, name)
    got = O.pad_mode_forward(base.astype(dtype), pad, om, fill)
    assert got.dtype == dtype and got.shape == want.shape
    assert np.array_equal(got, want.astype(dtype)), (mode, name)


@pytest.mark.parametrize("mode,name", CASES)
def test_pad_mode_forward_with_leading_axes(mode, name):
    """the (N, C, ...) layout the layers use: every plane is padded alone"""
    base, pad, om, fill, want = golden_case(mode, name)
    x = np.stack([base, -base, 2 * base])[None]
    got = O.pad_mode_forward(x, pad, om, fill)
    scale = np.array([1.0, -1.0, 2.0]).reshape((1, 3) + (1,) * len(pad))
    inner = tuple(slice(p, p + s) for p, s in zip(pad, base.shape))
    border = np.ones(want.shape, bool)
    border[inner] = False
    if om == "constant":   # the fill does not scale with the plane
        assert np.array_equal(got[0][:, border], np.full((3, int(border.sum())), fill)), (mode, name)
        assert np.array_equal(got[0][(slice(None),) + inner], x[0]), (mode, name)
    else:
        assert np.array_equal(got, want[None, None] * scale), (mode, name)
