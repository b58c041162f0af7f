"""The kernel-ABI calls of nkg_cross_entropy, over the recording stub of tests/graph_trace.py: one nk_cross_entropy_fwd
per forward and one nk_cross_entropy_bwd per backward into the input's gradient (beta 0 at its first write, then 1),
no log_softmax or nll call, the forward's saved lse and denominator feeding the backward, no backward for a frozen
input, and nothing recorded by an invalid call."""
import re

import numpy as np
import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
MEAN, SUM = 0, 1


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_cross_entropy"))))


def ce(g, x, t, w=None, reduction=MEAN, ignore_index=-100, eps=0.0):
    return g.call("nkg_cross_entropy", x.h, t.h, w.h if w is not None else None, reduction, ignore_index, eps)


def names(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def args_of(lines, name):
    return [l[len(name) + 1:-1].split(", ") for l in lines if l.startswith(name + "(")]


CASES = {
    # x shape, target shape, x dtype, gradient dtype, target dtype, weighted, reduction, ignore_index, label_smoothing
    "rows_f32_mean": ((6, 10), (6,), F32, None, F32, False, MEAN, -100, 0.0),
    "rows_bf16_f32grad_weighted_sum": ((6, 10), (6,), BF16, F32, BF16, True, SUM, 0, 0.1),
    "spatial_f32_mean": ((2, 5, 3, 4), (2, 3, 4), F32, None, F32, True, MEAN, 3, 1.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_one_forward_call_and_one_backward_call_per_pass(graph, case):
    xs, ts, xd, gd, td, weighted, red, ig, eps = CASES[case]

    def scenario(g):
        x = g.param(xs, xd, gd)
        t = g.leaf(ts, td)
        w = g.leaf((xs[1],), F32) if weighted else None
        loss = ce(g, x, t, w, red, ig, eps)
        loss.describe("loss")
        loss.forward()
        for r in range(2):
            g.note("backward %d" % r)
            loss.backward(1.0)
        x.grad_ptr()

    lines = graph.run(scenario)
    assert lines[-1].endswith("never freed: []"), lines[-1]
    calls = [n for n in names(lines) if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free", "nk_fill")]
    assert calls == ["loss", "nk_cross_entropy_fwd", "backward 0", "nk_cross_entropy_bwd", "backward 1",
                     "nk_cross_entropy_bwd", "grad"]
    assert not any(l.startswith(("nk_log_softmax", "nk_nll", "nk_softmax")) for l in lines)
    assert "loss: diff=1 shape=[] dtype=%d" % F32 in "\n".join(lines)
    n, c = xs[0], xs[1]
    s = 1
    for d in xs[2:]:
        s *= d
    f = args_of(lines, "nk_cross_entropy_fwd")
    assert len(f) == 1
    f = f[0]
    # loss, lse, denom, x, dtype, target, target_dtype, weight, n, c, s, ignore_index, label_smoothing, mean
    assert f[4] == str(xd) and f[6] == str(td) and (f[7] != "0") == weighted
    assert f[8:] == [str(n), str(c), str(s), str(ig), "%.9g" % float(np.float32(eps)), str(int(red == MEAN))]
    b = args_of(lines, "nk_cross_entropy_bwd")
    # dx, dx_dtype, x, dtype, target, target_dtype, weight, lse, denom, g, n, c, s, ignore_index, label_smoothing,
    # mean, beta
    assert [a[-1] for a in b] == ["0", "1"]
    want_gd = xd if gd is None else gd
    for a in b:
        assert a[1] == str(want_gd) and a[2] == f[3] and a[3] == str(xd) and a[4] == f[5] and a[6] == f[7]
        assert a[7] == f[1] and a[8] == f[2]        # the forward's saved lse and denominator feed the backward
        assert a[10:16] == f[8:14]


def test_frozen_input_records_no_backward(graph):
    def scenario(g):
        x = g.leaf((4, 7), F32)
        t = g.leaf((4,), F32)
        p = g.param((4, 7), F32)
        loss = ce(g, x, t) + (p * x).sum()
        loss.forward()
        loss.backward(1.0)

    lines = graph.run(scenario)
    assert "nk_cross_entropy_fwd" in names(lines) and "nk_cross_entropy_bwd" not in names(lines)


ERRORS = [
    (lambda g, x, t, w: ce(g, x, g.leaf((5,), F32)), "input must be (N, C, d1, ..., dk)"),
    (lambda g, x, t, w: ce(g, g.param((4, 7, 3), F32), g.leaf((4, 2), F32)), "input must be (N, C, d1, ..., dk)"),
    (lambda g, x, t, w: ce(g, g.param((4,), F32), g.leaf((4,), F32)), "input must be (N, C, d1, ..., dk)"),
    (lambda g, x, t, w: ce(g, x, t, g.leaf((6,), F32)), "weight must be an f32 tensor of shape (7,)"),
    (lambda g, x, t, w: ce(g, x, t, g.leaf((7,), BF16)), "weight must be an f32 tensor"),
    (lambda g, x, t, w: ce(g, x, t, g.param((7,), F32)), "the weight must not be differentiable"),
    (lambda g, x, t, w: ce(g, x, t.requires_grad()), "the target must not be differentiable"),
    (lambda g, x, t, w: ce(g, x, t, w, eps=-0.1), "label_smoothing must be between 0.0 and 1.0"),
    (lambda g, x, t, w: ce(g, x, t, w, eps=1.5), "label_smoothing must be between 0.0 and 1.0"),
    (lambda g, x, t, w: ce(g, x, t, w, eps=float("nan")), "label_smoothing must be between 0.0 and 1.0"),
    (lambda g, x, t, w: ce(g, g.param((4, 257), F32), g.leaf((4,), BF16)), "a bf16 target cannot hold class ids"),
    (lambda g, x, t, w: ce(g, x, g.leaf((4,), F32, g.other_ctx)), "operands live on different devices"),
    (lambda g, x, t, w: ce(g, x, t, g.leaf((7,), F32, g.other_ctx)), "operands live on different devices"),
    (lambda g, x, t, w: ce(g, x, t, w, reduction=2), "unknown reduction 2"),
    (lambda g, x, t, w: g.call("nkg_cross_entropy", x.h, None, None, 0, -100, 0.0), "NULL"),
]


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_invalid_arguments_fail_and_record_nothing(graph, case):
    op, msg = ERRORS[case]

    def scenario(g):
        x = g.param((4, 7), F32)
        t = g.leaf((4,), F32)
        w = g.leaf((7,), F32)
        x.describe("before")
        g.expect_error(op, g, x, t, w)
        x.describe("after")

    lines = graph.run(scenario)
    err = [l for l in lines if l.startswith("error ")]
    assert len(err) == 1 and msg in err[0] and err[0].startswith("error -1 "), err
    assert not any(l.startswith("nk_cross_entropy") for l in lines)
    before = [l for l in lines if l.startswith("before")][0]
    assert before.replace("before", "after") in lines
