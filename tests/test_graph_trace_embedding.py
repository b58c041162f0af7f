"""The kernel-ABI calls of nkg_embedding and nkg_reshape, over the recording stub of tests/graph_trace.py: one forward
call per pass and one backward call into the weight's gradient (beta 0 at its first write, 1 when a tied Linear head
wrote first), none for a frozen weight; errors record nothing; reshape records no call and shares the gradient."""
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_embedding"))))


def embedding(g, ids, w, pad=-1):
    return g.call("nkg_embedding", ids.h, w.h, pad)


def reshape(g, x, shape):
    return g.call("nkg_reshape", x.h, len(shape), T._i64s(shape))


def names(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def args_of(lines, name):
    return [l[len(name) + 1:-1].split(", ") for l in lines if l.startswith(name + "(")]


@pytest.mark.parametrize("grad_dtype", [None, F32])
def test_one_forward_call_and_one_backward_call_per_pass(graph, grad_dtype):
    def scenario(g):
        ids = g.leaf((5, 7), F32)
        w = g.param((100, 16), BF16, grad_dtype)
        y = embedding(g, ids, w, 3)
        y.describe("y")
        loss = y.sum()
        loss.forward()
        for r in range(2):
            g.note("backward %d" % r)
            loss.backward(1.0)
        w.grad_ptr()

    lines = graph.run(scenario)
    assert lines[-1].endswith("never freed: []"), lines[-1]
    calls = [n for n in names(lines) if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free", "nk_fill", "nk_sum_bwd")]
    assert calls == ["y", "nk_embedding_fwd", "nk_sum_fwd", "backward 0", "nk_embedding_bwd", "backward 1",
                     "nk_embedding_bwd", "grad"]
    assert "y: diff=1 shape=[5, 7, 16] dtype=%d" % BF16 in "\n".join(lines)
    f = args_of(lines, "nk_embedding_fwd")[0]
    # y, w, ids, ids_dtype, n, v, e, dtype
    assert f[3:] == [str(F32), "35", "100", "16", str(BF16)]
    b = args_of(lines, "nk_embedding_bwd")
    gd = BF16 if grad_dtype is None else grad_dtype
    # dw, dw_dtype, ids, ids_dtype, g, g_dtype, n, v, e, padding_idx, beta
    assert [a[1] for a in b] == [str(gd)] * 2 and [a[5] for a in b] == [str(BF16)] * 2
    assert [a[6:10] for a in b] == [["35", "100", "16", "3"]] * 2
    assert [a[-1] for a in b] == ["0", "1"]
    assert b[0][2] == f[2]                              # the forward's ids feed the backward


def test_tied_head_writes_first(graph):
    """the head's dW GEMM runs before the embedding's backward: the embedding accumulates with beta 1"""
    def scenario(g):
        ids = g.leaf((6,), F32)
        w = g.param((50, 8), F32)
        loss = embedding(g, ids, w).mm_t(w).sum()
        loss.forward()
        loss.backward(1.0)

    lines = graph.run(scenario)
    b = args_of(lines, "nk_embedding_bwd")
    assert len(b) == 1 and b[0][-1] == "1"
    assert names(lines).index("nk_embedding_bwd") > max(i for i, n in enumerate(names(lines)) if n == "nk_gemm_bias_act")


def test_frozen_weight_has_no_backward(graph):
    def scenario(g):
        ids = g.leaf((4,), F32)
        w = g.leaf((10, 3), F32)
        x = g.param((4, 3), F32)
        loss = (embedding(g, ids, w) * x).sum()
        loss.describe("loss")
        loss.forward()
        loss.backward(1.0)

    lines = graph.run(scenario)
    assert "nk_embedding_fwd" in names(lines) and "nk_embedding_bwd" not in names(lines)


ERRORS = [
    (lambda g, ids, w: embedding(g, ids.requires_grad(), w), "ids must not be differentiable"),
    (lambda g, ids, w: embedding(g, ids, g.param((20,), F32)), "weight must be 2-D"),
    (lambda g, ids, w: embedding(g, ids, w, 20), "padding_idx 20 outside"),
    (lambda g, ids, w: embedding(g, ids, w, -2), "padding_idx -2 outside"),
    (lambda g, ids, w: embedding(g, g.leaf((4,), BF16), g.param((257, 3), F32)), "bf16 ids"),
    (lambda g, ids, w: embedding(g, g.leaf((1, 1, 1, 1, 1, 1), F32), w), "more than 6 dimensions"),
    (lambda g, ids, w: g.call("nkg_embedding", ids.h, None, -1), "NULL"),
]


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_invalid_arguments_fail_and_record_nothing(graph, case):
    op, msg = ERRORS[case]

    def scenario(g):
        ids = g.leaf((4,), F32)
        w = g.param((20, 3), F32)
        w.describe("before")
        g.expect_error(op, g, ids, w)
        w.describe("after")

    lines = graph.run(scenario)
    err = [l for l in lines if l.startswith("error ")]
    assert len(err) == 1 and msg in err[0], err
    assert not any(l.startswith("nk_embedding") for l in lines)
    before = [l for l in lines if l.startswith("before")][0]
    assert before.replace("before", "after") in lines


def test_reshape_is_a_view_sharing_the_gradient(graph):
    def scenario(g):
        x = g.param((3, 4, 5), F32)
        y = reshape(g, x, (12, 5))
        y.describe("y")
        loss = y.sum()
        loss.forward()
        loss.backward(1.0)
        x.grad_ptr("x grad")
        y.grad_ptr("y grad")
        g.expect_error(reshape, g, x, (7, 8))

    lines = graph.run(scenario)
    assert "y: diff=1 shape=[12, 5] dtype=0 grad_dtype=0 history=0 backward_history=0" in lines
    xg = [l for l in lines if l.startswith("x grad")][0].split(" -> ")[1]
    yg = [l for l in lines if l.startswith("y grad")][0].split(" -> ")[1]
    assert xg == yg
    calls = [n for n in names(lines) if n.startswith("nk_") and n not in ("nk_alloc", "nk_alloc_uninit", "nk_free",
                                                                          "nk_fill")]
    assert calls == ["nk_sum_fwd", "nk_sum_bwd"]     # reshape itself launches nothing
    assert any(l.startswith("error -1 shape '(7, 8)' is invalid for input of size 60") for l in lines)
