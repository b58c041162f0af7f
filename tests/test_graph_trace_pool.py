"""The kernel-ABI calls of the pooling nodes (nkg_max_pool / nkg_avg_pool / nkg_adaptive_avg_pool), over the recording
stub of tests/graph_trace.py: one forward call per node; the max pool's index buffer only for a differentiable operand
(NULL otherwise); one backward call per pass into the operand's gradient, beta 0 and then 1 over repeated passes; every
invalid argument fails with its message and records nothing."""
import ctypes as C
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
POOL = ("nk_max_pool_nd_fwd", "nk_max_pool_nd_bwd", "nk_avg_pool_nd_fwd", "nk_avg_pool_nd_bwd",
        "nk_adaptive_avg_pool_nd_fwd", "nk_adaptive_avg_pool_nd_bwd")
# the pooling entry points' shape arguments are host arrays of nsp entries
T.HOST_ARRAYS.update({(f, p): "nsp" for f in POOL for p in ("in_sp", "out_sp", "k", "stride", "pad", "dilation")})


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_pool"))))


def max_pool(g, x, k, s, p, d, ceil=0):
    return g.call("nkg_max_pool", x.h, len(k), T._i64s(k), T._i64s(s), T._i64s(p), T._i64s(d), ceil)


def avg_pool(g, x, k, s, p, ceil=0, include_pad=1):
    return g.call("nkg_avg_pool", x.h, len(k), T._i64s(k), T._i64s(s), T._i64s(p), ceil, include_pad)


def adaptive(g, x, o):
    return g.call("nkg_adaptive_avg_pool", x.h, len(o), T._i64s(o))


def names(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def args_of(lines, name):
    return [l[len(name) + 1:-1].split(", ") for l in lines if l.startswith(name + "(")]


OPS = {
    "max": ((2, 3, 9, 10), lambda g, x: max_pool(g, x, (3, 3), (2, 2), (1, 1), (1, 1), 1), (2, 3, 5, 6)),
    "avg": ((2, 4, 6, 5, 7), lambda g, x: avg_pool(g, x, (2, 2, 3), (2, 1, 2), (1, 0, 1), 0, 0), (2, 4, 4, 4, 4)),
    "adaptive": ((3, 2, 11), lambda g, x: adaptive(g, x, (4,)), (3, 2, 4)),
}


@pytest.mark.parametrize("grad_dtype", [None, F32])
@pytest.mark.parametrize("op", sorted(OPS))
def test_one_forward_call_and_one_backward_call_per_pass(graph, op, grad_dtype):
    xs, build, ys = OPS[op]
    fwd, bwd = "nk_%s_pool_nd_fwd" % (op if op != "adaptive" else "adaptive_avg"), None
    bwd = fwd[:-3] + "bwd"

    def scenario(g):
        x = g.param(xs, BF16, grad_dtype)
        y = build(g, x)
        y.describe("y")
        loss = y.sum()
        loss.forward()
        for r in range(3):
            g.note("backward %d" % r)
            loss.backward(1.0)
        x.grad_ptr()

    lines = graph.run(scenario)
    assert lines[-1].endswith("never freed: []"), lines[-1]
    calls = [n for n in names(lines) if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free", "nk_fill", "nk_sum_bwd")]
    assert calls == ["y", fwd, "nk_sum_fwd", "backward 0", bwd, "backward 1", bwd, "backward 2", bwd, "grad"]
    assert "y: diff=1 shape=%s dtype=%d" % (list(ys), BF16) in "\n".join(lines)
    f = args_of(lines, fwd)[0]
    b = args_of(lines, bwd)
    # y, [idx,] x, planes, nsp, in_sp, out_sp, ...
    off = 3 if op == "max" else 2
    assert f[off:off + 4] == [str(xs[0] * xs[1]), str(len(xs) - 2), str(list(xs[2:])).replace(" ", ""),
                              str(list(ys[2:])).replace(" ", "")]
    gd = BF16 if grad_dtype is None else grad_dtype
    # dx, dx_dtype, g, g_dtype, ...; beta is last: 0 on the first pass, then accumulating
    assert [a[1] for a in b] == [str(gd)] * 3 and [a[3] for a in b] == [str(BF16)] * 3
    assert [a[-1] for a in b] == ["0", "1", "1"]
    assert len({a[0] for a in b}) == 1
    if op == "max":
        assert f[1] != "0" and all(a[4] == f[1] for a in b)     # the forward's indices feed every backward
        allocs = [l for l in lines if l.startswith("nk_alloc")]
        assert allocs[1].startswith("nk_alloc_uninit(%d) = %s" % (4 * 2 * 3 * 5 * 6, f[1]))   # built with the node


def test_max_pool_of_a_constant_keeps_no_indices(graph):
    def scenario(g):
        x = g.leaf((2, 3, 8, 8))
        y = max_pool(g, x, (2, 2), (2, 2), (0, 0), (1, 1))
        y.describe("y")
        y.forward()

    lines = graph.run(scenario)
    assert names(lines) == ["nk_alloc", "y", "nk_alloc_uninit", "nk_max_pool_nd_fwd"]   # no index buffer
    assert args_of(lines, "nk_max_pool_nd_fwd")[0][1] == "0"


def test_two_pools_in_a_chain(graph):
    """max pool into global average pool: the gradient of the middle tensor feeds the max pool's backward"""
    def scenario(g):
        x = g.param((2, 4, 8, 8))
        z = adaptive(g, max_pool(g, x, (2, 2), (2, 2), (0, 0), (1, 1)), (1, 1))
        loss = z.sum()
        loss.forward()
        loss.backward(1.0)

    calls = [n for n in names(graph.run(scenario)) if n.startswith("nk_") and "pool" in n]
    assert calls == ["nk_max_pool_nd_fwd", "nk_adaptive_avg_pool_nd_fwd", "nk_adaptive_avg_pool_nd_bwd",
                     "nk_max_pool_nd_bwd"]


ERRORS = [
    ("max_pool", lambda g, x: max_pool(g, x, (0, 2), (1, 1), (0, 0), (1, 1)), "kernel size, stride and dilation"),
    ("max_pool", lambda g, x: max_pool(g, x, (2, 2), (0, 1), (0, 0), (1, 1)), "kernel size, stride and dilation"),
    ("max_pool", lambda g, x: max_pool(g, x, (2, 2), (1, 1), (0, 0), (1, 0)), "kernel size, stride and dilation"),
    ("max_pool", lambda g, x: max_pool(g, x, (3, 3), (1, 1), (2, 0), (1, 1)), "at most half the kernel size"),
    ("max_pool", lambda g, x: max_pool(g, x, (3, 3), (1, 1), (-1, 0), (1, 1)), "at most half the kernel size"),
    ("max_pool", lambda g, x: max_pool(g, x, (5, 2), (1, 1), (0, 0), (3, 1)), "output size would be"),
    ("max_pool", lambda g, x: max_pool(g, x, (2,), (1,), (0,), (1,)), "sample dimensions"),
    ("avg_pool", lambda g, x: avg_pool(g, x, (2, 4), (1, 1), (0, 3)), "at most half the kernel size"),
    ("avg_pool", lambda g, x: avg_pool(g, x, (9, 2), (1, 1), (0, 0)), "output size would be"),
    ("avg_pool", lambda g, x: avg_pool(g, x, (2, 2, 2, 2), (1,) * 4, (0,) * 4), "sample dimensions"),
    ("adaptive_avg_pool", lambda g, x: adaptive(g, x, (0, 2)), "sizes must be >= 1"),
    ("adaptive_avg_pool", lambda g, x: adaptive(g, x, (2, 2, 2)), "sample dimensions"),
    ("max_pool", lambda g, x: g.call("nkg_max_pool", x.h, 2, None, T._i64s((1, 1)), T._i64s((0, 0)),
                                     T._i64s((1, 1)), 0), "NULL"),
    ("avg_pool", lambda g, x: g.call("nkg_avg_pool", None, 2, T._i64s((1, 1)), T._i64s((1, 1)), T._i64s((0, 0)),
                                     0, 1), "NULL"),
    ("adaptive_avg_pool", lambda g, x: g.call("nkg_adaptive_avg_pool", x.h, 2, None), "NULL"),
]


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_invalid_arguments_fail_and_record_nothing(graph, case):
    who, op, msg = ERRORS[case]

    def scenario(g):
        x = g.param((2, 3, 7, 6))
        x.describe("before")
        g.expect_error(op, g, x)
        x.describe("after")

    lines = graph.run(scenario)[1:]                         # after the operand's allocation
    assert len(lines) == 4, lines
    assert lines[1].startswith("error -1 %s: " % who) and msg in lines[1], lines[1]
    assert lines[0].replace("before", "after") == lines[2]
