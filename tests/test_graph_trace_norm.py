"""The kernel-ABI calls of the normalization nodes (nkg_batch_norm / nkg_layer_norm), over the recording stub of
tests/graph_trace.py: one forward call and one backward call per pass, in train and in eval; beta 0 and then 1 over
repeated passes for dx, dw and db; NULL for an absent weight, bias or running statistic and for the dx of an operand
that is not differentiable; the backward follows the forward's statistics after the status flips; every invalid
argument fails with its message and records nothing.  (Kernel launches per call are pinned in tests/test_gpu_norm.py.)"""
import ctypes as C
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
SKIP = ("nk_alloc", "nk_alloc_uninit", "nk_free", "nk_fill", "nk_sum_bwd", "nk_sum_fwd", "nk_memset0")


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_norm"))))


def status(g, train):
    h = C.c_void_p()
    g.ck(g.lib.nkg_status_create(int(train), C.byref(h)))
    return h


def batch_norm(g, x, w, b, rm, rv, st, momentum=0.1, eps=1e-5):
    h = lambda v: v.h if v is not None else None
    return g.call("nkg_batch_norm", x.h, h(w), h(b), h(rm), h(rv), st, momentum, eps)


def layer_norm(g, x, k, w, b, eps=1e-5):
    h = lambda v: v.h if v is not None else None
    return g.call("nkg_layer_norm", x.h, k, h(w), h(b), eps)


def names(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def calls(lines):
    return [n for n in names(lines) if n not in SKIP]


def args_of(lines, name):
    return [l[len(name) + 1:-1].split(", ") for l in lines if l.startswith(name + "(")]


# nk_batch_norm_fwd(y, x, dtype, n, c, s, w, b, rm, rv, save_mean, save_rstd, training, momentum, eps)
# nk_batch_norm_bwd(dx, dx_dtype, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype, db_beta, g, g_dtype, x, dtype, n, c, s,
#                   w, save_mean, save_rstd, batch_stats)
@pytest.mark.parametrize("train", [1, 0])
def test_batch_norm_calls_per_pass(graph, train):
    def scenario(g):
        st = status(g, train)
        x = g.param((4, 3, 5, 6), BF16, F32)
        w, b = g.param((3,), BF16), g.param((3,), BF16, F32)
        rm, rv = g.leaf((3,)), g.leaf((3,))
        y = batch_norm(g, x, w, b, rm, rv, st, 0.25, 1e-3)
        loss = y.sum()
        loss.forward()
        for r in range(3):
            g.note("backward %d" % r)
            loss.backward(1.0)
        g.lib.nkg_status_release(st)

    lines = graph.run(scenario)
    assert lines[-1].endswith("never freed: []"), lines[-1]
    assert calls(lines) == ["nk_batch_norm_fwd", "backward 0", "nk_batch_norm_bwd", "backward 1", "nk_batch_norm_bwd",
                            "backward 2", "nk_batch_norm_bwd"]
    f = args_of(lines, "nk_batch_norm_fwd")[0]
    assert f[2:6] == [str(BF16), "4", "3", "30"] and f[12:] == [str(train), "0.25", "0.00100000005"]
    assert all(a != "0" for a in f[6:12])
    bw = args_of(lines, "nk_batch_norm_bwd")
    assert [a[1] for a in bw] == [str(F32)] * 3 and [a[4] for a in bw] == [str(BF16)] * 3
    assert [a[7] for a in bw] == [str(F32)] * 3
    for i in (2, 5, 8):                                        # dx, dw, db: overwrite, then accumulate
        assert [a[i] for a in bw] == ["0", "1", "1"]
    assert all(a[-1] == str(train) for a in bw)                # batch statistics in training mode only
    assert all(a[17:19] == f[10:12] for a in bw)               # the forward's saved statistics
    allocs = [l for l in lines if l.startswith("nk_alloc")]
    assert any(l.endswith(" = " + f[10]) and l.startswith("nk_alloc_uninit(12)") for l in allocs)


def test_batch_norm_null_operands(graph):
    """no affine, no running statistics; the operand is a constant while the weight is learned: no dx"""
    def scenario(g):
        st = status(g, 1)
        x = g.leaf((8, 5))
        y = batch_norm(g, x, None, None, None, None, st)
        y.forward()
        x2 = g.leaf((8, 5))
        w = g.param((5,))
        z = batch_norm(g, x2, w, None, None, None, st).sum()
        z.forward()
        z.backward(1.0)
        g.lib.nkg_status_release(st)

    lines = graph.run(scenario)
    f = args_of(lines, "nk_batch_norm_fwd")
    assert f[0][6:10] == ["0", "0", "0", "0"] and f[1][7:10] == ["0", "0", "0"] and f[1][6] != "0"
    (bw,) = args_of(lines, "nk_batch_norm_bwd")
    assert bw[0] == "0" and bw[3] != "0" and bw[6] == "0"


def test_batch_norm_backward_follows_the_forward_after_the_status_flips(graph):
    def scenario(g):
        st = status(g, 1)
        x = g.param((4, 2, 3))
        loss = batch_norm(g, x, None, None, g.leaf((2,)), g.leaf((2,)), st).sum()
        loss.forward()
        g.ck(g.lib.nkg_status_set(st, 0))
        loss.backward(1.0)            # the forward used batch statistics
        loss.forward()
        g.ck(g.lib.nkg_status_set(st, 1))
        loss.backward(1.0)            # the forward used the running ones
        g.lib.nkg_status_release(st)

    lines = graph.run(scenario)
    assert [a[12] for a in args_of(lines, "nk_batch_norm_fwd")] == ["1", "0"]
    assert [a[-1] for a in args_of(lines, "nk_batch_norm_bwd")] == ["1", "0"]


def test_one_value_per_channel_fails_on_a_training_forward_after_an_eval_build(graph):
    """built in eval mode with running statistics (allowed), then the status turns to training: the forward fails with
    torch's message and launches nothing"""
    def scenario(g):
        st = status(g, 0)
        y = batch_norm(g, g.param((1, 3)), None, None, g.leaf((3,)), g.leaf((3,)), st)
        g.ck(g.lib.nkg_status_set(st, 1))
        g.expect_error(y.forward)
        g.ck(g.lib.nkg_status_set(st, 0))
        y.forward()
        g.lib.nkg_status_release(st)

    lines = graph.run(scenario)
    errors = [l for l in lines if l.startswith("error")]
    assert errors == ["error -1 Expected more than 1 value per channel when training, got input size "
                      "torch.Size([1, 3])"], errors
    assert [a[12] for a in args_of(lines, "nk_batch_norm_fwd")] == ["0"]   # only the eval forward ran


# nk_layer_norm_fwd(y, x, dtype, rows, cols, w, b, save_mean, save_rstd, eps)
# nk_layer_norm_bwd(dx, dx_dtype, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype, db_beta, g, g_dtype, x, dtype, rows,
#                   cols, w, save_mean, save_rstd)
def test_layer_norm_calls_per_pass(graph):
    def scenario(g):
        x = g.param((2, 3, 4, 5), F32, BF16)
        w, b = g.param((4, 5)), g.param((4, 5))
        loss = layer_norm(g, x, 2, w, b, 1e-6).sum()
        loss.forward()
        for r in range(2):
            g.note("backward %d" % r)
            loss.backward(1.0)

    lines = graph.run(scenario)
    assert lines[-1].endswith("never freed: []"), lines[-1]
    assert calls(lines) == ["nk_layer_norm_fwd", "backward 0", "nk_layer_norm_bwd", "backward 1", "nk_layer_norm_bwd"]
    (f,) = args_of(lines, "nk_layer_norm_fwd")
    assert f[2:5] == [str(F32), "6", "20"] and f[-1] == "9.99999997e-07"
    bw = args_of(lines, "nk_layer_norm_bwd")
    assert [a[1] for a in bw] == [str(BF16)] * 2
    for i in (2, 5, 8):
        assert [a[i] for a in bw] == ["0", "1"]
    assert all(a[13:15] == ["6", "20"] and a[16:] == f[7:9] for a in bw)


def test_layer_norm_without_affine_or_bias(graph):
    def scenario(g):
        x = g.param((3, 7))
        w = g.param((7,))
        loss = layer_norm(g, x, 1, w, None).sum()
        loss.forward()
        loss.backward(1.0)
        layer_norm(g, g.leaf((3, 7)), 1, None, None).forward()

    lines = graph.run(scenario)
    f = args_of(lines, "nk_layer_norm_fwd")
    assert f[0][5] != "0" and f[0][6] == "0" and f[1][5:7] == ["0", "0"]
    (bw,) = args_of(lines, "nk_layer_norm_bwd")
    assert bw[0] != "0" and bw[3] != "0" and bw[6] == "0"


ERRORS = [
    ("batch_norm", lambda g, x, st: batch_norm(g, x, g.param((4,)), None, None, None, st), "weight must have shape"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, g.param((3,), BF16), None, None, None, st),
     "different element types"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, None, None, g.leaf((3,)), None, st), "both given or both NULL"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, None, None, g.leaf((3,), BF16), g.leaf((3,)), st), "must be f32"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, None, None, g.param((3,)), g.leaf((3,)), st),
     "must not be differentiable"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, None, None, g.leaf((3,)), g.leaf((3,)).relu(), st),
     "running_var must be a leaf"),
    ("batch_norm", lambda g, x, st: batch_norm(g, x, None, None, None, None, st, 0.1, -1.0), "eps must be >= 0"),
    ("batch_norm", lambda g, x, st: batch_norm(g, g.param((5,)), None, None, None, None, st), "(N, C, ...)"),
    ("Expected more than 1 value per channel when training, got input size torch.Size([1, 3])",
     lambda g, x, st: batch_norm(g, g.param((1, 3)), None, None, None, None, st), ""),
    ("batch_norm", lambda g, x, st: g.call("nkg_batch_norm", x.h, None, None, None, None, None, 0.1, 1e-5), "NULL"),
    ("layer_norm", lambda g, x, st: layer_norm(g, x, 5, None, None), "normalized_shape has 5 dimensions"),
    ("layer_norm", lambda g, x, st: layer_norm(g, x, 0, None, None), "normalized_shape has 0 dimensions"),
    ("layer_norm", lambda g, x, st: layer_norm(g, x, 2, g.param((7, 6)), None), "weight must have shape"),
    ("layer_norm", lambda g, x, st: layer_norm(g, x, 1, None, g.param((7,), BF16)), "different element types"),
]


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_invalid_arguments_fail_and_record_nothing(graph, case):
    who, op, msg = ERRORS[case]

    def scenario(g):
        st = status(g, 1)
        x = g.param((2, 3, 6, 7))
        x.describe("before")
        g.expect_error(op, g, x, st)
        x.describe("after")
        g.lib.nkg_status_release(st)

    lines = [l for l in graph.run(scenario) if not l.startswith(("nk_alloc", "nk_free"))]   # the operands made here
    assert len(lines) == 4, lines
    assert lines[1].startswith("error -1 %s" % who) and msg in lines[1], lines[1]
    assert lines[0].replace("before", "after") == lines[2]
