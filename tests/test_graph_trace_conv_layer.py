"""The kernel-ABI calls of the 1-d / 3-d convolution layer node (nkg_conv_layer), over the recording stub of
tests/graph_trace.py, so the node's structure is checked without a GPU: one nk_conv_layer_nd_fwd forward (no padded copy,
no separate bias add); backward one nk_conv_layer_nd_bwd_input for a differentiable input and one
nk_conv_layer_nd_bwd_kernel that also produces the bias gradient when it has the weight gradient's element type."""
import ctypes as C
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
ZERO, REFLECTIVE, REPLICATIVE = 0, 1, 2
LAYER = ("nk_conv_layer_nd_fwd", "nk_conv_layer_nd_bwd_input", "nk_conv_layer_nd_bwd_kernel")
# the layer entry points' shape arguments are host arrays of nsp entries
T.HOST_ARRAYS.update({(f, p): "nsp" for f in LAYER for p in ("in_sp", "k", "stride", "dilation", "pad")})


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_conv_layer"))))


def layer(g, x, w, b, pad, mode=ZERO, value=0.0, stride=None, dil=None):
    nsp = len(pad)
    out = C.c_void_p()
    g.ck(g.lib.nkg_conv_layer(x.h if x else None, w.h if w else None, b.h if b else None, nsp, T._i64s(pad), mode, value,
                              T._i64s(stride or (1,) * nsp), T._i64s(dil or (1,) * nsp), C.byref(out)))
    return g.wrap(out)


# nsp: (input, weight, bias, padding, mode, stride, dilation)
GEOMETRY = {
    1: ((2, 4, 10), (8, 4, 3), (8, 1), (2,), REFLECTIVE, (2,), (1,)),
    3: ((1, 3, 4, 5, 6), (8, 3, 2, 2, 2), (8, 1, 1, 1), (1, 0, 2), REPLICATIVE, (1, 2, 1), (1, 1, 2)),
}


def scenario(g, nsp, x_diff, grad_dtype, padded, passes):
    xs, ws, bs, pad, mode, stride, dil = GEOMETRY[nsp]
    pad = pad if padded else (0,) * nsp
    x = g.param(xs, BF16, grad_dtype) if x_diff else g.leaf(xs, BF16)
    w, b = g.param(ws, BF16, grad_dtype), g.param(bs, BF16, grad_dtype)
    y = layer(g, x, w, b, pad, mode, 0.0, stride, dil)
    y.describe("y")
    loss = y.mean()
    loss.forward()
    for r in range(passes):
        g.note("backward %d" % r)
        loss.backward(1.0)


def calls(graph, *args):
    lines = graph.run(lambda g: scenario(g, *args))
    assert lines[-1].endswith("never freed: []"), lines[-1]
    names = [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]
    return [n for n in names if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free")], lines


def args_of(lines, name):
    return [l[len(name) + 1:-1].split(", ") for l in lines if l.startswith(name + "(")]


@pytest.mark.parametrize("padded", [True, False])
@pytest.mark.parametrize("nsp", [1, 3])
def test_one_call_forward_and_two_backward(graph, nsp, padded):
    """a bf16 layer with bf16 gradients: forward is one layer call; backward is dX then dW with the bias gradient riding
    along; the padding goes to the layer calls as given, never to a pad kernel"""
    names, lines = calls(graph, nsp, True, None, padded, 1)
    assert names == ["y", LAYER[0], "nk_sum_fwd", "backward 0", "nk_fill", "nk_sum_bwd", LAYER[1], LAYER[2]]
    xs, ws, bs, pad, mode, stride, dil = GEOMETRY[nsp]
    pad = list(pad if padded else (0,) * nsp)
    fwd = args_of(lines, LAYER[0])[0]
    # y, x, w, bias, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, mode, value, dtype
    assert fwd[4:] == [str(nsp), str(xs[0]), str(xs[1]), str(list(xs[2:])).replace(" ", ""), str(ws[0]),
                       str(list(ws[2:])).replace(" ", ""), str(list(stride)).replace(" ", ""),
                       str(list(dil)).replace(" ", ""), str(pad).replace(" ", ""), str(mode), "0", str(BF16)]
    dx = args_of(lines, LAYER[1])[0]
    assert dx[-3:] == [str(mode), str(BF16), "0"]                                  # mode, dtype, beta
    dw = args_of(lines, LAYER[2])[0]
    assert dw[1] == str(BF16) and dw[2] != "0" and dw[-1] == "0"                 # dw dtype, dbias given, beta 0


@pytest.mark.parametrize("nsp", [1, 3])
def test_input_as_var_costs_no_dx(graph, nsp):
    names, lines = calls(graph, nsp, False, None, True, 1)
    assert LAYER[1] not in names
    assert names[names.index("backward 0"):] == ["backward 0", "nk_fill", "nk_sum_bwd", LAYER[2]]


@pytest.mark.parametrize("nsp", [1, 3])
def test_f32_gradients_of_bf16_data(graph, nsp):
    """dX is produced in the data type and added into the f32 gradient (accumulate's temporary); dW and db are written
    in f32 by the layer call itself"""
    names, lines = calls(graph, nsp, True, F32, True, 1)
    assert names[names.index("backward 0"):] == ["backward 0", "nk_fill", "nk_sum_bwd", LAYER[1], "nk_unbroadcast_acc",
                                                 LAYER[2]]
    assert args_of(lines, LAYER[1])[0][-1] == "0"
    dw = args_of(lines, LAYER[2])[0]
    assert dw[1] == str(F32) and dw[2] != "0"


@pytest.mark.parametrize("grad_dtype", [None, F32])
def test_second_backward_accumulates(graph, grad_dtype):
    """the second backward() runs the same calls with beta = 1 into every gradient"""
    names, lines = calls(graph, 1, True, grad_dtype, True, 2)
    k = names.index("backward 1")
    assert names[k + 1:] == names[names.index("backward 0") + 1:k]
    dxs, dws = args_of(lines, LAYER[1]), args_of(lines, LAYER[2])
    assert [d[-1] for d in dws] == ["0", "1"]
    if grad_dtype is None:
        assert [d[-1] for d in dxs] == ["0", "1"]
    else:     # into a temporary, then added with beta = 1
        assert [d[-1] for d in dxs] == ["0", "0"]
        assert [a[-1] for a in args_of(lines, "nk_unbroadcast_acc")] == ["0", "1"]


def test_bias_of_another_gradient_type_is_summed_apart(graph):
    """f32 weight gradient, bf16 bias gradient: dW without dbias, then the un-broadcast of g onto the (Cout, 1, 1, 1)
    bias"""
    def run(g):
        x = g.leaf((1, 3, 4, 5, 6), F32)
        w, b = g.param((2, 3, 2, 2, 2)), g.param((2, 1, 1, 1), F32, BF16)
        y = layer(g, x, w, b, (0, 1, 0), ZERO, 0.0, (1, 2, 1), (1, 1, 2))
        y.forward()
        y.backward(1.0)
    lines = graph.run(run)
    dw = args_of(lines, LAYER[2])[0]
    assert dw[2] == "0"
    ub = args_of(lines, "nk_unbroadcast_acc")[0]
    assert ub[1:4] == [str(BF16), "4", "[2,1,1,1]"] and ub[5:8] == [str(F32), "5", "[1,2,3,3,4]"]


def test_no_bias(graph):
    def run(g):
        x, w = g.param((2, 4, 9)), g.param((8, 4, 3))
        y = layer(g, x, w, None, (1,), REPLICATIVE)
        y.describe("y")
        y.forward()
        y.backward(1.0)
    lines = graph.run(run)
    assert args_of(lines, LAYER[0])[0][3] == "0" and args_of(lines, LAYER[2])[0][2] == "0"
    assert not args_of(lines, "nk_unbroadcast_acc")


def test_argument_errors(graph):
    def run(g):
        E, L = g.expect_error, g.lib
        x1, w1, b1 = g.leaf((2, 4, 5)), g.param((8, 4, 3)), g.param((8, 1))
        E(lambda: layer(g, None, w1, b1, (1,)))
        E(lambda: layer(g, x1, w1, b1, (1, 1)))                                   # nsp = 2
        E(lambda: layer(g, g.leaf((2, 4, 5, 5)), g.param((8, 4, 3, 3)), b1, (1, 1)))
        E(lambda: layer(g, x1, g.param((8, 4, 3, 3)), b1, (1,)))                 # kernel rank
        E(lambda: layer(g, x1, g.param((8, 3, 3)), b1, (1,)))                    # in-channels
        E(lambda: layer(g, x1, w1, g.param((8,)), (1,)))                         # bias shape
        E(lambda: layer(g, x1, w1, g.param((8, 1), BF16), (1,)))                 # bias dtype
        E(lambda: layer(g, x1, w1, b1, (5,), REFLECTIVE))                        # reflection as long as the input
        E(lambda: layer(g, x1, w1, b1, (-1,)))
        E(lambda: layer(g, x1, w1, b1, (1,), 3))                                  # mode
        E(lambda: layer(g, x1, w1, b1, (1,), ZERO, 0.0, (0,)))                   # stride
        E(lambda: layer(g, x1, g.param((8, 4, 9)), b1, (1,)))                    # kernel longer than the padded input
        out = C.c_void_p()
        E(lambda: g.ck(L.nkg_conv_layer(x1.h, w1.h, b1.h, 1, None, 0, 0.0, T._i64s((1,)), T._i64s((1,)), C.byref(out))))
    lines = graph.run(run)
    errors = [l for l in lines if l.startswith("error ")]
    assert len(errors) == 13 and not any(l.startswith(LAYER) for l in lines), lines
    for want in ("conv_layer: NULL", "1 or 3 sample dimensions (got 2)", "Invalid kernel shape for 1d conv",
                 "kernel in-channels 3", "bias must be (8, 1), got (8,)", "operands have different element types",
                 "reflective padding 5 must be smaller than the dimension 5", "padding must be >= 0", "bad mode 3",
                 "Invalid stride/dilation for 1d conv.", "The kernel size can't be greater than actual input size."):
        assert any(want in e for e in errors), want
