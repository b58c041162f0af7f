"""The kernel-ABI calls of the LSTM / GRU sequence node (nkg_lstm / nkg_gru), over the recording stub of
tests/graph_trace.py, so the node's launch structure is checked without a GPU: one whole-sequence GEMM plus a GEMM and a
gate kernel per step forward; per step a step kernel and one GEMM backward, then every whole-sequence product once."""
import ctypes as C
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
N, I, H = 4, 8, 16


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_rnn_seq"))))


def sequence(g, lstm, steps, state_diff, x_diff, through_cell=False):
    G = (4 if lstm else 3) * H
    w_ih, w_hh = g.param((G, I), BF16, F32), g.param((G, H), BF16, F32)
    b_ih, b_hh = g.param((G,), BF16, F32), g.param((G,), BF16, F32)
    w_ih.set_hook("w_ih")
    w_hh.set_rs("w_hh", 2, 0)
    h = g.param((N, H), BF16, F32) if state_diff else g.leaf((N, H), BF16)
    c = g.param((N, H), BF16, F32) if state_diff else g.leaf((N, H), BF16)
    x = g.param((steps, N, I), BF16, F32) if x_diff else g.leaf((steps, N, I), BF16)
    y, oc = C.c_void_p(), C.c_void_p()
    if lstm:
        g.ck(g.lib.nkg_lstm(x.h, c.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y), C.byref(oc)))
        y, oc = g.wrap(y), g.wrap(oc)
    else:
        g.ck(g.lib.nkg_gru(x.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y)))
        y = g.wrap(y)
    loss = oc.sum() if through_cell else y.mean()
    loss.forward()
    g.note("backward")
    loss.backward(1.0)


def calls(graph, *args, **kw):
    lines = graph.run(lambda g: sequence(g, *args, **kw))
    assert lines[-1].endswith("never freed: []"), lines[-1]
    names = [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]
    names = [n for n in names if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free")]
    k = names.index("backward")
    return names[:k], names[k + 1:], lines


@pytest.mark.parametrize("lstm", [True, False])
@pytest.mark.parametrize("steps", [1, 3])
def test_forward_is_one_gemm_plus_two_calls_per_step(graph, lstm, steps):
    fwd, _, _ = calls(graph, lstm, steps, True, True)
    gate = "nk_lstm_cell_fwd" if lstm else "nk_gru_cell_fwd"
    assert fwd == ["nk_gemm_bias_act"] + ["nk_gemm_bias_act", gate] * steps + ["nk_sum_fwd"]


@pytest.mark.parametrize("lstm", [True, False])
def test_backward_with_every_operand_differentiable(graph, lstm):
    steps = 3
    _, bwd, lines = calls(graph, lstm, steps, True, True)
    step = "nk_lstm_seq_bwd_step" if lstm else "nk_gru_seq_bwd_step"
    assert bwd == (["nk_fill", "nk_sum_bwd", "nk_memset0"] + [step, "nk_gemm_bias_act"] * steps +
                   ["nk_gemm_bias_act", "nk_gemm_bias_act", "rs w_hh pushed", "nk_gemm_bias_act", "hook w_ih"] +
                   ["nk_unbroadcast_acc"] * 2 + ["nk_gemm_bias_act"] + ["nk_unbroadcast_acc"] * (2 if lstm else 1))
    # the whole-sequence products: dW_hh over K = (T-1)*N then step 0 (beta 1), dW_ih over K = T*N, dX over T*N rows
    gemms = [l for l in lines[lines.index("backward"):] if l.startswith("nk_gemm_bias_act(")]
    G = (4 if lstm else 3) * H
    heads = [",".join(l[len("nk_gemm_bias_act("):].split(", ")[:5]) for l in gemms[steps:]]
    assert heads == ["1,0,%d,%d,%d" % (G, H, (steps - 1) * N), "1,0,%d,%d,%d" % (G, H, N), "1,0,%d,%d,%d" % (G, I, steps * N),
                     "0,0,%d,%d,%d" % (steps * N, I, G)]


@pytest.mark.parametrize("lstm", [True, False])
def test_backward_does_no_work_for_plain_operands(graph, lstm):
    """input and states are plain Vars: no dX product, no state conversion, and step 0 sends nothing back"""
    steps = 3
    _, bwd, _ = calls(graph, lstm, steps, False, False)
    step = "nk_lstm_seq_bwd_step" if lstm else "nk_gru_seq_bwd_step"
    assert bwd == (["nk_fill", "nk_sum_bwd", "nk_memset0"] + [step, "nk_gemm_bias_act"] * (steps - 1) + [step] +
                   ["nk_gemm_bias_act", "nk_gemm_bias_act", "rs w_hh pushed", "nk_gemm_bias_act", "hook w_ih"] +
                   ["nk_unbroadcast_acc"] * 2)


def test_lstm_running_cell_gradient_starts_from_the_last_cell_state_gradient(graph):
    """the loss reads only the last cell state: dc starts as its gradient converted to f32, and every dh_out is NULL"""
    _, bwd, lines = calls(graph, True, 2, False, False, through_cell=True)
    assert bwd[:3] == ["nk_fill", "nk_sum_bwd", "nk_cast"]
    steps = [l for l in lines if l.startswith("nk_lstm_seq_bwd_step(")]
    assert len(steps) == 2 and all(l.split(", ")[5] == "0" for l in steps), steps   # dh_out
    assert steps[0].split(", ")[6] == "0" and steps[1].split(", ")[6] != "0"            # dh_rec: NULL at step T-1 only
