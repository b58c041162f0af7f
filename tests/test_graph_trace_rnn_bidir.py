"""The kernel-ABI calls of the LSTM / GRU layer node (nkg_lstm_layer / nkg_gru_layer), over the recording stub of
tests/graph_trace.py.  Two directions: two whole-sequence GEMMs, then per step ONE batched GEMM for both directions'
recurrent products and ONE two-direction step kernel; backward, per step one step kernel and one batched GEMM, then the
whole-sequence products once per direction.  One direction: the calls of nkg_lstm / nkg_gru plus one copy into h_n."""
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
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_rnn_bidir"))))


def layer(g, lstm, steps, dirs, state_diff, x_diff, loss_on="output"):
    G = (4 if lstm else 3) * H
    w_ih, w_hh = g.param((dirs, G, I), BF16, F32), g.param((dirs, G, H), BF16, F32)
    b_ih, b_hh = g.param((dirs, G), BF16, F32), g.param((dirs, G), BF16, F32)
    w_ih.set_hook("w_ih")
    w_hh.set_hook("w_hh")
    b_ih.set_hook("b_ih")
    h = g.param((dirs, N, H), BF16, F32) if state_diff else g.leaf((dirs, N, H), BF16)
    c = g.param((dirs, N, H), BF16, F32) if state_diff else g.leaf((dirs, N, H), BF16)
    x = g.param((steps, N, I), BF16, F32) if x_diff else g.leaf((steps, N, I), BF16)
    y, hn, cn = C.c_void_p(), C.c_void_p(), C.c_void_p()
    if lstm:
        g.ck(g.lib.nkg_lstm_layer(x.h, c.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y), C.byref(hn), C.byref(cn)))
        y, hn, cn = g.wrap(y), g.wrap(hn), g.wrap(cn)
    else:
        g.ck(g.lib.nkg_gru_layer(x.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y), C.byref(hn)))
        y, hn = g.wrap(y), g.wrap(hn)
    loss = {"output": lambda: y.mean(), "h_n": lambda: hn.sum()}[loss_on]()
    loss.forward()
    g.note("backward")
    loss.backward(1.0)


def calls(graph, *args, **kw):
    lines = graph.run(lambda g: layer(g, *args, **kw))
    assert lines[-1].endswith("never freed: []"), lines[-1]
    names = [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]
    names = [n for n in names if n not in ("nk_alloc", "nk_alloc_uninit", "nk_free")]
    k = names.index("backward")
    return names[:k], names[k + 1:], lines


def args(line):
    return line[line.index("(") + 1:-1].split(", ")


@pytest.mark.parametrize("lstm", [True, False])
@pytest.mark.parametrize("steps", [1, 3])
def test_bidirectional_forward_is_two_gemms_plus_two_calls_per_step(graph, lstm, steps):
    fwd, _, lines = calls(graph, lstm, steps, 2, True, True)
    step = "nk_lstm_bidir_fwd_step" if lstm else "nk_gru_bidir_fwd_step"
    assert fwd == ["nk_gemm_bias_act"] * 2 + ["nk_gemm_strided_batched", step] * steps + ["nk_sum_fwd"]
    G, NG = (4 if lstm else 3) * H, N * (4 if lstm else 3) * H
    batched = [args(l) for l in lines[:lines.index("backward")] if l.startswith("nk_gemm_strided_batched(")]
    for s, a in enumerate(batched):
        # NT, (N, G, H), both directions (batch 2): W_hh G*H apart, gates (2T-1-2s)*N*G apart, biases G apart
        assert a[:5] == ["0", "1", str(N), str(G), str(H)], a
        assert a[8] == str(N * H) and a[11] == str(G * H) and a[15] == str((2 * steps - 1 - 2 * s) * NG), a
        assert a[16] == "2" and a[20] == str(G), a
        assert a[12] == ("1" if lstm else "0"), a   # the LSTM's recurrent product adds to the input gates


@pytest.mark.parametrize("lstm", [True, False])
def test_bidirectional_backward_with_every_operand_differentiable(graph, lstm):
    steps = 3
    _, bwd, lines = calls(graph, lstm, steps, 2, True, True)
    step = "nk_lstm_bidir_bwd_step" if lstm else "nk_gru_bidir_bwd_step"
    start = ["nk_fill", "nk_sum_bwd", "nk_memset0"]
    assert bwd == (start + [step, "nk_gemm_strided_batched"] * steps +
                   ["nk_gemm_bias_act"] * 4 + ["hook w_hh"] + ["nk_gemm_bias_act"] * 2 + ["hook w_ih"] +
                   ["nk_unbroadcast_acc"] * 2 + ["hook b_ih"] + ["nk_unbroadcast_acc"] * 2 + ["nk_gemm_bias_act"] * 2 +
                   ["nk_unbroadcast_acc"] * (2 if lstm else 1))
    for hook in ("hook w_hh", "hook w_ih", "hook b_ih"):
        assert bwd.count(hook) == 1
    # the reverse direction's dW_hh reads output rows 1.. at column offset H (ld 2H), then h0[1]
    gemms = [args(l) for l in lines[lines.index("backward"):] if l.startswith("nk_gemm_bias_act(")]
    G = (4 if lstm else 3) * H
    assert [a[:5] for a in gemms[:4]] == [["1", "0", str(G), str(H), str((steps - 1) * N)], ["1", "0", str(G), str(H), str(N)]] * 2
    assert gemms[0][9] == str(2 * H) and gemms[2][9] == str(2 * H)
    assert gemms[2][8].endswith("+%d" % ((N * 2 * H + H) * 2)), gemms[2][8]
    assert gemms[3][8].endswith("+%d" % (N * H * 2)), gemms[3][8]


@pytest.mark.parametrize("lstm", [True, False])
def test_bidirectional_backward_does_no_work_for_plain_operands(graph, lstm):
    """input and states are plain Vars: no dX product, no state conversion, and step 0 sends nothing back"""
    steps = 3
    _, bwd, _ = calls(graph, lstm, steps, 2, False, False)
    step = "nk_lstm_bidir_bwd_step" if lstm else "nk_gru_bidir_bwd_step"
    assert bwd == (["nk_fill", "nk_sum_bwd", "nk_memset0"] + [step, "nk_gemm_strided_batched"] * (steps - 1) + [step] +
                   ["nk_gemm_bias_act"] * 4 + ["hook w_hh"] + ["nk_gemm_bias_act"] * 2 + ["hook w_ih"] +
                   ["nk_unbroadcast_acc"] * 2 + ["hook b_ih"] + ["nk_unbroadcast_acc"] * 2)


@pytest.mark.parametrize("lstm", [True, False])
@pytest.mark.parametrize("steps", [1, 3])
def test_one_direction_is_the_sequence_node_plus_one_copy(graph, lstm, steps):
    fwd, bwd, _ = calls(graph, lstm, steps, 1, True, True)
    gate = "nk_lstm_cell_fwd" if lstm else "nk_gru_cell_fwd"
    assert fwd == ["nk_gemm_bias_act"] + ["nk_gemm_bias_act", gate] * steps + ["nk_cast", "nk_sum_fwd"]
    step = "nk_lstm_seq_bwd_step" if lstm else "nk_gru_seq_bwd_step"
    assert bwd == (["nk_fill", "nk_sum_bwd", "nk_memset0"] + [step, "nk_gemm_bias_act"] * steps +
                   ["nk_gemm_bias_act"] * (2 if steps > 1 else 1) + ["hook w_hh", "nk_gemm_bias_act", "hook w_ih",
                                                                     "nk_unbroadcast_acc", "hook b_ih",
                                                                     "nk_unbroadcast_acc", "nk_gemm_bias_act"] +
                   ["nk_unbroadcast_acc"] * (2 if lstm else 1))


@pytest.mark.parametrize("lstm", [True, False])
@pytest.mark.parametrize("dirs", [1, 2])
def test_last_hidden_state_gradient_seeds_the_carried_gradient(graph, lstm, dirs):
    """the loss reads only h_n: the carried f32 dh starts as its gradient (one conversion), every dh_out is NULL, and the
    last step reads it"""
    _, bwd, lines = calls(graph, lstm, 2, dirs, False, False, loss_on="h_n")
    if lstm:
        assert bwd[:4] == ["nk_fill", "nk_sum_bwd", "nk_memset0", "nk_cast"], bwd   # dc zero, dh from h_n's gradient
    else:
        assert bwd[:3] == ["nk_fill", "nk_sum_bwd", "nk_cast"], bwd
    name = ("nk_lstm_" if lstm else "nk_gru_") + ("bidir_bwd_step" if dirs == 2 else "seq_bwd_step")
    steps = [args(l) for l in lines if l.startswith(name + "(")]
    assert len(steps) == 2
    dh_out = {"nk_lstm_seq_bwd_step": 5, "nk_gru_seq_bwd_step": 7, "nk_lstm_bidir_bwd_step": 7,
              "nk_gru_bidir_bwd_step": 10}[name]
    assert all(a[dh_out] == "0" for a in steps), steps
    if lstm:
        dh_rec = 6 if dirs == 1 else 10
        assert all(a[dh_rec] != "0" for a in steps), steps


def test_layer_operand_errors(graph):
    def run(g):
        G = 4 * H
        x = g.leaf((3, N, I), BF16)
        w_ih, w_hh = g.leaf((2, G, I), BF16), g.leaf((2, G, H), BF16)
        b_ih, b_hh = g.leaf((2, G), BF16), g.leaf((2, G), BF16)
        y, hn, cn = C.c_void_p(), C.c_void_p(), C.c_void_p()
        for h in (g.leaf((3, N, H), BF16), g.leaf((N, H), BF16)):
            g.expect_error(lambda: g.ck(g.lib.nkg_lstm_layer(x.h, h.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y),
                                                             C.byref(hn), C.byref(cn))))
        h = g.leaf((1, N, H), BF16)   # one direction against parameters of two
        g.expect_error(lambda: g.ck(g.lib.nkg_lstm_layer(x.h, h.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y),
                                                         C.byref(hn), C.byref(cn))))
        h = g.leaf((2, N, H), BF16)
        g.expect_error(lambda: g.ck(g.lib.nkg_lstm_layer(x.h, h.h, h.h, w_ih.h, w_hh.h, b_ih.h, b_hh.h, C.byref(y),
                                                         None, C.byref(cn))))
    lines = graph.run(run)
    errors = [l for l in lines if l.startswith("error")]
    assert len(errors) == 4, lines
    assert "hidden must be (num_directions = 1 or 2" in errors[0] and "hidden must be (num_directions" in errors[1]
    assert "cell_state must be (1, 4, 16)" in errors[2] or "weight_ih must be (1, 64, 8)" in errors[2], errors[2]
    assert "NULL output" in errors[3]
