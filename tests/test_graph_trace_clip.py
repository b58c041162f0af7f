"""The kernel-ABI calls of the gradient-clipping graph entry points (nkg_grad_norm, nkg_clip_grads_with_norm,
nkg_clip_grad_value), over the recording stub of tests/graph_trace.py: every parameter is checked first, then each
gradient is materialised in parameter order (a pending zero_grad() gets its zero fill) and ONE ABI call takes every
table in parameter order, whatever the dtypes; an error launches nothing.  The traces are pinned in
tests/golden/graph_trace_clip.json (tests/golden/make_graph_trace_clip.py)."""
import ctypes as C
import json
import os
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graph_trace_clip.json")
CLIP_CALLS = ("nk_grad_norm", "nk_grad_scale_by_norm", "nk_grad_clamp")
# the clipping calls' host tables, written by content like the optimizers' (added before the stub is generated)
T.HOST_ARRAYS.update({(f, p): "count" for f in CLIP_CALLS for p in ("g", "g_dtype", "n")})

# 70 parameters whose gradients mix f32 and bf16 (bf16 data with f32 gradients, f32 data with bf16 gradients, ...)
MIXED = [(1 + 37 * i % 4099, BF16 if i % 3 == 1 else F32, BF16 if i % 5 == 2 else F32) for i in range(70)]


def _arr(ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


def _params(g, specs):
    return [g.param((n,), dt, gd) for n, dt, gd in specs]


def _hs(ps):
    return _arr([p.h.value for p in ps])


def norm_mixed(g):
    ps = _params(g, MIXED)
    total = g.ext(4)
    g.ck(g.lib.nkg_grad_norm(_hs(ps), len(ps), 2.0, 1.0, total))
    g.ck(g.lib.nkg_clip_grads_with_norm(_hs(ps), len(ps), 0.25, total))


def every_norm_type(g):
    ps = _params(g, MIXED[:4])
    for p in (1.0, 2.0, 3.0, 0.5, float("inf")):
        g.ck(g.lib.nkg_grad_norm(_hs(ps), len(ps), p, 0.5, g.ext(4)))


def pending_zero_grad(g):
    """a backward pass, zero_grad() on one weight, then clip_grad_norm_: the norm sees that weight's zeros"""
    x = g.leaf((3, 6), BF16)
    w = g.param((4, 6), BF16, F32)
    b = g.param((4,), BF16, F32)
    s = (x.mm_t(w) + b).sum()
    s.forward()
    s.backward(1.0)
    w.zero_grad()
    total = g.ext(4)
    g.ck(g.lib.nkg_grad_norm(_hs([w, b]), 2, 2.0, 1.0, total))
    g.ck(g.lib.nkg_clip_grads_with_norm(_hs([w, b]), 2, 1.0, total))
    s.backward(1.0)      # the clipped gradients are nonzero now: the next pass accumulates into them


def not_differentiable(g):
    ps = _params(g, [(4, F32, None)] * 3)
    ps[1] = g.leaf((4,), F32)
    hs, total = _hs(ps), g.ext(4)
    g.expect_error(lambda: g.ck(g.lib.nkg_grad_norm(hs, 3, 2.0, 1.0, total)))
    g.expect_error(lambda: g.ck(g.lib.nkg_clip_grads_with_norm(hs, 3, 1.0, total)))
    g.expect_error(lambda: g.ck(g.lib.nkg_clip_grad_value(hs, 3, 1.0, 1.0)))


def bad_arguments(g):
    ps = _params(g, [(4, F32, None)] * 2)
    hs, total = _hs(ps), g.ext(4)
    for p in (0.0, -2.0, float("-inf"), float("nan")):
        g.expect_error(lambda: g.ck(g.lib.nkg_grad_norm(hs, 2, p, 1.0, total)))
    g.expect_error(lambda: g.ck(g.lib.nkg_grad_norm(hs, 0, 2.0, 1.0, total)))
    g.expect_error(lambda: g.ck(g.lib.nkg_grad_norm(None, 2, 2.0, 1.0, total)))
    g.ck(g.lib.nkg_clip_grads_with_norm(hs, 0, 1.0, total))     # no parameters: nothing to do
    g.ck(g.lib.nkg_clip_grad_value(hs, 0, 1.0, 1.0))
    g.note("empty lists done")


def clip_value_with_grad_scale(g):
    ps = _params(g, [(5, F32, None), (6, BF16, None), (7, BF16, F32)])
    g.ck(g.lib.nkg_clip_grad_value(_hs(ps), len(ps), 0.5, 0.25))


SCENARIOS = {"norm_mixed": norm_mixed, "every_norm_type": every_norm_type, "pending_zero_grad": pending_zero_grad,
             "not_differentiable": not_differentiable, "bad_arguments": bad_arguments,
             "clip_value_with_grad_scale": clip_value_with_grad_scale}


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_clip"))))


def calls(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def arg(line, name, field):
    """one argument of a traced call, by position in the header's parameter list"""
    params = [p for _, n, ps in T.header_functions() if n == name for p in ps][1:]   # the context is not traced
    args = re.findall(r"\[[^\]]*\]|[^,\s][^,]*", line[len(name) + 1:-1])
    return args[[p[1] for p in params].index(field)]


def test_every_scenario_has_a_golden():
    with open(GOLDEN) as fh:
        assert sorted(json.load(fh)) == sorted(SCENARIOS)


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_trace_matches_golden(graph, name):
    with open(GOLDEN) as fh:
        want = json.load(fh)[name]
    got = graph.run(SCENARIOS[name])
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, "%s: first difference at call %d:\n  got  %s\n  want %s" % (name, i, a, b)
    assert len(got) == len(want)


def test_one_call_with_every_table_in_parameter_order(graph):
    lines = graph.run(norm_mixed)
    names = [n for n in calls(lines) if n not in ("nk_alloc", "nk_alloc_uninit")]
    assert names == ["nk_grad_norm", "nk_grad_scale_by_norm"]
    for name in ("nk_grad_norm", "nk_grad_scale_by_norm"):
        line = next(l for l in lines if l.startswith(name + "("))
        assert int(arg(line, name, "count")) == len(MIXED)
        assert json.loads(arg(line, name, "n")) == [n for n, _, _ in MIXED]
        assert json.loads(arg(line, name, "g_dtype")) == [gd for _, _, gd in MIXED]
        assert len(set(arg(line, name, "g").strip("[]").split(","))) == len(MIXED)
    norm = next(l for l in lines if l.startswith("nk_grad_norm("))
    assert (arg(norm, "nk_grad_norm", "norm_type"), arg(norm, "nk_grad_norm", "grad_scale")) == ("2", "1")


def test_pending_zero_grad_is_filled_before_the_norm(graph):
    lines = graph.run(pending_zero_grad)
    names = calls(lines)
    i = names.index("nk_grad_norm")
    assert "nk_memset0" in names[:i] and names.index("nk_memset0") > max(
        k for k, n in enumerate(names[:i]) if n.startswith("nk_gemm") or n == "nk_unbroadcast_acc")
    assert names[i + 1] == "nk_grad_scale_by_norm"


def test_errors_launch_nothing(graph):
    lines = graph.run(not_differentiable)
    errors = [l for l in lines if l.startswith("error ")]
    assert len(errors) == 3 and all("parameter 1 is not differentiable" in e for e in errors), errors
    after = lines[lines.index(errors[0]):]
    assert not any(l.startswith(("nk_grad_", "nk_alloc", "nk_memset0", "nk_fill")) for l in after), after
    lines = graph.run(bad_arguments)
    errors = [l for l in lines if l.startswith("error ")]
    assert len(errors) == 6 and sum("norm_type must be > 0" in e for e in errors) == 4, errors
    after = lines[lines.index(errors[0]):]
    assert not any(l.startswith(("nk_grad_", "nk_alloc", "nk_memset0", "nk_fill")) for l in after), after


def test_clip_value_passes_the_grad_scale(graph):
    lines = graph.run(clip_value_with_grad_scale)
    line = next(l for l in lines if l.startswith("nk_grad_clamp("))
    assert (arg(line, "nk_grad_clamp", "clip_value"), arg(line, "nk_grad_clamp", "grad_scale")) == ("0.5", "0.25")
    assert json.loads(arg(line, "nk_grad_clamp", "g_dtype")) == [F32, BF16, F32]
