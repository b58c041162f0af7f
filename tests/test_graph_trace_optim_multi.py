"""The kernel-ABI calls of the optimizers' graph entry points (nkg_multi_*_step), over the recording stub of
tests/graph_trace.py, so their structure is checked without a GPU: every parameter's gradient is materialised in
parameter order (a zeroed one is cleared first), Adam and Adagrad launch their prologue once, and each (data, gradient)
dtype group is updated by one nk_multi_*_step call per 64 tensors, in parameter order; a parameter that is not
differentiable fails the call before anything is launched.  Every variant runs once on a single parameter too.  The traces are pinned in tests/golden/graph_trace_optim_multi.json
(tests/golden/make_graph_trace_optim_multi.py)."""
import ctypes as C
import json
import os
import re

import pytest

import graph_trace as T

BF16, F32 = T.BF16, T.F32
PER_LAUNCH = 64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graph_trace_optim_multi.json")


def _arr(ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


def _params(g, specs):
    """specs: [(numel, data dtype, gradient dtype or None)]"""
    return [g.param((n,), dt, gd) for n, dt, gd in specs]


def _states(g, specs, present=True):
    return _arr([g.ext(n * 4) for n, _, _ in specs]) if present else None


def _masters(g, specs):
    return _arr([g.ext(n * 4) if dt == BF16 else None for n, dt, _ in specs])


# 70 parameters: f32 ones with two bf16 ones (f32 gradients, master weights) among them
MIXED = [(1 + 37 * i % 4099, BF16 if i in (3, 50) else F32, F32 if i in (3, 50) else None) for i in range(70)]
# every (data, gradient) pair, in an order that interleaves them
PAIRS = [(5, F32, None), (6, BF16, None), (7, BF16, F32), (8, F32, BF16), (9, F32, None), (10, BF16, F32)]


def adam_mixed(g):
    ps = _params(g, MIXED)
    hyper = g.ext(24)
    g.ck(g.lib.nkg_multi_adam_step(_arr([p.h.value for p in ps]), len(ps), _states(g, MIXED), _states(g, MIXED),
                                   _states(g, MIXED), _masters(g, MIXED), hyper, 0.9, 0.999, 1e-8, 0.0, 0.01, 0.5))


def sgd_pairs(g):
    ps = _params(g, PAIRS)
    g.ck(g.lib.nkg_multi_sgd_step(_arr([p.h.value for p in ps]), len(ps), _states(g, PAIRS), None, g.ext(24), 0.01,
                                  0.9, 0.1, 1, 1.0))


def rmsprop_pairs(g):
    ps = _params(g, PAIRS)
    g.ck(g.lib.nkg_multi_rmsprop_step(_arr([p.h.value for p in ps]), len(ps), _states(g, PAIRS), _states(g, PAIRS),
                                      None, _masters(g, PAIRS), g.ext(24), 0.99, 1e-8, 0.0, 0.0, 0.0, 1.0))


def adagrad_twice(g):
    specs = [(130, F32, None)] * 3
    ps = _params(g, specs)
    hyper, st = g.ext(24), _states(g, specs)
    for r in range(2):
        g.note("step %d" % r)
        g.ck(g.lib.nkg_multi_adagrad_step(_arr([p.h.value for p in ps]), len(ps), st, None, hyper, 0.1, 1e-10, 0.0,
                                          0.0, 1.0))


def not_differentiable(g):
    specs = [(4, F32, None)] * 3
    ps = _params(g, specs)
    ps[1] = g.leaf((4,), F32)
    hs = _arr([p.h.value for p in ps])
    for name, args in (("nkg_multi_adam_step", (None, None, None, None, g.ext(24), 0.9, 0.999, 1e-8, 0.0, 0.0, 1.0)),
                       ("nkg_multi_sgd_step", (None, None, g.ext(24), 0.0, 0.0, 0.0, 0, 1.0)),
                       ("nkg_multi_rmsprop_step", (None, None, None, None, g.ext(24), 0.99, 1e-8, 0.0, 0.0, 0.0, 1.0)),
                       ("nkg_multi_adagrad_step", (None, None, g.ext(24), 0.0, 1e-10, 0.0, 0.0, 1.0))):
        g.expect_error(lambda: g.ck(getattr(g.lib, name)(hs, 3, *args)))


def one_parameter_variants(g):
    """each optimizer variant on one parameter after a backward pass, then a step after zero_grad(), whose deferred
    zero fill the step materialises"""
    x = g.leaf((3, 6), BF16)
    w = g.param((4, 6), BF16, F32)
    s = x.mm_t(w).sum()
    s.forward()
    s.backward(1.0)
    spec = [(24, BF16, F32)]
    hs, hyper = _arr([w.h.value]), g.ext(24)
    g.ck(g.lib.nkg_multi_sgd_step(hs, 1, _states(g, spec), _masters(g, spec), hyper, 0.01, 0.9, 0.0, 1, 0.5))
    g.ck(g.lib.nkg_multi_sgd_step(hs, 1, None, None, hyper, 0.01, 0.0, 0.0, 0, 0.5))
    g.ck(g.lib.nkg_multi_adam_step(hs, 1, _states(g, spec), _states(g, spec), _states(g, spec), _masters(g, spec), hyper,
                                   0.9, 0.999, 1e-8, 0.0, 0.01, 1.0))
    g.ck(g.lib.nkg_multi_adam_step(hs, 1, _states(g, spec), _states(g, spec), None, None, hyper, 0.9, 0.999, 1e-8, 0.0,
                                   0.01, 1.0))
    g.ck(g.lib.nkg_multi_rmsprop_step(hs, 1, _states(g, spec), _states(g, spec), _states(g, spec), None, hyper, 0.99,
                                      1e-8, 0.5, 0.001, 0.0, 1.0))
    g.ck(g.lib.nkg_multi_rmsprop_step(hs, 1, _states(g, spec), None, None, None, hyper, 0.99, 1e-8, 0.0, 0.001, 0.0,
                                      1.0))
    g.ck(g.lib.nkg_multi_adagrad_step(hs, 1, _states(g, spec), None, hyper, 0.1, 1e-10, 0.0, 0.0, 0.25))
    w.zero_grad()
    g.ck(g.lib.nkg_multi_sgd_step(hs, 1, None, None, hyper, 0.01, 0.0, 0.0, 0, 0.5))


SCENARIOS = {"adam_mixed": adam_mixed, "sgd_pairs": sgd_pairs, "rmsprop_pairs": rmsprop_pairs,
             "adagrad_twice": adagrad_twice, "not_differentiable": not_differentiable,
             "one_parameter_variants": one_parameter_variants}


@pytest.fixture(scope="module")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace_optim_multi"))))


def calls(lines):
    return [re.match(r"[\w ]+", l).group(0).strip() for l in lines[:-1]]


def table(line, name, field):
    """one host-array argument of a traced nk_multi_* call, by position in the header's parameter list"""
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


def test_one_call_per_64_tensors_per_dtype_group_in_parameter_order(graph):
    lines = graph.run(adam_mixed)
    names = [n for n in calls(lines) if n not in ("nk_alloc", "nk_alloc_uninit")]
    assert names == ["nk_optim_prologue"] + ["nk_multi_adam_step"] * 3
    multi = [l for l in lines if l.startswith("nk_multi_adam_step(")]
    f32_idx = [i for i, (_, dt, _) in enumerate(MIXED) if dt == F32]
    bf16_idx = [i for i, (_, dt, _) in enumerate(MIXED) if dt == BF16]
    counts = [int(table(l, "nk_multi_adam_step", "count")) for l in multi]
    assert counts == [PER_LAUNCH, len(f32_idx) - PER_LAUNCH, len(bf16_idx)]
    sizes = [json.loads(table(l, "nk_multi_adam_step", "n")) for l in multi]
    assert sizes == [[MIXED[i][0] for i in f32_idx[:PER_LAUNCH]], [MIXED[i][0] for i in f32_idx[PER_LAUNCH:]],
                     [MIXED[i][0] for i in bf16_idx]]
    dtypes = [(table(l, "nk_multi_adam_step", "w_dtype"), table(l, "nk_multi_adam_step", "g_dtype")) for l in multi]
    assert dtypes == [(str(F32), str(F32))] * 2 + [(str(BF16), str(F32))]
    masters = [table(l, "nk_multi_adam_step", "master") for l in multi]
    assert masters[0] == "[" + ",".join(["0"] * PER_LAUNCH) + "]" and "0" not in masters[2].strip("[]").split(",")


def test_dtype_groups_in_order_of_first_appearance(graph):
    lines = graph.run(sgd_pairs)
    multi = [l for l in lines if l.startswith("nk_multi_sgd_step(")]
    got = [(table(l, "nk_multi_sgd_step", "w_dtype"), table(l, "nk_multi_sgd_step", "g_dtype"),
            json.loads(table(l, "nk_multi_sgd_step", "n"))) for l in multi]
    assert got == [(str(F32), str(F32), [5, 9]), (str(BF16), str(BF16), [6]), (str(BF16), str(F32), [7, 10]),
                   (str(F32), str(BF16), [8])]
    assert "nk_optim_prologue" not in calls(lines)          # SGD reads lr straight from the block


def test_prologue_once_per_step(graph):
    names = calls(graph.run(adagrad_twice))
    names = [n for n in names if n not in ("nk_alloc", "nk_alloc_uninit")]
    assert names == ["step 0", "nk_optim_prologue", "nk_multi_adagrad_step"] * 1 + \
        ["step 1", "nk_optim_prologue", "nk_multi_adagrad_step"]


def test_non_differentiable_parameter_launches_nothing(graph):
    lines = graph.run(not_differentiable)
    errors = [l for l in lines if l.startswith("error ")]
    assert len(errors) == 4 and all("parameter 1 is not differentiable" in e for e in errors), errors
    after = lines[lines.index(errors[0]):]       # the leaves' own allocations come before
    assert not any(l.startswith(("nk_multi_", "nk_optim_prologue", "nk_alloc")) for l in after), after
