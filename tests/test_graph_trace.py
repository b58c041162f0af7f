"""The host-side graph (neuronika_b200/csrc/nk_graph.cpp) makes exactly the kernel-ABI calls recorded in
tests/golden/graph_trace.json, scenario by scenario: same functions, same arguments, same order, same hook timing and
the same error messages.  The graph is compiled with the host C++ compiler against a recording stub of nk_b200.h
(tests/graph_trace.py), so this runs without a GPU.  Fusion decisions show up here and nowhere else: a lost fusion
changes no result, only the launches."""
import json

import pytest

import graph_trace as T


@pytest.fixture(scope="session")
def graph(tmp_path_factory):
    if T.compiler() is None:
        pytest.skip("no host C++ compiler (g++, c++ or clang++) to build the graph against the ABI stub")
    return T.Graph(T.build_library(str(tmp_path_factory.mktemp("graph_trace"))))


@pytest.fixture(scope="session")
def golden():
    with open(T.GOLDEN) as fh:
        return json.load(fh)


def test_every_scenario_has_a_golden(golden):
    assert sorted(golden) == sorted(T.SCENARIOS)


@pytest.mark.parametrize("name", sorted(T.SCENARIOS))
def test_trace_matches_golden(graph, golden, name):
    got = graph.run(T.SCENARIOS[name])
    want = golden[name]
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, "%s: first difference at call %d:\n  got  %s\n  want %s" % (name, i, a, b)
    assert len(got) == len(want), "%s: %d calls, golden has %d" % (name, len(got), len(want))
