#!/usr/bin/env python
"""Write graph_trace.json: the kernel-ABI call trace of every scenario of tests/graph_trace.py, recorded from
neuronika_b200/csrc/nk_graph.cpp compiled against a recording stub of include/nk_b200.h (no GPU needed).

    python tests/golden/make_graph_trace.py [--graph-src other/nk_graph.cpp] [--out path.json]

Regenerate it when a change to the graph is meant to change which kernels it launches, with which arguments or in
which order, and review the diff of the golden: it is exactly that change."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import graph_trace as T  # noqa: E402


def record(graph_src=T.GRAPH_SRC):
    with tempfile.TemporaryDirectory() as tmp:
        g = T.Graph(T.build_library(tmp, graph_src))
        return {name: g.run(fn) for name, fn in T.SCENARIOS.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--graph-src", default=T.GRAPH_SRC)
    ap.add_argument("--out", default=T.GOLDEN)
    args = ap.parse_args()
    traces = record(args.graph_src)
    with open(args.out, "w") as fh:
        json.dump(traces, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%d scenarios, %d calls -> %s" % (len(traces), sum(len(t) for t in traces.values()), args.out))


if __name__ == "__main__":
    main()
