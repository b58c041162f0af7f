#!/usr/bin/env python
"""Write graph_trace_clip.json: the kernel-ABI call traces of the gradient-clipping graph entry points
(the scenarios of tests/test_graph_trace_clip.py), recorded as make_graph_trace.py records the graph's.

    python tests/golden/make_graph_trace_clip.py"""
from __future__ import annotations

import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import graph_trace as T  # noqa: E402
import test_graph_trace_clip as M  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as tmp:
        g = T.Graph(T.build_library(tmp))
        traces = {name: g.run(fn) for name, fn in M.SCENARIOS.items()}
    with open(M.GOLDEN, "w") as fh:
        json.dump(traces, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print("%d scenarios, %d calls -> %s" % (len(traces), sum(len(t) for t in traces.values()), M.GOLDEN))


if __name__ == "__main__":
    main()
