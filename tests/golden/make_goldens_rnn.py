#!/usr/bin/env python
"""Transcribe the reference's chunk goldens (neuronika-variable/src/node/chunk/test.rs) into tensors_rnn.json.

Same rules as make_goldens.py (whose parser this reuses): nothing is computed, every number is lifted verbatim from the
reference's test.rs together with the file:line it came from.  Per test fn: the `from_shape_vec` literals in order,
the chunk indices passed to Chunk::new / ChunkBackward::new in order, and the `Array::linspace(a, b, n).into_shape(s)`
operands.  The reference has no tests of its recurrent cells.

    NK_REFERENCE=<reference checkout> python tests/golden/make_goldens_rnn.py
"""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens as MG  # noqa: E402

LINSPACE = re.compile(rf"Array::linspace\(\s*({MG.NUM})\s*,\s*({MG.NUM})\s*,\s*(\d+)\s*\)\s*\.into_shape\(\(([^)]*)\)\)")
INDEX = re.compile(r"\b(Chunk|ChunkBackward)::new\(.*?,\s*(\d+),?\s*\)\s*;", re.S)


def gen_chunk():
    out = MG.gen_tensors(["chunk"])["chunk"]
    text = open(os.path.join(MG.NV, "chunk", "test.rs")).read()
    for name, line, body in MG.fn_blocks(text):
        for blk in out.get(name, []):
            if blk["source"].endswith(f":{line}"):
                blk["indices"] = [int(m.group(2)) for m in INDEX.finditer(body)]
                blk["linspace"] = [{"start": float(m.group(1)), "stop": float(m.group(2)), "num": int(m.group(3)),
                                    "shape": MG.tuple_ints(m.group(4))} for m in LINSPACE.finditer(body)]
    return out


def main():
    if not os.path.isdir(MG.REF):
        sys.exit(f"{MG.REF} not present: goldens can only be regenerated where the reference is mounted")
    chunk = gen_chunk()
    with open(os.path.join(HERE, "tensors_rnn.json"), "w") as fh:
        json.dump({"chunk": chunk}, fh, indent=0, separators=(",", ":"))
    print("chunk", {k: [(len(b["tensors"]), b.get("indices")) for b in v] for k, v in chunk.items()})


if __name__ == "__main__":
    main()
