#!/usr/bin/env python
"""Transcribe the reference's concatenation goldens into tensors_cat.json: node/concatenate/test.rs (enabled) and the
disabled node/{multi_concatenate,stack,multi_stack,unsqueeze}/test.rs, whose numbers still state the intended results.

Same rules as make_goldens.py (whose parser this reuses): nothing is computed, every number is lifted verbatim from the
reference's test.rs together with the file:line it came from.  Per test fn, in source order:
  - "arrays": every array expression -- `new_input` / `new_backward_input` / `new_tensor` / `from_shape_vec` literals,
    `Array::linspace(a, b, n).into_shape(s)`, `Array::zeros(s)` / `Array::ones(s)` / `Array::from_elem(s, v)` -- with
    its kind and line;
  - "nodes": every `Name::new(...)` constructor with its first and last line and its integer-literal arguments in order (the
    axis, and the split offset of ConcatenateBackwardRight).

    NK_REFERENCE=<reference checkout> python tests/golden/make_goldens_cat.py
"""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens as MG  # noqa: E402

FILES = ["concatenate", "multi_concatenate", "stack", "multi_stack", "unsqueeze"]
SHAPE = r"\(?([\d,\s]+?)\)?"
ARRAY = re.compile(
    rf"(?P<lit>(?:new_input|new_backward_input|new_tensor|from_shape_vec))\(\s*{SHAPE}\s*,\s*vec!\[(?P<vals>[^\]]*)\]"
    rf"|Array::linspace\(\s*(?P<a>{MG.NUM})\.?\s*,\s*(?P<b>{MG.NUM})\.?\s*,\s*(?P<n>\d+)\s*\)\s*\.into_shape\(\(([^)]*)\)\)"
    rf"|(?:Array|Tensor)::(?P<fill>zeros|ones)\(\s*(?:\((?P<fshape>[\d,\s]+)\)|(?P<fshape1>\d+))\s*\)"
    rf"|(?:Array|Tensor)::from_elem\(\s*(?:\((?P<eshape>[\d,\s]+)\)|(?P<eshape1>\d+))\s*,\s*(?P<ev>{MG.NUM})\.?\s*\)",
    re.S)
NODE = re.compile(r"\b([A-Z]\w*)::new\(")


def line_of(text, pos):
    return text.count("\n", 0, pos) + 1


def arrays(text, start, body):
    out = []
    for m in ARRAY.finditer(body):
        line = line_of(text, start + m.start())
        if m.group("lit"):
            shape = MG.tuple_ints(m.group(2))
            vals = MG.parse_vec(m.group("vals"))
            out.append({"kind": m.group("lit"), "shape": shape, "values": vals, "line": line})
        elif m.group("a") is not None:
            out.append({"kind": "linspace", "start": float(m.group("a")), "stop": float(m.group("b")),
                        "num": int(m.group("n")), "shape": MG.tuple_ints(m.group(7)), "line": line})
        elif m.group("fill"):
            out.append({"kind": m.group("fill"), "shape": MG.tuple_ints(m.group("fshape") or m.group("fshape1")), "line": line})
        else:
            out.append({"kind": "from_elem", "shape": MG.tuple_ints(m.group("eshape") or m.group("eshape1")), "value": float(m.group("ev")),
                        "line": line})
    return out


def nodes(text, start, body):
    out = []
    for m in NODE.finditer(body):
        depth, i = 1, m.end()
        while depth and i < len(body):
            depth += (body[i] == "(") - (body[i] == ")")
            i += 1
        args, parts, depth, cur = body[m.end():i - 1], [], 0, ""
        for c in args:
            if c in "([{":
                depth += 1
            elif c in ")]}":
                depth -= 1
            if c == "," and depth == 0:
                parts.append(cur.strip())
                cur = ""
            else:
                cur += c
        parts.append(cur.strip())
        ints = [int(p) for p in parts if re.fullmatch(r"\d+", p)]
        out.append({"name": m.group(1), "first_line": line_of(text, start + m.start()),
                    "last_line": line_of(text, start + i - 1), "int_args": ints})
    return out


def gen():
    out = {}
    for f in FILES:
        path = os.path.join(MG.NV, f, "test.rs")
        text = open(path).read()
        per_fn = {}
        for name, line, body in MG.fn_blocks(text):
            start = text.index(body, sum(len(l) + 1 for l in text.split("\n")[:line - 1]))
            mod = "backward" if "mod backward" in text[:start] and text.rfind("mod backward", 0, start) > text.rfind(
                "mod forward", 0, start) else "forward"
            arr = arrays(text, start, body)
            if not arr:
                continue
            per_fn.setdefault(f"{mod}::{name}", []).append({
                "source": f"neuronika-variable/src/node/{f}/test.rs:{line}",
                "arrays": arr, "nodes": nodes(text, start, body)})
        out[f] = per_fn
    return out


def main():
    if not os.path.isdir(MG.REF):
        sys.exit(f"{MG.REF} not present: goldens can only be regenerated where the reference is mounted")
    data = gen()
    with open(os.path.join(HERE, "tensors_cat.json"), "w") as fh:
        json.dump(data, fh, indent=0, separators=(",", ":"))
    for f, d in data.items():
        print(f, {k: [(len(b["arrays"]), [n["int_args"] for n in b["nodes"]]) for b in v] for k, v in d.items()})


if __name__ == "__main__":
    main()
