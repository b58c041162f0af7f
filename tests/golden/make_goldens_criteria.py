#!/usr/bin/env python
"""Transcribe the reference's dropout and criterion goldens into tensors_criteria.json: node/dropout/test.rs,
node/absolute_error/test.rs and node/bce/test.rs (enabled), and node/bce_with_logits/test.rs and node/kldiv/test.rs
(disabled; their numbers still state the intended results).

Same rules as make_goldens.py (whose fn-block parser this reuses): nothing is computed, every number is lifted verbatim
from the reference's test.rs with the file:line of its test fn.  Per test fn, in source order:
  - "arrays": `Array::linspace(a, b, n)` (with its `.into_shape` shape, if any), `from_shape_vec(shape, vec![..])`,
    `new_input(shape, vec![..])` / `new_backward_input(shape, vec![..])` and `Array::zeros` / `ones` / `from_elem`;
  - "vecs": every other `vec![..]` literal (kldiv's input is `ln` of one, which the test applies);
  - "arr0": every `arr0(v)` value (seeds and expected losses);
  - "reductions": every `Reduction::Mean` / `Reduction::Sum`;
  - "probabilities": the float literals among a `Dropout::new(..)` / `DropoutBackward::new(..)` call's arguments.

    NK_REFERENCE=<reference checkout> python tests/golden/make_goldens_criteria.py
"""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens as MG  # noqa: E402

FILES = ["dropout", "absolute_error", "bce", "bce_with_logits", "kldiv"]
NUM = r"-?\d+(?:\.\d*)?(?:[eE]-?\d+)?(?:_?f32)?"
SHAPE = r"\(?(?P<shape>[\d,\s]+?)\)?"
ARRAY = re.compile(
    rf"Array::linspace\(\s*(?P<a>{NUM})\s*,\s*(?P<b>{NUM})\s*,\s*(?P<n>\d+)\s*\)(?:\s*\.into_shape\(\s*\((?P<ls>[^)]*)\)\s*\))?"
    rf"|(?P<lit>from_shape_vec|new_input|new_backward_input)\(\s*{SHAPE}\s*,\s*vec!\[(?P<vals>[^\]]*)\]"
    rf"|Array::(?P<fill>zeros|ones)\(\s*(?:\((?P<fshape>[\d,\s]*)\)|(?P<fshape1>\d+))\s*\)"
    rf"|Array::from_elem\(\s*(?:\((?P<eshape>[\d,\s]+)\)|(?P<eshape1>\d+))\s*,\s*(?P<ev>{NUM})\s*\)",
    re.S)
VEC = re.compile(r"vec!\[([^\]]*)\]", re.S)
ARR0 = re.compile(rf"arr0\(\s*({NUM})\s*\)")
RED = re.compile(r"Reduction::(Mean|Sum)")
DROPOUT_NEW = re.compile(r"\bDropout(?:Backward)?::new\(")


def num(s):
    return float(re.sub(r"_?f32$", "", s))


def parse_fn(body):
    arrays, covered = [], []
    for m in ARRAY.finditer(body):
        covered.append((m.start(), m.end()))
        if m.group("a") is not None:
            arrays.append({"kind": "linspace", "start": num(m.group("a")), "stop": num(m.group("b")),
                           "num": int(m.group("n")), "shape": MG.tuple_ints(m.group("ls")) if m.group("ls") else None})
        elif m.group("lit"):
            arrays.append({"kind": m.group("lit"), "shape": MG.tuple_ints(m.group("shape")),
                           "values": MG.parse_vec(m.group("vals"))})
        elif m.group("fill"):
            arrays.append({"kind": m.group("fill"), "shape": MG.tuple_ints(m.group("fshape") or m.group("fshape1") or "")})
        else:
            arrays.append({"kind": "from_elem", "shape": MG.tuple_ints(m.group("eshape") or m.group("eshape1")),
                           "value": num(m.group("ev"))})
    vecs = [MG.parse_vec(m.group(1)) for m in VEC.finditer(body)
            if not any(a <= m.start() < b for a, b in covered)]
    probs = []
    for m in DROPOUT_NEW.finditer(body):
        depth, i = 1, m.end()
        while depth:
            depth += (body[i] == "(") - (body[i] == ")")
            i += 1
        args = body[m.end():i - 1]
        while re.search(r"\([^()]*\)", args):   # the call's own arguments only
            args = re.sub(r"\([^()]*\)", "", args)
        probs += [num(v) for v in re.findall(rf"(?<![\w.])({NUM})(?=\s*,|\s*$)", args)]
    return {"arrays": arrays, "vecs": vecs, "arr0": [num(v) for v in ARR0.findall(body)],
            "reductions": RED.findall(body), "probabilities": probs}


def main():
    ref = os.environ.get("NK_REFERENCE")
    if not ref:
        sys.exit("set NK_REFERENCE to a checkout of the reference")
    out = {}
    for name in FILES:
        rel = f"neuronika-variable/src/node/{name}/test.rs"
        text = open(os.path.join(ref, rel)).read()
        cases = {}
        for fn, line, body in MG.fn_blocks(text):
            if fn in cases:   # `mod forward` and `mod backward` both have `creation` etc.: keep both
                fn = f"{fn}@{line}"
            cases[fn] = {"source": f"{rel}:{line}", **parse_fn(body)}
        out[name] = cases
    path = os.path.join(HERE, "tensors_criteria.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1)
        fh.write("\n")
    print("wrote", path, {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
