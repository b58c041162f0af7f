#!/usr/bin/env python
"""Transcribe the reference's padding goldens into tensors_pad.json: node/pad/{reflective,replicative,constant,zero}/test.rs,
each an `Array::range` input padded by one mode and the exact padded array it must equal (reflective and replicative in
1-D, 2-D and 3-D; constant with fill 8 and zero in 2-D).

Same rules as make_goldens.py (whose number handling this reuses): nothing is computed, every number is lifted verbatim
from the reference's test.rs together with the file:line it came from.  Per test fn:
  - "base": `Array::range(start, stop, step)` and the `.into_shape(...)` it is given (the 1-D tests have none);
  - "padding": the `[..].into_dimension()` per-axis padding;
  - "fill": the argument of `Constant(v)` (the constant mode only);
  - "padded_shape": the `Array::zeros(..)` the padding writes into;
  - "expected": the nested `ndarray::array![..]` literal of the assert, as nested lists.

    NK_REFERENCE=<reference checkout> python tests/golden/make_goldens_pad.py
"""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens as MG  # noqa: E402

MODES = ["reflective", "replicative", "constant", "zero"]


def nested_array(text: str, start: int):
    """the `ndarray::array![ ... ]` literal whose `[` is at text[start], as nested lists of floats, and its end"""
    depth, i = 0, start
    while True:
        depth += (text[i] == "[") - (text[i] == "]")
        i += 1
        if depth == 0:
            break
    body = re.sub(r"//[^\n]*", "", text[start:i])
    body = re.sub(MG.NUM, lambda m: repr(float(m.group(0))), body)
    body = re.sub(r",\s*\]", "]", body)
    return json.loads(body), i


def shape_of(s: str):
    return MG.tuple_ints(s)


def gen_pad():
    out = {}
    for mode in MODES:
        rel = f"neuronika-variable/src/node/pad/{mode}/test.rs"
        text = open(os.path.join(MG.REF, rel)).read()
        cases = {}
        for name, line, body in MG.fn_blocks(text):
            m_base = re.search(rf"Array::range\(\s*({MG.NUM})\s*,\s*({MG.NUM})\s*,\s*({MG.NUM})\s*\)"
                               r"(?:\s*\.into_shape\(\(([\d,\s]+)\)\))?", body)
            m_zeros = re.search(r"Array::<f32,\s*_>::zeros\(\s*(\(?[\d,\s]+\)?)\s*\)", body)
            m_pad = re.search(r"\[([\d,\s]+)\]\s*\.into_dimension\(\)", body)
            m_fill = re.search(rf"Constant\(\s*({MG.NUM})\s*\)", body)
            m_arr = re.search(r"ndarray::array!\[", body)
            assert m_base and m_zeros and m_pad and m_arr, (mode, name)
            expected, _ = nested_array(body, m_arr.end() - 1)
            start, stop, step = (float(m_base.group(k)) for k in (1, 2, 3))
            case = {
                "source": f"{rel}:{line}",
                "expected_line": line + body.count("\n", 0, m_arr.start()),
                "base_range": [start, stop, step],
                "base_shape": shape_of(m_base.group(4)) if m_base.group(4) else [int((stop - start) / step)],
                "padding": shape_of(m_pad.group(1)),
                "padded_shape": shape_of(m_zeros.group(1)),
                "expected": expected,
            }
            if m_fill:
                case["fill"] = float(m_fill.group(1))
            cases[name] = case
        out[mode] = cases
    assert sorted(out["reflective"]) == sorted(out["replicative"]) == ["test_1d", "test_2d", "test_3d"], out.keys()
    assert list(out["constant"]) == list(out["zero"]) == ["test"]
    return out


def main():
    if not os.path.isdir(MG.REF):
        sys.exit(f"{MG.REF} not present: goldens can only be regenerated where the reference is mounted")
    pad = gen_pad()
    with open(os.path.join(HERE, "tensors_pad.json"), "w") as fh:
        json.dump(pad, fh, indent=0, separators=(",", ":"))
        fh.write("\n")
    for mode, cases in pad.items():
        print(mode, {k: (c["base_shape"], c["padding"], c["padded_shape"]) for k, c in cases.items()})


if __name__ == "__main__":
    main()
