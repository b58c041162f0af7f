#!/usr/bin/env python
"""Transcribe the reference's learning-rate scheduler tests (neuronika-optim/src/lr_scheduler/*/test.rs) into
lr_scheduler.json.

Per test: the optimizer's initial lr (`StochasticGD::new(lr, ...)`), the scheduler constructor's arguments as written,
EPOCHS, the epochs passed to set_current_epoch, and every `get_*_lr() - <value>` assertion with its source line.  The
values are the literals of the test (`16_f32`), or `b_f32.powi(e)` written out as b**e (exact in f32 for these
operands); an assertion inside the epoch loop (`2_f32.powi(epoch as i32)`, `epoch as f32`) is kept as its expression
with the loop variable, together with the loop's guard when it has one.

    NK_REFERENCE=<reference checkout> python tests/golden/make_goldens_lr_scheduler.py
"""
from __future__ import annotations

import json
import os
import re
import sys

REF = os.environ.get("NK_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "neuronika-optim", "src", "lr_scheduler")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lr_scheduler.json")
TESTS = {"step_lr": "StepLR", "multi_step_lr": "MultiStepLR", "exponential_lr": "ExponentialLR",
         "multiplicative_lr": "MultiplicativeLR", "lambda_lr": "LambdaLR"}


def value(expr):
    """`16_f32`, `2_f32.powi(4)` -> number; anything with the loop variable stays an expression"""
    m = re.fullmatch(r"(\d+)_f32(?:\.powi\((\d+)\))?", expr.strip())
    if m:
        return float(int(m.group(1)) ** int(m.group(2) or 1))
    return None


def transcribe(mod, cls):
    path = os.path.join(SRC, mod, "test.rs")
    lines = open(path).read().splitlines()
    text = "\n".join(lines)
    rel = os.path.relpath(path, REF)
    out = {"source": rel, "scheduler": cls}
    out["optimizer_lr"] = float(re.search(r"StochasticGD::new\(\s*([\d.]+)", text).group(1))
    ctor = re.search(cls + r"::new\(&optim,\s*(.*)\);", text).group(1)
    out["args"] = ctor
    out["epochs"] = int(re.search(r"const EPOCHS: usize = (\d+);", text).group(1))
    out["set_current_epoch"] = [int(v) for v in re.findall(r"set_current_epoch\((\d+)\)", text)]
    asserts, guard = [], None
    for no, line in enumerate(lines, 1):
        g = re.search(r"if (epoch > \d+)", line)
        if g:
            guard = g.group(1)
        m = re.search(r"get_(last|current)_lr\(\) - (.*?)\)\.abs\(\) <= f32::EPSILON", line)
        if m:
            expr = m.group(2).strip()
            if expr.startswith("(") and not expr.endswith(")"):
                expr = expr[1:]
            in_loop = "epoch" in expr
            asserts.append({"line": f"{rel}:{no}", "which": m.group(1), "expr": expr, "value": value(expr),
                            "in_loop": in_loop, "guard": guard if in_loop else None})
    out["asserts"] = asserts
    return out


def main():
    if not os.path.isdir(SRC):
        sys.exit(f"{SRC} not present: goldens can only be regenerated where the reference is mounted")
    data = {mod: transcribe(mod, cls) for mod, cls in TESTS.items()}
    with open(OUT, "w") as fh:
        json.dump(data, fh, indent=1)
        fh.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
