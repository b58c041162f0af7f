"""The numpy oracle of concatenation (tests/cat_oracle.py), pinned on the CPU against the reference's own test vectors
(tests/golden/tensors_cat.json: node/concatenate, multi_concatenate, stack, multi_stack and unsqueeze), bit for bit,
and against the identities cat(chunks(x)) == x and stack == cat of unsqueezed operands."""
import json
import os

import numpy as np
import pytest

import cat_oracle as O
import rnn_oracle as R

F32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tensors_cat.json")


@pytest.fixture(scope="module")
def goldens():
    with open(GOLDEN) as fh:
        return json.load(fh)


def same(got, want, what):
    assert got.shape == want.shape and np.array_equal(got, want), (what, got, want)


def block(goldens, f, name):
    (b,) = goldens[f][name]
    return b


# ------------------------------------------------------------------------------ node/concatenate (enabled)
@pytest.mark.parametrize("name", ["forward::rows", "forward::columns"])
def test_concatenate_forward(goldens, name):
    b = block(goldens, "concatenate", name)
    arrs = [O.golden_array(a) for a in b["arrays"]]
    axis = b["nodes"][0]["int_args"][0]
    same(O.cat_forward(arrs[:2], axis), arrs[3], b["source"])


@pytest.mark.parametrize("name", ["backward::left_rows", "backward::left_columns", "backward::right_rows",
                                  "backward::right_columns"])
def test_concatenate_backward_one_side(goldens, name):
    b = block(goldens, "concatenate", name)
    g, once, twice = (O.golden_array(a) for a in b["arrays"])
    args = b["nodes"][0]["int_args"]
    axis = args[0]
    n = once.shape[axis]
    grad = np.zeros_like(once)
    if "left" in name:
        grads, lens = [grad, None], [n, g.shape[axis] - n]
    else:
        grads, lens = [None, grad], [args[1], g.shape[axis] - args[1]]
    O.cat_backward(g, grads, axis, lens)
    same(grad, once, b["source"])
    O.cat_backward(g, grads, axis, lens)
    same(grad, twice, b["source"])


def test_concatenate_backward_base_case(goldens):
    b = block(goldens, "concatenate", "backward::base_case")
    g, l1, r1, l2, r2 = (O.golden_array(a) for a in b["arrays"])
    axis = b["nodes"][2]["int_args"][0]
    grads = [np.zeros_like(l1), np.zeros_like(r1)]
    O.cat_backward(g, grads, axis)
    same(grads[0], l1, "left once")
    same(grads[1], r1, "right once")
    O.cat_backward(g, grads, axis)
    same(grads[0], l2, "left twice")
    same(grads[1], r2, "right twice")


# ------------------------------------------------------------------------------ disabled multi / stack / unsqueeze tests
def node_of(b):
    return b["nodes"][0]


def after(b, arrays):
    last = node_of(b)["last_line"]
    return [(a, O.golden_array(a)) for a in arrays if a["line"] > last]


FORWARD = [("multi_concatenate", "forward::forward", "cat"), ("stack", "forward::forward_rows", "stack"),
           ("stack", "forward::forward_columns", "stack"), ("multi_stack", "forward::forward", "stack"),
           ("unsqueeze", "forward::forward_rows", "unsqueeze"), ("unsqueeze", "forward::forward_columns", "unsqueeze"),
           ("unsqueeze", "forward::forward_depths", "unsqueeze")]


def run_forward(op, xs, axis):
    if op == "cat":
        return O.cat_forward(xs, axis)
    if op == "stack":
        return O.stack_forward(xs, axis)
    return O.unsqueeze(xs[0], axis)


@pytest.mark.parametrize("f,name,op", FORWARD)
def test_forward_goldens(goldens, f, name, op):
    """first evaluation, and the evaluation after the first operand was incremented by one"""
    b = block(goldens, f, name)
    axis = node_of(b)["int_args"][0]
    xs = [O.golden_array(a) for a in b["arrays"] if a["kind"] == "new_input"]
    want = run_forward(op, xs, axis)
    outs = [v for a, v in after(b, b["arrays"]) if v.shape == want.shape]
    same(want, outs[0], b["source"] + " first evaluation")
    same(run_forward(op, [xs[0] + 1] + xs[1:], axis), outs[-1], b["source"] + " second evaluation")


BACKWARD = [("multi_concatenate", "backward::backward", "cat"), ("stack", "backward::backward_rows", "stack"),
            ("stack", "backward::backward_columns", "stack"), ("stack", "backward::backward_left_rows", "stack"),
            ("stack", "backward::backward_left_columns", "stack"), ("stack", "backward::backward_right_rows", "stack"),
            ("stack", "backward::backward_right_columns", "stack"), ("multi_stack", "backward::backward", "stack"),
            ("unsqueeze", "backward::backward_rows", "unsqueeze"),
            ("unsqueeze", "backward::backward_columns", "unsqueeze"),
            ("unsqueeze", "backward::backward_depths", "unsqueeze")]


@pytest.mark.parametrize("f,name,op", BACKWARD)
def test_backward_goldens(goldens, f, name, op):
    """one backward, a second one (accumulate), then one onto cleared gradients (the reference's overwrite)"""
    b = block(goldens, f, name)
    node = node_of(b)
    axis = node["int_args"][0]
    diff = [O.golden_array(a) for a in b["arrays"] if a["kind"] == "new_backward_input"]
    n_ops = 2 if op == "stack" else len(diff)
    side = 0 if node["name"].endswith("Left") else 1 if node["name"].endswith("Right") else None
    tail = after(b, b["arrays"])
    seed = tail[0][1]
    expect = [v for _, v in tail[1:] if v.shape != seed.shape]
    grads = [np.zeros_like(d) for d in diff]

    def backward():
        bufs = list(grads) if side is None else [grads[0] if i == side else None for i in range(n_ops)]
        if op == "cat":
            O.cat_backward(seed, bufs, axis)
        elif op == "stack":
            O.stack_backward(seed, bufs, axis)
        else:
            bufs[0] += seed.reshape(bufs[0].shape)

    rounds = [expect[i:i + len(grads)] for i in range(0, len(expect), len(grads))]
    assert len(rounds) == 3, (b["source"], len(expect))
    for r, want in enumerate(rounds):
        if r == 2:
            for d in grads:
                d[...] = 0
        backward()
        for d, w in zip(grads, want):
            same(d, w, f"{b['source']} round {r}")


# ------------------------------------------------------------------------------ identities
@pytest.mark.parametrize("shape,chunk_shape,axis", [((6, 4), (2, 4), 0), ((3, 8), (3, 2), 1),
                                                    ((2, 6, 5), (2, 3, 5), 1), ((4, 3, 10), (4, 3, 1), 2)])
def test_cat_inverts_chunks(shape, chunk_shape, axis):
    """chunks along one axis, cat back: the original bit for bit; gradients make the same round trip"""
    x = np.random.default_rng(1).standard_normal(shape).astype(F32)
    parts = R.chunks(x, chunk_shape)
    same(O.cat_forward(parts, axis), x, "cat(chunks(x))")
    g = np.random.default_rng(2).standard_normal(shape).astype(F32)
    grads = [np.zeros_like(p) for p in parts]
    O.cat_backward(g, grads, axis)
    dx = np.zeros_like(x)
    for i, d in enumerate(grads):
        R.chunk_backward(dx, d, i)
    same(dx, g, "chunk backward of the cat backward")


@pytest.mark.parametrize("shape", [(3,), (2, 5), (2, 3, 4)])
def test_stack_is_cat_of_unsqueezed(shape):
    rng = np.random.default_rng(3)
    xs = [rng.standard_normal(shape).astype(F32) for _ in range(3)]
    for axis in range(len(shape) + 1):
        same(O.stack_forward(xs, axis), O.cat_forward([O.unsqueeze(x, axis) for x in xs], axis), f"axis {axis}")
        g = rng.standard_normal(O.stack_forward(xs, axis).shape).astype(F32)
        a = O.stack_backward(g, [np.zeros(shape, F32) for _ in xs], axis)
        c = O.cat_backward(g, [np.zeros(O.unsqueeze(x, axis).shape, F32) for x in xs], axis)
        for u, v in zip(a, c):
            same(u, v.reshape(shape), f"backward axis {axis}")
