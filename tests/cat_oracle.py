"""numpy oracle of concatenation: `cat` / `stack` forward and backward, and `unsqueeze`
(neuronika-variable/src/node/{multi_concatenate,multi_stack,unsqueeze}/mod.rs).

The backward functions add into the given gradient buffers, one operand after the other, as the reference's loops do;
an operand whose buffer is None gets nothing.  Kept beside its tests, like rnn_oracle.py, so the oracle/ package stays
as it is."""
from __future__ import annotations

import numpy as np


def cat_forward(xs, axis):
    """MultiConcatenate::forward: the operands side by side along `axis`"""
    return np.concatenate([np.asarray(x) for x in xs], axis=axis)


def cat_backward(g, grads, axis, lens=None):
    """MultiConcatenateBackward::backward: grads[i] += slice i of g along `axis`.  `lens` gives each operand's length
    along `axis` (needed only when some buffer is None)."""
    g = np.asarray(g)
    lens = [np.shape(d)[axis] for d in grads] if lens is None else list(lens)
    start = 0
    for d, n in zip(grads, lens):
        if d is not None:
            d += np.take(g, np.arange(start, start + n), axis=axis)
        start += n
    return grads


def stack_forward(xs, axis):
    """MultiStack::forward: the operands (one shape) along a new axis"""
    return np.stack([np.asarray(x) for x in xs], axis=axis)


def stack_backward(g, grads, axis):
    """MultiStackBackward::backward: grads[i] += g.index_axis(axis, i)"""
    g = np.asarray(g)
    for i, d in enumerate(grads):
        if d is not None:
            d += np.take(g, i, axis=axis)
    return grads


def unsqueeze(x, axis):
    """Unsqueeze::forward (and, reshaped back, its backward): a new axis of length 1"""
    return np.expand_dims(np.asarray(x), axis)


def golden_array(a):
    """an array expression of tests/golden/tensors_cat.json as float32"""
    shape = tuple(a["shape"])
    k = a["kind"]
    if k == "linspace":
        return np.linspace(a["start"], a["stop"], a["num"]).astype(np.float32).reshape(shape)
    if k == "zeros":
        return np.zeros(shape, np.float32)
    if k == "ones":
        return np.ones(shape, np.float32)
    if k == "from_elem":
        return np.full(shape, a["value"], np.float32)
    return np.asarray(a["values"], np.float32).reshape(shape)
