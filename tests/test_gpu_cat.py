"""`cat` / `stack` / `unsqueeze` on the GPU: the two entry points of csrc/nk_cat.cu, the graph nodes and a model.

A concatenation is a copy and its backward one addition per element (f32 g + beta*dx, then one round-to-nearest-even
to bf16 for a bf16 gradient), so every operator and graph comparison here is bit exact against tests/cat_oracle.py.
Operator level: operands are views into canary-filled buffers at offset 0 (16-byte aligned: vector path) or 1 element
(element path); every element outside a view keeps its canary and outputs written with beta = 0 start as NaN."""
import math

import numpy as np
import pytest

import cat_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0
UB = 2.0 ** -8
OPS = 64   # NK_CAT_OPS_PER_LAUNCH


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


@pytest.fixture
def fusion(nk):
    yield nk.set_fusion
    nk.set_fusion(1)


def bf16_round(x):
    from oracle import bf16_round as r
    return r(np.asarray(x, F32))


def held(x, dt):
    x = np.asarray(x, F32)
    return bf16_round(x) if dt == "bf16" else x


def D(nk, dt):
    return nk.BF16 if dt == "bf16" else nk.F32


def bits_equal(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (what, f"{bad.size} of {got.size} differ", got.ravel()[bad[0]], want.ravel()[bad[0]])


class Guarded:
    """`data` (float32 values the storage type holds) at element `off` of a canary-filled device buffer"""

    def __init__(self, nk, dev, data, dt, off=0, tail=24):
        data = np.asarray(data, F32)
        self.shape, self.n, self.off = data.shape, data.size, off
        host = np.full(off + self.n + tail, CANARY, F32)
        host[off:off + self.n] = data.ravel()
        self.buf = dev.from_ndarray(host, D(nk, dt))
        self.view = self.buf.slice_flat(off, self.shape)

    def read(self):
        flat = self.buf.as_ndarray().ravel()
        outside = np.concatenate([flat[:self.off], flat[self.off + self.n:]])
        bad = np.flatnonzero(outside.view(np.uint32) != F32(CANARY).view(np.uint32))
        assert bad.size == 0, f"{bad.size} elements outside the view were written"
        return flat[self.off:self.off + self.n].reshape(self.shape)


def shapes_along(base, axis, lens):
    out = []
    for n in lens:
        s = list(base)
        s[axis] = n
        out.append(tuple(s))
    return out


def want_bwd(g_slice, d0, beta, dx_dt):
    """the kernel's arithmetic: f32 g + beta*dx (exact products for the betas used here), one rounding to dx's type"""
    v = np.asarray(g_slice, F32)
    if beta != 0:
        v = (v + F32(beta) * np.asarray(d0, F32)).astype(F32)
    return held(v, dx_dt)


def check_bwd(nk, dev, gv, dt_g, dx_dt, shapes, axis, off, rng, betas):
    """nk_cat_bwd over the given shapes; betas[i] None = NULL operand (its buffer must stay untouched)"""
    from neuronika_b200 import ops
    G = Guarded(nk, dev, gv, dt_g, off)
    d0 = [held(rng.standard_normal(s), dx_dt) for s in shapes]
    DX = [Guarded(nk, dev, d if b else np.full(s, np.nan, F32), dx_dt, off) for d, s, b in zip(d0, shapes, betas)]
    lens = [s[axis] for s in shapes]
    before = dev.launches
    ops.cat_bwd([X.view if b is not None else None for X, b in zip(DX, betas)], G.view, axis,
                [b or 0.0 for b in betas], lens=lens)
    launches = dev.launches - before
    slices, start = [], 0
    for n in lens:
        slices.append(np.take(gv, np.arange(start, start + n), axis=axis))
        start += n
    for i, (X, b) in enumerate(zip(DX, betas)):
        got = X.read()
        if b is None:
            bits_equal(got, np.full(shapes[i], np.nan, F32), f"NULL operand {i} untouched")
        else:
            bits_equal(got, want_bwd(slices[i], d0[i], b, dx_dt), f"dx[{i}] beta {b}")
    bits_equal(G.read(), gv, "g unchanged")
    return launches


# ------------------------------------------------------------------------------------------------ operator level
BASE = (3, 5, 8)
LENS = [4, 0, 1, 7, 2]


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("off", [0, 1])
def test_cat_fwd_ops(nk, dev, dt, axis, off):
    from neuronika_b200 import ops
    rng = np.random.default_rng(axis * 2 + off)
    shapes = shapes_along(BASE, axis, LENS)
    xs = [held(rng.standard_normal(s), dt) for s in shapes]
    X = [Guarded(nk, dev, x, dt, off) for x in xs]
    want = O.cat_forward(xs, axis)
    Y = Guarded(nk, dev, np.full(want.shape, np.nan, F32), dt, off)
    before = dev.launches
    ops.cat([x.view for x in X], axis, out=Y.view)
    assert dev.launches - before == 1
    bits_equal(Y.read(), want, "cat")
    for x, g in zip(xs, X):
        bits_equal(g.read(), x, "input unchanged")


@pytest.mark.parametrize("g_dt", ["f32", "bf16"])
@pytest.mark.parametrize("dx_dt", ["f32", "bf16"])
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("off", [0, 1])
def test_cat_bwd_ops(nk, dev, g_dt, dx_dt, axis, off):
    """every (g, dx) element-type pair, mixed betas and a NULL operand"""
    rng = np.random.default_rng([axis, off, len(g_dt), len(dx_dt)])
    shapes = shapes_along(BASE, axis, LENS)
    gv = held(rng.standard_normal(O.cat_forward([np.zeros(s) for s in shapes], axis).shape), g_dt)
    betas = [0.0, 1.0, None, 0.5, 2.0]
    assert check_bwd(nk, dev, gv, g_dt, dx_dt, shapes, axis, off, rng, betas) == 1


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("count", [1, 2, 64, 65, 130])
def test_cat_launches_per_64_operands(nk, dev, dt, count):
    """one launch per NK_CAT_OPS_PER_LAUNCH operands in each direction"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(count)
    lens = [(i * 7) % 4 for i in range(count)]   # lengths 0..3, every group of 64 holds non-empty ones
    for i in range(0, count, OPS):
        lens[i] = max(lens[i], 1)
    shapes = [(2, n, 3) for n in lens]
    xs = [held(rng.standard_normal(s), dt) for s in shapes]
    arrs = [dev.from_ndarray(x, D(nk, dt)) for x in xs]
    before = dev.launches
    y = ops.cat(arrs, 1)
    assert dev.launches - before == math.ceil(count / OPS)
    bits_equal(y.as_ndarray(), O.cat_forward(xs, 1), "cat")
    gv = held(rng.standard_normal(y.shape), dt)
    betas = [[0.0, 1.0, 0.5][i % 3] for i in range(count)]
    assert check_bwd(nk, dev, gv, dt, "f32", shapes, 1, 0, rng, betas) == math.ceil(count / OPS)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("case", ["rows", "interleave"])
def test_cat_past_one_wave(nk, dev, dt, case):
    """more CTAs (rows: the per-operand copy) or grid-stride iterations (interleave: the in-order gather) than one wave"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(9)
    wave = dev.sm_count * 8 * 256
    if case == "rows":
        shapes, axis = [(3, 16 * wave // 1000 + 1, 1000), (3, 1, 1000), (3, 8 * wave // 1000, 1000)], 1
        xs = [held(rng.standard_normal(s), dt) for s in shapes]
        y = ops.cat([dev.from_ndarray(x, D(nk, dt)) for x in xs], axis)
        want = O.cat_forward(xs, axis)
    else:
        xs = [held(rng.standard_normal(2 * wave + 3), dt) for _ in range(3)]
        shapes, axis = [(x.size, 1) for x in xs], 1
        y = ops.cat([dev.from_ndarray(x, D(nk, dt)).view(s) for x, s in zip(xs, shapes)], axis)
        want = O.stack_forward(xs, 1)
    bits_equal(y.as_ndarray().reshape(want.shape), want, "cat")
    gv = held(rng.standard_normal(want.shape), dt)
    check_bwd(nk, dev, gv.reshape(y.shape), dt, "bf16" if dt == "f32" else "f32", shapes, axis, 0, rng,
              [1.0, 0.0, 0.5])


def test_cat_output_past_2_31_elements(nk, dev):
    """(2, 2^30 + 29, 2) bf16 output: 64-bit row offsets; every slice boundary of both rows and sampled positions"""
    from neuronika_b200 import ops
    lens = [2 ** 29 + 8, 5, 2 ** 29 + 16]
    shapes = [(2, n, 2) for n in lens]
    a = dev.full(shapes[0], 1.0, nk.BF16)
    bv = np.arange(20, dtype=F32).reshape(shapes[1]) - 7
    b = dev.from_ndarray(bv, nk.BF16)
    c = dev.full(shapes[2], 3.0, nk.BF16)
    y = dev.full((2, sum(lens), 2), np.nan, nk.BF16)
    assert y.size > 2 ** 31
    ops.cat([a, b, c], 1, out=y)
    pitch = sum(lens) * 2
    cols = np.cumsum([0] + [n * 2 for n in lens])

    def owner(j):
        """expected value at output column j"""
        k = int(np.searchsorted(cols, j, side="right") - 1)
        return k, j - cols[k]

    def at(buf, flat, n=1):
        return buf.slice_flat(int(flat), (n,)).as_ndarray()

    def expect_y(o, j):
        k, c_ = owner(j)
        return [1.0, None, 3.0][k] if k != 1 else bv[o].ravel()[c_]

    positions = []
    for o in range(2):
        for edge in list(cols) + [pitch]:
            positions += [(o, j) for j in range(max(0, edge - 3), min(pitch, edge + 3))]
    rng = np.random.default_rng(0)
    positions += [(int(rng.integers(2)), int(rng.integers(pitch))) for _ in range(48)]
    for o, j in positions:
        assert at(y, o * pitch + j)[0] == expect_y(o, j), (o, j)
    # backward: the three slices back, a into f32, b and c into bf16, all with beta 0 (NaN beforehand)
    da = dev.full(shapes[0], np.nan, nk.F32)
    db = dev.full(shapes[1], np.nan, nk.BF16)
    dc = dev.full(shapes[2], np.nan, nk.BF16)
    ops.cat_bwd([da, db, dc], y, 1, [0.0, 0.0, 0.0])
    bits_equal(db.as_ndarray(), bv, "db")
    for d, val, n in ((da, 1.0, lens[0]), (dc, 3.0, lens[2])):
        per_row = n * 2
        for o in range(2):
            for j in [0, 1, 2, per_row - 3, per_row - 2, per_row - 1] + [int(v) for v in rng.integers(per_row, size=24)]:
                assert at(d, o * per_row + j)[0] == val, (o, j)


def test_cat_argument_errors(nk, dev):
    from neuronika_b200 import _lib as L
    a = dev.zeros((2, 3))
    xs = (L.vp * 2)(a.ptr.value, a.ptr.value)
    lens = (L.i64 * 2)(2, 2)
    bad = (L.i64 * 2)(2, -1)
    before = dev.launches
    assert L.lib.nk_cat_fwd(dev.ctx, a.ptr, xs, bad, 2, 1, 3, nk.F32) == -1
    assert "negative length" in L.last_error(dev.ctx)
    assert L.lib.nk_cat_fwd(dev.ctx, a.ptr, xs, lens, 2, 1, 3, 7) == -1
    dts = (L.i32 * 2)(nk.F32, nk.F32)
    betas = (L.f32 * 2)(0.0, 0.0)
    same = (L.vp * 2)(a.ptr.value, a.ptr.value)
    assert L.lib.nk_cat_bwd(dev.ctx, same, dts, betas, a.ptr, nk.F32, lens, 2, 1, 3) == -1
    assert "share one gradient" in L.last_error(dev.ctx)
    assert dev.launches == before


# ------------------------------------------------------------------------------------------------ graph level
@pytest.fixture(scope="module")
def goldens():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tensors_cat.json")) as fh:
        return json.load(fh)


golden_value = O.golden_array


@pytest.mark.parametrize("f,name,op", [("multi_concatenate", "forward::forward", "cat"),
                                       ("stack", "forward::forward_rows", "stack"),
                                       ("stack", "forward::forward_columns", "stack"),
                                       ("multi_stack", "forward::forward", "stack"),
                                       ("unsqueeze", "forward::forward_rows", "unsqueeze"),
                                       ("unsqueeze", "forward::forward_depths", "unsqueeze")])
def test_goldens_forward_through_vars(nk, dev, goldens, f, name, op):
    (b,) = goldens[f][name]
    axis = b["nodes"][0]["int_args"][0]
    xs = [golden_value(a) for a in b["arrays"] if a["kind"] == "new_input"]
    vs = [nk.from_ndarray(dev, x) for x in xs]
    y = vs[0].unsqueeze(axis) if op == "unsqueeze" else getattr(vs[0], op)(vs[1:], axis)
    y.forward()
    last = b["nodes"][0]["last_line"]
    want = {"cat": O.cat_forward, "stack": O.stack_forward}.get(op, lambda x, a: O.unsqueeze(x[0], a))(xs, axis)
    outs = [golden_value(a) for a in b["arrays"] if a["line"] > last and tuple(a["shape"]) == want.shape]
    bits_equal(y.data(), outs[0], b["source"])


@pytest.mark.parametrize("f,name,op", [("multi_concatenate", "backward::backward", "cat"),
                                       ("stack", "backward::backward_columns", "stack"),
                                       ("stack", "backward::backward_left_rows", "stack"),
                                       ("stack", "backward::backward_right_columns", "stack"),
                                       ("multi_stack", "backward::backward", "stack")])
def test_goldens_backward_through_vars(nk, dev, goldens, f, name, op):
    """backward(1) is the all-ones seed of the reference's tests; a second backward() accumulates (their second round)"""
    (b,) = goldens[f][name]
    node = b["nodes"][0]
    axis = node["int_args"][0]
    diff = [golden_value(a) for a in b["arrays"] if a["kind"] == "new_backward_input"]
    if node["name"].endswith("Left"):
        vs = [nk.from_ndarray(dev, diff[0]).requires_grad(), nk.from_ndarray(dev, np.zeros_like(diff[0]))]
    elif node["name"].endswith("Right"):
        vs = [nk.from_ndarray(dev, np.zeros_like(diff[0])), nk.from_ndarray(dev, diff[0]).requires_grad()]
    else:
        vs = [nk.from_ndarray(dev, d).requires_grad() for d in diff]
    y = getattr(vs[0], op)(vs[1:], axis)
    y.forward()
    tail = [golden_value(a) for a in b["arrays"] if a["line"] > node["last_line"]]
    assert np.all(tail[0] == 1.0)
    expect = [v for v in tail[1:] if v.shape != tail[0].shape]
    diffs = [v for v in vs if isinstance(v, nk.VarDiff)]
    for r in range(2):
        y.backward(1.0)
        for k, v in enumerate(diffs):
            bits_equal(v.grad(), expect[r * len(diffs) + k], f"{b['source']} round {r}")


def test_history_lengths(nk, dev):
    """test.rs:420-500: one node per cat / stack whatever the operand kinds; multi_cat = 3 operand nodes + 1"""
    ones, zeros, full = nk.ones, nk.zeros, nk.full
    one = full(dev, (1,), 1.0)
    for diff_l, diff_r in ((False, False), (False, True), (True, False), (True, True)):
        lhs = ones(dev, (2, 2))
        rhs = zeros(dev, (2, 2))
        lhs = lhs.requires_grad() if diff_l else lhs
        rhs = rhs.requires_grad() if diff_r else rhs
        assert nk.cat(lhs, rhs, 1).history_len() == 1
        assert nk.stack(lhs, rhs, 1).history_len() == 1
        assert isinstance(nk.cat(lhs, rhs, 1), nk.VarDiff) == (diff_l or diff_r)
    for diff in (False, True):
        rg = (lambda v: v.requires_grad()) if diff else (lambda v: v)
        a = rg(ones(dev, (2, 2))) + one
        b = full(dev, (1,), 18.0) / rg(full(dev, (2, 2), 9.0))
        c = rg(full(dev, (2, 1), 3.0)) * full(dev, (1,), 4.0)
        d = a.cat([b, c], 1)
        assert d.history_len() == 4 and d.shape == (2, 5)
        c2 = rg(full(dev, (2, 2), 3.0)) * full(dev, (1,), 4.0)
        s = a.stack([b, c2], 0)
        assert s.history_len() == 4 and s.shape == (3, 2, 2)
        d.forward()
        bits_equal(d.data(), np.array([[2, 2, 2, 2, 12], [2, 2, 2, 2, 12]], F32), "multi_cat values")


def test_unsqueeze_is_a_view(nk, dev):
    """unlike the reference (test.rs:404-417: one node), unsqueeze records nothing and launches nothing"""
    x = nk.from_ndarray(dev, np.arange(6, dtype=F32).reshape(2, 3))
    for v in (x, x.requires_grad()):
        before = dev.launches
        u = v.unsqueeze(1)
        assert u.shape == (2, 1, 3) and u.history_len() == v.history_len() == 0
        u.forward()
        assert dev.launches == before
        bits_equal(u.data(), np.arange(6, dtype=F32).reshape(2, 1, 3), "unsqueeze")
    xd = x.requires_grad()
    u = xd.unsqueeze(2)
    y = u.cat([u], 2)
    y.forward()
    y.backward(1.0)
    bits_equal(xd.grad(), np.full((2, 3), 2.0, F32), "gradient through the view")


def test_mixed_operands_and_second_backward(nk, dev):
    """only the differentiable operands receive gradients; a second backward() on the cat's own output doubles them
    (its gradient is refilled with the seed, the node accumulates into the operands')"""
    rng = np.random.default_rng(4)
    a_, b_, c_ = (rng.standard_normal(s).astype(F32) for s in ((2, 3, 4), (2, 1, 4), (2, 5, 4)))
    a = nk.from_ndarray(dev, a_).requires_grad()
    b = nk.from_ndarray(dev, b_)
    c = nk.from_ndarray(dev, c_).requires_grad()
    w_ = rng.standard_normal((2, 9, 4)).astype(F32)
    y = a.cat([b, c], 1)
    loss = (y * nk.from_ndarray(dev, w_)).sum()
    loss.forward()
    bits_equal(y.data(), O.cat_forward([a_, b_, c_], 1), "mixed cat")
    loss.backward(1.0)
    bits_equal(a.grad(), w_[:, :3], "a")
    bits_equal(c.grad(), w_[:, 4:], "c")
    assert not isinstance(b, nk.VarDiff)
    a.zero_grad()
    c.zero_grad()
    y.forward()
    y.backward(0.7)
    bits_equal(a.grad(), np.full(a_.shape, 0.7, F32), "a, first backward")
    y.backward(0.7)
    bits_equal(a.grad(), np.full(a_.shape, 2 * F32(0.7), F32), "a after a second backward")
    bits_equal(c.grad(), np.full(c_.shape, 2 * F32(0.7), F32), "c after a second backward")


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("axis", [0, 1])
def test_operand_repeated(nk, dev, fusion, level, axis):
    """x.cat([x, x]) gives x the sum of the three slices; also two views of x (one gradient root) side by side"""
    fusion(level)
    rng = np.random.default_rng(level)
    x_ = rng.standard_normal((3, 4)).astype(F32)
    w_ = rng.standard_normal(O.cat_forward([x_] * 3, axis).shape).astype(F32)
    x = nk.from_ndarray(dev, x_).requires_grad()
    y = x.cat([x, x], axis)
    loss = (y * nk.from_ndarray(dev, w_)).sum()
    loss.forward()
    loss.backward(1.0)
    parts = np.split(w_, 3, axis=axis)
    bits_equal(x.grad(), (parts[0] + parts[1]).astype(F32) + parts[2], "sum of the slices")
    x3 = nk.from_ndarray(dev, x_.reshape(3, 2, 2)).requires_grad()
    z = x3.flatten().cat([x3.flatten()], axis)
    loss = (z * nk.from_ndarray(dev, w_[:, :8] if axis else w_[:6])).sum()
    loss.forward()
    loss.backward(1.0)
    ws = np.split(w_[:, :8] if axis else w_[:6], 2, axis=axis)
    bits_equal(x3.grad(), (ws[0] + ws[1]).reshape(3, 2, 2), "two views of one gradient")


def test_cat_inverts_chunks(nk, dev):
    rng = np.random.default_rng(5)
    x_ = rng.standard_normal((6, 10)).astype(F32)
    w_ = rng.standard_normal((6, 10)).astype(F32)
    x = nk.from_ndarray(dev, x_).requires_grad()
    parts = x.chunks((6, 2))
    y = parts[0].cat(parts[1:], 1)
    loss = (y * nk.from_ndarray(dev, w_)).sum()
    loss.forward()
    bits_equal(y.data(), x_, "cat(chunks(x))")
    loss.backward(1.0)
    bits_equal(x.grad(), w_, "gradient round trip")


def test_bf16_data_f32_gradients(nk, dev):
    rng = np.random.default_rng(6)
    a_, b_ = held(rng.standard_normal((4, 8)), "bf16"), held(rng.standard_normal((4, 8)), "bf16")
    a = nk.from_ndarray(dev, a_, nk.BF16).requires_grad(nk.F32)
    b = nk.from_ndarray(dev, b_, nk.BF16).requires_grad()
    y = a.stack([b], 1)
    y.forward()
    bits_equal(y.data(), O.stack_forward([a_, b_], 1), "bf16 stack")
    y.backward(0.3)
    assert a.grad_dtype == nk.F32 and b.grad_dtype == nk.BF16
    bits_equal(a.grad(), np.full((4, 8), bf16_round(0.3)), "f32 gradient")
    bits_equal(b.grad(), np.full((4, 8), bf16_round(0.3)), "bf16 gradient")
    y.backward(0.3)
    bits_equal(a.grad(), np.full((4, 8), 2 * bf16_round(0.3)), "f32 gradient, second pass")


def test_graph_errors_record_nothing(nk, dev):
    a = nk.zeros(dev, (2, 3)).requires_grad()
    b = nk.zeros(dev, (2, 4))
    c = nk.zeros(dev, (2, 3), nk.BF16)
    cases = [(lambda: a.cat([b], 0), "differs from operand 0 on axis 1"),
             (lambda: a.cat([b], 2), "axis 2 out of range"),
             (lambda: a.cat([c], 0), "another element type"),
             (lambda: a.stack([b], 0), "differs from operand 0"),
             (lambda: a.stack([a], 3), "axis 3 out of range"),
             (lambda: a.unsqueeze(3), "axis 3 out of range"),
             (lambda: nk.cat(a, nk.zeros(dev, (2, 3, 1)), 0), "dimensions")]
    for fn, msg in cases:
        with pytest.raises(nk.NkError, match=msg):
            fn()
    with pytest.raises(nk.NkError, match="at least one dimension"):
        nk.variable.from_ndarray(dev, np.zeros((), F32)).cat([], 0)
    assert a.history_len() == 0 and a.backward_history_len() == 0
    ok = a.cat([a], 0)
    assert ok.history_len() == 1 and ok.backward_history_len() == 1


# ------------------------------------------------------------------------------------------------ a model
def test_lstm_sequence_head_against_torch_and_captured(nk, dev):
    """unrolled 8-step bf16 LSTMCell, the hidden states cat-ed along axis 0 into one Linear head, mse, one SGD step:
    against torch CPU float64 on the same bf16-rounded parameters, then captured as a whole step (two replays equal the
    eager step; bias gradients are f32 atomics and equal to rounding)"""
    import torch
    from neuronika_b200 import optim
    n, n_in, hidden, out, T, lr = 16, 32, 48, 24, 8, 0.05
    rng = np.random.default_rng(31)
    cell = nk.nn.LSTMCell(dev, n_in, hidden, nk.BF16, grad_dtype=nk.F32, rng=np.random.default_rng(2))
    head = nk.nn.Linear(dev, hidden, out, nk.BF16, grad_dtype=nk.F32, rng=np.random.default_rng(3))
    params = cell.parameters() + head.parameters()
    init = [p.data().copy() for p in params]
    xs_ = [held(rng.standard_normal((n, n_in)), "bf16") for _ in range(T)]
    tgt_ = held(rng.standard_normal((T * n, out)), "bf16")
    xs = [nk.from_ndarray(dev, x, nk.BF16) for x in xs_]
    tgt = nk.from_ndarray(dev, tgt_, nk.BF16)
    zeros = nk.from_ndarray(dev, np.zeros((n, hidden), F32), nk.BF16)
    opt = optim.StochasticGD.new(lr)
    for p in params:
        opt.register(p)
    live = {}

    def step():
        opt.zero_grad()
        state, hs = (zeros, zeros), []
        for x in xs:
            state = cell.forward(state, x)
            hs.append(state[1])
        y = head.forward(hs[0].cat(hs[1:], 0))
        loss = y.mse_loss(tgt)
        loss.forward()
        loss.backward(1.0)
        live["loss"], live["y"] = loss, y
        live["grads"] = [p.grad_array() for p in params]
        opt.step()

    def reset():
        for p, v in zip(params, init):
            p.set_data(v)

    step()
    dev.synchronize()
    loss_eager = live["loss"].item()
    grads = [g.as_ndarray().copy() for g in live["grads"]]
    new_w = [p.data().copy() for p in params]

    tc = torch.nn.LSTMCell(n_in, hidden).double()
    th = torch.nn.Linear(hidden, out).double()
    tps = [tc.weight_ih, tc.weight_hh, tc.bias_ih, tc.bias_hh, th.weight, th.bias]
    with torch.no_grad():
        for p, v in zip(tps, init):
            p.copy_(torch.from_numpy(v.astype(np.float64)))
    h = c = torch.zeros(n, hidden, dtype=torch.float64)
    hs = []
    for x in xs_:
        h, c = tc(torch.from_numpy(x.astype(np.float64)), (h, c))
        hs.append(h)
    loss = torch.nn.functional.mse_loss(th(torch.cat(hs, 0)), torch.from_numpy(tgt_.astype(np.float64)))
    loss.backward()
    assert abs(loss_eager - loss.item()) <= 0.02 * abs(loss.item())
    names = ["weight_ih", "weight_hh", "bias_ih", "bias_hh", "head.weight", "head.bias"]
    for name, g, w0, w1, p in zip(names, grads, init, new_w, tps):
        want = p.grad.numpy()
        # bf16 states and gate gradients over T = 8 steps: within 5% of the largest float64 gradient of the tensor
        tol = 0.05 * np.abs(want).max() + 1e-6
        assert np.max(np.abs(g - want)) <= tol, name
        assert np.all(np.abs(w1 - (w0 - lr * want)) <= UB * np.abs(w0) + lr * tol + 1e-7), name

    reset()
    step()
    dev.synchronize()
    eager = [live["y"].data()] + [g.as_ndarray().copy() for g in live["grads"]] + [p.data().copy() for p in params]
    reset()
    with dev.capture(256 << 20) as cap:
        step()
    replays = []
    for _ in range(2):
        reset()
        cap.graph.launch()
        dev.synchronize()
        replays.append([live["y"].data()] + [g.as_ndarray().copy() for g in live["grads"]] +
                       [p.data().copy() for p in params])
    labels = ["y"] + names + ["w." + k for k in names]
    for r in replays:
        for name, a, b in zip(labels, eager, r):
            if "bias" in name:
                assert np.all(np.abs(a - b) <= 1e-6 * np.abs(a) + 1e-7), name
            else:
                bits_equal(b, a, f"replay {name}")
    for name, a, b in zip(labels, replays[0], replays[1]):
        if "bias" not in name:
            bits_equal(b, a, f"second replay {name}")
    cap.graph.close()
