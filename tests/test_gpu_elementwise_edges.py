"""The HBM-bound kernels of a training step that are neither GEMM nor convolution, at their vector, alignment and
grid-stride boundaries: elementwise and unary / binary maps, broadcast add and un-broadcast sums, scalar reductions,
softmax, mv / vm / vv, SGD and the Adam family, transpose and padding.

Every operand is a view into a larger buffer filled with a canary value (`Guarded`).  Offset 0 is 16-byte aligned and
takes the vector body; offset 1 is not, for f32 and bf16 alike, and must take the scalar body with the same result.
Both are asserted from the pointer.  After each call every element outside the output view must still hold the
canary, bit for bit.  Outputs written with beta = 0 are pre-filled with NaN, so a kernel that reads them fails.
"Past one wave" sizes come from the SM count: one wave is 8 CTAs x 256 threads per SM.

The reference is float64 on the same (bf16-rounded) inputs.  Copies, selects and sums of two f32 values round once,
so their results are compared bit for bit with the float64 value rounded as the kernel rounds it.  Other f32 results
must lie within k * 2^-24 * S of it, where S is the sum of the magnitudes of the terms and k is stated at each
assertion; for a reduction k is its per-thread chain length.  A bf16 output adds 2^-8 * |want| (one rounding).
Long inputs repeat a random block of P = 4099 elements (a prime, so no vector width, stride or tile aliases it).

These kernels report no kernel name; each case names the path it is meant to take and cites the host predicate that
picks it.  The device-memory peak of the file is the 2^31-element pad case: 13.1 GB (torch's allocator, one H100
80GB HBM3 at a 400 W power limit); the whole file runs in about 50 s there."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0          # exact in bf16 and f32, far outside every value below
U = 2.0 ** -24            # f32 unit roundoff
UB = 2.0 ** -8            # bf16 unit roundoff: one rounding of the output
P = 4099
VEC = {"f32": 4, "bf16": 8}     # NkVec<T>::N, elements per 16-byte access


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


@pytest.fixture(scope="module")
def O():
    import oracle
    return oracle


def D(nk, dt):
    return nk.BF16 if dt == "bf16" else nk.F32


def wave(dev):
    """threads in one wave of an elementwise grid (ew_blocks caps grids at 8 CTAs of 256 threads per SM)"""
    return dev.sm_count * 8 * 256


def cdiv(a, b):
    return -(-a // b)


def held(x, dt):
    """float32 x as a `dt` tensor holds it"""
    from oracle import bf16_round
    x = np.asarray(x, F32)
    return bf16_round(x) if dt == "bf16" else x


def stored(v, dt):
    """what a kernel stores for the exact value v when it rounds once to f32 and then to the storage type"""
    return held(np.asarray(v, np.float64).astype(F32), dt)


def tol(k, S, want, dt):
    return k * U * np.asarray(S, np.float64) + (UB * np.abs(want) if dt == "bf16" else 0.0)


def periodic(rng, n, lo, hi, dt, signs=False):
    """n values that repeat a random block of P elements, as a `dt` tensor holds them"""
    b = rng.uniform(lo, hi, min(n, P))
    if signs:
        b = b * rng.choice([-1.0, 1.0], b.size)
    return np.resize(held(b.astype(F32), dt), n)


def upload_periodic(nk, dev, block, n, dt):
    """np.resize(block, n) as a device array, converting only the block to the storage format"""
    import ctypes as C
    from neuronika_b200 import _lib as L
    host = np.resize(L.f32_to_bf16_bits(block) if dt == "bf16" else np.asarray(block, F32), n)
    a = dev.zeros((n,), D(nk, dt))
    L.check(L.lib.nk_h2d(dev.ctx, a.ptr, host.ctypes.data_as(C.c_void_p), a.nbytes), dev.ctx)
    dev.synchronize()
    return a


def to_device(dev, host, dtype):
    """host (float32 values the storage type holds exactly) as a device array: bf16 by truncation, which is exact
    for such values (f32_to_bf16_bits rounds, and takes longer)"""
    import ctypes as C
    from neuronika_b200 import _lib as L
    from neuronika_b200.device import CuArray
    host = np.ascontiguousarray(host, F32)
    if dtype == L.NK_BF16:
        u = host.view(np.uint32)
        assert not (u & 0xFFFF).any(), "not a bf16 value"
        host = (u >> 16).astype(np.uint16)
    a = CuArray(dev, host.shape, dtype)
    L.check(L.lib.nk_h2d(dev.ctx, a.ptr, host.ctypes.data_as(C.c_void_p), a.nbytes), dev.ctx)
    dev.synchronize()
    return a


class Guarded:
    """`data` at element `off` (0 or 1) of a device buffer whose other elements -- `off` before the view and `tail`
    after it -- hold CANARY.  off = 0 is 16-byte aligned, off = 1 is not: asserted from the view's pointer."""

    def __init__(self, dev, data, dtype, off=0, tail=24):
        assert off in (0, 1)
        data = np.asarray(data, F32)
        self.shape, self.n, self.off = data.shape, data.size, off
        host = np.full(off + self.n + tail, CANARY, F32)
        host[off:off + self.n] = data.ravel()
        self.buf = to_device(dev, host, dtype)
        self.view = self.buf.slice_flat(off, self.shape)
        assert (self.view.ptr.value % 16 == 0) == (off == 0), (off, self.view.ptr.value % 16)

    def read(self):
        """(the view, after asserting that nothing outside it changed)"""
        flat = self.buf.as_ndarray().ravel()
        outside = np.concatenate([flat[:self.off], flat[self.off + self.n:]])
        bad = np.flatnonzero(outside.view(np.uint32) != F32(CANARY).view(np.uint32))
        assert bad.size == 0, f"{bad.size} elements outside the view were written (first at outside index {bad[0]})"
        return flat[self.off:self.off + self.n].reshape(self.shape)


def out_buf(dev, want_shape, dtype, beta, d0, off=0):
    """an output view: NaN when beta = 0 (the kernel must not read it), else d0"""
    return Guarded(dev, np.full(want_shape, np.nan, F32) if beta == 0 else d0, dtype, off)


def exact(got, want, what):
    g, w = np.ascontiguousarray(got, F32).ravel(), np.ascontiguousarray(want, F32).ravel()
    bad = np.flatnonzero(g.view(np.uint32) != w.view(np.uint32))
    assert bad.size == 0, (what, f"{bad.size} differ", int(bad[0]), float(g[bad[0]]), float(w[bad[0]]))


def near(got, want, t, what):
    got, want, t = (a.ravel() for a in np.broadcast_arrays(np.asarray(got, np.float64), np.asarray(want, np.float64),
                                                           np.asarray(t, np.float64)))
    err = np.abs(got - want)
    bad = np.flatnonzero(~(err <= t))       # NaN fails
    assert bad.size == 0, (what, f"{bad.size} outside", int(bad[0]), float(got[bad[0]]), float(want[bad[0]]),
                           float(t[bad[0]]))


def ulp2(got, want64, what):
    """within 2 ulp of the float64 value rounded to f32"""
    w = F32(want64)
    assert abs(float(got) - float(w)) <= 2.0 * float(np.spacing(abs(w))), (what, float(got), float(w), want64)


# ============================================================================================ launch_ew / launch_map
# Dispatch: launch_ew's `vec` (nk_elementwise.cu:65) and launch_map's `vec` (nk_pointwise.cu:141) take the 16-byte
# body when every pointer is 16-byte aligned; the first n % V elements after it (and every element otherwise) run in
# the scalar loop, which must start at `done + tid`.
#
# Each op: (input kinds, read-modify-write?, call(out, ins, beta, g), ref(ins, n) -> (f, S, k)).  f is the op's exact
# value in float64; k = 0 means the kernel rounds f (+ beta * d0) once -- f is an f32 value or the op is not RMW --
# so the result is compared bit for bit; otherwise |got - want| <= (k [+ 2 for the beta term]) * 2^-24 * S.
G0 = 0.7            # the scalar gradient of mse / sum backward
FILL = 0.3          # rounds in bf16 (and in f32)
SYM, POS, DEN, UNIT, TANH = (-2.0, 2.0, False), (0.25, 2.0, False), (0.5, 2.0, True), (0.05, 0.95, False), (-0.95, 0.95, False)


def _ew_specs():
    from neuronika_b200 import ops
    lk = float(F32(0.01))   # leaky_relu slope as the kernel holds it (0.01f)
    g0 = float(F32(G0))

    def un(op, ip=0):
        return lambda o, i, b, g: ops.unary(op, i[0], ip, out=o)

    def unb(op, ip=0):
        return lambda o, i, b, g: ops.unary_bwd(op, o, i[1] if len(i) > 1 else None, i[0], ip, beta=b)

    def binb(op, side):
        return lambda o, i, b, g: ops.binary_bwd(op, side, o, i[0], i[1], i[2], beta=b)

    def powi(x, e):
        return x ** e

    S = {
        "fill": ((), False, lambda o, i, b, g: o.fill_(FILL), lambda a, n: (float(F32(FILL)), 0, 0)),
        "relu_fwd": ((SYM,), False, lambda o, i, b, g: ops.relu(i[0], out=o),
                     lambda a, n: (np.where(a[0] > 0, a[0], 0.0), 0, 0)),
        "relu_bwd": ((SYM, SYM), True, lambda o, i, b, g: ops.relu_bwd(o, i[0], i[1], beta=b),
                     lambda a, n: (np.where(a[0] > 0, a[1], 0.0), 0, 0)),
        # 2 (x - t) * g [/ n]: three roundings (x - t, * g, / n)
        "mse_bwd_mean": ((SYM, SYM), True, lambda o, i, b, g: ops.mse_bwd(o, i[0], i[1], g, True, beta=b),
                         lambda a, n: ((f := 2 * (a[0] - a[1]) * g0 / n), np.abs(f), 3)),
        "mse_bwd_sum": ((SYM, SYM), True, lambda o, i, b, g: ops.mse_bwd(o, i[0], i[1], g, False, beta=b),
                        lambda a, n: ((f := 2 * (a[0] - a[1]) * g0), np.abs(f), 2)),
        # g / n: one rounding
        "sum_bwd_mean": ((), True, lambda o, i, b, g: ops.reduce_sum_bwd(o, g, True, beta=b),
                         lambda a, n: (g0 / n, g0 / n, 1)),
        "sum_bwd_sum": ((), True, lambda o, i, b, g: ops.reduce_sum_bwd(o, g, False, beta=b),
                        lambda a, n: (g0, 0, 0)),
        # same-shape, same-type un-broadcast = dst = beta*dst + g through launch_ew (nk_elementwise.cu:699)
        "acc": ((SYM,), True, lambda o, i, b, g: ops.unbroadcast_acc(o, i[0], beta=b), lambda a, n: (a[0], 0, 0)),
        # unary forward: expf / tanhf within 2 ulp (4 * 2^-24 relative), logf 1 ulp, sqrtf exact, compositions add one
        # rounding per step; softplus' error is absolute (log of 1 + e^x), hence S = 1 + |f|
        "neg": ((SYM,), False, un("neg"), lambda a, n: (-a[0], 0, 0)),
        "exp": ((SYM,), False, un("exp"), lambda a, n: ((f := np.exp(a[0])), f, 6)),
        "ln": ((POS,), False, un("ln"), lambda a, n: ((f := np.log(a[0])), np.abs(f), 3)),
        "sqrt": ((POS,), False, un("sqrt"), lambda a, n: ((f := np.sqrt(a[0])), f, 1)),
        "sigmoid": ((SYM,), False, un("sigmoid"), lambda a, n: ((f := 1 / (1 + np.exp(-a[0]))), f, 8)),
        "tanh": ((SYM,), False, un("tanh"), lambda a, n: ((f := np.tanh(a[0])), np.abs(f), 6)),
        "softplus": ((SYM,), False, un("softplus"), lambda a, n: ((f := np.log1p(np.exp(a[0]))), 1 + f, 8)),
        "leaky_relu": ((SYM,), False, un("leaky_relu"), lambda a, n: (np.where(a[0] > 0, a[0], lk * a[0]), 0, 0)),
        "powi3": ((SYM,), False, un("powi", 3), lambda a, n: ((f := powi(a[0], 3)), np.abs(f), 3)),
        "powi-2": ((POS,), False, un("powi", -2), lambda a, n: ((f := powi(a[0], -2)), f, 3)),
        # unary backward (g, saved): one rounding per product / quotient, tanh / sigmoid bounded by their terms
        "neg_bwd": ((SYM,), True, unb("neg"), lambda a, n: (-a[0], 0, 0)),
        "exp_bwd": ((SYM, SYM), True, unb("exp"), lambda a, n: ((f := a[0] * a[1]), np.abs(f), 1)),
        "ln_bwd": ((SYM, POS), True, unb("ln"), lambda a, n: ((f := a[0] / a[1]), np.abs(f), 1)),
        "sqrt_bwd": ((SYM, POS), True, unb("sqrt"), lambda a, n: ((f := a[0] / (2 * a[1])), np.abs(f), 1)),
        "sigmoid_bwd": ((SYM, UNIT), True, unb("sigmoid"),
                        lambda a, n: (a[0] * a[1] * (1 - a[1]), np.abs(a[0] * a[1]) * (1 + a[1]), 3)),
        "tanh_bwd": ((SYM, TANH), True, unb("tanh"), lambda a, n: (a[0] * (1 - a[1] ** 2), np.abs(a[0]) * (1 + a[1] ** 2), 3)),
        "softplus_bwd": ((SYM, SYM), True, unb("softplus"),
                         lambda a, n: ((f := a[0] / (1 + np.exp(-a[1]))), np.abs(f), 6)),
        "leaky_relu_bwd": ((SYM, SYM), True, unb("leaky_relu"),
                           lambda a, n: ((f := np.where(a[1] > 0, a[0], lk * a[0])), np.abs(f), 1)),
        "powi3_bwd": ((SYM, SYM), True, unb("powi", 3), lambda a, n: ((f := a[0] * a[1] ** 2 * 3), np.abs(f), 3)),
        "powi-2_bwd": ((SYM, POS), True, unb("powi", -2), lambda a, n: ((f := a[0] * a[1] ** -3 * -2), np.abs(f), 4)),
        # same-shape binary forward: one rounding of an exact product / difference; division correctly rounded
        "sub": ((SYM, SYM), False, lambda o, i, b, g: ops.binary("sub", i[0], i[1], out=o), lambda a, n: (a[0] - a[1], 0, 0)),
        "mul": ((SYM, SYM), False, lambda o, i, b, g: ops.binary("mul", i[0], i[1], out=o), lambda a, n: (a[0] * a[1], 0, 0)),
        "div": ((SYM, DEN), False, lambda o, i, b, g: ops.binary("div", i[0], i[1], out=o),
                lambda a, n: ((f := a[0] / a[1]), np.abs(f), 1)),
        # same-shape binary backward (g, l, r): the fused launch_map<T, 3> (nk_pointwise.cu:433)
        "sub_bwd_l": ((SYM, SYM, SYM), True, binb("sub", 0), lambda a, n: (a[0], 0, 0)),
        "sub_bwd_r": ((SYM, SYM, SYM), True, binb("sub", 1), lambda a, n: (-a[0], 0, 0)),
        "mul_bwd_l": ((SYM, SYM, SYM), True, binb("mul", 0), lambda a, n: ((f := a[0] * a[2]), np.abs(f), 1)),
        "mul_bwd_r": ((SYM, SYM, SYM), True, binb("mul", 1), lambda a, n: ((f := a[0] * a[1]), np.abs(f), 1)),
        "div_bwd_l": ((SYM, SYM, DEN), True, binb("div", 0), lambda a, n: ((f := a[0] / a[2]), np.abs(f), 1)),
        "div_bwd_r": ((SYM, SYM, DEN), True, binb("div", 1),
                      lambda a, n: ((f := -a[0] * a[1] / a[2] ** 2), np.abs(f), 3)),
    }
    return S


EW_OPS = ["fill", "relu_fwd", "relu_bwd", "mse_bwd_mean", "mse_bwd_sum", "sum_bwd_mean", "sum_bwd_sum", "acc",
          "neg", "exp", "ln", "sqrt", "sigmoid", "tanh", "softplus", "leaky_relu", "powi3", "powi-2",
          "neg_bwd", "exp_bwd", "ln_bwd", "sqrt_bwd", "sigmoid_bwd", "tanh_bwd", "softplus_bwd", "leaky_relu_bwd",
          "powi3_bwd", "powi-2_bwd", "sub", "mul", "div", "sub_bwd_l", "sub_bwd_r", "mul_bwd_l", "mul_bwd_r",
          "div_bwd_l", "div_bwd_r"]


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("op", EW_OPS)
def test_elementwise_vector_scalar_and_grid_stride(nk, dev, op, dt):
    """n in {1, V-1, V, V+1, 1023, 2*wave*V + 5}: the vector body, its scalar tail, the scalar loop on unaligned
    operands and, at the last size, a third trip round the vector loop (and 2V trips round the scalar one).  Layouts:
    every operand aligned; each operand alone one element off (the output included); all of them off."""
    kinds, rmw, call, ref = _ew_specs()[op]
    V, D_ = VEC[dt], D(nk, dt)
    g = dev.from_ndarray(np.asarray(G0, F32))
    nops = len(kinds) + 1                                        # inputs, then the output
    layouts = list(dict.fromkeys([(0,) * nops] + [tuple(int(j == i) for j in range(nops)) for i in range(nops)]
                                 + [(1,) * nops]))
    big = 2 * wave(dev) * V + 5
    seed = EW_OPS.index(op) * 10 + (dt == "bf16")
    for n in (1, V - 1, V, V + 1, 1023, big):
        rng = np.random.default_rng(seed + n)
        ins = [periodic(rng, n, lo, hi, dt, sg) for lo, hi, sg in kinds]
        d0 = periodic(rng, n, -2, 2, dt)
        m = min(n, P)                          # inputs and d0 repeat their first m elements, and so does the result
        f, S, k = ref([a[:m].astype(np.float64) for a in ins], n)
        d0m = d0[:m].astype(np.float64)
        cases = []
        for li, offs in enumerate(layouts):
            if n == big and li not in (0, len(layouts) - 1):
                continue
            if not rmw:
                betas = (0.0,)
            elif n == big:
                betas = (0.5,) if li == 0 else (0.0,)
            elif li in (0, len(layouts) - 1):
                betas = (0.0, 1.0, 0.5)
            else:
                betas = ((0.0, 1.0, 0.5)[li % 3],)
            cases += [(offs, b) for b in betas]
        for offs, beta in cases:
            gins = [Guarded(dev, a, D_, o) for a, o in zip(ins, offs)]
            out = out_buf(dev, (n,), D_, beta, d0, offs[-1])
            call(out.view, [x.view for x in gins], beta, g)
            got = out.read()
            for x, a in zip(gins, ins):
                exact(x.read(), a, (op, "input changed"))
            want = f + beta * d0m
            what = (op, dt, n, offs, beta)
            if k == 0:
                exact(got, np.resize(stored(want, dt), n), what)    # one rounding of an exact value
            else:
                kk = k + (2 if beta else 0)                          # the op's k (see _ew_specs) + 2 for beta*d0 + f
                near(got, np.resize(want, n), np.resize(tol(kk, np.abs(S) + np.abs(beta * d0m), want, dt), n), what)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_relu_special_values(nk, dev, dt):
    """ReLU is f32::max(x, 0) (nk_elementwise.cu:97): NaN -> 0, +inf -> inf, -inf -> 0, -0 -> 0; its backward passes g
    only where x > 0.  Written out literally: numpy's maximum would propagate the NaN.  11 elements: an 8-wide vector
    body and a scalar tail when aligned, all scalar when not."""
    from neuronika_b200 import ops
    nan, inf = float("nan"), float("inf")
    x = np.array([nan, inf, -inf, -0.0, 0.0, 1.5, -1.5, nan, 2.0, -inf, nan], F32)
    want = np.array([0, inf, 0, 0, 0, 1.5, 0, 0, 2.0, 0, 0], F32)
    g = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], F32)
    for off in (0, 1):
        X = Guarded(dev, x, D(nk, dt), off)
        Y = out_buf(dev, x.shape, D(nk, dt), 0, None, off)
        ops.relu(X.view, out=Y.view)
        exact(Y.read(), want, ("relu", off))
        G = Guarded(dev, g, D(nk, dt), off)
        DX = out_buf(dev, x.shape, D(nk, dt), 0, None, off)
        ops.relu_bwd(DX.view, X.view, G.view, beta=0.0)
        exact(DX.read(), np.where(want > 0, g, 0).astype(F32), ("relu_bwd", off))


# ============================================================================================ broadcast add
def _bcast_cases(dev, V):
    """(name, left shape, right shape, offset of the full-size operand).  Paths: add_bcast_channel's vector body
    needs y and the big operand 16-byte aligned and, for inner = 1, C % V == 0, else inner % V == 0
    (nk_elementwise.cu:636); inner > 1 or a 0-d / all-ones small operand (C = 1, inner = n) uses the channel index
    (e / inner) % C; anything else with a broadcast on both sides is add_bcast_generic (nk_elementwise.cu:656)."""
    w = wave(dev)
    return [
        ("row_vector", (37, 8 * V), (8 * V,), 0),
        ("row_scalar", (37, 8 * V + 1), (8 * V + 1,), 0),
        ("channel_vector", (3, 5, 8, 8), (5, 1, 1), 0),
        ("channel_scalar", (3, 5, 7, 7), (5, 1, 1), 0),
        ("zero_dim", (6, 8 * V), (), 0),
        ("ones_1x1", (6, 8 * V), (1, 1), 0),
        ("small_left_row", (8 * V,), (37, 8 * V), 0),
        ("small_left_channel", (5, 1, 1), (3, 5, 8, 8), 0),
        ("row_big_off", (37, 8 * V), (8 * V,), 1),
        ("channel_big_off", (3, 5, 8, 8), (5, 1, 1), 1),
        ("generic_6d", (2, 1, 3, 1, 5, 1), (1, 4, 1, 2, 1, 3), 0),
        # past one wave: 3 trips of the vector body, 2+ of the scalar and generic loops
        ("channel_vector_waves", (cdiv(2 * w * V + 1, 16 * 64), 16, 8, 8), (16, 1, 1), 0),
        ("channel_scalar_waves", (cdiv(2 * w + 1, 16 * 49), 16, 7, 7), (16, 1, 1), 0),
        ("generic_6d_waves", (cdiv(2 * w + 1, 360), 1, 3, 1, 5, 1), (1, 4, 1, 2, 1, 3), 0),
    ]


@pytest.mark.parametrize("op", ["add", "sub", "mul", "div"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_broadcast_binary_forward(nk, dev, op, dt):
    """add through nk_add_bcast_fwd's channel / generic kernels; sub / mul / div through nk_binary_bcast_fwd's
    strided kernel, on the same shapes.  add, sub and mul round an exact value once: bit exact.  div: within 1 rounding."""
    from neuronika_b200 import ops
    D_ = D(nk, dt)
    for ci, (name, ls, rs, big_off) in enumerate(_bcast_cases(dev, VEC[dt])):
        rng = np.random.default_rng(ci)
        lo = 0.5 if op == "div" else -2.0
        l = held(rng.uniform(lo, 2, ls).astype(F32), dt)
        r = held((rng.uniform(lo, 2, rs) * (rng.choice([-1.0, 1.0], rs) if op == "div" else 1)).astype(F32), dt)
        ys = np.broadcast_shapes(ls, rs)
        lbig = int(np.prod(ls)) == int(np.prod(ys))
        L_ = Guarded(dev, l, D_, big_off if lbig else 0)
        R_ = Guarded(dev, r, D_, 0 if lbig else big_off)
        Y = out_buf(dev, ys, D_, 0, None, 0)
        if op == "add":
            ops.add(L_.view, R_.view, out=Y.view)
        else:
            ops.binary(op, L_.view, R_.view, out=Y.view)
        got = Y.read()
        exact(L_.read(), l, "left changed")
        exact(R_.read(), r, "right changed")
        l64, r64 = l.astype(np.float64), r.astype(np.float64)
        want = {"add": l64 + r64, "sub": l64 - r64, "mul": l64 * r64, "div": l64 / r64}[op]
        if op == "div":
            near(got, want, tol(1, np.abs(want), want, dt), (name, dt))     # one correctly rounded quotient
        else:
            exact(got, stored(want, dt), (name, dt))


# ============================================================================================ un-broadcast
def unb_plan(sm, gshape, dshape, g_dtype, aligned=True):
    """(kernel, chain length) nk_unbroadcast_acc picks (nk_elementwise.cu:696-788).  The chain is the longest run of
    f32 additions any term goes through: per-thread loop, shared-memory / warp combine, one atomic per row chunk."""
    nd = len(gshape)
    dsh = (1,) * (nd - len(dshape)) + tuple(dshape)
    if int(np.prod(dsh)) == int(np.prod(gshape)):
        return "axpy", 1
    keep = [k for k in range(nd) if dsh[k] != 1]
    red = [k for k in range(nd) if dsh[k] == 1 and gshape[k] != 1]
    if keep and any(keep[0] < k < keep[-1] for k in red):
        return "unbroadcast_generic", int(np.prod([gshape[k] for k in red]))
    if keep:
        R0 = int(np.prod(gshape[:keep[0]]))
        K = int(np.prod(gshape[keep[0]:keep[-1] + 1]))
        R1 = int(np.prod(gshape[keep[-1] + 1:]))
    else:
        R0, K, R1 = int(np.prod(gshape)), 1, 1
    V = 8 if g_dtype == "bf16" else 4
    if R1 == 1:
        # nk_elementwise.cu:737: colsum_vec needs K % V == 0, an aligned g and K >= 32 V
        vec = K % V == 0 and aligned and K >= 32 * V
        want_y = cdiv(sm * 8, cdiv(K, 32 * V if vec else 32))
        rpb = max(64, cdiv(R0, want_y))
        return ("colsum_vec" if vec else "colsum"), cdiv(rpb, 8) + 1 + 8 + cdiv(R0, rpb)
    want_y = min(max(cdiv(sm * 8, K), 1), R0)
    r0pb = cdiv(R0, want_y)
    return "chansum", r0pb * cdiv(R1, 256) + 5 + 8 + cdiv(R0, r0pb)


def unbroadcast_ref(g64, dshape):
    nd = g64.ndim
    dsh = (1,) * (nd - len(dshape)) + tuple(dshape)
    axes = tuple(k for k in range(nd) if dsh[k] == 1 and g64.shape[k] != 1)
    return g64.sum(axis=axes, keepdims=True).reshape(dshape)


def run_unbroadcast(nk, dev, g, gdt, dshape, ddt, beta, goff, rng, what, expect):
    from neuronika_b200 import ops
    kern, L = unb_plan(dev.sm_count, g.shape, dshape, gdt, goff == 0)
    assert kern == expect, (what, kern)
    d0 = held(rng.uniform(-1, 1, dshape).astype(F32), ddt)
    G_ = Guarded(dev, g, D(nk, gdt), goff)
    Dst = out_buf(dev, dshape, D(nk, ddt), beta, d0)
    ops.unbroadcast_acc(Dst.view, G_.view, beta=beta)
    got = Dst.read()
    exact(G_.read(), g, "g changed")
    g64 = g.astype(np.float64)
    want = unbroadcast_ref(g64, dshape) + beta * d0
    # chain L of additions over the terms, + 1 for finalize_acc's beta*dst + v
    near(got, want, tol(L + 1, unbroadcast_ref(np.abs(g64), dshape) + np.abs(beta * d0), want, ddt),
         what + (kern, L, beta))


@pytest.mark.parametrize("ddt", ["f32", "bf16"])
@pytest.mark.parametrize("gdt", ["f32", "bf16"])
@pytest.mark.parametrize("ki", [0, 1, 2])
def test_unbroadcast_column_sums(nk, dev, gdt, ddt, ki):
    """colsum_vec: K = 32V (one column block), 32V + V (a partial one) and a many-block K; R0 from 2 (R0 = 1 is the
    same-shape accumulate) across the two-rows-in-
    flight loop (r + 8 < r_end), its 8-row tail and the rows_per_block chunks, whose size is 64 until R0 > 64 * want_y.
    The same g one element off must fall back to colsum with the same sums."""
    K = {"f32": (128, 132, 4100), "bf16": (256, 264, 4096)}[gdt][ki]
    R0s = (2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 8192, 65537) if ki == 0 else (2, 7, 9, 17, 65, 2049)
    for R0 in R0s:
        rng = np.random.default_rng(R0 * 7 + ki)
        g = periodic(rng, R0 * K, -1, 1, gdt).reshape(R0, K)
        for beta in (0.0, 1.0):
            run_unbroadcast(nk, dev, g, gdt, (K,), ddt, beta, 0, rng, ("colsum_vec", R0, K), "colsum_vec")
            if R0 <= 8192:
                run_unbroadcast(nk, dev, g, gdt, (K,), ddt, beta, 1, rng, ("colsum g+1", R0, K), "colsum")


@pytest.mark.parametrize("ddt", ["f32", "bf16"])
@pytest.mark.parametrize("gdt", ["f32", "bf16"])
def test_unbroadcast_colsum_chansum_generic(nk, dev, gdt, ddt):
    """colsum at K around one 32-column block; chansum (R1 > 1) with R0 = 40 and K = 3, so that each of the 40 row
    chunks is one r0 (want_y = min(ceil(8 * SMs / 3), R0)), and R1 around the 256-thread block; unbroadcast_generic where the kept axes are not contiguous."""
    rng = np.random.default_rng(5)
    cases = [((R0, K), (K,), "colsum") for K in (1, 31, 32, 33, 124) for R0 in (2, 9, 65, 5000)]
    cases += [((40, 3, R1), (3, 1), "chansum") for R1 in (2, 255, 256, 257, 4096)]
    cases += [((4, 5, 6), (4, 1, 6), "unbroadcast_generic"),
              ((2, 3, 4, 5, 6, 7), (2, 1, 4, 1, 6, 1), "unbroadcast_generic")]
    for gs, ds, kern in cases:
        g = periodic(rng, int(np.prod(gs)), -1, 1, gdt).reshape(gs)
        for beta in (0.0, 1.0):
            run_unbroadcast(nk, dev, g, gdt, ds, ddt, beta, 0, rng, (gs, ds), kern)


@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("gdt,ddt", [("f32", "bf16"), ("bf16", "f32")])
def test_accumulate_mixed_types(nk, dev, gdt, ddt, beta):
    """same-shape accumulate between types: axpy_mixed (nk_elementwise.cu:700); of one term, so bit exact.  Same types
    go through launch_ew (test_elementwise_vector_scalar_and_grid_stride, op "acc")."""
    from neuronika_b200 import ops
    n = 2 * wave(dev) + 7
    rng = np.random.default_rng(9)
    g, d0 = periodic(rng, n, -2, 2, gdt), periodic(rng, n, -2, 2, ddt)
    G_ = Guarded(dev, g, D(nk, gdt), 1)
    Dst = out_buf(dev, (n,), D(nk, ddt), beta, d0, 1)
    ops.unbroadcast_acc(Dst.view, G_.view, beta=beta)
    exact(Dst.read(), stored(g.astype(np.float64) + beta * d0, ddt), (gdt, ddt, beta))


BWD_SHAPES = [((512, 256), (256,)), ((8, 16, 5, 5), (16, 1, 1)), ((4, 1, 6), (3, 6)), ((3, 1), (1, 4)),
              ((256,), (64, 256))]


@pytest.mark.parametrize("op", ["add", "sub", "mul", "div"])
@pytest.mark.parametrize("dt,ddt", [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32")])
def test_binary_backward_with_broadcast(nk, dev, op, dt, ddt):
    """nk_binary_bcast_bwd for each side that is broadcast: the factor over the broadcast shape (f32, in a
    cudaMallocAsync buffer for mul / div / sub-right, nk_pointwise.cu:442), then un-broadcast into the operand
    gradient; bf16 operands with an f32 gradient included.  Bound: the factor's roundings + the reduction's chain."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(11)
    for ls, rs in BWD_SHAPES:
        ys = np.broadcast_shapes(ls, rs)
        l = held(rng.uniform(0.5, 2, ls).astype(F32), dt)
        r = held((rng.uniform(0.5, 2, rs) * rng.choice([-1.0, 1.0], rs)).astype(F32), dt)
        g = held(rng.uniform(-1, 1, ys).astype(F32), dt)
        l64, r64, g64 = (np.broadcast_to(a.astype(np.float64), ys) for a in (l, r, g))
        for side, shape in ((0, ls), (1, rs)):
            if int(np.prod(shape)) == int(np.prod(ys)):
                continue
            fac, kf = {("add", 0): (g64, 0), ("add", 1): (g64, 0), ("sub", 0): (g64, 0), ("sub", 1): (-g64, 0),
                       ("mul", 0): (g64 * r64, 1), ("mul", 1): (g64 * l64, 1), ("div", 0): (g64 / r64, 1),
                       ("div", 1): (-g64 * l64 / r64 ** 2, 3)}[(op, side)]
            buffered = not (op == "add" or (op == "sub" and side == 0))
            kern, L = unb_plan(dev.sm_count, ys, shape, "f32" if buffered else dt)
            for beta in (0.0, 1.0):
                d0 = held(rng.uniform(-1, 1, shape).astype(F32), ddt)
                Dst = out_buf(dev, shape, D(nk, ddt), beta, d0)
                ops.binary_bwd(op, side, Dst.view, dev.from_ndarray(g, D(nk, dt)), dev.from_ndarray(l, D(nk, dt)),
                               dev.from_ndarray(r, D(nk, dt)), beta=beta)
                got = Dst.read()
                want = unbroadcast_ref(fac, shape) + beta * d0
                # kf roundings of the factor + the chain L of the reduction + 1 for beta
                S = unbroadcast_ref(np.abs(fac), shape) + np.abs(beta * d0)
                near(got, want, tol(kf + L + 1, S, want, ddt), (op, side, ls, rs, kern, beta))


# ============================================================================================ scalar reductions
def _sum_block(rng, n, dt):
    """1000 + N(0, 1): a large common offset, where an f32 running sum would lose the small parts"""
    return held((1000.0 + rng.standard_normal(min(n, P))).astype(F32), dt)


def _periodic_sum(block64, n):
    """sum of np.resize(block, n) in float64, without materialising it"""
    reps, rem = divmod(n, block64.size)
    return reps * block64.sum() + block64[:rem].sum()


@pytest.mark.parametrize("fn", ["sum", "mean", "mse", "dot"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_scalar_reductions_within_two_ulp(nk, dev, fn, dt):
    """nk_sum_fwd / nk_mse_fwd (reduce_stage1: f32 runs of 64 carried in f64, f64 across threads and blocks) and nk_dot
    (the same with fmaf): the result must be within 2 ulp of the float64 value rounded to f32, at n = 1, a block of 256
    and its neighbours, one grid wave +- 1 and 2^26 + 3 (about 250 elements per thread)."""
    from neuronika_b200 import ops
    w = wave(dev)
    for n in (1, 255, 256, 257, w - 1, w + 1, 2 ** 26 + 3):
        rng = np.random.default_rng(n)
        xb = _sum_block(rng, n, dt)
        X = upload_periodic(nk, dev, xb, n, dt)
        if fn in ("sum", "mean"):
            got = ops.reduce_sum(X, mean=fn == "mean").as_ndarray()
            want = _periodic_sum(xb.astype(np.float64), n) / (n if fn == "mean" else 1)
        else:
            tb = _sum_block(rng, n, dt)
            T_ = upload_periodic(nk, dev, tb, n, dt)
            x64, t64 = xb.astype(np.float64), tb.astype(np.float64)
            if fn == "mse":
                got = ops.mse(X, T_, mean=False).as_ndarray()
                want = _periodic_sum((x64 - t64) ** 2, n)
            else:
                got = ops.dot(X, T_).as_ndarray()
                want = _periodic_sum(x64 * t64, n)
        ulp2(got, want, (fn, dt, n))


@pytest.mark.parametrize("ldt,tdt", [("f32", "f32"), ("bf16", "f32"), ("f32", "bf16"), ("bf16", "bf16")])
def test_nll_forward_and_backward(nk, dev, ldt, tdt):
    """nk_nll_fwd: f64 partials, within 2 ulp of the float64 value, with class ids 0 and c - 1 present; nk_nll_bwd
    over n * c past one wave: -g/n at the target, 0 elsewhere, + beta*d -- each a single rounding, so bit exact."""
    from neuronika_b200 import ops
    combos = [(n, c) for n in (1, 257, 300000) for c in (1, 10, 1000) if n * c <= 3_000_000] + [(3000, 1000)]
    for n, c in combos:
        if tdt == "bf16" and c > 256:
            continue                                   # a bf16 target holds class ids up to 256 (nll_target_ok)
        rng = np.random.default_rng(n + c)
        logp = held(rng.uniform(-6, 0, (n, c)).astype(F32), ldt)
        tgt = rng.integers(0, c, n)
        tgt[0], tgt[-1] = 0, c - 1
        LP = dev.from_ndarray(logp, D(nk, ldt))
        T_ = dev.from_ndarray(tgt.astype(F32), D(nk, tdt))
        picked = logp.astype(np.float64)[np.arange(n), tgt]
        for mean in (True, False):
            got = ops.nll(LP, T_, mean=mean).as_ndarray()
            ulp2(got, -picked.sum() / (n if mean else 1), ("nll", n, c, mean))
        if n * c > wave(dev):
            g = dev.from_ndarray(np.asarray(G0, F32))
            gv = F32(G0) * (F32(1) / F32(n))           # (*g) * scale, scale = 1.f / float(n) on the host
            hit = np.zeros((n, c), bool)
            hit[np.arange(n), tgt] = True
            for beta in (0.0, 1.0):
                d0 = held(rng.uniform(-1, 1, (n, c)).astype(F32), ldt)
                Dl = out_buf(dev, (n, c), D(nk, ldt), beta, d0)
                ops.nll_bwd(Dl.view, T_, g, mean=True, beta=beta)
                want = np.where(hit, -float(gv), 0.0) + beta * d0
                exact(Dl.read(), stored(want, ldt), ("nll_bwd", n, c, beta))


# ============================================================================================ softmax
@pytest.mark.parametrize("log", [False, True])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_softmax_lanes_lengths_and_strides(nk, dev, dt, log):
    """One warp per lane (outer * inner lanes, stride `inner`), grid-strided over lanes (nk_softmax.cu:19).  Lengths
    around one warp and past 2^15; inner = 1 (last axis), 3 and 64; more lanes than warps in the grid (3 trips);
    lanes offset by +-1e4, where exp without the max subtraction overflows.  Forward bound, relative to y: the
    rounding of x - max, expf (2 ulp), the sum's chain (ceil(len/32) + 5) and the divide; log-softmax computes
    x - ln(sum) - max in the reference's order and its error is absolute: ~2^-24 (|x| + |max| + |ln sum|)."""
    from neuronika_b200 import ops
    D_ = D(nk, dt)
    configs = [(2 if ln * inner < 2 ** 21 else 1, ln, inner) for ln in (1, 31, 32, 33, 1000, 32769) for inner in (1, 3, 64)]
    configs += [(3 * dev.sm_count * 64 + 5, 10, 1)]          # lanes > 8 * 256 / 32 warps per SM
    fwd = ops.softmax
    for ci, (outer, ln, inner) in enumerate(configs):
        rng = np.random.default_rng(ci)
        lanes = outer * inner
        off = np.array([0.0, 1e4, -1e4])[np.arange(lanes) % 3].reshape(outer, 1, inner)
        x = held((off + 3 * rng.standard_normal((outer, ln, inner))).astype(F32), dt)
        shape = (outer, ln, inner)
        X = Guarded(dev, x, D_, 0)
        Y = out_buf(dev, shape, D_, 0, None)
        fwd(X.view, 1, out=Y.view, log=log)
        y = Y.read()
        x64 = x.astype(np.float64)
        m = x64.max(axis=1, keepdims=True)
        e = np.exp(x64 - m)
        s = e.sum(axis=1, keepdims=True)
        L = cdiv(ln, 32) + 5
        M = np.abs(x64 - m).max(axis=1, keepdims=True)
        if log:
            want = x64 - np.log(s) - m
            t = U * (2 * np.abs(x64) + 3 * np.abs(np.log(s)) + np.abs(m) + np.abs(want) + L + M + 10)
        else:
            want = e / s
            t = U * want * (np.abs(x64 - m) + M + L + 10) + 2.0 ** -140
        near(y, want, t + (UB * np.abs(want) if dt == "bf16" else 0), ("fwd", dt, log, shape))

        yb = held((rng.uniform(-8, 0, shape) if log else rng.uniform(0, 1, shape)).astype(F32), dt)
        g = held(rng.standard_normal(shape).astype(F32), dt)
        y64, g64 = yb.astype(np.float64), g.astype(np.float64)
        for beta in (0.0, 1.0):
            d0 = held(rng.uniform(-1, 1, shape).astype(F32), dt)
            DX = out_buf(dev, shape, D_, beta, d0)
            ops.softmax_bwd(DX.view, dev.from_ndarray(yb, D_), dev.from_ndarray(g, D_), 1, beta=beta, log=log)
            got = DX.read()
            if log:      # dx = g - exp(y) * sum(g)
                sg = g64.sum(axis=1, keepdims=True)
                v = g64 - np.exp(y64) * sg
                t = U * (np.exp(y64) * (6 * np.abs(sg) + L * np.abs(g64).sum(axis=1, keepdims=True))
                         + 2 * np.abs(v) + 2 * np.abs(beta * d0))
            else:        # dx = y * (g - sum(g * y))
                sg = (g64 * y64).sum(axis=1, keepdims=True)
                v = y64 * (g64 - sg)
                t = U * (np.abs(y64) * ((L + 1) * np.abs(g64 * y64).sum(axis=1, keepdims=True) + np.abs(g64 - sg))
                         + 2 * np.abs(v) + 2 * np.abs(beta * d0))
            want = v + beta * d0
            near(got, want, t + (UB * np.abs(want) if dt == "bf16" else 0), ("bwd", dt, log, shape, beta))


# ============================================================================================ mv / vm / vv
@pytest.mark.parametrize("ydt", ["f32", "bf16"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_gemv_n(nk, dev, dt, ydt):
    """y = A.x, one warp per row, grid-strided over rows (20000 > 8 warps x 8 CTAs x SMs).  The 16-byte body needs A
    and x aligned and cols % V == 0 (nk_gemv.cu:158): cols = 16V takes it, 16V + 1 and an A or x one element off do
    not.  Chain per lane: ceil(cols / 32) + V fmas, + 5 for the warp sum, + 1 for beta."""
    from neuronika_b200 import ops
    V, rows = VEC[dt], 20000
    for cols in (16 * V, 16 * V + 1):
        rng = np.random.default_rng(cols)
        a = periodic(rng, rows * cols, -1, 1, dt).reshape(rows, cols)
        x = held(rng.uniform(-1, 1, cols).astype(F32), dt)
        prod = a.astype(np.float64) @ x.astype(np.float64)
        mag = np.abs(a.astype(np.float64)) @ np.abs(x.astype(np.float64))
        L = cdiv(cols, 32) + V + 5
        for aoff, xoff in ((0, 0), (1, 0), (0, 1)):
            for beta in (0.0, 1.0):
                y0 = held(rng.uniform(-1, 1, rows).astype(F32), ydt)
                A_, X_ = Guarded(dev, a, D(nk, dt), aoff), Guarded(dev, x, D(nk, dt), xoff)
                Y = out_buf(dev, (rows,), D(nk, ydt), beta, y0)
                ops.gemv(A_.view, X_.view, Y.view, trans=False, beta=beta)
                want = prod + beta * y0
                near(Y.read(), want, tol(L + 1, mag + np.abs(beta * y0), want, ydt), (cols, aoff, xoff, beta))


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_gemv_t(nk, dev, dt):
    """y = A^T.x: threads own columns, row chunks of rows_per_block (>= 32) combined with atomics (nk_gemv.cu:172).
    Rows around one chunk and 100000 rows (1000+ chunks); columns around one 256-thread block.  (100000 rows are run
    with 1 and 257 columns only: 100000 x 5000 would be 2 GB of host data.)  Chain: rows_per_block fmas + the row
    chunks' atomics + 1 for beta."""
    from neuronika_b200 import ops
    sm = dev.sm_count
    for rows in (1, 31, 32, 33, 100000):
        for cols in (1, 255, 256, 257, 5000):
            if rows == 100000 and cols not in (1, 257):
                continue
            rng = np.random.default_rng(rows * 7 + cols)
            a = periodic(rng, rows * cols, -1, 1, dt).reshape(rows, cols)
            x = held(rng.uniform(-1, 1, rows).astype(F32), dt)
            want0 = x.astype(np.float64) @ a.astype(np.float64)
            mag = np.abs(x.astype(np.float64)) @ np.abs(a.astype(np.float64))
            rpb = max(32, cdiv(rows, cdiv(sm * 8, cdiv(cols, 256))))
            L = rpb + cdiv(rows, rpb) + 1
            for beta in (0.0, 1.0):
                y0 = held(rng.uniform(-1, 1, cols).astype(F32), dt)
                Y = out_buf(dev, (cols,), D(nk, dt), beta, y0)
                ops.gemv(dev.from_ndarray(a, D(nk, dt)), dev.from_ndarray(x, D(nk, dt)), Y.view, trans=True, beta=beta)
                want = want0 + beta * y0
                near(Y.read(), want, tol(L, mag + np.abs(beta * y0), want, dt), (rows, cols, beta))


@pytest.mark.parametrize("ddt", ["f32", "bf16"])
@pytest.mark.parametrize("sdt", ["f32", "bf16"])
def test_outer_and_scale_accumulate(nk, dev, ddt, sdt):
    """A = beta*A + u (x) v and dst = beta*dst + x*s in every (dst, src) type pair, past one wave (grid-strided).
    Two roundings: the product and the beta sum."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(3)
    rows, cols = 600, 1000
    u = held(rng.uniform(-2, 2, rows).astype(F32), sdt)
    v = held(rng.uniform(-2, 2, cols).astype(F32), sdt)
    n = 2 * wave(dev) + 7
    x = periodic(rng, n, -2, 2, sdt)
    s = F32(-0.37)
    for beta in (0.0, 1.0):
        a0 = held(rng.uniform(-2, 2, (rows, cols)).astype(F32), ddt)
        A_ = out_buf(dev, (rows, cols), D(nk, ddt), beta, a0)
        ops.outer_acc(A_.view, dev.from_ndarray(u, D(nk, sdt)), dev.from_ndarray(v, D(nk, sdt)), beta=beta)
        uv = np.outer(u.astype(np.float64), v.astype(np.float64))
        want = uv + beta * a0
        near(A_.read(), want, tol(2, np.abs(uv) + np.abs(beta * a0), want, ddt), ("outer", beta))

        d0 = periodic(rng, n, -2, 2, ddt)
        Dst = out_buf(dev, (n,), D(nk, ddt), beta, d0)
        ops.scale_acc(Dst.view, dev.from_ndarray(x, D(nk, sdt)), dev.from_ndarray(np.asarray(s, F32)), beta=beta)
        xs = x.astype(np.float64) * float(s)
        want = xs + beta * d0
        near(Dst.read(), want, tol(2, np.abs(xs) + np.abs(beta * d0), want, ddt), ("scale", beta))


# ============================================================================================ optimizers
def optim_hyper(dev, lr, step=0):
    """an nk_optim_hyper block holding lr and the step count"""
    import ctypes as C
    from neuronika_b200 import _lib as L
    from neuronika_b200.device import CuArray
    h = CuArray(dev, (C.sizeof(L.OptimHyper) // 4,), L.NK_F32)
    L.check(L.lib.nk_optim_hyper_set(dev.ctx, h.ptr, C.byref(L.OptimHyper(lr=lr, step=step))), dev.ctx)
    return h


def one(a):
    """the pointer array of a count = 1 call: the device array's pointer, or NULL"""
    import ctypes as C
    return None if a is None else (C.c_void_p * 1)(a.ptr.value)


def one_n(n):
    import ctypes as C
    return (C.c_int64 * 1)(n)


SGD_CFGS = {
    "plain": dict(momentum=0.0, dampening=0.0, nesterov=False, l2=0.0, grad_scale=1.0, wbg=1),
    "momentum_dampening_l2_scaled": dict(momentum=0.9, dampening=0.1, nesterov=False, l2=0.01, grad_scale=0.5, wbg=1),
    "nesterov_l2_no_writeback": dict(momentum=0.9, dampening=0.0, nesterov=True, l2=0.01, grad_scale=1.0, wbg=0),
    "scaled": dict(momentum=0.0, dampening=0.0, nesterov=False, l2=0.0, grad_scale=0.5, wbg=1),
}


@pytest.mark.parametrize("cfg", list(SGD_CFGS))
@pytest.mark.parametrize("wdt,gdt", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
def test_multi_sgd_vector_and_element_bodies_agree(nk, dev, wdt, gdt, cfg):
    """nk_multi_sgd_step on one tensor takes 4-element accesses (the last n % 4 elements one by one, by the thread that
    owns them) when w, g, buf and master all allow them (`vec` in nk_optim_multi.cu's multi_step), element accesses
    otherwise, with the same per-element arithmetic: the aligned run and runs with w, g, buf or master one element off
    (each alone, then all) must agree bit for bit, and with a float64 single step.  bf16 weights keep f32 master
    weights and must equal bf16_round(master); g is unchanged unless it is written back with a penalty or a scale."""
    from neuronika_b200 import _lib as L
    c = SGD_CFGS[cfg]
    lr, mu, l2x2 = float(F32(0.1)), float(F32(c["momentum"])), 2 * F32(c["l2"])   # f32 arguments
    omd = float(F32(1) - F32(c["dampening"]))
    mom, master_on = mu > 0, wdt == "bf16"
    hyper = optim_hyper(dev, 0.1)
    for n in (1, 3, 4, 5, 4001, 4002, 4003, 4 * wave(dev) + 3):
        rng = np.random.default_rng(n)
        m0 = rng.uniform(-1, 1, n).astype(F32)
        w0 = held(m0, wdt)
        g0 = held(rng.standard_normal(n).astype(F32), gdt)
        b0 = (0.1 * rng.standard_normal(n)).astype(F32)
        names = ["w", "g"] + (["buf"] if mom else []) + (["master"] if master_on else [])
        runs = {}
        for lay in ["aligned"] + [nm + "+1" for nm in names] + ["all+1"]:
            off = {nm: int(lay == "all+1" or lay == nm + "+1") for nm in names}
            W = Guarded(dev, w0, D(nk, wdt), off["w"])
            Gr = Guarded(dev, g0, D(nk, gdt), off["g"])
            B = Guarded(dev, b0, nk.F32, off["buf"]) if mom else None
            M = Guarded(dev, m0, nk.F32, off["master"]) if master_on else None
            L.check(L.lib.nk_multi_sgd_step(dev.ctx, 1, one(W.view), one(Gr.view), W.view.dtype, Gr.view.dtype,
                                            one(B.view if mom else None), one(M.view if master_on else None), one_n(n),
                                            hyper.ptr, c["l2"], mu, c["dampening"], int(c["nesterov"]),
                                            c["grad_scale"], c["wbg"]), dev.ctx)
            runs[lay] = [W.read(), Gr.read(), B.read() if mom else None, M.read() if master_on else None]
        base = runs["aligned"]
        for lay, r in runs.items():
            for i, (a, b) in enumerate(zip(base, r)):
                if a is not None:
                    exact(b, a, (cfg, n, lay, ["w", "g", "buf", "master"][i], "differs from the aligned run"))
        w1, g1, b1, mst = base
        wv = (m0 if master_on else w0).astype(np.float64)
        gs = g0.astype(np.float64) * c["grad_scale"]
        gv = gs + float(l2x2) * wv
        Sg = np.abs(gs) + float(l2x2) * np.abs(wv)
        if mom:
            bn = b0 * mu + gv * omd
            upd = gv + bn * mu if c["nesterov"] else bn
            Sb = mu * np.abs(b0) + Sg
            near(b1, bn, 6 * U * Sb, (cfg, n, "buf"))                          # gv 2, 2 products + 1 sum (+1)
        else:
            upd, Sb = gv, Sg
        wn = wv - upd * lr
        Sw = np.abs(wv) + lr * (1 + mu) * Sb
        if master_on:
            near(mst, wn, 8 * U * Sw, (cfg, n, "master"))                     # gv 2, buf 3, nesterov 2, w 2 roundings
            exact(w1, held(mst, "bf16"), (cfg, n, "w != bf16_round(master)"))
        else:
            near(w1, wn, 8 * U * Sw, (cfg, n, "w"))
        if c["wbg"] and not (c["l2"] == 0 and c["grad_scale"] == 1):
            near(g1, gv, tol(2, Sg, gv, gdt), (cfg, n, "g written back"))     # scale, then + l2 term
        else:
            exact(g1, g0, (cfg, n, "g must be unchanged"))


# ============================================================================================ Adam family
ADAM_KINDS = ["adam", "amsgrad", "rmsprop", "rmsprop_centered", "rmsprop_momentum", "rmsprop_centered_momentum",
              "adagrad"]


@pytest.mark.parametrize("kind", ADAM_KINDS)
@pytest.mark.parametrize("wdt,gdt", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
def test_multi_adam_family_one_step(nk, dev, O, kind, wdt, gdt):
    """One fused step over 2 * wave + 7 elements (nk_multi_*_step on one tensor), against the oracle's restatement
    (f32, the reference's operation order) on random optimizer state: grad_scale 0.5, an L1 penalty with w = +0 and -0
    (signum(+-0) = +-1), write_back_grad = 0 (g must not change), Adam and Adagrad at step 10000 (bias correction and
    learning-rate decay from nk_optim_prologue, which advances the block's step count from 9999).  bf16 weights keep f32 master weights.  Bound: 2 * 2^-24 * |w| for the
    final subtraction + 32 * 2^-24 * the update's term magnitudes (fused vs separate roundings in the moments)."""
    from neuronika_b200 import _lib as L
    n = 2 * wave(dev) + 7
    rng = np.random.default_rng(ADAM_KINDS.index(kind))
    m0 = rng.uniform(-1, 1, n).astype(F32)
    m0[::1000] = 0.0
    m0[1::1000] = -0.0
    w0 = held(m0, wdt)
    master_on = wdt == "bf16"
    g0 = held(rng.standard_normal(n).astype(F32), gdt)
    gs, l1, step, lr, eps = 0.5, 0.01, 10000, 1e-2, 1e-8
    st = {"ea": rng.standard_normal(n).astype(F32) * F32(0.1), "sq": rng.uniform(1, 2, n).astype(F32),
          "mx": rng.uniform(1, 2, n).astype(F32), "ga": rng.uniform(-0.1, 0.1, n).astype(F32),
          "bf": rng.standard_normal(n).astype(F32) * F32(0.1)}
    W, Gr = Guarded(dev, w0, D(nk, wdt)), Guarded(dev, g0, D(nk, gdt))
    M = Guarded(dev, m0, nk.F32) if master_on else None
    dS = {k: dev.from_ndarray(v) for k, v in st.items()}
    ctx, mp = dev.ctx, one(M.view if master_on else None)
    hyper = optim_hyper(dev, lr, step - 1)
    wref = (m0 if master_on else w0).copy()
    go = (g0 * F32(gs)).astype(F32)                      # the kernel scales in f32 before adding the penalty
    sign = np.where(np.signbit(wref), -1.0, 1.0)
    gv = go.astype(np.float64) + l1 * sign
    ref = {k: v.copy() for k, v in st.items()}
    if kind in ("adam", "amsgrad"):
        ams = kind == "amsgrad"
        L.check(L.lib.nk_optim_prologue(ctx, hyper.ptr, L.NK_OPTIM_ADAM, 0.9, 0.999, 0.0), ctx)
        L.check(L.lib.nk_multi_adam_step(ctx, 1, one(W.view), one(Gr.view), W.view.dtype, Gr.view.dtype, one(dS["ea"]),
                                         one(dS["sq"]), one(dS["mx"] if ams else None), mp, one_n(n), hyper.ptr, 0.9,
                                         0.999, eps, l1, 0.0, gs, 0), ctx)
        O.adam_step(wref, go, ref["ea"], ref["sq"], step, lr, 0.9, 0.999, eps, l1, 0.0,
                    max_exp_avg_sq=ref["mx"] if ams else None)
        Mm = np.abs(st["ea"]) * 0.9 + np.abs(gv) * 0.1
        Mv = st["sq"] * 0.999 + gv * gv * 0.001
        vv = np.maximum(ref["mx"], ref["sq"]) if ams else ref["sq"]
        bc2 = 1 - 0.999 ** step
        Mw = lr / (1 - 0.9 ** step) * Mm / (np.sqrt(vv) / np.sqrt(bc2) + eps)
        checks = {"ea": Mm, "sq": Mv} | ({"mx": Mv} if ams else {})
    elif kind == "adagrad":
        L.check(L.lib.nk_optim_prologue(ctx, hyper.ptr, L.NK_OPTIM_ADAGRAD, 0.0, 0.0, 0.1), ctx)
        L.check(L.lib.nk_multi_adagrad_step(ctx, 1, one(W.view), one(Gr.view), W.view.dtype, Gr.view.dtype,
                                            one(dS["sq"]), mp, one_n(n), hyper.ptr, eps, l1, 0.0, gs, 0), ctx)
        O.adagrad_step(wref, go, ref["sq"], step, lr, 0.1, eps, l1, 0.0)
        Ms = st["sq"] + gv * gv
        Mw = lr / (1 + (step - 1) * 0.1) * np.abs(gv) / (np.sqrt(Ms) + eps)
        checks = {"sq": Ms}
    else:
        centered, mom = "centered" in kind, "momentum" in kind
        L.check(L.lib.nk_multi_rmsprop_step(ctx, 1, one(W.view), one(Gr.view), W.view.dtype, Gr.view.dtype,
                                            one(dS["sq"]), one(dS["ga"] if centered else None),
                                            one(dS["bf"] if mom else None), mp, one_n(n), hyper.ptr, 0.99, eps,
                                            0.9 if mom else 0.0, l1, 0.0, gs, 0), ctx)
        O.rmsprop_step(wref, go, ref["sq"], lr, 0.99, eps, momentum=0.9 if mom else None, centered=centered,
                       grad_avg=ref["ga"], buffer=ref["bf"], l1=l1, l2=0.0)
        Msq = st["sq"] * 0.99 + gv * gv * 0.01
        Mga = np.abs(st["ga"]) * 0.99 + np.abs(gv) * 0.01
        denom = np.sqrt(ref["sq"].astype(np.float64) - (ref["ga"].astype(np.float64) ** 2 if centered else 0)) + eps
        Mb = (np.abs(st["bf"]) * 0.9 if mom else 0) + np.abs(gv) / denom
        Mw = lr * Mb
        checks = {"sq": Msq} | ({"ga": Mga} if centered else {}) | ({"bf": Mb} if mom else {})
    exact(Gr.read(), g0, (kind, "g must be unchanged with write_back_grad = 0"))
    for k, mag in checks.items():
        near(dS[k].as_ndarray(), ref[k], 16 * U * mag, (kind, k))       # a few fused-vs-separate roundings
    wgot = M.read() if master_on else W.read()
    near(wgot, wref, U * (2 * np.abs(wref) + 32 * Mw), (kind, "w"))
    if master_on:
        exact(W.read(), held(wgot, "bf16"), (kind, "w != bf16_round(master)"))


# ============================================================================================ shape ops, bit exact
@pytest.mark.parametrize("ddt", ["f32", "bf16"])
@pytest.mark.parametrize("sdt", ["f32", "bf16"])
def test_transpose_bit_exact(nk, dev, sdt, ddt):
    """transpose2d: 32 x 32 tiles, grid-strided over tiles (nk_pointwise.cu:249): rows and cols at 31 / 32 / 33, and
    2049 x 2081 (65 x 66 tiles, more than the grid); transpose_nd: a 6-d reversal.  All four type pairs; bf16 <- f32
    is bf16_round of the source; beta = 1 rounds the exact sum once."""
    from neuronika_b200 import ops
    shapes = [(r, c) for r in (31, 32, 33) for c in (31, 32, 33)] + [(2049, 2081), (3, 4, 5, 6, 7, 8)]
    for si, shape in enumerate(shapes):
        rng = np.random.default_rng(si)
        x = held(rng.uniform(-2, 2, shape).astype(F32), sdt)
        X = Guarded(dev, x, D(nk, sdt), 0)
        xt = np.ascontiguousarray(x.T).astype(np.float64)
        for beta in (0.0, 1.0):
            d0 = held(rng.uniform(-2, 2, xt.shape).astype(F32), ddt)
            Y = out_buf(dev, xt.shape, D(nk, ddt), beta, d0)
            ops.transpose(X.view, out=Y.view, beta=beta)
            exact(Y.read(), stored(xt + beta * d0, ddt), (shape, beta))


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_pad2d_pair_and_single_stores(nk, dev, dt):
    """pad2d_fwd stores 2 elements per thread when the output row is even and y is aligned to 2 elements, else 1
    (nk_elementwise.cu:933); pad2d_bwd likewise on the input row and dx (:956).  Odd and even widths, y or dx one
    element off, beta 0 and 1, and a case past one wave.  Copies, so bit exact."""
    from neuronika_b200 import ops
    D_ = D(nk, dt)
    cases = [((3, 5, 6), (1, 2), 0), ((3, 5, 7), (1, 2), 0), ((3, 5, 6), (1, 2), 1), ((3, 5, 7), (2, 1), 1),
             ((700, 30, 30), (1, 1), 0), ((700, 30, 31), (1, 1), 0)]
    for ci, (shape, (ph, pw), off) in enumerate(cases):
        rng = np.random.default_rng(ci)
        x = held(rng.uniform(-2, 2, shape).astype(F32), dt)
        ys = (shape[0], shape[1] + 2 * ph, shape[2] + 2 * pw)
        X = Guarded(dev, x, D_, 0)
        Y = out_buf(dev, ys, D_, 0, None, off)
        ops.pad2d(X.view, (ph, pw), value=0.5, out=Y.view)
        want = np.pad(x, ((0, 0), (ph, ph), (pw, pw)), constant_values=0.5)
        exact(Y.read(), want, ("fwd", shape, ph, pw, off))
        g = held(rng.uniform(-2, 2, ys).astype(F32), dt)
        G_ = Guarded(dev, g, D_, 0)
        for beta in (0.0, 1.0):
            d0 = held(rng.uniform(-2, 2, shape).astype(F32), dt)
            DX = out_buf(dev, shape, D_, beta, d0, off)
            ops.pad2d_bwd(DX.view, G_.view, (ph, pw), beta=beta)
            want = g[:, ph:ph + shape[1], pw:pw + shape[2]].astype(np.float64) + beta * d0
            exact(DX.read(), stored(want, dt), ("bwd", shape, ph, pw, off, beta))


@pytest.mark.parametrize("mode", ["constant", "reflective", "replicative"])
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_padnd_modes_at_full_reflection(nk, dev, dt, mode):
    """padnd over 1 to 3 sample dims with pad = len - 1 (the largest reflection) on some axes and 0 on others; the
    3-d case has more output elements than two grid waves.  Forward and backward (the interior, whatever the mode,
    beta 0 and 1), bit exact against the oracle."""
    from neuronika_b200 import ops
    D_ = D(nk, dt)
    w = wave(dev)
    cases = [((4, 9), (8,)), ((2, 3, 4, 5), (3, 0)), ((cdiv(2 * w + 1, 13 * 6 * 19), 5, 6, 7), (4, 0, 6))]
    for ci, (shape, pad) in enumerate(cases):
        rng = np.random.default_rng(ci)
        x = held(rng.uniform(-2, 2, shape).astype(F32), dt)
        want = O_pad(x, pad, mode)
        X = Guarded(dev, x, D_, 0)
        Y = out_buf(dev, want.shape, D_, 0, None)
        ops.pad_nd(X.view, pad, mode=mode, value=0.5, out=Y.view)
        exact(Y.read(), want, ("fwd", shape, pad))
        g = held(rng.uniform(-2, 2, want.shape).astype(F32), dt)
        for beta in (0.0, 1.0):
            d0 = held(rng.uniform(-2, 2, shape).astype(F32), dt)
            DX = out_buf(dev, shape, D_, beta, d0)
            ops.pad_nd_bwd(DX.view, dev.from_ndarray(g, D_), pad, beta=beta)
            sl = tuple([slice(None)] * (len(shape) - len(pad)) + [slice(p, s + p) for p, s in zip(pad, shape[-len(pad):])])
            exact(DX.read(), stored(g[sl].astype(np.float64) + beta * d0, dt), ("bwd", shape, pad, beta))


def O_pad(x, pad, mode):
    from oracle import pad_mode_forward
    return pad_mode_forward(x, pad, mode, F32(0.5))


@pytest.mark.parametrize("planes", [2047, 2049])
def test_pad2d_index_width_at_2_31(nk, dev, planes):
    """nk_pad2d_fwd / _bwd index in 32 bits below 2^31 output elements and in 64 bits from there
    (nk_elementwise.cu:934, 957).  (planes, 1022, 1022) bf16 padded by 1: each output plane is 2^20 elements, so
    plane 2048 starts at element 2^31.  The input is filled on the device with (i + 3j + 5p) mod 256, exact in bf16.
    Checked: plane 0, planes 2046-2048 (those that exist) and the last plane of y, no NaN left anywhere in y, the
    guard past its end, and the backward (the interior, beta = 0) equal to x everywhere.  x, y and dx take 12.9 GB."""
    import torch
    from neuronika_b200 import ops
    from neuronika_b200.device import CuArray
    h = 1022
    ho = h + 2
    need = planes * (h * h * 2 + ho * ho) * 2 + (1 << 30)     # x, dx, y + scratch
    free, _ = torch.cuda.mem_get_info()
    if free < max(need, 12 << 30):
        pytest.skip(f"needs about {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    base = (torch.arange(h, device="cuda", dtype=torch.int32)[:, None]
            + 3 * torch.arange(h, device="cuda", dtype=torch.int32)[None, :])
    xt = torch.empty((planes, h, h), dtype=torch.bfloat16, device="cuda")
    for p0 in range(0, planes, 256):
        p = torch.arange(p0, min(p0 + 256, planes), device="cuda", dtype=torch.int32)
        xt[p0:p0 + p.numel()] = ((base[None] + 5 * p[:, None, None]) % 256).to(torch.bfloat16)
    del base
    tail = 64
    yt = torch.full((planes * ho * ho + tail,), float("nan"), dtype=torch.bfloat16, device="cuda")
    yt[planes * ho * ho:] = CANARY
    dxt = torch.full((planes, h, h), float("nan"), dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()
    x = CuArray(dev, (planes, h, h), nk.BF16, ptr=xt.data_ptr(), owner=xt)
    ybuf = CuArray(dev, (yt.numel(),), nk.BF16, ptr=yt.data_ptr(), owner=yt)
    y = ybuf.slice_flat(0, (planes, ho, ho))
    dx = CuArray(dev, (planes, h, h), nk.BF16, ptr=dxt.data_ptr(), owner=dxt)
    ops.pad2d(x, (1, 1), value=0.0, out=y)
    ops.pad2d_bwd(dx, y, (1, 1), beta=0.0)
    dev.synchronize()
    ij = (np.arange(h)[:, None] + 3 * np.arange(h)[None, :])
    for p in sorted({0, 2046, 2047, 2048, planes - 1} & set(range(planes))):
        plane = y.slice_flat(p * ho * ho, (ho, ho)).as_ndarray()
        want = np.zeros((ho, ho), F32)
        want[1:-1, 1:-1] = (ij + 5 * p) % 256
        exact(plane, want, ("y plane", p))
    assert not any(bool(torch.isnan(c).any()) for c in yt.split(1 << 28)), "y has elements the forward did not write"
    assert bool((yt[planes * ho * ho:] == CANARY).all()), "the forward wrote past the end of y"
    assert all(torch.equal(a, b) for a, b in zip(dxt.view(torch.int16).split(256), xt.view(torch.int16).split(256))), \
        "backward: dx != x"
    del x, y, ybuf, dx, xt, yt, dxt
    torch.cuda.empty_cache()
