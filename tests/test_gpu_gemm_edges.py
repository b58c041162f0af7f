"""The wgmma GEMM engine at its edges, through the C ABI with explicit leading dimensions: every form x tile width, a
multi-wave persistent schedule with a partial group of m-blocks, the epilogue (alpha, bias, ReLU, beta) on both drains,
leading dimensions above their minimum and bases that TMA cannot address, and the fused ReLU backward with and without
column sums.

Operands and C are views into larger buffers filled with a canary value.  The view is checked against a float64
reference on the same bf16-rounded operands, relu(alpha.op(A)op(B) + bias + beta.C0) (nk_gemm_simt.cu's epilogue order);
every element outside the view -- the ldc - N gap of each row included -- must still hold the canary, bit for bit.
Tolerances: f32 output 2e-3.rms(want) + 1e-6; bf16 output + 2^-8.|want|; bf16 output accumulated into (beta != 0)
+ 2^-7.|want|."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0          # exact in bf16 and f32, far outside every product below
FORMS = {"NN": (0, 0), "NT": (0, 1), "TN": (1, 0), "TT": (1, 1)}


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


def ceil8(v):
    return (v + 7) // 8 * 8


def rms(x):
    return float(np.sqrt((np.asarray(x, np.float64) ** 2).mean())) if np.size(x) else 0.0


class Strided:
    """A rows x cols matrix at element `off` of a buffer, rows `ld` elements apart; every other element of the buffer
    (row gaps, the bytes before `off`, a tail guard) holds CANARY."""

    def __init__(self, dev, data, dtype, ld=None, off=0, tail=40):
        data = np.asarray(data, F32)
        if data.ndim == 1:
            data = data[None, :]
        self.rows, self.cols = data.shape
        self.ld = self.cols if ld is None else ld
        self.off = off
        assert self.ld >= self.cols
        self.size = off + self.rows * self.ld + tail
        host = np.full(self.size, CANARY, F32)
        self._inner(host)[:] = data
        self.buf = dev.from_ndarray(host, dtype)
        self.view = self.buf.slice_flat(off, (self.rows * self.ld,))
        self.ptr = self.view.ptr

    def _inner(self, flat):
        return flat[self.off:self.off + self.rows * self.ld].reshape(self.rows, self.ld)[:, :self.cols]

    def read(self):
        """(the view, after asserting that nothing outside it changed)"""
        flat = self.buf.as_ndarray()
        outside = np.ones(self.size, bool)
        self._inner(outside)[:] = False
        bad = np.flatnonzero(flat[outside] != CANARY)
        assert bad.size == 0, f"{bad.size} elements outside the view were written (first at outside index {bad[0]})"
        return self._inner(flat).copy()


def check(got, want, c_bf16, accumulated, what):
    want = np.asarray(want, np.float64)
    rel = (2.0 ** -7 if accumulated else 2.0 ** -8) if c_bf16 else 0.0
    tol = 2e-3 * rms(want) + rel * np.abs(want) + 1e-6
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= tol), (what, float(err.max()), int(np.argmax(err > tol)), rms(want))


def operands(O, rng, form, M, N, K, pad_a=0, pad_b=0):
    """bf16-rounded op(A) (M x K), op(B) (K x N) and their stored layouts with leading dimensions rounded up to 8
    elements (TMA row pitch) plus pad_a / pad_b"""
    ta, tb = FORMS[form]
    a = O.bf16_round(rng.uniform(-1, 1, (K, M) if ta else (M, K)).astype(F32))
    b = O.bf16_round(rng.uniform(-1, 1, (N, K) if tb else (K, N)).astype(F32))
    lda = ceil8(a.shape[1]) + pad_a
    ldb = ceil8(b.shape[1]) + pad_b
    opa = (a.T if ta else a).astype(np.float64)
    opb = (b.T if tb else b).astype(np.float64)
    return (a, lda), (b, ldb), opa @ opb


def run_gemm(nk, dev, O, form, M, N, K, cdt, *, alpha=1.0, beta=0.0, bias=None, relu=False, ldc=None, off_c=0,
             pad_a=0, pad_b=0, off_a=0, seed=0):
    """nk_gemm_bias_act on canary-guarded views; bias in {None, "f32", "bf16"} with an optional "+1" suffix (the bias
    view one element off its 16-byte alignment).  Returns (C view, reference, kernel name)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ta, tb = FORMS[form]
    (a, lda), (b, ldb), prod = operands(O, rng, form, M, N, K, pad_a, pad_b)
    A = Strided(dev, a, nk.BF16, lda, off_a)
    B = Strided(dev, b, nk.BF16, ldb)
    c_bf16 = cdt == nk.BF16
    c0 = rng.uniform(-1, 1, (M, N)).astype(F32)
    if c_bf16:
        c0 = O.bf16_round(c0)
    Cm = Strided(dev, c0, cdt, N if ldc is None else ldc, off_c)
    want = alpha * prod
    bptr, bdt = None, nk.F32
    if bias is not None:
        bdt = nk.BF16 if bias.startswith("bf16") else nk.F32
        bv = rng.uniform(-1, 1, N).astype(F32)
        if bdt == nk.BF16:
            bv = O.bf16_round(bv)
        Bias = Strided(dev, bv, bdt, off=1 if bias.endswith("+1") else 0)
        bptr = Bias.ptr
        want = want + bv[None, :]
    want = want + beta * c0
    if relu:
        want = np.maximum(want, 0.0)
    rc = ops.lib.nk_gemm_bias_act(dev.ctx, ta, tb, M, N, K, float(alpha), A.ptr, lda, B.ptr, ldb, float(beta), Cm.ptr,
                                  Cm.ld, nk.BF16, cdt, bptr, bdt, int(relu))
    nk._lib.check(rc, dev.ctx)
    kern = dev.last_gemm_kernel
    return Cm.read(), want, kern


# ------------------------------------------------------------------------------------------- form x tile width
WIDTH_N = {16: 13, 32: 27, 64: 50, 128: 100, 256: 300}
FORM_WIDTHS = [(f, w) for f in ("NT", "TT") for w in (16, 32, 64, 128, 256)] + \
              [(f, w) for f in ("NN", "TN") for w in (64, 128, 256)]


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("form,width", FORM_WIDTHS)
def test_every_form_and_tile_width(nk, dev, O, form, width, cdt):
    """every BLOCK_N the dispatcher can choose (16 / 32 only with a K-major B), M not a multiple of 128, K not a multiple
    of 64 (K = 8 < 16 on the narrow tiles), leading dimensions 8 elements above their minimum and a gap after each C row"""
    c = nk.F32 if cdt == "f32" else nk.BF16
    N = WIDTH_N[width]
    K = 8 if width == 16 else 136
    beta = 1.0 if c == nk.BF16 else 0.0
    got, want, kern = run_gemm(nk, dev, O, form, 200, N, K, c, beta=beta, ldc=ceil8(N) + 8, pad_a=8, pad_b=8,
                               seed=width * 10 + len(cdt))
    assert kern == f"wgmma_{form.lower()}_128x{width}"
    check(got, want, c == nk.BF16, beta != 0, (form, width, cdt))


# ------------------------------------------------------------------------------------------- persistent schedule
@pytest.mark.parametrize("form", ["NT", "NN", "TN", "TT"])
def test_multi_wave_schedule_with_a_partial_group(nk, dev, O, form):
    """more than two waves of 128 x 256 tiles whose m-blocks (18) leave a partial group of kGroupM = 16; K = 3 k-blocks,
    so the 4-stage ring wraps across tiles.  The whole output is checked."""
    sm = dev.sm_count
    m_blocks = 18
    n_blocks = max(17, -(-2 * sm // m_blocks) + 1)
    M, N, K = m_blocks * 128 - 104, n_blocks * 256 - 104, 192
    assert m_blocks * n_blocks > 2 * sm and m_blocks % 16 != 0
    got, want, kern = run_gemm(nk, dev, O, form, M, N, K, nk.F32, ldc=N + 8, seed=7)
    assert kern == f"wgmma_{form.lower()}_128x256"
    check(got, want, False, False, form)


# ------------------------------------------------------------------------------------------- epilogue matrix
# (C dtype, drain) -> (N, ldc, C offset): the row drain needs 16-byte aligned rows; the column drain takes the rest
DRAINS = {
    ("f32", "rows"): (200, 208, 0),
    ("bf16", "rows"): (200, 216, 0),
    ("f32", "columns"): (201, 203, 0),      # N % 4 != 0
    ("bf16", "columns"): (203, 205, 0),     # N % 8 != 0
    ("f32", "c+1"): (200, 208, 1),          # C base one element off 16-byte alignment
    ("bf16", "c+1"): (200, 208, 1),
}


@pytest.mark.parametrize("cdt,drain", list(DRAINS))
def test_epilogue_matrix(nk, dev, O, cdt, drain):
    """alpha x beta x bias (none, f32, bf16; aligned and one element off) x ReLU on each drain of the epilogue"""
    c = nk.F32 if cdt == "f32" else nk.BF16
    N, ldc, off_c = DRAINS[(cdt, drain)]
    biases = [None, "f32", "f32+1"] + (["bf16", "bf16+1"] if c == nk.BF16 else [])
    i = 0
    for alpha in (1.0, -0.75):
        for beta in (0.0, 0.5, 1.0):
            for bias in biases:
                for relu in (False, True):
                    i += 1
                    got, want, kern = run_gemm(nk, dev, O, "NT", 200, N, 72, c, alpha=alpha, beta=beta, bias=bias,
                                               relu=relu, ldc=ldc, off_c=off_c, seed=i)
                    assert kern == "wgmma_nt_128x256"
                    check(got, want, c == nk.BF16, beta != 0, (cdt, drain, alpha, beta, bias, relu))


# ------------------------------------------------------------------------------------------- leading dimensions
@pytest.mark.parametrize("form", ["NT", "NN", "TN", "TT"])
def test_leading_dimensions_and_unaligned_base(nk, dev, O, form):
    """lda / ldb above their minimum and ldc > N stay on wgmma; an A base one element off 16-byte alignment falls back to
    the SIMT engine with the same numbers, and is an error when the tensor-core engine is forced"""
    M, N, K = 150, 180, 100
    got, want, kern = run_gemm(nk, dev, O, form, M, N, K, nk.BF16, beta=1.0, ldc=N + 12, pad_a=24, pad_b=16, seed=11)
    assert kern.startswith(f"wgmma_{form.lower()}_")
    check(got, want, True, True, form)
    got, want, kern = run_gemm(nk, dev, O, form, M, N, K, nk.F32, beta=0.5, ldc=N + 3, pad_a=24, off_a=1, seed=12)
    assert kern.startswith("simt")
    check(got, want, False, True, form)
    dev.gemm_engine("wgmma")
    try:
        with pytest.raises(nk.NkError, match="not TMA-addressable"):
            run_gemm(nk, dev, O, form, M, N, K, nk.F32, off_a=1, seed=13)
    finally:
        dev.gemm_engine("auto")
    got, want, kern = run_gemm(nk, dev, O, form, M, N, K, nk.F32, seed=14)    # the context still works
    assert kern.startswith(f"wgmma_{form.lower()}_")
    check(got, want, False, False, form)


# ------------------------------------------------------------------------------------------- fused ReLU backward
def mask_values(rng, shape):
    """exact zeros, negatives and positives in equal parts"""
    return rng.choice(np.array([-1.0, 0.0, 1.0], F32), shape) * rng.uniform(0.25, 1.0, shape).astype(F32)


def run_relu_bwd(nk, dev, O, form, M, N, K, cdt, *, beta=0.0, ldc=None, off_c=0, off_mask=0, colsum=False, lda=None,
                 seed=0):
    """nk_gemm_relu_bwd(_colsum): C = beta.C0 + (mask > 0).op(A)op(B), mask (M, N) with C's type and leading dimension;
    colsum (N floats, starting from random values) += column sums of the stored C.  Returns (C, reference, colsum,
    colsum start, kernel name)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ta, tb = FORMS[form]
    (a, lda_), (b, ldb), prod = operands(O, rng, form, M, N, K)
    if lda is not None:
        lda_ = lda
    A = Strided(dev, a, nk.BF16, lda_)
    B = Strided(dev, b, nk.BF16, ldb)
    c_bf16 = cdt == nk.BF16
    rnd = (lambda v: O.bf16_round(v)) if c_bf16 else (lambda v: v)
    c0 = rnd(rng.uniform(-1, 1, (M, N)).astype(F32))
    mk = rnd(mask_values(rng, (M, N)))
    ld = N if ldc is None else ldc
    Cm = Strided(dev, c0, cdt, ld, off_c)
    Mk = Strided(dev, mk, cdt, ld, off_mask)
    want = beta * c0 + np.where(mk > 0, prod, 0.0)
    s0 = rng.uniform(-1, 1, N).astype(F32)
    S = Strided(dev, s0, nk.F32) if colsum else None
    if colsum:
        rc = ops.lib.nk_gemm_relu_bwd_colsum(dev.ctx, ta, tb, M, N, K, A.ptr, lda_, B.ptr, ldb, float(beta), Cm.ptr, ld,
                                             nk.BF16, cdt, Mk.ptr, S.ptr)
    else:
        rc = ops.lib.nk_gemm_relu_bwd(dev.ctx, ta, tb, M, N, K, A.ptr, lda_, B.ptr, ldb, float(beta), Cm.ptr, ld,
                                      nk.BF16, cdt, Mk.ptr)
    nk._lib.check(rc, dev.ctx)
    kern = dev.last_gemm_kernel
    got = Cm.read()
    assert np.array_equal(Mk.read(), mk)
    return got, want, (S.read()[0] if colsum else None), s0, kern


# (name, ldc, C offset, mask offset): the vector mask path needs C, mask and their rows 16-byte aligned
ROW_LAYOUTS = [("aligned", lambda n: ceil8(n) + 8, 0, 0), ("odd_ldc", lambda n: n + 1 if n % 2 == 0 else n + 2, 0, 0),
               ("mask+1", lambda n: ceil8(n) + 8, 0, 1)]


@pytest.mark.parametrize("layout", [r[0] for r in ROW_LAYOUTS])
@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("form", ["NN", "NT", "TN"])
def test_fused_relu_backward(nk, dev, O, form, cdt, layout):
    """nk_gemm_relu_bwd at ragged M / N with a mask of exact zeros and negatives, beta 0 and 1, on the vector and the
    scalar mask paths"""
    c = nk.F32 if cdt == "f32" else nk.BF16
    _, ldf, off_c, off_m = next(r for r in ROW_LAYOUTS if r[0] == layout)
    M, N, K = 333, 290, 88
    for beta in (0.0, 1.0):
        got, want, _, _, kern = run_relu_bwd(nk, dev, O, form, M, N, K, c, beta=beta, ldc=ldf(N), off_c=off_c,
                                             off_mask=off_m, seed=int(beta) + 3)
        assert kern == f"wgmma_{form.lower()}_128x256"
        check(got, want, c == nk.BF16, beta != 0, (form, cdt, layout, beta))


@pytest.mark.parametrize("layout", [r[0] for r in ROW_LAYOUTS])
@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("form,N", [("NN", 290), ("NT", 100), ("TN", 40)])
def test_fused_relu_backward_column_sums(nk, dev, O, form, N, cdt, layout):
    """nk_gemm_relu_bwd_colsum: C against the reference, and the column sums against the float64 sums of the C the device
    stored (rounded to C's type), within 1e-5 of the column's L1 norm (f32 atomics); M % 128 != 0, so the rows past M of
    the last m-block must count as zero"""
    c = nk.F32 if cdt == "f32" else nk.BF16
    _, ldf, off_c, off_m = next(r for r in ROW_LAYOUTS if r[0] == layout)
    M, K = 333, 88
    got, want, cs, s0, kern = run_relu_bwd(nk, dev, O, form, M, N, K, c, ldc=ldf(N), off_c=off_c, off_mask=off_m,
                                           colsum=True, seed=5)
    assert kern.startswith(f"wgmma_{form.lower()}_")
    check(got, want, c == nk.BF16, False, (form, cdt, layout))
    stored = got.astype(np.float64)
    tol = 1e-5 * (np.abs(stored).sum(0) + np.abs(s0)) + 1e-6
    err = np.abs(cs.astype(np.float64) - (s0 + stored.sum(0)))
    assert np.all(err <= tol), (form, cdt, layout, float(err.max()))


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
def test_fused_relu_backward_skinny_nn(nk, dev, O, cdt):
    """the skinny NN shape (K = 10 <= 16, N >= 256, lda = 10 not TMA-addressable) is fused by the CUDA-core kernel"""
    c = nk.F32 if cdt == "f32" else nk.BF16
    M, N, K = 300, 300, 10
    for beta in (0.0, 1.0):
        got, want, _, _, kern = run_relu_bwd(nk, dev, O, "NN", M, N, K, c, beta=beta, ldc=N + 5, lda=K, seed=8)
        assert kern == "simt_small_k"
        check(got, want, c == nk.BF16, beta != 0, (cdt, beta))
    got, want, cs, s0, kern = run_relu_bwd(nk, dev, O, "NN", M, N, K, c, ldc=N + 5, lda=K, colsum=True, seed=9)
    assert kern == "simt_small_k"
    check(got, want, c == nk.BF16, False, cdt)
    stored = got.astype(np.float64)
    err = np.abs(cs.astype(np.float64) - (s0 + stored.sum(0)))
    assert np.all(err <= 1e-5 * (np.abs(stored).sum(0) + np.abs(s0)) + 1e-6), float(err.max())


@pytest.mark.parametrize("form", ["NT", "NN"])
def test_fused_column_sums_contract(nk, dev, O, form):
    """beta != 0 with column sums is an argument error; a product that no engine fuses (N <= 16) returns
    NK_ERR_UNSUPPORTED with C, mask and the column sums untouched"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(21)
    ta, tb = FORMS[form]
    M, N, K = 200, 16, 64
    (a, lda), (b, ldb), _ = operands(O, rng, form, M, N, K)
    A, B = Strided(dev, a, nk.BF16, lda), Strided(dev, b, nk.BF16, ldb)
    c0 = O.bf16_round(rng.uniform(-1, 1, (M, N)).astype(F32))
    mk = O.bf16_round(mask_values(rng, (M, N)))
    s0 = rng.uniform(-1, 1, N).astype(F32)
    Cm, Mk, S = Strided(dev, c0, nk.BF16, N + 8), Strided(dev, mk, nk.BF16, N + 8), Strided(dev, s0, nk.F32)
    with pytest.raises(nk.NkError, match="beta must be 0"):
        nk._lib.check(ops.lib.nk_gemm_relu_bwd_colsum(dev.ctx, ta, tb, M, N, K, A.ptr, lda, B.ptr, ldb, 1.0, Cm.ptr,
                                                      N + 8, nk.BF16, nk.BF16, Mk.ptr, S.ptr), dev.ctx)
    rc = ops.lib.nk_gemm_relu_bwd_colsum(dev.ctx, ta, tb, M, N, K, A.ptr, lda, B.ptr, ldb, 0.0, Cm.ptr, N + 8, nk.BF16,
                                         nk.BF16, Mk.ptr, S.ptr)
    assert rc == -5
    dev.synchronize()
    assert np.array_equal(Cm.read(), c0)
    assert np.array_equal(Mk.read(), mk)
    assert np.array_equal(S.read()[0], s0)
