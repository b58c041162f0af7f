"""The CUDA-core GEMM engine (nk_gemm_simt.cu) at its split, dispatch and tail boundaries, through the C ABI with explicit
leading dimensions:

- simt_64x64x16: every form at M, N around the 64-wide tile, K around the 16-wide step and the 512 split-K threshold,
  K = 8200 on one tile (a split-K with a ragged last split), the epilogue matrix on the direct store and on the split-K
  reduce, every (operand, output) dtype pair, K = 0, and the grid limit on M;
- simt_small_k (NN, K <= 16, N >= 256): every KP bucket edge, N = 255 / 256, ragged rows and columns, and the scalar
  paths of B, C and the ReLU mask (row pitch not a multiple of 4, base off 16 bytes), with the mask and column sums;
- simt_small_m (TN, M <= 16, N >= 256, K >= 256): every MP bucket edge, K = 255 / 256, ragged k slabs, blocks that hold
  more than one 512-row slab, a misaligned B, and the epilogue in the finalize;
- the f32 ReLU backward, which stores the product into a temporary and then applies the mask.

Operands and C are views into larger buffers filled with a canary value: every element outside C's view, the ldc - N
gap of each row included, must still hold the canary bit for bit.  The reference is float64 on the operands as stored,
in the epilogue order of store_out, relu(alpha.AB + beta.C0 + bias).  The bound is elementwise:
|got - want| <= (K + splits + 4).2^-24.(|alpha|.(|A||B|) + |beta.C0| + |bias|), plus 2^-8.|want| for a bf16 C (2^-7 when
beta != 0).  One dropped or repeated 16-wide k step breaks it even at K = 8200."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24
CANARY = -1152.0          # exact in bf16 and f32, far outside every value below
FORMS = {"NN": (0, 0), "NT": (0, 1), "TN": (1, 0), "TT": (1, 1)}
NK_ERR_UNSUPPORTED = -5


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


class Strided:
    """A rows x cols matrix at element `off` of a buffer, rows `ld` elements apart; every other element of the buffer
    (row gaps, the elements before `off`, a tail guard) holds CANARY."""

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
        self.ptr = self.buf.slice_flat(off, (self.rows * self.ld,)).ptr

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


def simt_splits(sm, M, N, K):
    """the split-K choice of nk_gemm_simt.cu's launch(): (splits, k per split)"""
    tiles = -(-M // 64) * -(-N // 64)
    splits = 1
    if tiles < sm and K >= 512:
        s = min(-(-2 * sm // tiles), K // 128, 64)
        if s > 1:
            splits = s
    kps = -(-K // splits)
    kps = max(16, -(-kps // 16) * 16)
    return max(1, -(-K // kps)), kps


def small_m_blocks(sm, N, K):
    """the k partition of launch_skinny()'s small-M kernel: (k per block, blocks along k)"""
    gx = -(-N // 128)
    gy = -(-(4 * sm) // gx)
    kpb = -(-K // gy)
    kpb = -(-kpb // 512) * 512
    return kpb, -(-K // kpb)


def rounded(O, v, bf16):
    v = np.asarray(v, F32)
    return O.bf16_round(v) if bf16 else v


def check(got, want, mag, terms, c_bf16, accumulated, what):
    """|got - want| <= terms.2^-24.mag (+ 2^-8 / 2^-7 of |want| for a bf16 output)"""
    want = np.asarray(want, np.float64)
    rel = (2.0 ** -7 if accumulated else 2.0 ** -8) if c_bf16 else 0.0
    tol = terms * U * mag + rel * np.abs(want)
    err = np.abs(np.asarray(got, np.float64) - want)
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), np.unravel_index(int(np.argmax(err - tol)), err.shape),
                           float(err.max()), float(tol.ravel()[np.argmax(err - tol)]))


def run_gemm(nk, dev, O, form, M, N, K, ab="f32", c="f32", *, alpha=1.0, beta=0.0, bias=None, relu=False, lda=None,
             ldb=None, ldc=None, off_a=0, off_b=0, off_c=0, seed=0, inputs=None):
    """nk_gemm_bias_act on canary-guarded views; ab / c / bias in {"f32", "bf16"} (bias None: no bias).  bf16 operands
    run with the CUDA-core engine forced.  Returns (C view, reference, magnitude, kernel, launches); C0 and the bias go
    into the dict `inputs` when one is given."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ta, tb = FORMS[form]
    ab_bf, c_bf = ab == "bf16", c == "bf16"
    a = rounded(O, rng.uniform(-1, 1, (K, M) if ta else (M, K)), ab_bf)
    b = rounded(O, rng.uniform(-1, 1, (N, K) if tb else (K, N)), ab_bf)
    A = Strided(dev, a, nk.BF16 if ab_bf else nk.F32, lda or max(1, a.shape[1]), off_a)
    B = Strided(dev, b, nk.BF16 if ab_bf else nk.F32, ldb or max(1, b.shape[1]), off_b)
    c0 = rounded(O, rng.uniform(-1, 1, (M, N)), c_bf)
    C = Strided(dev, c0, nk.BF16 if c_bf else nk.F32, ldc or N, off_c)
    opa = (a.T if ta else a).astype(np.float64)
    opb = (b.T if tb else b).astype(np.float64)
    want = alpha * (opa @ opb) + beta * c0.astype(np.float64)
    mag = abs(alpha) * (np.abs(opa) @ np.abs(opb)) + np.abs(beta * c0.astype(np.float64))
    bptr, bdt = None, nk.F32
    if bias is not None:
        bdt = nk.BF16 if bias == "bf16" else nk.F32
        bv = rounded(O, rng.uniform(-1, 1, N), bias == "bf16")
        Bias = Strided(dev, bv, bdt)
        bptr = Bias.ptr
        want = want + bv[None, :]
        mag = mag + np.abs(bv)[None, :]
        if inputs is not None:
            inputs["bias"] = bv
    if inputs is not None:
        inputs["c0"] = c0
    if relu:
        want = np.maximum(want, 0.0)
    if ab_bf:
        dev.gemm_engine("simt")
    try:
        before = dev.launches
        rc = ops.lib.nk_gemm_bias_act(dev.ctx, ta, tb, M, N, K, float(alpha), A.ptr if K else None, A.ld,
                                      B.ptr if K else None, B.ld, float(beta), C.ptr, C.ld,
                                      nk.BF16 if ab_bf else nk.F32, nk.BF16 if c_bf else nk.F32, bptr, bdt, int(relu))
        nk._lib.check(rc, dev.ctx)
        launches = dev.launches - before
    finally:
        if ab_bf:
            dev.gemm_engine("auto")
    return C.read(), want, mag, dev.last_gemm_kernel, launches


# ------------------------------------------------------------------------------------------- simt_64x64x16
EDGE_MN = (1, 63, 64, 65, 130)


@pytest.mark.parametrize("K", [1, 15, 16, 17, 511, 512, 8200])
@pytest.mark.parametrize("form", list(FORMS))
def test_tile_form_and_step_edges(nk, dev, O, form, K):
    """M, N on both sides of the 64-wide tile, K on both sides of the 16-wide step and of the split-K threshold (512);
    at K = 8200 a single tile takes 57 splits of 144 with a ragged last split on a 132-SM H100.  ldc = N + 3 and an A
    base one element off its alignment; beta = 1 reads the old C."""
    for M in EDGE_MN:
        for N in EDGE_MN:
            splits, _ = simt_splits(dev.sm_count, M, N, K)
            got, want, mag, kern, launches = run_gemm(nk, dev, O, form, M, N, K, beta=1.0, ldc=N + 3, off_a=1,
                                                      seed=M * 1000 + N)
            assert kern == "simt_64x64x16", (form, M, N, K, kern)
            assert launches == (2 if splits > 1 else 1), (form, M, N, K, splits, launches)
            check(got, want, mag, K + splits + 4, False, True, (form, M, N, K))


def test_split_k_shapes_are_the_intended_ones(dev):
    """the cases below split where they are meant to: K = 511 never, K = 8200 on one tile with a ragged last split"""
    sm = dev.sm_count
    assert simt_splits(sm, 64, 64, 511)[0] == 1
    s, kps = simt_splits(sm, 64, 64, 8200)
    assert s > 1 and 8200 % kps != 0 and (s - 1) * kps < 8200
    if sm == 132:
        assert (s, kps) == (57, 144)
    s, kps = simt_splits(sm, 70, 90, 1000)
    assert s > 1 and 1000 % kps != 0


# (path) -> (M, N, K): the direct store (no split) and the split-K reduce (7 splits of 144, the last 136 long, on 132 SMs)
EPI_SHAPES = {"direct": (130, 70, 300), "splitk": (70, 90, 1000)}


@pytest.mark.parametrize("c", ["f32", "bf16"])
@pytest.mark.parametrize("path", list(EPI_SHAPES))
def test_epilogue_matrix(nk, dev, O, path, c):
    """alpha x beta in {0, 0.5, 1} x bias (none, f32, bf16) x ReLU on the direct store and on the split-K reduce"""
    M, N, K = EPI_SHAPES[path]
    splits, _ = simt_splits(dev.sm_count, M, N, K)
    assert (splits > 1) == (path == "splitk")
    i = 0
    for alpha in (0.0, 0.5, 1.0):
        for beta in (0.0, 0.5, 1.0):
            for bias in (None, "f32", "bf16"):
                for relu in (False, True):
                    i += 1
                    got, want, mag, kern, launches = run_gemm(nk, dev, O, "NT", M, N, K, "f32", c, alpha=alpha,
                                                              beta=beta, bias=bias, relu=relu, ldc=N + 3, off_a=1,
                                                              seed=i)
                    assert kern == "simt_64x64x16" and launches == (2 if splits > 1 else 1)
                    check(got, want, mag, K + splits + 4, c == "bf16", beta != 0, (path, c, alpha, beta, bias, relu))


@pytest.mark.parametrize("ab,c", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
@pytest.mark.parametrize("form", ["NN", "TT"])
def test_operand_and_output_dtype_pairs(nk, dev, O, form, ab, c):
    """every (operands, C) dtype pair, f32 operands into a bf16 C included, on the direct store and the split-K reduce"""
    for M, N, K in EPI_SHAPES.values():
        splits, _ = simt_splits(dev.sm_count, M, N, K)
        got, want, mag, kern, launches = run_gemm(nk, dev, O, form, M, N, K, ab, c, alpha=0.5, beta=0.5, bias="bf16",
                                                  relu=True, ldc=N + 3, off_a=1, seed=K)
        assert kern == "simt_64x64x16" and launches == (2 if splits > 1 else 1)
        check(got, want, mag, K + splits + 4, c == "bf16", True, (form, ab, c, M, N, K))


@pytest.mark.parametrize("c", ["f32", "bf16"])
def test_split_k_is_deterministic(nk, dev, O, c):
    """the split-K reduce sums the splits in a fixed order: two calls on the same data agree bit for bit"""
    runs = [run_gemm(nk, dev, O, "TN", 50, 40, 8200, "f32", c, beta=0.5, bias="f32", ldc=43, seed=3) for _ in range(2)]
    assert runs[0][4] == 2
    assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32))


@pytest.mark.parametrize("ab,c", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
def test_zero_k_is_the_epilogue_alone(nk, dev, O, ab, c):
    """K = 0 (A and B NULL): C = beta.C0 + bias exactly, in f32 arithmetic, for beta 0, 0.5 and 1, with and without
    ReLU"""
    for beta in (0.0, 0.5, 1.0):
        for relu in (False, True):
            M, N = 70, 90
            inputs = {}
            got, _, _, kern, launches = run_gemm(nk, dev, O, "NN", M, N, 0, ab, c, beta=beta, bias="f32", relu=relu,
                                                 ldc=N + 3, seed=int(beta * 2) + 3 * relu, inputs=inputs)
            c0, bv = inputs["c0"], inputs["bias"]
            v = (F32(beta) * c0 if beta else np.zeros_like(c0)) + bv[None, :]
            if relu:
                v = np.maximum(v, F32(0))
            assert kern == "simt_64x64x16" and launches == 1
            assert np.array_equal(got, rounded(O, v, c == "bf16")), (ab, c, beta, relu)


# ------------------------------------------------------------------------------------------- simt_small_k
@pytest.mark.parametrize("N", [255, 256, 1027])
@pytest.mark.parametrize("K", [1, 4, 5, 8, 9, 12, 13, 16, 17])
def test_small_k_bucket_edges(nk, dev, O, K, N):
    """K at every KP bucket edge (4 | 5, 8 | 9, 12 | 13, 16 | 17) and N = 255 / 256: K = 17 or N = 255 is not small-K.
    M = 77 is neither a multiple of the 64-row block nor of the 8-row flight; N = 1027 ends in a partial 4-column group
    and a partial 1024-column block."""
    M = 77
    small = K <= 16 and N >= 256
    for ab, c in (("f32", "f32"), ("bf16", "bf16")):
        got, want, mag, kern, _ = run_gemm(nk, dev, O, "NN", M, N, K, ab, c, alpha=0.5, beta=1.0, bias="f32",
                                           relu=True, ldb=N + (-N % 4) + 4, ldc=N + (-N % 4) + 8, seed=K * 10 + N)
        assert kern == ("simt_small_k" if small else "simt_64x64x16"), (K, N, ab, kern)
        check(got, want, mag, K + 5, c == "bf16", True, (K, N, ab, c))


# (name) -> (ldb, ldc, B offset, C offset) for N = 300; the vector paths need ldb / ldc % 4 == 0 and 16-byte bases
SMALL_K_LAYOUTS = {
    "vector": (304, 308, 0, 0),
    "ldb%4": (301, 308, 0, 0),
    "ldc%4": (304, 303, 0, 0),
    "b+1": (304, 308, 1, 0),
    "c+1": (304, 308, 0, 1),
}


@pytest.mark.parametrize("ab,c", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
@pytest.mark.parametrize("layout", list(SMALL_K_LAYOUTS))
def test_small_k_scalar_paths(nk, dev, O, layout, ab, c):
    """B and C rows that the 8 / 16-byte accesses cannot take, for every dtype pair, with beta 0 and 1"""
    ldb, ldc, ob, oc = SMALL_K_LAYOUTS[layout]
    for beta in (0.0, 1.0):
        got, want, mag, kern, _ = run_gemm(nk, dev, O, "NN", 77, 300, 10, ab, c, beta=beta, bias="bf16", ldb=ldb,
                                           ldc=ldc, off_b=ob, off_c=oc, seed=int(beta) + len(layout))
        assert kern == "simt_small_k"
        check(got, want, mag, 10 + 5, c == "bf16", beta != 0, (layout, ab, c, beta))


def mask_values(rng, shape):
    """exact zeros, negatives and positives in equal parts"""
    return rng.choice(np.array([-1.0, 0.0, 1.0], F32), shape) * rng.uniform(0.25, 1.0, shape).astype(F32)


def run_relu_bwd(nk, dev, O, form, M, N, K, *, beta=0.0, ldc=None, off_c=0, off_mask=0, colsum=False, seed=0):
    """nk_gemm_relu_bwd(_colsum) with f32 operands and C: C = beta.C0 + (mask > 0).op(A)op(B), the mask (M, N) with C's
    leading dimension; colsum (N floats, starting from random values) += column sums of the stored C.  Returns (rc, C
    view, reference, magnitude, colsum, colsum start, C0, kernel)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ta, tb = FORMS[form]
    a = rng.uniform(-1, 1, (K, M) if ta else (M, K)).astype(F32)
    b = rng.uniform(-1, 1, (N, K) if tb else (K, N)).astype(F32)
    A, B = Strided(dev, a, nk.F32), Strided(dev, b, nk.F32)
    c0 = rng.uniform(-1, 1, (M, N)).astype(F32)
    mk = mask_values(rng, (M, N))
    ld = N if ldc is None else ldc
    C, Mk = Strided(dev, c0, nk.F32, ld, off_c), Strided(dev, mk, nk.F32, ld, off_mask)
    opa = (a.T if ta else a).astype(np.float64)
    opb = (b.T if tb else b).astype(np.float64)
    keep = mk > 0
    want = beta * c0 + np.where(keep, opa @ opb, 0.0)
    mag = np.where(keep, np.abs(opa) @ np.abs(opb), 0.0) + np.abs(beta * c0)
    s0 = rng.uniform(-1, 1, N).astype(F32)
    S = Strided(dev, s0, nk.F32) if colsum else None
    args = (dev.ctx, ta, tb, M, N, K, A.ptr, A.ld, B.ptr, B.ld, float(beta), C.ptr, ld, nk.F32, nk.F32, Mk.ptr)
    rc = ops.lib.nk_gemm_relu_bwd_colsum(*args, S.ptr) if colsum else ops.lib.nk_gemm_relu_bwd(*args)
    got = C.read()
    assert np.array_equal(Mk.read(), mk)
    return rc, got, want, mag, (S.read()[0] if colsum else None), s0, c0, dev.last_gemm_kernel


# (name) -> (ldc, C offset, mask offset) for N = 300
MASK_LAYOUTS = {"vector": (308, 0, 0), "mask+1": (308, 0, 1), "ldc%4": (303, 0, 0), "c+1": (308, 1, 0)}


@pytest.mark.parametrize("layout", list(MASK_LAYOUTS))
def test_small_k_mask_and_column_sums(nk, dev, O, layout):
    """the fused ReLU backward of the small-K kernel with f32 operands: the mask on its vector and scalar paths with beta
    0 and 1, and the column sums against the float64 sums of the stored C (f32 atomics: 1e-5 of the column's L1 norm)"""
    ldc, oc, om = MASK_LAYOUTS[layout]
    M, N, K = 77, 300, 13
    for beta in (0.0, 1.0):
        rc, got, want, mag, _, _, _, kern = run_relu_bwd(nk, dev, O, "NN", M, N, K, beta=beta, ldc=ldc, off_c=oc,
                                                         off_mask=om, seed=int(beta))
        nk._lib.check(rc, dev.ctx)
        assert kern == "simt_small_k"
        check(got, want, mag, K + 5, False, beta != 0, (layout, beta))
    rc, got, want, mag, cs, s0, _, kern = run_relu_bwd(nk, dev, O, "NN", M, N, K, ldc=ldc, off_c=oc, off_mask=om,
                                                       colsum=True, seed=5)
    nk._lib.check(rc, dev.ctx)
    assert kern == "simt_small_k"
    check(got, want, mag, K + 5, False, False, layout)
    stored = got.astype(np.float64)
    err = np.abs(cs.astype(np.float64) - (s0 + stored.sum(0)))
    assert np.all(err <= 1e-5 * (np.abs(stored).sum(0) + np.abs(s0)) + 1e-6), (layout, float(err.max()))


# ------------------------------------------------------------------------------------------- simt_small_m
@pytest.mark.parametrize("K", [255, 256, 1537, 70000])
def test_small_m_bucket_edges(nk, dev, O, K):
    """M at every MP bucket edge (4 | 5, 8 | 9, 12 | 13, 16 | 17) and K = 255 / 256: M = 17 or K = 255 is not small-M.
    N = 301 ends in a partial 128-column block and a partial 4-column group; K = 1537 and 70000 end in a ragged k slab.
    beta, bias and ReLU run through the finalize."""
    N = 301
    for M in (1, 4, 5, 8, 9, 12, 13, 16, 17):
        small = M <= 16 and K >= 256
        splits = 1 if small else simt_splits(dev.sm_count, M, N, K)[0]
        got, want, mag, kern, _ = run_gemm(nk, dev, O, "TN", M, N, K, beta=0.5, bias="f32", relu=True, ldb=N + 3,
                                           ldc=N + 3, seed=M * 7 + K)
        assert kern == ("simt_small_m" if small else "simt_64x64x16"), (M, K, kern)
        check(got, want, mag, K + splits + 4, False, True, (M, K))


# (name) -> (ldb, B offset) for N = 301
SMALL_M_LAYOUTS = {"ldb%4": (301, 0), "b+1": (304, 1), "vector": (304, 0)}


@pytest.mark.parametrize("ab,c", [("f32", "f32"), ("f32", "bf16"), ("bf16", "f32"), ("bf16", "bf16")])
@pytest.mark.parametrize("layout", list(SMALL_M_LAYOUTS))
def test_small_m_layouts_and_dtypes(nk, dev, O, layout, ab, c):
    """B rows that the vector loads cannot take (pitch not a multiple of 4, base off 16 bytes), every dtype pair"""
    ldb, ob = SMALL_M_LAYOUTS[layout]
    M, N, K = 13, 301, 1537
    got, want, mag, kern, _ = run_gemm(nk, dev, O, "TN", M, N, K, ab, c, alpha=0.5, beta=1.0, bias="bf16", ldb=ldb,
                                       ldc=N + 3, off_b=ob, seed=len(layout))
    assert kern == "simt_small_m"
    check(got, want, mag, K + 5, c == "bf16", True, (layout, ab, c))


def test_small_m_blocks_of_several_slabs(nk, dev, O):
    """N wide enough that the k range falls into so few blocks that one block runs two 512-row slabs of A through shared
    memory, and the last block ends in a ragged slab"""
    sm = dev.sm_count
    gx = -(-(4 * sm) // 3)
    N, K = gx * 128 - 3, 1537
    kpb, gy = small_m_blocks(sm, N, K)
    assert kpb > 512 and (K - (gy - 1) * kpb) % 512 != 0, (kpb, gy)
    got, want, mag, kern, _ = run_gemm(nk, dev, O, "TN", 16, N, K, beta=1.0, bias="f32", relu=True, ldb=N + 3,
                                       ldc=N + 3, seed=4)
    assert kern == "simt_small_m"
    check(got, want, mag, K + 5, False, True, (N, K, kpb, gy))


# ------------------------------------------------------------------------------------------- contracts
def test_m_beyond_the_grid_is_a_clean_error(nk, dev, O):
    """M = 65535.64 + 1 needs 65536 row tiles: "M too large", C untouched, and the context still works"""
    from neuronika_b200 import ops
    M = 65535 * 64 + 1
    rng = np.random.default_rng(1)
    a = rng.uniform(-1, 1, (M, 1)).astype(F32)
    c0 = rng.uniform(-1, 1, (M, 1)).astype(F32)
    A, B, C = Strided(dev, a, nk.F32), Strided(dev, np.ones((1, 1), F32), nk.F32), Strided(dev, c0, nk.F32)
    with pytest.raises(nk.NkError, match="M too large"):
        nk._lib.check(ops.lib.nk_gemm_bias_act(dev.ctx, 0, 0, M, 1, 1, 1.0, A.ptr, 1, B.ptr, 1, 1.0, C.ptr, 1, nk.F32,
                                               nk.F32, None, nk.F32, 0), dev.ctx)
    dev.synchronize()
    assert np.array_equal(C.read(), c0)
    got, want, mag, kern, _ = run_gemm(nk, dev, O, "NN", 65, 63, 17, beta=1.0, ldc=66, seed=2)
    assert kern == "simt_64x64x16"
    check(got, want, mag, 17 + 5, False, True, "after the error")


@pytest.mark.parametrize("form,K", [("NN", 40), ("NT", 40), ("TN", 40), ("TT", 40), ("NT", 10)])
def test_f32_relu_backward_fallback(nk, dev, O, form, K):
    """f32 operands outside the small-K kernel: the product goes into a temporary and nk_relu_bwd masks it into C; with
    ldc == N it is right for beta 0 and 1, with ldc != N it is NK_ERR_UNSUPPORTED ("strided output") and C is untouched"""
    M, N = 150, 70
    for beta in (0.0, 1.0):
        rc, got, want, mag, _, _, _, kern = run_relu_bwd(nk, dev, O, form, M, N, K, beta=beta, seed=int(beta) + K)
        nk._lib.check(rc, dev.ctx)
        assert kern == "simt_64x64x16"
        check(got, want, mag, K + 5, False, beta != 0, (form, K, beta))
    rc, got, _, _, _, _, c0, _ = run_relu_bwd(nk, dev, O, form, M, N, K, beta=1.0, ldc=N + 3, seed=9)
    assert rc == NK_ERR_UNSUPPORTED
    with pytest.raises(nk.NkError, match="strided output"):
        nk._lib.check(rc, dev.ctx)
    assert np.array_equal(got, c0)


@pytest.mark.parametrize("form", ["NN", "NT", "TN"])
def test_f32_column_sums_are_unsupported(nk, dev, O, form):
    """the column-sum variant of an f32 product that the small-K kernel does not take returns NK_ERR_UNSUPPORTED with
    C, the mask and the column sums untouched (the caller then sums the columns itself)"""
    rc, got, _, _, cs, s0, c0, _ = run_relu_bwd(nk, dev, O, form, 150, 70, 40, colsum=True, seed=11)
    assert rc == NK_ERR_UNSUPPORTED
    assert np.array_equal(got, c0)
    assert np.array_equal(cs, s0)
