"""The wgmma GEMM engine's TMA-store epilogue (beta == 0; alpha, column bias, ReLU; a C that TMA can address) and its
main loop with one wgmma group in flight, through the C ABI with explicit leading dimensions.

C is a view into a larger buffer filled with a canary value: the view is checked against a float64 reference on the same
bf16-rounded operands, relu(alpha.op(A)op(B) + bias), and every element outside it -- the ldc - N gap of each row and
the guard after the last row included -- must still hold the canary, bit for bit (the store boxes are clipped at M and
N).  The same product written by the TMA store and by the shared-memory drain (forced with beta = 1 on a zeroed C) must
agree bit for bit: both round alpha.acc before adding the bias, so nothing but the accumulation order could differ, and
that is the same.  Tolerances: f32 output 2e-3.rms(want) + 1e-6; bf16 output + 2^-8.|want|."""
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
    """A rows x cols matrix at element `off` of a buffer, rows `ld` elements apart; everything else holds CANARY"""

    def __init__(self, dev, data, dtype, ld=None, off=0, tail=64):
        data = np.asarray(data, F32)
        if data.ndim == 1:
            data = data[None, :]
        self.rows, self.cols = data.shape
        self.ld = self.cols if ld is None else ld
        self.off = off
        self.size = off + self.rows * self.ld + tail
        host = np.full(self.size, CANARY, F32)
        self._inner(host)[:] = data
        self.buf = dev.from_ndarray(host, dtype)
        self.ptr = self.buf.slice_flat(off, (self.rows * self.ld,)).ptr

    def _inner(self, flat):
        return flat[self.off:self.off + self.rows * self.ld].reshape(self.rows, self.ld)[:, :self.cols]

    def read(self):
        flat = self.buf.as_ndarray()
        outside = np.ones(self.size, bool)
        self._inner(outside)[:] = False
        bad = np.flatnonzero(flat[outside] != CANARY)
        assert bad.size == 0, f"{bad.size} elements outside the view were written (first at outside index {bad[0]})"
        return self._inner(flat).copy()


def check(got, want, c_bf16, what):
    want = np.asarray(want, np.float64)
    tol = 2e-3 * rms(want) + (2.0 ** -8 if c_bf16 else 0.0) * np.abs(want) + 1e-6
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(err <= tol), (what, float(err.max()), int(np.argmax(err > tol)), rms(want))


def run(nk, dev, O, form, M, N, K, cdt, *, alpha=1.0, bias=None, relu=False, ldc=None, drain=False, seed=0):
    """nk_gemm_bias_act into a canary-guarded C view: beta = 0 (the TMA store), or with drain=True beta = 1 on a zeroed C
    (the shared-memory drain, same values).  bias in {None, "f32", "bf16"} with an optional "+1" suffix (one element off
    16-byte alignment).  Returns (C view, float64 reference, kernel name)."""
    from neuronika_b200 import ops
    rng = np.random.default_rng(seed)
    ta, tb = FORMS[form]
    a = O.bf16_round(rng.uniform(-1, 1, (K, M) if ta else (M, K)).astype(F32))
    b = O.bf16_round(rng.uniform(-1, 1, (N, K) if tb else (K, N)).astype(F32))
    lda, ldb = ceil8(a.shape[1]), ceil8(b.shape[1])
    A, B = Strided(dev, a, nk.BF16, lda), Strided(dev, b, nk.BF16, ldb)
    want = alpha * ((a.T if ta else a).astype(np.float64) @ (b.T if tb else b).astype(np.float64))
    c0 = np.zeros((M, N), F32) if drain else np.full((M, N), CANARY, F32)
    Cm = Strided(dev, c0, cdt, ceil8(N) + 8 if ldc is None else ldc)
    bptr, bdt = None, nk.F32
    if bias is not None:
        bdt = nk.BF16 if bias.startswith("bf16") else nk.F32
        bv = rng.uniform(-1, 1, N).astype(F32)
        if bdt == nk.BF16:
            bv = O.bf16_round(bv)
        Bias = Strided(dev, bv, bdt, off=1 if bias.endswith("+1") else 0)
        bptr = Bias.ptr
        want = want + bv[None, :]
    if relu:
        want = np.maximum(want, 0.0)
    rc = ops.lib.nk_gemm_bias_act(dev.ctx, ta, tb, M, N, K, float(alpha), A.ptr, lda, B.ptr, ldb, 1.0 if drain else 0.0,
                                  Cm.ptr, Cm.ld, nk.BF16, cdt, bptr, bdt, int(relu))
    nk._lib.check(rc, dev.ctx)
    return Cm.read(), want, dev.last_gemm_kernel


def cdtype(nk, name):
    return nk.F32 if name == "f32" else nk.BF16


# (M, N): M = 1, 63, 65 mod 128 (the 64-row boxes of each warpgroup); N = 8, 24, 40, 56, 72 mod 256 around the 32 / 64-
# column chunks of f32 / bf16 output -- rows that end on a 16-byte boundary, stored by TMA -- and N = 1, 31, 33, 63, 65
# mod 256, whose rows do not (a store box would clip them only to the 16-byte unit), so those go through the drain
RAGGED = [(129, 264), (191, 280), (193, 296), (129, 312), (191, 328), (65, 264),
          (129, 257), (191, 287), (193, 289), (129, 319), (191, 321)]


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("form", list(FORMS))
def test_every_form_ragged_at_box_and_chunk_edges(nk, dev, O, form, cdt):
    """ragged M and N at the store boxes' edges, ldc 8 .. 15 elements above N: nothing past row M or column N is written"""
    c = cdtype(nk, cdt)
    for i, (M, N) in enumerate(RAGGED):
        got, want, kern = run(nk, dev, O, form, M, N, 136, c, seed=i)
        assert kern == f"wgmma_{form.lower()}_128x256"
        check(got, want, c == nk.BF16, (form, cdt, M, N))


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
def test_bias_relu_alpha(nk, dev, O, cdt):
    """column bias f32 / bf16, aligned and one element off, x ReLU x alpha != 1"""
    c = cdtype(nk, cdt)
    i = 0
    for alpha in (1.0, -0.75):
        for bias in (None, "f32", "f32+1", "bf16", "bf16+1"):
            for relu in (False, True):
                i += 1
                got, want, kern = run(nk, dev, O, "NT", 200, 296, 72, c, alpha=alpha, bias=bias, relu=relu, ldc=304,
                                      seed=100 + i)
                assert kern == "wgmma_nt_128x256"
                check(got, want, c == nk.BF16, (cdt, alpha, bias, relu))


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
def test_persistent_schedule_reuses_staging_buffers(nk, dev, O, cdt):
    """at least three 128 x 256 tiles per CTA, so the staging buffers and their pending stores carry over from tile to
    tile; ragged M and N, the whole output checked"""
    c = cdtype(nk, cdt)
    sm = dev.sm_count
    m_blocks = 16
    n_blocks = -(-3 * sm // m_blocks) + 1
    tiles = m_blocks * n_blocks
    waves = -(-tiles // sm)
    assert waves >= 3 and tiles // -(-tiles // waves) >= 3
    M, N = m_blocks * 128 - 37, n_blocks * 256 - 104
    got, want, kern = run(nk, dev, O, "NT", M, N, 200, c, bias="bf16", relu=True, seed=7)
    assert kern == "wgmma_nt_128x256"
    check(got, want, c == nk.BF16, cdt)


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("form", list(FORMS))
def test_same_bits_as_the_drain(nk, dev, O, form, cdt):
    """the TMA store and the shared-memory drain (beta = 1 on a zeroed C) store the same values (-0 and +0 equal)"""
    c = cdtype(nk, cdt)
    for alpha, bias, relu in ((1.0, None, False), (-0.75, "f32", True), (1.5, "bf16+1", False)):
        tma, want, _ = run(nk, dev, O, form, 333, 296, 200, c, alpha=alpha, bias=bias, relu=relu, seed=11)
        drn, _, _ = run(nk, dev, O, form, 333, 296, 200, c, alpha=alpha, bias=bias, relu=relu, drain=True, seed=11)
        check(tma, want, c == nk.BF16, (form, cdt, alpha, bias, relu))
        neq = np.flatnonzero(tma != drn)
        assert neq.size == 0, (form, cdt, alpha, bias, relu, neq.size, tma.flat[neq[0]], drn.flat[neq[0]])


@pytest.mark.parametrize("form", list(FORMS))
def test_k_block_edges(nk, dev, O, form):
    """one k-block (K <= 64: the slot is released after the tile's last wait), and K not a multiple of 64"""
    for i, K in enumerate((8, 64, 65, 100, 1000)):
        for cdt in ("f32", "bf16"):
            c = cdtype(nk, cdt)
            got, want, kern = run(nk, dev, O, form, 300, 272, K, c, bias="f32", seed=200 + i)
            assert kern == f"wgmma_{form.lower()}_128x256"
            check(got, want, c == nk.BF16, (form, K, cdt))
