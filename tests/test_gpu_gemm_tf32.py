"""f32 GEMMs on the tensor cores (nk_gemm_f32_config, csrc/nk_gemm_tf32.cu) through the C ABI with explicit leading
dimensions: every form x mode x tile width, M / N around the 128 / 256 tile edges, K around the 32-wide k-block and
K = 1, leading dimensions and K that are not multiples of 4 and bases TMA cannot address (the pack kernel takes all of
them), and the epilogue (alpha, beta, f32 / bf16 bias, ReLU, f32 / bf16 C).

Operands and C are views into larger buffers filled with a canary; every element outside a view must still hold it.
Bounds (tests/tf32_oracle.py models the operand rounding exactly, so only accumulation is left):
  tf32   vs float64 on the TF32-rounded operands:   |alpha| K 2^-22 (|A^|.|B^|)
  tf32x3 vs float64 on the unrounded operands:      |alpha| (3K + 4) 2^-22 (|A|.|B|)  (the dropped lo.lo term and lo's
         own rounding are <= 3 2^-22 of each product; 3K terms are accumulated)
plus the epilogue's f32 rounding, 2^-22 (|alpha| |A|.|B| + |bias| + |beta C0|), and 2^-8 |want| for a bf16 C."""
import numpy as np
import pytest

import tf32_oracle as T

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0
FORMS = {"NN": (0, 0), "NT": (0, 1), "TN": (1, 0), "TT": (1, 1)}
MODES = ["tf32", "tf32x3"]


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


@pytest.fixture(autouse=True)
def ieee_after(dev):
    yield
    dev.f32_matmul("ieee")
    dev.gemm_engine("auto")


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


class Case:
    """One nk_gemm_bias_act call with f32 operands op(A) (M x K), op(B) (K x N) on canary-guarded views."""

    def __init__(self, nk, dev, form, M, N, K, cdt="f32", *, alpha=1.0, beta=0.0, bias=None, relu=False, ldc=None,
                 off_c=0, pad_a=0, pad_b=0, off_a=0, off_b=0, seed=0, a=None, b=None):
        from neuronika_b200 import ops
        self.nk, self.dev, self.ops = nk, dev, ops
        rng = np.random.default_rng(seed)
        self.ta, self.tb = FORMS[form]
        self.a = rng.uniform(-1, 1, (M, K)).astype(F32) if a is None else a
        self.b = rng.uniform(-1, 1, (K, N)).astype(F32) if b is None else b
        sa = self.a.T if self.ta else self.a
        sb = self.b.T if self.tb else self.b
        self.A = Strided(dev, sa, nk.F32, sa.shape[1] + pad_a, off_a)
        self.B = Strided(dev, sb, nk.F32, sb.shape[1] + pad_b, off_b)
        self.c_bf16 = cdt == "bf16"
        self.cdt = nk.BF16 if self.c_bf16 else nk.F32
        c0 = rng.uniform(-1, 1, (M, N)).astype(F32)
        self.c0 = bf16(c0) if self.c_bf16 else c0
        self.ldc = N if ldc is None else ldc
        self.off_c = off_c
        self.M, self.N, self.K, self.alpha, self.beta, self.relu = M, N, K, alpha, beta, relu
        self.bias, self.bptr, self.bdt = None, None, nk.F32
        if bias is not None:
            self.bdt = nk.BF16 if bias.startswith("bf16") else nk.F32
            bv = rng.uniform(-1, 1, N).astype(F32)
            self.bias = bf16(bv) if self.bdt == nk.BF16 else bv
            self.Bias = Strided(dev, self.bias, self.bdt, off=1 if bias.endswith("+1") else 0)
            self.bptr = self.Bias.ptr

    def run(self):
        """(C view after the call, kernel name); C starts from C0 on every call"""
        self.C = Strided(self.dev, self.c0, self.cdt, self.ldc, self.off_c)
        rc = self.ops.lib.nk_gemm_bias_act(self.dev.ctx, self.ta, self.tb, self.M, self.N, self.K, float(self.alpha),
                                           self.A.ptr, self.A.ld, self.B.ptr, self.B.ld, float(self.beta), self.C.ptr,
                                           self.C.ld, self.nk.F32, self.cdt, self.bptr, self.bdt, int(self.relu))
        self.nk._lib.check(rc, self.dev.ctx)
        return self.C.read(), self.dev.last_gemm_kernel

    def want_and_tol(self, mode):
        if mode == "tf32":
            prod, absprod = T.matmul_tf32(self.a, self.b), np.abs(T.tf32_round(self.a)).astype(np.float64) @ np.abs(
                T.tf32_round(self.b)).astype(np.float64)
            acc = self.K * 2.0 ** -22
        else:
            prod = self.a.astype(np.float64) @ self.b.astype(np.float64)
            absprod = np.abs(self.a).astype(np.float64) @ np.abs(self.b).astype(np.float64)
            acc = (3 * self.K + 4) * 2.0 ** -22
        want = self.alpha * prod + self.beta * self.c0
        mag = abs(self.alpha) * absprod + abs(self.beta) * np.abs(self.c0)
        if self.bias is not None:
            want = want + self.bias[None, :]
            mag = mag + np.abs(self.bias)[None, :]
        if self.relu:
            want = np.maximum(want, 0.0)
        tol = abs(self.alpha) * acc * absprod + 2.0 ** -22 * mag + 1e-30
        if self.c_bf16:
            tol = tol + 2.0 ** -8 * np.abs(want)
        return want, tol


def bf16(x):
    import oracle
    return oracle.bf16_round(np.asarray(x, F32))


def check(got, want, tol, what):
    err = np.abs(got.astype(np.float64) - want)
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), float(err.max()), float((err / tol).max()))


def width(mode, N):
    """the tile width the dispatcher picks: 64 / 128 / 256 by N, at most 128 in 3xTF32 mode (two accumulators)"""
    return 64 if N <= 64 else 128 if N <= 128 or mode == "tf32x3" else 256


def run_checked(nk, dev, mode, form, M, N, K, cdt="f32", **kw):
    c = Case(nk, dev, form, M, N, K, cdt, **kw)
    dev.f32_matmul(mode)
    got, kern = c.run()
    want, tol = c.want_and_tol(mode)
    check(got, want, tol, (mode, form, M, N, K, cdt, kw))
    return got, kern


# ------------------------------------------------------------------------------------------- form x mode x tile width
WIDTH_N = {64: 50, 128: 100, 256: 300}


@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("width", [64, 128, 256])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("mode", MODES)
def test_every_form_mode_and_tile_width(nk, dev, mode, form, width, cdt):
    """M = 200 (a partial second m-block), K = 136 (a partial k-block), leading dimensions above their minimum, a gap
    after each C row; beta = 1 on a bf16 C.  (3xTF32 runs N = 300 on 128-wide tiles.)"""
    N = WIDTH_N[width]
    beta = 1.0 if cdt == "bf16" else 0.0
    _, kern = run_checked(nk, dev, mode, form, 200, N, 136, cdt, beta=beta, ldc=N + 6, pad_a=4, pad_b=8,
                          seed=width + len(form + cdt + mode))
    assert kern == f"{mode}_{form.lower()}_128x{min(width, 128) if mode == 'tf32x3' else width}"


# ------------------------------------------------------------------------------------------- tile and k-block edges
SIZES = [(128, 256, 32), (127, 255, 31), (129, 257, 33), (256, 128, 1), (255, 129, 64), (1, 1, 1), (257, 65, 95),
         (130, 520, 257)]


@pytest.mark.parametrize("form", ["NT", "NN", "TN"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K", SIZES)
def test_tile_and_k_block_edges(nk, dev, mode, form, M, N, K):
    _, kern = run_checked(nk, dev, mode, form, M, N, K, seed=M * 7 + N + K)
    assert kern == f"{mode}_{form.lower()}_128x{width(mode, N)}"


# ------------------------------------------------------------------------------------------- layouts TMA cannot read
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("mode", MODES)
def test_unaddressable_operands_are_packed(nk, dev, mode, form):
    """K = 37 and odd leading dimensions, operand bases 4 and 12 bytes off 16-byte alignment, C one element off its
    alignment with an odd ldc (the drain's scalar stores)"""
    _, kern = run_checked(nk, dev, mode, form, 150, 133, 37, "f32", ldc=137, off_c=1, pad_a=3, pad_b=5, off_a=1,
                          off_b=3, seed=11)
    assert kern == f"{mode}_{form.lower()}_128x{width(mode, 133)}"
    _, kern = run_checked(nk, dev, mode, form, 150, 90, 37, "bf16", beta=0.5, ldc=91, off_c=1, pad_a=1, off_a=3, seed=12)
    assert kern == f"{mode}_{form.lower()}_128x128"


# ------------------------------------------------------------------------------------------- epilogue
@pytest.mark.parametrize("cdt", ["f32", "bf16"])
@pytest.mark.parametrize("mode", MODES)
def test_epilogue_matrix(nk, dev, mode, cdt):
    """alpha x beta x bias (none, f32, f32 off alignment, bf16) x ReLU, in nk_gemm_simt.cu's order"""
    i = 0
    for alpha in (1.0, -0.75):
        for beta in (0.0, 0.5, 1.0):
            for bias in (None, "f32", "f32+1", "bf16"):
                for relu in (False, True):
                    i += 1
                    _, kern = run_checked(nk, dev, mode, "NT", 140, 200, 72, cdt, alpha=alpha, beta=beta, bias=bias,
                                          relu=relu, ldc=202, seed=i)
                    assert kern == f"{mode}_nt_128x{width(mode, 200)}"


# ------------------------------------------------------------------------------------------- the rounding, bit for bit
def test_tf32_rounding_is_cvt_rna(nk, dev):
    """K = 1: C = tf32(a) tf32(b) is one exact product, rounded once to f32 -- the model's rounding (to nearest, ties
    away) must hold for every element, including ties and values a truncating conversion would round down"""
    rng = np.random.default_rng(5)
    base = rng.uniform(1, 2, (256, 1)).astype(F32)
    u = (base.view(np.uint32) & np.uint32(0xFFFFE000)) | rng.choice(np.array([0x0FFF, 0x1000, 0x1001, 0x1FFF, 0], np.uint32),
                                                                    base.shape)
    a = (u.view(F32) * rng.choice(np.array([1, -1], F32), base.shape)).astype(F32)
    b = a[:200].T.copy()
    c = Case(nk, dev, "NT", 256, 200, 1, a=a, b=b)
    dev.f32_matmul("tf32")
    got, kern = c.run()
    want = (T.tf32_round(a).astype(np.float64) @ T.tf32_round(b).astype(np.float64)).astype(F32)
    assert kern == "tf32_nt_128x256"
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------- determinism and forms
@pytest.mark.parametrize("mode", MODES)
def test_forms_give_the_same_bits_and_calls_repeat(nk, dev, mode):
    rng = np.random.default_rng(3)
    a = rng.uniform(-1, 1, (300, 520)).astype(F32)
    b = rng.uniform(-1, 1, (520, 200)).astype(F32)
    dev.f32_matmul(mode)
    outs = {}
    for form in FORMS:
        c = Case(nk, dev, form, 300, 200, 520, a=a, b=b, pad_a=form.count("T"))
        outs[form], kern = c.run()
        assert kern == f"{mode}_{form.lower()}_128x{width(mode, 200)}"
        again, _ = c.run()
        assert np.array_equal(again.view(np.uint32), outs[form].view(np.uint32)), form
    for form in FORMS:
        assert np.array_equal(outs[form].view(np.uint32), outs["NT"].view(np.uint32)), form


@pytest.mark.parametrize("mode", MODES)
def test_captured_call_equals_eager(nk, dev, mode):
    c = Case(nk, dev, "NN", 260, 300, 200, beta=1.0, bias="f32", seed=9)
    dev.f32_matmul(mode)
    eager, _ = c.run()
    C = Strided(dev, c.c0, nk.F32)
    launches = dev.launches
    with dev.capture(1 << 26) as cap:
        nk._lib.check(c.ops.lib.nk_gemm_bias_act(dev.ctx, 0, 0, 260, 300, 200, 1.0, c.A.ptr, c.A.ld, c.B.ptr, c.B.ld, 1.0,
                                                 C.ptr, 300, nk.F32, nk.F32, c.bptr, c.bdt, 0), dev.ctx)
    assert dev.launches - launches == 3   # two operand packs, one GEMM
    dev.f32_matmul("ieee")                # the graph keeps the mode it was captured with
    cap.graph.launch()
    assert np.array_equal(C.read().view(np.uint32), eager.view(np.uint32))
    cap.graph.close()


# ------------------------------------------------------------------------------------------- accuracy against SIMT
def test_tf32x3_accuracy_against_simt_and_tf32(nk, dev):
    """rms error against float64 on the unrounded operands: 3xTF32 within 8x of the CUDA-core engine's and at least 64x
    below one TF32 pass"""
    rng = np.random.default_rng(21)
    M, N, K = 256, 256, 2048
    a = rng.uniform(-1, 1, (M, K)).astype(F32)
    b = rng.uniform(-1, 1, (K, N)).astype(F32)
    want = a.astype(np.float64) @ b.astype(np.float64)
    err = {}
    for mode in ("ieee", "tf32", "tf32x3"):
        dev.f32_matmul(mode)
        got, kern = Case(nk, dev, "NT", M, N, K, a=a, b=b).run()
        assert kern == ("simt_64x64x16" if mode == "ieee" else f"{mode}_nt_128x{width(mode, N)}")
        err[mode] = float(np.sqrt(np.mean((got.astype(np.float64) - want) ** 2)))
    print(f"rms error vs float64 (K = {K}): {err}; tf32x3 / simt = {err['tf32x3'] / err['ieee']:.2f}, "
          f"tf32 / tf32x3 = {err['tf32'] / err['tf32x3']:.1f}")
    assert err["tf32x3"] <= 8 * err["ieee"], err
    assert 64 * err["tf32x3"] <= err["tf32"], err


# ------------------------------------------------------------------------------------------- settings
def test_simt_engine_overrides_the_mode_and_ieee_restores_simt_bits(nk, dev):
    c = Case(nk, dev, "TN", 200, 180, 90, bias="bf16", relu=True, seed=4)
    dev.f32_matmul("ieee")
    ref, kern = c.run()
    assert kern.startswith("simt")
    for mode in MODES:
        dev.f32_matmul(mode)
        dev.gemm_engine("simt")
        got, k2 = c.run()
        assert k2 == kern and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
        dev.gemm_engine("auto")
        _, k3 = c.run()
        assert k3 == f"{mode}_tn_128x{width(mode, 180)}"
    dev.f32_matmul("ieee")
    got, k4 = c.run()
    assert k4 == kern and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_forced_wgmma_engine(nk, dev):
    """gemm_engine("wgmma") keeps its error for f32 operands in IEEE mode and runs them on the tf32 engine otherwise"""
    c = Case(nk, dev, "NT", 64, 64, 64, seed=2)
    dev.gemm_engine("wgmma")
    with pytest.raises(RuntimeError, match="not bf16"):
        c.run()
    dev.f32_matmul("tf32")
    _, kern = c.run()
    assert kern == "tf32_nt_128x64"


def test_bad_mode_is_rejected(nk, dev):
    from neuronika_b200 import ops
    assert ops.lib.nk_gemm_f32_config(dev.ctx, 3) == -1
    assert ops.lib.nk_gemm_f32_config(dev.ctx, -1) == -1
    with pytest.raises(ValueError):
        dev.f32_matmul("fp16")


# ------------------------------------------------------------------------------------------- the other entry points
@pytest.mark.parametrize("mode", MODES)
def test_relu_bwd_products_follow_the_mode(nk, dev, mode):
    """nk_gemm_relu_bwd with f32 operands: the product on the tf32 engine into a temporary, then the ReLU backward; the
    fused column sums stay unsupported (the caller sums them itself)"""
    from neuronika_b200 import ops
    rng = np.random.default_rng(8)
    M, N, K = 200, 150, 96
    a = rng.uniform(-1, 1, (M, K)).astype(F32)
    w = rng.uniform(-1, 1, (N, K)).astype(F32)
    x = rng.uniform(-1, 1, (M, N)).astype(F32)
    c0 = rng.uniform(-1, 1, (M, N)).astype(F32)
    A, W, X, C = (dev.from_ndarray(v) for v in (a, w, x, c0))
    dev.f32_matmul(mode)
    nk._lib.check(ops.lib.nk_gemm_relu_bwd(dev.ctx, 0, 1, M, N, K, A.ptr, K, W.ptr, K, 1.0, C.ptr, N, nk.F32, nk.F32, X.ptr),
                  dev.ctx)
    assert dev.last_gemm_kernel == f"{mode}_nt_128x{width(mode, N)}"
    case = Case(nk, dev, "NT", M, N, K, a=a, b=w.T.copy())
    prod, tol = case.want_and_tol(mode)
    want = c0 + (x > 0) * prod
    check(C.as_ndarray(), want, tol + 2.0 ** -22 * np.abs(c0), "relu_bwd")
    colsum = dev.zeros((N,))
    rc = ops.lib.nk_gemm_relu_bwd_colsum(dev.ctx, 0, 1, M, N, K, A.ptr, K, W.ptr, K, 0.0, C.ptr, N, nk.F32, nk.F32, X.ptr,
                                         colsum.ptr)
    assert rc == -5


@pytest.mark.parametrize("mode", MODES)
def test_strided_batched_products_follow_the_mode(nk, dev, mode):
    from neuronika_b200 import ops
    rng = np.random.default_rng(6)
    batch, M, N, K = 3, 70, 90, 40
    a = rng.uniform(-1, 1, (batch, M, K)).astype(F32)
    b = rng.uniform(-1, 1, (batch, N, K)).astype(F32)
    bias = rng.uniform(-1, 1, (batch, N)).astype(F32)
    A, B, Bias = dev.from_ndarray(a), dev.from_ndarray(b), dev.from_ndarray(bias)
    C = dev.zeros((batch, M, N))
    dev.f32_matmul(mode)
    ops.gemm_strided_batched(A, B, C, M, N, K, batch, K, K, N, M * K, N * K, M * N, trans_b=True, bias=Bias, bias_stride=N)
    assert dev.last_gemm_kernel == f"{mode}_nt_128x128"
    got = C.as_ndarray()
    for i in range(batch):
        case = Case(nk, dev, "NT", M, N, K, a=a[i], b=b[i].T.copy())
        want, tol = case.want_and_tol(mode)
        check(got[i], want + bias[i][None, :], tol + 2.0 ** -22 * np.abs(bias[i])[None, :], ("batched", i))
