"""The TMA-store epilogue's column bias staged in shared memory: the producer copies each tile's bf16 bias slice with
the tile's first k-block into one of two slots, and the consumer warps release a slot once they have read it.  An f32
bias, a bias that is not 16-byte aligned (and N % 8 != 0) keep the bias loads of the epilogue.

Every case runs twice through nk_gemm_bias_act on the same operands: beta = 0 (the TMA store) and beta = 1 on a zeroed C
(the shared-memory drain, which never stages the bias).  Both must match the float64 reference within the tolerances of
test_gpu_gemm_tma_store.py, and each other bit for bit; nothing outside the C view may be written.  The kernel that ran
is checked by name in every case."""
import numpy as np
import pytest

from test_gpu_gemm_tma_store import cdtype, check, run

pytestmark = pytest.mark.gpu

# bf16: staged; f32 and bf16 one element off 16-byte alignment: the epilogue's own loads
BIASES = ["bf16", "f32", "bf16+1"]


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


def same_bits_as_drain(nk, dev, O, form, M, N, K, cdt, bias, alpha, relu, seed):
    c = cdtype(nk, cdt)
    tma, want, kern = run(nk, dev, O, form, M, N, K, c, alpha=alpha, bias=bias, relu=relu, seed=seed)
    assert kern == f"wgmma_{form.lower()}_128x256", kern
    check(tma, want, c == nk.BF16, (form, M, N, K, cdt, bias, alpha, relu))
    drn, _, kern = run(nk, dev, O, form, M, N, K, c, alpha=alpha, bias=bias, relu=relu, drain=True, seed=seed)
    assert kern == f"wgmma_{form.lower()}_128x256", kern
    neq = np.flatnonzero(tma != drn)
    assert neq.size == 0, (form, M, N, K, cdt, bias, neq.size, tma.flat[neq[0]], drn.flat[neq[0]])


@pytest.mark.parametrize("alpha,relu", [(1.0, False), (-0.75, True)])
@pytest.mark.parametrize("bias", BIASES)
@pytest.mark.parametrize("cdt", ["bf16", "f32"])
@pytest.mark.parametrize("form", ["NT", "NN", "TN"])
def test_partial_last_tile(nk, dev, O, form, cdt, bias, alpha, relu):
    """N = 264: the last tile's bias slice is one 16-byte unit; ragged M"""
    same_bits_as_drain(nk, dev, O, form, 333, 264, 200, cdt, bias, alpha, relu, seed=1)


@pytest.mark.parametrize("bias", BIASES)
@pytest.mark.parametrize("cdt", ["bf16", "f32"])
@pytest.mark.parametrize("K", [64, 128])
def test_producer_runs_ahead_of_the_bias_slots(nk, dev, O, K, cdt, bias):
    """one or two k-blocks per tile and more than 8 tiles per CTA: the producer reaches a bias slot before the consumers
    have released it, so every reuse waits on the slot's barrier.  N = 4096 + 8 leaves a partial last tile"""
    M, N = 9216, 4096 + 8
    sm = dev.sm_count
    tiles = -(-M // 128) * -(-N // 256)
    waves = -(-tiles // sm)
    grid = -(-tiles // waves)
    assert tiles // grid > 8, (tiles, grid)
    same_bits_as_drain(nk, dev, O, "NT", M, N, K, cdt, bias, -0.75, True, seed=K)


@pytest.mark.parametrize("cdt", ["bf16", "f32"])
def test_bias_rows_not_a_multiple_of_8(nk, dev, O, cdt):
    """f32 output with N % 8 == 4: the TMA store still runs (rows end on 16-byte units), but the last tile's bf16 bias
    slice is not a whole number of 16-byte units, so the epilogue loads the bias itself; bf16 output (N % 8 != 0) drains"""
    same_bits_as_drain(nk, dev, O, "NT", 200, 300, 136, cdt, "bf16", 1.5, True, seed=3)
