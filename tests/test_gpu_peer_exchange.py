"""The data-parallel exchange kernels (nk_peer.cu) and the reduce-scatter epilogue of the wgmma GEMM (nk_gemm_rs) on ONE
GPU, with every rank emulated in this process.

A peer pointer is a device pointer, so `world` ranks are `world` sets of ordinary buffers on one device, and each rank's
launch runs in turn on one stream.  What is checked here: the data path, the slot and offset arithmetic, the rank-order
summation, the signal addressing and the device-resident epoch.  Cross-GPU memory ordering and concurrent progress are
left to tests/test_gpu_dp.py, which needs two GPUs.

No launch may spin.  Before every launch `Flags.arm(epoch)` writes epoch + 0x100 to every word of every flag buffer
(64 words each, more than the 2 * world a kernel addresses) and reads them back.  The kernels wait for
int32(word - epoch) >= 0, so every wait returns on its first read, whatever index it reads; their signals write exactly
`epoch`.  After the launch, the words that should have been signalled hold `epoch` and every other word still holds the
armed value.  A call that the host rejects launches nothing: `dev.launches` is pinned for every call.

Every output is a view into a buffer whose other elements hold a canary (`Guarded`), checked bit for bit.  Outputs the
kernel must not read are pre-filled with NaN.  Sums are compared bit for bit with the float32 rank-order sum
((s0 + s1) + s2) ..., which is what makes every replica receive the same bits.  Each case names the path it is meant
to take and cites the host predicate that picks it.

The file's buffers peak at about 0.4 GB (the 4096 x 4096 reduce-scatter case); the process peaked at 882 MiB, CUDA
context included, and the file ran in about 20 s (one H100 80GB HBM3 at a 700 W power limit)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
CANARY = -1152.0          # exact in f32, far outside every value below
U = 2.0 ** -24            # f32 unit roundoff
ARM = 0x100
FLAG_WORDS = 64
MASK32 = 0xFFFFFFFF
INVALID_ARG = -1


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def L():
    from neuronika_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def dev(nk):
    d = nk.Device(0)
    yield d
    d.synchronize()


def table(ptrs):
    return (C.c_void_p * max(1, len(ptrs)))(*[int(p) for p in ptrs])


def h2d(L, dev, dst, host):
    host = np.ascontiguousarray(host)
    L.check(L.lib.nk_h2d(dev.ctx, C.c_void_p(int(dst)), host.ctypes.data_as(C.c_void_p), host.nbytes), dev.ctx)
    dev.synchronize()


def d2h(L, dev, src, n, dtype):
    host = np.empty(n, dtype)
    L.check(L.lib.nk_d2h(dev.ctx, host.ctypes.data_as(C.c_void_p), C.c_void_p(int(src)), host.nbytes), dev.ctx)
    return host


class Guarded:
    """f32 `data` at element `lead` of a device buffer whose other elements -- `lead` before the view and `tail` after
    it -- hold CANARY.  lead = 4 keeps the view 16-byte aligned, lead = 1 puts it one float off: asserted from the
    view's pointer."""

    def __init__(self, L, dev, data, lead=4, tail=12):
        data = np.ascontiguousarray(data, F32)
        self.L, self.dev = L, dev
        self.shape, self.n, self.lead = data.shape, data.size, lead
        host = np.full(lead + self.n + tail, CANARY, F32)
        host[lead:lead + self.n] = data.ravel()
        self.buf = dev.from_ndarray(host)
        self.ptr = int(self.buf.ptr.value) + 4 * lead
        assert (self.ptr % 16 == 0) == (lead % 4 == 0), (lead, self.ptr % 16)

    def view(self):
        """the view as a CuArray (a gradient buffer handed to the graph)"""
        return self.buf.slice_flat(self.lead, self.shape)

    def write(self, data):
        h2d(self.L, self.dev, self.ptr, np.ascontiguousarray(data, F32).reshape(self.n))

    def read(self):
        """(the view, after asserting that nothing outside it changed)"""
        flat = self.buf.as_ndarray().ravel()
        outside = np.concatenate([flat[:self.lead], flat[self.lead + self.n:]])
        bad = np.flatnonzero(outside.view(np.uint32) != F32(CANARY).view(np.uint32))
        assert bad.size == 0, f"{bad.size} elements outside the view were written (first at outside index {bad[0]})"
        return flat[self.lead:self.lead + self.n].reshape(self.shape)


class Flags:
    """rank r's flag words (`ptrs[r]`), armed before every launch so that no wait can spin"""

    def __init__(self, L, dev, world):
        self.L, self.dev = L, dev
        self.bufs = [dev.zeros((FLAG_WORDS,)) for _ in range(world)]
        self.ptrs = [int(b.ptr.value) for b in self.bufs]
        self.armed = None

    def arm(self, epoch):
        words = np.full(FLAG_WORDS, (epoch + ARM) & MASK32, np.uint32)
        for p in self.ptrs:
            h2d(self.L, self.dev, p, words)
        for p in self.ptrs:
            got = d2h(self.L, self.dev, p, FLAG_WORDS, np.uint32)
            assert np.array_equal(got, words), "flag words did not take the armed value"
        self.armed = int(words[0])

    def check(self, epoch, signalled):
        """signalled: the (flag buffer, word) pairs the launch must have set to `epoch`; the rest keep the armed value"""
        for j, p in enumerate(self.ptrs):
            want = np.full(FLAG_WORDS, self.armed, np.uint32)
            for jj, k in signalled:
                if jj == j:
                    want[k] = epoch
            got = d2h(self.L, self.dev, p, FLAG_WORDS, np.uint32)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (f"flag buffer {j}", [(int(k), hex(int(got[k])), hex(int(want[k]))) for k in bad[:8]])


class State:
    """one rank's ExState {epoch, done, next_chunk, error}: 16 bytes of local device memory"""

    def __init__(self, L, dev, epoch=0):
        self.L, self.dev = L, dev
        self.buf = dev.zeros((4,))
        self.ptr = int(self.buf.ptr.value)
        h2d(L, dev, self.ptr, np.array([epoch & MASK32, 0, 0, 0], np.uint32))

    def words(self):
        return d2h(self.L, self.dev, self.ptr, 4, np.uint32)

    def next_epoch(self):
        return (int(self.words()[0]) + 1) & MASK32


def summands(rng, world, n):
    """world rows of n f32 values over 24 binades: their float32 sum depends on the order of the terms"""
    mag = np.exp2(rng.integers(-12, 12, (world, n))).astype(F32)
    return (rng.standard_normal((world, n)).astype(F32) * mag).astype(F32)


def rank_sum(vals):
    """((v0 + v1) + v2) ... in float32: the order every replica sums in"""
    acc = np.array(vals[0], F32, copy=True)
    for v in vals[1:]:
        acc = (acc + np.asarray(v, F32)).astype(F32)
    return acc


def exact(got, want, what):
    g, w = np.ascontiguousarray(got, F32).ravel(), np.ascontiguousarray(want, F32).ravel()
    assert g.size == w.size, (what, g.size, w.size)
    bad = np.flatnonzero(g.view(np.uint32) != w.view(np.uint32))
    assert bad.size == 0, (what, f"{bad.size} differ", int(bad[0]), float(g[bad[0]]), float(w[bad[0]]))


def all_nan(x, what):
    assert np.isnan(x).all(), (what, f"{int((~np.isnan(x)).sum())} elements written")


def launched(dev, n0, k, what):
    assert dev.launches - n0 == k, (what, dev.launches - n0, k)


def rejected(L, dev, rc, text, n0):
    msg = L.last_error(dev.ctx)
    assert rc == INVALID_ARG, (rc, msg)
    assert text in msg, msg
    launched(dev, n0, 0, msg)


# ============================================================================================ nk_reduce_exchange
# One launch per rank: phase A signals word `rank` of every rank's flags and waits for words [0, world) of its own,
# phase B sums 32 KB chunks (kExChunkVec = 2048 float4) handed out by an atomic counter, phase C's last CTA signals word
# world + rank everywhere, waits for words [world, 2 world) of its own and resets done / next_chunk.  The grid is
# max_ctas (0: the SM count) clamped to the chunk count (nk_peer.cu nk_reduce_exchange).
CHUNK = 8192   # floats per chunk


def _exchange_round(L, dev, world, shard, max_ctas, rng, states, flags):
    """one emulated exchange: fresh slots of random summands, NaN gradients; rank r's launch runs in turn; after each,
    the owner's shard of every replica and nothing else is written"""
    vals = [summands(rng, world, shard) for _ in range(world)]        # vals[o][s]: source s's shard for owner o
    slots = [Guarded(L, dev, vals[o]) for o in range(world)]
    grads = [Guarded(L, dev, np.full(world * shard, np.nan, F32)) for _ in range(world)]
    gtab, ftab = table([g.ptr for g in grads]), table(flags.ptrs)
    want = [rank_sum(vals[o]) for o in range(world)]
    for r in range(world):
        e = states[r].next_epoch()
        flags.arm(e)
        n0 = dev.launches
        L.check(L.lib.nk_reduce_exchange(dev.ctx, C.c_void_p(slots[r].ptr), gtab, ftab, world, r, shard,
                                         C.c_void_p(states[r].ptr), max_ctas), dev.ctx)
        launched(dev, n0, 1, "reduce_exchange")
        dev.synchronize()
        flags.check(e, [(j, r) for j in range(world)] + [(j, world + r) for j in range(world)])
        assert list(states[r].words()) == [e, 0, 0, 0], ("ExState after the call", list(states[r].words()), e)
        for x in range(world):
            g = grads[x].read().reshape(world, shard)
            for o in range(world):
                if o <= r:
                    exact(g[o], want[o], f"replica {x}, owner {o}'s shard after rank {r}")
                else:
                    all_nan(g[o], f"replica {x}, owner {o}'s shard before its owner ran")
    for o in range(world):
        exact(slots[o].read(), vals[o], f"slots of rank {o} (read only)")


def _shard(spec, dev):
    return 8192 * dev.sm_count + 4 if spec == "sm" else spec


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("shard", [4, 8188, 8192, 8196])
@pytest.mark.parametrize("max_ctas", [0, 1, 3])
def test_reduce_exchange(L, dev, world, shard, max_ctas):
    """shards at the chunk boundary (one chunk, one chunk, two chunks the second with one float4); two calls in a row,
    each advancing the device epoch by one"""
    rng = np.random.default_rng(1000 * world + shard + max_ctas)
    states = [State(L, dev) for _ in range(world)]
    flags = Flags(L, dev, world)
    for rnd in range(2):
        _exchange_round(L, dev, world, shard, max_ctas, rng, states, flags)
        assert all(int(s.words()[0]) == rnd + 1 for s in states)


@pytest.mark.parametrize("world,shard,max_ctas", [
    (3, "sm", 0),            # one more chunk than CTAs: the first CTA to finish takes the tail chunk
    (3, "sm", 1),            # one CTA walks every chunk
    (2, 1 << 22, 0),         # 512 chunks over sm_count CTAs
    (8, 3 * CHUNK + 4, 1000),  # max_ctas above the chunk count: clamped to 4
])
def test_reduce_exchange_many_chunks(L, dev, world, shard, max_ctas):
    shard = _shard(shard, dev)
    rng = np.random.default_rng(shard + world)
    states = [State(L, dev) for _ in range(world)]
    _exchange_round(L, dev, world, shard, max_ctas, rng, states, Flags(L, dev, world))


def test_reduce_exchange_epoch_wraps(L, dev):
    """ExState.epoch 0xFFFFFFFE: the calls use epochs 0xFFFFFFFF, 0 and 1, and the waits compare modulo 2^32"""
    world, shard = 3, 8196
    rng = np.random.default_rng(7)
    states = [State(L, dev, epoch=0xFFFFFFFE) for _ in range(world)]
    flags = Flags(L, dev, world)
    for want in (0xFFFFFFFF, 0, 1):
        assert all(s.next_epoch() == want for s in states)
        _exchange_round(L, dev, world, shard, 0, rng, states, flags)
        assert all(int(s.words()[0]) == want for s in states)


def test_reduce_exchange_graph_replay(L, dev):
    """rank 0's call captured once (dev.capture) and replayed twice, re-armed before each replay: the launch is the same
    every step because the epoch lives on the device"""
    world, shard = 3, 2 * CHUNK + 4
    rng = np.random.default_rng(11)
    states = [State(L, dev) for _ in range(world)]
    flags = Flags(L, dev, world)
    slots = [Guarded(L, dev, np.zeros((world, shard), F32)) for _ in range(world)]
    grads = [Guarded(L, dev, np.full(world * shard, np.nan, F32)) for _ in range(world)]
    gtab, ftab = table([g.ptr for g in grads]), table(flags.ptrs)

    def eager(r):
        L.check(L.lib.nk_reduce_exchange(dev.ctx, C.c_void_p(slots[r].ptr), gtab, ftab, world, r, shard,
                                         C.c_void_p(states[r].ptr), 0), dev.ctx)

    with dev.capture(1 << 20) as cap:
        eager(0)
    graph = cap.graph
    assert graph.kernel_count == 1
    dev.synchronize()
    assert list(states[0].words()) == [0, 0, 0, 0], "capturing ran the kernel"
    for rep in (1, 2):
        vals = [summands(rng, world, shard) for _ in range(world)]
        for o in range(world):
            slots[o].write(vals[o])
        for g in grads:
            g.write(np.full(world * shard, np.nan, F32))
        for r in range(world):
            e = states[r].next_epoch()
            assert e == rep
            flags.arm(e)
            n0 = dev.launches
            graph.launch() if r == 0 else eager(r)
            launched(dev, n0, 1, "replay" if r == 0 else "reduce_exchange")
            dev.synchronize()
            flags.check(e, [(j, r) for j in range(world)] + [(j, world + r) for j in range(world)])
            assert list(states[r].words()) == [e, 0, 0, 0]
        for x in range(world):
            g = grads[x].read().reshape(world, shard)
            for o in range(world):
                exact(g[o], rank_sum(vals[o]), f"replay {rep}: replica {x}, owner {o}")
    graph.close()


@pytest.mark.parametrize("case", ["world0", "world9", "rank_eq_world", "shard0", "shard6", "shard-4", "null_state"])
def test_reduce_exchange_rejects(L, dev, case):
    """host-side rejections (nk_peer.cu nk_reduce_exchange's NK_REQUIREs): nothing launched, nothing written"""
    world, shard = 2, 8
    slots = Guarded(L, dev, np.zeros(world * shard, F32))
    grads = [Guarded(L, dev, np.full(world * shard, np.nan, F32)) for _ in range(world)]
    flags = Flags(L, dev, world)
    st = State(L, dev)
    w, r, n, sp = world, 0, shard, st.ptr
    text = "nk_reduce_exchange: bad arguments"
    if case == "world0":
        w = 0
    elif case == "world9":
        w = 9
    elif case == "rank_eq_world":
        r = world
    elif case == "null_state":
        sp = 0
    else:
        n = {"shard0": 0, "shard6": 6, "shard-4": -4}[case]
        text = "is not a positive multiple of 4"
    n0 = dev.launches
    rc = L.lib.nk_reduce_exchange(dev.ctx, C.c_void_p(slots.ptr), table([g.ptr for g in grads] * 5),
                                  table(flags.ptrs * 5), w, r, n, C.c_void_p(sp) if sp else None, 0)
    rejected(L, dev, rc, text, n0)
    for g in grads:
        all_nan(g.read(), "gradient of a rejected call")
    assert list(st.words()) == [0, 0, 0, 0]


# ============================================================================================ nk_reduce_bcast
# The three-launch form's middle kernel: grid = max_ctas (0: 20) of 1024 threads, cut to ceil(shard / 4 / 1024); each
# thread sums U = 4 float4 per grid stride, so 20 CTAs cover U * stride = 327680 floats per pass (nk_peer.cu
# nk_reduce_bcast).  shard 0 returns before the launch.
BCAST_CASES = [(w, n, c) for w in (1, 2, 3, 8) for n in (0, 4, 4096, 4100, 327676, 327680, 327684) for c in (0, 1, 7)
               if w < 8 or n <= 4100 or c == 0]     # the wide shards at world 8 with the default grid only


@pytest.mark.parametrize("world,shard,max_ctas", BCAST_CASES)
def test_reduce_bcast(L, dev, world, shard, max_ctas):
    rng = np.random.default_rng(world * 7 + shard + max_ctas)
    vals = [summands(rng, world, shard) for _ in range(world)]
    slots = [Guarded(L, dev, vals[o]) for o in range(world)]
    grads = [Guarded(L, dev, np.full(world * shard, np.nan, F32)) for _ in range(world)]
    gtab = table([g.ptr for g in grads])
    want = [rank_sum(vals[o]) if shard else np.zeros(0, F32) for o in range(world)]
    for r in range(world):
        n0 = dev.launches
        L.check(L.lib.nk_reduce_bcast(dev.ctx, C.c_void_p(slots[r].ptr), gtab, world, r, shard, max_ctas), dev.ctx)
        launched(dev, n0, 1 if shard else 0, "reduce_bcast")
        dev.synchronize()
        for x in range(world):
            g = grads[x].read().reshape(world, shard)
            for o in range(world):
                if o <= r:
                    exact(g[o], want[o], f"replica {x}, owner {o}'s shard after rank {r}")
                else:
                    all_nan(g[o], f"replica {x}, owner {o}'s shard before its owner ran")
    for o in range(world):
        exact(slots[o].read(), vals[o], f"slots of rank {o} (read only)")


def test_reduce_bcast_rejects(L, dev):
    g = Guarded(L, dev, np.full(16, np.nan, F32))
    s = Guarded(L, dev, np.zeros(16, F32))
    for w, r, n, text in ((9, 0, 8, "bad arguments"), (2, 2, 8, "bad arguments"), (0, 0, 8, "bad arguments"),
                          (2, 0, 6, "not a multiple of 4")):
        n0 = dev.launches
        rejected(L, dev, L.lib.nk_reduce_bcast(dev.ctx, C.c_void_p(s.ptr), table([g.ptr] * 9), w, r, n, 0), text, n0)
    all_nan(g.read(), "gradient of a rejected call")


# ============================================================================================ nk_peer_barrier
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("epoch", [1, 0x80000000, 0xFFFFFFFF])
def test_peer_barrier(L, dev, world, epoch):
    """one thread per peer stores `epoch` into word `rank` of that peer's flags and waits for word r of its own"""
    flags = Flags(L, dev, world)
    for r in range(world):
        flags.arm(epoch)
        n0 = dev.launches
        L.check(L.lib.nk_peer_barrier(dev.ctx, table(flags.ptrs), world, r, epoch), dev.ctx)
        launched(dev, n0, 1, "peer_barrier")
        dev.synchronize()
        flags.check(epoch, [(j, r) for j in range(world)])


def test_peer_barrier_rejects(L, dev):
    flags = Flags(L, dev, 2)
    for w, r in ((0, 0), (9, 0), (2, 2), (2, -1)):
        n0 = dev.launches
        rejected(L, dev, L.lib.nk_peer_barrier(dev.ctx, table(flags.ptrs * 5), w, r, 1), "bad world", n0)


# ============================================================================================ nk_peer_allreduce_small
# One CTA of 1024 threads.  The vector body runs when n % 4 == 0 and both `grad` and the rank's own slot base are
# 16-byte aligned (nk_peer.cu small_allreduce_kernel `vec`; every rank's slots sit at the same byte offset, as
# parallel.py allocates them); it moves U = 8 float4 per thread and pass, so 32768 floats is one pass exactly.
# Everything else takes the scalar body.
#
# The ranks run one after the other, so rank r sums before the ranks s > r have pushed.  The test stands in for those
# pushes: region s of rank r's slots holds rank s's values for s > r and NaN for s <= r, so a push that does not land
# leaves a NaN in the sum.  The second round runs the ranks in the order world-1 .. 0 on fresh buffers, so that every
# (sender, receiver) pair is covered by a real push.
SMALL_N = [1, 3, 4, 5, 4096, 32764, 32768, 32772]


def _small_round(L, dev, world, n, align, order, rng):
    vals = summands(rng, world, n)
    glead = 1 if align == "grad+1" else 4
    slead = 1 if align == "slot+1" else 4
    grads = [Guarded(L, dev, vals[r], lead=glead) for r in range(world)]
    pos = {r: i for i, r in enumerate(order)}
    slots = []
    for r in range(world):
        init = np.full((world, n), np.nan, F32)
        for s in range(world):
            if pos[s] > pos[r]:
                init[s] = vals[s]
        slots.append(Guarded(L, dev, init, lead=slead))
    vec = n % 4 == 0 and grads[0].ptr % 16 == 0 and slots[0].ptr % 16 == 0
    assert vec == (align == "aligned" and n % 4 == 0)
    stab = table([s.ptr for s in slots])
    flags = Flags(L, dev, world)
    states = [State(L, dev, epoch=5) for _ in range(world)]
    for r in order:
        e = states[r].next_epoch()
        flags.arm(e)
        n0 = dev.launches
        L.check(L.lib.nk_peer_allreduce_small(dev.ctx, C.c_void_p(grads[r].ptr), stab, table(flags.ptrs), world, r, n,
                                              C.c_void_p(states[r].ptr)), dev.ctx)
        launched(dev, n0, 1, "peer_allreduce_small")
        dev.synchronize()
        flags.check(e, [(j, r) for j in range(world)] + [(j, world + r) for j in range(world)])
        assert list(states[r].words()) == [e, 0, 0, 0]
    want = rank_sum(vals)
    for r in range(world):
        exact(grads[r].read(), want, f"grad of rank {r} ({'vector' if vec else 'scalar'} body)")
        exact(slots[r].read(), vals, f"slots of rank {r}: region s holds rank s's values")


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("n", SMALL_N)
@pytest.mark.parametrize("align", ["aligned", "grad+1", "slot+1"])
def test_peer_allreduce_small(L, dev, world, n, align):
    rng = np.random.default_rng(world * 100003 + n * 3 + len(align))
    _small_round(L, dev, world, n, align, list(range(world)), rng)
    _small_round(L, dev, world, n, align, list(range(world))[::-1], rng)


@pytest.mark.parametrize("world,align", [(2, "aligned"), (3, "aligned"), (3, "grad+1")])
def test_peer_allreduce_small_largest(L, dev, world, align):
    """n = 2^20, the largest the kernel takes: 32 vector passes"""
    rng = np.random.default_rng(world)
    _small_round(L, dev, world, 1 << 20, align, list(range(world)), rng)


def test_peer_allreduce_small_rejects(L, dev):
    g = Guarded(L, dev, np.full(8, np.nan, F32))
    s = Guarded(L, dev, np.zeros(16, F32))
    flags = Flags(L, dev, 2)
    st = State(L, dev)
    for w, r, n, text in ((2, 0, 0, "outside (0, 2^20]"), (2, 0, (1 << 20) + 1, "outside (0, 2^20]"),
                          (9, 0, 8, "bad arguments"), (2, 2, 8, "bad arguments")):
        n0 = dev.launches
        rc = L.lib.nk_peer_allreduce_small(dev.ctx, C.c_void_p(g.ptr), table([s.ptr] * 9), table(flags.ptrs * 5), w, r, n,
                                           C.c_void_p(st.ptr))
        rejected(L, dev, rc, text, n0)
    all_nan(g.read(), "grad of a rejected call")
    assert list(st.words()) == [0, 0, 0, 0]


# ============================================================================================ nk_gemm_rs
# nk_gemm_rs sets the reduce-scatter plan and calls nk_gemm_bias_act with the engine forced to the tensor cores: one
# launch of the 128 x 256 wgmma kernel whose drain epilogue stores row shard o (rows [o M/W, (o+1) M/W)) to
# slots[o] + rank * shard, in the rotated tile order of tile_m_block.  The plain product it must match bit for bit is
# nk_gemm_bias_act on the same operands, engine forced to the tensor cores, f32 C, beta 0: the same kernel with the
# TMA-store epilogue.  Both epilogues round alpha * acc once (__fmul_rn) and store f32, so they store the same bits.
# op(A) is (M, K), op(B) is (K, N); "TN" (A stored (K, M), B stored (K, N)) is the graph's dW form.  Leading
# dimensions are padded to a multiple of 8 elements (TMA) with NaN that the kernel must not read.
# The rotated tile order (tile_m_block's m_rot) only permutes the tiles over the CTAs: no result depends on it, so
# these cases check the stores it leads to, not the order itself.
FORMS = {"TN": (1, 0), "NT": (0, 1), "NN": (0, 0), "TT": (1, 1)}


def _pad8(x):
    return -(-x // 8) * 8


class Operands:
    """bf16 A, B of one rank for op(A).op(B) in the given form, in padded buffers"""

    def __init__(self, L, dev, rng, form, M, N, K, a_off=0):
        from neuronika_b200.device import CuArray
        self.tA, self.tB = FORMS[form]
        self.a = rng.uniform(-1, 1, (M, K)).astype(F32)
        self.b = rng.uniform(-1, 1, (K, N)).astype(F32)
        self.a = L.bf16_bits_to_f32(L.f32_to_bf16_bits(self.a))
        self.b = L.bf16_bits_to_f32(L.f32_to_bf16_bits(self.b))
        sa = self.a.T if self.tA else self.a          # as stored
        sb = self.b.T if self.tB else self.b
        self.lda, self.ldb = _pad8(sa.shape[1]), _pad8(sb.shape[1])
        self.bufs = []
        self.A = self._upload(L, dev, CuArray, sa, self.lda, a_off)
        self.B = self._upload(L, dev, CuArray, sb, self.ldb, 0)

    def _upload(self, L, dev, CuArray, stored, ld, off):
        rows, cols = stored.shape
        host = np.full((rows * ld + off + 8,), np.nan, F32)
        host[off:off + rows * ld].reshape(rows, ld)[:, :cols] = stored
        buf = CuArray(dev, host.shape, L.NK_BF16)
        bits = L.f32_to_bf16_bits(host)
        L.check(L.lib.nk_h2d(dev.ctx, buf.ptr, bits.ctypes.data_as(C.c_void_p), buf.nbytes), dev.ctx)
        dev.synchronize()
        self.bufs.append(buf)
        return int(buf.ptr.value) + 2 * off

    def bound(self, alpha, got, what):
        """|got - alpha.AB| <= (K + 4) 2^-24 |alpha| (|A||B|) elementwise, against float64"""
        a, b = self.a.astype(np.float64), self.b.astype(np.float64)
        want = alpha * (a @ b)
        tol = (a.shape[1] + 4) * U * abs(alpha) * (np.abs(a) @ np.abs(b))
        err = np.abs(got.astype(np.float64) - want)
        bad = np.flatnonzero(~(err <= tol))
        assert bad.size == 0, (what, f"{bad.size} outside", int(bad[0]), float(got.ravel()[bad[0]]),
                               float(want.ravel()[bad[0]]), float(tol.ravel()[bad[0]]))


def plain_product(L, dev, ops, M, N, K, alpha):
    """nk_gemm_bias_act, engine forced to the tensor cores, f32 C (NaN-filled: beta 0 must not read it)"""
    c = Guarded(L, dev, np.full((M, N), np.nan, F32))
    dev.gemm_engine("wgmma")
    try:
        n0 = dev.launches
        L.check(L.lib.nk_gemm_bias_act(dev.ctx, ops.tA, ops.tB, M, N, K, alpha, C.c_void_p(ops.A), ops.lda,
                                       C.c_void_p(ops.B), ops.ldb, 0.0, C.c_void_p(c.ptr), N, L.NK_BF16, L.NK_F32, None,
                                       L.NK_F32, 0), dev.ctx)
        launched(dev, n0, 1, "plain wgmma GEMM")
    finally:
        dev.gemm_engine("auto")
    return c.read()


def _gemm_rs_case(L, dev, world, form, M, N, K, alpha, seed, bound_ranks=(0,)):
    rng = np.random.default_rng(seed)
    shard_rows = M // world
    slots = [Guarded(L, dev, np.full((world, shard_rows, N), np.nan, F32)) for _ in range(world)]
    stab = table([s.ptr for s in slots])
    products = []
    for r in range(world):
        ops = Operands(L, dev, rng, form, M, N, K)
        c = plain_product(L, dev, ops, M, N, K, alpha)
        if r in bound_ranks:
            ops.bound(alpha, c, f"plain product of rank {r}")
        n0 = dev.launches
        L.check(L.lib.nk_gemm_rs(dev.ctx, ops.tA, ops.tB, M, N, K, alpha, C.c_void_p(ops.A), ops.lda, C.c_void_p(ops.B),
                                 ops.ldb, stab, world, r, L.NK_BF16), dev.ctx)
        launched(dev, n0, 1, "nk_gemm_rs")
        assert dev.last_gemm_kernel == f"wgmma_{form.lower()}_128x256", dev.last_gemm_kernel
        products.append(c)
        del ops
    dev.synchronize()
    for o in range(world):
        got = slots[o].read()
        for r in range(world):
            exact(got[r], products[r][o * shard_rows:(o + 1) * shard_rows], f"slot {o}, region {r}")


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("N", [136, 200, 256, 264])
@pytest.mark.parametrize("K", [1, 64, 65])
def test_gemm_rs(L, dev, world, N, K):
    """M = world * 128 (one m block per owner), the graph's TN form; N = 200 ends in a 32-column chunk of 8 columns"""
    _gemm_rs_case(L, dev, world, "TN", world * 128, N, K, 0.75, world * 1000 + N * 10 + K)


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("form", ["TN", "NT", "NN", "TT"])
def test_gemm_rs_forms(L, dev, world, form):
    """M = 3 * world * 128: three m blocks per owner, walked in the rotated order; every operand form TMA takes"""
    _gemm_rs_case(L, dev, world, form, 3 * world * 128, 200, 65, -1.5, world * 10 + len(form) + ord(form[0]))


@pytest.mark.parametrize("world,form,M,N,K", [
    (2, "TN", 256, 264, 8192),      # a long main loop
    (2, "NT", 256, 136, 8192),
    (2, "TN", 256, 4096, 64),       # 16 n blocks
    (4, "TN", 4096, 4096, 64),      # 512 tiles: more than the SMs, each CTA takes several in the rotated order
])
def test_gemm_rs_large(L, dev, world, form, M, N, K):
    _gemm_rs_case(L, dev, world, form, M, N, K, 0.375, M + N + K)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("null_operands", [False, True])
def test_gemm_rs_empty_batch(L, dev, world, null_operands):
    """K = 0 (an empty local batch): the product is zero, and every owner receives this rank's zero shard without a
    launch, so the ranks still agree on the calls that follow"""
    M, N = world * 128, 200
    rng = np.random.default_rng(world)
    slots = [Guarded(L, dev, np.full((world, M // world, N), np.nan, F32)) for _ in range(world)]
    stab = table([s.ptr for s in slots])
    ops = Operands(L, dev, rng, "TN", M, N, 8)
    for r in range(world):
        n0 = dev.launches
        A, B = (None, None) if null_operands else (C.c_void_p(ops.A), C.c_void_p(ops.B))
        L.check(L.lib.nk_gemm_rs(dev.ctx, 1, 0, M, N, 0, 1.0, A, M, B, N, stab, world, r, L.NK_BF16), dev.ctx)
        launched(dev, n0, 0, "nk_gemm_rs with K = 0")
        dev.synchronize()
        for o in range(world):
            got = slots[o].read()
            for s in range(world):
                if s <= r:
                    exact(got[s], np.zeros((M // world, N), F32), f"slot {o}, region {s}")
                else:
                    all_nan(got[s], f"slot {o}, region {s} before rank {s} ran")


# Each rejection leaves the slots as they were, and the context as it was: the next plain GEMM writes C (the plan is
# cleared) and an f32 GEMM runs (the engine is no longer forced to the tensor cores).
RS_ERRORS = {
    "world1": (dict(world=1), "bad world"),
    "world9": (dict(world=9), "bad world"),
    "rank_eq_world": (dict(rank=2), "bad world"),
    "f32_operands": (dict(ab=0), "bf16 operands"),
    "M_not_world_x128": (dict(M=384), "is not a multiple of world * 128"),
    "N128": (dict(N=128), "N > 128"),
    "N64": (dict(N=64), "N > 128"),
    "N_not_x4": (dict(N=202), "N % 4 == 0"),
    "A_misaligned": (dict(a_off=1), "not TMA-addressable"),
    "lda_not_x8": (dict(lda=260), "not TMA-addressable"),
    "slot_misaligned": (dict(slot_off=1), "not 16-byte aligned"),
    "lda_too_small": (dict(lda=128), "leading dimension too small"),   # rejected inside nk_gemm_bias_act, plan set
    "negative_K": (dict(K=-1), "negative dimension"),
}


@pytest.mark.parametrize("case", list(RS_ERRORS))
def test_gemm_rs_rejects(L, dev, case):
    over, text = RS_ERRORS[case]
    world, M, N, K = 2, 256, 264, 64
    rng = np.random.default_rng(3)
    ops = Operands(L, dev, rng, "TN", M, 264, K, a_off=over.get("a_off", 0))
    slots = [Guarded(L, dev, np.full(M * 264 + 8, np.nan, F32)) for _ in range(world)]
    stab = table([s.ptr + 4 * over.get("slot_off", 0) * (o == 1) for o, s in enumerate(slots)] * 5)
    n0 = dev.launches
    rc = L.lib.nk_gemm_rs(dev.ctx, 1, 0, over.get("M", M), over.get("N", N), over.get("K", K), 1.0, C.c_void_p(ops.A),
                          over.get("lda", M), C.c_void_p(ops.B), ops.ldb, stab, over.get("world", world),
                          over.get("rank", 0), over.get("ab", L.NK_BF16))
    msg = L.last_error(dev.ctx)
    rejected(L, dev, rc, text, n0)
    # the next plain GEMM (engine auto) writes C, not the slots
    ops = Operands(L, dev, rng, "TN", M, N, K)
    c = Guarded(L, dev, np.full((M, N), np.nan, F32))
    n0 = dev.launches
    L.check(L.lib.nk_gemm_bias_act(dev.ctx, 1, 0, M, N, K, 1.0, C.c_void_p(ops.A), ops.lda, C.c_void_p(ops.B), ops.ldb,
                                   0.0, C.c_void_p(c.ptr), N, L.NK_BF16, L.NK_F32, None, L.NK_F32, 0), dev.ctx)
    launched(dev, n0, 1, "plain GEMM after a rejection")
    ops.bound(1.0, c.read(), "plain GEMM after a rejection")
    # ... and f32 operands still run (the tensor-core engine is not left forced)
    a = rng.uniform(-1, 1, (16, 8)).astype(F32)
    b = rng.uniform(-1, 1, (8, 24)).astype(F32)
    da, db = dev.from_ndarray(a), dev.from_ndarray(b)
    dc = Guarded(L, dev, np.full((16, 24), np.nan, F32))
    L.check(L.lib.nk_gemm_bias_act(dev.ctx, 0, 0, 16, 24, 8, 1.0, da.ptr, 8, db.ptr, 24, 0.0, C.c_void_p(dc.ptr), 24,
                                   L.NK_F32, L.NK_F32, None, L.NK_F32, 0), dev.ctx)
    want = a.astype(np.float64) @ b
    assert np.all(np.abs(dc.read() - want) <= 12 * U * (np.abs(a) @ np.abs(b)))
    for s in slots:
        all_nan(s.read(), "slot after a rejected nk_gemm_rs")


# ============================================================================================ graph integration
# MatMulBackward pushes dW through nk_gemm_rs when the gradient starts from zero (beta 0), G is bf16, the gradient is
# f32, this node is its only writer, rows % (world * 128) == 0 and cols > 128, cols % 8 == 0 (nk_graph.cpp, the `push`
# predicate); then it calls the hook with 1.  Otherwise it computes the gradient locally and calls the hook with 0.
def _net(V, nk, dev, w, b, x, t, dt, grad_view=None):
    Wv = V.from_ndarray(dev, w, dt).requires_grad(nk.F32, grad_view)
    bv = V.from_ndarray(dev, b, dt).requires_grad(nk.F32)
    loss = (V.from_ndarray(dev, x, dt).mm_t(Wv) + bv).relu().mse_loss(V.from_ndarray(dev, t, dt))
    return Wv, bv, loss


def _replicas(L, dev, nk, world, rows, cols, batch, dt, seed):
    """world replicas with the fused plan (gradient view in a NaN-filled guarded bucket of their own) and world plain
    replicas; the weights are equal, the inputs differ"""
    from neuronika_b200 import variable as V
    rng = np.random.default_rng(seed)
    w = rng.uniform(-0.1, 0.1, (rows, cols)).astype(F32)
    b = rng.uniform(-0.1, 0.1, (rows,)).astype(F32)
    slots = [Guarded(L, dev, np.full(rows * cols, np.nan, F32)) for _ in range(world)]
    slot_ptrs = [s.ptr for s in slots]
    fused, plain, hooks = [], [], []
    for r in range(world):
        x = rng.uniform(-1, 1, (batch, cols)).astype(F32)
        t = rng.uniform(-1, 1, (batch, rows)).astype(F32)
        bucket = Guarded(L, dev, np.full((rows, cols), np.nan, F32))
        Wv, bv, loss = _net(V, nk, dev, w, b, x, t, dt, bucket.view())
        got = []
        hooks.append(got)
        Wv.set_grad_rs(world, r, slot_ptrs, got.append)
        Wv.zero_grad()
        bv.zero_grad()
        fused.append((Wv, bv, loss, bucket))
        plain.append(_net(V, nk, dev, w, b, x, t, dt))
    return fused, plain, hooks, slots


def _backward_all(dev, fused, plain):
    for (_, _, loss, _), (_, _, ploss) in zip(fused, plain):
        loss.forward()
        loss.backward(1.0)
        ploss.forward()
        ploss.backward(1.0)
    dev.synchronize()


def _exchange(L, dev, fused, slots, world, shard):
    flags = Flags(L, dev, world)
    states = [State(L, dev) for _ in range(world)]
    gtab = table([f[3].ptr for f in fused])
    for r in range(world):
        flags.arm(states[r].next_epoch())
        n0 = dev.launches
        L.check(L.lib.nk_reduce_exchange(dev.ctx, C.c_void_p(slots[r].ptr), gtab, table(flags.ptrs), world, r, shard,
                                         C.c_void_p(states[r].ptr), 0), dev.ctx)
        launched(dev, n0, 1, "reduce_exchange")
        dev.synchronize()


@pytest.mark.parametrize("world", [2, 3])
def test_graph_fused_exchange(L, dev, nk, world):
    """backward of every replica pushes its dW shards; the exchange then hands every replica the rank-order sum of
    the plain graphs' dW, bit for bit.  A second backward without zero_grad computes locally (pushed = 0) on top."""
    rows, cols, batch = world * 128, 264, 96
    fused, plain, hooks, slots = _replicas(L, dev, nk, world, rows, cols, batch, nk.BF16, world)
    _backward_all(dev, fused, plain)
    assert hooks == [[1]] * world, hooks
    dws = [p[0].grad() for p in plain]
    for f in fused:
        all_nan(f[3].read(), "bucket after a pushed backward (the local product is never written)")
    _exchange(L, dev, fused, slots, world, rows * cols // world)
    want = rank_sum(dws)
    for r, f in enumerate(fused):
        exact(f[3].read(), want, f"W_{r}.grad after the exchange")
        exact(f[0].grad(), want, f"W_{r}.grad() after the exchange")
    # second backward without zero_grad: beta = 1, no push; the plain replica starts from the same gradient
    before = [s.read().copy() for s in slots]
    for f, p in zip(fused, plain):
        p[0].grad_array().copy_from(f[3].read())
        f[2].backward(1.0)
        p[2].backward(1.0)
    dev.synchronize()
    assert hooks == [[1, 0]] * world, hooks
    for r, (f, p) in enumerate(zip(fused, plain)):
        exact(f[3].read(), p[0].grad(), f"W_{r}.grad after a second backward")
    for o in range(world):
        exact(slots[o].read(), before[o], f"slots of rank {o} after a backward that did not push")


@pytest.mark.parametrize("case", ["rows_not_world_x128", "cols128", "f32_graph"])
def test_graph_no_push(L, dev, nk, case):
    """each case misses one term of the push predicate: pushed = 0, the gradient is the plain graph's, slots untouched"""
    world = 2
    rows, cols, dt = {"rows_not_world_x128": (200, 264, nk.BF16), "cols128": (256, 128, nk.BF16),
                      "f32_graph": (256, 264, nk.F32)}[case]
    fused, plain, hooks, slots = _replicas(L, dev, nk, world, rows, cols, 64, dt, 5)
    _backward_all(dev, fused, plain)
    assert hooks == [[0]] * world, hooks
    for r, (f, p) in enumerate(zip(fused, plain)):
        exact(f[3].read(), p[0].grad(), f"W_{r}.grad computed locally")
    for s in slots:
        all_nan(s.read(), "slot of a gradient that was not pushed")


def test_graph_empty_batch_is_rejected(L, dev, nk):
    """a replica with no rows in its batch does not reach the fused exchange through this net: the MSE forward rejects
    empty input, so backward never runs, no hook fires and no slot is written.  nk_gemm_rs's own K = 0 path (zero
    shards, no launch) is test_gemm_rs_empty_batch."""
    world, rows, cols = 2, 256, 264
    fused, plain, hooks, slots = _replicas(L, dev, nk, world, rows, cols, 0, nk.BF16, 9)
    for f in fused:
        with pytest.raises(L.NkError, match="nk_mse_fwd: NULL pointer or empty input"):
            f[2].forward()
    assert hooks == [[]] * world, hooks
    for s in slots:
        all_nan(s.read(), "slot of a replica whose forward was rejected")
