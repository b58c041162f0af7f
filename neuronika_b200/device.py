"""Device and CuArray: the host-side mirror of the reference's embryonic `cuda` module
(neuronika-variable/src/cuda/device.rs:11-75, cuda/cuarray.rs:10-171) over the C ABI."""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Tuple

import numpy as np

from . import _lib as L

F32, BF16 = L.NK_F32, L.NK_BF16
_DT_NAME = {F32: "f32", BF16: "bf16"}


def as_shape(shape) -> Tuple[int, ...]:
    if isinstance(shape, (int, np.integer)):
        return (int(shape),)
    return tuple(int(s) for s in shape)


def dtype_of(name) -> int:
    if name in (F32, BF16):
        return int(name)
    return {"f32": F32, "float32": F32, "bf16": BF16, "bfloat16": BF16}[str(name)]


class Device:
    """Handle to a CUDA device (`Device::new(idx)`, cuda/device.rs:34-52; Default = device 0).

    Owns the nk_ctx: stream, workspace arena, error string.  Creation fails loudly when there
    is no GPU -- the package has no CPU path."""

    def __init__(self, device: int = 0, stream=None):
        ctx = C.c_void_p()
        rc = L.lib.nk_ctx_create(int(device), C.byref(ctx))
        if rc != 0:
            raise L.NkError(rc, L.last_error(None))
        self.ctx = ctx
        self.index = int(device)
        self.capturing = False          # inside `with capture()`: host reads of device results are refused
        if stream is not None:
            self.set_stream(stream)

    # -- plumbing
    def set_stream(self, cuda_stream_handle: int) -> None:
        L.check(L.lib.nk_ctx_set_stream(self.ctx, C.c_void_p(int(cuda_stream_handle))), self.ctx)

    def synchronize(self) -> None:
        L.check(L.lib.nk_sync(self.ctx), self.ctx)

    @property
    def launches(self) -> int:
        return int(L.lib.nk_launch_count(self.ctx))

    @property
    def sm_count(self) -> int:
        return int(L.lib.nk_sm_count(self.ctx))

    def gemm_engine(self, engine: str) -> None:
        L.check(L.lib.nk_gemm_config(self.ctx, {"auto": 0, "simt": 1, "wgmma": 2}[engine]), self.ctx)

    F32_MATMUL_MODES = {"ieee": 0, "tf32": 1, "tf32x3": 2}

    def f32_matmul(self, mode: str) -> None:
        """How f32 matrix products use the tensor cores (off by default, like torch's allow_tf32):
        "ieee": on the CUDA cores in full f32; "tf32": operands rounded to TF32 (10-bit mantissa, to nearest, ties away
        from zero), products on the wgmma engine with f32 accumulation; "tf32x3": each operand split into a TF32 high
        and low part and three TF32 products summed, close to f32 accuracy.  Applies to every f32 GEMM (mm, mm_t,
        Linear forward and backward, the RNN cells and sequence layers); gemm_engine("simt") still keeps them all on the
        CUDA cores.  The mode is read when a GEMM is launched: a captured step replays with the mode it was captured with."""
        if mode not in self.F32_MATMUL_MODES:
            raise ValueError(f"f32_matmul: mode must be one of {sorted(self.F32_MATMUL_MODES)}, got {mode!r}")
        L.check(L.lib.nk_gemm_f32_config(self.ctx, self.F32_MATMUL_MODES[mode]), self.ctx)

    def f32_conv(self, mode: str) -> None:
        """How f32 convolutions use the tensor cores (off by default, like torch's cudnn.allow_tf32), separately from
        f32_matmul: "ieee": the CUDA-core kernels in full f32; "tf32" / "tf32x3": im2col + the TF32 / 3xTF32 wgmma GEMM
        (operands rounded as f32_matmul describes) for every f32, groups = 1 convolution -- Var.convolution in 1-D,
        2-D and 3-D and the Conv1d / Conv2d / Conv3d layers, forward and backward.  Grouped convolutions stay on the
        CUDA cores, and conv_engine("direct") keeps every convolution there.  The mode is read when a convolution is
        launched: a captured step replays with the mode it was captured with."""
        if mode not in self.F32_MATMUL_MODES:
            raise ValueError(f"f32_conv: mode must be one of {sorted(self.F32_MATMUL_MODES)}, got {mode!r}")
        L.check(L.lib.nk_conv_f32_config(self.ctx, self.F32_MATMUL_MODES[mode]), self.ctx)

    def conv_engine(self, engine: str) -> None:
        """"auto": tensor-core kernels wherever they apply; "direct": CUDA-core kernels only"""
        L.check(L.lib.nk_conv_config(self.ctx, {"auto": 0, "direct": 1}[engine]), self.ctx)

    @property
    def last_gemm_kernel(self) -> str:
        return L.lib.nk_last_gemm_kernel(self.ctx).decode()

    @property
    def last_conv_kernel(self) -> str:
        return L.lib.nk_last_conv_kernel(self.ctx).decode()

    def manual_seed(self, seed: int) -> None:
        """Seed the device's dropout generator and reset its call counter (nk_rng_seed): the masks drawn afterwards are
        a function of the seed and of how many dropout forwards ran since.  Not while capturing.  Without it the seed
        comes from OS entropy.  Data-parallel replicas that should draw different masks need different seeds."""
        L.check(L.lib.nk_rng_seed(self.ctx, int(seed) & (2 ** 64 - 1)), self.ctx)

    def rng_state(self) -> Tuple[int, int]:
        """(seed, dropout calls since seeding) of the device's generator (nk_rng_state; synchronises)."""
        seed, calls = C.c_uint64(), C.c_uint64()
        L.check(L.lib.nk_rng_state(self.ctx, C.byref(seed), C.byref(calls)), self.ctx)
        return int(seed.value), int(calls.value)

    def timer_start(self) -> None:
        L.check(L.lib.nk_timer_start(self.ctx), self.ctx)

    def timer_stop(self) -> float:
        ms = C.c_float()
        L.check(L.lib.nk_timer_stop(self.ctx, C.byref(ms)), self.ctx)
        return float(ms.value)

    def capture(self, arena_bytes: int = 1 << 30) -> "_Capture":
        """Record everything the enclosed step launches into a CUDA graph (nk_capture_begin / nk_capture_end):

            with dev.capture(arena_bytes) as cap:
                step()                      # builds the tape, forward, backward, exchange, optimizer -- recorded, not run
            cap.graph.launch()              # replays the whole step with one driver call

        Run the step once eagerly first (first-use allocations cannot be captured)."""
        return _Capture(self, int(arena_bytes))

    def close(self) -> None:
        if getattr(self, "ctx", None) is not None and self.ctx:
            L.lib.nk_ctx_destroy(self.ctx)
            self.ctx = None

    # -- array constructors (CuArray::zeroed / from_ndarray)
    def zeros(self, shape, dtype=F32) -> "CuArray":
        return CuArray(self, shape, dtype)

    def full(self, shape, value: float, dtype=F32) -> "CuArray":
        a = CuArray(self, shape, dtype)
        L.check(L.lib.nk_fill(self.ctx, a.ptr, a.dtype, a.size, float(value)), self.ctx)
        return a

    def from_ndarray(self, array: np.ndarray, dtype=F32) -> "CuArray":
        a = CuArray(self, np.shape(array), dtype)
        a.copy_from(array)
        return a


class CapturedStep:
    """An instantiated CUDA graph of one step plus the arena its intermediates live in (nk_graph)."""

    def __init__(self, device: Device, handle):
        self.device, self._h = device, handle

    def launch(self) -> None:
        L.check(L.lib.nk_graph_launch(self.device.ctx, self._h), self.device.ctx)

    @property
    def kernel_count(self) -> int:
        return int(L.lib.nk_graph_kernel_count(self._h))

    @property
    def arena_used(self) -> int:
        return int(L.lib.nk_graph_arena_used(self._h))

    def close(self) -> None:
        if self._h and self.device.ctx:
            L.lib.nk_graph_destroy(self.device.ctx, self._h)
        self._h = None


class _Capture:
    def __init__(self, device: Device, arena_bytes: int):
        self.device, self.arena_bytes, self.graph = device, arena_bytes, None

    def __enter__(self):
        L.check(L.lib.nk_capture_begin(self.device.ctx, self.arena_bytes), self.device.ctx)
        self.device.capturing = True
        return self

    def __exit__(self, exc_type, exc, tb):
        self.device.capturing = False
        h = C.c_void_p()
        rc = L.lib.nk_capture_end(self.device.ctx, C.byref(h))
        if exc_type is None:
            L.check(rc, self.device.ctx)
            self.graph = CapturedStep(self.device, h)
        return False


class CuArray:
    """Dense C-order device buffer + shape (CuArray{buffer, dim, strides, device}, cuarray.rs:10-19).
    Zero-filled on allocation like `CuArray::zeroed` (:35)."""

    def __init__(self, device: Device, shape, dtype=F32, ptr: int | None = None, owner=None):
        self.device = device
        self.shape: Tuple[int, ...] = as_shape(shape)
        self.dtype = dtype_of(dtype)
        self.size = int(np.prod(self.shape)) if len(self.shape) else 1
        self.itemsize = 2 if self.dtype == BF16 else 4
        self.nbytes = self.size * self.itemsize
        self._owner = owner
        if ptr is None:
            p = C.c_void_p()
            L.check(L.lib.nk_alloc(device.ctx, self.nbytes, C.byref(p)), device.ctx)
            self.ptr = C.c_void_p(p.value)
            self._owned = True
        else:
            self.ptr = C.c_void_p(int(ptr))
            self._owned = False

    def __del__(self):
        try:
            if self._owned and self.ptr and self.device.ctx:
                L.lib.nk_free(self.device.ctx, self.ptr)
        except Exception:
            pass

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def view(self, shape) -> "CuArray":
        """Same memory, different shape (e.g. flatten (N,C,H,W) -> (N, C*H*W): bit-exact no-op)."""
        shape = tuple(int(s) for s in shape)
        assert int(np.prod(shape)) == self.size, (shape, self.shape)
        return CuArray(self.device, shape, self.dtype, ptr=self.ptr.value, owner=self)

    def slice_flat(self, offset: int, shape) -> "CuArray":
        shape = tuple(int(s) for s in shape)
        n = int(np.prod(shape)) if shape else 1
        assert offset + n <= self.size
        return CuArray(self.device, shape, self.dtype, ptr=self.ptr.value + offset * self.itemsize, owner=self)

    def copy_from(self, array: np.ndarray) -> None:
        """H2D (`from_ndarray`, cuarray.rs:114-116).  f32 host data is rounded to bf16 for bf16 arrays."""
        a = np.ascontiguousarray(array, dtype=np.float32)
        assert a.size == self.size, (a.shape, self.shape)
        host = L.f32_to_bf16_bits(a) if self.dtype == BF16 else a
        L.check(L.lib.nk_h2d(self.device.ctx, self.ptr, host.ctypes.data_as(C.c_void_p), self.nbytes), self.device.ctx)
        self.device.synchronize()  # host buffer may be a temporary

    def as_ndarray(self) -> np.ndarray:
        """D2H copy as float32 (`as_ndarray`, cuarray.rs:101-105)."""
        host = np.empty(self.size, dtype=np.uint16 if self.dtype == BF16 else np.float32)
        L.check(L.lib.nk_d2h(self.device.ctx, host.ctypes.data_as(C.c_void_p), self.ptr, self.nbytes), self.device.ctx)
        out = L.bf16_bits_to_f32(host) if self.dtype == BF16 else host
        return out.reshape(self.shape)

    def zero_(self) -> None:
        L.check(L.lib.nk_memset0(self.device.ctx, self.ptr, self.nbytes), self.device.ctx)

    def fill_(self, value: float) -> None:
        L.check(L.lib.nk_fill(self.device.ctx, self.ptr, self.dtype, self.size, float(value)), self.device.ctx)

    def astype(self, dtype) -> "CuArray":
        out = CuArray(self.device, self.shape, dtype)
        L.check(L.lib.nk_cast(self.device.ctx, out.ptr, out.dtype, self.ptr, self.dtype, self.size), self.device.ctx)
        return out

    def cuda_array_interface(self) -> dict:
        """For wrapping as a torch tensor (f32 -> float32, bf16 -> viewed as int16)."""
        return {"shape": self.shape, "typestr": "<f4" if self.dtype == F32 else "<i2",
                "data": (self.ptr.value, False), "version": 2}

    def __repr__(self) -> str:
        return f"CuArray(shape={self.shape}, dtype={_DT_NAME[self.dtype]}, device={self.device.index})"
