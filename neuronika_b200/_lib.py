"""ctypes binding of libnk_b200.so (the C ABI declared in include/nk_b200.h).

The library is the product: if it cannot be loaded this module raises -- there is no CPU
fallback anywhere in the package.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnk_b200.so")

NK_F32, NK_BF16 = 0, 1
NK_GEMM_AUTO, NK_GEMM_SIMT, NK_GEMM_TC = 0, 1, 2
NK_BIN_ADD, NK_BIN_SUB, NK_BIN_MUL, NK_BIN_DIV = 0, 1, 2, 3
(NK_UN_NEG, NK_UN_EXP, NK_UN_LN, NK_UN_SQRT, NK_UN_SIGMOID, NK_UN_TANH, NK_UN_SOFTPLUS, NK_UN_LEAKY_RELU,
 NK_UN_POWI) = range(9)
NK_PAD_CONSTANT, NK_PAD_REFLECTIVE, NK_PAD_REPLICATIVE = 0, 1, 2
NK_OPTIM_TENSORS_PER_LAUNCH = 64
NK_OPTIM_ADAM, NK_OPTIM_ADAGRAD = 0, 1
NK_LR_STEP, NK_LR_MULTI_STEP, NK_LR_EXPONENTIAL, NK_LR_MULTIPLICATIVE, NK_LR_LAMBDA = range(5)
NK_OK = 0
NK_ERR = {-1: "NK_ERR_INVALID_ARG", -2: "NK_ERR_CUDA", -3: "NK_ERR_NCCL", -4: "NK_ERR_OOM",
          -5: "NK_ERR_UNSUPPORTED"}


class NkError(RuntimeError):
    """Raised for every non-zero status (the Rust wrapper `.unwrap()`s, the reference panics)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"{NK_ERR.get(code, code)}: {message}")
        self.code = code
        self.message = message


class OptimHyper(C.Structure):
    """nk_optim_hyper: the device-resident lr and step count of an optimizer"""
    _fields_ = [("lr", C.c_float), ("step_size", C.c_float), ("sqrt_bc2", C.c_float), ("clr", C.c_float),
                ("step", C.c_int64)]


class LrSched(C.Structure):
    """nk_lr_sched: the device-resident state of a learning-rate scheduler"""
    _fields_ = [("epoch", C.c_int64), ("step_size", C.c_int64), ("table", C.c_void_p), ("table_len", C.c_int64),
                ("gamma", C.c_float), ("initial_lr", C.c_float), ("last_lr", C.c_float), ("current_lr", C.c_float),
                ("kind", C.c_int32), ("past_horizon", C.c_int32)]


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(or `make -C neuronika_b200/csrc`).  neuronika_b200 has no CPU fallback.")

lib = C.CDLL(LIB_PATH)

vp, i64, i32, f32, sz, u64 = C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_size_t, C.c_uint64
pi64 = C.POINTER(C.c_int64)
pvp = C.POINTER(C.c_void_p)

_PROTOS = {
    "nk_ctx_create": (i32, [i32, C.POINTER(vp)]),
    "nk_ctx_destroy": (i32, [vp]),
    "nk_ctx_set_stream": (i32, [vp, vp]),
    "nk_ctx_stream": (vp, [vp]),
    "nk_last_error": (C.c_char_p, [vp]),
    "nk_version": (C.c_char_p, []),
    "nk_sync": (i32, [vp]),
    "nk_launch_count": (u64, [vp]),
    "nk_sm_count": (i32, [vp]),
    "nk_gemm_config": (i32, [vp, i32]),
    "nk_gemm_f32_config": (i32, [vp, i32]),
    "nk_conv_config": (i32, [vp, i32]),
    "nk_conv_f32_config": (i32, [vp, i32]),
    "nk_last_gemm_kernel": (C.c_char_p, [vp]),
    "nk_last_conv_kernel": (C.c_char_p, [vp]),
    "nk_alloc": (i32, [vp, sz, C.POINTER(vp)]),
    "nk_alloc_uninit": (i32, [vp, sz, C.POINTER(vp)]),
    "nk_free": (i32, [vp, vp]),
    "nk_h2d": (i32, [vp, vp, vp, sz]),
    "nk_d2h": (i32, [vp, vp, vp, sz]),
    "nk_d2d": (i32, [vp, vp, vp, sz]),
    "nk_memset0": (i32, [vp, vp, sz]),
    "nk_host_alloc": (i32, [vp, sz, C.POINTER(vp)]),
    "nk_host_free": (i32, [vp, vp]),
    "nk_fill": (i32, [vp, vp, i32, sz, f32]),
    "nk_cast": (i32, [vp, vp, i32, vp, i32, sz]),
    "nk_capture_begin": (i32, [vp, sz]),
    "nk_capture_end": (i32, [vp, C.POINTER(vp)]),
    "nk_graph_launch": (i32, [vp, vp]),
    "nk_graph_destroy": (i32, [vp, vp]),
    "nk_graph_kernel_count": (i64, [vp]),
    "nk_graph_arena_used": (sz, [vp]),
    "nk_timer_start": (i32, [vp]),
    "nk_timer_stop": (i32, [vp, C.POINTER(f32)]),
    "nk_gemm": (i32, [vp, i32, i32, i64, i64, i64, f32, vp, i64, vp, i64, f32, vp, i64, i32, i32]),
    "nk_gemm_bias_act": (i32, [vp, i32, i32, i64, i64, i64, f32, vp, i64, vp, i64, f32, vp, i64, i32, i32,
                               vp, i32, i32]),
    "nk_gemm_strided_batched": (i32, [vp, i32, i32, i64, i64, i64, f32, vp, i64, i64, vp, i64, i64, f32, vp, i64, i64,
                                      i64, i32, i32, vp, i64, i32]),
    "nk_gemm_relu_bwd": (i32, [vp, i32, i32, i64, i64, i64, vp, i64, vp, i64, f32, vp, i64, i32, i32, vp]),
    "nk_gemm_relu_bwd_colsum": (i32, [vp, i32, i32, i64, i64, i64, vp, i64, vp, i64, f32, vp, i64, i32, i32, vp, vp]),
    "nk_add_bcast_fwd": (i32, [vp, vp, vp, vp, i32, i32, pi64, i32, pi64, i32, pi64]),
    "nk_unbroadcast_acc": (i32, [vp, vp, i32, i32, pi64, vp, i32, i32, pi64, f32]),
    "nk_relu_fwd": (i32, [vp, vp, vp, sz, i32]),
    "nk_relu_bwd": (i32, [vp, vp, vp, vp, sz, i32, f32]),
    "nk_softmax_fwd": (i32, [vp, vp, vp, i64, i64, i64, i32]),
    "nk_softmax_bwd": (i32, [vp, vp, vp, vp, i64, i64, i64, i32, f32]),
    "nk_log_softmax_fwd": (i32, [vp, vp, vp, i64, i64, i64, i32]),
    "nk_log_softmax_bwd": (i32, [vp, vp, vp, vp, i64, i64, i64, i32, f32]),
    "nk_mse_fwd": (i32, [vp, vp, vp, vp, sz, i32, i32]),
    "nk_mse_bwd": (i32, [vp, vp, vp, vp, vp, sz, i32, i32, f32]),
    "nk_nll_fwd": (i32, [vp, vp, vp, vp, i32, i64, i64, i32, i32]),
    "nk_nll_bwd": (i32, [vp, vp, vp, i32, vp, i64, i64, i32, i32, f32]),
    "nk_sum_fwd": (i32, [vp, vp, vp, sz, i32, i32]),
    "nk_sum_bwd": (i32, [vp, vp, vp, sz, i32, i32, f32]),
    "nk_pad2d_fwd": (i32, [vp, vp, vp, i64, i64, i64, i64, i64, f32, i32]),
    "nk_pad2d_bwd": (i32, [vp, vp, vp, i64, i64, i64, i64, i64, i32, f32]),
    "nk_conv2d_fwd": (i32, [vp, vp, vp, vp, vp, i32] + [i64] * 12 + [i32]),
    "nk_conv2d_bwd_input": (i32, [vp, vp, vp, vp] + [i64] * 12 + [i32, f32]),
    "nk_conv2d_bwd_kernel": (i32, [vp, vp, i32, vp, vp, vp] + [i64] * 12 + [i32, f32]),
    "nk_ipc_alloc": (i32, [vp, sz, pvp]),
    "nk_ipc_free": (i32, [vp, vp]),
    "nk_ipc_export": (i32, [vp, vp, vp]),
    "nk_ipc_open": (i32, [vp, vp, pvp]),
    "nk_ipc_close": (i32, [vp, vp]),
    "nk_peer_barrier": (i32, [vp, pvp, i32, i32, C.c_uint32]),
    "nk_gemm_rs": (i32, [vp, i32, i32, i64, i64, i64, f32, vp, i64, vp, i64, pvp, i32, i32, i32]),
    "nk_reduce_bcast": (i32, [vp, vp, pvp, i32, i32, i64, i32]),
    "nk_reduce_exchange": (i32, [vp, vp, pvp, pvp, i32, i32, i64, vp, i32]),
    "nk_peer_allreduce_small": (i32, [vp, vp, pvp, pvp, i32, i32, i64, vp]),
    "nk_binary_bcast_fwd": (i32, [vp, i32, vp, vp, vp, i32, i32, pi64, i32, pi64, i32, pi64]),
    "nk_binary_bcast_bwd": (i32, [vp, i32, i32, vp, i32, vp, vp, vp, i32, i32, pi64, i32, pi64, f32]),
    "nk_unary_fwd": (i32, [vp, i32, vp, vp, sz, i32, i32]),
    "nk_unary_bwd": (i32, [vp, i32, vp, vp, vp, sz, i32, i32, f32]),
    "nk_transpose": (i32, [vp, vp, i32, vp, i32, i32, pi64, f32]),
    "nk_padnd_fwd": (i32, [vp, vp, vp, i64, i32, pi64, pi64, i32, f32, i32]),
    "nk_padnd_bwd": (i32, [vp, vp, vp, i64, i32, pi64, pi64, i32, f32]),
    "nk_max_pool_nd_fwd": (i32, [vp, vp, vp, vp, i64, i32, pi64, pi64, pi64, pi64, pi64, pi64, i32]),
    "nk_max_pool_nd_bwd": (i32, [vp, vp, i32, vp, i32, vp, i64, i32, pi64, pi64, pi64, pi64, pi64, pi64, f32]),
    "nk_avg_pool_nd_fwd": (i32, [vp, vp, vp, i64, i32, pi64, pi64, pi64, pi64, pi64, i32, i32]),
    "nk_avg_pool_nd_bwd": (i32, [vp, vp, i32, vp, i32, i64, i32, pi64, pi64, pi64, pi64, pi64, i32, f32]),
    "nk_adaptive_avg_pool_nd_fwd": (i32, [vp, vp, vp, i64, i32, pi64, pi64, i32]),
    "nk_adaptive_avg_pool_nd_bwd": (i32, [vp, vp, i32, vp, i32, i64, i32, pi64, pi64, f32]),
    "nk_batch_norm_fwd": (i32, [vp, vp, vp, i32, i64, i64, i64, vp, vp, vp, vp, vp, vp, i32, f32, f32]),
    "nk_batch_norm_bwd": (i32, [vp, vp, i32, f32, vp, i32, f32, vp, i32, f32, vp, i32, vp, i32, i64, i64, i64, vp, vp,
                                vp, i32]),
    "nk_layer_norm_fwd": (i32, [vp, vp, vp, i32, i64, i64, vp, vp, vp, vp, f32]),
    "nk_layer_norm_bwd": (i32, [vp, vp, i32, f32, vp, i32, f32, vp, i32, f32, vp, i32, vp, i32, i64, i64, vp, vp, vp]),
    "nk_embedding_fwd": (i32, [vp, vp, vp, vp, i32, i64, i64, i64, i32]),
    "nk_embedding_bwd": (i32, [vp, vp, i32, vp, i32, vp, i32, i64, i64, i64, i64, f32]),
    "nk_cross_entropy_fwd": (i32, [vp, vp, vp, vp, vp, i32, vp, i32, vp, i64, i64, i64, i64, f32, i32]),
    "nk_cross_entropy_bwd": (i32, [vp, vp, i32, vp, i32, vp, i32, vp, vp, vp, vp, i64, i64, i64, i64, f32, i32, f32]),
    "nk_gemv": (i32, [vp, i32, i64, i64, vp, vp, f32, vp, i32, i32]),
    "nk_outer_acc": (i32, [vp, vp, i32, vp, vp, i64, i64, i32, f32]),
    "nk_dot": (i32, [vp, vp, vp, vp, sz, i32]),
    "nk_scale_acc": (i32, [vp, vp, i32, vp, i32, vp, sz, f32]),
    "nk_convnd_fwd": (i32, [vp, vp, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, i64, i32]),
    "nk_convnd_bwd_input": (i32, [vp, vp, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, i64, i32, f32]),
    "nk_convnd_bwd_kernel": (i32, [vp, vp, i32, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, i64, i32, f32]),
    "nk_conv_layer_nd_fwd": (i32, [vp, vp, vp, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, pi64, i32, f32, i32]),
    "nk_conv_layer_nd_bwd_input": (i32, [vp, vp, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, pi64, i32, i32, f32]),
    "nk_conv_layer_nd_bwd_kernel": (i32, [vp, vp, i32, vp, vp, vp, i32, i64, i64, pi64, i64, pi64, pi64, pi64, pi64, i32,
                                          f32, i32, f32]),
    "nk_optim_hyper_set": (i32, [vp, vp, vp]),
    "nk_optim_hyper_get": (i32, [vp, vp, vp]),
    "nk_optim_prologue": (i32, [vp, vp, i32, f32, f32, f32]),
    "nk_multi_sgd_step": (i32, [vp, i32, pvp, pvp, i32, i32, pvp, pvp, pi64, vp, f32, f32, f32, i32, f32, i32]),
    "nk_multi_adam_step": (i32, [vp, i32, pvp, pvp, i32, i32, pvp, pvp, pvp, pvp, pi64, vp, f32, f32, f32, f32, f32, f32,
                                 i32]),
    "nk_multi_rmsprop_step": (i32, [vp, i32, pvp, pvp, i32, i32, pvp, pvp, pvp, pvp, pi64, vp, f32, f32, f32, f32, f32,
                                    f32, i32]),
    "nk_multi_adagrad_step": (i32, [vp, i32, pvp, pvp, i32, i32, pvp, pvp, pi64, vp, f32, f32, f32, f32, i32]),
    "nk_lr_sched_set": (i32, [vp, vp, vp]),
    "nk_lr_sched_get": (i32, [vp, vp, vp]),
    "nk_lr_sched_step": (i32, [vp, vp, vp]),
    "nk_grad_norm": (i32, [vp, i32, pvp, C.POINTER(i32), pi64, f32, f32, vp]),
    "nk_grad_scale_by_norm": (i32, [vp, i32, pvp, C.POINTER(i32), pi64, vp, f32]),
    "nk_grad_clamp": (i32, [vp, i32, pvp, C.POINTER(i32), pi64, f32, f32]),
    "nk_comm_unique_id": (i32, [vp, vp]),
    "nk_comm_init_rank": (i32, [vp, i32, i32, vp]),
    "nk_comm_destroy": (i32, [vp]),
    "nk_comm_world": (i32, [vp]),
    "nk_comm_rank": (i32, [vp]),
    "nk_allreduce_sum": (i32, [vp, vp, sz, i32]),
    "nk_lstm_cell_fwd": (i32, [vp, vp, vp, vp, vp, i64, i64, i32]),
    "nk_lstm_cell_bwd": (i32, [vp, vp, i32, vp, f32, vp, vp, vp, vp, i64, i64, i32]),
    "nk_gru_cell_fwd": (i32, [vp, vp, vp, vp, vp, i64, i64, i32]),
    "nk_gru_cell_bwd": (i32, [vp, vp, vp, i32, vp, f32, vp, vp, vp, vp, i64, i64, i32]),
    "nk_lstm_seq_bwd_step": (i32, [vp, vp, i32, vp, vp, vp, vp, vp, i64, i64, i32]),
    "nk_gru_seq_bwd_step": (i32, [vp, vp, vp, i32, vp, vp, vp, vp, vp, i64, i64, i32]),
    "nk_lstm_bidir_fwd_step": (i32, [vp, vp, i64, i64, vp, vp, i64, vp, i64, vp, i64, i64, i64, i32]),
    "nk_gru_bidir_fwd_step": (i32, [vp, vp, i64, i64, vp, vp, vp, i64, vp, i64, i64, i64, i32]),
    "nk_lstm_bidir_bwd_step": (i32, [vp, vp, i32, i64, vp, vp, vp, i64, vp, i64, i64, vp, i64, i64, i32]),
    "nk_gru_bidir_bwd_step": (i32, [vp, vp, vp, i32, i64, vp, vp, vp, vp, i64, i64, vp, i64, i64, i64, i64, i32]),
    "nk_chunk_fwd": (i32, [vp, vp, vp, i32, pi64, pi64, i64, i32]),
    "nk_chunk_bwd": (i32, [vp, vp, i32, vp, i32, i32, pi64, pi64, i64, f32]),
    "nk_cat_fwd": (i32, [vp, vp, pvp, pi64, i32, i64, i64, i32]),
    "nk_cat_bwd": (i32, [vp, pvp, C.POINTER(i32), C.POINTER(f32), vp, i32, pi64, i32, i64, i64]),
    "nk_mae_fwd": (i32, [vp, vp, vp, vp, sz, i32, i32]),
    "nk_mae_bwd": (i32, [vp, vp, i32, vp, vp, vp, sz, i32, i32, f32]),
    "nk_bce_fwd": (i32, [vp, vp, vp, vp, sz, i32, i32]),
    "nk_bce_bwd": (i32, [vp, vp, i32, vp, vp, vp, sz, i32, i32, f32]),
    "nk_bce_with_logits_fwd": (i32, [vp, vp, vp, vp, sz, i32, i32]),
    "nk_bce_with_logits_bwd": (i32, [vp, vp, i32, vp, vp, vp, sz, i32, i32, f32]),
    "nk_kldiv_fwd": (i32, [vp, vp, vp, vp, sz, i64, i32, i32]),
    "nk_kldiv_bwd": (i32, [vp, vp, i32, vp, vp, sz, i64, i32, i32, f32]),
    "nk_dropout_fwd": (i32, [vp, vp, vp, vp, sz, i32, C.c_double]),
    "nk_dropout_bwd": (i32, [vp, vp, i32, vp, vp, sz, i32, C.c_double, f32]),
    "nk_rng_seed": (i32, [vp, u64]),
    "nk_rng_state": (i32, [vp, C.POINTER(u64), C.POINTER(u64)]),
}

for _name, (_res, _args) in _PROTOS.items():
    _fn = getattr(lib, _name)  # AttributeError here = the .so does not export a declared symbol
    _fn.restype = _res
    _fn.argtypes = _args


def exported_symbols():
    """Names this binding declares (tests compare them with include/nk_b200.h)."""
    return sorted(_PROTOS)


def last_error(ctx) -> str:
    msg = lib.nk_last_error(ctx)
    return msg.decode() if msg else ""


def check(rc: int, ctx=None) -> None:
    if rc != NK_OK:
        raise NkError(rc, last_error(ctx))


def shape_arr(shape):
    return (C.c_int64 * max(1, len(shape)))(*[int(s) for s in shape])


# ---- host-side element-format conversion (data marshalling, not compute) -------------------
def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit patterns (uint16), round-to-nearest-even."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    bits = x.view(np.uint32).astype(np.uint64)
    bias = ((bits >> 16) & 1) + 0x7FFF
    out = ((bits + bias) >> 16).astype(np.uint16)
    if np.any(np.isnan(x)):   # the rounding carry would turn a NaN with a high mantissa into +-0 / inf: keep it a quiet NaN
        out = np.where(np.isnan(x), ((x.view(np.uint32) >> 16) | 0x0040).astype(np.uint16), out.reshape(x.shape))
    return out.reshape(x.shape)


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    b = np.ascontiguousarray(b, dtype=np.uint16)
    return (b.astype(np.uint32) << 16).view(np.float32).reshape(b.shape)
