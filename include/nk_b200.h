/*
 * nk_b200.h -- C ABI of the H100-native (sm_90a) dense forward/backward hot path of neuronika.
 *
 * This is the drop-in boundary (SURVEY.md section 8-b): one C function per
 * (operator, direction), taking device pointers and sizes, launched asynchronously on
 * the context's CUDA stream.  A Rust `Forward`/`Backward` node (reference trait objects,
 * neuronika-variable/src/autograd.rs:7-12, 20-25) keeps `Shared<CuArray>` handles exactly
 * like the reference's only device node does (cuda/cunode/binary_op/mod.rs:11-82) and
 * calls one of these functions from `forward()` / `backward()`.
 *
 * Conventions
 *   - every function returns 0 (NK_OK) or a negative nk_status; the message is available
 *     through nk_last_error().  Nothing aborts or throws across the ABI (the reference
 *     `.unwrap()`s every CUDA result, cuda/device.rs:36-45; the Rust wrapper does the same
 *     on our status codes).
 *   - all tensors are dense, C-order (row-major); images are NCHW (reference layout).
 *   - `beta` on a backward entry point selects the reference's accumulate protocol:
 *     beta = 1 -> `grad += ...` (what every reference Backward node does), beta = 0 ->
 *     overwrite (used by the host for a gradient buffer that is known to be all-zero,
 *     which gives identical results without the read).
 *   - element types: NK_F32 (reference type) and NK_BF16 (tensor-core operand type).
 *   - a context is single-threaded (like the reference's Rc graph, utils.rs:9); use one
 *     context per host thread / per GPU.
 *   - there is NO CPU fallback: every entry point fails with NK_ERR_CUDA when no device
 *     is present.
 */
#ifndef NK_B200_H
#define NK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nk_ctx nk_ctx;

typedef enum {
  NK_OK = 0,
  NK_ERR_INVALID_ARG = -1,
  NK_ERR_CUDA = -2,
  NK_ERR_NCCL = -3,
  NK_ERR_OOM = -4,
  NK_ERR_UNSUPPORTED = -5
} nk_status;

typedef enum { NK_F32 = 0, NK_BF16 = 1 } nk_dtype;

/* GEMM engine selection (nk_gemm_config): AUTO picks the wgmma tensor-core engine
 * whenever the operands are bf16 and TMA-addressable, else the SIMT kernel. */
typedef enum { NK_GEMM_AUTO = 0, NK_GEMM_SIMT = 1, NK_GEMM_TC = 2, NK_GEMM_TCGEN05 = NK_GEMM_TC /* former name */ } nk_gemm_engine;
/* How f32 products use the tensor cores (nk_gemm_f32_config).  IEEE (the default): f32 operands run on the CUDA cores,
 * as they always did.  TF32: every operand element is rounded to TF32 (cvt.rna: to nearest, ties away from zero) and the
 * product runs on the wgmma engine with f32 accumulation.  TF32X3: each element x is split into hi = tf32(x) and
 * lo = tf32(x - hi), and C = A_hi.B_hi + A_hi.B_lo + A_lo.B_hi (the lo.lo term, ~2^-22 of each product, is dropped):
 * close to f32 accuracy, at about a fifth of the TF32 rate (README).  The mode is read when a GEMM is called; a captured step keeps the
 * mode it was captured with. */
typedef enum { NK_F32_GEMM_IEEE = 0, NK_F32_GEMM_TF32 = 1, NK_F32_GEMM_TF32X3 = 2 } nk_f32_gemm_mode;
/* Convolution engine selection (nk_conv_config): AUTO = tensor-core kernels wherever they apply; DIRECT = the CUDA-core
 * kernels only (the parity path the reference's goldens run on), in every f32 convolution mode.  f32 convolutions stay on
 * the CUDA cores under AUTO too unless nk_conv_f32_config opts them into TF32 / 3xTF32; grouped (groups > 1) ones stay
 * there in every mode. */
typedef enum { NK_CONV_AUTO = 0, NK_CONV_DIRECT = 1 } nk_conv_engine;

/* ---- context (replaces cuda::Device, neuronika-variable/src/cuda/device.rs:11-75) ---- */
int nk_ctx_create(int device, nk_ctx** out);
int nk_ctx_destroy(nk_ctx* ctx);
/* adopt an external cudaStream_t (e.g. torch's) so events / NCCL order with our kernels */
int nk_ctx_set_stream(nk_ctx* ctx, void* cuda_stream);
void* nk_ctx_stream(nk_ctx* ctx);
const char* nk_last_error(nk_ctx* ctx);
const char* nk_version(void);
int nk_sync(nk_ctx* ctx);
/* number of kernels this library launched on ctx since creation */
uint64_t nk_launch_count(nk_ctx* ctx);
int nk_sm_count(nk_ctx* ctx);
int nk_gemm_config(nk_ctx* ctx, int engine /* nk_gemm_engine */);
int nk_conv_config(nk_ctx* ctx, int engine /* nk_conv_engine */);
/* f32 products of nk_gemm / nk_gemm_bias_act / nk_gemm_strided_batched / nk_gemm_relu_bwd (and every graph node built on
 * them) in `mode` (nk_f32_gemm_mode).  The GEMM engine setting wins: NK_GEMM_SIMT keeps every product on the CUDA cores.
 * Errors: NK_ERR_INVALID_ARG for an unknown mode. */
int nk_gemm_f32_config(nk_ctx* ctx, int mode /* nk_f32_gemm_mode */);
/* f32, groups = 1 convolutions of nk_conv2d_* / nk_convnd_* / nk_conv_layer_nd_* (and every graph node built on them) in
 * `mode` (nk_f32_gemm_mode values), separately from nk_gemm_f32_config.  IEEE (the default): the CUDA-core kernels, as
 * always.  TF32 / TF32X3: im2col + the TF32 / 3xTF32 wgmma GEMM for every such call with a non-empty batch, whatever its
 * shape, with x (fill values included), w and g rounded as nk_gemm_f32_config describes; nk_last_conv_kernel names it
 * "tf32_im2col_*" / "tf32x3_im2col_*" (2-D) or "tf32_im2col_nd_*" / "tf32x3_im2col_nd_*" (1-D / 3-D).
 * nk_conv_config(DIRECT) wins.  The mode is read when a convolution is called; a captured step keeps the mode it was
 * captured with.  Errors: NK_ERR_INVALID_ARG for an unknown mode. */
int nk_conv_f32_config(nk_ctx* ctx, int mode /* nk_f32_gemm_mode */);
/* name of the kernel variant the last nk_gemm call used ("wgmma_nt_128x256", "simt", ...) */
const char* nk_last_gemm_kernel(nk_ctx* ctx);

/* ---- buffers (replaces cuda::CuArray, cuda/cuarray.rs:10-171) ---- */
int nk_alloc(nk_ctx* ctx, size_t bytes, void** dptr);      /* zero-filled, like CuArray::zeroed :35 */
int nk_alloc_uninit(nk_ctx* ctx, size_t bytes, void** dptr); /* for buffers the next kernel fully overwrites */
int nk_free(nk_ctx* ctx, void* dptr);
int nk_h2d(nk_ctx* ctx, void* dst, const void* src, size_t bytes);   /* from_ndarray :114 */
int nk_d2h(nk_ctx* ctx, void* dst, const void* src, size_t bytes);   /* as_ndarray :101 (blocks) */
int nk_d2d(nk_ctx* ctx, void* dst, const void* src, size_t bytes);
int nk_memset0(nk_ctx* ctx, void* dptr, size_t bytes);
int nk_host_alloc(nk_ctx* ctx, size_t bytes, void** hptr);           /* pinned host memory */
int nk_host_free(nk_ctx* ctx, void* hptr);
int nk_fill(nk_ctx* ctx, void* dptr, int dtype, size_t n, float value);
int nk_cast(nk_ctx* ctx, void* dst, int dst_dtype, const void* src, int src_dtype, size_t n);
/* ---- whole-step capture.  A training step launches the same kernels every iteration (the reference rebuilds the
 * same define-by-run graph each time, examples/quickstart.rs:216-227), so the step can be recorded once and replayed
 * with one driver call: between nk_capture_begin and nk_capture_end every kernel / copy / memset this library
 * enqueues on the context stream -- and on streams that join it through events, e.g. the exchange side stream -- is
 * recorded into a CUDA graph instead of running.  While capturing, nk_alloc / nk_alloc_uninit take memory from an
 * arena of `arena_bytes` owned by the graph (fixed addresses on every replay; blocks freed inside the capture are
 * recycled) and nk_free of arena memory is a no-op for as long as the graph lives.  Things that cannot be captured
 * (nk_d2h, nk_sync, growth of the scratch workspace) fail: run the step once eagerly first.  nk_graph_launch replays
 * the step on the context stream; results are in the same buffers every time. */
typedef struct nk_graph nk_graph;
int nk_capture_begin(nk_ctx* ctx, size_t arena_bytes);
int nk_capture_end(nk_ctx* ctx, nk_graph** out);
int nk_graph_launch(nk_ctx* ctx, nk_graph* graph);
int nk_graph_destroy(nk_ctx* ctx, nk_graph* graph);
int64_t nk_graph_kernel_count(nk_graph* graph);   /* kernel nodes per replay (counted into nk_launch_count) */
size_t nk_graph_arena_used(nk_graph* graph);
/* CUDA-event stopwatch on the context stream */
int nk_timer_start(nk_ctx* ctx);
int nk_timer_stop(nk_ctx* ctx, float* ms);

/* ---- matrix multiply: C = alpha * op(A) . op(B) + beta * C  (row-major, like ndarray's
 * general_mat_mul call sites: matrix_matrix_mul/mod.rs:33,65,97; matrix_matrix_mul_t/mod.rs:33,65,97)
 *   op(A) is M x K: transA=0 -> A stored (M,K) lda>=K ; transA=1 -> A stored (K,M) lda>=M
 *   op(B) is K x N: transB=0 -> B stored (K,N) ldb>=N ; transB=1 -> B stored (N,K) ldb>=K
 *   mm fwd: NN; mm dA: NT; mm dB: TN; mm_t fwd: NT; mm_t dX: NN; mm_t dW: TN.
 *   Optional fused epilogue: + bias[N] (row broadcast, Linear fwd) and ReLU. */
int nk_gemm(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
            const void* A, int64_t lda, const void* B, int64_t ldb, float beta, void* C,
            int64_t ldc, int ab_dtype, int c_dtype);
int nk_gemm_bias_act(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K,
                     float alpha, const void* A, int64_t lda, const void* B, int64_t ldb,
                     float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype,
                     const void* bias /* N elements, c_dtype or f32 */, int bias_dtype,
                     int relu);
/* `batch` independent products C_b = alpha * op(A_b).op(B_b) + beta*C_b + bias_b, where X_b = X + b*strideX elements and
 * bias_b (N elements, column-indexed, or NULL) = bias + b*bias_stride.  bf16 operands that TMA can address (16-byte
 * aligned bases, leading dimensions and operand strides multiples of 8 elements, strides >= 0, every C_b 16-byte
 * aligned; not TT) run as ONE launch of the batched wgmma kernel; anything else as one nk_gemm_bias_act per product. */
int nk_gemm_strided_batched(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
                            const void* A, int64_t lda, int64_t strideA, const void* B, int64_t ldb, int64_t strideB,
                            float beta, void* C, int64_t ldc, int64_t strideC, int64_t batch, int ab_dtype, int c_dtype,
                            const void* bias, int64_t bias_stride, int bias_dtype);

/* C = beta*C + relu'(relu_operand) (.) (op(A).op(B)): the input gradient of a matmul whose left operand is the output
 * of a ReLU, with that ReLU's backward (relu/mod.rs:71-78: dx += (x > 0) * g) applied in the GEMM epilogue instead of a
 * separate pass over the (M, N) gradient.  relu_operand is (M, N) with C's element type and leading dimension; either
 * the ReLU's input or its output (y = max(x, 0) > 0  <=>  x > 0). */
int nk_gemm_relu_bwd(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A,
                     int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype,
                     int c_dtype, const void* relu_operand);
/* The same with beta = 0 and, in the same epilogue, colsum[n] += sum_m C[m][n] (N floats, f32 atomics; the caller zeroes or
 * keeps them): the bias gradient of the layer below -- the un-broadcast of its Addition's right operand,
 * addition/mod.rs:81-135 -- without a separate pass over the (M, N) gradient.  The sums are those of the values as stored
 * (after rounding to C's element type).  NK_ERR_UNSUPPORTED (nothing done) where no engine has the fused epilogue.
 * The graph uses it at fusion level 3 (nkg_set_fusion); measured equal to the separate column-sum pass at config 4. */
int nk_gemm_relu_bwd_colsum(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A,
                            int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype,
                            int c_dtype, const void* relu_operand, float* colsum);

/* ---- broadcasting add (addition/mod.rs:39-50, 81-135; utils.rs:97-125, 152-192) ----
 * shapes are right-aligned, up to NK_MAX_DIMS dims. */
#define NK_MAX_DIMS 6
int nk_add_bcast_fwd(nk_ctx* ctx, void* y, const void* l, const void* r, int dtype,
                     int y_ndim, const int64_t* y_shape, int l_ndim, const int64_t* l_shape,
                     int r_ndim, const int64_t* r_shape);
/* dst = beta*dst + unbroadcast(g -> dst_shape); an empty g leaves dst = beta*dst (g may then be NULL) */
int nk_unbroadcast_acc(nk_ctx* ctx, void* dst, int dst_dtype, int dst_ndim,
                       const int64_t* dst_shape, const void* g, int g_dtype, int g_ndim,
                       const int64_t* g_shape, float beta);

/* ---- relu (relu/mod.rs:29-38, 67-79) ---- */
int nk_relu_fwd(nk_ctx* ctx, void* y, const void* x, size_t n, int dtype);
int nk_relu_bwd(nk_ctx* ctx, void* dx, const void* x, const void* g, size_t n, int dtype, float beta);

/* ---- softmax / log-softmax along one axis of an (outer, len, inner) view
 * (softmax/mod.rs:37-53, 84-104; logsoftmax/mod.rs:37-53, 84-102) ---- */
int nk_softmax_fwd(nk_ctx* ctx, void* y, const void* x, int64_t outer, int64_t len, int64_t inner, int dtype);
int nk_softmax_bwd(nk_ctx* ctx, void* dx, const void* y, const void* g, int64_t outer, int64_t len,
                   int64_t inner, int dtype, float beta);
int nk_log_softmax_fwd(nk_ctx* ctx, void* y, const void* x, int64_t outer, int64_t len, int64_t inner, int dtype);
int nk_log_softmax_bwd(nk_ctx* ctx, void* dx, const void* y, const void* g, int64_t outer, int64_t len,
                       int64_t inner, int dtype, float beta);

/* ---- losses and scalar reductions; scalar outputs / seeds are device f32 ----
 * (squared_error/mod.rs:46-58, 98-122; nll/mod.rs:42-68, 100-133; sum/mod.rs, mean/mod.rs) */
int nk_mse_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean);
int nk_mse_bwd(nk_ctx* ctx, void* dx, const void* x, const void* t, const float* g, size_t n,
               int dtype, int mean, float beta);
/* NLL: `target` holds the class ids as floats (`target as usize`, nll/mod.rs:55) in element type
 * target_dtype -- NK_F32 whatever the input's type, or NK_BF16 (exact only for ids <= 256, so
 * rejected when c > 256). */
int nk_nll_fwd(nk_ctx* ctx, float* loss, const void* logp, const void* target, int target_dtype,
               int64_t n, int64_t c, int dtype, int mean);
int nk_nll_bwd(nk_ctx* ctx, void* dlogp, const void* target, int target_dtype, const float* g,
               int64_t n, int64_t c, int dtype, int mean, float beta);
int nk_sum_fwd(nk_ctx* ctx, float* out, const void* x, size_t n, int dtype, int mean);
int nk_sum_bwd(nk_ctx* ctx, void* dx, const float* g, size_t n, int dtype, int mean, float beta);

/* ---- the other criteria (csrc/nk_criteria.cu): absolute_error/mod.rs, bce/mod.rs, bce_with_logits/mod.rs,
 * kldiv/mod.rs.  x and t share the element type `dtype`; the loss is a device f32 scalar; the backward writes
 * dx = beta*dx + dloss/dx * (*g) in its own element type dx_dtype (f32 gradients of bf16 data).  The forward sums in a
 * fixed order (f32 partials carried into double, one block summing the per-block partials), so repeated calls are
 * bitwise equal.  mean divides by n for mae / bce / bce_with_logits and by `batch` (x's leading dimension) for kldiv --
 * the reference's batch mean, torch's reduction='batchmean', not torch's 'mean'.
 *   mae              |x - t|                                          dx: sign(x - t) * g, 0 where x == t
 *   bce              -t*max(ln x, -100) + (t - 1)*max(ln(1 - x), -100)  dx: (x - t) / max((1 - x)*x, FLT_EPSILON) * g
 *   bce_with_logits  (1 - t)*x + m + ln(e^-m + e^(-x-m)), m = max(-x, 0)  dx: (sigmoid(x) - t) * g
 *   kldiv            t*(ln t - x) where t > 0, else 0 (x = log-probabilities)   dx: -t * g */
int nk_mae_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean);
int nk_mae_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n, int dtype,
               int mean, float beta);
int nk_bce_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean);
int nk_bce_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n, int dtype,
               int mean, float beta);
int nk_bce_with_logits_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean);
int nk_bce_with_logits_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n,
                           int dtype, int mean, float beta);
int nk_kldiv_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int64_t batch, int dtype, int mean);
int nk_kldiv_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* t, const float* g, size_t n, int64_t batch, int dtype,
                 int mean, float beta);

/* ---- dropout (dropout/mod.rs; csrc/nk_dropout.cu) with a counter-based generator ----
 * Philox4x32-10 (Salmon et al., SC'11, the Random123 generator): key = the context's 64-bit seed; counter = (e/4 as a
 * 64-bit value in words 0-1, the call id as a 64-bit value in words 2-3); element e uses output word e%4:
 *   u = (r >> 8) * 2^-24,  q = 1 - (float)p,  keep iff u < q,  y = x / q in f32 (then rounded to dtype), else 0.
 * The call id is a 64-bit counter kept in device memory by the context: every nk_dropout_fwd that draws a mask reads it
 * and the last of its blocks to start advances it by one (a ticket in the same device state), so a captured step draws
 * a new mask on every replay.  The state is allocated on first use (run one step eagerly before capturing), seeded from
 * OS entropy unless nk_rng_seed ran first.
 * nk_dropout_fwd: p == 0 copies x (no draw, mask untouched, may be NULL); p == 1 writes zeros (no draw); otherwise draws
 * and writes the keep mask, bit e%32 of word e/32 (ceil(n/32) words, bits past n are 0).  p outside [0, 1] is an error.
 * nk_dropout_bwd: dx = beta*dx + g*keep/q in dx's element type; g has element type dtype.  p == 0: the identity
 * (dx = beta*dx + g); p == 1: dx = beta*dx; otherwise mask == NULL is the identity too (the backward of a forward that
 * ran in eval mode).
 * nk_rng_seed sets the seed and resets the call counter; it cannot be captured (NK_ERR_UNSUPPORTED while capturing).
 * nk_rng_state reads both back (blocks). */
int nk_dropout_fwd(nk_ctx* ctx, void* y, uint32_t* mask, const void* x, size_t n, int dtype, double p);
int nk_dropout_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const uint32_t* mask, const void* g, size_t n, int dtype,
                   double p, float beta);
int nk_rng_seed(nk_ctx* ctx, uint64_t seed);
int nk_rng_state(nk_ctx* ctx, uint64_t* seed, uint64_t* calls);

/* ---- the rest of the elementwise family (SURVEY.md 8-f rank 1; csrc/nk_pointwise.cu) ----
 * binary ops broadcast like nk_add_bcast_fwd (utils.rs:97-125):
 *   subtraction/mod.rs:44-49, multiplication/mod.rs:44-49, division/mod.rs:44-49.
 * nk_binary_bcast_bwd accumulates ONE operand's gradient (side 0 = left, 1 = right):
 *   dst = beta*dst + unbroadcast(factor(g, l, r) -> shape of that operand), factor =
 *   SUB: g | -g (subtraction/mod.rs:87-92,130-135); MUL: g*r | g*l (multiplication/mod.rs:90-148);
 *   DIV: g/r | -g*l/r^2 (division/mod.rs:90-151).  l / r may be NULL where the factor ignores them. */
typedef enum { NK_BIN_ADD = 0, NK_BIN_SUB = 1, NK_BIN_MUL = 2, NK_BIN_DIV = 3 } nk_binary_op;
int nk_binary_bcast_fwd(nk_ctx* ctx, int op, void* y, const void* l, const void* r, int dtype,
                        int y_ndim, const int64_t* y_shape, int l_ndim, const int64_t* l_shape,
                        int r_ndim, const int64_t* r_shape);
int nk_binary_bcast_bwd(nk_ctx* ctx, int op, int side, void* dst, int dst_dtype, const void* g,
                        const void* l, const void* r, int dtype, int l_ndim, const int64_t* l_shape,
                        int r_ndim, const int64_t* r_shape, float beta);
/* unary ops: y = f(x); dx = beta*dx + g * f'(saved), where `saved` is the tensor the reference's
 * Backward node keeps -- the OUTPUT y for EXP, SQRT, SIGMOID, TANH; the INPUT x for LN, SOFTPLUS,
 * LEAKY_RELU (slope 0.01), POWI; ignored for NEG.  iparam = the integer exponent of POWI
 * (negation/mod.rs:32-68, exp/mod.rs:32-74, logn/mod.rs:32-74, sqrt/mod.rs:32-74, sigmoid/mod.rs:32-76,
 * tanh/mod.rs:32-76, softplus/mod.rs:32-76, leaky_relu/mod.rs:33-81, power/mod.rs:41-88). */
typedef enum { NK_UN_NEG = 0, NK_UN_EXP = 1, NK_UN_LN = 2, NK_UN_SQRT = 3, NK_UN_SIGMOID = 4,
               NK_UN_TANH = 5, NK_UN_SOFTPLUS = 6, NK_UN_LEAKY_RELU = 7, NK_UN_POWI = 8 } nk_unary_op;
int nk_unary_fwd(nk_ctx* ctx, int op, void* y, const void* x, size_t n, int dtype, int iparam);
int nk_unary_bwd(nk_ctx* ctx, int op, void* dx, const void* saved, const void* g, size_t n, int dtype,
                 int iparam, float beta);
/* dst (reversed shape) = beta*dst + src^T : ndarray's `.t()` reverses every axis
 * (transpose/mod.rs:32-36 forward with beta = 0; :66-68 backward `dX += G^T` with beta = 1). Bit exact. */
int nk_transpose(nk_ctx* ctx, void* dst, int dst_dtype, const void* src, int src_dtype, int ndim,
                 const int64_t* src_shape, float beta);
/* padding of the last nsp (1..3) dims of (planes, s...) with a mode; backward is the interior slice
 * for every mode, as in the reference (pad/mod.rs:157-182). */
typedef enum { NK_PAD_CONSTANT = 0, NK_PAD_REFLECTIVE = 1, NK_PAD_REPLICATIVE = 2 } nk_pad_mode;
int nk_padnd_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                 const int64_t* pad, int mode, float value, int dtype);
int nk_padnd_bwd(nk_ctx* ctx, void* dx, const void* g, int64_t planes, int nsp, const int64_t* in_sp,
                 const int64_t* pad, int dtype, float beta);

/* ---- pooling over the last nsp (1..3) dims of (planes, s...), torch's semantics (csrc/nk_pool.cu) ----
 * in_sp / out_sp / k / stride / pad / dilation are host arrays of nsp entries.  Per axis out_sp must be torch's extent
 * floor((L + 2p - d(k-1) - 1)/s) + 1 or its ceil_mode value (the last window dropped when it would start in the right
 * padding); k, s, d >= 1, 0 <= p <= k/2.  Anything else is NK_ERR_INVALID_ARG and launches nothing; more than 2^31 - 1
 * elements in one plane is NK_ERR_UNSUPPORTED.  planes = 0 launches nothing.
 * max: padded positions are never candidates; each window is scanned in row-major order from -inf, an element replacing
 *   the maximum when it is greater or NaN (the first of equal maxima, the last NaN); idx (int32, may be NULL) gets the
 *   in-plane flat index of the winner.  Bit exact.
 * avg: the f32 sum of the in-bounds elements divided once by prod(e - a) (count_include_pad, a = o*s - p,
 *   e = min(a + k, L + p)) or by the number of in-bounds elements; adaptive: window [floor(iL/O), ceil((i+1)L/O)) per
 *   axis, divided by its element count.
 * Backward: dx = beta*dx + sum, the sum gathered per input element in f32 and ascending output order (max: g[o] where
 *   idx[o] is the element; averages: g[o] / divisor), the product and the add rounded separately; no atomics, so
 *   repeated calls are bitwise equal.  dx and g are each f32 or bf16 (dx_dtype, g_dtype). */
int nk_max_pool_nd_fwd(nk_ctx* ctx, void* y, int32_t* idx, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                       const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
                       const int64_t* dilation, int dtype);
int nk_max_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, const int32_t* idx,
                       int64_t planes, int nsp, const int64_t* in_sp, const int64_t* out_sp, const int64_t* k,
                       const int64_t* stride, const int64_t* pad, const int64_t* dilation, float beta);
int nk_avg_pool_nd_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                       const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
                       int count_include_pad, int dtype);
int nk_avg_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int64_t planes, int nsp,
                       const int64_t* in_sp, const int64_t* out_sp, const int64_t* k, const int64_t* stride,
                       const int64_t* pad, int count_include_pad, float beta);
int nk_adaptive_avg_pool_nd_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                                const int64_t* out_sp, int dtype);
int nk_adaptive_avg_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int64_t planes,
                                int nsp, const int64_t* in_sp, const int64_t* out_sp, float beta);

/* ---- batch norm over (N, C, S) and layer norm over (rows, cols), torch's semantics (csrc/nk_norm.cu) ----
 * x / y are f32 or bf16 (dtype); w and b (may be NULL: 1 and 0) have x's dtype; every statistic is f32.
 * Batch norm, S = product of the sample dims (1 for (N, C)), M = N*S per channel:
 *   batch statistics when training or running_mean is NULL: y = (x - mean) * rstd * w + b, mean and the biased var of
 *   the channel, rstd = 1/sqrt(var + eps), saved to save_mean / save_rstd (C floats each); when training with running
 *   stats, rm = (1 - momentum) rm + momentum mean, rv = (1 - momentum) rv + momentum var M/(M - 1).  Otherwise the
 *   running statistics normalize, and save_mean = rm, save_rstd = 1/sqrt(rv + eps).  M = 1 with batch statistics is
 *   NK_ERR_INVALID_ARG (torch's message); N = 0 launches nothing.  Training: 3 launches (partial statistics, per-channel
 *   finalize, apply); running statistics: 1.
 *   Backward with the saved statistics, xhat = (x - save_mean) * save_rstd: db = sum g, dw = sum g*xhat per channel;
 *   dx = w*rstd/M * (M g - sum g - xhat sum g*xhat) when batch_stats, else g*w*rstd.  Each of dx / dw / db may be NULL
 *   (not computed), has its own dtype and is accumulated as d = beta*d + value.  Launches: partial sums and finalize
 *   when dw, db or a batch-statistics dx is wanted, then dx.
 * Layer norm: each of `rows` rows of `cols` elements is normalized by its own mean and biased variance, then w and b
 *   (cols elements) apply elementwise; save_mean / save_rstd hold `rows` floats.  One launch.  Backward, g' = g*w:
 *   dx = rstd/D * (D g' - sum g' - xhat sum g'*xhat) over the row (D = cols), dw / db = the column sums of g*xhat / g;
 *   at most 2 launches (column partials, then dx and the column finalize).
 * Every reduction runs in a fixed order without atomics: repeated calls give identical bits for every output. */
int nk_batch_norm_fwd(nk_ctx* ctx, void* y, const void* x, int dtype, int64_t n, int64_t c, int64_t s, const void* w,
                      const void* b, float* running_mean, float* running_var, float* save_mean, float* save_rstd,
                      int training, float momentum, float eps);
int nk_batch_norm_bwd(nk_ctx* ctx, void* dx, int dx_dtype, float dx_beta, void* dw, int dw_dtype, float dw_beta,
                      void* db, int db_dtype, float db_beta, const void* g, int g_dtype, const void* x, int dtype,
                      int64_t n, int64_t c, int64_t s, const void* w, const float* save_mean, const float* save_rstd,
                      int batch_stats);
int nk_layer_norm_fwd(nk_ctx* ctx, void* y, const void* x, int dtype, int64_t rows, int64_t cols, const void* w,
                      const void* b, float* save_mean, float* save_rstd, float eps);
int nk_layer_norm_bwd(nk_ctx* ctx, void* dx, int dx_dtype, float dx_beta, void* dw, int dw_dtype, float dw_beta,
                      void* db, int db_dtype, float db_beta, const void* g, int g_dtype, const void* x, int dtype,
                      int64_t rows, int64_t cols, const void* w, const float* save_mean, const float* save_rstd);

/* ---- embedding: a gather of weight rows and its deterministic gradient, torch's semantics (csrc/nk_embedding.cu) ----
 * w / dw are (v, e) row-major, y / g are (n, e).  `ids` holds n ids stored as floats, like nll's class ids: ids_dtype
 * NK_F32, or NK_BF16 when v <= 256 (otherwise NK_ERR_INVALID_ARG); v <= 2^24, where every integer is exact in f32.  A
 * value x is a valid id when 0 <= x < v (tested on the float: NaN, negative and x >= v are invalid) and its id is
 * trunc(x).  An INVALID ID gives a zero output row and adds nothing to any gradient row, as nll ignores an out-of-range
 * target.
 * nk_embedding_fwd: y[p, :] = w[id(p), :], a bit-exact copy in `dtype`, 16-byte accesses when e * esize and both bases
 *   allow them.  One launch; n = 0 or e = 0 launches nothing.
 * nk_embedding_bwd: dw[r, :] = beta*dw[r, :] + sum of g[p, :] over the positions p with id(p) == r, r != padding_idx
 *   (-1: none).  dw and g are each f32 or bf16.  No float atomics: the positions are grouped by id with a stable LSD
 *   radix sort (ceil(bits(v + 1) / 8) passes of 8 bits), so each row's positions ascend; the sorted sequence is cut into
 *   slots of 32 entries, each row's run inside a slot is summed sequentially in f32, and a row spanning several slots
 *   adds its runs' partials in slot order.  The sum is rounded once into dw's type, the product beta*dw and the add
 *   rounded separately (beta = 0 never reads dw).  Rows without a valid position: untouched when beta == 1, else
 *   beta*dw (zeros for beta = 0), so a beta = 0 call writes every row.  The order depends on the ids alone: repeated
 *   calls give identical bits.  Nothing syncs with the host (launch sizes depend on n, v and e only).
 *   Launches: 3 per sort pass, then 1 (slots), then 1 more when beta != 1 or n > 32; with n = 0 only the last, and
 *   none at all when beta == 1.  Workspace (nk_alloc_uninit, freed stream-ordered): 16n + 1024*ceil(n/4096) bytes for
 *   the sort, plus 8*ceil(n/32)*e bytes of f32 partials when n > 32.  n >= 2^31 is NK_ERR_UNSUPPORTED. */
int nk_embedding_fwd(nk_ctx* ctx, void* y, const void* w, const void* ids, int ids_dtype, int64_t n, int64_t v, int64_t e,
                     int dtype);
int nk_embedding_bwd(nk_ctx* ctx, void* dw, int dw_dtype, const void* ids, int ids_dtype, const void* g, int g_dtype,
                     int64_t n, int64_t v, int64_t e, int64_t padding_idx, float beta);

/* ---- cross-entropy with class-index targets, torch's F.cross_entropy (csrc/nk_cross_entropy.cu) ----
 * x is (n, c, s) row-major in `dtype` (f32 or bf16): the class axis is the middle one, s = prod(d1..dk) for an
 * (N, C, d1, ..., dk) input and 1 for (N, C).  `target` holds n*s class ids stored as floats, like nll's: target_dtype
 * NK_F32, or NK_BF16 when c <= 256 (otherwise NK_ERR_INVALID_ARG); 1 <= c <= 2^24.  A position is IGNORED when its id
 * is invalid (NaN, < 0, >= c; torch raises instead) or trunc(id) == ignore_index; otherwise its class is t = trunc(id).
 * `weight` is NULL (every weight 1) or c f32 class weights w, W = sum w.  With lse = ln sum_k exp(x_k), eps =
 * label_smoothing in [0, 1] (otherwise NK_ERR_INVALID_ARG), a non-ignored position's loss is
 *   l = (1 - eps)*w_t*(lse - x_t) + eps/c * sum_k w_k*(lse - x_k),
 * and an ignored one's 0.  Sum: loss = sum l; mean (torch's): loss = sum l / sum of w_t over non-ignored positions,
 * NaN (0/0) when every position is ignored or n = 0.
 * nk_cross_entropy_fwd writes the device f32 scalars *loss and *denom (that denominator, whatever `mean`) and lse
 *   (n*s f32, 0 for ignored positions), which the backward reads.  One read of x.
 * nk_cross_entropy_bwd: with p = softmax(x) of the position and gs = *g (Sum) or *g / *denom (mean),
 *   dx_k = beta*dx_k + gs*((1 - eps)*w_t*(p_k - [k == t]) + eps/c*(W*p_k - w_k))
 *   in dx_dtype (f32 or bf16, independently of x), the product and the add rounded separately; beta = 0 never reads
 *   dx; an ignored position gets beta*dx (untouched when beta == 1).  One read of x and lse, one write of dx.
 * Layouts, chosen from the shape: s == 1 rows of <= 4096 bytes, or 4096 rows and more, a warp per row; fewer longer
 * rows a CTA per row, or a CTA per (row, chunk) when there are fewer than 2*SMs rows of at least 65536 classes (the
 * chunks' partial (max, sum) pairs merged in ascending chunk order); s > 1 a thread per position walking the classes
 * with stride s.  16-byte loads of rows whenever x (and dx) are 16-byte aligned, with a scalar head and tail per row.
 * A -inf logit (a masked class) adds nothing to the sum, wherever it falls; a NaN logit makes the position's loss NaN.  Fixed reduction orders, no float
 * atomics: repeated calls give identical bits; nothing is synchronised with the host, so a captured step replays with
 * new targets (and a new ignored count).
 * Launches: forward 1 (finish only, n = 0), 2, or 3 for split rows, plus 1 for W when both weight and eps > 0;
 * backward 1 (none for n = 0), plus the same W launch.  Workspace (nk_alloc_uninit, freed stream-ordered): forward
 * 16 bytes per block of the main kernel (at most 8 per SM), 16 bytes per (row, chunk) for split rows, 16 for W;
 * backward 16 bytes for W. */
int nk_cross_entropy_fwd(nk_ctx* ctx, float* loss, float* lse, float* denom, const void* x, int dtype,
                         const void* target, int target_dtype, const float* weight, int64_t n, int64_t c, int64_t s,
                         int64_t ignore_index, float label_smoothing, int mean);
int nk_cross_entropy_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, int dtype, const void* target,
                         int target_dtype, const float* weight, const float* lse, const float* denom, const float* g,
                         int64_t n, int64_t c, int64_t s, int64_t ignore_index, float label_smoothing, int mean,
                         float beta);

/* ---- matrix-vector / vector-matrix / vector-vector products (8-f rank 3; csrc/nk_gemv.cu) ----
 * A is (rows, cols) row-major.  trans = 0: y[rows] = beta*y + A.x[cols] (MatrixVectorMul::forward,
 * matrix_vector_mul/mod.rs:32-40; vm dv, vector_matrix_mul/mod.rs:64-72); trans = 1: y[cols] = beta*y +
 * A^T.x[rows] (VectorMatrixMul::forward :32-40; mv dv, matrix_vector_mul/mod.rs:93-101).
 * nk_outer_acc: A = beta*A + u (x) v (mv dA :64-69, vm dA vector_matrix_mul/mod.rs:96-101).
 * nk_dot: *out = <a, b> (vector_vector_mul/mod.rs:32-34); nk_scale_acc: dst = beta*dst + x * (*scalar)
 * with the scalar on the device (the 0-d gradient of vv, :58-63). */
int nk_gemv(nk_ctx* ctx, int trans, int64_t rows, int64_t cols, const void* A, const void* x, float beta,
            void* y, int ax_dtype, int y_dtype);
int nk_outer_acc(nk_ctx* ctx, void* A, int a_dtype, const void* u, const void* v, int64_t rows,
                 int64_t cols, int uv_dtype, float beta);
int nk_dot(nk_ctx* ctx, float* out, const void* a, const void* b, size_t n, int dtype);
int nk_scale_acc(nk_ctx* ctx, void* dst, int dst_dtype, const void* x, int x_dtype, const float* scalar,
                 size_t n, float beta);

/* ---- 2-D constant/zero padding of (planes, H, W) (pad/mod.rs:97-129, 157-182) ---- */
int nk_pad2d_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int64_t h, int64_t w,
                 int64_t ph, int64_t pw, float value, int dtype);
int nk_pad2d_bwd(nk_ctx* ctx, void* dx, const void* g, int64_t planes, int64_t h, int64_t w,
                 int64_t ph, int64_t pw, int dtype, float beta);

/* ---- 2-D convolution (cross-correlation, NCHW, no implicit padding)
 * (convolution/mod.rs:85-123 fwd, 146-189 dX, 191-226 dW; arg checks utils.rs:427-496).
 *   x (N,Cin,H,W)  w (Cout,Cin/groups,kh,kw)  y (N,Cout,Ho,Wo),
 *   Ho = (H - dh*(kh-1) - 1)/sh + 1.
 *   fwd optionally fuses + bias[Cout] (the Conv2d layer's (Cout,1,1) bias,
 *   neuronika-nn/src/lib.rs:774) and ReLU; bwd_kernel optionally also accumulates
 *   dbias[Cout] += sum_{n,p,q} g.  With N = 0, bwd_kernel scales dW (and dbias) by beta and
 *   g / x may be NULL. */
int nk_conv2d_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu,
                  int64_t n, int64_t cin, int64_t h, int64_t wd, int64_t cout, int64_t kh,
                  int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw, int64_t groups,
                  int dtype);
int nk_conv2d_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int64_t n,
                        int64_t cin, int64_t h, int64_t wd, int64_t cout, int64_t kh, int64_t kw,
                        int64_t sh, int64_t sw, int64_t dh, int64_t dw, int64_t groups, int dtype,
                        float beta);
int nk_conv2d_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, void* dbias, const void* g,
                         const void* x, int64_t n, int64_t cin, int64_t h, int64_t wd,
                         int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh,
                         int64_t dw, int64_t groups, int dtype, float beta);
/* 1-D / 3-D convolution, x (N, Cin, s[0..nsp)), w (Cout, Cin/groups, k[0..nsp)), nsp = 1..3 sample dims
 * (the reference's convolution is generic over them: convolution/mod.rs:85-226, goldens
 * convolution/test.rs:144-239, 306-444 and the strided / dilated / grouped siblings).  CUDA-core gather
 * kernels; the 2-D entry points above are the tensor-core path. */
int nk_convnd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, int nsp, int64_t n, int64_t cin,
                  const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                  const int64_t* dilation, int64_t groups, int dtype);
int nk_convnd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n,
                        int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k,
                        const int64_t* stride, const int64_t* dilation, int64_t groups, int dtype,
                        float beta);
int nk_convnd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp,
                         int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k,
                         const int64_t* stride, const int64_t* dilation, int64_t groups, int dtype,
                         float beta);
/* 1-D / 3-D convolution LAYERS (nn.Conv1d / nn.Conv3d, neuronika-nn/src/lib.rs:630-916): y = conv(pad(x), w) + bias,
 * x (N, Cin, s[0..nsp)), w (Cout, Cin, k[0..nsp)), nsp = 1 or 3, groups = 1, pad[a] on both sides of axis a with an
 * nk_pad_mode (pad_value: the constant mode's fill), bias (Cout) or NULL.  bf16 shapes of the im2col engine run on the
 * tensor cores with the padding applied inside the column gather ("wgmma_im2col_nd_*"); f32, the other shapes and
 * nk_conv_config(DIRECT) pad into a stream-ordered temporary and run the CUDA-core kernels of nk_convnd_* ("direct_nd_*"),
 * bit-identical to nk_padnd_fwd -> nk_convnd_* -> nk_add_bcast_fwd.  dx gets the interior slice of the padded input's
 * gradient for every mode (the reference's pad backward, pad/mod.rs:157-182; torch instead folds the border gradient of
 * reflect / replicate padding back onto the input).  bwd_kernel also accumulates dbias[Cout] (dw_dtype) when non-NULL.
 * With N = 0 nothing is computed and dW (and dbias) become beta * dW; g and x may then be NULL.  Reflective padding must
 * be smaller than the input extent. */
int nk_conv_layer_nd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int nsp, int64_t n,
                         int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                         const int64_t* dilation, const int64_t* pad, int pad_mode, float pad_value, int dtype);
int nk_conv_layer_nd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                               const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                               const int64_t* dilation, const int64_t* pad, int pad_mode, int dtype, float beta);
int nk_conv_layer_nd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, void* dbias, const void* g, const void* x, int nsp,
                                int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k,
                                const int64_t* stride, const int64_t* dilation, const int64_t* pad, int pad_mode,
                                float pad_value, int dtype, float beta);
/* name of the kernel variant the last conv call used */
const char* nk_last_conv_kernel(nk_ctx* ctx);

/* ---- recurrent cells and `chunks` (SURVEY.md 8-f rank 4; csrc/nk_rnn.cu) ----
 * The gate pre-activations are f32, written by the cell's own GEMMs; states, outputs and gradients have the cell's element
 * type `dtype`; all maths is f32.  The backward entry points recompute the activations (and c') from the f32 gates.
 * LSTM (neuronika-nn/src/lib.rs:510-540 with the intended gate assignment, SURVEY.md 8-c defect 7 = torch.nn.LSTMCell):
 *   gates = x.W_ih^T + b_ih + h.W_hh^T + b_hh, (n, 4H), chunks [i | f | g | o] along the columns:
 *   c' = sigmoid(f)*c + sigmoid(i)*tanh(g);  h' = sigmoid(o)*tanh(c').
 * nk_lstm_cell_bwd writes dgates (beta 0, element type dgates_dtype) and dc_prev = beta_dc*dc_prev + sigmoid(f)*dc_total,
 * dc_total = dc_out + dh_out*sigmoid(o)*(1 - tanh^2(c')).  dh_out / dc_out may be NULL (an output nobody used: zero
 * gradient); dc_prev may be NULL (c not differentiable). */
int nk_lstm_cell_fwd(nk_ctx* ctx, void* c_out, void* h_out, const float* gates, const void* c_prev, int64_t n,
                     int64_t hidden, int dtype);
int nk_lstm_cell_bwd(nk_ctx* ctx, void* dgates, int dgates_dtype, void* dc_prev, float beta_dc, const float* gates,
                     const void* c_prev, const void* dh_out, const void* dc_out, int64_t n, int64_t hidden, int dtype);
/* GRU (torch.nn.GRUCell = neuronika-nn/src/lib.rs:607-624): igates = x.W_ih^T + b_ih, hgates = h.W_hh^T + b_hh, (n, 3H)
 * each, chunks [r | z | n]:  r = sigmoid(i_r + h_r); z = sigmoid(i_z + h_z); nn = tanh(i_n + r*h_n); h' = (h - nn)*z + nn.
 * nk_gru_cell_bwd writes digates and dhgates (beta 0; they differ only in the n chunk) and the pointwise part of the
 * hidden-state gradient, dh_prev = beta_dh*dh_prev + z*dh_out (dh_prev may be NULL). */
int nk_gru_cell_fwd(nk_ctx* ctx, void* h_out, const float* igates, const float* hgates, const void* h_prev, int64_t n,
                    int64_t hidden, int dtype);
int nk_gru_cell_bwd(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, void* dh_prev, float beta_dh,
                    const float* igates, const float* hgates, const void* h_prev, const void* dh_out, int64_t n,
                    int64_t hidden, int dtype);
/* Backward time steps of the LSTM / GRU sequence nodes (nk_graph.h, nkg_lstm / nkg_gru).  As nk_lstm_cell_bwd /
 * nk_gru_cell_bwd, except that the hidden-state gradient of the step is the sum of two sources, dh_out (element type
 * `dtype`: this step's slice of the output gradient) and dh_rec (f32: what the later steps sent back through the hidden
 * state), either of which may be NULL = zero, and that the gradient carried from step to step is f32 whatever `dtype`
 * and is updated in place:
 *   LSTM  dc (n, H) f32 holds dc_out on entry and dc_prev = sigmoid(f)*dc_total on return;
 *   GRU   dh_rec holds the pointwise part z*dh of the previous step's gradient on return (the caller adds
 *         dhgates.W_hh); it is left alone when NULL. */
int nk_lstm_seq_bwd_step(nk_ctx* ctx, void* dgates, int dgates_dtype, float* dc, const float* gates, const void* c_prev,
                         const void* dh_out, const float* dh_rec, int64_t n, int64_t hidden, int dtype);
int nk_gru_seq_bwd_step(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, float* dh_rec, const float* igates,
                        const float* hgates, const void* h_prev, const void* dh_out, int64_t n, int64_t hidden, int dtype);
/* One time step of BOTH directions of a bidirectional sequence layer (nk_graph.h, nkg_lstm_layer / nkg_gru_layer) in one
 * launch, with the gate maths above.  Every per-direction operand X is passed as direction 0's pointer plus X_dstride,
 * the distance in elements (any sign) to direction 1's.  Rows of y, dh_out and the GRU backward's h_prev are ld* apart
 * (2H for the layer's (T, N, 2H) output); every other (n, H) operand is dense.  h_next (forward), dc and dh_rec
 * (backward, f32) are (2, n, H) buffers with direction stride n*H.
 *   forward:  writes h' into y and h_next (and, LSTM, c' into c_out);
 *   backward: as nk_lstm_seq_bwd_step / nk_gru_seq_bwd_step per direction; dgates / digates / dhgates share the gates'
 *             layout (gates_dstride); dh_out and dh_rec may be NULL. */
int nk_lstm_bidir_fwd_step(nk_ctx* ctx, void* y, int64_t y_dstride, int64_t ldy, void* h_next, void* c_out,
                           int64_t c_out_dstride, const float* gates, int64_t gates_dstride, const void* c_prev,
                           int64_t c_prev_dstride, int64_t n, int64_t hidden, int dtype);
int nk_gru_bidir_fwd_step(nk_ctx* ctx, void* y, int64_t y_dstride, int64_t ldy, void* h_next, const float* igates,
                          const float* hgates, int64_t gates_dstride, const void* h_prev, int64_t h_prev_dstride, int64_t n,
                          int64_t hidden, int dtype);
int nk_lstm_bidir_bwd_step(nk_ctx* ctx, void* dgates, int dgates_dtype, int64_t gates_dstride, float* dc, const float* gates,
                           const void* c_prev, int64_t c_prev_dstride, const void* dh_out, int64_t dh_out_dstride,
                           int64_t ld_dh_out, const float* dh_rec, int64_t n, int64_t hidden, int dtype);
int nk_gru_bidir_bwd_step(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, int64_t gates_dstride, float* dh_rec,
                          const float* igates, const float* hgates, const void* h_prev, int64_t h_prev_dstride,
                          int64_t ld_h_prev, const void* dh_out, int64_t dh_out_dstride, int64_t ld_dh_out, int64_t n,
                          int64_t hidden, int dtype);
/* chunks (chunk/mod.rs): y = block `index` of x in row-major block order (ndarray's exact_chunks: trailing partial blocks
 * are dropped); a bit-exact copy.  Backward: dx[block] = beta*dx[block] + g, nothing else of dx is touched. */
int nk_chunk_fwd(nk_ctx* ctx, void* y, const void* x, int ndim, const int64_t* x_shape, const int64_t* chunk_shape,
                 int64_t index, int dtype);
int nk_chunk_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int ndim, const int64_t* x_shape,
                 const int64_t* chunk_shape, int64_t index, float beta);

/* ---- concatenation (multi_concatenate/mod.rs, multi_stack/mod.rs; csrc/nk_cat.cu) ----
 * Operand i is an (outer, lens[i], inner) block; the output is (outer, sum lens, inner) with operand i at offset
 * sum_{j<i} lens[j] along the middle axis.  A stack is the same call with every lens[i] = 1.  xs / lens (and the
 * backward's per-operand arrays) are host arrays of `count` entries, passed to the kernel by value: one launch per
 * NK_CAT_OPS_PER_LAUNCH operands in each direction, no allocation and no host-to-device copy, so both calls can be
 * captured (nk_capture_begin).
 * nk_cat_fwd: a bit-exact copy; an operand with no elements contributes nothing (its pointer may be NULL).
 * nk_cat_bwd: dxs[i] = betas[i]*dxs[i] + (block i of g), element type dx_dtypes[i] (f32 or bf16, independently of g's;
 * bf16 results are rounded to nearest even); dxs[i] == NULL: operand i gets no gradient.  The non-NULL dxs must be
 * pairwise distinct (two slices summed into one buffer are two calls). */
#define NK_CAT_OPS_PER_LAUNCH 64
int nk_cat_fwd(nk_ctx* ctx, void* y, const void* const* xs, const int64_t* lens, int count, int64_t outer,
               int64_t inner, int dtype);
int nk_cat_bwd(nk_ctx* ctx, void* const* dxs, const int* dx_dtypes, const float* betas, const void* g, int g_dtype,
               const int64_t* lens, int count, int64_t outer, int64_t inner);

/* ---- optimizers and learning-rate schedulers (csrc/nk_optim_multi.cu) ----
 * lr and the step count live in device memory, in a caller-allocated nk_optim_hyper block that the kernels read (and
 * the prologue and the scheduler write), so a captured step advances them on every replay.
 *   nk_optim_hyper_set / _get copy the whole block to / from the device and synchronise; NK_ERR_UNSUPPORTED while
 *   capturing (a replay would not repeat them).
 *   nk_optim_prologue (one thread): step += 1, then, for NK_OPTIM_ADAM (Adam and AMSGrad), step_size = lr/(1-b1^t) and
 *   sqrt_bc2 = sqrt(1-b2^t), b^t by repeated squaring; for NK_OPTIM_ADAGRAD clr = lr/(1+(t-1)*lr_decay).  Every
 *   operation is rounded on its own in f32, in the order written.  SGD and RMSProp need no prologue: their kernels read
 *   lr.
 *   nk_multi_*_step: one optimizer step over `count` <= NK_OPTIM_TENSORS_PER_LAUNCH tensors of one (w_dtype, g_dtype)
 *   pair in ONE launch.  w, g and n are arrays of `count` entries; each state / master argument is an array of `count`
 *   device pointers or NULL (= every entry NULL).  State arrays are f32, n elements, zero before the first step.
 *   `master` (f32, optional; a NULL entry means that tensor has none) keeps an f32 copy of bf16 weights: the update is
 *   applied to master and w receives its rounding.  The tensor table travels in the kernel parameters: no allocation,
 *   no host-to-device copy, so the call can be captured.  A tensor takes 4-element (16-byte f32) accesses when all its
 *   pointers allow them, element accesses otherwise.  grad_scale = 1/world_size for data parallel.  Per element, with t
 *   the step count and lr, step_size, sqrt_bc2, clr read from `hyper`:
 *   sgd      (sgd/mod.rs:191-231, penalty.rs:63-67) g' = grad_scale*g + 2*l2*w ; no momentum: w -= lr*g' ;
 *            momentum: buf = mu*buf + (1-damp)*g' ; w -= lr*(nesterov ? g' + mu*buf : buf).  `momentum_buf` may be
 *            NULL when momentum <= FLT_EPSILON.  g' is written back into g when write_back_grad, except when l2 = 0 and
 *            grad_scale = 1 (then g' = g).
 *   The Adam family: g' = grad_scale*g + l1*signum(w) + 2*l2*w (penalty.rs:63-79: L1, L2, ElasticNet), written back into
 *   g when write_back_grad (the reference adds the penalty into the gradient).
 *   adam     m = b1*m + (1-b1)g'; v = b2*v + (1-b2)g'^2; w -= m / (sqrt(v)/sqrt_bc2 + eps) * step_size
 *            (adam/mod.rs:131-169); max_exp_avg_sq != NULL -> AMSGrad: v^ = max(v^, v) replaces v in the
 *            denominator (amsgrad/mod.rs:159-204).
 *   rmsprop  s = a*s + (1-a)g'^2; centered (grad_avg != NULL): ga = a*ga + (1-a)g', denom = sqrt(s - ga^2)+eps
 *            else sqrt(s)+eps; momentum (> f32::EPSILON, momentum_buf != NULL): b = mu*b + g'/denom, w -= lr*b;
 *            else w -= g'/denom*lr (rmsprop/mod.rs:193-300).
 *   adagrad  s += g'^2; w -= g' / (sqrt(s) + eps) * clr   (adagrad/mod.rs:113-140).
 * Learning-rate schedulers (lr_scheduler/{step_lr,multi_step_lr,exponential_lr,multiplicative_lr,lambda_lr}/mod.rs):
 * nk_lr_sched_step (one thread) advances epoch to t = epoch + 1 and applies the rule to the optimizer block's lr in f32:
 *   STEP           lr *= gamma when t % step_size == 0        MULTI_STEP  lr *= gamma when t is one of the milestones
 *   EXPONENTIAL    lr *= gamma                                MULTIPLICATIVE  lr *= f(t)    LAMBDA  lr = initial_lr * f(t)
 * last_lr receives lr before the step and current_lr after it.  `table` is a device array of table_len entries: the
 * milestones (int64) or f(1..table_len) (f32).  A closure-based step with t > table_len changes nothing and sets
 * past_horizon, which stays set: nk_lr_sched_get then fails with NK_ERR_INVALID_ARG until nk_lr_sched_set clears it.
 * nk_lr_sched_set / _get copy the block like nk_optim_hyper_set / _get (synchronous, refused while capturing). */
#define NK_OPTIM_TENSORS_PER_LAUNCH 64
typedef enum { NK_OPTIM_ADAM = 0, NK_OPTIM_ADAGRAD = 1 } nk_optim_prologue_kind;
typedef struct nk_optim_hyper {
  float lr;
  float step_size;  /* Adam: lr / (1 - beta1^step) */
  float sqrt_bc2;   /* Adam: sqrt(1 - beta2^step) */
  float clr;        /* Adagrad: lr / (1 + (step - 1) * lr_decay) */
  int64_t step;     /* optimizer steps taken */
} nk_optim_hyper;
typedef enum { NK_LR_STEP = 0, NK_LR_MULTI_STEP = 1, NK_LR_EXPONENTIAL = 2, NK_LR_MULTIPLICATIVE = 3,
               NK_LR_LAMBDA = 4 } nk_lr_kind;
typedef struct nk_lr_sched {
  int64_t epoch;
  int64_t step_size;   /* NK_LR_STEP, >= 1 */
  const void* table;   /* milestones (int64) or factors f(1..table_len) (f32), device memory */
  int64_t table_len;
  float gamma;
  float initial_lr;    /* NK_LR_LAMBDA */
  float last_lr;
  float current_lr;
  int32_t kind;        /* nk_lr_kind */
  int32_t past_horizon;
} nk_lr_sched;
int nk_optim_hyper_set(nk_ctx* ctx, nk_optim_hyper* hyper, const nk_optim_hyper* host);
int nk_optim_hyper_get(nk_ctx* ctx, const nk_optim_hyper* hyper, nk_optim_hyper* host);
int nk_optim_prologue(nk_ctx* ctx, nk_optim_hyper* hyper, int kind, float beta1, float beta2, float lr_decay);
int nk_multi_sgd_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                      void* const* momentum_buf, void* const* master, const int64_t* n, const nk_optim_hyper* hyper,
                      float l2, float momentum, float dampening, int nesterov, float grad_scale, int write_back_grad);
int nk_multi_adam_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                       void* const* exp_avg, void* const* exp_avg_sq, void* const* max_exp_avg_sq, void* const* master,
                       const int64_t* n, const nk_optim_hyper* hyper, float beta1, float beta2, float eps, float l1,
                       float l2, float grad_scale, int write_back_grad);
int nk_multi_rmsprop_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                          void* const* square_avg, void* const* grad_avg, void* const* momentum_buf, void* const* master,
                          const int64_t* n, const nk_optim_hyper* hyper, float alpha, float eps, float momentum,
                          float l1, float l2, float grad_scale, int write_back_grad);
int nk_multi_adagrad_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                          void* const* grad_sq, void* const* master, const int64_t* n, const nk_optim_hyper* hyper,
                          float eps, float l1, float l2, float grad_scale, int write_back_grad);
int nk_lr_sched_set(nk_ctx* ctx, nk_lr_sched* sched, const nk_lr_sched* host);
int nk_lr_sched_get(nk_ctx* ctx, const nk_lr_sched* sched, nk_lr_sched* host);
int nk_lr_sched_step(nk_ctx* ctx, nk_lr_sched* sched, nk_optim_hyper* hyper);

/* ---- gradient clipping, torch.nn.utils' get_total_norm / clip_grads_with_norm_ / clip_grad_value_ (csrc/nk_optim_multi.cu)
 * Each call takes `count` gradients of any dtypes (g_dtype[i]: NK_F32 or NK_BF16) with n[i] elements each.  Inside a
 * call the tensors are grouped by dtype in order of first appearance, and each group takes one launch per
 * NK_OPTIM_TENSORS_PER_LAUNCH tensors (a group of empty tensors takes none); the table travels in the kernel parameters.
 * A tensor takes 4-element (16-byte f32, 8-byte bf16) accesses when its base allows them, element accesses otherwise.
 * Nothing is read back to the host, so every call can be captured.  Invalid arguments (a bad dtype, a negative n, a
 * NULL pointer where elements are, a bad norm_type) fail with NK_ERR_INVALID_ARG before anything is launched.
 *   nk_grad_norm: with k = grad_scale and v = f32(k*g) (one f32 multiply) over every element of every tensor,
 *     p = 2: sqrt(sum v^2)   p = 1: sum |v|   p = +inf: max |v|   other p > 0: (sum |v|^p)^(1/p)  (powf only here),
 *     written to *total (device, one f32).  A NaN element makes the total NaN (for p = +inf too), an infinite one
 *     makes it +inf; count = 0 gives 0.  norm_type <= 0, -inf and NaN are rejected.  Launches: one per group, each
 *     CTA writing one f32 partial (its elements folded in a fixed tree) to a workspace from nk_alloc_uninit that is
 *     freed stream-ordered, then one CTA that merges every partial in a fixed order in double, takes the root in
 *     double and rounds once to f32.  No float atomics: repeated calls give identical bits.
 *   nk_grad_scale_by_norm: torch's coefficient, each operation rounded on its own in f32,
 *     c = (1 / (*total + 1e-6)) * max_norm (torch evaluates max_norm / x as x.reciprocal() * max_norm), c = 1 when
 *     c > 1 (a compare: a NaN total gives c = NaN); then g = dtype(f32(g) * c), one rounding.  When c == 1 nothing is
 *     written (g * 1 == g).  One launch per group.
 *   nk_grad_clamp: b = clip_value / grad_scale in f32; g = min(max(g, -b), b), clamp_min first as torch applies them, a
 *     NaN element stays NaN; clip_value < 0 makes every other element b.  One launch per group. */
int nk_grad_norm(nk_ctx* ctx, int count, const void* const* g, const int* g_dtype, const int64_t* n, float norm_type,
                 float grad_scale, float* total);
int nk_grad_scale_by_norm(nk_ctx* ctx, int count, void* const* g, const int* g_dtype, const int64_t* n,
                          const float* total, float max_norm);
int nk_grad_clamp(nk_ctx* ctx, int count, void* const* g, const int* g_dtype, const int64_t* n, float clip_value,
                  float grad_scale);

/* ---- NCCL all-reduce behind the ABI (SURVEY.md 8-b, 8-e; csrc/nk_comm.cu) ----
 * The context owns the communicator; libnccl.so.2 is bound at run time (dlopen), so the library loads
 * without it.  Rank 0 creates the 128-byte id and ships it to the others by any means; every rank then
 * calls nk_comm_init_rank (collective).  nk_allreduce_sum sums `n` elements in place over the replicas,
 * enqueued on the context stream (ordered with the kernels that produced the gradients and with the
 * nk_multi_sgd_step that follows).  Errors: NK_ERR_NCCL. */
int nk_comm_unique_id(nk_ctx* ctx, void* id128);
int nk_comm_init_rank(nk_ctx* ctx, int world, int rank, const void* id128);
int nk_comm_destroy(nk_ctx* ctx);
int nk_comm_world(nk_ctx* ctx);
int nk_comm_rank(nk_ctx* ctx);
int nk_allreduce_sum(nk_ctx* ctx, void* ptr, size_t n, int dtype);

/* ---- data-parallel gradient exchange over NVLink peer memory (SURVEY.md 8-e) ----
 * The reference has no multi-device path; under data parallel the only exchange on the hot path is
 * the sum of the weight gradients over the replicas before the SGD step above (which then runs
 * identically on every replica).  Rather than a library all-reduce after the dW GEMM, the exchange
 * is fused into the kernels around it (neuronika_b200/csrc/nk_peer.cu):
 *   nk_gemm_rs       the wgmma GEMM whose epilogue stores row shard o of the (M,N) f32 product
 *                    into rank o's slot buffer `slots[o]` (world*M/world*N floats, slot index = the
 *                    calling rank) over NVLink, tile by tile while the MMAs run (reduce-scatter).
 *                    Needs 2 <= world <= 8, bf16 operands that TMA can address, M % (world*128) == 0,
 *                    N > 128, N % 4 == 0 and 16-byte aligned slots; K = 0 (an empty local batch) stores
 *                    zero shards.  An error launches nothing and leaves the slots untouched;
 *   nk_peer_barrier  flag exchange through peer memory: returns (on the stream) once every rank has
 *                    reached the same `epoch`; `flags[r]` is rank r's flag array (>= world words);
 *   nk_reduce_bcast  the owner sums its `world` slots in rank order and stores the result into every
 *                    replica's gradient `grads[r]` at element rank*shard_elems (all-gather half).
 * Buffers that peers touch come from nk_ipc_alloc (cudaMalloc; pool memory cannot be exported) and
 * are mapped by the other processes with nk_ipc_export (64-byte handle) / nk_ipc_open. */
int nk_ipc_alloc(nk_ctx* ctx, size_t bytes, void** out);
int nk_ipc_free(nk_ctx* ctx, void* ptr);
int nk_ipc_export(nk_ctx* ctx, void* ptr, void* handle64);
int nk_ipc_open(nk_ctx* ctx, const void* handle64, void** peer_ptr);
int nk_ipc_close(nk_ctx* ctx, void* peer_ptr);
int nk_peer_barrier(nk_ctx* ctx, void* const* flags, int world, int rank, uint32_t epoch);
int nk_gemm_rs(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
               const void* A, int64_t lda, const void* B, int64_t ldb, void* const* slots, int world,
               int rank, int ab_dtype);
int nk_reduce_bcast(nk_ctx* ctx, const float* slots, void* const* grads, int world, int rank,
                    int64_t shard_elems, int max_ctas);
/* barrier -> owner reduce + broadcast -> barrier as ONE kernel whose epoch lives on the device (`state`: 16 bytes of
 * zero-initialised LOCAL device memory per exchange sequence), so the launch is identical every step and can be
 * captured in a CUDA graph.  flags[r] = rank r's flag words (>= 2*world, zero-initialised, peer-mapped).  Work is
 * handed out in 32 KB chunks, so max_ctas may be the SM count (0 = that): CTAs that do not fit beside a running
 * GEMM start when it retires.  All ranks must issue the same sequence of calls on the same (flags, state). */
int nk_reduce_exchange(nk_ctx* ctx, const float* slots, void* const* grads, void* const* flags, int world,
                       int rank, int64_t shard_elems, void* state, int max_ctas);
/* all-reduce (sum, rank order: bit-identical on every replica) of a small local vector `grad` (n <= 2^20 floats: biases,
 * the 10-wide layer) through peer memory in one single-CTA kernel: slots[r] = rank r's receive buffer (world*n floats),
 * flags / state as above but separate from nk_reduce_exchange's. */
int nk_peer_allreduce_small(nk_ctx* ctx, float* grad, void* const* slots, void* const* flags, int world, int rank,
                            int64_t n, void* state);

#ifdef __cplusplus
}
#endif
#endif /* NK_B200_H */
