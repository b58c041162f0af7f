/*
 * nk_graph.h -- C handle API of the host-side graph (C++), the mirror of the reference's
 * Var / VarDiff op surface over device tensors.
 *
 * The reference's host code is Rust (neuronika-variable/src/{var,vardiff,history,gradient}.rs);
 * no Rust toolchain exists in this environment, so the define-by-run graph above the kernel ABI
 * (nk_b200.h) is written in C++ (neuronika_b200/csrc/nk_graph.cpp) with the same semantics:
 *   - a variable is a handle to (data, tape); differentiable variables add (grad, backward tape)
 *     (var.rs:34-61, vardiff.rs:35-65);
 *   - op methods only record nodes; nothing is computed until forward() (lazy), which runs every
 *     node of the tape in creation order (var.rs:110-128); backward(seed) fills the root gradient
 *     with `seed` and runs the backward nodes in reverse order (vardiff.rs:125-141);
 *   - every backward node ACCUMULATES into its operands' gradients (beta = 1); leaf gradients
 *     persist until zero_grad() (vardiff.rs:100-102);
 *   - differentiability is sticky: Var (x) VarDiff -> VarDiff, and only the needed backward
 *     halves are built (var.rs:1048-1061).
 * This header exists so that Python (ctypes) and any other FFI can drive that C++ graph; a Rust
 * binding would not use it (it would implement Forward/Backward over nk_b200.h directly, see
 * INTEGRATION.md).
 *
 * All functions return 0 or a negative nk_status; nkg_last_error() gives the message (shape
 * errors carry the reference's own panic text where it has one).
 */
#ifndef NK_GRAPH_H
#define NK_GRAPH_H

#include "nk_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nkg_var nkg_var; /* Var or VarDiff */

typedef enum { NKG_MEAN = 0, NKG_SUM = 1 } nkg_reduction; /* neuronika-variable/src/lib.rs:29-36 */

const char* nkg_last_error(void);

/* ---- leaves (neuronika-variable/src/lib.rs:51-240 constructors; data zero-filled) ---- */
int nkg_leaf(nk_ctx* ctx, int ndim, const int64_t* shape, int dtype, nkg_var** out);
/* wrap caller-owned device memory as a leaf (flat parameter / gradient buckets for data parallel) */
int nkg_leaf_external(nk_ctx* ctx, int ndim, const int64_t* shape, int dtype, void* data_ptr, nkg_var** out);
/* Var::requires_grad (var.rs:104-107): returns a NEW differentiable handle sharing the data.
 * grad_dtype < 0 -> same as data; grad_ptr may supply caller-owned gradient storage (or NULL). */
int nkg_requires_grad(nkg_var* v, int grad_dtype, void* grad_ptr, nkg_var** out);
int nkg_clone(nkg_var* v, nkg_var** out);
int nkg_release(nkg_var* v);

/* ---- introspection ---- */
int nkg_is_diff(nkg_var* v);
int nkg_ndim(nkg_var* v);
int nkg_shape(nkg_var* v, int64_t* shape_out);
int nkg_dtype(nkg_var* v);
int nkg_grad_dtype(nkg_var* v);
void* nkg_data_ptr(nkg_var* v);  /* device pointer (allocates the buffer if still lazy) */
void* nkg_grad_ptr(nkg_var* v);  /* NULL for Var or after no_grad() */
int nkg_history_len(nkg_var* v); /* number of forward nodes on the tape (test.rs:748-806 checks) */
int nkg_backward_history_len(nkg_var* v);

/* ---- execution (var.rs:110-128, vardiff.rs:100-165) ---- */
int nkg_forward(nkg_var* v);
int nkg_backward(nkg_var* v, float seed);
int nkg_zero_grad(nkg_var* v);
int nkg_no_grad(nkg_var* v);
int nkg_with_grad(nkg_var* v);
/* host-side peephole fusion over the tape.  level 0: off.  level 1 (default): mm_t + bias add (+ ReLU) -> one GEMM
 * epilogue, conv + bias -> one kernel, gradient aliasing through single-consumer adds; invisible to results for ANY
 * use of the tape (a repeated backward() un-aliases first).  level 2: additionally the ReLU backward of a layer is
 * applied in the epilogue of the dX GEMM above it (nk_gemm_relu_bwd), which never stores the intermediate gradient --
 * exact for one backward() per tape (what a training loop does); a second backward() on such a tape fails loudly. */
int nkg_set_fusion(int level);

/* ---- operators (names follow the reference's methods) ---- */
int nkg_mm(nkg_var* a, nkg_var* b, nkg_var** out);      /* var.rs:1034-1061, vardiff.rs:1073-1106 */
int nkg_mm_t(nkg_var* a, nkg_var* b, nkg_var** out);    /* var.rs:1065-1094 */
int nkg_add(nkg_var* a, nkg_var* b, nkg_var** out);     /* vardiff.rs:902-924, broadcasting */
int nkg_relu(nkg_var* a, nkg_var** out);
int nkg_softmax(nkg_var* a, int axis, nkg_var** out);
int nkg_log_softmax(nkg_var* a, int axis, nkg_var** out);
int nkg_sum(nkg_var* a, nkg_var** out);
int nkg_mean(nkg_var* a, nkg_var** out);
int nkg_mse_loss(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_nll_loss(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_pad(nkg_var* a, int64_t ph, int64_t pw, float value, nkg_var** out); /* Zero = Constant(0) */
/* receiver is the KERNEL, argument the input, as in the reference (var.rs:704-716) */
int nkg_convolution(nkg_var* kernel, nkg_var* input, int64_t sh, int64_t sw, int64_t dh, int64_t dw,
                    int64_t groups, nkg_var** out);
/* (N, C, H, W) -> (N, C*H*W): bit-exact view; not in the reference (SURVEY.md 2.2 "missing") */
int nkg_flatten(nkg_var* a, nkg_var** out);

/* ---- the rest of the op surface (SURVEY.md 8-f): broadcasting arithmetic (vardiff.rs Sub/Mul/Div impls over
 * subtraction/, multiplication/, division/), unary maths (var.rs `exp`, `ln`, `sqrt`, `sigmoid`, `tanh`, `softplus`,
 * `leaky_relu`, `pow(i32)`, `Neg`), `t()` (reverses every axis), n-d padding with a mode, mv / vm / vv and 1-d / 3-d
 * convolution.  nkg_unary takes an nk_unary_op; the named functions are the reference's method names. */
int nkg_sub(nkg_var* a, nkg_var* b, nkg_var** out);
int nkg_mul(nkg_var* a, nkg_var* b, nkg_var** out);
int nkg_div(nkg_var* a, nkg_var* b, nkg_var** out);
int nkg_unary(nkg_var* a, int op, int iparam, nkg_var** out);
int nkg_neg(nkg_var* a, nkg_var** out);
int nkg_exp(nkg_var* a, nkg_var** out);
int nkg_ln(nkg_var* a, nkg_var** out);
int nkg_sqrt(nkg_var* a, nkg_var** out);
int nkg_sigmoid(nkg_var* a, nkg_var** out);
int nkg_tanh(nkg_var* a, nkg_var** out);
int nkg_softplus(nkg_var* a, nkg_var** out);
int nkg_leaky_relu(nkg_var* a, nkg_var** out);
int nkg_pow(nkg_var* a, int exp, nkg_var** out);
int nkg_transpose(nkg_var* a, nkg_var** out);
/* pad the nsp (1..3) sample dims of (N, C, ...) with an nk_pad_mode (pad/mod.rs:20-182) */
int nkg_pad_mode(nkg_var* a, int nsp, const int64_t* padding, int mode, float value, nkg_var** out);
/* Pooling of the nsp (1..3) sample dims of (N, C, ...), torch's semantics (nk_b200.h nk_*_pool_nd_*), one forward and
 * one backward node each.  kernel / stride / padding / dilation / output_size: nsp entries; ceil_mode as in torch.  The
 * max pool of a differentiable operand keeps the winners' int32 indices (numel(out) * 4 bytes, allocated when the node
 * is built) for its backward.  Invalid arguments fail with NK_ERR_INVALID_ARG and record nothing. */
int nkg_max_pool(nkg_var* a, int nsp, const int64_t* kernel, const int64_t* stride, const int64_t* padding,
                 const int64_t* dilation, int ceil_mode, nkg_var** out);
int nkg_avg_pool(nkg_var* a, int nsp, const int64_t* kernel, const int64_t* stride, const int64_t* padding,
                 int ceil_mode, int count_include_pad, nkg_var** out);
int nkg_adaptive_avg_pool(nkg_var* a, int nsp, const int64_t* output_size, nkg_var** out);
int nkg_mv(nkg_var* matrix, nkg_var* vector, nkg_var** out);   /* matrix_vector_mul/mod.rs */
int nkg_vm(nkg_var* vector, nkg_var* matrix, nkg_var** out);   /* vector_matrix_mul/mod.rs */
int nkg_vv(nkg_var* a, nkg_var* b, nkg_var** out);             /* vector_vector_mul/mod.rs: 0-d result */
/* 1-d (N,C,L) / 3-d (N,C,D,H,W) convolution; the receiver is the kernel, as in nkg_convolution */
int nkg_convolution_nd(nkg_var* kernel, nkg_var* input, int nsp, const int64_t* stride, const int64_t* dilation,
                       int64_t groups, nkg_var** out);
/* The 1-d / 3-d convolution LAYER (nn.Conv1d / nn.Conv3d) as ONE node: out = conv(pad(input), weight) + bias, input
 * (N, Cin, s...) with nsp = 1 or 3 sample dims, weight (Cout, Cin, k...), bias (Cout, 1, ..) with nsp ones, or NULL;
 * `padding` per sample dim with an nk_pad_mode (`value`: the constant mode's fill).  The same results as the nodes
 * pad_mode -> convolution_nd -> add, without the padded copy of the input or its gradient: forward and backward are
 * nk_conv_layer_nd_* (tensor cores for bf16).  The backward writes only the gradients of differentiable operands. */
int nkg_conv_layer(nkg_var* input, nkg_var* weight, nkg_var* bias, int nsp, const int64_t* padding, int mode, float value,
                   const int64_t* stride, const int64_t* dilation, nkg_var** out);

/* ---- chunks and recurrent cells (SURVEY.md 8-f rank 4) ----
 * nkg_chunks (var.rs:401-417): every block of ndarray's exact_chunks(chunk_shape) in row-major block order, one lazy
 * node each (a bit-exact copy; backward adds into that block of the operand's gradient).  *count receives the number of
 * blocks; nothing is recorded when it exceeds `capacity` (call with capacity 0 to ask).
 * nkg_lstm_cell / nkg_gru_cell: one step of neuronika-nn's LSTMCell / GRUCell (lib.rs:450-626) as ONE forward and ONE
 * backward node: x (N, I), hidden and cell_state (N, H), weight_ih (G*H, I), weight_hh (G*H, H), biases (G*H,), G = 4
 * (LSTM, gate chunks [i | f | g | o], the intended assignment of SURVEY.md 8-c defect 7 = torch.nn.LSTMCell) or 3 (GRU,
 * [r | z | n] = torch.nn.GRUCell).  All operands share one element type and one context.  The outputs are differentiable
 * if any operand is; the LSTM's two outputs carry the same node in their histories. */
int nkg_chunks(nkg_var* a, int ndim, const int64_t* chunk_shape, int capacity, nkg_var** outs, int* count);
int nkg_lstm_cell(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh,
                  nkg_var* bias_ih, nkg_var* bias_hh, nkg_var** new_cell_state, nkg_var** new_hidden);
int nkg_gru_cell(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
                 nkg_var* bias_hh, nkg_var** new_hidden);

/* ---- recurrent sequence layers (one layer, one direction, time-major) ----
 * nkg_lstm / nkg_gru: the cell above applied to every step of input (T, N, I), T >= 1, from the initial states hidden
 * (and cell_state) (N, H), with the cells' weight layout.  `output` (T, N, H) holds every step's hidden state, so the
 * last hidden state is output[T-1]; `last_cell_state` (N, H) is the LSTM's cell state after step T-1.  Each call records
 * ONE forward and ONE backward node whatever T is: the products that do not depend on the recurrence (x.W_ih^T + b_ih,
 * dW_ih, dW_hh, dx, the bias gradients) run once over all T*N rows, and the state gradient is carried from step to step
 * in f32.  The node keeps the f32 gate pre-activations of all steps (T*N*G values; twice that for the GRU, as T cell nodes
 * do) and the backward allocates T*N*G elements of the operands' type for its own duration.  Operands are validated as
 * the cells': one element type, one context, any mix of differentiable and plain operands; only the differentiable
 * ones get gradient work, and the outputs are differentiable if any operand is. */
int nkg_lstm(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
             nkg_var* bias_hh, nkg_var** output, nkg_var** last_cell_state);
int nkg_gru(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih, nkg_var* bias_hh,
            nkg_var** output);
/* nkg_lstm_layer / nkg_gru_layer: one layer of torch.nn.LSTM / GRU, one or two directions (D = hidden's first dimension).
 * input (T, N, I); hidden and cell_state (D, N, H); parameters stacked over the directions, weight_ih (D, G*H, I),
 * weight_hh (D, G*H, H), biases (D, G*H), direction 1 = torch's `_reverse` parameters.  `output` (T, N, D*H) holds every
 * time step's hidden state, the reverse direction's (which runs from time T-1 down to 0) in columns [H, 2H);
 * `last_hidden` / `last_cell_state` (D, N, H) are each direction's state after its last step (time T-1 forward, time 0
 * reverse).  ONE forward and ONE backward node.  D = 1 issues the calls of nkg_lstm / nkg_gru plus one N*H copy into
 * last_hidden.  D = 2 runs both directions' step t in one nk_gemm_strided_batched and one nk_*_bidir_*_step launch
 * (2 + 2T launches forward, 2T + the whole-sequence products backward) and keeps D times what one direction keeps. */
int nkg_lstm_layer(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh,
                   nkg_var* bias_ih, nkg_var* bias_hh, nkg_var** output, nkg_var** last_hidden, nkg_var** last_cell_state);
int nkg_gru_layer(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
                  nkg_var* bias_hh, nkg_var** output, nkg_var** last_hidden);

/* ---- concatenation (var.rs:564-645, vardiff.rs:627-; multi_concatenate/mod.rs, multi_stack/mod.rs) ----
 * nkg_cat: the `count` operands side by side along `axis` (0 <= axis < ndim; equal shapes on every other axis, any length
 * along `axis`, 0 included).  nkg_stack: identical shapes, joined along a new axis 0 <= axis <= ndim.  Both record ONE
 * forward and ONE backward node whatever the count; the result's history is the union of the operands' plus that node.
 * All operands share one element type and one context; the result is differentiable if any operand is, and only the
 * differentiable operands receive gradients.  count >= 1 (one operand: a copy).
 * nkg_unsqueeze (var.rs:425-431): a new axis of length 1 at 0 <= axis <= ndim.  A view, like nkg_flatten: no kernel,
 * no node (the reference records one), and the gradient is the operand's. */
int nkg_cat(nkg_var* const* vars, int count, int axis, nkg_var** out);
int nkg_stack(nkg_var* const* vars, int count, int axis, nkg_var** out);
int nkg_unsqueeze(nkg_var* a, int axis, nkg_var** out);
/* nkg_reshape: the operand under `shape` (ndim <= NK_MAX_DIMS entries, same element count).  A view like nkg_flatten
 * and nkg_unsqueeze: no kernel, no node, and the gradient is the operand's. */
int nkg_reshape(nkg_var* a, int ndim, const int64_t* shape, nkg_var** out);
/* nkg_embedding: out = weight[ids], torch's embedding (nk_b200.h nk_embedding_*): weight (v, e) f32 or bf16; ids of
 * any shape holding float ids (f32, or bf16 when v <= 256), never differentiable; out has shape ids.shape + (e,) and
 * the weight's dtype, and is differentiable iff the weight is.  An invalid id gives a zero row and no gradient;
 * padding_idx (-1: none, else 0 <= padding_idx < v) gets no gradient either.  ONE forward and ONE backward node; the
 * backward writes the weight's gradient. */
int nkg_embedding(nkg_var* ids, nkg_var* weight, int64_t padding_idx, nkg_var** out);
/* nkg_cross_entropy: torch's F.cross_entropy with class-index targets (nk_b200.h nk_cross_entropy_*): input (N, C) or
 * (N, C, d1, ..., dk), f32 or bf16; target (N) or (N, d1, ..., dk) holding float class ids (f32, or bf16 when C <= 256),
 * never differentiable; weight NULL or an f32 (C) tensor, never differentiable; reduction NKG_MEAN (torch's: divided by
 * the summed weights of the non-ignored positions, NaN when there are none) or NKG_SUM; label_smoothing in [0, 1].
 * Positions whose id equals ignore_index or is invalid (NaN, < 0, >= C) are ignored.  The result is a 0-d f32 scalar.
 * ONE forward node, which owns the saved per-position lse and the denominator, and, for a differentiable input, ONE
 * backward node into the input's gradient.  Invalid arguments (shapes, weight, label_smoothing, bf16 target with
 * C > 256, devices) are NK_ERR_INVALID_ARG and record nothing. */
int nkg_cross_entropy(nkg_var* input, nkg_var* target, nkg_var* weight, int reduction, int64_t ignore_index,
                      float label_smoothing, nkg_var** out);

/* ---- the other criteria and dropout (var.rs:375-521, vardiff.rs:418-583) ----
 * nkg_mae / nkg_bce / nkg_bce_with_logits / nkg_kldiv take (input, target, reduction) like nkg_mse_loss: same shape and
 * element type, a non-differentiable target, a 0-d f32 result; ONE forward node and, for a differentiable input, ONE
 * backward node (nk_b200.h gives the maths).  kldiv's Mean divides by the input's leading dimension (batch mean).
 * Dropout's status is a shared flag (the reference's Rc<Cell<bool>>): 1 = train, 0 = eval; every node built with it
 * sees later changes.  nkg_dropout: p outside [0, 1] fails with "Wrong probability received" and records nothing.
 * The node owns its keep mask (allocated when the node is built, for 0 < p < 1).  Every forward() reads the status:
 * train with 0 < p < 1 draws a new mask (nk_dropout_fwd), train with p == 1 writes zeros, eval or p == 0 copies.  The
 * backward applies what the last forward did, whatever the status says by then.  A captured step replays the status it
 * was captured with: the choice between drawing and copying is made on the host when the kernels are recorded. */
typedef struct nkg_status nkg_status;
int nkg_mae(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_bce(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_bce_with_logits(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_kldiv(nkg_var* input, nkg_var* target, int reduction, nkg_var** out);
int nkg_status_create(int train, nkg_status** out);
int nkg_status_set(nkg_status* status, int train);
int nkg_status_get(nkg_status* status);   /* 1 train, 0 eval */
int nkg_status_release(nkg_status* status);
int nkg_dropout(nkg_var* a, double p, nkg_status* status, nkg_var** out);
/* Batch norm of an (N, C, ...) operand over N and the sample dims, torch's semantics (nk_b200.h nk_batch_norm_*), one
 * node.  weight / bias: (C,) of the operand's dtype, or NULL; running_mean / running_var: non-differentiable f32 (C,)
 * leaves updated in place by every training forward, or both NULL (batch statistics in both modes).  `status` is read
 * on each forward() (train: batch statistics); the backward follows what the last forward did.  The node's (C,) f32
 * saved statistics are allocated when it is built.  Invalid arguments fail with NK_ERR_INVALID_ARG and record
 * nothing, batch statistics of one value per channel with torch's message. */
int nkg_batch_norm(nkg_var* x, nkg_var* weight, nkg_var* bias, nkg_var* running_mean, nkg_var* running_var,
                   nkg_status* status, float momentum, float eps, nkg_var** out);
/* Layer norm over the last k dims of the operand (torch's normalized_shape = those dims), one node; weight / bias have
 * that shape and the operand's dtype, or are NULL. */
int nkg_layer_norm(nkg_var* x, int k, nkg_var* weight, nkg_var* bias, float eps, nkg_var** out);

/* ---- gradient-ready hook (data parallel overlap): `cb(user, begin, end)` is called from inside nkg_backward(), on
 * the calling thread, right after the LAST kernel that accumulates into elements [begin, end) of this leaf's gradient
 * in the running backward pass has been launched -- so the caller can start the all-reduce of that range while the
 * rest of backward runs.  Normally one call with [0, numel).  With row_chunks > 1, a matmul backward node that is the
 * last writer of the gradient computes it in that many row blocks (one GEMM each, same arithmetic per element) and
 * reports every block as soon as it is launched, so a single large layer's exchange overlaps its own dW GEMMs. */
typedef void (*nkg_grad_hook)(void* user, int64_t elem_begin, int64_t elem_end);
int nkg_set_grad_hook(nkg_var* leaf, nkg_grad_hook cb, void* user, int row_chunks);

/* ---- fused exchange (nk_b200.h "data-parallel gradient exchange"): when the matmul backward node that writes this
 * leaf's gradient finds it all-zero (beta = 0), it runs nk_gemm_rs into `slots` instead of the plain dW GEMM and calls
 * `cb(user, 1)`; otherwise (accumulating into an existing gradient, shape not shardable) it computes the gradient
 * locally as usual and calls `cb(user, 0)` so that the caller can fall back to an all-reduce.  world <= 8. */
typedef void (*nkg_grad_rs_hook)(void* user, int pushed);
int nkg_set_grad_rs(nkg_var* leaf, int world, int rank, void* const* slots, nkg_grad_rs_hook cb, void* user);

/* ---- optimizers over many leaves (neuronika-optim/src/{sgd,adam,amsgrad,rmsprop,adagrad}/mod.rs; nk_b200.h
 * nk_multi_*_step): one optimizer step over `count` parameters, lr and the step count in the device block `hyper`.
 * State and master arguments are arrays of `count` caller-owned f32 device buffers of the parameters' sizes, in
 * parameter order (or NULL: none).  Each parameter's gradient is taken as the backward pass left it (zeros after
 * nkg_zero_grad) and receives the penalised gradient; Adam and Adagrad then launch nk_optim_prologue once; the
 * parameters are grouped by (data, gradient) element types and each group is updated by one nk_multi_*_step call per
 * NK_OPTIM_TENSORS_PER_LAUNCH tensors, in parameter order.  A parameter that is not differentiable fails the call
 * before anything is launched. */
int nkg_multi_sgd_step(nkg_var* const* params, int count, void* const* momentum_buf, void* const* master,
                       nk_optim_hyper* hyper, float l2, float momentum, float dampening, int nesterov, float grad_scale);
int nkg_multi_adam_step(nkg_var* const* params, int count, void* const* exp_avg, void* const* exp_avg_sq,
                        void* const* max_exp_avg_sq, void* const* master, nk_optim_hyper* hyper, float beta1,
                        float beta2, float eps, float l1, float l2, float grad_scale);
int nkg_multi_rmsprop_step(nkg_var* const* params, int count, void* const* square_avg, void* const* grad_avg,
                           void* const* momentum_buf, void* const* master, nk_optim_hyper* hyper, float alpha, float eps,
                           float momentum, float l1, float l2, float grad_scale);
int nkg_multi_adagrad_step(nkg_var* const* params, int count, void* const* grad_sq, void* const* master,
                           nk_optim_hyper* hyper, float lr_decay, float eps, float l1, float l2, float grad_scale);

/* ---- gradient clipping over many leaves (torch.nn.utils; nk_b200.h nk_grad_norm / nk_grad_scale_by_norm /
 * nk_grad_clamp).  Every parameter must be differentiable and on one context, or the call fails before anything is
 * materialised or launched.  Then each gradient is materialised in parameter order (a pending zero_grad() gets its
 * zero fill) and ONE ABI call takes the tables in parameter order.  nkg_grad_norm writes the total norm of the
 * gradients times grad_scale to `total` (device, one f32) and needs at least one parameter (the total's device);
 * nkg_clip_grads_with_norm scales them by torch's coefficient from max_norm and that total; nkg_clip_grad_value clamps
 * them to +-clip_value / grad_scale.  The two writing calls mark the gradients nonzero; with count = 0 they do
 * nothing. */
int nkg_grad_norm(nkg_var* const* params, int count, float norm_type, float grad_scale, float* total);
int nkg_clip_grads_with_norm(nkg_var* const* params, int count, float max_norm, const float* total);
int nkg_clip_grad_value(nkg_var* const* params, int count, float clip_value, float grad_scale);

#ifdef __cplusplus
}
#endif
#endif
