// Host-side define-by-run graph in C++ over the kernel ABI (nk_b200.h): the mirror of the
// reference's Var / VarDiff / History / Gradient and of its Forward / Backward node structs.
//
//   reference (Rust, neuronika-variable/src)                     here
//   --------------------------------------------------------------------------------------------
//   Var<D>{data, history}                     var.rs:34-61        Variable{data, fwd tape}
//   VarDiff<D>{var, grad, history}            vardiff.rs:35-65    Variable{+ grad, bwd tape}
//   History<T> (BTreeMap in insertion order)  history.rs:54-124   std::map<op id, node> + buffer
//   Gradient<T,D> (RefCell<Option<array>>)    gradient.rs:14-79   Gradient (lazy device buffer)
//   trait Forward / trait Backward            autograd.rs:7-25    struct Forward / struct Backward
//   node structs (one Forward + 1..3 Backward per op)  node/*/mod.rs   classes of the same names
//
// Protocol kept bit-for-bit: op methods only record nodes; forward() recomputes the whole tape in
// creation order; backward(seed) fills the root gradient and runs the backward tape in reverse;
// every Backward accumulates into its operand gradients.  Two host-side optimisations are
// invisible to results: (1) buffers are allocated lazily and a gradient known to be all-zero is
// overwritten (beta = 0) instead of read-modify-written; (2) a peephole over the tape fuses
// mm_t + bias-add into one GEMM epilogue and aliases the gradient of a single-consumer addend.
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "nk_graph.h"

namespace nkg {

static thread_local std::string g_error;
static int g_fusion = 1;  // 0 off, 1 exact for any use of the tape, 2 additionally assumes ONE backward() per tape,
                          // 3 = 2 + the bias-gradient column sums in the dX GEMM epilogue (no measured gain: see fuse())
static uint64_t g_next_op_id = 1;  // creation order == a topological order (history.rs:84-88)

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

[[noreturn]] static void fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw Error(code, buf);
}

static inline void ck(nk_ctx* ctx, int rc) {
  if (rc != NK_OK) throw Error(rc, nk_last_error(ctx));
}

using Shape = std::vector<int64_t>;
static int64_t numel(const Shape& s) {
  int64_t n = 1;
  for (auto d : s) n *= d;
  return n;
}
static size_t esize(int dt) { return dt == NK_BF16 ? 2 : 4; }

// ------------------------------------------------------------------------------- Tensor
struct Tensor {
  nk_ctx* ctx;
  Shape shape;
  int dtype;
  void* ptr = nullptr;
  bool owned = true;
  std::shared_ptr<Tensor> base;  // view of another tensor (flatten)
  Tensor(nk_ctx* c, Shape s, int dt) : ctx(c), shape(std::move(s)), dtype(dt) {}
  ~Tensor() {
    if (owned && ptr && !base) nk_free(ctx, ptr);
  }
  int64_t n() const { return numel(shape); }
  // buffer about to be fully overwritten by a forward kernel: no zero fill needed
  void* wptr() {
    if (base) return base->wptr();
    if (!ptr) ck(ctx, nk_alloc_uninit(ctx, size_t(n()) * esize(dtype), &ptr));
    return ptr;
  }
  // a reader of a tensor nothing has written yet sees zeros (CuArray::zeroed; test.rs:748-806 laziness checks)
  void* rptr() {
    if (base) return base->rptr();
    if (!ptr) ck(ctx, nk_alloc(ctx, size_t(n()) * esize(dtype), &ptr));
    return ptr;
  }
};
using TensorP = std::shared_ptr<Tensor>;

// ------------------------------------------------------------------------------- Gradient
struct Gradient {
  nk_ctx* ctx;
  Shape shape;
  int dtype;
  void* ptr = nullptr;
  bool owned = true;
  bool enabled = true;   // false after no_grad()
  bool is_zero = true;   // content known to be all zeros -> first accumulate may overwrite
  bool stale = false;    // logically zero but the memory has not been cleared yet (lazy zero_grad)
  std::shared_ptr<Gradient> alias;  // fusion: this gradient IS that gradient
  nkg_grad_hook hook = nullptr;     // data-parallel overlap: called when the last writer of a backward pass is done
  void* hook_user = nullptr;
  int hook_chunks = 1;              // a matmul that is the last writer may deliver the gradient in this many row blocks
  int writers = 0;                  // backward nodes accumulating into it in the running pass
  uint64_t pass_id = 0;
  int rs_world = 0, rs_rank = 0;    // fused reduce-scatter plan (nkg_set_grad_rs)
  void* rs_slots[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  nkg_grad_rs_hook rs_hook = nullptr;
  void* rs_user = nullptr;
  int last_writer = -1;             // index (in reverse tape order) of the last node writing it in this pass
  bool hook_fired = false;
  // fill(v) is deferred: the gradient is "v everywhere" until somebody needs the bytes (get / acc materialise it).
  // A consumer that takes a uniform gradient as a value (ConvolutionBackward -> nk_conv2d_bwd_uniform) only needs the
  // bytes for the duration of its own call: backward(seed) on a convolution's own output keeps no materialised G.
  bool is_const = false;
  float const_val = 0.f;
  bool is_leaf = false;             // created by requires_grad(): owned by the user, never aliased away by the peephole
  Gradient(nk_ctx* c, Shape s, int dt) : ctx(c), shape(std::move(s)), dtype(dt) {}
  ~Gradient() {
    if (owned && ptr) nk_free(ctx, ptr);
  }
  Gradient* root() { return alias ? alias->root() : this; }
  int64_t n() const { return numel(shape); }
  void* get() {
    Gradient* r = root();
    if (!r->enabled)
      fail(NK_ERR_INVALID_ARG,
           "Trying to get a de-allocated gradient. Switch on the gradients first by using `.with_grad()`");
    if (!r->ptr) {
      if (r->is_const)   // a deferred fill writes every element right below: the zero fill of nk_alloc would only move bytes
        ck(r->ctx, nk_alloc_uninit(r->ctx, size_t(r->n()) * esize(r->dtype), &r->ptr));
      else
        ck(r->ctx, nk_alloc(r->ctx, size_t(r->n()) * esize(r->dtype), &r->ptr));
      r->is_zero = true;
      r->stale = false;
    }
    if (r->stale) {  // a reader wants the zeros that zero_grad() promised
      ck(r->ctx, nk_memset0(r->ctx, r->ptr, size_t(r->n()) * esize(r->dtype)));
      r->stale = false;
    }
    if (r->is_const) {  // a reader wants the bytes of a deferred fill
      r->is_const = false;
      r->is_zero = false;
      ck(r->ctx, nk_fill(r->ctx, r->ptr, r->dtype, size_t(r->n()), r->const_val));
    }
    return r->ptr;
  }
  // pointer + beta for an accumulating write that covers the whole buffer: beta = 0 when the content is
  // known to be zero (then stale memory is simply overwritten), and the buffer counts as touched afterwards
  void* acc(float* beta) {
    Gradient* r = root();
    if (r->is_const) get();  // accumulating on top of a deferred fill: make it real first
    if (r->enabled && !r->ptr) {  // first touch is a full overwrite (beta = 0): no need to clear the new buffer
      ck(r->ctx, nk_alloc_uninit(r->ctx, size_t(r->n()) * esize(r->dtype), &r->ptr));
      r->is_zero = true;
      r->stale = false;
    }
    if (!r->enabled || !r->ptr) get();
    *beta = r->is_zero ? 0.f : 1.f;
    r->is_zero = false;
    r->stale = false;
    return r->ptr;
  }
  void zero() {
    Gradient* r = root();
    r->is_const = false;
    if (r->ptr && !r->is_zero) {
      if (r->owned || (r->rs_world > 1 && r->rs_slots[0]))
        // owned memory: clear lazily (first full overwrite or first read).  Also a slice of a data-parallel bucket with
        // a fused-exchange plan: the exchange rewrites the whole slice every step, so clearing 64 MB first only moves
        // bytes; a reader through the graph still gets its zeros (get() honours `stale`)
        r->stale = true;
      else
        ck(r->ctx, nk_memset0(r->ctx, r->ptr, size_t(r->n()) * esize(r->dtype)));  // caller-visible memory
    }
    r->is_zero = true;
  }
  void fill(float v) {  // deferred: see is_const
    Gradient* r = root();
    if (!r->enabled)
      fail(NK_ERR_INVALID_ARG,
           "Trying to get a de-allocated gradient. Switch on the gradients first by using `.with_grad()`");
    if (!r->owned) {  // caller-visible memory: write it now
      float unused;
      r->is_const = false;
      ck(r->ctx, nk_fill(r->ctx, acc(&unused), r->dtype, size_t(r->n()), v));
      r->is_zero = false;
      return;
    }
    r->is_const = true;
    r->const_val = v;
    r->is_zero = false;
    r->stale = false;
  }
  void no_grad() {  // gradient.rs:68-71
    Gradient* r = root();
    r->is_const = false;
    if (r->owned && r->ptr) nk_free(r->ctx, r->ptr);
    if (r->owned) r->ptr = nullptr;
    r->enabled = false;
  }
  void with_grad() {  // gradient.rs:73-78 (fresh zeros)
    Gradient* r = root();
    if (!r->enabled) {
      r->enabled = true;
      r->is_zero = true;
      if (!r->owned && r->ptr) ck(r->ctx, nk_memset0(r->ctx, r->ptr, size_t(r->n()) * esize(r->dtype)));
    }
  }
};
using GradientP = std::shared_ptr<Gradient>;

// ------------------------------------------------------------------------------- node traits
struct Forward {
  bool skip = false;  // fused into a consumer
  virtual ~Forward() {}
  virtual void forward() = 0;
  virtual const char* name() const = 0;
};
// set by nkg_backward around each node: position of the running node in the reverse tape
static thread_local int g_bwd_pos = -1;
static inline void grad_written(const GradientP& g) {
  if (!g) return;
  Gradient* r = g->root();
  if (r->hook && r->last_writer == g_bwd_pos && !r->hook_fired) {
    r->hook_fired = true;
    r->hook(r->hook_user, 0, r->n());
  }
}

struct Backward {
  GradientP gradient;  // gradient of this node's output
  bool skip = false;
  bool single_pass = false;  // a fusion that is exact for ONE backward pass was applied to this node
  int runs = 0;        // backward() calls so far (a second pass over the same tape must see un-aliased gradients)
  virtual ~Backward() {}
  virtual void backward() = 0;
  virtual void targets(std::vector<Gradient*>& out) = 0;  // gradients this node accumulates into
  virtual const char* name() const = 0;
  virtual void no_grad() {
    if (gradient) gradient->no_grad();
  }
  virtual void with_grad() {
    if (gradient) gradient->with_grad();
  }
};
using ForwardP = std::shared_ptr<Forward>;
using BackwardP = std::shared_ptr<Backward>;

static void gemm(nk_ctx* ctx, bool ta, bool tb, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                 const void* B, int64_t ldb, float beta, void* C, int ab_dt, int c_dt, const void* bias = nullptr,
                 int bias_dt = NK_F32, int relu = 0) {
  ck(ctx, nk_gemm_bias_act(ctx, ta, tb, M, N, K, 1.f, A, lda, B, ldb, beta, C, N, ab_dt, c_dt, bias, bias_dt, relu));
}

// A backward kernel that produces its result in element type `kdt` accumulating into a gradient that may have another
// element type (a bf16 leaf with an f32 gradient, requires_grad(grad_dtype)): same type -> the kernel writes the
// gradient directly with the accumulate mode `beta`; otherwise it writes a temporary (beta = 0) which is then added
// with the mixed-type axpy of nk_unbroadcast_acc.
template <typename F>
static void acc_typed(nk_ctx* ctx, const GradientP& g, int kdt, F&& kernel) {
  float beta;
  void* d = g->acc(&beta);
  if (g->dtype == kdt) {
    kernel(d, beta);
    return;
  }
  void* tmp = nullptr;
  ck(ctx, nk_alloc_uninit(ctx, size_t(g->n()) * esize(kdt), &tmp));
  try {
    kernel(tmp, 0.f);
    ck(ctx, nk_unbroadcast_acc(ctx, d, g->dtype, (int)g->shape.size(), g->shape.data(), tmp, kdt, (int)g->shape.size(),
                               g->shape.data(), beta));
  } catch (...) {
    nk_free(ctx, tmp);
    throw;
  }
  ck(ctx, nk_free(ctx, tmp));
}

// ------------------------------------------------------------------------------- matmul nodes
// MatrixMatrixMul (matrix_matrix_mul/mod.rs:11-41) and MatrixMatrixMulT (matrix_matrix_mul_t/mod.rs:11-41)
struct MatMul : Forward {
  nk_ctx* ctx;
  TensorP left, right, data;
  bool t;  // true: C = A.B^T (mm_t)
  MatMul(nk_ctx* c, TensorP l, TensorP r, TensorP d, bool tt) : ctx(c), left(l), right(r), data(d), t(tt) {}
  const char* name() const override { return t ? "MatrixMatrixMulT" : "MatrixMatrixMul"; }
  void forward() override { run(nullptr); }
  void run(Tensor* bias, Tensor* out = nullptr, int relu = 0) {
    Tensor* o = out ? out : data.get();
    const int64_t M = left->shape[0], K = left->shape[1], N = t ? right->shape[0] : right->shape[1];
    gemm(ctx, false, t, M, N, K, left->rptr(), left->shape[1], right->rptr(), right->shape[1], 0.f, o->wptr(),
         left->dtype, o->dtype, bias ? bias->rptr() : nullptr, bias ? bias->dtype : NK_F32, relu);
  }
};

// dA += G.B^T | G.B ; dB += A^T.G | G^T.A   (matrix_matrix_mul/mod.rs:43-126, matrix_matrix_mul_t/mod.rs:43-126)
struct MatMulBackward : Backward {
  nk_ctx* ctx;
  TensorP left_data, right_data;
  GradientP left_grad, right_grad;  // either may be null (operand not differentiable)
  bool t;
  // fusion level 2: the left operand is the output of a ReLU whose backward is the only reader of left_grad -- the
  // masked product goes straight into the ReLU operand's gradient (nk_gemm_relu_bwd), left_grad is never materialised
  TensorP left_mask;
  GradientP left_dst;
  // ... and the bias gradient of the layer below (the un-broadcast of its Addition's (K) row bias) is summed in the
  // same epilogue (nk_gemm_relu_bwd_colsum): the AdditionBackward then skips its right operand
  GradientP left_colsum;
  const char* name() const override { return t ? "MatrixMatrixMulTBackward" : "MatrixMatrixMulBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (left_dst)
      out.push_back(left_dst->root());
    else if (left_grad)
      out.push_back(left_grad->root());
    if (left_dst && left_colsum) out.push_back(left_colsum->root());
    if (right_grad) out.push_back(right_grad->root());
  }
  void backward() override {
    const int64_t M = left_data->shape[0], K = left_data->shape[1];
    const int64_t N = t ? right_data->shape[0] : right_data->shape[1];
    const void* G = gradient->get();
    const int gdt = gradient->dtype;
    // the right operand is the parameter in Linear (dW): issue it first so that its all-reduce can overlap the
    // dX GEMM under data parallel; the two results are independent, so the order is invisible
    if (right_grad) {
      float beta;
      void* d = right_grad->acc(&beta);
      // TN in both cases: dW += G^T.X : (M,N)^T.(M,K) -> (N,K) | dB += A^T.G : (M,K)^T.(M,N) -> (K,N)
      const void* A = t ? G : left_data->rptr();
      const void* B = t ? left_data->rptr() : G;
      const int64_t rows = t ? N : K, cols = t ? K : N;
      Gradient* r = right_grad->root();
      int chunks = 1;
      if (r->rs_world > 1) {
        // data parallel: the epilogue of the dW GEMM pushes each row shard to its owner over NVLink (nk_gemm_rs);
        // only when this node alone produces the gradient in this pass and the gradient starts from zero
        const bool push = beta == 0.f && gdt == NK_BF16 && right_grad->dtype == NK_F32 && r == right_grad.get() &&
                          r->writers == 1 && rows % (int64_t(r->rs_world) * 128) == 0 && cols > 128 && cols % 8 == 0;
        if (push)
          ck(ctx, nk_gemm_rs(ctx, 1, 0, rows, cols, M, 1.f, A, rows, B, cols, r->rs_slots, r->rs_world, r->rs_rank, gdt));
        else
          gemm(ctx, true, false, rows, cols, M, A, rows, B, cols, beta, d, gdt, right_grad->dtype);
        if (r->rs_hook) r->rs_hook(r->rs_user, push ? 1 : 0);
        chunks = 0;
      } else if (r == right_grad.get() && r->hook && r->hook_chunks > 1 && r->last_writer == g_bwd_pos && !r->hook_fired &&
          rows % (int64_t(r->hook_chunks) * 128) == 0)
        chunks = r->hook_chunks;
      if (chunks == 0) {
        // handled above
      } else if (chunks == 1) {
        gemm(ctx, true, false, rows, cols, M, A, rows, B, cols, beta, d, gdt, right_grad->dtype);
        grad_written(right_grad);
      } else {
        // row blocks of the gradient, each final (and handed to the hook) as soon as its GEMM is launched
        const int64_t rc = rows / chunks;
        for (int c = 0; c < chunks; ++c) {
          const int64_t r0 = c * rc;
          gemm(ctx, true, false, rc, cols, M, static_cast<const char*>(A) + r0 * esize(gdt), rows, B, cols, beta,
               static_cast<char*>(d) + r0 * cols * esize(right_grad->dtype), gdt, right_grad->dtype);
          r->hook(r->hook_user, r0 * cols, (r0 + rc) * cols);
        }
        r->hook_fired = true;
      }
    }
    if (left_dst) {  // (M,K), ReLU backward of the layer below in the epilogue: dZ += (Y > 0) * (G.W | G.B^T)
      float beta;
      void* d = left_dst->acc(&beta);
      bool summed = false;
      if (left_colsum && beta == 0.f) {
        float bbeta;
        void* db = left_colsum->acc(&bbeta);
        if (bbeta == 0.f) ck(ctx, nk_memset0(ctx, db, size_t(K) * sizeof(float)));
        const int rc = nk_gemm_relu_bwd_colsum(ctx, 0, t ? 0 : 1, M, K, N, G, N, right_data->rptr(), t ? K : N, 0.f, d, K, gdt,
                                               left_dst->dtype, left_mask->rptr(), static_cast<float*>(db));
        if (rc == NK_OK)
          summed = true;
        else if (rc != NK_ERR_UNSUPPORTED)
          ck(ctx, rc);
        else if (bbeta == 0.f)
          left_colsum->root()->is_zero = true;   // nothing was added: the plain un-broadcast below overwrites
      }
      if (!summed) {
        ck(ctx, nk_gemm_relu_bwd(ctx, 0, t ? 0 : 1, M, K, N, G, N, right_data->rptr(), t ? K : N, beta, d, K, gdt,
                                 left_dst->dtype, left_mask->rptr()));
        if (left_colsum) {   // no fused epilogue for this shape / accumulate mode: the ordinary column sums of dZ
          float bbeta;
          void* db = left_colsum->acc(&bbeta);
          const int64_t dshape[1] = {K}, gshape[2] = {M, K};
          ck(ctx, nk_unbroadcast_acc(ctx, db, left_colsum->dtype, 1, dshape, d, left_dst->dtype, 2, gshape, bbeta));
        }
      }
      grad_written(left_dst);
      grad_written(left_colsum);
    } else if (left_grad) {  // (M,K)
      float beta;
      void* d = left_grad->acc(&beta);
      if (t)  // dX += G.W      : (M,N).(N,K)   NN
        gemm(ctx, false, false, M, K, N, G, N, right_data->rptr(), K, beta, d, gdt, left_grad->dtype);
      else    // dA += G.B^T    : (M,N).(K,N)^T NT
        gemm(ctx, false, true, M, K, N, G, N, right_data->rptr(), N, beta, d, gdt, left_grad->dtype);
      grad_written(left_grad);
    }
  }
};

// ------------------------------------------------------------------------------- addition
struct Convolution;
struct Addition : Forward {  // addition/mod.rs:11-50
  nk_ctx* ctx;
  TensorP left, right, data;
  std::shared_ptr<MatMul> fused_gemm;        // peephole: data = mm_t(..) + right in one kernel
  std::shared_ptr<Convolution> fused_conv;   // peephole: data = convolution(..) + bias(Cout,1,1) in one kernel
  TensorP fused_relu_out;                    // peephole: the consumer ReLU's output, written by the GEMM epilogue
  void run_fused_conv();
  const char* name() const override { return "Addition"; }
  void forward() override {
    if (fused_gemm) {
      if (fused_relu_out)
        fused_gemm->run(right.get(), fused_relu_out.get(), 1);  // y = relu(x.W^T + b); z itself is never stored
      else
        fused_gemm->run(right.get(), data.get());
      return;
    }
    if (fused_conv) {
      run_fused_conv();
      return;
    }
    ck(ctx, nk_add_bcast_fwd(ctx, data->wptr(), left->rptr(), right->rptr(), data->dtype, (int)data->shape.size(),
                             data->shape.data(), (int)left->shape.size(), left->shape.data(),
                             (int)right->shape.size(), right->shape.data()));
  }
};

struct AdditionBackward : Backward {  // addition/mod.rs:52-135 (Left, Right and the composite)
  nk_ctx* ctx;
  GradientP left_grad, right_grad;
  bool left_aliased = false, right_aliased = false;  // right_aliased: the bias gradient is produced by the fused conv dW
  bool right_fused = false;   // the bias gradient is summed in the epilogue of the dX GEMM above (MatMulBackward::left_colsum)
  const char* name() const override { return "AdditionBackward"; }
  void acc(GradientP& dst, bool aliased) {
    if (!dst || aliased) return;
    float beta;
    void* d = dst->acc(&beta);
    ck(ctx, nk_unbroadcast_acc(ctx, d, dst->dtype, (int)dst->shape.size(), dst->shape.data(), gradient->get(),
                               gradient->dtype, (int)gradient->shape.size(), gradient->shape.data(), beta));
    grad_written(dst);
  }
  void targets(std::vector<Gradient*>& out) override {
    if (left_grad) out.push_back(left_grad->root());
    if (right_grad && !right_fused) out.push_back(right_grad->root());
  }
  void backward() override {
    acc(left_grad, left_aliased);
    acc(right_grad, right_aliased || right_fused);
  }
};

// ------------------------------------------------------------------------------- unary / softmax
struct ReLU : Forward {  // relu/mod.rs:11-38
  nk_ctx* ctx;
  TensorP operand, data;
  const char* name() const override { return "ReLU"; }
  void forward() override {
    ck(ctx, nk_relu_fwd(ctx, data->wptr(), operand->rptr(), size_t(data->n()), data->dtype));
  }
};
struct ReLUBackward : Backward {  // relu/mod.rs:40-79
  nk_ctx* ctx;
  TensorP operand_data;
  GradientP operand_grad;
  const char* name() const override { return "ReLUBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    const void* g = gradient->get();
    acc_typed(ctx, operand_grad, operand_data->dtype, [&](void* d, float beta) {
      ck(ctx, nk_relu_bwd(ctx, d, operand_data->rptr(), g, size_t(operand_data->n()), operand_data->dtype, beta));
    });
  }
};

static void lanes(const Shape& s, int axis, int64_t& outer, int64_t& len, int64_t& inner) {
  outer = inner = 1;
  for (int i = 0; i < axis; ++i) outer *= s[i];
  len = s[axis];
  for (size_t i = axis + 1; i < s.size(); ++i) inner *= s[i];
}

struct Softmax : Forward {  // softmax/mod.rs:11-53, logsoftmax/mod.rs:11-53
  nk_ctx* ctx;
  TensorP operand, data;
  int axis;
  bool log;
  const char* name() const override { return log ? "LogSoftmax" : "Softmax"; }
  void forward() override {
    int64_t o, l, i;
    lanes(data->shape, axis, o, l, i);
    ck(ctx, (log ? nk_log_softmax_fwd : nk_softmax_fwd)(ctx, data->wptr(), operand->rptr(), o, l, i, data->dtype));
  }
};
struct SoftmaxBackward : Backward {  // softmax/mod.rs:55-104, logsoftmax/mod.rs:55-102
  nk_ctx* ctx;
  TensorP data;
  GradientP operand_grad;
  int axis;
  bool log;
  const char* name() const override { return log ? "LogSoftmaxBackward" : "SoftmaxBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    int64_t o, l, i;
    lanes(data->shape, axis, o, l, i);
    const void* g = gradient->get();
    acc_typed(ctx, operand_grad, data->dtype, [&](void* d, float beta) {
      ck(ctx, (log ? nk_log_softmax_bwd : nk_softmax_bwd)(ctx, d, data->rptr(), g, o, l, i, data->dtype, beta));
    });
  }
};

// ------------------------------------------------------------------------------- reductions / losses
struct SumMean : Forward {  // sum/mod.rs:11-34, mean/mod.rs:11-34
  nk_ctx* ctx;
  TensorP operand, data;
  bool mean;
  const char* name() const override { return mean ? "Mean" : "Sum"; }
  void forward() override {
    ck(ctx, nk_sum_fwd(ctx, (float*)data->wptr(), operand->rptr(), size_t(operand->n()), operand->dtype, mean));
  }
};
struct SumMeanBackward : Backward {  // sum/mod.rs:36-66, mean/mod.rs:36-71
  nk_ctx* ctx;
  GradientP operand_grad;
  bool mean;
  const char* name() const override { return mean ? "MeanBackward" : "SumBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    float beta;
    void* d = operand_grad->acc(&beta);
    ck(ctx, nk_sum_bwd(ctx, d, (const float*)gradient->get(), size_t(operand_grad->n()), operand_grad->dtype, mean,
                       beta));
  }
};

struct Loss : Forward {  // squared_error/mod.rs:11-58, nll/mod.rs:11-68
  nk_ctx* ctx;
  TensorP input, target, data;
  bool mean, nll;
  const char* name() const override { return nll ? "NegativeLogLikelihood" : "SquaredError"; }
  void forward() override {
    if (nll)
      ck(ctx, nk_nll_fwd(ctx, (float*)data->wptr(), input->rptr(), target->rptr(), target->dtype, input->shape[0],
                         input->shape[1], input->dtype, mean));
    else
      ck(ctx, nk_mse_fwd(ctx, (float*)data->wptr(), input->rptr(), target->rptr(), size_t(input->n()), input->dtype,
                         mean));
  }
};
struct LossBackward : Backward {  // squared_error/mod.rs:60-122, nll/mod.rs:70-133
  nk_ctx* ctx;
  TensorP input, target;
  GradientP input_grad;
  bool mean, nll;
  const char* name() const override { return nll ? "NegativeLogLikelihoodBackward" : "SquaredErrorBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (input_grad) out.push_back(input_grad->root());
  }
  void backward() override {
    const float* g = (const float*)gradient->get();
    acc_typed(ctx, input_grad, input->dtype, [&](void* d, float beta) {
      if (nll)
        ck(ctx, nk_nll_bwd(ctx, d, target->rptr(), target->dtype, g, input->shape[0], input->shape[1], input->dtype,
                           mean, beta));
      else
        ck(ctx, nk_mse_bwd(ctx, d, input->rptr(), target->rptr(), g, size_t(input->n()), input->dtype, mean, beta));
    });
  }
};

// ------------------------------------------------------------------------------- pad / conv / flatten
struct Pad : Forward {  // pad/mod.rs:63-129 with Constant / Zero modes
  nk_ctx* ctx;
  TensorP operand, data;
  int64_t ph, pw;
  float value;
  const char* name() const override { return "Pad"; }
  void forward() override {
    const Shape& s = operand->shape;
    ck(ctx, nk_pad2d_fwd(ctx, data->wptr(), operand->rptr(), s[0] * s[1], s[2], s[3], ph, pw, value, data->dtype));
  }
};
struct PadBackward : Backward {  // pad/mod.rs:131-182
  nk_ctx* ctx;
  GradientP operand_grad;
  int64_t ph, pw;
  const char* name() const override { return "PadBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    const Shape& s = operand_grad->shape;
    const void* g = gradient->get();
    acc_typed(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_pad2d_bwd(ctx, d, g, s[0] * s[1], s[2], s[3], ph, pw, gradient->dtype, beta));
    });
  }
};

struct ConvArgs {
  int64_t n, cin, h, w, cout, kh, kw, sh, sw, dh, dw, groups;
};
struct Convolution : Forward {  // convolution/mod.rs:296-355
  nk_ctx* ctx;
  TensorP input, kernel, data;
  ConvArgs a;
  const char* name() const override { return "Convolution"; }
  void forward() override { run(nullptr, nullptr); }
  void run(Tensor* bias, Tensor* out, int relu = 0) {
    Tensor* o = out ? out : data.get();
    ck(ctx, nk_conv2d_fwd(ctx, o->wptr(), input->rptr(), kernel->rptr(), bias ? bias->rptr() : nullptr, relu, a.n, a.cin,
                          a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh, a.dw, a.groups, o->dtype));
  }
};
void Addition::run_fused_conv() {
  if (fused_relu_out)
    fused_conv->run(right.get(), fused_relu_out.get(), 1);  // y = relu(conv + b) in the convolution's epilogue
  else
    fused_conv->run(right.get(), data.get());
}
struct ConvolutionBackward : Backward {  // convolution/mod.rs:357-510: input first, then kernel (:380-388)
  nk_ctx* ctx;
  TensorP input, kernel;
  GradientP input_grad, kernel_grad;
  GradientP bias_grad;  // set by the peephole when the (Cout,1,1) bias add was fused: db rides along with dW
  ConvArgs a;
  const char* name() const override { return "ConvolutionBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (input_grad) out.push_back(input_grad->root());
    if (kernel_grad) out.push_back(kernel_grad->root());
    if (bias_grad) out.push_back(bias_grad->root());
  }
  void backward() override {
    void* dbias = nullptr;
    if (bias_grad) {
      float bbeta;
      void* db = bias_grad->acc(&bbeta);
      Gradient* kr = kernel_grad ? kernel_grad->root() : nullptr;
      const float kbeta = kr ? (kr->is_zero ? 0.f : 1.f) : -1.f;
      if (kr && kbeta == bbeta && bias_grad->dtype == kernel_grad->dtype) {
        dbias = db;  // same accumulate mode and type as dW: one kernel produces both
      } else {
        const int64_t dshape[3] = {a.cout, 1, 1};
        ck(ctx, nk_unbroadcast_acc(ctx, db, bias_grad->dtype, 3, dshape, gradient->get(), gradient->dtype, 4,
                                   gradient->shape.data(), bbeta));
      }
    }
    // dX is produced in the element type of the output gradient; an input gradient of another type goes through
    // acc_typed (and then the two halves run as separate kernels)
    const bool dx_same = !input_grad || input_grad->dtype == gradient->dtype;
    Gradient* gr = gradient->root();
    if (input_grad && kernel_grad && dx_same) {  // both halves: one pass over the output gradient where the kernels allow it
      float bx, bw;
      void* dxp = input_grad->acc(&bx);
      void* dwp = kernel_grad->acc(&bw);
      int rc = NK_ERR_UNSUPPORTED;
      if (gr->is_const && (!bias_grad || dbias))
        // the output gradient is a deferred fill (backward(seed) on this convolution's own output): filled into a
        // temporary for the duration of the call
        rc = nk_conv2d_bwd_uniform(ctx, dxp, bx, dwp, kernel_grad->dtype, dbias, bw, gr->const_val, input->rptr(),
                                   kernel->rptr(), a.n, a.cin, a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh, a.dw,
                                   a.groups, gradient->dtype);
      if (rc == NK_ERR_UNSUPPORTED)
        rc = nk_conv2d_bwd(ctx, dxp, bx, dwp, kernel_grad->dtype, dbias, bw, gradient->get(), input->rptr(),
                           kernel->rptr(), a.n, a.cin, a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh, a.dw, a.groups,
                           gradient->dtype);
      ck(ctx, rc);
      grad_written(kernel_grad);
      grad_written(input_grad);
    } else {
      if (input_grad) {
        const void* g = gradient->get();
        acc_typed(ctx, input_grad, gradient->dtype, [&](void* d, float beta) {
          ck(ctx, nk_conv2d_bwd_input(ctx, d, g, kernel->rptr(), a.n, a.cin, a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw,
                                      a.dh, a.dw, a.groups, gradient->dtype, beta));
        });
        grad_written(input_grad);
      }
      if (kernel_grad) {
        float beta;
        void* d = kernel_grad->acc(&beta);
        ck(ctx, nk_conv2d_bwd_kernel(ctx, d, kernel_grad->dtype, dbias, gradient->get(), input->rptr(), a.n, a.cin,
                                     a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh, a.dw, a.groups, gradient->dtype,
                                     beta));
        grad_written(kernel_grad);
      }
    }
    if (bias_grad) grad_written(bias_grad);
  }
};

// ------------------------------------------------------------------------------- sub / mul / div (broadcasting)
// subtraction/mod.rs:11-172, multiplication/mod.rs:11-185, division/mod.rs:11-185
struct Binary : Forward {
  nk_ctx* ctx;
  TensorP left, right, data;
  int op;
  const char* name() const override {
    return op == NK_BIN_SUB ? "Subtraction" : op == NK_BIN_MUL ? "Multiplication" : "Division";
  }
  void forward() override {
    ck(ctx, nk_binary_bcast_fwd(ctx, op, data->wptr(), left->rptr(), right->rptr(), data->dtype, (int)data->shape.size(),
                                data->shape.data(), (int)left->shape.size(), left->shape.data(),
                                (int)right->shape.size(), right->shape.data()));
  }
};
struct BinaryBackward : Backward {
  nk_ctx* ctx;
  TensorP left_data, right_data;
  GradientP left_grad, right_grad;  // either may be null
  int op;
  const char* name() const override {
    return op == NK_BIN_SUB ? "SubtractionBackward" : op == NK_BIN_MUL ? "MultiplicationBackward" : "DivisionBackward";
  }
  void targets(std::vector<Gradient*>& out) override {
    if (left_grad) out.push_back(left_grad->root());
    if (right_grad) out.push_back(right_grad->root());
  }
  void side(int sd, const GradientP& dst) {
    if (!dst) return;
    float beta;
    void* d = dst->acc(&beta);
    ck(ctx, nk_binary_bcast_bwd(ctx, op, sd, d, dst->dtype, gradient->get(), left_data->rptr(), right_data->rptr(),
                                gradient->dtype, (int)left_data->shape.size(), left_data->shape.data(),
                                (int)right_data->shape.size(), right_data->shape.data(), beta));
    grad_written(dst);
  }
  void backward() override {  // left first, then right, like the composite nodes (e.g. multiplication/mod.rs:176-181)
    side(0, left_grad);
    side(1, right_grad);
  }
};

// ------------------------------------------------------------------------------- unary family
// negation, exp, logn, sqrt, sigmoid, tanh, softplus, leaky_relu, power (node/*/mod.rs; see nk_b200.h nk_unary_*)
static const char* unary_name(int op, bool bwd) {
  static const char* f[] = {"Negation", "Exp", "Logn", "Sqrt", "Sigmoid", "TanH", "SoftPlus", "LeakyReLU", "Power"};
  static const char* b[] = {"NegationBackward", "ExpBackward", "LognBackward", "SqrtBackward", "SigmoidBackward",
                            "TanHBackward", "SoftPlusBackward", "LeakyReLUBackward", "PowerBackward"};
  return (bwd ? b : f)[op];
}
struct Unary : Forward {
  nk_ctx* ctx;
  TensorP operand, data;
  int op, iparam;
  const char* name() const override { return unary_name(op, false); }
  void forward() override {
    ck(ctx, nk_unary_fwd(ctx, op, data->wptr(), operand->rptr(), size_t(data->n()), data->dtype, iparam));
  }
};
struct UnaryBackward : Backward {
  nk_ctx* ctx;
  TensorP saved;  // the node's output (exp, sqrt, sigmoid, tanh) or its input (ln, softplus, leaky_relu, powi)
  GradientP operand_grad;
  int op, iparam;
  const char* name() const override { return unary_name(op, true); }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    const void* g = gradient->get();
    const void* sv = saved ? saved->rptr() : nullptr;
    acc_typed(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_unary_bwd(ctx, op, d, sv, g, size_t(gradient->n()), gradient->dtype, iparam, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- transpose (transpose/mod.rs:11-75)
struct Transpose : Forward {
  nk_ctx* ctx;
  TensorP operand, data;
  const char* name() const override { return "Transpose"; }
  void forward() override {
    ck(ctx, nk_transpose(ctx, data->wptr(), data->dtype, operand->rptr(), operand->dtype, (int)operand->shape.size(),
                         operand->shape.data(), 0.f));
  }
};
struct TransposeBackward : Backward {
  nk_ctx* ctx;
  GradientP operand_grad;
  const char* name() const override { return "TransposeBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {  // dX += G^T
    float beta;
    void* d = operand_grad->acc(&beta);
    ck(ctx, nk_transpose(ctx, d, operand_grad->dtype, gradient->get(), gradient->dtype, (int)gradient->shape.size(),
                         gradient->shape.data(), beta));
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- n-d padding with a mode
// Pad<D, T: PaddingMode> over (N, C, s...) with 1..3 sample dims (pad/mod.rs:20-182; modes pad/{constant,zero,
// reflective,replicative}/mod.rs).  The 2-d constant case keeps its own node (Pad above).
struct PadNd : Forward {
  nk_ctx* ctx;
  TensorP operand, data;
  int nsp, mode;
  int64_t pad[3];
  float value;
  const char* name() const override { return "Pad"; }
  void forward() override {
    const Shape& s = operand->shape;
    ck(ctx, nk_padnd_fwd(ctx, data->wptr(), operand->rptr(), s[0] * s[1], nsp, s.data() + 2, pad, mode, value,
                         data->dtype));
  }
};
struct PadNdBackward : Backward {
  nk_ctx* ctx;
  GradientP operand_grad;
  int nsp;
  int64_t pad[3];
  const char* name() const override { return "PadBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    const Shape& s = operand_grad->shape;
    const void* g = gradient->get();
    acc_typed(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_padnd_bwd(ctx, d, g, s[0] * s[1], nsp, s.data() + 2, pad, gradient->dtype, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- mv / vm / vv
// matrix_vector_mul/mod.rs:11-129, vector_matrix_mul/mod.rs:11-129, vector_vector_mul/mod.rs:11-91
struct MatVec : Forward {
  nk_ctx* ctx;
  TensorP mat, vec, data;
  bool vm;  // true: y = v.A
  const char* name() const override { return vm ? "VectorMatrixMul" : "MatrixVectorMul"; }
  void forward() override {
    ck(ctx, nk_gemv(ctx, vm ? 1 : 0, mat->shape[0], mat->shape[1], mat->rptr(), vec->rptr(), 0.f, data->wptr(),
                    mat->dtype, data->dtype));
  }
};
struct MatVecBackward : Backward {
  nk_ctx* ctx;
  TensorP mat, vec;
  GradientP mat_grad, vec_grad;
  bool vm;
  const char* name() const override { return vm ? "VectorMatrixMulBackward" : "MatrixVectorMulBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (mat_grad) out.push_back(mat_grad->root());
    if (vec_grad) out.push_back(vec_grad->root());
  }
  void backward() override {
    const void* g = gradient->get();
    const int64_t rows = mat->shape[0], cols = mat->shape[1];
    auto do_mat = [&] {
      if (!mat_grad) return;
      float beta;
      void* d = mat_grad->acc(&beta);
      // mv: dA += g (x) v ; vm: dA += v (x) g
      ck(ctx, nk_outer_acc(ctx, d, mat_grad->dtype, vm ? vec->rptr() : g, vm ? g : vec->rptr(), rows, cols,
                           gradient->dtype, beta));
      grad_written(mat_grad);
    };
    auto do_vec = [&] {
      if (!vec_grad) return;
      float beta;
      void* d = vec_grad->acc(&beta);
      // mv: dv += A^T.g ; vm: dv += A.g
      ck(ctx, nk_gemv(ctx, vm ? 0 : 1, rows, cols, mat->rptr(), g, beta, d, mat->dtype, vec_grad->dtype));
      grad_written(vec_grad);
    };
    if (vm) {  // left operand first
      do_vec();
      do_mat();
    } else {
      do_mat();
      do_vec();
    }
  }
};
struct VecVec : Forward {
  nk_ctx* ctx;
  TensorP left, right, data;
  const char* name() const override { return "VectorVectorMul"; }
  void forward() override {
    ck(ctx, nk_dot(ctx, (float*)data->wptr(), left->rptr(), right->rptr(), size_t(left->n()), left->dtype));
  }
};
struct VecVecBackward : Backward {
  nk_ctx* ctx;
  TensorP left, right;
  GradientP left_grad, right_grad;
  const char* name() const override { return "VectorVectorMulBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (left_grad) out.push_back(left_grad->root());
    if (right_grad) out.push_back(right_grad->root());
  }
  void backward() override {
    const float* g = (const float*)gradient->get();
    auto one = [&](const GradientP& dst, const TensorP& other) {
      if (!dst) return;
      float beta;
      void* d = dst->acc(&beta);
      ck(ctx, nk_scale_acc(ctx, d, dst->dtype, other->rptr(), other->dtype, g, size_t(other->n()), beta));
      grad_written(dst);
    };
    one(left_grad, right);
    one(right_grad, left);
  }
};

// ------------------------------------------------------------------------------- 1-d / 3-d convolution
struct ConvNdArgs {
  int nsp;
  int64_t n, cin, cout, groups;
  int64_t in[3], k[3], s[3], d[3];
};
struct ConvolutionNd : Forward {  // convolution/mod.rs:296-355 for Ix3 / Ix5 operands
  nk_ctx* ctx;
  TensorP input, kernel, data;
  ConvNdArgs a;
  const char* name() const override { return "Convolution"; }
  void forward() override {
    ck(ctx, nk_convnd_fwd(ctx, data->wptr(), input->rptr(), kernel->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k, a.s,
                          a.d, a.groups, data->dtype));
  }
};
struct ConvolutionNdBackward : Backward {  // convolution/mod.rs:357-510
  nk_ctx* ctx;
  TensorP input, kernel;
  GradientP input_grad, kernel_grad;
  ConvNdArgs a;
  const char* name() const override { return "ConvolutionBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (input_grad) out.push_back(input_grad->root());
    if (kernel_grad) out.push_back(kernel_grad->root());
  }
  void backward() override {
    const void* g = gradient->get();
    if (input_grad) {
      acc_typed(ctx, input_grad, gradient->dtype, [&](void* d, float beta) {
        ck(ctx, nk_convnd_bwd_input(ctx, d, g, kernel->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k, a.s, a.d, a.groups,
                                    gradient->dtype, beta));
      });
      grad_written(input_grad);
    }
    if (kernel_grad) {
      float beta;
      void* d = kernel_grad->acc(&beta);
      ck(ctx, nk_convnd_bwd_kernel(ctx, d, kernel_grad->dtype, g, input->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k,
                                   a.s, a.d, a.groups, gradient->dtype, beta));
      grad_written(kernel_grad);
    }
  }
};

// ------------------------------------------------------------------------------- chunks (chunk/mod.rs)
struct Chunk : Forward {
  nk_ctx* ctx;
  TensorP operand, data;
  int64_t index;
  const char* name() const override { return "Chunk"; }
  void forward() override {
    ck(ctx, nk_chunk_fwd(ctx, data->wptr(), operand->rptr(), (int)operand->shape.size(), operand->shape.data(),
                         data->shape.data(), index, data->dtype));
  }
};
struct ChunkBackward : Backward {
  nk_ctx* ctx;
  GradientP operand_grad;
  int64_t index;
  const char* name() const override { return "ChunkBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (operand_grad) out.push_back(operand_grad->root());
  }
  void backward() override {
    // a write into one block: Gradient::acc() would let the first writer overwrite the whole buffer, so the block is
    // added onto materialised zeros (get()) instead
    void* d = operand_grad->get();
    Gradient* r = operand_grad->root();
    ck(ctx, nk_chunk_bwd(ctx, d, r->dtype, gradient->get(), gradient->dtype, (int)r->shape.size(), r->shape.data(),
                         gradient->shape.data(), index, 1.f));
    r->is_zero = false;
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- cat / stack
// MultiConcatenate / MultiStack (multi_concatenate/mod.rs, multi_stack/mod.rs) as ONE node whatever the operand count:
// operand i is an (outer, lens[i], inner) block of the output (a stacked operand has length 1 along the new axis).
struct Concatenate : Forward {
  nk_ctx* ctx;
  std::vector<TensorP> operands;
  TensorP data;
  std::vector<int64_t> lens;
  int64_t outer, inner;
  bool stack;
  const char* name() const override { return stack ? "MultiStack" : "MultiConcatenate"; }
  void forward() override {
    if (data->n() == 0) return;
    std::vector<const void*> xs;
    for (size_t i = 0; i < operands.size(); ++i) xs.push_back(lens[i] ? operands[i]->rptr() : nullptr);
    ck(ctx, nk_cat_fwd(ctx, data->wptr(), xs.data(), lens.data(), (int)lens.size(), outer, inner, data->dtype));
  }
};
struct ConcatenateBackward : Backward {
  nk_ctx* ctx;
  std::vector<GradientP> operand_grads;   // null for an operand that is not differentiable
  std::vector<int64_t> lens;
  int64_t outer, inner;
  bool stack;
  const char* name() const override { return stack ? "MultiStackBackward" : "MultiConcatenateBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    for (const GradientP& g : operand_grads)
      if (g && std::find(out.begin(), out.end(), g->root()) == out.end()) out.push_back(g->root());
  }
  void backward() override {
    // Every slice covers its operand's whole gradient, so each one accumulates with Gradient::acc()'s beta.  Operands
    // that share a gradient (x.cat([x, x]), or gradients the peephole aliased to one root) go to separate calls:
    // pass p holds the p-th occurrence of each root and adds onto what the earlier passes wrote.
    const size_t n = operand_grads.size();
    std::vector<int> pass(n, -1);
    int passes = 0;
    std::map<Gradient*, int> seen;
    for (size_t i = 0; i < n; ++i)
      if (operand_grads[i] && operand_grads[i]->n() > 0)
        passes = std::max(passes, (pass[i] = seen[operand_grads[i]->root()]++) + 1);
    if (passes == 0) return;
    const void* g = gradient->get();
    for (int p = 0; p < passes; ++p) {
      std::vector<void*> dxs(n, nullptr);
      std::vector<int> dts(n, NK_F32);
      std::vector<float> betas(n, 0.f);
      for (size_t i = 0; i < n; ++i) {
        if (pass[i] != p) continue;
        dxs[i] = operand_grads[i]->acc(&betas[i]);
        dts[i] = operand_grads[i]->root()->dtype;
      }
      ck(ctx, nk_cat_bwd(ctx, dxs.data(), dts.data(), betas.data(), g, gradient->dtype, lens.data(), (int)n, outer,
                         inner));
    }
  }
};

// ------------------------------------------------------------------------------- recurrent cells
// LSTMCell / GRUCell (neuronika-nn/src/lib.rs:450-626) as ONE forward and ONE backward node per step instead of the
// ~15 nodes the reference composes them from: the two GEMMs write the gate pre-activations in f32 (kept for the tape's
// lifetime, so a second backward() still works), one kernel applies the gates (nk_lstm_cell_fwd / nk_gru_cell_fwd).
// The backward runs the gate kernel, then the weight gradients (dW += dG^T.x, TN), the bias gradients (column sums of
// dG) and the input / state gradients (dx += dG.W, NN), only for the operands that are differentiable.
struct CellOperands {
  TensorP x, h, c, w_ih, w_hh, b_ih, b_hh;   // c: LSTM only
};
struct CellGrads {
  GradientP x, h, c, w_ih, w_hh, b_ih, b_hh;
};
struct RnnCell : Forward {
  nk_ctx* ctx;
  bool lstm;
  CellOperands o;
  TensorP gi, gh;               // f32 gate pre-activations: LSTM (N, 4H) in gi; GRU (N, 3H) in gi (input) and gh (hidden)
  TensorP h_out, c_out;
  const char* name() const override { return lstm ? "LSTMCell" : "GRUCell"; }
  void forward() override {
    const int64_t N = o.x->shape[0], I = o.x->shape[1], H = o.h->shape[1], G = o.w_ih->shape[0];
    const int dt = o.x->dtype;
    gemm(ctx, false, true, N, G, I, o.x->rptr(), I, o.w_ih->rptr(), I, 0.f, gi->wptr(), dt, NK_F32, o.b_ih->rptr(),
         o.b_ih->dtype);
    if (lstm) {
      gemm(ctx, false, true, N, G, H, o.h->rptr(), H, o.w_hh->rptr(), H, 1.f, gi->rptr(), dt, NK_F32, o.b_hh->rptr(),
           o.b_hh->dtype);
      ck(ctx, nk_lstm_cell_fwd(ctx, c_out->wptr(), h_out->wptr(), (const float*)gi->rptr(), o.c->rptr(), N, H, dt));
    } else {
      gemm(ctx, false, true, N, G, H, o.h->rptr(), H, o.w_hh->rptr(), H, 0.f, gh->wptr(), dt, NK_F32, o.b_hh->rptr(),
           o.b_hh->dtype);
      ck(ctx, nk_gru_cell_fwd(ctx, h_out->wptr(), (const float*)gi->rptr(), (const float*)gh->rptr(), o.h->rptr(), N, H,
                              dt));
    }
  }
};
// the content of a gradient nobody has written in this pass is known to be zero: the kernels take NULL for it
static const void* grad_or_null(const GradientP& g) {
  if (!g) return nullptr;
  Gradient* r = g->root();
  if (r->is_zero && !r->is_const) return nullptr;
  return g->get();
}
struct RnnCellBackward : Backward {  // `gradient` is the new hidden state's; c_out_grad the new cell state's (LSTM)
  nk_ctx* ctx;
  bool lstm;
  CellOperands o;
  CellGrads d;
  TensorP gi, gh;
  GradientP c_out_grad;
  const char* name() const override { return lstm ? "LSTMCellBackward" : "GRUCellBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    for (const GradientP* g : {&d.w_hh, &d.w_ih, &d.b_ih, &d.b_hh, &d.x, &d.h, &d.c})
      if (*g) out.push_back((*g)->root());
  }
  // dW += dG^T.A (TN).  A weight with a data-parallel reduce-scatter plan is computed locally and reported as not pushed
  // ONCE per backward pass, by its last writer: in an unrolled sequence every time step's node accumulates into the same
  // weight gradient, and the caller exchanges the whole gradient for every report it gets.
  void weight(const GradientP& g, const void* dG, const TensorP& a, int64_t G, int64_t N, int dt) {
    if (!g) return;
    float beta;
    void* p = g->acc(&beta);
    const int64_t K = a->shape[1];
    gemm(ctx, true, false, G, K, N, dG, G, a->rptr(), K, beta, p, dt, g->dtype);
    Gradient* r = g->root();
    if (r->rs_world > 1 && r->rs_hook && r->last_writer == g_bwd_pos) r->rs_hook(r->rs_user, 0);
    grad_written(g);
  }
  void bias(const GradientP& g, const void* dG, int64_t G, int64_t N, int dt) {
    if (!g) return;
    float beta;
    void* p = g->acc(&beta);
    const int64_t ds[1] = {G}, gs[2] = {N, G};
    ck(ctx, nk_unbroadcast_acc(ctx, p, g->dtype, 1, ds, dG, dt, 2, gs, beta));
    grad_written(g);
  }
  // dA += dG.W (NN)
  void input(const GradientP& g, const void* dG, const TensorP& w, int64_t G, int64_t N, int dt) {
    if (!g) return;
    float beta;
    void* p = g->acc(&beta);
    const int64_t K = w->shape[1];
    gemm(ctx, false, false, N, K, G, dG, G, w->rptr(), K, beta, p, dt, g->dtype);
    grad_written(g);
  }
  void backward() override {
    const int64_t N = o.x->shape[0], H = o.h->shape[1], G = o.w_ih->shape[0];
    const int dt = o.x->dtype;
    const size_t gbytes = size_t(N) * size_t(G) * esize(dt);
    void* dI = nullptr;
    void* dH = nullptr;
    try {
      ck(ctx, nk_alloc_uninit(ctx, gbytes, &dI));
      if (lstm) {
        const void* dh = grad_or_null(gradient);
        const void* dc = grad_or_null(c_out_grad);
        if (d.c)
          acc_typed(ctx, d.c, dt, [&](void* p, float beta) {
            ck(ctx, nk_lstm_cell_bwd(ctx, dI, dt, p, beta, (const float*)gi->rptr(), o.c->rptr(), dh, dc, N, H, dt));
          });
        else
          ck(ctx, nk_lstm_cell_bwd(ctx, dI, dt, nullptr, 0.f, (const float*)gi->rptr(), o.c->rptr(), dh, dc, N, H, dt));
        dH = dI;   // one gate gradient for both products
      } else {
        ck(ctx, nk_alloc_uninit(ctx, gbytes, &dH));
        const void* dh = gradient->get();
        if (d.h)
          acc_typed(ctx, d.h, dt, [&](void* p, float beta) {
            ck(ctx, nk_gru_cell_bwd(ctx, dI, dH, dt, p, beta, (const float*)gi->rptr(), (const float*)gh->rptr(),
                                    o.h->rptr(), dh, N, H, dt));
          });
        else
          ck(ctx, nk_gru_cell_bwd(ctx, dI, dH, dt, nullptr, 0.f, (const float*)gi->rptr(), (const float*)gh->rptr(),
                                  o.h->rptr(), dh, N, H, dt));
      }
      // the parameters first (their data-parallel exchange can then overlap the rest), as MatMulBackward does
      weight(d.w_hh, dH, o.h, G, N, dt);
      weight(d.w_ih, dI, o.x, G, N, dt);
      bias(d.b_ih, dI, G, N, dt);
      bias(d.b_hh, dH, G, N, dt);
      input(d.x, dI, o.w_ih, G, N, dt);
      input(d.h, dH, o.w_hh, G, N, dt);
      if (d.c) grad_written(d.c);
    } catch (...) {
      if (dH && dH != dI) nk_free(ctx, dH);
      if (dI) nk_free(ctx, dI);
      throw;
    }
    if (dH != dI) ck(ctx, nk_free(ctx, dH));
    ck(ctx, nk_free(ctx, dI));
  }
  void no_grad() override {
    Backward::no_grad();
    if (c_out_grad) c_out_grad->no_grad();
  }
  void with_grad() override {
    Backward::with_grad();
    if (c_out_grad) c_out_grad->with_grad();
  }
};

}  // namespace nkg

// ------------------------------------------------------------------------------- Variable (handle)
using namespace nkg;

struct nkg_var {
  nk_ctx* ctx = nullptr;
  TensorP data;
  std::map<uint64_t, ForwardP> fwd;  // History<(Rc<dyn Forward>, Cell<bool>)>
  std::vector<ForwardP> fwd_buf;
  GradientP grad;                    // null => Var
  std::map<uint64_t, BackwardP> bwd; // History<(Rc<dyn Backward>, Rc<dyn NoGrad>)>
  std::vector<BackwardP> bwd_buf;
  bool diff() const { return grad != nullptr; }
};

namespace {

nkg_var* new_like(nkg_var* a) {
  nkg_var* v = new nkg_var();
  v->ctx = a->ctx;
  return v;
}

void merge(nkg_var* dst, const nkg_var* a, const nkg_var* b = nullptr) {  // History::merge
  dst->fwd = a->fwd;
  dst->bwd = a->bwd;
  if (b) {
    dst->fwd.insert(b->fwd.begin(), b->fwd.end());
    dst->bwd.insert(b->bwd.begin(), b->bwd.end());
  }
}

uint64_t push(nkg_var* v, ForwardP op) {
  uint64_t id = g_next_op_id++;
  v->fwd[id] = std::move(op);
  return id;
}
void push_bwd(nkg_var* v, uint64_t id, BackwardP op) { v->bwd[id] = std::move(op); }

void require_same_dtype(nkg_var* a, nkg_var* b, const char* who) {
  if (a->data->dtype != b->data->dtype) fail(NK_ERR_INVALID_ARG, "%s: operands have different element types", who);
  if (a->ctx != b->ctx) fail(NK_ERR_INVALID_ARG, "%s: operands live on different devices", who);
}

Shape cobroadcast(const Shape& l, const Shape& r) {  // utils.rs:97-125
  const Shape& big = l.size() >= r.size() ? l : r;
  const Shape& small = l.size() >= r.size() ? r : l;
  Shape out = big;
  size_t off = big.size() - small.size();
  for (size_t i = 0; i < small.size(); ++i) {
    int64_t& o = out[off + i];
    if (o != small[i]) {
      if (o == 1)
        o = small[i];
      else if (small[i] != 1)
        fail(NK_ERR_INVALID_ARG, "The two tensors have incompatible shape.");
    }
  }
  return out;
}

// ---- peephole fusion, run when the tapes are materialised by forward()
void fuse(nkg_var* v) {
  if (!g_fusion) return;
  // producer lookup: output tensor -> MatMul op
  std::map<Tensor*, std::shared_ptr<MatMul>> producers;
  for (auto& kv : v->fwd)
    if (auto mm = std::dynamic_pointer_cast<MatMul>(kv.second)) producers[mm->data.get()] = mm;
  for (auto& kv : v->fwd) {
    auto add = std::dynamic_pointer_cast<Addition>(kv.second);
    if (!add || add->fused_gemm) continue;
    auto it = producers.find(add->left.get());
    if (it == producers.end()) continue;
    auto mm = it->second;
    // bias must be a (N) row broadcast of the (M,N) product, same element type; the product must have no
    // other holder than its producer and this consumer (no live variable handle, no second consumer)
    const Shape& os = add->data->shape;
    if (!mm->t || os.size() != 2 || add->right->shape.size() != 1 || add->right->shape[0] != os[1]) continue;
    if (add->right->dtype != add->data->dtype || add->left->shape != os) continue;
    if (add->left.use_count() != 2) continue;
    add->fused_gemm = mm;
    mm->skip = true;
  }
  // ... followed by ReLU: relu(mm_t + bias) in the same epilogue.  The pre-activation z is then never stored, so the
  // ReLU backward node masks with y > 0 instead of z > 0 (identical: y = max(z, 0)).
  {
    std::map<Tensor*, std::shared_ptr<Addition>> fused_adds;
    for (auto& kv : v->fwd)
      if (auto add = std::dynamic_pointer_cast<Addition>(kv.second))
        if (add->fused_gemm && !add->fused_relu_out) fused_adds[add->data.get()] = add;
    for (auto& kv : v->fwd) {
      auto relu = std::dynamic_pointer_cast<ReLU>(kv.second);
      if (!relu || relu->skip) continue;
      auto it = fused_adds.find(relu->operand.get());
      if (it == fused_adds.end()) continue;
      auto add = it->second;
      std::shared_ptr<ReLUBackward> rb;
      for (auto& kb : v->bwd)
        if (auto c = std::dynamic_pointer_cast<ReLUBackward>(kb.second))
          if (c->operand_data.get() == add->data.get()) rb = c;
      // holders of z: the Addition, the ReLU, (the ReLU backward) -- anything else (a live handle, another consumer)
      // needs z in memory
      if (add->data.use_count() != (rb ? 3 : 2)) continue;
      if (relu->data->dtype != add->data->dtype) continue;
      add->fused_relu_out = relu->data;
      relu->skip = true;
      if (rb) rb->operand_data = relu->data;
    }
  }
  // convolution + (Cout,1,1) bias add -> one kernel with a bias epilogue (the Conv2d layer's intended forward)
  std::map<Tensor*, std::shared_ptr<Convolution>> conv_producers;
  for (auto& kv : v->fwd)
    if (auto cv = std::dynamic_pointer_cast<Convolution>(kv.second)) conv_producers[cv->data.get()] = cv;
  for (auto& kv : v->fwd) {
    auto add = std::dynamic_pointer_cast<Addition>(kv.second);
    if (!add || add->fused_gemm || add->fused_conv) continue;
    auto it = conv_producers.find(add->left.get());
    if (it == conv_producers.end()) continue;
    const Shape& os = add->data->shape;
    const Shape& bs = add->right->shape;
    if (os.size() != 4 || bs.size() != 3 || bs[0] != os[1] || bs[1] != 1 || bs[2] != 1) continue;
    if (add->right->dtype != add->data->dtype || add->left->shape != os) continue;
    if (add->left.use_count() != 2) continue;
    add->fused_conv = it->second;
    it->second->skip = true;
  }
  // ... followed by ReLU: relu(conv + bias) in the convolution's epilogue, exactly as for the Linear layer above (the
  // ReLU backward masks with y > 0, identical to z > 0)
  {
    std::map<Tensor*, std::shared_ptr<Addition>> fused_adds;
    for (auto& kv : v->fwd)
      if (auto add = std::dynamic_pointer_cast<Addition>(kv.second))
        if (add->fused_conv && !add->fused_relu_out) fused_adds[add->data.get()] = add;
    for (auto& kv : v->fwd) {
      auto relu = std::dynamic_pointer_cast<ReLU>(kv.second);
      if (!relu || relu->skip || fused_adds.empty()) continue;
      auto it = fused_adds.find(relu->operand.get());
      if (it == fused_adds.end()) continue;
      auto add = it->second;
      std::shared_ptr<ReLUBackward> rb;
      for (auto& kb : v->bwd)
        if (auto c = std::dynamic_pointer_cast<ReLUBackward>(kb.second))
          if (c->operand_data.get() == add->data.get()) rb = c;
      if (add->data.use_count() != (rb ? 3 : 2)) continue;
      if (relu->data->dtype != add->data->dtype) continue;
      add->fused_relu_out = relu->data;
      relu->skip = true;
      if (rb) rb->operand_data = relu->data;
    }
  }
  // level 2: ReLU backward into the epilogue of the matmul that produces its output gradient
  if (g_fusion >= 2) {
    for (auto& kv : v->bwd) {
      auto rb = std::dynamic_pointer_cast<ReLUBackward>(kv.second);
      if (!rb || rb->skip || !rb->gradient || !rb->operand_grad) continue;
      Gradient* gh = rb->gradient.get();
      if (gh->alias || gh->ptr || gh->is_leaf || gh->hook || rb->gradient.use_count() != 2) continue;
      if (rb->operand_grad->dtype != gh->dtype || rb->operand_data->dtype != gh->dtype) continue;
      for (auto& kv2 : v->bwd) {
        auto mb = std::dynamic_pointer_cast<MatMulBackward>(kv2.second);
        if (!mb || mb->left_dst || mb->left_grad.get() != gh) continue;
        mb->left_mask = rb->operand_data;
        mb->left_dst = rb->operand_grad;
        mb->single_pass = true;
        rb->skip = true;
        // the Addition below the ReLU (z = x.W^T + b): its (K) row-bias gradient is the column sum of the dZ this GEMM
        // writes -- take it in the same epilogue when it is an f32 gradient nobody else aliases.  LEVEL 3 ONLY: correct
        // (the GPU suite runs it) and four launches fewer per config-4 step, but no faster: 0.791 vs 0.793 ms -- the
        // butterfly and the 1.3 M f32 atomics cost what the two column-sum passes did (a first version with scalar mask
        // loads was 0.2 ms SLOWER: its epilogue outlasted the main loop).  One atomic per column and CTA would be next.
        for (auto& kv3 : v->bwd) {
          if (g_fusion < 3) break;
          auto ab = std::dynamic_pointer_cast<AdditionBackward>(kv3.second);
          if (!ab || ab->skip || ab->right_fused || ab->right_aliased || !ab->right_grad) continue;
          if (ab->gradient.get() != rb->operand_grad.get()) continue;
          Gradient* bg = ab->right_grad.get();
          const Shape& gs = rb->operand_grad->shape;
          if (bg->alias || bg->dtype != NK_F32 || gs.size() != 2 || bg->shape.size() != 1 || bg->shape[0] != gs[1]) continue;
          mb->left_colsum = ab->right_grad;
          ab->right_fused = true;
          break;
        }
        break;
      }
    }
  }
  // gradient aliasing: dL += G with identical shape/dtype and a single consumer => L.grad is G
  for (auto& kv : v->bwd) {
    auto ab = std::dynamic_pointer_cast<AdditionBackward>(kv.second);
    if (!ab) continue;
    auto try_alias = [&](GradientP& g, bool& flag) {
      if (!g || flag || g->alias || g->ptr) return;
      if (g->shape != ab->gradient->shape || g->dtype != ab->gradient->dtype) return;
      if (!g->owned) return;
      // only a gradient produced by a Backward node may be aliased: a leaf's gradient belongs to the user (hooks and
      // reduce-scatter plans sit on it, it accumulates over backward() calls and outlives this graph)
      if (g->is_leaf || g->hook || g->rs_world > 1) return;
      if (g.use_count() != 2) return;  // the producer's Backward node + this node
      g->alias = ab->gradient;
      flag = true;
    };
    try_alias(ab->left_grad, ab->left_aliased);
  }
  // bias gradient of a fused Conv2d: let the dW kernel produce it (its all-ones K-row) instead of re-reading G
  for (auto& kv : v->bwd) {
    auto ab = std::dynamic_pointer_cast<AdditionBackward>(kv.second);
    if (!ab || !ab->left_aliased || ab->right_aliased || !ab->right_grad) continue;
    const Shape& bs = ab->right_grad->shape;
    if (ab->gradient->shape.size() != 4 || bs.size() != 3 || bs[0] != ab->gradient->shape[1] || bs[1] != 1 || bs[2] != 1)
      continue;
    for (auto& kv2 : v->bwd) {
      auto cb = std::dynamic_pointer_cast<ConvolutionBackward>(kv2.second);
      if (!cb || cb->bias_grad || cb->gradient->root() != ab->gradient->root()) continue;
      cb->bias_grad = ab->right_grad;
      ab->right_aliased = true;
      break;
    }
  }
}

void materialise(nkg_var* v) {
  if (v->fwd_buf.size() != v->fwd.size()) {
    fuse(v);
    v->fwd_buf.clear();
    for (auto& kv : v->fwd) v->fwd_buf.push_back(kv.second);
  }
  if (v->bwd_buf.size() != v->bwd.size()) {
    v->bwd_buf.clear();
    for (auto& kv : v->bwd) v->bwd_buf.push_back(kv.second);
  }
}

template <typename F>
int guard(F&& f) {
  try {
    f();
    return NK_OK;
  } catch (const Error& e) {
    g_error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_error = e.what();
    return NK_ERR_INVALID_ARG;
  }
}

nkg_var* unary_node(nkg_var* a, const Shape& out_shape, int out_dtype, TensorP& out_data) {
  nkg_var* v = new_like(a);
  merge(v, a);
  out_data = std::make_shared<Tensor>(a->ctx, out_shape, out_dtype);
  v->data = out_data;
  return v;
}

// a view: the operand's memory and tapes under another shape (no kernel, no node); the gradient of a view is the same
// memory with the view's shape
nkg_var* view_of(nkg_var* a, const Shape& shape) {
  nkg_var* v = new nkg_var(*a);
  auto t = std::make_shared<Tensor>(a->ctx, shape, a->data->dtype);
  t->base = a->data;
  t->owned = false;
  v->data = t;
  if (a->diff()) {
    auto g = std::make_shared<Gradient>(a->ctx, shape, a->grad->dtype);
    g->alias = a->grad;
    v->grad = g;
  }
  v->fwd_buf.clear();
  v->bwd_buf.clear();
  return v;
}

}  // namespace

extern "C" {

const char* nkg_last_error(void) { return g_error.c_str(); }

int nkg_set_fusion(int level) {
  g_fusion = level < 0 ? 0 : (level > 3 ? 3 : level);
  return NK_OK;
}

int nkg_leaf(nk_ctx* ctx, int ndim, const int64_t* shape, int dtype, nkg_var** out) {
  return guard([&] {
    if (!ctx || !out || ndim < 0 || ndim > NK_MAX_DIMS) fail(NK_ERR_INVALID_ARG, "nkg_leaf: bad arguments");
    if (dtype != NK_F32 && dtype != NK_BF16) fail(NK_ERR_INVALID_ARG, "nkg_leaf: bad dtype %d", dtype);
    nkg_var* v = new nkg_var();
    v->ctx = ctx;
    v->data = std::make_shared<Tensor>(ctx, Shape(shape, shape + ndim), dtype);
    v->data->wptr();  // leaves are allocated (zero-filled) eagerly
    *out = v;
  });
}

int nkg_leaf_external(nk_ctx* ctx, int ndim, const int64_t* shape, int dtype, void* data_ptr, nkg_var** out) {
  return guard([&] {
    if (!ctx || !out || !data_ptr || ndim < 0 || ndim > NK_MAX_DIMS)
      fail(NK_ERR_INVALID_ARG, "nkg_leaf_external: bad arguments");
    nkg_var* v = new nkg_var();
    v->ctx = ctx;
    v->data = std::make_shared<Tensor>(ctx, Shape(shape, shape + ndim), dtype);
    v->data->ptr = data_ptr;
    v->data->owned = false;
    *out = v;
  });
}

int nkg_requires_grad(nkg_var* a, int grad_dtype, void* grad_ptr, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "nkg_requires_grad: NULL");
    nkg_var* v = new nkg_var(*a);  // shares data and forward tape (VarDiff::leaf(self, zeros))
    v->grad = std::make_shared<Gradient>(a->ctx, a->data->shape, grad_dtype < 0 ? a->data->dtype : grad_dtype);
    v->grad->is_leaf = true;
    if (grad_ptr) {
      v->grad->ptr = grad_ptr;
      v->grad->owned = false;
      v->grad->is_zero = false;  // caller-owned memory: contents unknown
    }
    v->bwd.clear();
    v->bwd_buf.clear();
    *out = v;
  });
}

int nkg_clone(nkg_var* a, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "nkg_clone: NULL");
    *out = new nkg_var(*a);
  });
}

int nkg_release(nkg_var* v) {
  delete v;
  return NK_OK;
}

int nkg_is_diff(nkg_var* v) { return v && v->diff(); }
int nkg_ndim(nkg_var* v) { return v ? (int)v->data->shape.size() : -1; }
int nkg_shape(nkg_var* v, int64_t* s) {
  if (!v || !s) return NK_ERR_INVALID_ARG;
  for (size_t i = 0; i < v->data->shape.size(); ++i) s[i] = v->data->shape[i];
  return NK_OK;
}
int nkg_dtype(nkg_var* v) { return v ? v->data->dtype : -1; }
int nkg_grad_dtype(nkg_var* v) { return v && v->grad ? v->grad->dtype : -1; }
void* nkg_data_ptr(nkg_var* v) {
  void* p = nullptr;
  guard([&] { p = v ? v->data->rptr() : nullptr; });
  return p;
}
void* nkg_grad_ptr(nkg_var* v) {
  void* p = nullptr;
  guard([&] {
    if (v && v->grad && v->grad->root()->enabled) p = v->grad->get();
  });
  return p;
}
int nkg_history_len(nkg_var* v) { return v ? (int)v->fwd.size() : -1; }
int nkg_backward_history_len(nkg_var* v) { return v ? (int)v->bwd.size() : -1; }

int nkg_forward(nkg_var* v) {
  return guard([&] {
    if (!v) fail(NK_ERR_INVALID_ARG, "nkg_forward: NULL");
    materialise(v);
    for (auto& op : v->fwd_buf)
      if (!op->skip) op->forward();
  });
}

int nkg_backward(nkg_var* v, float seed) {
  return guard([&] {
    if (!v || !v->diff()) fail(NK_ERR_INVALID_ARG, "nkg_backward: not a differentiable variable");
    if (v->fwd_buf.size() != v->fwd.size() || v->bwd_buf.size() != v->bwd.size())
      fail(NK_ERR_INVALID_ARG, "Perhaps you forgot to call .forward()?");  // vardiff.rs:126-130
    // The aliasing peephole (dL += G with one consumer => L.grad IS G) is exact for ONE backward pass per tape.  The
    // reference accumulates into every gradient, intermediates included, on every pass (nothing zeroes them), so on a
    // repeated backward() the addend's gradient and the sum's gradient diverge: give the addend its own buffer, holding
    // what the reference would hold after the passes so far (= the sum's gradient at the end of the last pass).
    for (auto& op : v->bwd_buf)
      if (op->single_pass && op->runs > 0)
        fail(NK_ERR_UNSUPPORTED, "this tape was optimised for ONE backward pass (fusion level 2: %s never stores the "
             "gradient it would have to accumulate); build the graph again or use nkg_set_fusion(1)", op->name());
    for (auto& op : v->bwd_buf) {
      auto ab = std::dynamic_pointer_cast<AdditionBackward>(op);
      if (!ab || !ab->left_aliased || ab->runs == 0 || !ab->left_grad || !ab->left_grad->alias) continue;
      Gradient* g = ab->left_grad.get();
      Gradient* src = g->root();
      const size_t bytes = size_t(g->n()) * esize(g->dtype);
      void* own = nullptr;
      ck(g->ctx, nk_alloc_uninit(g->ctx, bytes, &own));
      ck(g->ctx, nk_d2d(g->ctx, own, src->get(), bytes));
      g->alias.reset();
      g->ptr = own;
      g->owned = true;
      g->is_zero = false;
      g->stale = false;
      ab->left_aliased = false;
      if (ab->right_aliased) {  // the bias gradient rode along with the convolution's dW: back to its own un-broadcast
        for (auto& op2 : v->bwd_buf)
          if (auto cb = std::dynamic_pointer_cast<ConvolutionBackward>(op2))
            if (cb->bias_grad == ab->right_grad) cb->bias_grad.reset();
        ab->right_aliased = false;
      }
    }
    v->grad->fill(seed);
    // last writer (reverse tape position) of every hooked gradient in this pass
    std::vector<Gradient*> tg;
    bool any_hook = false;
    int pos = 0;
    static thread_local uint64_t pass_counter = 0;
    const uint64_t pass = ++pass_counter;
    for (auto it = v->bwd_buf.rbegin(); it != v->bwd_buf.rend(); ++it, ++pos) {
      if ((*it)->skip) continue;
      tg.clear();
      (*it)->targets(tg);
      for (Gradient* g : tg)
        if (g->hook || g->rs_world > 1) {
          if (g->pass_id != pass) {
            g->pass_id = pass;
            g->writers = 0;
          }
          ++g->writers;
          g->last_writer = pos;
          g->hook_fired = false;
          any_hook = true;
        }
    }
    pos = 0;
    for (auto it = v->bwd_buf.rbegin(); it != v->bwd_buf.rend(); ++it, ++pos) {
      g_bwd_pos = any_hook ? pos : -2;
      if (!(*it)->skip) {
        (*it)->backward();
        (*it)->runs++;
      }
      if (any_hook) {  // nodes that do not report their writes individually: fire at node granularity
        tg.clear();
        (*it)->targets(tg);
        for (Gradient* g : tg)
          if (g->hook && g->last_writer == pos && !g->hook_fired) {
            g->hook_fired = true;
            g->hook(g->hook_user, 0, g->n());
          }
      }
    }
    g_bwd_pos = -1;
  });
}

int nkg_zero_grad(nkg_var* v) {
  return guard([&] {
    if (!v || !v->diff()) fail(NK_ERR_INVALID_ARG, "nkg_zero_grad: not a differentiable variable");
    v->grad->zero();
  });
}

int nkg_no_grad(nkg_var* v) {
  return guard([&] {
    if (!v || !v->diff()) fail(NK_ERR_INVALID_ARG, "nkg_no_grad: not a differentiable variable");
    materialise(v);
    for (auto& op : v->bwd_buf) op->no_grad();
  });
}

int nkg_with_grad(nkg_var* v) {
  return guard([&] {
    if (!v || !v->diff()) fail(NK_ERR_INVALID_ARG, "nkg_with_grad: not a differentiable variable");
    materialise(v);
    for (auto& op : v->bwd_buf) op->with_grad();
  });
}

// ---------------------------------------------------------------- operators
static int matmul_impl(nkg_var* a, nkg_var* b, bool t, nkg_var** out) {
  return guard([&] {
    if (!a || !b || !out) fail(NK_ERR_INVALID_ARG, "mm: NULL");
    require_same_dtype(a, b, t ? "mm_t" : "mm");
    const Shape &ls = a->data->shape, &rs = b->data->shape;
    if (ls.size() != 2 || rs.size() != 2) fail(NK_ERR_INVALID_ARG, "mm: operands must be 2-dimensional");
    const int64_t inner_r = t ? rs[1] : rs[0];
    if (ls[1] != inner_r)
      fail(NK_ERR_INVALID_ARG, "mm: incompatible shapes (%lld, %lld) and (%lld, %lld)%s", (long long)ls[0],
           (long long)ls[1], (long long)rs[0], (long long)rs[1], t ? " (transposed rhs)" : "");
    nkg_var* v = new_like(a);
    merge(v, a, b);
    Shape os{ls[0], t ? rs[0] : rs[1]};
    v->data = std::make_shared<Tensor>(a->ctx, os, a->data->dtype);
    uint64_t id = push(v, std::make_shared<MatMul>(a->ctx, a->data, b->data, v->data, t));
    if (a->diff() || b->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, os, a->data->dtype);
      auto bw = std::make_shared<MatMulBackward>();
      bw->ctx = a->ctx;
      bw->t = t;
      bw->gradient = v->grad;
      bw->left_data = a->data;
      bw->right_data = b->data;
      bw->left_grad = a->grad;   // null when the operand is a Var: that half is never built
      bw->right_grad = b->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_mm(nkg_var* a, nkg_var* b, nkg_var** out) { return matmul_impl(a, b, false, out); }
int nkg_mm_t(nkg_var* a, nkg_var* b, nkg_var** out) { return matmul_impl(a, b, true, out); }

int nkg_add(nkg_var* a, nkg_var* b, nkg_var** out) {
  return guard([&] {
    if (!a || !b || !out) fail(NK_ERR_INVALID_ARG, "add: NULL");
    require_same_dtype(a, b, "add");
    Shape os = cobroadcast(a->data->shape, b->data->shape);
    nkg_var* v = new_like(a);
    merge(v, a, b);
    v->data = std::make_shared<Tensor>(a->ctx, os, a->data->dtype);
    auto op = std::make_shared<Addition>();
    op->ctx = a->ctx;
    op->left = a->data;
    op->right = b->data;
    op->data = v->data;
    uint64_t id = push(v, op);
    if (a->diff() || b->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, os, a->data->dtype);
      auto bw = std::make_shared<AdditionBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->left_grad = a->grad;
      bw->right_grad = b->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_relu(nkg_var* a, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "relu: NULL");
    TensorP od;
    nkg_var* v = unary_node(a, a->data->shape, a->data->dtype, od);
    auto op = std::make_shared<ReLU>();
    op->ctx = a->ctx;
    op->operand = a->data;
    op->data = od;
    uint64_t id = push(v, op);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, od->shape, od->dtype);
      auto bw = std::make_shared<ReLUBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_data = a->data;
      bw->operand_grad = a->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

static int softmax_impl(nkg_var* a, int axis, bool log, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "softmax: NULL");
    if (axis < 0 || axis >= (int)a->data->shape.size()) fail(NK_ERR_INVALID_ARG, "softmax: axis %d out of range", axis);
    TensorP od;
    nkg_var* v = unary_node(a, a->data->shape, a->data->dtype, od);
    auto op = std::make_shared<Softmax>();
    op->ctx = a->ctx;
    op->operand = a->data;
    op->data = od;
    op->axis = axis;
    op->log = log;
    uint64_t id = push(v, op);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, od->shape, od->dtype);
      auto bw = std::make_shared<SoftmaxBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->data = od;
      bw->operand_grad = a->grad;
      bw->axis = axis;
      bw->log = log;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_softmax(nkg_var* a, int axis, nkg_var** out) { return softmax_impl(a, axis, false, out); }
int nkg_log_softmax(nkg_var* a, int axis, nkg_var** out) { return softmax_impl(a, axis, true, out); }

static int summean_impl(nkg_var* a, bool mean, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "sum: NULL");
    TensorP od;
    nkg_var* v = unary_node(a, Shape{}, NK_F32, od);
    auto op = std::make_shared<SumMean>();
    op->ctx = a->ctx;
    op->operand = a->data;
    op->data = od;
    op->mean = mean;
    uint64_t id = push(v, op);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, Shape{}, NK_F32);
      auto bw = std::make_shared<SumMeanBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_grad = a->grad;
      bw->mean = mean;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_sum(nkg_var* a, nkg_var** out) { return summean_impl(a, false, out); }
int nkg_mean(nkg_var* a, nkg_var** out) { return summean_impl(a, true, out); }

static int loss_impl(nkg_var* input, nkg_var* target, int reduction, bool nll, nkg_var** out) {
  return guard([&] {
    if (!input || !target || !out) fail(NK_ERR_INVALID_ARG, "loss: NULL");
    if (nll) {
      // class ids are stored as floats (nll/mod.rs:55 `target as usize`): an f32 target is accepted whatever the
      // input's element type; a bf16 target represents integers exactly only up to 256
      if (input->ctx != target->ctx) fail(NK_ERR_INVALID_ARG, "nll_loss: operands live on different devices");
      if (target->data->dtype == NK_BF16 && input->data->shape.size() == 2 && input->data->shape[1] > 256)
        fail(NK_ERR_INVALID_ARG, "nll_loss: a bf16 target cannot hold class ids above 256; pass the target as f32");
    } else {
      require_same_dtype(input, target, "mse_loss");
    }
    if (nll) {
      if (input->data->shape.size() != 2 || target->data->shape.size() != 1 ||
          target->data->shape[0] != input->data->shape[0])
        fail(NK_ERR_INVALID_ARG, "nll_loss: input must be (N, C) and target (N)");
    } else if (input->data->shape != target->data->shape) {
      fail(NK_ERR_INVALID_ARG, "mse_loss: input and target shapes differ");
    }
    if (target->diff()) fail(NK_ERR_INVALID_ARG, "loss: the target must not be differentiable");
    nkg_var* v = new_like(input);
    merge(v, input, target);
    v->data = std::make_shared<Tensor>(input->ctx, Shape{}, NK_F32);
    auto op = std::make_shared<Loss>();
    op->ctx = input->ctx;
    op->input = input->data;
    op->target = target->data;
    op->data = v->data;
    op->mean = reduction == NKG_MEAN;
    op->nll = nll;
    uint64_t id = push(v, op);
    if (input->diff()) {
      v->grad = std::make_shared<Gradient>(input->ctx, Shape{}, NK_F32);
      auto bw = std::make_shared<LossBackward>();
      bw->ctx = input->ctx;
      bw->gradient = v->grad;
      bw->input = input->data;
      bw->target = target->data;
      bw->input_grad = input->grad;
      bw->mean = op->mean;
      bw->nll = nll;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_mse_loss(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, false, o); }
int nkg_nll_loss(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, true, o); }

int nkg_pad(nkg_var* a, int64_t ph, int64_t pw, float value, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "pad: NULL");
    const Shape& s = a->data->shape;
    if (s.size() != 4 || ph < 0 || pw < 0) fail(NK_ERR_INVALID_ARG, "pad: expects a (N, C, H, W) operand and padding >= 0");
    TensorP od;
    nkg_var* v = unary_node(a, Shape{s[0], s[1], s[2] + 2 * ph, s[3] + 2 * pw}, a->data->dtype, od);
    auto op = std::make_shared<Pad>();
    op->ctx = a->ctx;
    op->operand = a->data;
    op->data = od;
    op->ph = ph;
    op->pw = pw;
    op->value = value;
    uint64_t id = push(v, op);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, od->shape, od->dtype);
      auto bw = std::make_shared<PadBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_grad = a->grad;
      bw->ph = ph;
      bw->pw = pw;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_convolution(nkg_var* kernel, nkg_var* input, int64_t sh, int64_t sw, int64_t dh, int64_t dw, int64_t groups,
                    nkg_var** out) {
  return guard([&] {
    if (!kernel || !input || !out) fail(NK_ERR_INVALID_ARG, "convolution: NULL");
    require_same_dtype(kernel, input, "convolution");
    const Shape &ks = kernel->data->shape, &is = input->data->shape;
    // check_conv_args / check_groups_args, utils.rs:427-496 (same messages)
    if (is.size() != 4) fail(NK_ERR_UNSUPPORTED, "convolution: only 2d convolutions (N, C, H, W) run on the device");
    if (ks.size() != is.size()) fail(NK_ERR_INVALID_ARG, "Invalid kernel shape for 2d conv");
    if (sh < 1 || sw < 1 || dh < 1 || dw < 1 || groups < 1) fail(NK_ERR_INVALID_ARG, "Invalid stride/dilation/groups for 2d conv.");
    if (is[2] < (ks[2] - 1) * dh + 1 || is[3] < (ks[3] - 1) * dw + 1)
      fail(NK_ERR_INVALID_ARG, "The kernel size can't be greater than actual input size.");
    if (is[1] % groups) fail(NK_ERR_INVALID_ARG, "In channels %lld is not divisible by groups %lld", (long long)is[1], (long long)groups);
    if (ks[0] % groups) fail(NK_ERR_INVALID_ARG, "Out channels %lld is not divisible by groups %lld", (long long)ks[0], (long long)groups);
    if (ks[1] * groups != is[1]) fail(NK_ERR_INVALID_ARG, "convolution: kernel in-channels %lld x groups %lld != input channels %lld", (long long)ks[1], (long long)groups, (long long)is[1]);
    ConvArgs a{is[0], is[1], is[2], is[3], ks[0], ks[2], ks[3], sh, sw, dh, dw, groups};
    Shape os{is[0], ks[0], (is[2] - dh * (ks[2] - 1) - 1) / sh + 1, (is[3] - dw * (ks[3] - 1) - 1) / sw + 1};
    nkg_var* v = new_like(kernel);
    merge(v, kernel, input);
    v->data = std::make_shared<Tensor>(kernel->ctx, os, input->data->dtype);
    auto op = std::make_shared<Convolution>();
    op->ctx = kernel->ctx;
    op->input = input->data;
    op->kernel = kernel->data;
    op->data = v->data;
    op->a = a;
    uint64_t id = push(v, op);
    if (kernel->diff() || input->diff()) {
      v->grad = std::make_shared<Gradient>(kernel->ctx, os, input->data->dtype);
      auto bw = std::make_shared<ConvolutionBackward>();
      bw->ctx = kernel->ctx;
      bw->gradient = v->grad;
      bw->input = input->data;
      bw->kernel = kernel->data;
      bw->input_grad = input->grad;
      bw->kernel_grad = kernel->grad;
      bw->a = a;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_flatten(nkg_var* a, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "flatten: NULL");
    const Shape& s = a->data->shape;
    if (s.size() < 2) fail(NK_ERR_INVALID_ARG, "flatten: needs at least 2 dimensions");
    int64_t rest = 1;
    for (size_t i = 1; i < s.size(); ++i) rest *= s[i];
    *out = view_of(a, Shape{s[0], rest});
  });
}

// ---------------------------------------------------------------- 8-f operators
static int binary_impl(nkg_var* a, nkg_var* b, int op, nkg_var** out) {
  return guard([&] {
    if (!a || !b || !out) fail(NK_ERR_INVALID_ARG, "binary op: NULL");
    require_same_dtype(a, b, op == NK_BIN_SUB ? "sub" : op == NK_BIN_MUL ? "mul" : "div");
    Shape os = cobroadcast(a->data->shape, b->data->shape);
    nkg_var* v = new_like(a);
    merge(v, a, b);
    v->data = std::make_shared<Tensor>(a->ctx, os, a->data->dtype);
    auto fw = std::make_shared<Binary>();
    fw->ctx = a->ctx;
    fw->left = a->data;
    fw->right = b->data;
    fw->data = v->data;
    fw->op = op;
    uint64_t id = push(v, fw);
    if (a->diff() || b->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, os, a->data->dtype);
      auto bw = std::make_shared<BinaryBackward>();
      bw->ctx = a->ctx;
      bw->op = op;
      bw->gradient = v->grad;
      bw->left_data = a->data;
      bw->right_data = b->data;
      bw->left_grad = a->grad;
      bw->right_grad = b->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_sub(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_SUB, out); }
int nkg_mul(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_MUL, out); }
int nkg_div(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_DIV, out); }

int nkg_unary(nkg_var* a, int op, int iparam, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "unary op: NULL");
    if (op < NK_UN_NEG || op > NK_UN_POWI) fail(NK_ERR_INVALID_ARG, "unary op: bad op %d", op);
    TensorP od;
    nkg_var* v = unary_node(a, a->data->shape, a->data->dtype, od);
    auto fw = std::make_shared<Unary>();
    fw->ctx = a->ctx;
    fw->operand = a->data;
    fw->data = od;
    fw->op = op;
    fw->iparam = iparam;
    uint64_t id = push(v, fw);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, od->shape, od->dtype);
      auto bw = std::make_shared<UnaryBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_grad = a->grad;
      bw->op = op;
      bw->iparam = iparam;
      const bool keeps_output = op == NK_UN_EXP || op == NK_UN_SQRT || op == NK_UN_SIGMOID || op == NK_UN_TANH;
      bw->saved = op == NK_UN_NEG ? nullptr : (keeps_output ? od : a->data);
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_neg(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_NEG, 0, out); }
int nkg_exp(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_EXP, 0, out); }
int nkg_ln(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_LN, 0, out); }
int nkg_sqrt(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_SQRT, 0, out); }
int nkg_sigmoid(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_SIGMOID, 0, out); }
int nkg_tanh(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_TANH, 0, out); }
int nkg_softplus(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_SOFTPLUS, 0, out); }
int nkg_leaky_relu(nkg_var* a, nkg_var** out) { return nkg_unary(a, NK_UN_LEAKY_RELU, 0, out); }
int nkg_pow(nkg_var* a, int exp, nkg_var** out) { return nkg_unary(a, NK_UN_POWI, exp, out); }

int nkg_transpose(nkg_var* a, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "t: NULL");
    Shape os(a->data->shape.rbegin(), a->data->shape.rend());
    TensorP od;
    nkg_var* v = unary_node(a, os, a->data->dtype, od);
    auto fw = std::make_shared<Transpose>();
    fw->ctx = a->ctx;
    fw->operand = a->data;
    fw->data = od;
    uint64_t id = push(v, fw);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, os, od->dtype);
      auto bw = std::make_shared<TransposeBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_grad = a->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_pad_mode(nkg_var* a, int nsp, const int64_t* padding, int mode, float value, nkg_var** out) {
  return guard([&] {
    if (!a || !out || !padding) fail(NK_ERR_INVALID_ARG, "pad: NULL");
    const Shape& s = a->data->shape;
    if (nsp < 1 || nsp > 3 || (int)s.size() != nsp + 2)
      fail(NK_ERR_INVALID_ARG, "pad: expects a (N, C, ...) operand with %d sample dimensions", nsp);
    if (mode < NK_PAD_CONSTANT || mode > NK_PAD_REPLICATIVE) fail(NK_ERR_INVALID_ARG, "pad: bad mode %d", mode);
    Shape os = s;
    for (int k = 0; k < nsp; ++k) {
      if (padding[k] < 0) fail(NK_ERR_INVALID_ARG, "pad: padding must be >= 0");
      if (mode == NK_PAD_REFLECTIVE && padding[k] > 0 && padding[k] >= s[2 + k])
        fail(NK_ERR_INVALID_ARG, "pad: reflective padding %lld must be smaller than the dimension %lld",
             (long long)padding[k], (long long)s[2 + k]);
      os[2 + k] += 2 * padding[k];
    }
    TensorP od;
    nkg_var* v = unary_node(a, os, a->data->dtype, od);
    auto fw = std::make_shared<PadNd>();
    fw->ctx = a->ctx;
    fw->operand = a->data;
    fw->data = od;
    fw->nsp = nsp;
    fw->mode = mode;
    fw->value = value;
    for (int k = 0; k < 3; ++k) fw->pad[k] = k < nsp ? padding[k] : 0;
    uint64_t id = push(v, fw);
    if (a->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, os, od->dtype);
      auto bw = std::make_shared<PadNdBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->operand_grad = a->grad;
      bw->nsp = nsp;
      for (int k = 0; k < 3; ++k) bw->pad[k] = fw->pad[k];
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

static int matvec_impl(nkg_var* mat, nkg_var* vec, bool vm, nkg_var** out) {
  return guard([&] {
    if (!mat || !vec || !out) fail(NK_ERR_INVALID_ARG, "mv: NULL");
    require_same_dtype(mat, vec, vm ? "vm" : "mv");
    const Shape &ms = mat->data->shape, &vs = vec->data->shape;
    if (ms.size() != 2 || vs.size() != 1) fail(NK_ERR_INVALID_ARG, "%s: needs a matrix and a vector", vm ? "vm" : "mv");
    const int64_t need = vm ? ms[0] : ms[1];
    if (vs[0] != need)
      fail(NK_ERR_INVALID_ARG, "%s: incompatible shapes (%lld, %lld) and (%lld)", vm ? "vm" : "mv", (long long)ms[0],
           (long long)ms[1], (long long)vs[0]);
    nkg_var* first = vm ? vec : mat;
    nkg_var* second = vm ? mat : vec;
    nkg_var* v = new_like(first);
    merge(v, first, second);
    Shape os{vm ? ms[1] : ms[0]};
    v->data = std::make_shared<Tensor>(mat->ctx, os, mat->data->dtype);
    auto fw = std::make_shared<MatVec>();
    fw->ctx = mat->ctx;
    fw->mat = mat->data;
    fw->vec = vec->data;
    fw->data = v->data;
    fw->vm = vm;
    uint64_t id = push(v, fw);
    if (mat->diff() || vec->diff()) {
      v->grad = std::make_shared<Gradient>(mat->ctx, os, mat->data->dtype);
      auto bw = std::make_shared<MatVecBackward>();
      bw->ctx = mat->ctx;
      bw->gradient = v->grad;
      bw->mat = mat->data;
      bw->vec = vec->data;
      bw->mat_grad = mat->grad;
      bw->vec_grad = vec->grad;
      bw->vm = vm;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}
int nkg_mv(nkg_var* mat, nkg_var* vec, nkg_var** out) { return matvec_impl(mat, vec, false, out); }
int nkg_vm(nkg_var* vec, nkg_var* mat, nkg_var** out) { return matvec_impl(mat, vec, true, out); }

int nkg_vv(nkg_var* a, nkg_var* b, nkg_var** out) {
  return guard([&] {
    if (!a || !b || !out) fail(NK_ERR_INVALID_ARG, "vv: NULL");
    require_same_dtype(a, b, "vv");
    if (a->data->shape.size() != 1 || b->data->shape.size() != 1 || a->data->shape[0] != b->data->shape[0])
      fail(NK_ERR_INVALID_ARG, "vv: needs two vectors of the same length");
    nkg_var* v = new_like(a);
    merge(v, a, b);
    v->data = std::make_shared<Tensor>(a->ctx, Shape{}, NK_F32);
    auto fw = std::make_shared<VecVec>();
    fw->ctx = a->ctx;
    fw->left = a->data;
    fw->right = b->data;
    fw->data = v->data;
    uint64_t id = push(v, fw);
    if (a->diff() || b->diff()) {
      v->grad = std::make_shared<Gradient>(a->ctx, Shape{}, NK_F32);
      auto bw = std::make_shared<VecVecBackward>();
      bw->ctx = a->ctx;
      bw->gradient = v->grad;
      bw->left = a->data;
      bw->right = b->data;
      bw->left_grad = a->grad;
      bw->right_grad = b->grad;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

int nkg_convolution_nd(nkg_var* kernel, nkg_var* input, int nsp, const int64_t* stride, const int64_t* dilation,
                       int64_t groups, nkg_var** out) {
  return guard([&] {
    if (!kernel || !input || !out || !stride || !dilation) fail(NK_ERR_INVALID_ARG, "convolution: NULL");
    if (nsp == 2)
      fail(NK_ERR_INVALID_ARG, "convolution: use nkg_convolution for 2d operands");
    require_same_dtype(kernel, input, "convolution");
    const Shape &ks = kernel->data->shape, &is = input->data->shape;
    if (nsp < 1 || nsp > 3 || (int)is.size() != nsp + 2) fail(NK_ERR_INVALID_ARG, "convolution: input rank does not match %dd conv", nsp);
    if (ks.size() != is.size()) fail(NK_ERR_INVALID_ARG, "Invalid kernel shape for %dd conv", nsp);
    if (groups < 1) fail(NK_ERR_INVALID_ARG, "Invalid groups for %dd conv.", nsp);
    ConvNdArgs a;
    a.nsp = nsp, a.n = is[0], a.cin = is[1], a.cout = ks[0], a.groups = groups;
    Shape os{is[0], ks[0]};
    for (int k = 0; k < 3; ++k) a.in[k] = a.k[k] = a.s[k] = a.d[k] = 1;
    for (int k = 0; k < nsp; ++k) {
      if (stride[k] < 1 || dilation[k] < 1) fail(NK_ERR_INVALID_ARG, "Invalid stride/dilation for %dd conv.", nsp);
      if (is[2 + k] < (ks[2 + k] - 1) * dilation[k] + 1)
        fail(NK_ERR_INVALID_ARG, "The kernel size can't be greater than actual input size.");
      a.in[k] = is[2 + k], a.k[k] = ks[2 + k], a.s[k] = stride[k], a.d[k] = dilation[k];
      os.push_back((is[2 + k] - dilation[k] * (ks[2 + k] - 1) - 1) / stride[k] + 1);
    }
    if (is[1] % groups) fail(NK_ERR_INVALID_ARG, "In channels %lld is not divisible by groups %lld", (long long)is[1], (long long)groups);
    if (ks[0] % groups) fail(NK_ERR_INVALID_ARG, "Out channels %lld is not divisible by groups %lld", (long long)ks[0], (long long)groups);
    if (ks[1] * groups != is[1]) fail(NK_ERR_INVALID_ARG, "convolution: kernel in-channels %lld x groups %lld != input channels %lld", (long long)ks[1], (long long)groups, (long long)is[1]);
    nkg_var* v = new_like(kernel);
    merge(v, kernel, input);
    v->data = std::make_shared<Tensor>(kernel->ctx, os, input->data->dtype);
    auto fw = std::make_shared<ConvolutionNd>();
    fw->ctx = kernel->ctx;
    fw->input = input->data;
    fw->kernel = kernel->data;
    fw->data = v->data;
    fw->a = a;
    uint64_t id = push(v, fw);
    if (kernel->diff() || input->diff()) {
      v->grad = std::make_shared<Gradient>(kernel->ctx, os, input->data->dtype);
      auto bw = std::make_shared<ConvolutionNdBackward>();
      bw->ctx = kernel->ctx;
      bw->gradient = v->grad;
      bw->input = input->data;
      bw->kernel = kernel->data;
      bw->input_grad = input->grad;
      bw->kernel_grad = kernel->grad;
      bw->a = a;
      push_bwd(v, id, bw);
    }
    *out = v;
  });
}

// ---------------------------------------------------------------- chunks / recurrent cells
int nkg_chunks(nkg_var* a, int ndim, const int64_t* chunk_shape, int capacity, nkg_var** outs, int* count) {
  return guard([&] {
    if (!a || !chunk_shape || !count || (capacity > 0 && !outs)) fail(NK_ERR_INVALID_ARG, "chunks: NULL");
    const Shape& xs = a->data->shape;
    if (ndim != (int)xs.size()) fail(NK_ERR_INVALID_ARG, "chunks: chunk shape has %d dimensions, the operand %d", ndim, (int)xs.size());
    int64_t nblocks = 1;
    for (int k = 0; k < ndim; ++k) {
      if (chunk_shape[k] < 1 || chunk_shape[k] > xs[k])
        fail(NK_ERR_INVALID_ARG, "chunks: chunk dimension %d (%lld) must be in [1, %lld]", k, (long long)chunk_shape[k],
             (long long)xs[k]);
      nblocks *= xs[k] / chunk_shape[k];
    }
    *count = (int)nblocks;
    if (capacity < nblocks) return;   // size query: nothing recorded
    const Shape cs(chunk_shape, chunk_shape + ndim);
    for (int64_t i = 0; i < nblocks; ++i) {
      TensorP od;
      nkg_var* v = unary_node(a, cs, a->data->dtype, od);
      auto fw = std::make_shared<Chunk>();
      fw->ctx = a->ctx;
      fw->operand = a->data;
      fw->data = od;
      fw->index = i;
      uint64_t id = push(v, fw);
      if (a->diff()) {
        v->grad = std::make_shared<Gradient>(a->ctx, cs, od->dtype);
        auto bw = std::make_shared<ChunkBackward>();
        bw->ctx = a->ctx;
        bw->gradient = v->grad;
        bw->operand_grad = a->grad;
        bw->index = i;
        push_bwd(v, id, bw);
      }
      outs[i] = v;
    }
  });
}

// var.rs:564-587 / 622-645, vardiff.rs:627-641 / 681-: one node for every operand count and every mix of Var and
// VarDiff operands (the reference's four homogeneous methods and its Cat / Stack traits for mixed pairs)
static void cat_impl(nkg_var* const* vars, int count, int axis, bool stack, nkg_var** out) {
  const char* who = stack ? "stack" : "cat";
  if (!vars || !out) fail(NK_ERR_INVALID_ARG, "%s: NULL", who);
  if (count < 1) fail(NK_ERR_INVALID_ARG, "%s: needs at least one operand, got %d", who, count);
  for (int i = 0; i < count; ++i)
    if (!vars[i]) fail(NK_ERR_INVALID_ARG, "%s: operand %d is NULL", who, i);
  nkg_var* a = vars[0];
  const Shape& s0 = a->data->shape;
  const int nd = (int)s0.size();
  for (int i = 1; i < count; ++i) {
    if (vars[i]->data->dtype != a->data->dtype)
      fail(NK_ERR_INVALID_ARG, "%s: operand %d has another element type than operand 0", who, i);
    if (vars[i]->ctx != a->ctx) fail(NK_ERR_INVALID_ARG, "%s: operand %d lives on another device than operand 0", who, i);
    if ((int)vars[i]->data->shape.size() != nd)
      fail(NK_ERR_INVALID_ARG, "%s: operand %d has %d dimensions, operand 0 has %d", who, i,
           (int)vars[i]->data->shape.size(), nd);
  }
  Shape os = s0;
  std::vector<int64_t> lens(count, 1);
  int64_t outer = 1, inner = 1;
  if (stack) {
    if (axis < 0 || axis > nd) fail(NK_ERR_INVALID_ARG, "stack: axis %d out of range for %d-dimensional operands", axis, nd);
    if (nd + 1 > NK_MAX_DIMS) fail(NK_ERR_INVALID_ARG, "stack: the result would have more than %d dimensions", NK_MAX_DIMS);
    for (int i = 1; i < count; ++i)
      for (int k = 0; k < nd; ++k)
        if (vars[i]->data->shape[k] != s0[k])
          fail(NK_ERR_INVALID_ARG, "stack: operand %d differs from operand 0 on axis %d (%lld vs %lld)", i, k,
               (long long)vars[i]->data->shape[k], (long long)s0[k]);
    for (int k = 0; k < axis; ++k) outer *= s0[k];
    for (int k = axis; k < nd; ++k) inner *= s0[k];
    os.insert(os.begin() + axis, count);
  } else {
    if (nd < 1) fail(NK_ERR_INVALID_ARG, "cat: operands must have at least one dimension");
    if (axis < 0 || axis >= nd) fail(NK_ERR_INVALID_ARG, "cat: axis %d out of range for %d-dimensional operands", axis, nd);
    os[axis] = 0;
    for (int i = 0; i < count; ++i) {
      const Shape& si = vars[i]->data->shape;
      for (int k = 0; k < nd; ++k)
        if (k != axis && si[k] != s0[k])
          fail(NK_ERR_INVALID_ARG, "cat: operand %d differs from operand 0 on axis %d (%lld vs %lld)", i, k,
               (long long)si[k], (long long)s0[k]);
      lens[i] = si[axis];
      os[axis] += si[axis];
    }
    int64_t len;
    lanes(os, axis, outer, len, inner);
  }
  nk_ctx* ctx = a->ctx;
  const int dt = a->data->dtype;
  nkg_var* v = new_like(a);
  for (int i = 0; i < count; ++i) {   // History::merge over every operand
    v->fwd.insert(vars[i]->fwd.begin(), vars[i]->fwd.end());
    v->bwd.insert(vars[i]->bwd.begin(), vars[i]->bwd.end());
  }
  v->data = std::make_shared<Tensor>(ctx, os, dt);
  auto fw = std::make_shared<Concatenate>();
  fw->ctx = ctx;
  fw->data = v->data;
  fw->lens = lens;
  fw->outer = outer;
  fw->inner = inner;
  fw->stack = stack;
  bool diff = false;
  for (int i = 0; i < count; ++i) {
    fw->operands.push_back(vars[i]->data);
    diff = diff || vars[i]->diff();
  }
  const uint64_t id = push(v, fw);
  if (diff) {
    v->grad = std::make_shared<Gradient>(ctx, os, dt);
    auto bw = std::make_shared<ConcatenateBackward>();
    bw->ctx = ctx;
    bw->gradient = v->grad;
    for (int i = 0; i < count; ++i) bw->operand_grads.push_back(vars[i]->grad);
    bw->lens = lens;
    bw->outer = outer;
    bw->inner = inner;
    bw->stack = stack;
    push_bwd(v, id, bw);
  }
  *out = v;
}

int nkg_cat(nkg_var* const* vars, int count, int axis, nkg_var** out) {
  return guard([&] { cat_impl(vars, count, axis, false, out); });
}

int nkg_stack(nkg_var* const* vars, int count, int axis, nkg_var** out) {
  return guard([&] { cat_impl(vars, count, axis, true, out); });
}

int nkg_unsqueeze(nkg_var* a, int axis, nkg_var** out) {
  return guard([&] {
    if (!a || !out) fail(NK_ERR_INVALID_ARG, "unsqueeze: NULL");
    Shape s = a->data->shape;
    if (axis < 0 || axis > (int)s.size())
      fail(NK_ERR_INVALID_ARG, "unsqueeze: axis %d out of range for a %d-dimensional operand", axis, (int)s.size());
    if (s.size() + 1 > NK_MAX_DIMS) fail(NK_ERR_INVALID_ARG, "unsqueeze: the result would have more than %d dimensions", NK_MAX_DIMS);
    s.insert(s.begin() + axis, 1);
    *out = view_of(a, s);
  });
}

static void cell_impl(bool lstm, nkg_var* x, nkg_var* c, nkg_var* h, nkg_var* w_ih, nkg_var* w_hh, nkg_var* b_ih,
                      nkg_var* b_hh, nkg_var** new_c, nkg_var** new_h) {
  const char* who = lstm ? "lstm_cell" : "gru_cell";
  struct Arg {
    nkg_var* v;
    const char* name;
  };
  std::vector<Arg> args = {{x, "input"}, {h, "hidden"}, {w_ih, "weight_ih"}, {w_hh, "weight_hh"}, {b_ih, "bias_ih"},
                           {b_hh, "bias_hh"}};
  if (lstm) args.push_back({c, "cell_state"});
  for (const Arg& a : args)
    if (!a.v) fail(NK_ERR_INVALID_ARG, "%s: %s is NULL", who, a.name);
  if (!new_h || (lstm && !new_c)) fail(NK_ERR_INVALID_ARG, "%s: NULL output", who);
  for (const Arg& a : args) {
    if (a.v->data->dtype != x->data->dtype)
      fail(NK_ERR_INVALID_ARG, "%s: %s has another element type than the input", who, a.name);
    if (a.v->ctx != x->ctx) fail(NK_ERR_INVALID_ARG, "%s: %s lives on another device than the input", who, a.name);
  }
  const int64_t G = lstm ? 4 : 3;
  auto shape_str = [](const Shape& s) {
    std::string out = "(";
    for (size_t i = 0; i < s.size(); ++i) out += (i ? ", " : "") + std::to_string(s[i]);
    return out + (s.size() == 1 ? ",)" : ")");
  };
  const Shape& xs = x->data->shape;
  if (xs.size() != 2) fail(NK_ERR_INVALID_ARG, "%s: input must be (batch, input_size), got %s", who, shape_str(xs).c_str());
  const Shape& hs = h->data->shape;
  if (hs.size() != 2 || hs[0] != xs[0])
    fail(NK_ERR_INVALID_ARG, "%s: hidden must be (batch = %lld, hidden_size), got %s", who, (long long)xs[0],
         shape_str(hs).c_str());
  const int64_t N = xs[0], I = xs[1], H = hs[1];
  auto expect = [&](nkg_var* v, const char* name, const Shape& want) {
    if (v->data->shape != want)
      fail(NK_ERR_INVALID_ARG, "%s: %s must be %s, got %s", who, name, shape_str(want).c_str(),
           shape_str(v->data->shape).c_str());
  };
  if (lstm) expect(c, "cell_state", {N, H});
  expect(w_ih, "weight_ih", {G * H, I});
  expect(w_hh, "weight_hh", {G * H, H});
  expect(b_ih, "bias_ih", {G * H});
  expect(b_hh, "bias_hh", {G * H});

  nk_ctx* ctx = x->ctx;
  const int dt = x->data->dtype;
  auto fw = std::make_shared<RnnCell>();
  fw->ctx = ctx;
  fw->lstm = lstm;
  fw->o = CellOperands{x->data, h->data, lstm ? c->data : nullptr, w_ih->data, w_hh->data, b_ih->data, b_hh->data};
  fw->gi = std::make_shared<Tensor>(ctx, Shape{N, G * H}, NK_F32);
  if (!lstm) fw->gh = std::make_shared<Tensor>(ctx, Shape{N, G * H}, NK_F32);
  fw->h_out = std::make_shared<Tensor>(ctx, Shape{N, H}, dt);
  if (lstm) fw->c_out = std::make_shared<Tensor>(ctx, Shape{N, H}, dt);

  nkg_var* vh = new_like(x);
  vh->data = fw->h_out;
  for (const Arg& a : args) {   // History::merge over every operand
    vh->fwd.insert(a.v->fwd.begin(), a.v->fwd.end());
    vh->bwd.insert(a.v->bwd.begin(), a.v->bwd.end());
  }
  const uint64_t id = push(vh, fw);
  bool diff = false;
  for (const Arg& a : args) diff = diff || a.v->diff();
  if (diff) {
    vh->grad = std::make_shared<Gradient>(ctx, Shape{N, H}, dt);
    auto bw = std::make_shared<RnnCellBackward>();
    bw->ctx = ctx;
    bw->lstm = lstm;
    bw->o = fw->o;
    bw->gi = fw->gi;
    bw->gh = fw->gh;
    bw->gradient = vh->grad;
    bw->d = CellGrads{x->grad, h->grad, lstm ? c->grad : nullptr, w_ih->grad, w_hh->grad, b_ih->grad, b_hh->grad};
    if (lstm) bw->c_out_grad = std::make_shared<Gradient>(ctx, Shape{N, H}, dt);
    push_bwd(vh, id, bw);
  }
  if (lstm) {   // the second output: same tapes, same op id (merging the two histories keeps one node)
    nkg_var* vc = new nkg_var(*vh);
    vc->data = fw->c_out;
    if (diff) vc->grad = std::dynamic_pointer_cast<RnnCellBackward>(vh->bwd[id])->c_out_grad;
    *new_c = vc;
  }
  *new_h = vh;
}

int nkg_lstm_cell(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh,
                  nkg_var* bias_ih, nkg_var* bias_hh, nkg_var** new_cell_state, nkg_var** new_hidden) {
  return guard([&] {
    cell_impl(true, input, cell_state, hidden, weight_ih, weight_hh, bias_ih, bias_hh, new_cell_state, new_hidden);
  });
}

int nkg_gru_cell(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
                 nkg_var* bias_hh, nkg_var** new_hidden) {
  return guard([&] { cell_impl(false, input, nullptr, hidden, weight_ih, weight_hh, bias_ih, bias_hh, nullptr, new_hidden); });
}

// ---------------------------------------------------------------- optimizers on a leaf (neuronika-optim)
int nkg_adam_step(nkg_var* p, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, float* master, int64_t step,
                  float lr, float beta1, float beta2, float eps, float l1, float l2, float grad_scale) {
  return guard([&] {
    if (!p || !p->diff()) fail(NK_ERR_INVALID_ARG, "adam: parameter is not differentiable");
    Gradient* g = p->grad->root();
    ck(p->ctx, nk_adam_step(p->ctx, p->data->rptr(), p->data->dtype, p->grad->get(), g->dtype, exp_avg, exp_avg_sq,
                            max_exp_avg_sq, master, size_t(p->data->n()), step, lr, beta1, beta2, eps, l1, l2, grad_scale, 1));
    g->is_zero = false;
  });
}
int nkg_rmsprop_step(nkg_var* p, float* square_avg, float* grad_avg, float* momentum_buf, float* master, float lr,
                     float alpha, float eps, float momentum, float l1, float l2, float grad_scale) {
  return guard([&] {
    if (!p || !p->diff()) fail(NK_ERR_INVALID_ARG, "rmsprop: parameter is not differentiable");
    Gradient* g = p->grad->root();
    ck(p->ctx, nk_rmsprop_step(p->ctx, p->data->rptr(), p->data->dtype, p->grad->get(), g->dtype, square_avg, grad_avg,
                               momentum_buf, master, size_t(p->data->n()), lr, alpha, eps, momentum, l1, l2, grad_scale, 1));
    g->is_zero = false;
  });
}
int nkg_adagrad_step(nkg_var* p, float* grad_sq, float* master, int64_t step, float lr, float lr_decay, float eps,
                     float l1, float l2, float grad_scale) {
  return guard([&] {
    if (!p || !p->diff()) fail(NK_ERR_INVALID_ARG, "adagrad: parameter is not differentiable");
    Gradient* g = p->grad->root();
    ck(p->ctx, nk_adagrad_step(p->ctx, p->data->rptr(), p->data->dtype, p->grad->get(), g->dtype, grad_sq, master,
                               size_t(p->data->n()), step, lr, lr_decay, eps, l1, l2, grad_scale, 1));
    g->is_zero = false;
  });
}

int nkg_set_grad_rs(nkg_var* leaf, int world, int rank, void* const* slots, nkg_grad_rs_hook cb, void* user) {
  return guard([&] {
    if (!leaf || !leaf->diff()) fail(NK_ERR_INVALID_ARG, "nkg_set_grad_rs: not a differentiable variable");
    if (world < 0 || world > 8 || (world > 1 && (!slots || rank < 0 || rank >= world)))
      fail(NK_ERR_INVALID_ARG, "nkg_set_grad_rs: bad world / rank");
    Gradient* r = leaf->grad->root();
    r->rs_world = world > 1 ? world : 0;
    r->rs_rank = rank;
    for (int i = 0; i < 8; ++i) r->rs_slots[i] = (world > 1 && i < world) ? slots[i] : nullptr;
    r->rs_hook = world > 1 ? cb : nullptr;
    r->rs_user = user;
  });
}

int nkg_set_grad_hook(nkg_var* leaf, nkg_grad_hook cb, void* user, int row_chunks) {
  return guard([&] {
    if (!leaf || !leaf->diff()) fail(NK_ERR_INVALID_ARG, "nkg_set_grad_hook: not a differentiable variable");
    Gradient* r = leaf->grad->root();
    r->hook = cb;
    r->hook_user = user;
    r->hook_chunks = row_chunks > 1 ? row_chunks : 1;
  });
}

int nkg_sgd_step(nkg_var* p, float* momentum_buf, float* master, float lr, float l2, float momentum, float dampening,
                 int nesterov, float grad_scale) {
  return guard([&] {
    if (!p || !p->diff()) fail(NK_ERR_INVALID_ARG, "sgd: parameter is not differentiable");
    Gradient* g = p->grad->root();
    ck(p->ctx, nk_sgd_step(p->ctx, p->data->rptr(), p->data->dtype, p->grad->get(), g->dtype, momentum_buf, master,
                           size_t(p->data->n()), lr, l2, momentum, dampening, nesterov, grad_scale, 1));
    g->is_zero = false;
  });
}

}  // extern "C"
