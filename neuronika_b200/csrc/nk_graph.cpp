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
#include "nk_pool.h"

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
  // fill(v) is deferred: the gradient is "v everywhere" until somebody needs the bytes (get / acc materialise it).  The
  // nk_fill then runs right before the gradient's first reader, into a buffer allocated without nk_alloc's zero fill.
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
  nk_ctx* ctx;
  bool skip = false;  // fused into a consumer
  explicit Forward(nk_ctx* c) : ctx(c) {}
  virtual ~Forward() {}
  virtual void forward() = 0;
  virtual const char* name() const = 0;
};
// set by nkg_backward around each node: position of the running node in the reverse tape
static thread_local int g_bwd_pos = -1;
// A backward node reports every gradient it accumulates into once its last write to it is launched: the hook of a
// gradient fires when the node that reports it is that gradient's last writer in the running pass.
static inline void grad_written(const GradientP& g) {
  if (!g) return;
  Gradient* r = g->root();
  if (r->hook && r->last_writer == g_bwd_pos && !r->hook_fired) {
    r->hook_fired = true;
    r->hook(r->hook_user, 0, r->n());
  }
}

struct Backward {
  nk_ctx* ctx;
  GradientP gradient;  // gradient of this node's output
  bool skip = false;
  bool single_pass = false;  // a fusion that is exact for ONE backward pass was applied to this node
  int runs = 0;        // backward() calls so far (a second pass over the same tape must see un-aliased gradients)
  Backward(nk_ctx* c, GradientP g) : ctx(c), gradient(std::move(g)) {}
  virtual ~Backward() {}
  virtual void backward() = 0;
  virtual void targets(std::vector<Gradient*>& out) = 0;  // gradients this node accumulates into
  virtual const char* name() const = 0;
  // called before every backward pass after the first: undo what a fusion made exact for one pass only
  virtual void unalias() {}
  virtual void no_grad() {
    if (gradient) gradient->no_grad();
  }
  virtual void with_grad() {
    if (gradient) gradient->with_grad();
  }
};
using ForwardP = std::shared_ptr<Forward>;
using BackwardP = std::shared_ptr<Backward>;

// the non-null operand gradients of a node, as targets()
static void add_targets(std::vector<Gradient*>& out, std::initializer_list<const GradientP*> grads) {
  for (const GradientP* g : grads)
    if (*g) out.push_back((*g)->root());
}

static void gemm(nk_ctx* ctx, bool ta, bool tb, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                 const void* B, int64_t ldb, float beta, void* C, int ab_dt, int c_dt, const void* bias = nullptr,
                 int bias_dt = NK_F32, int relu = 0) {
  ck(ctx, nk_gemm_bias_act(ctx, ta, tb, M, N, K, 1.f, A, lda, B, ldb, beta, C, N, ab_dt, c_dt, bias, bias_dt, relu));
}

// The one write protocol of the backward nodes: kernel(dst, beta) accumulates a result it produces in element type
// `kdt` into the gradient g.  Same type -> the kernel writes the gradient directly with Gradient::acc()'s accumulate
// mode; otherwise (a bf16 leaf with an f32 gradient, requires_grad(grad_dtype)) it writes a temporary (beta = 0) which
// is then added with the mixed-type axpy of nk_unbroadcast_acc.
template <typename F>
static void accumulate(nk_ctx* ctx, const GradientP& g, int kdt, F&& kernel) {
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
// ... for a kernel that writes the gradient's own element type
template <typename F>
static void accumulate(nk_ctx* ctx, const GradientP& g, F&& kernel) {
  accumulate(ctx, g, g->dtype, kernel);
}

// ------------------------------------------------------------------------------- matmul nodes
// MatrixMatrixMul (matrix_matrix_mul/mod.rs:11-41) and MatrixMatrixMulT (matrix_matrix_mul_t/mod.rs:11-41)
struct MatMul : Forward {
  TensorP left, right, data;
  bool t;  // true: C = A.B^T (mm_t)
  MatMul(nk_ctx* c, TensorP l, TensorP r, TensorP d, bool tt)
      : Forward(c), left(std::move(l)), right(std::move(r)), data(std::move(d)), t(tt) {}
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
  MatMulBackward(nk_ctx* c, GradientP g, TensorP ld, TensorP rd, GradientP lg, GradientP rg, bool tt)
      : Backward(c, std::move(g)), left_data(std::move(ld)), right_data(std::move(rd)), left_grad(std::move(lg)),
        right_grad(std::move(rg)), t(tt) {}
  const char* name() const override { return t ? "MatrixMatrixMulTBackward" : "MatrixMatrixMulBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    if (left_dst)
      add_targets(out, {&left_dst, &left_colsum});
    else
      add_targets(out, {&left_grad});
    add_targets(out, {&right_grad});
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
        chunks = 0;  // reported after the dX GEMM, below
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
    grad_written(right_grad);  // a gradient with a reduce-scatter plan
  }
};

// ------------------------------------------------------------------------------- addition
struct Convolution;
struct Addition : Forward {  // addition/mod.rs:11-50
  TensorP left, right, data;
  std::shared_ptr<MatMul> fused_gemm;        // peephole: data = mm_t(..) + right in one kernel
  std::shared_ptr<Convolution> fused_conv;   // peephole: data = convolution(..) + bias(Cout,1,1) in one kernel
  TensorP fused_relu_out;                    // peephole: the consumer ReLU's output, written by the GEMM epilogue
  Addition(nk_ctx* c, TensorP l, TensorP r, TensorP d)
      : Forward(c), left(std::move(l)), right(std::move(r)), data(std::move(d)) {}
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
  GradientP left_grad, right_grad;
  bool left_aliased = false;
  bool right_fused = false;   // the bias gradient is summed in the epilogue of the dX GEMM above (MatMulBackward::left_colsum)
  AdditionBackward(nk_ctx* c, GradientP g, GradientP lg, GradientP rg)
      : Backward(c, std::move(g)), left_grad(std::move(lg)), right_grad(std::move(rg)) {}
  const char* name() const override { return "AdditionBackward"; }
  void acc(const GradientP& dst, bool aliased) {
    if (!dst || aliased) return;
    accumulate(ctx, dst, [&](void* d, float beta) {
      ck(ctx, nk_unbroadcast_acc(ctx, d, dst->dtype, (int)dst->shape.size(), dst->shape.data(), gradient->get(),
                                 gradient->dtype, (int)gradient->shape.size(), gradient->shape.data(), beta));
    });
    grad_written(dst);
  }
  void targets(std::vector<Gradient*>& out) override {
    add_targets(out, {&left_grad});
    if (!right_fused) add_targets(out, {&right_grad});
  }
  void backward() override {
    acc(left_grad, left_aliased);
    acc(right_grad, right_fused);
    if (left_aliased) grad_written(left_grad);    // written by the consumers of this node's output
  }
  void unalias() override;
};

// ------------------------------------------------------------------------------- unary / softmax
struct ReLU : Forward {  // relu/mod.rs:11-38
  TensorP operand, data;
  ReLU(nk_ctx* c, TensorP x, TensorP d) : Forward(c), operand(std::move(x)), data(std::move(d)) {}
  const char* name() const override { return "ReLU"; }
  void forward() override {
    ck(ctx, nk_relu_fwd(ctx, data->wptr(), operand->rptr(), size_t(data->n()), data->dtype));
  }
};
struct ReLUBackward : Backward {  // relu/mod.rs:40-79
  TensorP operand_data;
  GradientP operand_grad;
  ReLUBackward(nk_ctx* c, GradientP g, TensorP x, GradientP xg)
      : Backward(c, std::move(g)), operand_data(std::move(x)), operand_grad(std::move(xg)) {}
  const char* name() const override { return "ReLUBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const void* g = gradient->get();
    accumulate(ctx, operand_grad, operand_data->dtype, [&](void* d, float beta) {
      ck(ctx, nk_relu_bwd(ctx, d, operand_data->rptr(), g, size_t(operand_data->n()), operand_data->dtype, beta));
    });
    grad_written(operand_grad);
  }
};

static void lanes(const Shape& s, int axis, int64_t& outer, int64_t& len, int64_t& inner) {
  outer = inner = 1;
  for (int i = 0; i < axis; ++i) outer *= s[i];
  len = s[axis];
  for (size_t i = axis + 1; i < s.size(); ++i) inner *= s[i];
}

struct Softmax : Forward {  // softmax/mod.rs:11-53, logsoftmax/mod.rs:11-53
  TensorP operand, data;
  int axis;
  bool log;
  Softmax(nk_ctx* c, TensorP x, TensorP d, int ax, bool lg)
      : Forward(c), operand(std::move(x)), data(std::move(d)), axis(ax), log(lg) {}
  const char* name() const override { return log ? "LogSoftmax" : "Softmax"; }
  void forward() override {
    int64_t o, l, i;
    lanes(data->shape, axis, o, l, i);
    ck(ctx, (log ? nk_log_softmax_fwd : nk_softmax_fwd)(ctx, data->wptr(), operand->rptr(), o, l, i, data->dtype));
  }
};
struct SoftmaxBackward : Backward {  // softmax/mod.rs:55-104, logsoftmax/mod.rs:55-102
  TensorP data;
  GradientP operand_grad;
  int axis;
  bool log;
  SoftmaxBackward(nk_ctx* c, GradientP g, TensorP d, GradientP xg, int ax, bool lg)
      : Backward(c, std::move(g)), data(std::move(d)), operand_grad(std::move(xg)), axis(ax), log(lg) {}
  const char* name() const override { return log ? "LogSoftmaxBackward" : "SoftmaxBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    int64_t o, l, i;
    lanes(data->shape, axis, o, l, i);
    const void* g = gradient->get();
    accumulate(ctx, operand_grad, data->dtype, [&](void* d, float beta) {
      ck(ctx, (log ? nk_log_softmax_bwd : nk_softmax_bwd)(ctx, d, data->rptr(), g, o, l, i, data->dtype, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- reductions / losses
struct SumMean : Forward {  // sum/mod.rs:11-34, mean/mod.rs:11-34
  TensorP operand, data;
  bool mean;
  SumMean(nk_ctx* c, TensorP x, TensorP d, bool m) : Forward(c), operand(std::move(x)), data(std::move(d)), mean(m) {}
  const char* name() const override { return mean ? "Mean" : "Sum"; }
  void forward() override {
    ck(ctx, nk_sum_fwd(ctx, (float*)data->wptr(), operand->rptr(), size_t(operand->n()), operand->dtype, mean));
  }
};
struct SumMeanBackward : Backward {  // sum/mod.rs:36-66, mean/mod.rs:36-71
  GradientP operand_grad;
  bool mean;
  SumMeanBackward(nk_ctx* c, GradientP g, GradientP xg, bool m)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), mean(m) {}
  const char* name() const override { return mean ? "MeanBackward" : "SumBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    accumulate(ctx, operand_grad, [&](void* d, float beta) {
      ck(ctx, nk_sum_bwd(ctx, d, (const float*)gradient->get(), size_t(operand_grad->n()), operand_grad->dtype, mean,
                         beta));
    });
    grad_written(operand_grad);
  }
};

// the criteria: squared_error/, nll/, absolute_error/, bce/, bce_with_logits/, kldiv/ (node/*/mod.rs)
enum LossKind { kMse, kNll, kMae, kBce, kBceWithLogits, kKlDiv };
static const char* loss_name(int kind, bool bwd) {
  static const char* const fwd_names[] = {"SquaredError", "NegativeLogLikelihood", "AbsoluteError",
                                          "BinaryCrossEntropy", "BCEWithLogits", "KLDiv"};
  static const char* const bwd_names[] = {"SquaredErrorBackward", "NegativeLogLikelihoodBackward",
                                          "AbsoluteErrorBackward", "BinaryCrossEntropyBackward",
                                          "BCEWithLogitsBackward", "KLDivBackward"};
  return bwd ? bwd_names[kind] : fwd_names[kind];
}

struct Loss : Forward {  // squared_error/mod.rs:11-58, nll/mod.rs:11-68, and the four above
  TensorP input, target, data;
  bool mean;
  int kind;
  Loss(nk_ctx* c, TensorP x, TensorP t, TensorP d, bool m, int k)
      : Forward(c), input(std::move(x)), target(std::move(t)), data(std::move(d)), mean(m), kind(k) {}
  const char* name() const override { return loss_name(kind, false); }
  void forward() override {
    float* out = (float*)data->wptr();
    const void *x = input->rptr(), *t = target->rptr();
    const size_t n = size_t(input->n());
    const int dt = input->dtype;
    switch (kind) {
      case kNll:
        ck(ctx, nk_nll_fwd(ctx, out, x, t, target->dtype, input->shape[0], input->shape[1], dt, mean));
        break;
      case kMse: ck(ctx, nk_mse_fwd(ctx, out, x, t, n, dt, mean)); break;
      case kMae: ck(ctx, nk_mae_fwd(ctx, out, x, t, n, dt, mean)); break;
      case kBce: ck(ctx, nk_bce_fwd(ctx, out, x, t, n, dt, mean)); break;
      case kBceWithLogits: ck(ctx, nk_bce_with_logits_fwd(ctx, out, x, t, n, dt, mean)); break;
      default: ck(ctx, nk_kldiv_fwd(ctx, out, x, t, n, input->shape[0], dt, mean)); break;
    }
  }
};
struct LossBackward : Backward {  // squared_error/mod.rs:60-122, nll/mod.rs:70-133, and the four above
  TensorP input, target;
  GradientP input_grad;
  bool mean;
  int kind;
  LossBackward(nk_ctx* c, GradientP g, TensorP x, TensorP t, GradientP xg, bool m, int k)
      : Backward(c, std::move(g)), input(std::move(x)), target(std::move(t)), input_grad(std::move(xg)), mean(m),
        kind(k) {}
  const char* name() const override { return loss_name(kind, true); }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&input_grad}); }
  void backward() override {
    const float* g = (const float*)gradient->get();
    if (kind == kNll || kind == kMse) {  // kernels that write the input's element type
      accumulate(ctx, input_grad, input->dtype, [&](void* d, float beta) {
        if (kind == kNll)
          ck(ctx, nk_nll_bwd(ctx, d, target->rptr(), target->dtype, g, input->shape[0], input->shape[1], input->dtype,
                             mean, beta));
        else
          ck(ctx, nk_mse_bwd(ctx, d, input->rptr(), target->rptr(), g, size_t(input->n()), input->dtype, mean, beta));
      });
    } else {  // kernels that write the gradient's own element type
      accumulate(ctx, input_grad, [&](void* d, float beta) {
        const int ddt = input_grad->dtype, dt = input->dtype;
        const size_t n = size_t(input->n());
        const void* t = target->rptr();
        switch (kind) {
          case kMae: ck(ctx, nk_mae_bwd(ctx, d, ddt, input->rptr(), t, g, n, dt, mean, beta)); break;
          case kBce: ck(ctx, nk_bce_bwd(ctx, d, ddt, input->rptr(), t, g, n, dt, mean, beta)); break;
          case kBceWithLogits: ck(ctx, nk_bce_with_logits_bwd(ctx, d, ddt, input->rptr(), t, g, n, dt, mean, beta)); break;
          default: ck(ctx, nk_kldiv_bwd(ctx, d, ddt, t, g, n, input->shape[0], dt, mean, beta)); break;
        }
      });
    }
    grad_written(input_grad);
  }
};

// ------------------------------------------------------------------------------- dropout
// What a Dropout forward did last; its backward applies exactly that, whatever the status says by then.
enum DropoutDraw { kDropIdentity, kDropMasked, kDropZero };
struct DropoutState {
  int draw = kDropIdentity;
};

struct Dropout : Forward {  // dropout/mod.rs:15-78
  TensorP operand, data, mask;  // mask: ceil(n/32) keep words, allocated when the node is built (the reference's noise)
  double p;
  std::shared_ptr<bool> train;  // the shared status, Rc<Cell<bool>>
  std::shared_ptr<DropoutState> state;
  Dropout(nk_ctx* c, TensorP x, TensorP d, TensorP m, double pp, std::shared_ptr<bool> st, std::shared_ptr<DropoutState> s)
      : Forward(c), operand(std::move(x)), data(std::move(d)), mask(std::move(m)), p(pp), train(std::move(st)),
        state(std::move(s)) {}
  const char* name() const override { return "Dropout"; }
  void forward() override {
    const bool draw = *train && p != 0.0;
    ck(ctx, nk_dropout_fwd(ctx, data->wptr(), draw && mask ? (uint32_t*)mask->wptr() : nullptr, operand->rptr(),
                           size_t(data->n()), data->dtype, draw ? p : 0.0));
    state->draw = !draw ? kDropIdentity : (1.0 - p == 0.0 ? kDropZero : kDropMasked);
  }
};
struct DropoutBackward : Backward {  // dropout/mod.rs:80-132, with the forward's 1/(1-p) (SURVEY.md 8-c defect 8)
  GradientP operand_grad;
  TensorP mask;
  double p;
  std::shared_ptr<DropoutState> state;
  DropoutBackward(nk_ctx* c, GradientP g, GradientP xg, TensorP m, double pp, std::shared_ptr<DropoutState> s)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), mask(std::move(m)), p(pp), state(std::move(s)) {}
  const char* name() const override { return "DropoutBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const void* g = gradient->get();
    const bool identity = state->draw == kDropIdentity;
    accumulate(ctx, operand_grad, [&](void* d, float beta) {
      ck(ctx, nk_dropout_bwd(ctx, d, operand_grad->dtype, identity || !mask ? nullptr : (const uint32_t*)mask->rptr(), g,
                             size_t(operand_grad->n()), gradient->dtype, identity ? 0.0 : p, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- pad / conv / flatten
struct Pad : Forward {  // pad/mod.rs:63-129 with Constant / Zero modes
  TensorP operand, data;
  int64_t ph, pw;
  float value;
  Pad(nk_ctx* c, TensorP x, TensorP d, int64_t h, int64_t w, float v)
      : Forward(c), operand(std::move(x)), data(std::move(d)), ph(h), pw(w), value(v) {}
  const char* name() const override { return "Pad"; }
  void forward() override {
    const Shape& s = operand->shape;
    ck(ctx, nk_pad2d_fwd(ctx, data->wptr(), operand->rptr(), s[0] * s[1], s[2], s[3], ph, pw, value, data->dtype));
  }
};
struct PadBackward : Backward {  // pad/mod.rs:131-182
  GradientP operand_grad;
  int64_t ph, pw;
  PadBackward(nk_ctx* c, GradientP g, GradientP xg, int64_t h, int64_t w)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), ph(h), pw(w) {}
  const char* name() const override { return "PadBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const Shape& s = operand_grad->shape;
    const void* g = gradient->get();
    accumulate(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_pad2d_bwd(ctx, d, g, s[0] * s[1], s[2], s[3], ph, pw, gradient->dtype, beta));
    });
    grad_written(operand_grad);
  }
};

struct ConvArgs {
  int64_t n, cin, h, w, cout, kh, kw, sh, sw, dh, dw, groups;
};
struct Convolution : Forward {  // convolution/mod.rs:296-355
  TensorP input, kernel, data;
  ConvArgs a;
  Convolution(nk_ctx* c, TensorP x, TensorP k, TensorP d, const ConvArgs& args)
      : Forward(c), input(std::move(x)), kernel(std::move(k)), data(std::move(d)), a(args) {}
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
// dW first, as in MatMulBackward: a data-parallel hook on the kernel's gradient fires before dX is launched; the two
// results are independent, so the order is invisible
struct ConvolutionBackward : Backward {  // convolution/mod.rs:357-510
  TensorP input, kernel;
  GradientP input_grad, kernel_grad;
  ConvArgs a;
  ConvolutionBackward(nk_ctx* c, GradientP g, TensorP x, TensorP k, GradientP xg, GradientP kg, const ConvArgs& args)
      : Backward(c, std::move(g)), input(std::move(x)), kernel(std::move(k)), input_grad(std::move(xg)),
        kernel_grad(std::move(kg)), a(args) {}
  const char* name() const override { return "ConvolutionBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&input_grad, &kernel_grad}); }
  void backward() override {
    if (kernel_grad) {
      accumulate(ctx, kernel_grad, [&](void* d, float beta) {
        ck(ctx, nk_conv2d_bwd_kernel(ctx, d, kernel_grad->dtype, nullptr, gradient->get(), input->rptr(), a.n, a.cin, a.h,
                                     a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh, a.dw, a.groups, gradient->dtype, beta));
      });
      grad_written(kernel_grad);
    }
    if (input_grad) {
      const void* g = gradient->get();
      accumulate(ctx, input_grad, gradient->dtype, [&](void* d, float beta) {
        ck(ctx, nk_conv2d_bwd_input(ctx, d, g, kernel->rptr(), a.n, a.cin, a.h, a.w, a.cout, a.kh, a.kw, a.sh, a.sw, a.dh,
                                    a.dw, a.groups, gradient->dtype, beta));
      });
      grad_written(input_grad);
    }
  }
};

// The aliasing peephole (dL += G with one consumer => L.grad IS G) is exact for ONE backward pass per tape.  The
// reference accumulates into every gradient, intermediates included, on every pass (nothing zeroes them), so on a
// repeated backward() the addend's gradient and the sum's gradient diverge: give the addend its own buffer, holding
// what the reference would hold after the passes so far (= the sum's gradient at the end of the last pass).
void AdditionBackward::unalias() {
  if (!left_aliased || !left_grad || !left_grad->alias) return;
  Gradient* g = left_grad.get();
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
  left_aliased = false;
}

// ------------------------------------------------------------------------------- sub / mul / div (broadcasting)
// subtraction/mod.rs:11-172, multiplication/mod.rs:11-185, division/mod.rs:11-185
struct Binary : Forward {
  TensorP left, right, data;
  int op;
  Binary(nk_ctx* c, TensorP l, TensorP r, TensorP d, int o)
      : Forward(c), left(std::move(l)), right(std::move(r)), data(std::move(d)), op(o) {}
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
  TensorP left_data, right_data;
  GradientP left_grad, right_grad;  // either may be null
  int op;
  BinaryBackward(nk_ctx* c, GradientP g, TensorP ld, TensorP rd, GradientP lg, GradientP rg, int o)
      : Backward(c, std::move(g)), left_data(std::move(ld)), right_data(std::move(rd)), left_grad(std::move(lg)),
        right_grad(std::move(rg)), op(o) {}
  const char* name() const override {
    return op == NK_BIN_SUB ? "SubtractionBackward" : op == NK_BIN_MUL ? "MultiplicationBackward" : "DivisionBackward";
  }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&left_grad, &right_grad}); }
  void side(int sd, const GradientP& dst) {
    if (!dst) return;
    accumulate(ctx, dst, [&](void* d, float beta) {
      ck(ctx, nk_binary_bcast_bwd(ctx, op, sd, d, dst->dtype, gradient->get(), left_data->rptr(), right_data->rptr(),
                                  gradient->dtype, (int)left_data->shape.size(), left_data->shape.data(),
                                  (int)right_data->shape.size(), right_data->shape.data(), beta));
    });
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
  TensorP operand, data;
  int op, iparam;
  Unary(nk_ctx* c, TensorP x, TensorP d, int o, int ip)
      : Forward(c), operand(std::move(x)), data(std::move(d)), op(o), iparam(ip) {}
  const char* name() const override { return unary_name(op, false); }
  void forward() override {
    ck(ctx, nk_unary_fwd(ctx, op, data->wptr(), operand->rptr(), size_t(data->n()), data->dtype, iparam));
  }
};
struct UnaryBackward : Backward {
  TensorP saved;  // the node's output (exp, sqrt, sigmoid, tanh) or its input (ln, softplus, leaky_relu, powi)
  GradientP operand_grad;
  int op, iparam;
  UnaryBackward(nk_ctx* c, GradientP g, TensorP s, GradientP xg, int o, int ip)
      : Backward(c, std::move(g)), saved(std::move(s)), operand_grad(std::move(xg)), op(o), iparam(ip) {}
  const char* name() const override { return unary_name(op, true); }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const void* g = gradient->get();
    const void* sv = saved ? saved->rptr() : nullptr;
    accumulate(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_unary_bwd(ctx, op, d, sv, g, size_t(gradient->n()), gradient->dtype, iparam, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- transpose (transpose/mod.rs:11-75)
struct Transpose : Forward {
  TensorP operand, data;
  Transpose(nk_ctx* c, TensorP x, TensorP d) : Forward(c), operand(std::move(x)), data(std::move(d)) {}
  const char* name() const override { return "Transpose"; }
  void forward() override {
    ck(ctx, nk_transpose(ctx, data->wptr(), data->dtype, operand->rptr(), operand->dtype, (int)operand->shape.size(),
                         operand->shape.data(), 0.f));
  }
};
struct TransposeBackward : Backward {
  GradientP operand_grad;
  TransposeBackward(nk_ctx* c, GradientP g, GradientP xg) : Backward(c, std::move(g)), operand_grad(std::move(xg)) {}
  const char* name() const override { return "TransposeBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {  // dX += G^T
    accumulate(ctx, operand_grad, [&](void* d, float beta) {
      ck(ctx, nk_transpose(ctx, d, operand_grad->dtype, gradient->get(), gradient->dtype, (int)gradient->shape.size(),
                           gradient->shape.data(), beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- n-d padding with a mode
// Pad<D, T: PaddingMode> over (N, C, s...) with 1..3 sample dims (pad/mod.rs:20-182; modes pad/{constant,zero,
// reflective,replicative}/mod.rs).  The 2-d constant case keeps its own node (Pad above).
struct PadNd : Forward {
  TensorP operand, data;
  int nsp, mode;
  int64_t pad[3];
  float value;
  PadNd(nk_ctx* c, TensorP x, TensorP d, int n, const int64_t* p, int m, float v)
      : Forward(c), operand(std::move(x)), data(std::move(d)), nsp(n), mode(m), pad{p[0], p[1], p[2]}, value(v) {}
  const char* name() const override { return "Pad"; }
  void forward() override {
    const Shape& s = operand->shape;
    ck(ctx, nk_padnd_fwd(ctx, data->wptr(), operand->rptr(), s[0] * s[1], nsp, s.data() + 2, pad, mode, value,
                         data->dtype));
  }
};
struct PadNdBackward : Backward {
  GradientP operand_grad;
  int nsp;
  int64_t pad[3];
  PadNdBackward(nk_ctx* c, GradientP g, GradientP xg, int n, const int64_t* p)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), nsp(n), pad{p[0], p[1], p[2]} {}
  const char* name() const override { return "PadBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const Shape& s = operand_grad->shape;
    const void* g = gradient->get();
    accumulate(ctx, operand_grad, gradient->dtype, [&](void* d, float beta) {
      ck(ctx, nk_padnd_bwd(ctx, d, g, s[0] * s[1], nsp, s.data() + 2, pad, gradient->dtype, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- pooling (nk_pool.cu)
// Max / average / adaptive average pooling of the nsp sample dims of (N, C, ...), torch's semantics.  The max pool's
// int32 winner indices (idx, allocated when the node is built, only for a differentiable operand) carry the forward's
// choice to the backward.
enum PoolOp { kPoolMax, kPoolAvg, kPoolAdaptive };
struct PoolArgs {
  int op, nsp, include_pad;
  int64_t k[3], s[3], p[3], d[3];
};
static int pool_fwd(nk_ctx* ctx, const PoolArgs& a, void* y, int32_t* idx, const void* x, const Shape& xs,
                    const Shape& ys, int dtype) {
  const int64_t planes = xs[0] * xs[1];
  if (a.op == kPoolMax)
    return nk_max_pool_nd_fwd(ctx, y, idx, x, planes, a.nsp, xs.data() + 2, ys.data() + 2, a.k, a.s, a.p, a.d, dtype);
  if (a.op == kPoolAvg)
    return nk_avg_pool_nd_fwd(ctx, y, x, planes, a.nsp, xs.data() + 2, ys.data() + 2, a.k, a.s, a.p, a.include_pad,
                              dtype);
  return nk_adaptive_avg_pool_nd_fwd(ctx, y, x, planes, a.nsp, xs.data() + 2, ys.data() + 2, dtype);
}
struct Pool : Forward {
  TensorP operand, data, idx;
  PoolArgs a;
  Pool(nk_ctx* c, TensorP x, TensorP d, TensorP i, const PoolArgs& pa)
      : Forward(c), operand(std::move(x)), data(std::move(d)), idx(std::move(i)), a(pa) {}
  const char* name() const override {
    return a.op == kPoolMax ? "MaxPool" : a.op == kPoolAvg ? "AvgPool" : "AdaptiveAvgPool";
  }
  void forward() override {
    ck(ctx, pool_fwd(ctx, a, data->wptr(), idx ? (int32_t*)idx->wptr() : nullptr, operand->rptr(), operand->shape,
                     data->shape, data->dtype));
  }
};
struct PoolBackward : Backward {
  GradientP operand_grad;
  TensorP idx;
  PoolArgs a;
  PoolBackward(nk_ctx* c, GradientP g, GradientP xg, TensorP i, const PoolArgs& pa)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), idx(std::move(i)), a(pa) {}
  const char* name() const override {
    return a.op == kPoolMax ? "MaxPoolBackward" : a.op == kPoolAvg ? "AvgPoolBackward" : "AdaptiveAvgPoolBackward";
  }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
  void backward() override {
    const Shape &xs = operand_grad->shape, &ys = gradient->shape;
    const void* g = gradient->get();
    const int64_t planes = xs[0] * xs[1];
    accumulate(ctx, operand_grad, [&](void* d, float beta) {  // one launch for every (dx, g) dtype pair
      const int dt = operand_grad->dtype, gt = gradient->dtype;
      if (a.op == kPoolMax)
        ck(ctx, nk_max_pool_nd_bwd(ctx, d, dt, g, gt, (const int32_t*)idx->rptr(), planes, a.nsp, xs.data() + 2,
                                   ys.data() + 2, a.k, a.s, a.p, a.d, beta));
      else if (a.op == kPoolAvg)
        ck(ctx, nk_avg_pool_nd_bwd(ctx, d, dt, g, gt, planes, a.nsp, xs.data() + 2, ys.data() + 2, a.k, a.s, a.p,
                                   a.include_pad, beta));
      else
        ck(ctx, nk_adaptive_avg_pool_nd_bwd(ctx, d, dt, g, gt, planes, a.nsp, xs.data() + 2, ys.data() + 2, beta));
    });
    grad_written(operand_grad);
  }
};

// ------------------------------------------------------------------------------- embedding (nk_embedding.cu)
// out = weight[ids]: ids of any shape (float ids, never differentiable), weight (v, e); the backward writes only the
// weight's gradient.
struct Embedding : Forward {
  TensorP ids, weight, data;
  Embedding(nk_ctx* c, TensorP i, TensorP w, TensorP d)
      : Forward(c), ids(std::move(i)), weight(std::move(w)), data(std::move(d)) {}
  const char* name() const override { return "Embedding"; }
  void forward() override {
    const Shape& ws = weight->shape;
    ck(ctx, nk_embedding_fwd(ctx, data->wptr(), weight->rptr(), ids->rptr(), ids->dtype, ids->n(), ws[0], ws[1],
                             weight->dtype));
  }
};
struct EmbeddingBackward : Backward {
  TensorP ids;
  GradientP weight_grad;
  int64_t padding_idx;
  EmbeddingBackward(nk_ctx* c, GradientP g, TensorP i, GradientP wg, int64_t pad)
      : Backward(c, std::move(g)), ids(std::move(i)), weight_grad(std::move(wg)), padding_idx(pad) {}
  const char* name() const override { return "EmbeddingBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&weight_grad}); }
  void backward() override {
    const Shape& ws = weight_grad->shape;
    const void* g = gradient->get();
    accumulate(ctx, weight_grad, [&](void* d, float beta) {  // one call for every (dw, g) dtype pair
      ck(ctx, nk_embedding_bwd(ctx, d, weight_grad->dtype, ids->rptr(), ids->dtype, g, gradient->dtype, ids->n(), ws[0],
                               ws[1], padding_idx, beta));
    });
    grad_written(weight_grad);
  }
};

// ------------------------------------------------------------------------------- batch norm / layer norm (nk_norm.cu)
// Which statistics the last BatchNorm forward normalized with; its backward applies exactly that, whatever the status
// says by then (as DropoutState).
struct BatchNormState {
  bool batch = true;
};
// (N, C, S) view of a batch-norm operand: S = product of the sample dims
static void bn_dims(const Shape& s, int64_t& n, int64_t& c, int64_t& sp) {
  n = s[0], c = s[1], sp = 1;
  for (size_t i = 2; i < s.size(); ++i) sp *= s[i];
}
static void* opt_r(const TensorP& t) { return t ? t->rptr() : nullptr; }

// the size as torch prints it in its messages: torch.Size([2, 3])
static std::string torch_size(const Shape& s) {
  std::string out = "torch.Size([";
  for (size_t i = 0; i < s.size(); ++i) out += (i ? ", " : "") + std::to_string(s[i]);
  return out + "])";
}
// batch statistics need two values per channel (torch's _verify_batch_size): checked when the node is built and again
// on every forward, since the status may have turned to training in between
static void bn_check_batch(const Shape& s, bool batch) {
  int64_t n, c, sp;
  bn_dims(s, n, c, sp);
  if (batch && n * sp == 1)
    fail(NK_ERR_INVALID_ARG, "Expected more than 1 value per channel when training, got input size %s",
         torch_size(s).c_str());
}

struct BatchNorm : Forward {
  TensorP operand, weight, bias, running_mean, running_var, data, save_mean, save_rstd;
  std::shared_ptr<bool> train;
  std::shared_ptr<BatchNormState> state;
  float momentum, eps;
  BatchNorm(nk_ctx* c, TensorP x, TensorP w, TensorP b, TensorP rm, TensorP rv, TensorP d, TensorP sm, TensorP sr,
            std::shared_ptr<bool> st, std::shared_ptr<BatchNormState> s, float mom, float e)
      : Forward(c), operand(std::move(x)), weight(std::move(w)), bias(std::move(b)), running_mean(std::move(rm)),
        running_var(std::move(rv)), data(std::move(d)), save_mean(std::move(sm)), save_rstd(std::move(sr)),
        train(std::move(st)), state(std::move(s)), momentum(mom), eps(e) {}
  const char* name() const override { return "BatchNorm"; }
  void forward() override {
    bn_check_batch(operand->shape, *train || !running_mean);
    int64_t n, c, sp;
    bn_dims(operand->shape, n, c, sp);
    ck(ctx, nk_batch_norm_fwd(ctx, data->wptr(), operand->rptr(), data->dtype, n, c, sp, opt_r(weight), opt_r(bias),
                              (float*)opt_r(running_mean), (float*)opt_r(running_var), (float*)save_mean->wptr(),
                              (float*)save_rstd->wptr(), *train ? 1 : 0, momentum, eps));
    state->batch = *train || !running_mean;
  }
};
struct BatchNormBackward : Backward {
  GradientP operand_grad, weight_grad, bias_grad;
  TensorP operand, weight, save_mean, save_rstd;
  std::shared_ptr<BatchNormState> state;
  BatchNormBackward(nk_ctx* c, GradientP g, GradientP xg, GradientP wg, GradientP bg, TensorP x, TensorP w, TensorP sm,
                    TensorP sr, std::shared_ptr<BatchNormState> s)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), weight_grad(std::move(wg)), bias_grad(std::move(bg)),
        operand(std::move(x)), weight(std::move(w)), save_mean(std::move(sm)), save_rstd(std::move(sr)),
        state(std::move(s)) {}
  const char* name() const override { return "BatchNormBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad, &weight_grad, &bias_grad}); }
  void backward() override {
    int64_t n, c, sp;
    bn_dims(operand->shape, n, c, sp);
    const void* g = gradient->get();
    float bx = 0.f, bw = 0.f, bb = 0.f;  // one launch sequence writes all three, each with its own dtype and beta
    void* dx = operand_grad ? operand_grad->acc(&bx) : nullptr;
    void* dw = weight_grad ? weight_grad->acc(&bw) : nullptr;
    void* db = bias_grad ? bias_grad->acc(&bb) : nullptr;
    ck(ctx, nk_batch_norm_bwd(ctx, dx, operand_grad ? operand_grad->dtype : NK_F32, bx, dw,
                              weight_grad ? weight_grad->dtype : NK_F32, bw, db, bias_grad ? bias_grad->dtype : NK_F32,
                              bb, g, gradient->dtype, operand->rptr(), operand->dtype, n, c, sp, opt_r(weight),
                              (const float*)save_mean->rptr(), (const float*)save_rstd->rptr(), state->batch ? 1 : 0));
    grad_written(operand_grad);
    grad_written(weight_grad);
    grad_written(bias_grad);
  }
};

// the last k dims of the operand are one row
struct LayerNorm : Forward {
  TensorP operand, weight, bias, data, save_mean, save_rstd;
  int64_t cols;
  float eps;
  LayerNorm(nk_ctx* c, TensorP x, TensorP w, TensorP b, TensorP d, TensorP sm, TensorP sr, int64_t cl, float e)
      : Forward(c), operand(std::move(x)), weight(std::move(w)), bias(std::move(b)), data(std::move(d)),
        save_mean(std::move(sm)), save_rstd(std::move(sr)), cols(cl), eps(e) {}
  const char* name() const override { return "LayerNorm"; }
  void forward() override {
    ck(ctx, nk_layer_norm_fwd(ctx, data->wptr(), operand->rptr(), data->dtype, operand->n() / cols, cols, opt_r(weight),
                              opt_r(bias), (float*)save_mean->wptr(), (float*)save_rstd->wptr(), eps));
  }
};
struct LayerNormBackward : Backward {
  GradientP operand_grad, weight_grad, bias_grad;
  TensorP operand, weight, save_mean, save_rstd;
  int64_t cols;
  LayerNormBackward(nk_ctx* c, GradientP g, GradientP xg, GradientP wg, GradientP bg, TensorP x, TensorP w, TensorP sm,
                    TensorP sr, int64_t cl)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), weight_grad(std::move(wg)), bias_grad(std::move(bg)),
        operand(std::move(x)), weight(std::move(w)), save_mean(std::move(sm)), save_rstd(std::move(sr)), cols(cl) {}
  const char* name() const override { return "LayerNormBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad, &weight_grad, &bias_grad}); }
  void backward() override {
    const void* g = gradient->get();
    float bx = 0.f, bw = 0.f, bb = 0.f;
    void* dx = operand_grad ? operand_grad->acc(&bx) : nullptr;
    void* dw = weight_grad ? weight_grad->acc(&bw) : nullptr;
    void* db = bias_grad ? bias_grad->acc(&bb) : nullptr;
    ck(ctx, nk_layer_norm_bwd(ctx, dx, operand_grad ? operand_grad->dtype : NK_F32, bx, dw,
                              weight_grad ? weight_grad->dtype : NK_F32, bw, db, bias_grad ? bias_grad->dtype : NK_F32,
                              bb, g, gradient->dtype, operand->rptr(), operand->dtype, operand->n() / cols, cols,
                              opt_r(weight), (const float*)save_mean->rptr(), (const float*)save_rstd->rptr()));
    grad_written(operand_grad);
    grad_written(weight_grad);
    grad_written(bias_grad);
  }
};

// ------------------------------------------------------------------------------- cross-entropy (nk_cross_entropy.cu)
// input (N, C, d1..dk), target (N, d1..dk) of float class ids, weight (C) f32 or NULL; neither target nor weight is
// differentiable.  The forward node owns lse (N*S floats) and the denominator, allocated when the node is built; the
// backward reads both.
struct CeDims {
  int64_t n, c, s;
};
static CeDims ce_dims(const Shape& xs) {
  int64_t s = 1;
  for (size_t i = 2; i < xs.size(); ++i) s *= xs[i];
  return {xs[0], xs[1], s};
}
struct CrossEntropy : Forward {
  TensorP input, target, weight, data, lse, denom;
  bool mean;
  int64_t ignore_index;
  float label_smoothing;
  CrossEntropy(nk_ctx* c, TensorP x, TensorP t, TensorP w, TensorP d, TensorP l, TensorP dn, bool m, int64_t ig,
               float eps)
      : Forward(c), input(std::move(x)), target(std::move(t)), weight(std::move(w)), data(std::move(d)),
        lse(std::move(l)), denom(std::move(dn)), mean(m), ignore_index(ig), label_smoothing(eps) {}
  const char* name() const override { return "CrossEntropy"; }
  void forward() override {
    const CeDims d = ce_dims(input->shape);
    ck(ctx, nk_cross_entropy_fwd(ctx, (float*)data->wptr(), (float*)lse->wptr(), (float*)denom->wptr(), input->rptr(),
                                 input->dtype, target->rptr(), target->dtype, (const float*)opt_r(weight), d.n, d.c, d.s,
                                 ignore_index, label_smoothing, mean));
  }
};
struct CrossEntropyBackward : Backward {
  TensorP input, target, weight, lse, denom;
  GradientP input_grad;
  bool mean;
  int64_t ignore_index;
  float label_smoothing;
  CrossEntropyBackward(nk_ctx* c, GradientP g, TensorP x, TensorP t, TensorP w, TensorP l, TensorP dn, GradientP xg,
                       bool m, int64_t ig, float eps)
      : Backward(c, std::move(g)), input(std::move(x)), target(std::move(t)), weight(std::move(w)), lse(std::move(l)),
        denom(std::move(dn)), input_grad(std::move(xg)), mean(m), ignore_index(ig), label_smoothing(eps) {}
  const char* name() const override { return "CrossEntropyBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&input_grad}); }
  void backward() override {
    const CeDims d = ce_dims(input->shape);
    accumulate(ctx, input_grad, [&](void* dx, float beta) {  // one call for every (dx, x) dtype pair
      ck(ctx, nk_cross_entropy_bwd(ctx, dx, input_grad->dtype, input->rptr(), input->dtype, target->rptr(),
                                   target->dtype, (const float*)opt_r(weight), (const float*)lse->rptr(),
                                   (const float*)denom->rptr(), (const float*)gradient->get(), d.n, d.c, d.s,
                                   ignore_index, label_smoothing, mean, beta));
    });
    grad_written(input_grad);
  }
};

// ------------------------------------------------------------------------------- mv / vm / vv
// matrix_vector_mul/mod.rs:11-129, vector_matrix_mul/mod.rs:11-129, vector_vector_mul/mod.rs:11-91
struct MatVec : Forward {
  TensorP mat, vec, data;
  bool vm;  // true: y = v.A
  MatVec(nk_ctx* c, TensorP m, TensorP v, TensorP d, bool tvm)
      : Forward(c), mat(std::move(m)), vec(std::move(v)), data(std::move(d)), vm(tvm) {}
  const char* name() const override { return vm ? "VectorMatrixMul" : "MatrixVectorMul"; }
  void forward() override {
    ck(ctx, nk_gemv(ctx, vm ? 1 : 0, mat->shape[0], mat->shape[1], mat->rptr(), vec->rptr(), 0.f, data->wptr(),
                    mat->dtype, data->dtype));
  }
};
struct MatVecBackward : Backward {
  TensorP mat, vec;
  GradientP mat_grad, vec_grad;
  bool vm;
  MatVecBackward(nk_ctx* c, GradientP g, TensorP m, TensorP v, GradientP mg, GradientP vg, bool tvm)
      : Backward(c, std::move(g)), mat(std::move(m)), vec(std::move(v)), mat_grad(std::move(mg)),
        vec_grad(std::move(vg)), vm(tvm) {}
  const char* name() const override { return vm ? "VectorMatrixMulBackward" : "MatrixVectorMulBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&mat_grad, &vec_grad}); }
  void backward() override {
    const void* g = gradient->get();
    const int64_t rows = mat->shape[0], cols = mat->shape[1];
    auto do_mat = [&] {
      if (!mat_grad) return;
      // mv: dA += g (x) v ; vm: dA += v (x) g
      accumulate(ctx, mat_grad, [&](void* d, float beta) {
        ck(ctx, nk_outer_acc(ctx, d, mat_grad->dtype, vm ? vec->rptr() : g, vm ? g : vec->rptr(), rows, cols,
                             gradient->dtype, beta));
      });
      grad_written(mat_grad);
    };
    auto do_vec = [&] {
      if (!vec_grad) return;
      // mv: dv += A^T.g ; vm: dv += A.g
      accumulate(ctx, vec_grad, [&](void* d, float beta) {
        ck(ctx, nk_gemv(ctx, vm ? 0 : 1, rows, cols, mat->rptr(), g, beta, d, mat->dtype, vec_grad->dtype));
      });
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
  TensorP left, right, data;
  VecVec(nk_ctx* c, TensorP l, TensorP r, TensorP d)
      : Forward(c), left(std::move(l)), right(std::move(r)), data(std::move(d)) {}
  const char* name() const override { return "VectorVectorMul"; }
  void forward() override {
    ck(ctx, nk_dot(ctx, (float*)data->wptr(), left->rptr(), right->rptr(), size_t(left->n()), left->dtype));
  }
};
struct VecVecBackward : Backward {
  TensorP left, right;
  GradientP left_grad, right_grad;
  VecVecBackward(nk_ctx* c, GradientP g, TensorP l, TensorP r, GradientP lg, GradientP rg)
      : Backward(c, std::move(g)), left(std::move(l)), right(std::move(r)), left_grad(std::move(lg)),
        right_grad(std::move(rg)) {}
  const char* name() const override { return "VectorVectorMulBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&left_grad, &right_grad}); }
  void backward() override {
    const float* g = (const float*)gradient->get();
    auto one = [&](const GradientP& dst, const TensorP& other) {
      if (!dst) return;
      accumulate(ctx, dst, [&](void* d, float beta) {
        ck(ctx, nk_scale_acc(ctx, d, dst->dtype, other->rptr(), other->dtype, g, size_t(other->n()), beta));
      });
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
  TensorP input, kernel, data;
  ConvNdArgs a;
  ConvolutionNd(nk_ctx* c, TensorP x, TensorP k, TensorP d, const ConvNdArgs& args)
      : Forward(c), input(std::move(x)), kernel(std::move(k)), data(std::move(d)), a(args) {}
  const char* name() const override { return "Convolution"; }
  void forward() override {
    ck(ctx, nk_convnd_fwd(ctx, data->wptr(), input->rptr(), kernel->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k, a.s,
                          a.d, a.groups, data->dtype));
  }
};
struct ConvolutionNdBackward : Backward {  // convolution/mod.rs:357-510
  TensorP input, kernel;
  GradientP input_grad, kernel_grad;
  ConvNdArgs a;
  ConvolutionNdBackward(nk_ctx* c, GradientP g, TensorP x, TensorP k, GradientP xg, GradientP kg, const ConvNdArgs& args)
      : Backward(c, std::move(g)), input(std::move(x)), kernel(std::move(k)), input_grad(std::move(xg)),
        kernel_grad(std::move(kg)), a(args) {}
  const char* name() const override { return "ConvolutionBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&input_grad, &kernel_grad}); }
  void backward() override {
    const void* g = gradient->get();
    if (input_grad) {
      accumulate(ctx, input_grad, gradient->dtype, [&](void* d, float beta) {
        ck(ctx, nk_convnd_bwd_input(ctx, d, g, kernel->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k, a.s, a.d, a.groups,
                                    gradient->dtype, beta));
      });
      grad_written(input_grad);
    }
    if (kernel_grad) {
      accumulate(ctx, kernel_grad, [&](void* d, float beta) {
        ck(ctx, nk_convnd_bwd_kernel(ctx, d, kernel_grad->dtype, g, input->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k,
                                     a.s, a.d, a.groups, gradient->dtype, beta));
      });
      grad_written(kernel_grad);
    }
  }
};

// ------------------------------------------------------------------------------- 1-d / 3-d convolution layer
// nn.Conv1d / nn.Conv3d (neuronika-nn/src/lib.rs:630-916): pad -> convolution -> + bias as one node
struct ConvLayerArgs {
  int nsp, mode;
  float value;
  int64_t n, cin, cout;
  int64_t in[3], k[3], s[3], d[3], pad[3];
};
struct ConvLayer : Forward {
  TensorP input, weight, bias, data;  // bias may be null
  ConvLayerArgs a;
  ConvLayer(nk_ctx* c, TensorP x, TensorP w, TensorP b, TensorP d, const ConvLayerArgs& args)
      : Forward(c), input(std::move(x)), weight(std::move(w)), bias(std::move(b)), data(std::move(d)), a(args) {}
  const char* name() const override { return "ConvLayer"; }
  void forward() override {
    ck(ctx, nk_conv_layer_nd_fwd(ctx, data->wptr(), input->rptr(), weight->rptr(), bias ? bias->rptr() : nullptr, a.nsp, a.n,
                                 a.cin, a.in, a.cout, a.k, a.s, a.d, a.pad, a.mode, a.value, data->dtype));
  }
};
struct ConvLayerBackward : Backward {
  TensorP input, weight;
  GradientP input_grad, weight_grad, bias_grad;  // each may be null
  ConvLayerArgs a;
  ConvLayerBackward(nk_ctx* c, GradientP g, TensorP x, TensorP w, GradientP xg, GradientP wg, GradientP bg,
                    const ConvLayerArgs& args)
      : Backward(c, std::move(g)), input(std::move(x)), weight(std::move(w)), input_grad(std::move(xg)),
        weight_grad(std::move(wg)), bias_grad(std::move(bg)), a(args) {}
  const char* name() const override { return "ConvLayerBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&input_grad, &weight_grad, &bias_grad}); }
  void backward() override {
    const void* g = gradient->get();   // a deferred root fill is materialised here
    const int gdt = gradient->dtype;
    if (input_grad) {
      accumulate(ctx, input_grad, gdt, [&](void* d, float beta) {
        ck(ctx, nk_conv_layer_nd_bwd_input(ctx, d, g, weight->rptr(), a.nsp, a.n, a.cin, a.in, a.cout, a.k, a.s, a.d, a.pad,
                                           a.mode, gdt, beta));
      });
      grad_written(input_grad);
    }
    // the bias gradient rides along with dW when both have one element type and one accumulate mode
    bool bias_done = false;
    if (weight_grad) {
      void* dbias = nullptr;
      if (bias_grad && bias_grad->dtype == weight_grad->dtype) {
        Gradient* wr = weight_grad->root();
        Gradient* br = bias_grad->root();
        if (!wr->is_const && !br->is_const && wr->is_zero == br->is_zero) {
          float bbeta;
          dbias = bias_grad->acc(&bbeta);
          bias_done = true;
        }
      }
      accumulate(ctx, weight_grad, [&](void* d, float beta) {
        ck(ctx, nk_conv_layer_nd_bwd_kernel(ctx, d, weight_grad->dtype, dbias, g, input->rptr(), a.nsp, a.n, a.cin, a.in,
                                            a.cout, a.k, a.s, a.d, a.pad, a.mode, a.value, gdt, beta));
      });
      grad_written(weight_grad);
    }
    if (bias_grad && !bias_done) {
      accumulate(ctx, bias_grad, [&](void* d, float beta) {
        ck(ctx, nk_unbroadcast_acc(ctx, d, bias_grad->dtype, (int)bias_grad->shape.size(), bias_grad->shape.data(), g, gdt,
                                   (int)gradient->shape.size(), gradient->shape.data(), beta));
      });
    }
    grad_written(bias_grad);
  }
};

// ------------------------------------------------------------------------------- chunks (chunk/mod.rs)
struct Chunk : Forward {
  TensorP operand, data;
  int64_t index;
  Chunk(nk_ctx* c, TensorP x, TensorP d, int64_t i) : Forward(c), operand(std::move(x)), data(std::move(d)), index(i) {}
  const char* name() const override { return "Chunk"; }
  void forward() override {
    ck(ctx, nk_chunk_fwd(ctx, data->wptr(), operand->rptr(), (int)operand->shape.size(), operand->shape.data(),
                         data->shape.data(), index, data->dtype));
  }
};
struct ChunkBackward : Backward {
  GradientP operand_grad;
  int64_t index;
  ChunkBackward(nk_ctx* c, GradientP g, GradientP xg, int64_t i)
      : Backward(c, std::move(g)), operand_grad(std::move(xg)), index(i) {}
  const char* name() const override { return "ChunkBackward"; }
  void targets(std::vector<Gradient*>& out) override { add_targets(out, {&operand_grad}); }
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
  std::vector<TensorP> operands;
  TensorP data;
  std::vector<int64_t> lens;
  int64_t outer, inner;
  bool stack;
  Concatenate(nk_ctx* c, std::vector<TensorP> xs, TensorP d, const std::vector<int64_t>& l, int64_t o, int64_t i, bool s)
      : Forward(c), operands(std::move(xs)), data(std::move(d)), lens(l), outer(o), inner(i), stack(s) {}
  const char* name() const override { return stack ? "MultiStack" : "MultiConcatenate"; }
  void forward() override {
    if (data->n() == 0) return;
    std::vector<const void*> xs;
    for (size_t i = 0; i < operands.size(); ++i) xs.push_back(lens[i] ? operands[i]->rptr() : nullptr);
    ck(ctx, nk_cat_fwd(ctx, data->wptr(), xs.data(), lens.data(), (int)lens.size(), outer, inner, data->dtype));
  }
};
struct ConcatenateBackward : Backward {
  std::vector<GradientP> operand_grads;   // null for an operand that is not differentiable
  std::vector<int64_t> lens;
  int64_t outer, inner;
  bool stack;
  ConcatenateBackward(nk_ctx* c, GradientP g, std::vector<GradientP> xg, const std::vector<int64_t>& l, int64_t o,
                      int64_t i, bool s)
      : Backward(c, std::move(g)), operand_grads(std::move(xg)), lens(l), outer(o), inner(i), stack(s) {}
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
    if (passes > 0) {
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
    for (const GradientP& g : operand_grads) grad_written(g);
  }
};

// ------------------------------------------------------------------------------- recurrent cells
// LSTMCell / GRUCell (neuronika-nn/src/lib.rs:450-626) as ONE forward and ONE backward node per step instead of the
// ~15 nodes the reference composes them from: the two GEMMs write the gate pre-activations in f32 (kept for the tape's
// lifetime, so a second backward() still works), one kernel applies the gates (nk_lstm_cell_fwd / nk_gru_cell_fwd).
// The backward runs the gate kernel, then the weight gradients (dW += dG^T.x, TN), the bias gradients (column sums of
// dG) and the input / state gradients (dx += dG.W, NN), only for the operands that are differentiable.
// A whole sequence of such steps as one node is RnnSeq / RnnSeqBackward below ("recurrent sequence layers").
struct CellOperands {
  TensorP x, h, c, w_ih, w_hh, b_ih, b_hh;   // c: LSTM only
};
struct CellGrads {
  GradientP x, h, c, w_ih, w_hh, b_ih, b_hh;
};
struct RnnCell : Forward {
  bool lstm;
  CellOperands o;
  TensorP gi, gh;               // f32 gate pre-activations: LSTM (N, 4H) in gi; GRU (N, 3H) in gi (input) and gh (hidden)
  TensorP h_out, c_out;
  RnnCell(nk_ctx* c, bool l, CellOperands ops, TensorP h) : Forward(c), lstm(l), o(std::move(ops)), h_out(std::move(h)) {
    const int64_t N = o.x->shape[0], G = o.w_ih->shape[0];
    gi = std::make_shared<Tensor>(c, Shape{N, G}, NK_F32);
    if (!lstm) gh = std::make_shared<Tensor>(c, Shape{N, G}, NK_F32);
    if (lstm) c_out = std::make_shared<Tensor>(c, h_out->shape, h_out->dtype);
  }
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
  bool lstm;
  CellOperands o;
  CellGrads d;
  TensorP gi, gh;
  GradientP c_out_grad;
  RnnCellBackward(nk_ctx* c, GradientP g, const RnnCell& fw, CellGrads grads)
      : Backward(c, std::move(g)), lstm(fw.lstm), o(fw.o), d(std::move(grads)), gi(fw.gi), gh(fw.gh) {
    if (lstm) c_out_grad = std::make_shared<Gradient>(c, gradient->shape, gradient->dtype);
  }
  const char* name() const override { return lstm ? "LSTMCellBackward" : "GRUCellBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    add_targets(out, {&d.w_hh, &d.w_ih, &d.b_ih, &d.b_hh, &d.x, &d.h, &d.c});
  }
  // dW += dG^T.A (TN).  A weight with a data-parallel reduce-scatter plan is computed locally and reported as not pushed
  // ONCE per backward pass, by its last writer: in an unrolled sequence every time step's node accumulates into the same
  // weight gradient, and the caller exchanges the whole gradient for every report it gets.
  void weight(const GradientP& g, const void* dG, const TensorP& a, int64_t G, int64_t N, int dt) {
    if (!g) return;
    const int64_t K = a->shape[1];
    accumulate(ctx, g, [&](void* p, float beta) { gemm(ctx, true, false, G, K, N, dG, G, a->rptr(), K, beta, p, dt, g->dtype); });
    Gradient* r = g->root();
    if (r->rs_world > 1 && r->rs_hook && r->last_writer == g_bwd_pos) r->rs_hook(r->rs_user, 0);
    grad_written(g);
  }
  void bias(const GradientP& g, const void* dG, int64_t G, int64_t N, int dt) {
    if (!g) return;
    const int64_t ds[1] = {G}, gs[2] = {N, G};
    accumulate(ctx, g, [&](void* p, float beta) { ck(ctx, nk_unbroadcast_acc(ctx, p, g->dtype, 1, ds, dG, dt, 2, gs, beta)); });
    grad_written(g);
  }
  // dA += dG.W (NN)
  void input(const GradientP& g, const void* dG, const TensorP& w, int64_t G, int64_t N, int dt) {
    if (!g) return;
    const int64_t K = w->shape[1];
    accumulate(ctx, g, [&](void* p, float beta) { gemm(ctx, false, false, N, K, G, dG, G, w->rptr(), K, beta, p, dt, g->dtype); });
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
          accumulate(ctx, d.c, dt, [&](void* p, float beta) {
            ck(ctx, nk_lstm_cell_bwd(ctx, dI, dt, p, beta, (const float*)gi->rptr(), o.c->rptr(), dh, dc, N, H, dt));
          });
        else
          ck(ctx, nk_lstm_cell_bwd(ctx, dI, dt, nullptr, 0.f, (const float*)gi->rptr(), o.c->rptr(), dh, dc, N, H, dt));
        dH = dI;   // one gate gradient for both products
      } else {
        ck(ctx, nk_alloc_uninit(ctx, gbytes, &dH));
        const void* dh = gradient->get();
        if (d.h)
          accumulate(ctx, d.h, dt, [&](void* p, float beta) {
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
      grad_written(d.c);
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

// ------------------------------------------------------------------------------- recurrent sequence layers
// nn.LSTM / nn.GRU (time-major) as ONE forward and ONE backward node per layer whatever T is.  Of a cell's products only
// h_{t-1}.W_hh^T (forward) and dG_t.W_hh (backward) depend on the recurrence; the others run once over all T*N rows:
// X.W_ih^T + b_ih, dW_ih, dW_hh, dX and the bias column sums.  The node keeps the f32 gate pre-activations of every step
// (what T cell nodes keep) and, for the LSTM, the cell states.  The backward carries the state gradients (dc, and the
// part of dh that comes back through W_hh) in f32 from the last step down to step 0 (nk_lstm_seq_bwd_step /
// nk_gru_seq_bwd_step) and converts them once, into the gradients of the initial states.
// A bidirectional layer (D = 2) runs both directions in the same node: step s is time s of the forward direction and
// time T-1-s of the reverse one, and each step is ONE nk_gemm_strided_batched (the two directions' recurrent products)
// and ONE two-direction step kernel (nk_*_bidir_*_step), so it launches per step what a one-direction layer launches.
// The parameters are stacked over directions, (D, G, *), and the gates and gate gradients are (D, T*N, G) in time
// order, so the step-s operands of the two directions are a constant distance apart: (2T-1-2s)*N*G elements of the
// gates, G*H of W_hh, N*H of the (2, N, H) state buffers.
static inline char* at(void* p, int64_t elems, int dt) { return static_cast<char*>(p) + size_t(elems) * esize(dt); }
static inline const char* at(const void* p, int64_t elems, int dt) {
  return static_cast<const char*>(p) + size_t(elems) * esize(dt);
}
struct RnnDims {
  int64_t T, N, I, H, D;
};
struct RnnSeq : Forward {
  bool lstm;
  int64_t T, N, I, H, G, D;
  CellOperands o;      // x is (T, N, I); a layer's states are (D, N, H) and its parameters (D, G, *)
  TensorP gi, gh;      // f32 gate pre-activations of every step: LSTM (D, T*N, 4H) in gi; GRU (D, T*N, 3H) in gi and gh
  TensorP out;         // (T, N, D*H): every step's hidden state, the reverse direction in columns [H, 2H)
  TensorP cs, c_last;  // LSTM: the cell states of steps 0 .. T-2, (D, T-1, N, H), and the last one, (D, N, H) ((N, H) for
                       // nkg_lstm)
  TensorP h_n;         // layers (nkg_lstm_layer / nkg_gru_layer): the last hidden state of each direction, (D, N, H)
  RnnSeq(nk_ctx* c, bool l, bool layer, const RnnDims& dm, CellOperands ops, TensorP output)
      : Forward(c), lstm(l), T(dm.T), N(dm.N), I(dm.I), H(dm.H), G((l ? 4 : 3) * dm.H), D(dm.D), o(std::move(ops)),
        out(std::move(output)) {
    gi = std::make_shared<Tensor>(c, Shape{D, T * N, G}, NK_F32);
    if (!lstm) gh = std::make_shared<Tensor>(c, Shape{D, T * N, G}, NK_F32);
    const Shape state = layer ? Shape{D, N, H} : Shape{N, H};
    if (lstm) {
      cs = std::make_shared<Tensor>(c, Shape{D, T - 1, N, H}, out->dtype);
      c_last = std::make_shared<Tensor>(c, state, out->dtype);
    }
    if (layer) h_n = std::make_shared<Tensor>(c, state, out->dtype);
  }
  const char* name() const override { return lstm ? "LSTM" : "GRU"; }
  // D = 1: the state before step t, the initial one or what step t-1 wrote
  const void* h_prev(int64_t t, int64_t NH) const { return t ? at(out->rptr(), (t - 1) * NH, out->dtype) : o.h->rptr(); }
  const void* c_prev(int64_t t, int64_t NH) const { return t ? at(cs->rptr(), (t - 1) * NH, cs->dtype) : o.c->rptr(); }
  // D = 2: the cell state before step s of direction 0, and the distance to direction 1's
  const void* c_prev2(int64_t s, int64_t& dstride) const {
    dstride = s ? (T - 1) * N * H : N * H;
    return s ? at(cs->rptr(), (s - 1) * N * H, cs->dtype) : o.c->rptr();
  }
  void forward() override {
    if (D == 2) return forward_bidir();
    const int dt = o.x->dtype;
    gemm(ctx, false, true, T * N, G, I, o.x->rptr(), I, o.w_ih->rptr(), I, 0.f, gi->wptr(), dt, NK_F32, o.b_ih->rptr(),
         o.b_ih->dtype);
    void* y = out->wptr();
    for (int64_t t = 0; t < T; ++t) {
      float* gi_t = reinterpret_cast<float*>(at(gi->rptr(), t * N * G, NK_F32));
      void* y_t = at(y, t * N * H, dt);
      if (lstm) {
        gemm(ctx, false, true, N, G, H, h_prev(t, N * H), H, o.w_hh->rptr(), H, 1.f, gi_t, dt, NK_F32, o.b_hh->rptr(),
             o.b_hh->dtype);
        void* c_t = t == T - 1 ? c_last->wptr() : at(cs->wptr(), t * N * H, dt);
        ck(ctx, nk_lstm_cell_fwd(ctx, c_t, y_t, gi_t, c_prev(t, N * H), N, H, dt));
      } else {
        float* gh_t = reinterpret_cast<float*>(at(gh->wptr(), t * N * G, NK_F32));
        gemm(ctx, false, true, N, G, H, h_prev(t, N * H), H, o.w_hh->rptr(), H, 0.f, gh_t, dt, NK_F32, o.b_hh->rptr(),
             o.b_hh->dtype);
        ck(ctx, nk_gru_cell_fwd(ctx, y_t, gi_t, gh_t, h_prev(t, N * H), N, H, dt));
      }
    }
    if (h_n) ck(ctx, nk_cast(ctx, h_n->wptr(), dt, at(y, (T - 1) * N * H, dt), dt, size_t(N * H)));
  }
  void forward_bidir() {
    const int dt = o.x->dtype;
    const int64_t NH = N * H, NG = N * G;
    float* g = static_cast<float*>(gi->wptr());
    for (int64_t d = 0; d < 2; ++d)
      gemm(ctx, false, true, T * N, G, I, o.x->rptr(), I, at(o.w_ih->rptr(), d * G * I, dt), I, 0.f, g + d * T * NG, dt,
           NK_F32, at(o.b_ih->rptr(), d * G, o.b_ih->dtype), o.b_ih->dtype);
    float* gH = lstm ? g : static_cast<float*>(gh->wptr());   // the recurrent products: added to the LSTM's gates
    void* y = out->wptr();
    // (2, 2, N, H) ping-pong of the (2, N, H) hidden states that the next step's GEMM reads, for this pass only (the
    // backward reads the states from the output)
    void* hs = nullptr;
    if (T > 1) ck(ctx, nk_alloc_uninit(ctx, size_t(4 * NH) * esize(dt), &hs));
    try {
      steps_bidir(g, gH, y, hs);
    } catch (...) {
      if (hs) nk_free(ctx, hs);
      throw;
    }
    if (hs) ck(ctx, nk_free(ctx, hs));
  }
  void steps_bidir(float* g, float* gH, void* y, void* hs) {
    const int dt = o.x->dtype;
    const int64_t NH = N * H, NG = N * G;
    for (int64_t s = 0; s < T; ++s) {
      const void* hp = s ? at(hs, ((s - 1) & 1) * 2 * NH, dt) : o.h->rptr();
      void* hn = s == T - 1 ? h_n->wptr() : at(hs, (s & 1) * 2 * NH, dt);
      const int64_t gds = (2 * T - 1 - 2 * s) * NG;               // gates: time s of direction 0 -> time T-1-s of direction 1
      void* y_s = at(y, s * N * 2 * H, dt);
      const int64_t yds = (T - 1 - 2 * s) * N * 2 * H + H;         // output: row T-1-s, columns [H, 2H)
      ck(ctx, nk_gemm_strided_batched(ctx, 0, 1, N, G, H, 1.f, hp, H, NH, o.w_hh->rptr(), H, G * H, lstm ? 1.f : 0.f,
                                      gH + s * NG, G, gds, 2, dt, NK_F32, o.b_hh->rptr(), G, o.b_hh->dtype));
      if (lstm) {
        int64_t cpds;
        const void* cp = c_prev2(s, cpds);
        void* co = s == T - 1 ? c_last->wptr() : at(cs->wptr(), s * NH, dt);
        ck(ctx, nk_lstm_bidir_fwd_step(ctx, y_s, yds, 2 * H, hn, co, s == T - 1 ? NH : (T - 1) * NH, g + s * NG, gds, cp,
                                       cpds, N, H, dt));
      } else {
        ck(ctx, nk_gru_bidir_fwd_step(ctx, y_s, yds, 2 * H, hn, g + s * NG, gH + s * NG, gds, hp, NH, N, H, dt));
      }
    }
  }
};

struct RnnSeqBackward : Backward {  // `gradient` is the output's, (T, N, D*H); c_last_grad / h_n_grad the last states'
  std::shared_ptr<RnnSeq> fw;
  CellGrads d;
  GradientP c_last_grad, h_n_grad;
  RnnSeqBackward(nk_ctx* c, GradientP g, std::shared_ptr<RnnSeq> f, CellGrads grads)
      : Backward(c, std::move(g)), fw(std::move(f)), d(std::move(grads)) {
    if (fw->lstm) c_last_grad = std::make_shared<Gradient>(c, fw->c_last->shape, fw->c_last->dtype);
    if (fw->h_n) h_n_grad = std::make_shared<Gradient>(c, fw->h_n->shape, fw->h_n->dtype);
  }
  const char* name() const override { return fw->lstm ? "LSTMBackward" : "GRUBackward"; }
  void targets(std::vector<Gradient*>& out) override {
    add_targets(out, {&d.w_hh, &d.w_ih, &d.b_ih, &d.b_hh, &d.x, &d.h, &d.c});
  }
  // a weight with a data-parallel reduce-scatter plan is computed locally and reported as not pushed, as the cell does
  void weight_done(const GradientP& g) {
    Gradient* r = g->root();
    if (r->rs_world > 1 && r->rs_hook && r->last_writer == g_bwd_pos) r->rs_hook(r->rs_user, 0);
    grad_written(g);
  }
  // the column sums of each direction's (rows, G) slice of dG, into that direction's row of g
  void bias(const GradientP& g, const void* dG, int64_t G, int64_t rows, int dt, int64_t D = 1) {
    if (!g) return;
    const int64_t ds[1] = {G}, gs[2] = {rows, G};
    accumulate(ctx, g, [&](void* p, float beta) {
      for (int64_t k = 0; k < D; ++k)
        ck(ctx, nk_unbroadcast_acc(ctx, at(p, k * G, g->dtype), g->dtype, 1, ds, at(dG, k * rows * G, dt), dt, 2, gs, beta));
    });
    grad_written(g);
  }
  // g += the f32 (rows, H) state gradient the loop carried, converted into g's element type
  void state(const GradientP& g, const float* carried, int64_t rows, int64_t H) {
    if (!g) return;
    const int64_t s[2] = {rows, H};
    accumulate(ctx, g, [&](void* p, float beta) { ck(ctx, nk_unbroadcast_acc(ctx, p, g->dtype, 2, s, carried, NK_F32, 2, s, beta)); });
    grad_written(g);
  }
  // the carried f32 state gradient starts as the gradient of the last state (false: nobody wrote one)
  bool seed(void* carried, const GradientP& last, int64_t n) {
    const void* g = grad_or_null(last);
    if (g) ck(ctx, nk_cast(ctx, carried, NK_F32, g, last->dtype, size_t(n)));
    return g != nullptr;
  }
  void backward() override {
    const CellOperands& o = fw->o;
    const bool lstm = fw->lstm;
    const int64_t T = fw->T, N = fw->N, I = fw->I, H = fw->H, G = fw->G, D = fw->D;
    const int64_t NH = N * H, NG = N * G;
    const int dt = o.x->dtype;
    const size_t gbytes = size_t(D * T) * size_t(NG) * esize(dt), sbytes = size_t(D * NH) * sizeof(float);
    void *dI = nullptr, *dH = nullptr, *dh_rec = nullptr, *dc = nullptr;
    auto release = [&] {
      if (dc) nk_free(ctx, dc);
      if (dh_rec) nk_free(ctx, dh_rec);
      if (dH && dH != dI) nk_free(ctx, dH);
      if (dI) nk_free(ctx, dI);
    };
    try {
      ck(ctx, nk_alloc_uninit(ctx, gbytes, &dI));
      ck(ctx, nk_alloc_uninit(ctx, sbytes, &dh_rec));
      const void* dY = grad_or_null(gradient);
      const float* gi = reinterpret_cast<const float*>(fw->gi->rptr());
      const float* gh = lstm ? nullptr : reinterpret_cast<const float*>(fw->gh->rptr());
      bool dh_seeded = false;   // dh_rec holds the last hidden state's gradient before the last step
      if (lstm) {
        dH = dI;   // one gate gradient for both products
        ck(ctx, nk_alloc_uninit(ctx, sbytes, &dc));
        if (!seed(dc, c_last_grad, D * NH)) ck(ctx, nk_memset0(ctx, dc, sbytes));
        dh_seeded = seed(dh_rec, h_n_grad, D * NH);
      } else {
        ck(ctx, nk_alloc_uninit(ctx, gbytes, &dH));
        if (!seed(dh_rec, h_n_grad, D * NH)) ck(ctx, nk_memset0(ctx, dh_rec, sbytes));
      }
      const float* dh_last = dh_seeded ? static_cast<const float*>(dh_rec) : nullptr;
      if (D == 1) {
        for (int64_t t = T - 1; t >= 0; --t) {
          const void* dY_t = dY ? at(dY, t * NH, gradient->dtype) : nullptr;
          const bool send_back = t > 0 || d.h;   // somebody reads the gradient of the state before step t
          if (lstm) {
            ck(ctx, nk_lstm_seq_bwd_step(ctx, at(dI, t * NG, dt), dt, static_cast<float*>(dc), gi + t * NG,
                                         fw->c_prev(t, NH), dY_t, t == T - 1 ? dh_last : static_cast<const float*>(dh_rec),
                                         N, H, dt));
            if (send_back) gemm(ctx, false, false, N, H, G, at(dH, t * NG, dt), G, o.w_hh->rptr(), H, 0.f, dh_rec, dt, NK_F32);
          } else {
            ck(ctx, nk_gru_seq_bwd_step(ctx, at(dI, t * NG, dt), at(dH, t * NG, dt), dt, static_cast<float*>(dh_rec),
                                        gi + t * NG, gh + t * NG, fw->h_prev(t, NH), dY_t, N, H, dt));
            if (send_back) gemm(ctx, false, false, N, H, G, at(dH, t * NG, dt), G, o.w_hh->rptr(), H, 1.f, dh_rec, dt, NK_F32);
          }
        }
      } else {
        const void* y = fw->out->rptr();
        for (int64_t s = T - 1; s >= 0; --s) {
          const int64_t gds = (2 * T - 1 - 2 * s) * NG;
          const void* dY_s = dY ? at(dY, s * N * 2 * H, gradient->dtype) : nullptr;
          const int64_t yds = (T - 1 - 2 * s) * N * 2 * H + H;
          const bool send_back = s > 0 || d.h;
          if (lstm) {
            int64_t cpds;
            const void* cp = fw->c_prev2(s, cpds);
            ck(ctx, nk_lstm_bidir_bwd_step(ctx, at(dI, s * NG, dt), dt, gds, static_cast<float*>(dc), gi + s * NG, cp, cpds,
                                           dY_s, yds, 2 * H, s == T - 1 ? dh_last : static_cast<const float*>(dh_rec), N,
                                           H, dt));
          } else {
            // the hidden state before step s: the initial one, or output rows s-1 (direction 0) and T-s (direction 1)
            const void* hp = s ? at(y, (s - 1) * N * 2 * H, dt) : o.h->rptr();
            const int64_t hpds = s ? (T - 2 * s + 1) * N * 2 * H + H : NH;
            ck(ctx, nk_gru_bidir_bwd_step(ctx, at(dI, s * NG, dt), at(dH, s * NG, dt), dt, gds, static_cast<float*>(dh_rec),
                                          gi + s * NG, gh + s * NG, hp, hpds, s ? 2 * H : H, dY_s, yds, 2 * H, N, H, dt));
          }
          if (send_back)
            ck(ctx, nk_gemm_strided_batched(ctx, 0, 0, N, H, G, 1.f, at(dH, s * NG, dt), G, gds, o.w_hh->rptr(), H, G * H,
                                            lstm ? 0.f : 1.f, dh_rec, H, NH, 2, dt, NK_F32, nullptr, 0, NK_F32));
        }
      }
      // the parameters first (their data-parallel exchange can then overlap the rest), as the cell does.  Each weight
      // gradient is written by this node alone, so its hook and its reduce-scatter report fire once, after the last GEMM
      if (d.w_hh) {   // dW_hh += dG[later steps]^T.output[earlier steps] + dG[first step]^T.hidden (TN), per direction
        const void* y = fw->out->rptr();
        const int64_t ldy = D * H;
        accumulate(ctx, d.w_hh, [&](void* p, float beta) {
          for (int64_t k = 0; k < D; ++k) {
            void* pk = at(p, k * G * H, d.w_hh->dtype);
            const void* dG = at(dH, k * T * NG, dt);
            // direction 0 runs forward: step t >= 1 follows output row t-1; direction 1 runs backward: step t <= T-2
            // follows output row t+1, columns [H, 2H); the first step of each follows its initial state
            if (T > 1)
              gemm(ctx, true, false, G, H, (T - 1) * N, k ? dG : at(dG, NG, dt), G, k ? at(y, N * ldy + H, dt) : y, ldy,
                   beta, pk, dt, d.w_hh->dtype);
            gemm(ctx, true, false, G, H, N, k ? at(dG, (T - 1) * NG, dt) : dG, G, at(o.h->rptr(), k * NH, dt), H,
                 T > 1 ? 1.f : beta, pk, dt, d.w_hh->dtype);
          }
        });
        weight_done(d.w_hh);
      }
      if (d.w_ih) {   // dW_ih += dG^T.X (TN, K = T*N), per direction
        accumulate(ctx, d.w_ih, [&](void* p, float beta) {
          for (int64_t k = 0; k < D; ++k)
            gemm(ctx, true, false, G, I, T * N, at(dI, k * T * NG, dt), G, o.x->rptr(), I, beta, at(p, k * G * I, d.w_ih->dtype),
                 dt, d.w_ih->dtype);
        });
        weight_done(d.w_ih);
      }
      bias(d.b_ih, dI, G, T * N, dt, D);
      bias(d.b_hh, dH, G, T * N, dt, D);
      if (d.x) {      // dX += sum over directions of dG.W_ih (NN over T*N rows)
        accumulate(ctx, d.x, [&](void* p, float beta) {
          for (int64_t k = 0; k < D; ++k)
            gemm(ctx, false, false, T * N, I, G, at(dI, k * T * NG, dt), G, at(o.w_ih->rptr(), k * G * I, dt), I,
                 k ? 1.f : beta, p, dt, d.x->dtype);
        });
        grad_written(d.x);
      }
      state(d.h, static_cast<const float*>(dh_rec), D * N, H);
      state(d.c, static_cast<const float*>(dc), D * N, H);
    } catch (...) {
      release();
      throw;
    }
    ck(ctx, nk_free(ctx, dc));
    ck(ctx, nk_free(ctx, dh_rec));
    if (dH != dI) ck(ctx, nk_free(ctx, dH));
    ck(ctx, nk_free(ctx, dI));
  }
  void no_grad() override {
    Backward::no_grad();
    if (c_last_grad) c_last_grad->no_grad();
    if (h_n_grad) h_n_grad->no_grad();
  }
  void with_grad() override {
    Backward::with_grad();
    if (c_last_grad) c_last_grad->with_grad();
    if (h_n_grad) h_n_grad->with_grad();
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

struct nkg_status {  // the dropout status shared by the handle and every node built with it, Rc<Cell<bool>>
  std::shared_ptr<bool> train;
};

namespace {

void not_null(std::initializer_list<const void*> ptrs, const char* who) {
  for (const void* p : ptrs)
    if (!p) fail(NK_ERR_INVALID_ARG, "%s: NULL", who);
}

void require_same_dtype(nkg_var* a, nkg_var* b, const char* who) {
  if (a->data->dtype != b->data->dtype) fail(NK_ERR_INVALID_ARG, "%s: operands have different element types", who);
  if (a->ctx != b->ctx) fail(NK_ERR_INVALID_ARG, "%s: operands live on different devices", who);
}

// check_groups_args, utils.rs:427-496 (same messages): shared by the 2-d and the n-d convolution
void check_conv_channels(const Shape& ks, const Shape& is, int64_t groups) {
  if (is[1] % groups) fail(NK_ERR_INVALID_ARG, "In channels %lld is not divisible by groups %lld", (long long)is[1], (long long)groups);
  if (ks[0] % groups) fail(NK_ERR_INVALID_ARG, "Out channels %lld is not divisible by groups %lld", (long long)ks[0], (long long)groups);
  if (ks[1] * groups != is[1]) fail(NK_ERR_INVALID_ARG, "convolution: kernel in-channels %lld x groups %lld != input channels %lld", (long long)ks[1], (long long)groups, (long long)is[1]);
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

// "(2, 3)" / "(4,)" in the messages of the shape checks
std::string shape_str(const Shape& s) {
  std::string out = "(";
  for (size_t i = 0; i < s.size(); ++i) out += (i ? ", " : "") + std::to_string(s[i]);
  return out + (s.size() == 1 ? ",)" : ")");
}

// Records one op: the result's history is the union of the operands' (History::merge) plus one node; its data is a
// new (shape, dtype) tensor written by the Forward node make_fwd(data); if any operand is differentiable, the result
// gets a gradient of the same shape and type and the Backward node make_bwd(data, gradient) under the same op id.
template <typename MakeFwd, typename MakeBwd>
nkg_var* record(const std::vector<nkg_var*>& operands, const Shape& shape, int dtype, MakeFwd&& make_fwd,
                MakeBwd&& make_bwd) {
  nkg_var* v = new nkg_var();
  v->ctx = operands.front()->ctx;
  bool diff = false;
  for (nkg_var* a : operands) {
    v->fwd.insert(a->fwd.begin(), a->fwd.end());
    v->bwd.insert(a->bwd.begin(), a->bwd.end());
    diff = diff || a->diff();
  }
  v->data = std::make_shared<Tensor>(v->ctx, shape, dtype);
  const uint64_t id = g_next_op_id++;  // creation order == a topological order (history.rs:84-88)
  v->fwd[id] = make_fwd(v->data);
  if (diff) {
    v->grad = std::make_shared<Gradient>(v->ctx, shape, dtype);
    v->bwd[id] = make_bwd(v->data, v->grad);
  }
  return v;
}

// ---- peephole fusion, run when the tapes are materialised by forward()
void fuse(nkg_var* v) {
  if (!g_fusion) return;
  // lookups over the tapes, built once: output tensor -> its producer (matmul or convolution), operand tensor -> the
  // LAST ReLU backward reading it, output gradient -> its addition backward, left operand gradient -> the FIRST matmul
  // backward accumulating into it
  std::map<Tensor*, std::shared_ptr<MatMul>> gemms;
  std::map<Tensor*, std::shared_ptr<Convolution>> convs;
  for (auto& kv : v->fwd) {
    if (auto mm = std::dynamic_pointer_cast<MatMul>(kv.second)) gemms[mm->data.get()] = mm;
    if (auto cv = std::dynamic_pointer_cast<Convolution>(kv.second)) convs[cv->data.get()] = cv;
  }
  std::map<Tensor*, std::shared_ptr<ReLUBackward>> relu_bwds;
  std::map<Gradient*, std::shared_ptr<AdditionBackward>> add_bwds;
  std::map<Gradient*, std::shared_ptr<MatMulBackward>> mm_bwds;
  for (auto& kv : v->bwd) {
    if (auto rb = std::dynamic_pointer_cast<ReLUBackward>(kv.second)) relu_bwds[rb->operand_data.get()] = rb;
    if (auto ab = std::dynamic_pointer_cast<AdditionBackward>(kv.second)) add_bwds[ab->gradient.get()] = ab;
    if (auto mb = std::dynamic_pointer_cast<MatMulBackward>(kv.second)) mm_bwds.emplace(mb->left_grad.get(), mb);
  }

  // producer + bias add -> one kernel with a bias epilogue: mm_t + (N) row bias (the Linear layer) or convolution +
  // (Cout,1,1) bias (the Conv2d layer).  The bias has the sum's element type; the product has no other holder than its
  // producer and this consumer (no live variable handle, no second consumer).
  std::map<Tensor*, std::shared_ptr<Addition>> fused_adds;  // sum -> addition, for the ReLU pass below
  for (auto& kv : v->fwd) {
    auto add = std::dynamic_pointer_cast<Addition>(kv.second);
    if (!add || add->fused_gemm || add->fused_conv) continue;
    const Shape& os = add->data->shape;
    const Shape& bs = add->right->shape;
    if (add->right->dtype != add->data->dtype || add->left->shape != os || add->left.use_count() != 2) continue;
    auto mm = gemms.find(add->left.get());
    auto cv = convs.find(add->left.get());
    if (mm != gemms.end() && mm->second->t && os.size() == 2 && bs.size() == 1 && bs[0] == os[1]) {
      add->fused_gemm = mm->second;
      mm->second->skip = true;
    } else if (cv != convs.end() && os.size() == 4 && bs.size() == 3 && bs[0] == os[1] && bs[1] == 1 && bs[2] == 1) {
      add->fused_conv = cv->second;
      cv->second->skip = true;
    }
  }
  for (auto& kv : v->fwd)
    if (auto add = std::dynamic_pointer_cast<Addition>(kv.second))
      if ((add->fused_gemm || add->fused_conv) && !add->fused_relu_out) fused_adds[add->data.get()] = add;
  // ... followed by ReLU: relu(producer + bias) in the same epilogue.  The pre-activation z is then never stored, so the
  // ReLU backward node masks with y > 0 instead of z > 0 (identical: y = max(z, 0)).
  for (auto& kv : v->fwd) {
    auto relu = std::dynamic_pointer_cast<ReLU>(kv.second);
    if (!relu || relu->skip) continue;
    auto it = fused_adds.find(relu->operand.get());
    if (it == fused_adds.end()) continue;
    auto add = it->second;
    auto rbi = relu_bwds.find(add->data.get());
    ReLUBackward* rb = rbi == relu_bwds.end() ? nullptr : rbi->second.get();
    // holders of z: the Addition, the ReLU, (the ReLU backward) -- anything else (a live handle, another consumer)
    // needs z in memory
    if (add->data.use_count() != (rb ? 3 : 2)) continue;
    if (relu->data->dtype != add->data->dtype) continue;
    add->fused_relu_out = relu->data;
    relu->skip = true;
    if (rb) rb->operand_data = relu->data;
  }
  // level 2: ReLU backward into the epilogue of the matmul that produces its output gradient
  if (g_fusion >= 2) {
    for (auto& kv : v->bwd) {
      auto rb = std::dynamic_pointer_cast<ReLUBackward>(kv.second);
      if (!rb || rb->skip || !rb->gradient || !rb->operand_grad) continue;
      Gradient* gh = rb->gradient.get();
      if (gh->alias || gh->ptr || gh->is_leaf || gh->hook || rb->gradient.use_count() != 2) continue;
      if (rb->operand_grad->dtype != gh->dtype || rb->operand_data->dtype != gh->dtype) continue;
      auto mbi = mm_bwds.find(gh);
      if (mbi == mm_bwds.end() || mbi->second->left_dst) continue;
      MatMulBackward* mb = mbi->second.get();
      mb->left_mask = rb->operand_data;
      mb->left_dst = rb->operand_grad;
      mb->single_pass = true;
      rb->skip = true;
      // the Addition below the ReLU (z = x.W^T + b): its (K) row-bias gradient is the column sum of the dZ this GEMM
      // writes -- take it in the same epilogue when it is an f32 gradient nobody else aliases.  LEVEL 3 ONLY: correct
      // (the GPU suite runs it) and four launches fewer per config-4 step, but no faster: 0.791 vs 0.793 ms -- the
      // butterfly and the 1.3 M f32 atomics cost what the two column-sum passes did (a first version with scalar mask
      // loads was 0.2 ms SLOWER: its epilogue outlasted the main loop).  One atomic per column and CTA would be next.
      auto abi = add_bwds.find(rb->operand_grad.get());
      if (g_fusion < 3 || abi == add_bwds.end()) continue;
      AdditionBackward* ab = abi->second.get();
      if (ab->skip || ab->right_fused || !ab->right_grad) continue;
      Gradient* bg = ab->right_grad.get();
      const Shape& gs = rb->operand_grad->shape;
      if (bg->alias || bg->dtype != NK_F32 || gs.size() != 2 || bg->shape.size() != 1 || bg->shape[0] != gs[1]) continue;
      mb->left_colsum = ab->right_grad;
      ab->right_fused = true;
    }
  }
  // gradient aliasing: dL += G with identical shape/dtype and a single consumer => L.grad is G
  for (auto& kv : v->bwd) {
    auto ab = std::dynamic_pointer_cast<AdditionBackward>(kv.second);
    if (!ab) continue;
    GradientP& g = ab->left_grad;
    if (!g || ab->left_aliased || g->alias || g->ptr) continue;
    if (g->shape != ab->gradient->shape || g->dtype != ab->gradient->dtype) continue;
    if (!g->owned) continue;
    // only a gradient produced by a Backward node may be aliased: a leaf's gradient belongs to the user (hooks and
    // reduce-scatter plans sit on it, it accumulates over backward() calls and outlives this graph)
    if (g->is_leaf || g->hook || g->rs_world > 1) continue;
    if (g.use_count() != 2) continue;  // the producer's Backward node + this node
    g->alias = ab->gradient;
    ab->left_aliased = true;
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
    v->data->rptr();  // leaves are allocated (zero-filled) eagerly
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
    not_null({a, out}, "nkg_requires_grad");
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
    not_null({a, out}, "nkg_clone");
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
    not_null({v}, "nkg_forward");
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
    for (auto& op : v->bwd_buf)
      if (op->single_pass && op->runs > 0)
        fail(NK_ERR_UNSUPPORTED, "this tape was optimised for ONE backward pass (fusion level 2: %s never stores the "
             "gradient it would have to accumulate); build the graph again or use nkg_set_fusion(1)", op->name());
    for (auto& op : v->bwd_buf)
      if (op->runs > 0) op->unalias();
    v->grad->fill(seed);
    // last writer (reverse tape position) of every hooked gradient in this pass; every node reports its writes
    // (grad_written), and the hook fires on the report of the last writer
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
      if ((*it)->skip) continue;
      g_bwd_pos = any_hook ? pos : -2;
      (*it)->backward();
      (*it)->runs++;
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
    not_null({a, b, out}, "mm");
    require_same_dtype(a, b, t ? "mm_t" : "mm");
    const Shape &ls = a->data->shape, &rs = b->data->shape;
    if (ls.size() != 2 || rs.size() != 2) fail(NK_ERR_INVALID_ARG, "mm: operands must be 2-dimensional");
    const int64_t inner_r = t ? rs[1] : rs[0];
    if (ls[1] != inner_r)
      fail(NK_ERR_INVALID_ARG, "mm: incompatible shapes (%lld, %lld) and (%lld, %lld)%s", (long long)ls[0],
           (long long)ls[1], (long long)rs[0], (long long)rs[1], t ? " (transposed rhs)" : "");
    *out = record(
        {a, b}, Shape{ls[0], t ? rs[0] : rs[1]}, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<MatMul>(a->ctx, a->data, b->data, d, t); },
        // a null operand gradient (a Var) is a half that is never built
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<MatMulBackward>(a->ctx, g, a->data, b->data, a->grad, b->grad, t);
        });
  });
}

int nkg_mm(nkg_var* a, nkg_var* b, nkg_var** out) { return matmul_impl(a, b, false, out); }
int nkg_mm_t(nkg_var* a, nkg_var* b, nkg_var** out) { return matmul_impl(a, b, true, out); }

int nkg_add(nkg_var* a, nkg_var* b, nkg_var** out) {
  return guard([&] {
    not_null({a, b, out}, "add");
    require_same_dtype(a, b, "add");
    *out = record(
        {a, b}, cobroadcast(a->data->shape, b->data->shape), a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Addition>(a->ctx, a->data, b->data, d); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<AdditionBackward>(a->ctx, g, a->grad, b->grad);
        });
  });
}

int nkg_relu(nkg_var* a, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "relu");
    *out = record(
        {a}, a->data->shape, a->data->dtype, [&](const TensorP& d) { return std::make_shared<ReLU>(a->ctx, a->data, d); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<ReLUBackward>(a->ctx, g, a->data, a->grad); });
  });
}

static int softmax_impl(nkg_var* a, int axis, bool log, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "softmax");
    if (axis < 0 || axis >= (int)a->data->shape.size()) fail(NK_ERR_INVALID_ARG, "softmax: axis %d out of range", axis);
    *out = record(
        {a}, a->data->shape, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Softmax>(a->ctx, a->data, d, axis, log); },
        [&](const TensorP& d, const GradientP& g) {
          return std::make_shared<SoftmaxBackward>(a->ctx, g, d, a->grad, axis, log);
        });
  });
}
int nkg_softmax(nkg_var* a, int axis, nkg_var** out) { return softmax_impl(a, axis, false, out); }
int nkg_log_softmax(nkg_var* a, int axis, nkg_var** out) { return softmax_impl(a, axis, true, out); }

static int summean_impl(nkg_var* a, bool mean, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "sum");
    *out = record(
        {a}, Shape{}, NK_F32, [&](const TensorP& d) { return std::make_shared<SumMean>(a->ctx, a->data, d, mean); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<SumMeanBackward>(a->ctx, g, a->grad, mean); });
  });
}
int nkg_sum(nkg_var* a, nkg_var** out) { return summean_impl(a, false, out); }
int nkg_mean(nkg_var* a, nkg_var** out) { return summean_impl(a, true, out); }

static int loss_impl(nkg_var* input, nkg_var* target, int reduction, int kind, nkg_var** out) {
  return guard([&] {
    not_null({input, target, out}, "loss");
    const bool nll = kind == kNll;
    static const char* const who[] = {"mse_loss", "nll_loss", "mae", "bce", "bce_with_logits", "kldiv"};
    if (nll) {
      // class ids are stored as floats (nll/mod.rs:55 `target as usize`): an f32 target is accepted whatever the
      // input's element type; a bf16 target represents integers exactly only up to 256
      if (input->ctx != target->ctx) fail(NK_ERR_INVALID_ARG, "nll_loss: operands live on different devices");
      if (target->data->dtype == NK_BF16 && input->data->shape.size() == 2 && input->data->shape[1] > 256)
        fail(NK_ERR_INVALID_ARG, "nll_loss: a bf16 target cannot hold class ids above 256; pass the target as f32");
    } else {
      require_same_dtype(input, target, who[kind]);
    }
    if (nll) {
      if (input->data->shape.size() != 2 || target->data->shape.size() != 1 ||
          target->data->shape[0] != input->data->shape[0])
        fail(NK_ERR_INVALID_ARG, "nll_loss: input must be (N, C) and target (N)");
    } else if (input->data->shape != target->data->shape) {
      fail(NK_ERR_INVALID_ARG, "%s: input and target shapes differ", who[kind]);
    }
    if (kind == kKlDiv && (input->data->shape.empty() || input->data->shape[0] == 0))
      fail(NK_ERR_INVALID_ARG, "kldiv: the input needs a leading (batch) dimension");
    if (target->diff()) fail(NK_ERR_INVALID_ARG, "loss: the target must not be differentiable");
    const bool mean = reduction == NKG_MEAN;
    *out = record(
        {input, target}, Shape{}, NK_F32,
        [&](const TensorP& d) { return std::make_shared<Loss>(input->ctx, input->data, target->data, d, mean, kind); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<LossBackward>(input->ctx, g, input->data, target->data, input->grad, mean, kind);
        });
  });
}
int nkg_mse_loss(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kMse, o); }
int nkg_nll_loss(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kNll, o); }
int nkg_mae(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kMae, o); }
int nkg_bce(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kBce, o); }
int nkg_bce_with_logits(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kBceWithLogits, o); }
int nkg_kldiv(nkg_var* i, nkg_var* t, int r, nkg_var** o) { return loss_impl(i, t, r, kKlDiv, o); }

int nkg_status_create(int train, nkg_status** out) {
  return guard([&] {
    not_null({out}, "nkg_status_create");
    *out = new nkg_status{std::make_shared<bool>(train != 0)};
  });
}
int nkg_status_set(nkg_status* s, int train) {
  return guard([&] {
    not_null({s}, "nkg_status_set");
    *s->train = train != 0;
  });
}
int nkg_status_get(nkg_status* s) { return s ? int(*s->train) : NK_ERR_INVALID_ARG; }
int nkg_status_release(nkg_status* s) {
  delete s;
  return NK_OK;
}

int nkg_dropout(nkg_var* a, double p, nkg_status* status, nkg_var** out) {
  return guard([&] {
    not_null({a, status, out}, "dropout");
    if (!(p >= 0.0 && p <= 1.0)) fail(NK_ERR_INVALID_ARG, "Wrong probability received: %g.", p);  // dropout/mod.rs:38-40
    TensorP mask;
    if (p != 0.0 && 1.0 - p != 0.0) {  // only a drawing forward has a mask
      mask = std::make_shared<Tensor>(a->ctx, Shape{(a->data->n() + 31) / 32}, NK_F32);  // 32-bit words
      mask->wptr();
    }
    auto state = std::make_shared<DropoutState>();
    *out = record(
        {a}, a->data->shape, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Dropout>(a->ctx, a->data, d, mask, p, status->train, state); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<DropoutBackward>(a->ctx, g, a->grad, mask, p, state);
        });
  });
}

int nkg_pad(nkg_var* a, int64_t ph, int64_t pw, float value, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "pad");
    const Shape& s = a->data->shape;
    if (s.size() != 4 || ph < 0 || pw < 0) fail(NK_ERR_INVALID_ARG, "pad: expects a (N, C, H, W) operand and padding >= 0");
    *out = record(
        {a}, Shape{s[0], s[1], s[2] + 2 * ph, s[3] + 2 * pw}, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Pad>(a->ctx, a->data, d, ph, pw, value); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<PadBackward>(a->ctx, g, a->grad, ph, pw); });
  });
}

int nkg_convolution(nkg_var* kernel, nkg_var* input, int64_t sh, int64_t sw, int64_t dh, int64_t dw, int64_t groups,
                    nkg_var** out) {
  return guard([&] {
    not_null({kernel, input, out}, "convolution");
    require_same_dtype(kernel, input, "convolution");
    const Shape &ks = kernel->data->shape, &is = input->data->shape;
    // check_conv_args / check_groups_args, utils.rs:427-496 (same messages)
    if (is.size() != 4) fail(NK_ERR_UNSUPPORTED, "convolution: only 2d convolutions (N, C, H, W) run on the device");
    if (ks.size() != is.size()) fail(NK_ERR_INVALID_ARG, "Invalid kernel shape for 2d conv");
    if (sh < 1 || sw < 1 || dh < 1 || dw < 1 || groups < 1) fail(NK_ERR_INVALID_ARG, "Invalid stride/dilation/groups for 2d conv.");
    if (is[2] < (ks[2] - 1) * dh + 1 || is[3] < (ks[3] - 1) * dw + 1)
      fail(NK_ERR_INVALID_ARG, "The kernel size can't be greater than actual input size.");
    check_conv_channels(ks, is, groups);
    const ConvArgs a{is[0], is[1], is[2], is[3], ks[0], ks[2], ks[3], sh, sw, dh, dw, groups};
    *out = record(
        {kernel, input},
        Shape{is[0], ks[0], (is[2] - dh * (ks[2] - 1) - 1) / sh + 1, (is[3] - dw * (ks[3] - 1) - 1) / sw + 1},
        input->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Convolution>(kernel->ctx, input->data, kernel->data, d, a); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<ConvolutionBackward>(kernel->ctx, g, input->data, kernel->data, input->grad,
                                                       kernel->grad, a);
        });
  });
}

int nkg_flatten(nkg_var* a, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "flatten");
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
    not_null({a, b, out}, "binary op");
    require_same_dtype(a, b, op == NK_BIN_SUB ? "sub" : op == NK_BIN_MUL ? "mul" : "div");
    *out = record(
        {a, b}, cobroadcast(a->data->shape, b->data->shape), a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Binary>(a->ctx, a->data, b->data, d, op); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<BinaryBackward>(a->ctx, g, a->data, b->data, a->grad, b->grad, op);
        });
  });
}
int nkg_sub(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_SUB, out); }
int nkg_mul(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_MUL, out); }
int nkg_div(nkg_var* a, nkg_var* b, nkg_var** out) { return binary_impl(a, b, NK_BIN_DIV, out); }

int nkg_unary(nkg_var* a, int op, int iparam, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "unary op");
    if (op < NK_UN_NEG || op > NK_UN_POWI) fail(NK_ERR_INVALID_ARG, "unary op: bad op %d", op);
    *out = record(
        {a}, a->data->shape, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Unary>(a->ctx, a->data, d, op, iparam); },
        [&](const TensorP& d, const GradientP& g) {
          const bool keeps_output = op == NK_UN_EXP || op == NK_UN_SQRT || op == NK_UN_SIGMOID || op == NK_UN_TANH;
          TensorP saved = op == NK_UN_NEG ? nullptr : (keeps_output ? d : a->data);
          return std::make_shared<UnaryBackward>(a->ctx, g, std::move(saved), a->grad, op, iparam);
        });
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
    not_null({a, out}, "t");
    *out = record(
        {a}, Shape(a->data->shape.rbegin(), a->data->shape.rend()), a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Transpose>(a->ctx, a->data, d); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<TransposeBackward>(a->ctx, g, a->grad); });
  });
}

int nkg_pad_mode(nkg_var* a, int nsp, const int64_t* padding, int mode, float value, nkg_var** out) {
  return guard([&] {
    not_null({a, out, padding}, "pad");
    const Shape& s = a->data->shape;
    if (nsp < 1 || nsp > 3 || (int)s.size() != nsp + 2)
      fail(NK_ERR_INVALID_ARG, "pad: expects a (N, C, ...) operand with %d sample dimensions", nsp);
    if (mode < NK_PAD_CONSTANT || mode > NK_PAD_REPLICATIVE) fail(NK_ERR_INVALID_ARG, "pad: bad mode %d", mode);
    Shape os = s;
    int64_t pad[3] = {0, 0, 0};
    for (int k = 0; k < nsp; ++k) {
      if (padding[k] < 0) fail(NK_ERR_INVALID_ARG, "pad: padding must be >= 0");
      if (mode == NK_PAD_REFLECTIVE && padding[k] > 0 && padding[k] >= s[2 + k])
        fail(NK_ERR_INVALID_ARG, "pad: reflective padding %lld must be smaller than the dimension %lld",
             (long long)padding[k], (long long)s[2 + k]);
      os[2 + k] += 2 * padding[k];
      pad[k] = padding[k];
    }
    *out = record(
        {a}, os, a->data->dtype,
        [&](const TensorP& d) { return std::make_shared<PadNd>(a->ctx, a->data, d, nsp, pad, mode, value); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<PadNdBackward>(a->ctx, g, a->grad, nsp, pad); });
  });
}

// checks the operand and the per-axis arguments of a pooling op, then records it; nothing is recorded on an error
static int pool_record(int op, nkg_var* a, int nsp, const int64_t* kernel, const int64_t* stride,
                       const int64_t* padding, const int64_t* dilation, const int64_t* out_size, bool ceil_mode,
                       bool include_pad, nkg_var** out) {
  static const char* const who[] = {"max_pool", "avg_pool", "adaptive_avg_pool"};
  const char* name = who[op];
  return guard([&] {
    not_null({a, out}, name);
    if (op == kPoolAdaptive)
      not_null({out_size}, name);
    else
      not_null({kernel, stride, padding, op == kPoolMax ? dilation : kernel}, name);
    const Shape& s = a->data->shape;
    if (nsp < 1 || nsp > 3 || (int)s.size() != nsp + 2)
      fail(NK_ERR_INVALID_ARG, "%s: expects a (N, C, ...) operand with %d sample dimensions (1 to 3), got %d dimensions",
           name, nsp, (int)s.size());
    PoolArgs pa{op, nsp, include_pad, {1, 1, 1}, {1, 1, 1}, {0, 0, 0}, {1, 1, 1}};
    Shape os = s;
    for (int i = 0; i < nsp; ++i) {
      const int64_t L = s[2 + i];
      if (op == kPoolAdaptive) {
        if (out_size[i] < 1 || L < 1)
          fail(NK_ERR_INVALID_ARG, "%s: input and output sizes must be >= 1 (axis %d: %lld, %lld)", name, i,
               (long long)L, (long long)out_size[i]);
        os[2 + i] = out_size[i];
        continue;
      }
      pa.k[i] = kernel[i], pa.s[i] = stride[i], pa.p[i] = padding[i], pa.d[i] = op == kPoolMax ? dilation[i] : 1;
      char msg[160];
      if (nk_pool_check_axis(name, i, L, pa.k[i], pa.s[i], pa.p[i], pa.d[i], msg, sizeof msg))
        fail(NK_ERR_INVALID_ARG, "%s", msg);
      os[2 + i] = nk_pool_out_extent(L, pa.k[i], pa.s[i], pa.p[i], pa.d[i], ceil_mode);
      if (os[2 + i] < 1)
        fail(NK_ERR_INVALID_ARG, "%s: output size would be %lld (axis %d, input %lld)", name, (long long)os[2 + i], i,
             (long long)L);
    }
    TensorP idx;
    if (op == kPoolMax && a->diff()) {
      idx = std::make_shared<Tensor>(a->ctx, os, NK_F32);  // int32 words
      idx->wptr();
    }
    *out = record(
        {a}, os, a->data->dtype, [&](const TensorP& d) { return std::make_shared<Pool>(a->ctx, a->data, d, idx, pa); },
        [&](const TensorP&, const GradientP& g) { return std::make_shared<PoolBackward>(a->ctx, g, a->grad, idx, pa); });
  });
}

int nkg_max_pool(nkg_var* a, int nsp, const int64_t* kernel, const int64_t* stride, const int64_t* padding,
                 const int64_t* dilation, int ceil_mode, nkg_var** out) {
  return pool_record(kPoolMax, a, nsp, kernel, stride, padding, dilation, nullptr, ceil_mode != 0, true, out);
}

int nkg_avg_pool(nkg_var* a, int nsp, const int64_t* kernel, const int64_t* stride, const int64_t* padding,
                 int ceil_mode, int count_include_pad, nkg_var** out) {
  return pool_record(kPoolAvg, a, nsp, kernel, stride, padding, nullptr, nullptr, ceil_mode != 0,
                     count_include_pad != 0, out);
}

int nkg_adaptive_avg_pool(nkg_var* a, int nsp, const int64_t* output_size, nkg_var** out) {
  return pool_record(kPoolAdaptive, a, nsp, nullptr, nullptr, nullptr, nullptr, output_size, false, false, out);
}

// a (C,) operand of a normalization: w / b of the operand's dtype, or a running statistic: a non-differentiable f32
// leaf
static void norm_param(nkg_var* p, nkg_var* x, const Shape& want, const char* who, const char* what, bool stat) {
  if (!p) return;
  if (p->ctx != x->ctx) fail(NK_ERR_INVALID_ARG, "%s: %s lives on another device", who, what);
  if (p->data->shape != want)
    fail(NK_ERR_INVALID_ARG, "%s: %s must have shape %s, got %s", who, what, shape_str(want).c_str(),
         shape_str(p->data->shape).c_str());
  if (stat) {
    if (p->data->dtype != NK_F32) fail(NK_ERR_INVALID_ARG, "%s: %s must be f32", who, what);
    if (p->diff()) fail(NK_ERR_INVALID_ARG, "%s: %s must not be differentiable", who, what);
    // the forward writes it in place: only a leaf's buffer is the caller's alone, never another node's output
    if (!p->fwd.empty()) fail(NK_ERR_INVALID_ARG, "%s: %s must be a leaf", who, what);
  } else {
    require_same_dtype(p, x, who);
  }
}

int nkg_batch_norm(nkg_var* x, nkg_var* weight, nkg_var* bias, nkg_var* running_mean, nkg_var* running_var,
                   nkg_status* status, float momentum, float eps, nkg_var** out) {
  return guard([&] {
    static const char* who = "batch_norm";
    not_null({x, status, out}, who);
    const Shape& s = x->data->shape;
    if (s.size() < 2) fail(NK_ERR_INVALID_ARG, "%s: expects an (N, C, ...) operand, got %d dimensions", who, (int)s.size());
    if (s[1] < 1) fail(NK_ERR_INVALID_ARG, "%s: no channels", who);
    if (!running_mean != !running_var)
      fail(NK_ERR_INVALID_ARG, "%s: running_mean and running_var are both given or both NULL", who);
    if (!(eps >= 0.f)) fail(NK_ERR_INVALID_ARG, "%s: eps must be >= 0, got %g", who, eps);
    const Shape cs{s[1]};
    norm_param(weight, x, cs, who, "weight", false);
    norm_param(bias, x, cs, who, "bias", false);
    norm_param(running_mean, x, cs, who, "running_mean", true);
    norm_param(running_var, x, cs, who, "running_var", true);
    bn_check_batch(s, *status->train || !running_mean);
    auto sm = std::make_shared<Tensor>(x->ctx, cs, NK_F32), sr = std::make_shared<Tensor>(x->ctx, cs, NK_F32);
    sm->wptr();
    sr->wptr();
    auto state = std::make_shared<BatchNormState>();
    TensorP w = weight ? weight->data : nullptr, b = bias ? bias->data : nullptr;
    TensorP rm = running_mean ? running_mean->data : nullptr, rv = running_var ? running_var->data : nullptr;
    std::vector<nkg_var*> operands{x};
    if (weight) operands.push_back(weight);
    if (bias) operands.push_back(bias);
    *out = record(
        operands, s, x->data->dtype,
        [&](const TensorP& d) {
          return std::make_shared<BatchNorm>(x->ctx, x->data, w, b, rm, rv, d, sm, sr, status->train, state, momentum,
                                             eps);
        },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<BatchNormBackward>(x->ctx, g, x->grad, weight ? weight->grad : nullptr,
                                                     bias ? bias->grad : nullptr, x->data, w, sm, sr, state);
        });
  });
}

int nkg_layer_norm(nkg_var* x, int k, nkg_var* weight, nkg_var* bias, float eps, nkg_var** out) {
  return guard([&] {
    static const char* who = "layer_norm";
    not_null({x, out}, who);
    const Shape& s = x->data->shape;
    if (k < 1 || k > (int)s.size())
      fail(NK_ERR_INVALID_ARG, "%s: normalized_shape has %d dimensions, the input %d", who, k, (int)s.size());
    if (!(eps >= 0.f)) fail(NK_ERR_INVALID_ARG, "%s: eps must be >= 0, got %g", who, eps);
    const Shape ns(s.end() - k, s.end());
    const int64_t cols = numel(ns);
    if (cols < 1) fail(NK_ERR_INVALID_ARG, "%s: normalized_shape %s has no elements", who, shape_str(ns).c_str());
    norm_param(weight, x, ns, who, "weight", false);
    norm_param(bias, x, ns, who, "bias", false);
    const Shape rs{x->data->n() / cols};
    auto sm = std::make_shared<Tensor>(x->ctx, rs, NK_F32), sr = std::make_shared<Tensor>(x->ctx, rs, NK_F32);
    sm->wptr();
    sr->wptr();
    TensorP w = weight ? weight->data : nullptr, b = bias ? bias->data : nullptr;
    std::vector<nkg_var*> operands{x};
    if (weight) operands.push_back(weight);
    if (bias) operands.push_back(bias);
    *out = record(
        operands, s, x->data->dtype,
        [&](const TensorP& d) { return std::make_shared<LayerNorm>(x->ctx, x->data, w, b, d, sm, sr, cols, eps); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<LayerNormBackward>(x->ctx, g, x->grad, weight ? weight->grad : nullptr,
                                                     bias ? bias->grad : nullptr, x->data, w, sm, sr, cols);
        });
  });
}

static int matvec_impl(nkg_var* mat, nkg_var* vec, bool vm, nkg_var** out) {
  return guard([&] {
    not_null({mat, vec, out}, "mv");
    require_same_dtype(mat, vec, vm ? "vm" : "mv");
    const Shape &ms = mat->data->shape, &vs = vec->data->shape;
    if (ms.size() != 2 || vs.size() != 1) fail(NK_ERR_INVALID_ARG, "%s: needs a matrix and a vector", vm ? "vm" : "mv");
    const int64_t need = vm ? ms[0] : ms[1];
    if (vs[0] != need)
      fail(NK_ERR_INVALID_ARG, "%s: incompatible shapes (%lld, %lld) and (%lld)", vm ? "vm" : "mv", (long long)ms[0],
           (long long)ms[1], (long long)vs[0]);
    *out = record(
        {vm ? vec : mat, vm ? mat : vec}, Shape{vm ? ms[1] : ms[0]}, mat->data->dtype,
        [&](const TensorP& d) { return std::make_shared<MatVec>(mat->ctx, mat->data, vec->data, d, vm); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<MatVecBackward>(mat->ctx, g, mat->data, vec->data, mat->grad, vec->grad, vm);
        });
  });
}
int nkg_mv(nkg_var* mat, nkg_var* vec, nkg_var** out) { return matvec_impl(mat, vec, false, out); }
int nkg_vm(nkg_var* vec, nkg_var* mat, nkg_var** out) { return matvec_impl(mat, vec, true, out); }

int nkg_vv(nkg_var* a, nkg_var* b, nkg_var** out) {
  return guard([&] {
    not_null({a, b, out}, "vv");
    require_same_dtype(a, b, "vv");
    if (a->data->shape.size() != 1 || b->data->shape.size() != 1 || a->data->shape[0] != b->data->shape[0])
      fail(NK_ERR_INVALID_ARG, "vv: needs two vectors of the same length");
    *out = record(
        {a, b}, Shape{}, NK_F32, [&](const TensorP& d) { return std::make_shared<VecVec>(a->ctx, a->data, b->data, d); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<VecVecBackward>(a->ctx, g, a->data, b->data, a->grad, b->grad);
        });
  });
}

int nkg_convolution_nd(nkg_var* kernel, nkg_var* input, int nsp, const int64_t* stride, const int64_t* dilation,
                       int64_t groups, nkg_var** out) {
  return guard([&] {
    not_null({kernel, input, out, stride, dilation}, "convolution");
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
    check_conv_channels(ks, is, groups);
    *out = record(
        {kernel, input}, os, input->data->dtype,
        [&](const TensorP& d) { return std::make_shared<ConvolutionNd>(kernel->ctx, input->data, kernel->data, d, a); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<ConvolutionNdBackward>(kernel->ctx, g, input->data, kernel->data, input->grad,
                                                         kernel->grad, a);
        });
  });
}

int nkg_conv_layer(nkg_var* input, nkg_var* weight, nkg_var* bias, int nsp, const int64_t* padding, int mode, float value,
                   const int64_t* stride, const int64_t* dilation, nkg_var** out) {
  return guard([&] {
    not_null({input, weight, out, padding, stride, dilation}, "conv_layer");
    if (nsp != 1 && nsp != 3) fail(NK_ERR_INVALID_ARG, "conv_layer: 1 or 3 sample dimensions (got %d)", nsp);
    require_same_dtype(weight, input, "conv_layer");
    if (bias) require_same_dtype(bias, input, "conv_layer");
    const Shape &ks = weight->data->shape, &is = input->data->shape;
    if ((int)is.size() != nsp + 2) fail(NK_ERR_INVALID_ARG, "conv_layer: input rank does not match %dd conv", nsp);
    if (ks.size() != is.size()) fail(NK_ERR_INVALID_ARG, "Invalid kernel shape for %dd conv", nsp);
    if (mode < NK_PAD_CONSTANT || mode > NK_PAD_REPLICATIVE) fail(NK_ERR_INVALID_ARG, "pad: bad mode %d", mode);
    check_conv_channels(ks, is, 1);
    ConvLayerArgs a;
    a.nsp = nsp, a.mode = mode, a.value = value, a.n = is[0], a.cin = is[1], a.cout = ks[0];
    Shape os{is[0], ks[0]};
    for (int k = 0; k < nsp; ++k) {
      if (padding[k] < 0) fail(NK_ERR_INVALID_ARG, "pad: padding must be >= 0");
      if (mode == NK_PAD_REFLECTIVE && padding[k] > 0 && padding[k] >= is[2 + k])
        fail(NK_ERR_INVALID_ARG, "pad: reflective padding %lld must be smaller than the dimension %lld",
             (long long)padding[k], (long long)is[2 + k]);
      if (stride[k] < 1 || dilation[k] < 1) fail(NK_ERR_INVALID_ARG, "Invalid stride/dilation for %dd conv.", nsp);
      const int64_t padded = is[2 + k] + 2 * padding[k];
      if (padded < (ks[2 + k] - 1) * dilation[k] + 1)
        fail(NK_ERR_INVALID_ARG, "The kernel size can't be greater than actual input size.");
      a.in[k] = is[2 + k], a.k[k] = ks[2 + k], a.s[k] = stride[k], a.d[k] = dilation[k], a.pad[k] = padding[k];
      os.push_back((padded - dilation[k] * (ks[2 + k] - 1) - 1) / stride[k] + 1);
    }
    if (bias) {
      Shape bs(nsp + 1, 1);
      bs[0] = ks[0];
      if (bias->data->shape != bs)
        fail(NK_ERR_INVALID_ARG, "conv_layer: bias must be %s, got %s", shape_str(bs).c_str(), shape_str(bias->data->shape).c_str());
    }
    std::vector<nkg_var*> operands{input, weight};
    if (bias) operands.push_back(bias);
    *out = record(
        operands, os, input->data->dtype,
        [&](const TensorP& d) {
          return std::make_shared<ConvLayer>(input->ctx, input->data, weight->data, bias ? bias->data : nullptr, d, a);
        },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<ConvLayerBackward>(input->ctx, g, input->data, weight->data, input->grad, weight->grad,
                                                     bias ? bias->grad : nullptr, a);
        });
  });
}

// ---------------------------------------------------------------- chunks / recurrent cells / sequence layers
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
    for (int64_t i = 0; i < nblocks; ++i)
      outs[i] = record(
          {a}, cs, a->data->dtype, [&](const TensorP& d) { return std::make_shared<Chunk>(a->ctx, a->data, d, i); },
          [&](const TensorP&, const GradientP& g) { return std::make_shared<ChunkBackward>(a->ctx, g, a->grad, i); });
  });
}

// var.rs:564-587 / 622-645, vardiff.rs:627-641 / 681-: one node for every operand count and every mix of Var and
// VarDiff operands (the reference's four homogeneous methods and its Cat / Stack traits for mixed pairs)
static void cat_impl(nkg_var* const* vars, int count, int axis, bool stack, nkg_var** out) {
  const char* who = stack ? "stack" : "cat";
  not_null({vars, out}, who);
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
  std::vector<nkg_var*> operands(vars, vars + count);
  *out = record(
      operands, os, a->data->dtype,
      [&](const TensorP& d) {
        std::vector<TensorP> xs;
        for (nkg_var* x : operands) xs.push_back(x->data);
        return std::make_shared<Concatenate>(a->ctx, std::move(xs), d, lens, outer, inner, stack);
      },
      [&](const TensorP&, const GradientP& g) {
        std::vector<GradientP> grads;
        for (nkg_var* x : operands) grads.push_back(x->grad);
        return std::make_shared<ConcatenateBackward>(a->ctx, g, std::move(grads), lens, outer, inner, stack);
      });
}

int nkg_cat(nkg_var* const* vars, int count, int axis, nkg_var** out) {
  return guard([&] { cat_impl(vars, count, axis, false, out); });
}

int nkg_stack(nkg_var* const* vars, int count, int axis, nkg_var** out) {
  return guard([&] { cat_impl(vars, count, axis, true, out); });
}

int nkg_unsqueeze(nkg_var* a, int axis, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "unsqueeze");
    Shape s = a->data->shape;
    if (axis < 0 || axis > (int)s.size())
      fail(NK_ERR_INVALID_ARG, "unsqueeze: axis %d out of range for a %d-dimensional operand", axis, (int)s.size());
    if (s.size() + 1 > NK_MAX_DIMS) fail(NK_ERR_INVALID_ARG, "unsqueeze: the result would have more than %d dimensions", NK_MAX_DIMS);
    s.insert(s.begin() + axis, 1);
    *out = view_of(a, s);
  });
}

int nkg_reshape(nkg_var* a, int ndim, const int64_t* shape, nkg_var** out) {
  return guard([&] {
    not_null({a, out}, "reshape");
    if (ndim < 0 || ndim > NK_MAX_DIMS || (ndim > 0 && !shape))
      fail(NK_ERR_INVALID_ARG, "reshape: 0 to %d dimensions (got %d)", NK_MAX_DIMS, ndim);
    const Shape s(shape, shape + ndim);
    for (int64_t d : s)
      if (d < 0) fail(NK_ERR_INVALID_ARG, "reshape: negative dimension %lld", (long long)d);
    if (numel(s) != a->data->n())
      fail(NK_ERR_INVALID_ARG, "shape '%s' is invalid for input of size %lld", shape_str(s).c_str(),
           (long long)a->data->n());
    *out = view_of(a, s);
  });
}

int nkg_embedding(nkg_var* ids, nkg_var* weight, int64_t padding_idx, nkg_var** out) {
  return guard([&] {
    static const char* who = "embedding";
    not_null({ids, weight, out}, who);
    if (ids->ctx != weight->ctx) fail(NK_ERR_INVALID_ARG, "%s: operands live on different devices", who);
    const Shape& ws = weight->data->shape;
    if (ws.size() != 2) fail(NK_ERR_INVALID_ARG, "%s: weight must be 2-D (v, e), got %s", who, shape_str(ws).c_str());
    if (ids->diff()) fail(NK_ERR_INVALID_ARG, "%s: ids must not be differentiable", who);
    const int64_t v = ws[0];
    if (v > (int64_t(1) << 24)) fail(NK_ERR_INVALID_ARG, "%s: %lld rows exceed 2^24, where f32 ids are exact", who, (long long)v);
    if (ids->data->dtype == NK_BF16 && v > 256)
      fail(NK_ERR_INVALID_ARG, "%s: bf16 ids cannot hold ids above 256 (v = %lld); pass the ids as f32", who, (long long)v);
    if (padding_idx < -1 || padding_idx >= v)
      fail(NK_ERR_INVALID_ARG, "%s: padding_idx %lld outside [-1, %lld)", who, (long long)padding_idx, (long long)v);
    Shape os = ids->data->shape;
    if (os.size() + 1 > NK_MAX_DIMS)
      fail(NK_ERR_INVALID_ARG, "%s: the result would have more than %d dimensions", who, NK_MAX_DIMS);
    os.push_back(ws[1]);
    *out = record(
        {ids, weight}, os, weight->data->dtype,
        [&](const TensorP& d) { return std::make_shared<Embedding>(weight->ctx, ids->data, weight->data, d); },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<EmbeddingBackward>(weight->ctx, g, ids->data, weight->grad, padding_idx);
        });
  });
}

int nkg_cross_entropy(nkg_var* input, nkg_var* target, nkg_var* weight, int reduction, int64_t ignore_index,
                      float label_smoothing, nkg_var** out) {
  return guard([&] {
    static const char* who = "cross_entropy";
    not_null({input, target, out}, who);
    if (input->ctx != target->ctx || (weight && weight->ctx != input->ctx))
      fail(NK_ERR_INVALID_ARG, "%s: operands live on different devices", who);
    if (reduction != NKG_MEAN && reduction != NKG_SUM) fail(NK_ERR_INVALID_ARG, "%s: unknown reduction %d", who, reduction);
    const Shape &xs = input->data->shape, &ts = target->data->shape;
    if (xs.size() < 2 || ts.size() + 1 != xs.size() || ts[0] != xs[0] || !std::equal(ts.begin() + 1, ts.end(), xs.begin() + 2))
      fail(NK_ERR_INVALID_ARG, "%s: input must be (N, C, d1, ..., dk) and target (N, d1, ..., dk), got %s and %s", who,
           shape_str(xs).c_str(), shape_str(ts).c_str());
    const int64_t c = xs[1];
    if (c < 1) fail(NK_ERR_INVALID_ARG, "%s: the input has no classes", who);
    if (c > (int64_t(1) << 24))
      fail(NK_ERR_INVALID_ARG, "%s: %lld classes exceed 2^24, where f32 class ids are exact", who, (long long)c);
    if (target->data->dtype == NK_BF16 && c > 256)
      fail(NK_ERR_INVALID_ARG, "%s: a bf16 target cannot hold class ids above 256 (C = %lld); pass the target as f32", who,
           (long long)c);
    if (target->diff()) fail(NK_ERR_INVALID_ARG, "%s: the target must not be differentiable", who);
    if (weight) {
      if (weight->data->dtype != NK_F32 || weight->data->shape != Shape{c})
        fail(NK_ERR_INVALID_ARG, "%s: weight must be an f32 tensor of shape (%lld,), got %s", who, (long long)c,
             shape_str(weight->data->shape).c_str());
      if (weight->diff()) fail(NK_ERR_INVALID_ARG, "%s: the weight must not be differentiable", who);
    }
    if (!(label_smoothing >= 0.f && label_smoothing <= 1.f))
      fail(NK_ERR_INVALID_ARG, "%s: label_smoothing must be between 0.0 and 1.0, got %g", who, double(label_smoothing));
    const CeDims d = ce_dims(xs);
    auto lse = std::make_shared<Tensor>(input->ctx, Shape{d.n * d.s}, NK_F32);
    auto denom = std::make_shared<Tensor>(input->ctx, Shape{}, NK_F32);
    lse->wptr();
    denom->wptr();
    TensorP w = weight ? weight->data : nullptr;
    std::vector<nkg_var*> operands{input, target};
    if (weight) operands.push_back(weight);
    const bool mean = reduction == NKG_MEAN;
    *out = record(
        operands, Shape{}, NK_F32,
        [&](const TensorP& dt) {
          return std::make_shared<CrossEntropy>(input->ctx, input->data, target->data, w, dt, lse, denom, mean,
                                                ignore_index, label_smoothing);
        },
        [&](const TensorP&, const GradientP& g) {
          return std::make_shared<CrossEntropyBackward>(input->ctx, g, input->data, target->data, w, lse, denom,
                                                        input->grad, mean, ignore_index, label_smoothing);
        });
  });
}

// The operand checks of a cell step (`seq` false: input (N, I)) and of a sequence layer (`seq` true: input (T, N, I),
// T >= 1; `layer`: states (D, N, H) and parameters stacked over D = 1 or 2 directions).  Returns the operands in
// History::merge order.
static std::vector<nkg_var*> check_rnn_operands(const char* who, bool lstm, bool seq, nkg_var* x, nkg_var* c, nkg_var* h,
                                                nkg_var* w_ih, nkg_var* w_hh, nkg_var* b_ih, nkg_var* b_hh,
                                                bool outputs_given, RnnDims& dims, bool layer = false) {
  struct Arg {
    nkg_var* v;
    const char* name;
  };
  std::vector<Arg> args = {{x, "input"}, {h, "hidden"}, {w_ih, "weight_ih"}, {w_hh, "weight_hh"}, {b_ih, "bias_ih"},
                           {b_hh, "bias_hh"}};
  if (lstm) args.push_back({c, "cell_state"});
  for (const Arg& a : args)
    if (!a.v) fail(NK_ERR_INVALID_ARG, "%s: %s is NULL", who, a.name);
  if (!outputs_given) fail(NK_ERR_INVALID_ARG, "%s: NULL output", who);
  for (const Arg& a : args) {
    if (a.v->data->dtype != x->data->dtype)
      fail(NK_ERR_INVALID_ARG, "%s: %s has another element type than the input", who, a.name);
    if (a.v->ctx != x->ctx) fail(NK_ERR_INVALID_ARG, "%s: %s lives on another device than the input", who, a.name);
  }
  const int64_t G = lstm ? 4 : 3;
  const Shape& xs = x->data->shape;
  if (xs.size() != (seq ? 3u : 2u))
    fail(NK_ERR_INVALID_ARG, "%s: input must be %s, got %s", who, seq ? "(seq_len, batch, input_size)" : "(batch, input_size)",
         shape_str(xs).c_str());
  if (seq && xs[0] < 1) fail(NK_ERR_INVALID_ARG, "%s: input needs at least one time step, got %s", who, shape_str(xs).c_str());
  const Shape& hs = h->data->shape;
  const int64_t N = xs[seq ? 1 : 0], I = xs[seq ? 2 : 1];
  if (layer) {
    if (hs.size() != 3 || (hs[0] != 1 && hs[0] != 2) || hs[1] != N)
      fail(NK_ERR_INVALID_ARG, "%s: hidden must be (num_directions = 1 or 2, batch = %lld, hidden_size), got %s", who,
           (long long)N, shape_str(hs).c_str());
  } else if (hs.size() != 2 || hs[0] != N) {
    fail(NK_ERR_INVALID_ARG, "%s: hidden must be (batch = %lld, hidden_size), got %s", who, (long long)N,
         shape_str(hs).c_str());
  }
  const int64_t D = layer ? hs[0] : 1, H = hs.back();
  auto expect = [&](nkg_var* v, const char* name, Shape want) {
    if (layer) want.insert(want.begin(), D);
    if (v->data->shape != want)
      fail(NK_ERR_INVALID_ARG, "%s: %s must be %s, got %s", who, name, shape_str(want).c_str(),
           shape_str(v->data->shape).c_str());
  };
  if (lstm) expect(c, "cell_state", {N, H});
  expect(w_ih, "weight_ih", {G * H, I});
  expect(w_hh, "weight_hh", {G * H, H});
  expect(b_ih, "bias_ih", {G * H});
  expect(b_hh, "bias_hh", {G * H});
  dims = {seq ? xs[0] : 1, N, I, H, D};
  std::vector<nkg_var*> operands;   // History::merge over every operand
  for (const Arg& a : args) operands.push_back(a.v);
  return operands;
}

static void cell_impl(bool lstm, nkg_var* x, nkg_var* c, nkg_var* h, nkg_var* w_ih, nkg_var* w_hh, nkg_var* b_ih,
                      nkg_var* b_hh, nkg_var** new_c, nkg_var** new_h) {
  const char* who = lstm ? "lstm_cell" : "gru_cell";
  RnnDims dm;
  const std::vector<nkg_var*> operands =
      check_rnn_operands(who, lstm, false, x, c, h, w_ih, w_hh, b_ih, b_hh, new_h && (!lstm || new_c), dm);
  const int64_t N = dm.N, H = dm.H;
  std::shared_ptr<RnnCell> cell;
  std::shared_ptr<RnnCellBackward> cell_bwd;
  nkg_var* vh = record(
      operands, Shape{N, H}, x->data->dtype,
      [&](const TensorP& d) {
        cell = std::make_shared<RnnCell>(
            x->ctx, lstm, CellOperands{x->data, h->data, lstm ? c->data : nullptr, w_ih->data, w_hh->data, b_ih->data, b_hh->data},
            d);
        return cell;
      },
      [&](const TensorP&, const GradientP& g) {
        cell_bwd = std::make_shared<RnnCellBackward>(
            x->ctx, g, *cell,
            CellGrads{x->grad, h->grad, lstm ? c->grad : nullptr, w_ih->grad, w_hh->grad, b_ih->grad, b_hh->grad});
        return cell_bwd;
      });
  if (lstm) {   // the second output: same tapes, same op id (merging the two histories keeps one node)
    nkg_var* vc = new nkg_var(*vh);
    vc->data = cell->c_out;
    if (cell_bwd) vc->grad = cell_bwd->c_out_grad;
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

// `layer` (nkg_lstm_layer / nkg_gru_layer): states (D, N, H), stacked parameters, and the last hidden state as an output
static void seq_impl(bool lstm, bool layer, nkg_var* x, nkg_var* c, nkg_var* h, nkg_var* w_ih, nkg_var* w_hh, nkg_var* b_ih,
                     nkg_var* b_hh, nkg_var** output, nkg_var** last_h, nkg_var** last_c) {
  const char* who = layer ? (lstm ? "lstm_layer" : "gru_layer") : (lstm ? "lstm" : "gru");
  RnnDims dm;
  const std::vector<nkg_var*> operands = check_rnn_operands(
      who, lstm, true, x, c, h, w_ih, w_hh, b_ih, b_hh, output && (!layer || last_h) && (!lstm || last_c), dm, layer);
  std::shared_ptr<RnnSeq> seq;
  std::shared_ptr<RnnSeqBackward> seq_bwd;
  nkg_var* vy = record(
      operands, Shape{dm.T, dm.N, dm.D * dm.H}, x->data->dtype,
      [&](const TensorP& d) {
        seq = std::make_shared<RnnSeq>(
            x->ctx, lstm, layer, dm,
            CellOperands{x->data, h->data, lstm ? c->data : nullptr, w_ih->data, w_hh->data, b_ih->data, b_hh->data}, d);
        return seq;
      },
      [&](const TensorP&, const GradientP& g) {
        seq_bwd = std::make_shared<RnnSeqBackward>(
            x->ctx, g, seq,
            CellGrads{x->grad, h->grad, lstm ? c->grad : nullptr, w_ih->grad, w_hh->grad, b_ih->grad, b_hh->grad});
        return seq_bwd;
      });
  if (lstm) {   // the second output: same tapes, same op id (merging the two histories keeps one node)
    nkg_var* vc = new nkg_var(*vy);
    vc->data = seq->c_last;
    if (seq_bwd) vc->grad = seq_bwd->c_last_grad;
    *last_c = vc;
  }
  if (layer) {
    nkg_var* vh = new nkg_var(*vy);
    vh->data = seq->h_n;
    if (seq_bwd) vh->grad = seq_bwd->h_n_grad;
    *last_h = vh;
  }
  *output = vy;
}

int nkg_lstm(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
             nkg_var* bias_hh, nkg_var** output, nkg_var** last_cell_state) {
  return guard([&] {
    seq_impl(true, false, input, cell_state, hidden, weight_ih, weight_hh, bias_ih, bias_hh, output, nullptr,
             last_cell_state);
  });
}

int nkg_gru(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih, nkg_var* bias_hh,
            nkg_var** output) {
  return guard([&] {
    seq_impl(false, false, input, nullptr, hidden, weight_ih, weight_hh, bias_ih, bias_hh, output, nullptr, nullptr);
  });
}

int nkg_lstm_layer(nkg_var* input, nkg_var* cell_state, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh,
                   nkg_var* bias_ih, nkg_var* bias_hh, nkg_var** output, nkg_var** last_hidden, nkg_var** last_cell_state) {
  return guard([&] {
    seq_impl(true, true, input, cell_state, hidden, weight_ih, weight_hh, bias_ih, bias_hh, output, last_hidden,
             last_cell_state);
  });
}

int nkg_gru_layer(nkg_var* input, nkg_var* hidden, nkg_var* weight_ih, nkg_var* weight_hh, nkg_var* bias_ih,
                  nkg_var* bias_hh, nkg_var** output, nkg_var** last_hidden) {
  return guard([&] {
    seq_impl(false, true, input, nullptr, hidden, weight_ih, weight_hh, bias_ih, bias_hh, output, last_hidden, nullptr);
  });
}

// ---------------------------------------------------------------- optimizers over many leaves (neuronika-optim)
// Every parameter is checked to be differentiable before anything launches, so that an error launches nothing; then, in
// parameter order, each gradient is materialised (Gradient::get) and marked nonzero after the update, since the kernels
// write the penalised gradient back.  The tensors are grouped by (data dtype, gradient dtype) in the order each pair
// first appears, and each group is updated NK_OPTIM_TENSORS_PER_LAUNCH tensors per call.
extern "C++" {
namespace {
struct MultiGroup {
  int w_dtype, g_dtype;
  std::vector<int> idx;
};

// the context of `count` differentiable parameters on one device (nullptr for none); fails before anything else runs
nk_ctx* params_ctx(const char* who, nkg_var* const* params, int count) {
  if (count < 0 || (count > 0 && !params)) fail(NK_ERR_INVALID_ARG, "%s: bad parameter array", who);
  for (int i = 0; i < count; ++i)
    if (!params[i] || !params[i]->diff())
      fail(NK_ERR_INVALID_ARG, "%s: parameter %d is not differentiable", who, i);
  if (count == 0) return nullptr;
  nk_ctx* ctx = params[0]->ctx;
  for (int i = 1; i < count; ++i)
    if (params[i]->ctx != ctx) fail(NK_ERR_INVALID_ARG, "%s: parameters on different devices", who);
  return ctx;
}

template <typename Launch>
void multi_step(const char* who, nkg_var* const* params, int count, void* const* const* states, int nstates,
                void* const* master, Launch launch) {
  nk_ctx* ctx = params_ctx(who, params, count);
  if (count == 0) return;
  std::vector<void*> w(count), g(count);
  std::vector<int64_t> n(count);
  std::vector<Gradient*> roots(count);
  std::vector<MultiGroup> groups;
  for (int i = 0; i < count; ++i) {
    nkg_var* p = params[i];
    roots[i] = p->grad->root();
    w[i] = p->data->rptr();
    g[i] = p->grad->get();
    n[i] = p->data->n();
    const int wd = p->data->dtype, gd = roots[i]->dtype;
    auto it = std::find_if(groups.begin(), groups.end(), [&](const MultiGroup& m) { return m.w_dtype == wd && m.g_dtype == gd; });
    if (it == groups.end()) it = groups.insert(groups.end(), MultiGroup{wd, gd, {}});
    it->idx.push_back(i);
  }
  std::vector<void*> cw, cg, cm, cs[3];
  std::vector<int64_t> cn;
  for (const MultiGroup& m : groups)
    for (size_t first = 0; first < m.idx.size(); first += NK_OPTIM_TENSORS_PER_LAUNCH) {
      const size_t last = std::min(m.idx.size(), first + NK_OPTIM_TENSORS_PER_LAUNCH);
      cw.clear(), cg.clear(), cm.clear(), cn.clear();
      for (int k = 0; k < nstates; ++k) cs[k].clear();
      for (size_t j = first; j < last; ++j) {
        const int i = m.idx[j];
        cw.push_back(w[i]);
        cg.push_back(g[i]);
        cn.push_back(n[i]);
        cm.push_back(master ? master[i] : nullptr);
        for (int k = 0; k < nstates; ++k) cs[k].push_back(states[k] ? states[k][i] : nullptr);
      }
      void* const* st[3];
      for (int k = 0; k < nstates; ++k) st[k] = states[k] ? cs[k].data() : nullptr;
      ck(ctx, launch(ctx, int(cw.size()), cw.data(), cg.data(), m.w_dtype, m.g_dtype, st, master ? cm.data() : nullptr,
                     cn.data()));
    }
  for (Gradient* r : roots) r->is_zero = false;
}

// Gradient clipping: the parameters are checked as multi_step checks them, then each gradient is materialised in
// parameter order and `launch` makes one ABI call with the tables in parameter order.  The writing calls mark the
// gradients nonzero afterwards.
template <typename Launch>
void grad_call(const char* who, nkg_var* const* params, int count, bool writes, Launch launch) {
  nk_ctx* ctx = params_ctx(who, params, count);
  if (count == 0) return;
  std::vector<void*> g(count);
  std::vector<int> dt(count);
  std::vector<int64_t> n(count);
  std::vector<Gradient*> roots(count);
  for (int i = 0; i < count; ++i) {
    roots[i] = params[i]->grad->root();
    g[i] = params[i]->grad->get();
    dt[i] = roots[i]->dtype;
    n[i] = roots[i]->n();
  }
  ck(ctx, launch(ctx, g.data(), dt.data(), n.data()));
  if (writes)
    for (Gradient* r : roots) r->is_zero = false;
}
}  // namespace
}  // extern "C++"

int nkg_multi_sgd_step(nkg_var* const* params, int count, void* const* momentum_buf, void* const* master,
                       nk_optim_hyper* hyper, float l2, float momentum, float dampening, int nesterov, float grad_scale) {
  return guard([&] {
    void* const* states[1] = {momentum_buf};
    multi_step("multi_sgd", params, count, states, 1, master,
               [&](nk_ctx* ctx, int c, void* const* w, void* const* g, int wd, int gd, void* const* const* st,
                   void* const* m, const int64_t* n) {
                 return nk_multi_sgd_step(ctx, c, w, g, wd, gd, st[0], m, n, hyper, l2, momentum, dampening, nesterov,
                                          grad_scale, 1);
               });
  });
}

int nkg_multi_adam_step(nkg_var* const* params, int count, void* const* exp_avg, void* const* exp_avg_sq,
                        void* const* max_exp_avg_sq, void* const* master, nk_optim_hyper* hyper, float beta1,
                        float beta2, float eps, float l1, float l2, float grad_scale) {
  return guard([&] {
    bool first = true;
    void* const* states[3] = {exp_avg, exp_avg_sq, max_exp_avg_sq};
    multi_step("multi_adam", params, count, states, 3, master,
               [&](nk_ctx* ctx, int c, void* const* w, void* const* g, int wd, int gd, void* const* const* st,
                   void* const* m, const int64_t* n) {
                 if (first) {   // once per optimizer step, after every check, before the first update
                   first = false;
                   if (int rc = nk_optim_prologue(ctx, hyper, NK_OPTIM_ADAM, beta1, beta2, 0.f)) return rc;
                 }
                 return nk_multi_adam_step(ctx, c, w, g, wd, gd, st[0], st[1], st[2], m, n, hyper, beta1, beta2, eps,
                                           l1, l2, grad_scale, 1);
               });
  });
}

int nkg_multi_rmsprop_step(nkg_var* const* params, int count, void* const* square_avg, void* const* grad_avg,
                           void* const* momentum_buf, void* const* master, nk_optim_hyper* hyper, float alpha, float eps,
                           float momentum, float l1, float l2, float grad_scale) {
  return guard([&] {
    void* const* states[3] = {square_avg, grad_avg, momentum_buf};
    multi_step("multi_rmsprop", params, count, states, 3, master,
               [&](nk_ctx* ctx, int c, void* const* w, void* const* g, int wd, int gd, void* const* const* st,
                   void* const* m, const int64_t* n) {
                 return nk_multi_rmsprop_step(ctx, c, w, g, wd, gd, st[0], st[1], st[2], m, n, hyper, alpha, eps,
                                              momentum, l1, l2, grad_scale, 1);
               });
  });
}

int nkg_multi_adagrad_step(nkg_var* const* params, int count, void* const* grad_sq, void* const* master,
                           nk_optim_hyper* hyper, float lr_decay, float eps, float l1, float l2, float grad_scale) {
  return guard([&] {
    bool first = true;
    void* const* states[1] = {grad_sq};
    multi_step("multi_adagrad", params, count, states, 1, master,
               [&](nk_ctx* ctx, int c, void* const* w, void* const* g, int wd, int gd, void* const* const* st,
                   void* const* m, const int64_t* n) {
                 if (first) {
                   first = false;
                   if (int rc = nk_optim_prologue(ctx, hyper, NK_OPTIM_ADAGRAD, 0.f, 0.f, lr_decay)) return rc;
                 }
                 return nk_multi_adagrad_step(ctx, c, w, g, wd, gd, st[0], m, n, hyper, eps, l1, l2, grad_scale, 1);
               });
  });
}

int nkg_grad_norm(nkg_var* const* params, int count, float norm_type, float grad_scale, float* total) {
  return guard([&] {
    if (count == 0) fail(NK_ERR_INVALID_ARG, "grad_norm: no parameters, so no device for the total");
    if (!(norm_type > 0.f)) fail(NK_ERR_INVALID_ARG, "grad_norm: norm_type must be > 0 or +inf (got %g)", norm_type);
    grad_call("grad_norm", params, count, false, [&](nk_ctx* ctx, void* const* g, const int* dt, const int64_t* n) {
      return nk_grad_norm(ctx, count, g, dt, n, norm_type, grad_scale, total);
    });
  });
}

int nkg_clip_grads_with_norm(nkg_var* const* params, int count, float max_norm, const float* total) {
  return guard([&] {
    grad_call("clip_grads_with_norm", params, count, true,
              [&](nk_ctx* ctx, void* const* g, const int* dt, const int64_t* n) {
                return nk_grad_scale_by_norm(ctx, count, g, dt, n, total, max_norm);
              });
  });
}

int nkg_clip_grad_value(nkg_var* const* params, int count, float clip_value, float grad_scale) {
  return guard([&] {
    grad_call("clip_grad_value", params, count, true, [&](nk_ctx* ctx, void* const* g, const int* dt, const int64_t* n) {
      return nk_grad_clamp(ctx, count, g, dt, n, clip_value, grad_scale);
    });
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

}  // extern "C"
