// Optimizers: the update of every parameter tensor of one (w dtype, g dtype) pair in one launch per
// NK_OPTIM_TENSORS_PER_LAUNCH tensors, with lr and the step count in device memory (nk_optim_hyper), plus the
// learning-rate scheduler step as a one-thread kernel on the same block.
//
// The reference walks the parameter three to five times per step (one Zip per state array:
// neuronika-optim/src/adam/mod.rs:131-169, amsgrad/mod.rs:159-204, rmsprop/mod.rs:193-300, adagrad/mod.rs:113-140);
// here every element is read and written once.  Per-element arithmetic keeps the reference's operation order (f32), so
// the f32 path matches it to rounding.
//
// The tensor table travels in the kernel parameters (__grid_constant__), as nk_cat.cu's operand table does: the grid
// is the concatenation of every tensor's CTAs, the host computes the CTA prefix and each CTA finds its tensor with a
// binary search.  A CTA covers kChunk consecutive elements of its tensor.  Each thread takes 4 consecutive elements
// (16-byte f32 / 8-byte bf16 accesses) when all of the tensor's pointers are aligned for it, and walks the chunk with
// element accesses otherwise.
// HBM bound: algorithmic bytes per element = w (r+w) + g (r[+w]) + 2 states (r+w) = 24..28 B in f32.
//
// Gradient clipping (torch.nn.utils) shares the table layout: a norm pass that writes one partial per CTA and a
// one-CTA finish, and a scale / clamp pass over the gradients (include/nk_b200.h "gradient clipping").
#include <float.h>
#include <limits.h>

#include <algorithm>

#include "nk_internal.cuh"

// Per-element arithmetic of the five optimizers.  `wv` is the f32 weight (the master copy when there is one), `gv` the
// penalised gradient.
//
// SGD penalty (sgd/mod.rs:191-231, penalty.rs:63-67): g' = grad_scale*g + 2*l2*w.  The SGD update spells out its
// fused multiply-adds, so that its rounding does not depend on how nvcc contracts `a*b + c*d` where it is inlined.
__device__ __forceinline__ float nk_sgd_grad(float g, float wv, float grad_scale, float l2x2) {
  return __fmaf_rn(l2x2, wv, __fmul_rn(g, grad_scale));  // grad += penalty.penalize(w) = 2*lambda*w
}

__device__ __forceinline__ float nk_sgd_update(float wv, float gv, float& buf, float lr, float mu, float one_minus_damp,
                                               int use_momentum, int nesterov) {
  if (!use_momentum) return __fmaf_rn(-gv, lr, wv);
  const float b = __fmaf_rn(gv, one_minus_damp, __fmul_rn(buf, mu));
  buf = b;
  return __fmaf_rn(-(nesterov ? __fmaf_rn(b, mu, gv) : b), lr, wv);
}

// Adam-family penalties (penalty.rs:63-79): g' = grad_scale*g + l1*signum(w) + 2*l2*w
struct NkOptPenalty {
  float l1, l2x2, grad_scale;
  int write_back_grad;
};

__device__ __forceinline__ float nk_signum_f32(float w) {  // f32::signum: 1.0 for +0.0, -1.0 for -0.0, NaN for NaN
  return w != w ? w : copysignf(1.f, w);
}

__device__ __forceinline__ float nk_opt_grad(const NkOptPenalty& c, float g, float wv) {
  float gv = g * c.grad_scale;
  if (c.l1 != 0.f) gv += c.l1 * nk_signum_f32(wv);
  gv += c.l2x2 * wv;
  return gv;
}

// adam/mod.rs:150-166, amsgrad/mod.rs:177-200; `max_sq` is read and written only when `ams`
__device__ __forceinline__ float nk_adam_update(float wv, float gv, float& exp_avg, float& exp_avg_sq, bool ams,
                                                float& max_sq, float beta1, float beta2, float sqrt_bc2,
                                                float step_size, float eps) {
  const float m = exp_avg * beta1 + gv * (1.f - beta1);
  const float v = exp_avg_sq * beta2 + gv * gv * (1.f - beta2);
  exp_avg = m;
  exp_avg_sq = v;
  float vv = v;
  if (ams) {  // AMSGrad: running maximum of the second moment
    vv = fmaxf(max_sq, v);
    max_sq = vv;
  }
  wv -= m / ((sqrtf(vv) / sqrt_bc2) + eps) * step_size;
  return wv;
}

// rmsprop/mod.rs:193-300: the four (centered, momentum) variants
__device__ __forceinline__ float nk_rmsprop_update(float wv, float gv, float& square_avg, bool centered,
                                                   float& grad_avg, bool momentum_on, float& buf, float lr,
                                                   float alpha, float eps, float momentum) {
  const float sq = square_avg * alpha + gv * gv * (1.f - alpha);
  square_avg = sq;
  float denom;
  if (centered) {
    const float ga = grad_avg * alpha + gv * (1.f - alpha);
    grad_avg = ga;
    denom = sqrtf(sq + (-ga * ga)) + eps;
  } else {
    denom = sqrtf(sq) + eps;
  }
  if (momentum_on) {
    const float b = buf * momentum + gv / denom;
    buf = b;
    wv -= b * lr;
  } else {
    wv -= gv / denom * lr;
  }
  return wv;
}

// adagrad/mod.rs:113-140
__device__ __forceinline__ float nk_adagrad_update(float wv, float gv, float& grad_sq, float clr, float eps) {
  const float s = grad_sq + gv * gv;
  grad_sq = s;
  wv -= gv / (sqrtf(s) + eps) * clr;
  return wv;
}

// a named namespace: kernel symbol names stay the same from build to build (torch.profiler traces)
namespace nk_optim_multi {

constexpr int kThreads = 256;
constexpr int kTensors = NK_OPTIM_TENSORS_PER_LAUNCH;
constexpr int kChunk = kThreads * 4;  // elements per CTA

enum Kind { SGD = 0, ADAM = 1, RMSPROP = 2, ADAGRAD = 3 };

struct Tensor {
  void* w;
  void* g;
  float* s[3];     // optimizer state, by kind: SGD {buf}, Adam {exp_avg, exp_avg_sq, max_sq}, RMSProp {square_avg,
                   // grad_avg, buf}, Adagrad {grad_sq}
  float* master;
  int64_t n;
};
struct Table {
  Tensor t[kTensors];
  int32_t blk[kTensors + 1];  // CTA prefix
  uint64_t vec;               // bit i: tensor i takes the 4-element path
  int count;
};
// every hyperparameter that is not in the device block; uniform over the launch
struct Args {
  float beta1, beta2, eps;                       // Adam (eps: also RMSProp, Adagrad)
  float alpha, momentum;                         // RMSProp (momentum: also SGD)
  float one_minus_damp, sgd_l2x2;                // SGD
  NkOptPenalty pen;                              // Adam family; pen.grad_scale and write_back_grad serve SGD too
  int has[3];                                    // which of the state slots are in use
  int nesterov;
};
static_assert(sizeof(Table) + sizeof(Args) + sizeof(void*) <= 4096, "tensor table exceeds the kernel parameter limit");

static inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

__device__ __forceinline__ int find_tensor(const int32_t* blk, int count, int b) {
  int lo = 0, hi = count - 1;  // the largest i with blk[i] <= b (empty tensors own no CTA)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (blk[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// the scalars a launch reads from the device block
struct Derived {
  float lr, step_size, sqrt_bc2, clr;
};

// one element: wv (f32 weight or master) and the raw gradient in, the new weight out; st[] is the element's state
template <int K>
__device__ __forceinline__ float update(const Args& a, const Derived& d, float wv, float& graw, float (&st)[3]) {
  if (K == SGD) {
    const float gv = nk_sgd_grad(graw, wv, a.pen.grad_scale, a.sgd_l2x2);
    graw = gv;
    return nk_sgd_update(wv, gv, st[0], d.lr, a.momentum, a.one_minus_damp, a.has[0], a.nesterov);
  }
  const float gv = nk_opt_grad(a.pen, graw, wv);
  graw = gv;
  if (K == ADAM)
    return nk_adam_update(wv, gv, st[0], st[1], a.has[2], st[2], a.beta1, a.beta2, d.sqrt_bc2, d.step_size, a.eps);
  if (K == RMSPROP)
    return nk_rmsprop_update(wv, gv, st[0], a.has[1], st[1], a.has[2], st[2], d.lr, a.alpha, a.eps, a.momentum);
  return nk_adagrad_update(wv, gv, st[0], d.clr, a.eps);
}

template <typename T>
struct alignas(sizeof(T) * 4) Quad {
  T v[4];
};

template <int K, typename TW, typename TG>
__global__ void __launch_bounds__(kThreads) nk_optim_multi_kernel(const __grid_constant__ Table tab,
                                                                  const __grid_constant__ Args a,
                                                                  const nk_optim_hyper* __restrict__ hyper) {
  const int b = blockIdx.x;
  const int i = find_tensor(tab.blk, tab.count, b);
  const Tensor& t = tab.t[i];
  const Derived d{hyper->lr, hyper->step_size, hyper->sqrt_bc2, hyper->clr};
  TW* __restrict__ w = static_cast<TW*>(t.w);
  TG* __restrict__ g = static_cast<TG*>(t.g);
  float* __restrict__ master = t.master;
  const int wb = a.pen.write_back_grad;
  const int64_t base = int64_t(b - tab.blk[i]) * kChunk;
  if ((tab.vec >> i) & 1) {
    const int64_t e0 = base + int64_t(threadIdx.x) * 4;
    if (e0 + 4 <= t.n) {
      const int64_t q = e0 / 4;
      Quad<TW> wq = reinterpret_cast<const Quad<TW>*>(w)[q];
      Quad<TG> gq = reinterpret_cast<const Quad<TG>*>(g)[q];
      Quad<float> mq, sq[3];
      if (master) mq = reinterpret_cast<const Quad<float>*>(master)[q];
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (a.has[k]) sq[k] = reinterpret_cast<const Quad<float>*>(t.s[k])[q];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float st[3] = {sq[0].v[e], sq[1].v[e], sq[2].v[e]};
        float gv = nk_to_f32<TG>(gq.v[e]);
        const float wv = update<K>(a, d, master ? mq.v[e] : nk_to_f32<TW>(wq.v[e]), gv, st);
        gq.v[e] = nk_from_f32<TG>(gv);
#pragma unroll
        for (int k = 0; k < 3; ++k) sq[k].v[e] = st[k];
        mq.v[e] = wv;
        wq.v[e] = nk_from_f32<TW>(wv);
      }
      if (wb) reinterpret_cast<Quad<TG>*>(g)[q] = gq;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (a.has[k]) reinterpret_cast<Quad<float>*>(t.s[k])[q] = sq[k];
      if (master) reinterpret_cast<Quad<float>*>(master)[q] = mq;
      reinterpret_cast<Quad<TW>*>(w)[q] = wq;
      return;
    }
    // the last (n % 4) elements of the tensor: element accesses by the thread that owns them
    for (int64_t e = e0; e < t.n; ++e) {
      float st[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) st[k] = a.has[k] ? t.s[k][e] : 0.f;
      float gv = nk_to_f32<TG>(g[e]);
      const float wv = update<K>(a, d, master ? master[e] : nk_to_f32<TW>(w[e]), gv, st);
      if (wb) g[e] = nk_from_f32<TG>(gv);
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (a.has[k]) t.s[k][e] = st[k];
      if (master) master[e] = wv;
      w[e] = nk_from_f32<TW>(wv);
    }
    return;
  }
#pragma unroll 4
  for (int j = 0; j < kChunk / kThreads; ++j) {
    const int64_t e = base + int64_t(j) * kThreads + threadIdx.x;
    if (e >= t.n) break;
    float st[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) st[k] = a.has[k] ? t.s[k][e] : 0.f;
    float gv = nk_to_f32<TG>(g[e]);
    const float wv = update<K>(a, d, master ? master[e] : nk_to_f32<TW>(w[e]), gv, st);
    if (wb) g[e] = nk_from_f32<TG>(gv);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (a.has[k]) t.s[k][e] = st[k];
    if (master) master[e] = wv;
    w[e] = nk_from_f32<TW>(wv);
  }
}

// step += 1 and the per-step scalars, each operation rounded on its own in f32
__global__ void nk_optim_prologue_kernel(nk_optim_hyper* h, int kind, float beta1, float beta2, float lr_decay) {
  const int64_t step = h->step + 1;
  h->step = step;
  if (kind == NK_OPTIM_ADAM) {
    float p1 = 1.f, p2 = 1.f, b1 = beta1, b2 = beta2;
    for (uint64_t e = uint64_t(step); e; e >>= 1) {
      if (e & 1) p1 = __fmul_rn(p1, b1), p2 = __fmul_rn(p2, b2);
      b1 = __fmul_rn(b1, b1), b2 = __fmul_rn(b2, b2);
    }
    const float bc1 = __fsub_rn(1.f, p1), bc2 = __fsub_rn(1.f, p2);
    h->sqrt_bc2 = __fsqrt_rn(bc2);
    h->step_size = __fdiv_rn(h->lr, bc1);
  } else {
    h->clr = __fdiv_rn(h->lr, __fadd_rn(1.f, __fmul_rn(__ll2float_rn(step - 1), lr_decay)));
  }
}

__global__ void nk_lr_sched_kernel(nk_lr_sched* s, nk_optim_hyper* h) {
  const int64_t t = s->epoch + 1;
  const float lr = h->lr;
  float next = lr;
  switch (s->kind) {
    case NK_LR_STEP:
      if (t % s->step_size == 0) next = __fmul_rn(lr, s->gamma);
      break;
    case NK_LR_MULTI_STEP: {
      const int64_t* m = static_cast<const int64_t*>(s->table);
      for (int64_t k = 0; k < s->table_len; ++k)
        if (m[k] == t) {
          next = __fmul_rn(lr, s->gamma);
          break;
        }
      break;
    }
    case NK_LR_EXPONENTIAL:
      next = __fmul_rn(lr, s->gamma);
      break;
    default: {  // the closure-based schedulers: f(t) from the table
      if (t > s->table_len) {
        s->past_horizon = 1;
        return;
      }
      const float f = static_cast<const float*>(s->table)[t - 1];
      next = __fmul_rn(s->kind == NK_LR_LAMBDA ? s->initial_lr : lr, f);
    }
  }
  s->epoch = t;
  s->last_lr = lr;
  s->current_lr = next;
  h->lr = next;
}

// ------------------------------------------------------------------------------------------------- host side
static int copy_block(nk_ctx* ctx, const char* who, void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (ctx->capturing)
    return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "%s: a host copy of the block cannot be captured (a replay would not "
                        "repeat it)", who);
  NK_REQUIRE(ctx, dst && src, "%s: NULL pointer", who);
  NK_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, kind, ctx->stream));
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NK_OK;
}

static inline void* entry(void* const* a, int i) { return a ? a[i] : nullptr; }

// builds the table of one launch (checks everything first: an error launches nothing) and launches it
template <int K>
static int multi_step(nk_ctx* ctx, const char* who, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                      void* const* st[3], void* const* master, const int64_t* n, const nk_optim_hyper* hyper,
                      const Args& args) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(w_dtype) && nk_dtype_ok(g_dtype), "%s: bad dtype", who);
  NK_REQUIRE(ctx, count >= 0 && count <= kTensors, "%s: %d tensors (1..%d per launch)", who, count, kTensors);
  if (count == 0) return NK_OK;
  NK_REQUIRE(ctx, w && g && n && hyper, "%s: NULL pointer", who);
  Table tab = {};
  tab.count = count;
  int64_t blocks = 0;
  const size_t ws = nk_dtype_size(w_dtype), gs = nk_dtype_size(g_dtype);
  for (int i = 0; i < count; ++i) {
    Tensor& t = tab.t[i];
    NK_REQUIRE(ctx, n[i] >= 0, "%s: tensor %d has %lld elements", who, i, (long long)n[i]);
    t.w = w[i];
    t.g = g[i];
    t.n = n[i];
    t.master = static_cast<float*>(entry(master, i));
    bool vec = aligned(t.w, 4 * ws) && aligned(t.g, 4 * gs) && aligned(t.master, 16);
    for (int k = 0; k < 3; ++k) {
      t.s[k] = args.has[k] ? static_cast<float*>(entry(st[k], i)) : nullptr;
      vec = vec && aligned(t.s[k], 16);
    }
    tab.blk[i] = int32_t(blocks);
    if (t.n == 0) continue;
    NK_REQUIRE(ctx, t.w && t.g, "%s: tensor %d: NULL weight or gradient", who, i);
    for (int k = 0; k < 3; ++k)
      NK_REQUIRE(ctx, !args.has[k] || t.s[k], "%s: tensor %d: NULL state %d", who, i, k);
    if (vec) tab.vec |= uint64_t(1) << i;
    blocks += (t.n + kChunk - 1) / kChunk;
    NK_REQUIRE(ctx, blocks <= INT_MAX, "%s: %lld CTAs exceed the grid limit", who, (long long)blocks);
  }
  tab.blk[count] = int32_t(blocks);
  if (blocks == 0) return NK_OK;
  const int grid = int(blocks);
  if (w_dtype == NK_F32 && g_dtype == NK_F32)
    nk_optim_multi_kernel<K, float, float><<<grid, kThreads, 0, ctx->stream>>>(tab, args, hyper);
  else if (w_dtype == NK_BF16 && g_dtype == NK_BF16)
    nk_optim_multi_kernel<K, __nv_bfloat16, __nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(tab, args, hyper);
  else if (w_dtype == NK_BF16)
    nk_optim_multi_kernel<K, __nv_bfloat16, float><<<grid, kThreads, 0, ctx->stream>>>(tab, args, hyper);
  else
    nk_optim_multi_kernel<K, float, __nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(tab, args, hyper);
  NK_LAUNCHED(ctx, who);
  return NK_OK;
}

// ------------------------------------------------------------------------------------------- gradient clipping
// torch.nn.utils' get_total_norm, clip_grads_with_norm_ and clip_grad_value_ over tables of gradients of one dtype,
// laid out like the optimizer launches: the grid is the concatenation of every tensor's CTAs.
enum NormKind { NORM_2 = 0, NORM_1 = 1, NORM_INF = 2, NORM_P = 3 };
// 4-element vectors per thread in a CTA of the norm pass.  Captured get_total_norm (memset of the total, norm pass,
// finish) in us over f32 gradients, H100 80GB HBM3 at 700 W, two runs each: the language model (16.4 M elements, 7
// tensors) / config 4's MLP (21 M, 6 tensors) / 256 x 4096:
//   2 vectors (2048 elements per CTA) 29.5 / 34.1 / 12.0;  4: 29.0-29.5 / 33.5 / 12.1;  8: 28.5 / 34.3 / 14.9;
//   16: 31.6 / 35.1 / 14.9.
constexpr int kNormVecs = 4;
constexpr int kNormChunk = kThreads * 4 * kNormVecs;

struct GradTensor {
  void* g;
  int64_t n;
};
struct GradTable {
  GradTensor t[kTensors];
  int32_t blk[kTensors + 1];  // CTA prefix
  uint64_t vec;               // bit i: tensor i takes the 4-element path
  int count;
  int part;                   // norm: the workspace slot of this launch's first CTA partial
};
static_assert(sizeof(GradTable) + 3 * sizeof(void*) <= 4096, "gradient table exceeds the kernel parameter limit");

// the larger of a and b, NaN when either is (fmaxf returns the other operand)
template <typename T>
__device__ __forceinline__ T nan_max(T a, T b) {
  return (a != a || a >= b) ? a : b;
}

template <int P, typename T>
__device__ __forceinline__ T norm_merge(T a, T b) {
  return P == NORM_INF ? nan_max(a, b) : a + b;
}

// one element's share of the norm, v = f32(k * g)
template <int P>
__device__ __forceinline__ float norm_term(float g, float k, float p) {
  const float v = __fmul_rn(g, k);
  if (P == NORM_2) return v * v;
  if (P == NORM_P) return powf(fabsf(v), p);
  return fabsf(v);
}

// one f32 partial per CTA: each thread folds its elements in index order, then a fixed butterfly per warp and warp 0's
// partials in warp order
template <int P, typename TG>
__global__ void __launch_bounds__(kThreads) nk_grad_norm_kernel(const __grid_constant__ GradTable tab, float p, float k,
                                                                float* __restrict__ part) {
  const int b = blockIdx.x;
  const int i = find_tensor(tab.blk, tab.count, b);
  const GradTensor& t = tab.t[i];
  const TG* __restrict__ g = static_cast<const TG*>(t.g);
  const int64_t base = int64_t(b - tab.blk[i]) * kNormChunk;
  float s = 0.f;
  if ((tab.vec >> i) & 1) {
    if (base + kNormChunk <= t.n) {  // a whole chunk: every load in flight before the first use
      Quad<TG> q[kNormVecs];
#pragma unroll
      for (int j = 0; j < kNormVecs; ++j)
        q[j] = reinterpret_cast<const Quad<TG>*>(g)[(base >> 2) + j * kThreads + threadIdx.x];
#pragma unroll
      for (int j = 0; j < kNormVecs; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) s = norm_merge<P>(s, norm_term<P>(nk_to_f32<TG>(q[j].v[e]), k, p));
    } else {
      for (int j = 0; j < kNormVecs; ++j) {
        const int64_t e0 = base + (int64_t(j) * kThreads + threadIdx.x) * 4;
        if (e0 >= t.n) break;
        if (e0 + 4 <= t.n) {
          const Quad<TG> q = reinterpret_cast<const Quad<TG>*>(g)[e0 >> 2];
#pragma unroll
          for (int e = 0; e < 4; ++e) s = norm_merge<P>(s, norm_term<P>(nk_to_f32<TG>(q.v[e]), k, p));
        } else {  // the last (n % 4) elements of the tensor
          for (int64_t e = e0; e < t.n; ++e) s = norm_merge<P>(s, norm_term<P>(nk_to_f32<TG>(g[e]), k, p));
        }
      }
    }
  } else {
#pragma unroll 4
    for (int j = 0; j < kNormChunk / kThreads; ++j) {
      const int64_t e = base + int64_t(j) * kThreads + threadIdx.x;
      if (e >= t.n) break;
      s = norm_merge<P>(s, norm_term<P>(nk_to_f32<TG>(g[e]), k, p));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = norm_merge<P>(s, __shfl_xor_sync(0xffffffffu, s, o));
  __shared__ float warp_part[kThreads / 32];
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = warp_part[0];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) r = norm_merge<P>(r, warp_part[w]);
    part[tab.part + b] = r;
  }
}

// one CTA: every partial merged in a fixed order in double, the root taken in double, rounded once to f32
__global__ void __launch_bounds__(kThreads) nk_grad_norm_finish_kernel(const float* __restrict__ part, int nparts,
                                                                       int kind, float p, float* __restrict__ total) {
  const bool inf = kind == NORM_INF;
  double s = 0.0;
  for (int j = threadIdx.x; j < nparts; j += kThreads)
    s = inf ? norm_merge<NORM_INF>(s, double(part[j])) : s + double(part[j]);
  __shared__ double sh[kThreads];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      sh[threadIdx.x] = inf ? norm_merge<NORM_INF>(sh[threadIdx.x], sh[threadIdx.x + w])
                            : sh[threadIdx.x] + sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double r = sh[0];
    if (kind == NORM_2) r = sqrt(r);
    if (kind == NORM_P) r = pow(r, 1.0 / double(p));
    *total = float(r);
  }
}

enum PointOp { SCALE = 0, CLAMP = 1 };

// SCALE: g *= c with torch's coefficient from *total and a = max_norm (nothing is written when c == 1);
// CLAMP: g = min(max(g, -a), a) in torch's order (clamp_min, then clamp_max), a NaN element stays NaN
template <int OP, typename TG>
__global__ void __launch_bounds__(kThreads) nk_grad_pointwise_kernel(const __grid_constant__ GradTable tab,
                                                                     const float* __restrict__ total, float a) {
  float c = 1.f;
  if (OP == SCALE) {
    // torch: max_norm / (total + 1e-6) is Tensor.__rdiv__, reciprocal() * max_norm; then clamp(max=1), NaN kept
    c = __fmul_rn(__frcp_rn(__fadd_rn(*total, 1e-6f)), a);
    if (c > 1.f) c = 1.f;
    if (c == 1.f) return;  // x * 1 == x: the unconditional multiply would write the same bits
  }
  const auto op = [&](float v) {
    if (OP == SCALE) return __fmul_rn(v, c);
    if (v < -a) v = -a;
    if (v > a) v = a;
    return v;
  };
  const int b = blockIdx.x;
  const int i = find_tensor(tab.blk, tab.count, b);
  const GradTensor& t = tab.t[i];
  TG* __restrict__ g = static_cast<TG*>(t.g);
  const int64_t base = int64_t(b - tab.blk[i]) * kChunk;
  if ((tab.vec >> i) & 1) {
    const int64_t e0 = base + int64_t(threadIdx.x) * 4;
    if (e0 + 4 <= t.n) {
      Quad<TG> q = reinterpret_cast<const Quad<TG>*>(g)[e0 >> 2];
#pragma unroll
      for (int e = 0; e < 4; ++e) q.v[e] = nk_from_f32<TG>(op(nk_to_f32<TG>(q.v[e])));
      reinterpret_cast<Quad<TG>*>(g)[e0 >> 2] = q;
      return;
    }
    for (int64_t e = e0; e < t.n; ++e) g[e] = nk_from_f32<TG>(op(nk_to_f32<TG>(g[e])));
    return;
  }
#pragma unroll 4
  for (int j = 0; j < kChunk / kThreads; ++j) {
    const int64_t e = base + int64_t(j) * kThreads + threadIdx.x;
    if (e >= t.n) break;
    g[e] = nk_from_f32<TG>(op(nk_to_f32<TG>(g[e])));
  }
}

struct GradLaunch {
  GradTable tab;
  int dtype;
  int blocks;
};

// The launches of one clipping call, `chunk` elements per CTA: the tensors grouped by dtype in order of first
// appearance, kTensors per launch.  Every argument is checked before the caller launches anything; *parts receives the
// CTAs of all launches.
static int grad_launches(nk_ctx* ctx, const char* who, int count, void* const* g, const int* g_dtype, const int64_t* n,
                         int64_t chunk, std::vector<GradLaunch>& out, int64_t* parts) {
  *parts = 0;
  NK_REQUIRE(ctx, count >= 0, "%s: %d tensors", who, count);
  if (count == 0) return NK_OK;
  NK_REQUIRE(ctx, g && g_dtype && n, "%s: NULL pointer", who);
  std::vector<int> order;
  for (int i = 0; i < count; ++i) {
    NK_REQUIRE(ctx, nk_dtype_ok(g_dtype[i]), "%s: tensor %d: bad dtype %d", who, i, g_dtype[i]);
    NK_REQUIRE(ctx, n[i] >= 0, "%s: tensor %d has %lld elements", who, i, (long long)n[i]);
    NK_REQUIRE(ctx, n[i] == 0 || g[i], "%s: tensor %d: NULL gradient", who, i);
    if (std::find(order.begin(), order.end(), g_dtype[i]) == order.end()) order.push_back(g_dtype[i]);
  }
  for (int dt : order)
    for (int i = 0, first = 1; i < count; ++i) {
      if (g_dtype[i] != dt) continue;
      if (first || out.back().tab.count == kTensors) {
        out.push_back(GradLaunch{});
        out.back().dtype = dt;
        out.back().tab.part = int(*parts);
        first = 0;
      }
      GradLaunch& l = out.back();
      const int j = l.tab.count++;
      l.tab.t[j] = GradTensor{g[i], n[i]};
      l.tab.blk[j] = l.blocks;
      if (aligned(g[i], 4 * nk_dtype_size(dt))) l.tab.vec |= uint64_t(1) << j;
      const int64_t blocks = (n[i] + chunk - 1) / chunk;
      NK_REQUIRE(ctx, *parts + blocks <= INT_MAX, "%s: %lld CTAs exceed the grid limit", who,
                 (long long)(*parts + blocks));
      l.blocks += int(blocks);
      l.tab.blk[j + 1] = l.blocks;
      *parts += blocks;
    }
  return NK_OK;
}

template <int P>
static void launch_norm(nk_ctx* ctx, const GradLaunch& l, float p, float k, float* part) {
  if (l.dtype == NK_BF16)
    nk_grad_norm_kernel<P, __nv_bfloat16><<<l.blocks, kThreads, 0, ctx->stream>>>(l.tab, p, k, part);
  else
    nk_grad_norm_kernel<P, float><<<l.blocks, kThreads, 0, ctx->stream>>>(l.tab, p, k, part);
}

template <int OP>
static int pointwise(nk_ctx* ctx, const char* who, int count, void* const* g, const int* g_dtype, const int64_t* n,
                     const float* total, float a) {
  std::vector<GradLaunch> ls;
  int64_t parts;
  if (int rc = grad_launches(ctx, who, count, g, g_dtype, n, kChunk, ls, &parts)) return rc;
  for (const GradLaunch& l : ls) {
    if (!l.blocks) continue;
    if (l.dtype == NK_BF16)
      nk_grad_pointwise_kernel<OP, __nv_bfloat16><<<l.blocks, kThreads, 0, ctx->stream>>>(l.tab, total, a);
    else
      nk_grad_pointwise_kernel<OP, float><<<l.blocks, kThreads, 0, ctx->stream>>>(l.tab, total, a);
    NK_LAUNCHED(ctx, who);
  }
  return NK_OK;
}

}  // namespace nk_optim_multi

using namespace nk_optim_multi;

extern "C" {

int nk_optim_hyper_set(nk_ctx* ctx, nk_optim_hyper* hyper, const nk_optim_hyper* host) {
  return copy_block(ctx, "nk_optim_hyper_set", hyper, host, sizeof(nk_optim_hyper), cudaMemcpyHostToDevice);
}

int nk_optim_hyper_get(nk_ctx* ctx, const nk_optim_hyper* hyper, nk_optim_hyper* host) {
  return copy_block(ctx, "nk_optim_hyper_get", host, hyper, sizeof(nk_optim_hyper), cudaMemcpyDeviceToHost);
}

int nk_optim_prologue(nk_ctx* ctx, nk_optim_hyper* hyper, int kind, float beta1, float beta2, float lr_decay) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, hyper, "nk_optim_prologue: NULL block");
  NK_REQUIRE(ctx, kind == NK_OPTIM_ADAM || kind == NK_OPTIM_ADAGRAD, "nk_optim_prologue: bad kind %d", kind);
  nk_optim_prologue_kernel<<<1, 1, 0, ctx->stream>>>(hyper, kind, beta1, beta2, lr_decay);
  NK_LAUNCHED(ctx, "optim_prologue");
  return NK_OK;
}

int nk_multi_sgd_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                      void* const* momentum_buf, void* const* master, const int64_t* n, const nk_optim_hyper* hyper,
                      float l2, float momentum, float dampening, int nesterov, float grad_scale, int write_back_grad) {
  Args a = {};
  a.momentum = momentum;
  a.one_minus_damp = 1.f - dampening;
  a.sgd_l2x2 = 2.f * l2;
  a.nesterov = nesterov;
  a.has[0] = momentum > FLT_EPSILON;  // `.filter(|val| *val > f32::EPSILON)`, sgd/mod.rs:202
  a.pen.grad_scale = grad_scale;
  a.pen.write_back_grad = (a.sgd_l2x2 == 0.f && grad_scale == 1.f) ? 0 : write_back_grad;  // g' = g: nothing to write
  void* const* st[3] = {momentum_buf, nullptr, nullptr};
  return multi_step<SGD>(ctx, "nk_multi_sgd_step", count, w, g, w_dtype, g_dtype, st, master, n, hyper, a);
}

int nk_multi_adam_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                       void* const* exp_avg, void* const* exp_avg_sq, void* const* max_exp_avg_sq, void* const* master,
                       const int64_t* n, const nk_optim_hyper* hyper, float beta1, float beta2, float eps, float l1,
                       float l2, float grad_scale, int write_back_grad) {
  Args a = {};
  a.beta1 = beta1;
  a.beta2 = beta2;
  a.eps = eps;
  a.pen = NkOptPenalty{l1, 2.f * l2, grad_scale, write_back_grad};
  a.has[0] = a.has[1] = 1;
  a.has[2] = max_exp_avg_sq != nullptr;
  void* const* st[3] = {exp_avg, exp_avg_sq, max_exp_avg_sq};
  return multi_step<ADAM>(ctx, "nk_multi_adam_step", count, w, g, w_dtype, g_dtype, st, master, n, hyper, a);
}

int nk_multi_rmsprop_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                          void* const* square_avg, void* const* grad_avg, void* const* momentum_buf, void* const* master,
                          const int64_t* n, const nk_optim_hyper* hyper, float alpha, float eps, float momentum,
                          float l1, float l2, float grad_scale, int write_back_grad) {
  Args a = {};
  a.alpha = alpha;
  a.eps = eps;
  a.momentum = momentum;
  a.pen = NkOptPenalty{l1, 2.f * l2, grad_scale, write_back_grad};
  a.has[0] = 1;
  a.has[1] = grad_avg != nullptr;
  a.has[2] = momentum_buf != nullptr && momentum > FLT_EPSILON;  // rmsprop/mod.rs:213-216
  void* const* st[3] = {square_avg, grad_avg, momentum_buf};
  return multi_step<RMSPROP>(ctx, "nk_multi_rmsprop_step", count, w, g, w_dtype, g_dtype, st, master, n, hyper, a);
}

int nk_multi_adagrad_step(nk_ctx* ctx, int count, void* const* w, void* const* g, int w_dtype, int g_dtype,
                          void* const* grad_sq, void* const* master, const int64_t* n, const nk_optim_hyper* hyper,
                          float eps, float l1, float l2, float grad_scale, int write_back_grad) {
  Args a = {};
  a.eps = eps;
  a.pen = NkOptPenalty{l1, 2.f * l2, grad_scale, write_back_grad};
  a.has[0] = 1;
  void* const* st[3] = {grad_sq, nullptr, nullptr};
  return multi_step<ADAGRAD>(ctx, "nk_multi_adagrad_step", count, w, g, w_dtype, g_dtype, st, master, n, hyper, a);
}

int nk_lr_sched_set(nk_ctx* ctx, nk_lr_sched* sched, const nk_lr_sched* host) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, host, "nk_lr_sched_set: NULL pointer");
  NK_REQUIRE(ctx, host->kind >= NK_LR_STEP && host->kind <= NK_LR_LAMBDA, "nk_lr_sched_set: bad kind %d", host->kind);
  NK_REQUIRE(ctx, host->epoch >= 0, "nk_lr_sched_set: negative epoch %lld", (long long)host->epoch);
  NK_REQUIRE(ctx, host->kind != NK_LR_STEP || host->step_size >= 1, "nk_lr_sched_set: step_size must be >= 1 (got %lld)",
             (long long)host->step_size);
  NK_REQUIRE(ctx, host->table_len >= 0 && (host->table_len == 0 || host->table),
             "nk_lr_sched_set: table of %lld entries at NULL", (long long)host->table_len);
  return copy_block(ctx, "nk_lr_sched_set", sched, host, sizeof(nk_lr_sched), cudaMemcpyHostToDevice);
}

int nk_lr_sched_get(nk_ctx* ctx, const nk_lr_sched* sched, nk_lr_sched* host) {
  if (int rc = copy_block(ctx, "nk_lr_sched_get", host, sched, sizeof(nk_lr_sched), cudaMemcpyDeviceToHost)) return rc;
  if (host->past_horizon)
    return nk_set_error(ctx, NK_ERR_INVALID_ARG, "lr scheduler stepped past the end of its table of %lld factors "
                        "(epoch %lld): lr was left unchanged", (long long)host->table_len, (long long)host->epoch);
  return NK_OK;
}

int nk_lr_sched_step(nk_ctx* ctx, nk_lr_sched* sched, nk_optim_hyper* hyper) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, sched && hyper, "nk_lr_sched_step: NULL pointer");
  nk_lr_sched_kernel<<<1, 1, 0, ctx->stream>>>(sched, hyper);
  NK_LAUNCHED(ctx, "lr_sched");
  return NK_OK;
}

int nk_grad_norm(nk_ctx* ctx, int count, const void* const* g, const int* g_dtype, const int64_t* n, float norm_type,
                 float grad_scale, float* total) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, norm_type > 0.f, "nk_grad_norm: norm_type must be > 0 or +inf (got %g)", double(norm_type));
  NK_REQUIRE(ctx, total, "nk_grad_norm: NULL total");
  const int kind = norm_type == 2.f ? NORM_2 : norm_type == 1.f ? NORM_1 : isinf(norm_type) ? NORM_INF : NORM_P;
  std::vector<GradLaunch> ls;
  int64_t parts;
  if (int rc = grad_launches(ctx, "nk_grad_norm", count, const_cast<void* const*>(g), g_dtype, n, kNormChunk, ls, &parts))
    return rc;
  void* ws = nullptr;
  if (int rc = nk_alloc_uninit(ctx, size_t(std::max<int64_t>(parts, 1)) * sizeof(float), &ws)) return rc;
  float* part = static_cast<float*>(ws);
  const int rc = [&]() -> int {
    for (const GradLaunch& l : ls) {
      if (!l.blocks) continue;
      switch (kind) {
        case NORM_2: launch_norm<NORM_2>(ctx, l, norm_type, grad_scale, part); break;
        case NORM_1: launch_norm<NORM_1>(ctx, l, norm_type, grad_scale, part); break;
        case NORM_INF: launch_norm<NORM_INF>(ctx, l, norm_type, grad_scale, part); break;
        default: launch_norm<NORM_P>(ctx, l, norm_type, grad_scale, part);
      }
      NK_LAUNCHED(ctx, "grad_norm");
    }
    nk_grad_norm_finish_kernel<<<1, kThreads, 0, ctx->stream>>>(part, int(parts), kind, norm_type, total);
    NK_LAUNCHED(ctx, "grad_norm_finish");
    return NK_OK;
  }();
  const int frc = nk_free(ctx, ws);
  return rc ? rc : frc;
}

int nk_grad_scale_by_norm(nk_ctx* ctx, int count, void* const* g, const int* g_dtype, const int64_t* n,
                          const float* total, float max_norm) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, total, "nk_grad_scale_by_norm: NULL total");
  return pointwise<SCALE>(ctx, "nk_grad_scale_by_norm", count, g, g_dtype, n, total, max_norm);
}

int nk_grad_clamp(nk_ctx* ctx, int count, void* const* g, const int* g_dtype, const int64_t* n, float clip_value,
                  float grad_scale) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  return pointwise<CLAMP>(ctx, "nk_grad_clamp", count, g, g_dtype, n, nullptr, clip_value / grad_scale);
}

}  // extern "C"
