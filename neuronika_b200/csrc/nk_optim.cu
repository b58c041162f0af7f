// Adam-family parameter updates as single fused passes (SURVEY.md 8-f rank 2): the reference walks the parameter
// three to five times per step (one Zip per state array: neuronika-optim/src/adam/mod.rs:131-169,
// amsgrad/mod.rs:159-204, rmsprop/mod.rs:193-300, adagrad/mod.rs:113-140); here every element is read and written
// once.  Per-element arithmetic keeps the reference's operation order (f32), so the f32 path matches it to rounding.
// Penalties (penalty.rs:63-79): g += l1*signum(w) + 2*l2*w  (L1, L2, ElasticNet; signum(+-0) = +-1 like f32::signum).
// HBM bound: algorithmic bytes per element = w (r+w) + g (r[+w]) + 2 states (r+w) = 24..28 B in f32.
#include <float.h>

#include "nk_internal.cuh"
#include "nk_optim_math.cuh"

namespace {

constexpr int kThreads = 256;

inline int opt_blocks(nk_ctx* ctx, size_t n) {
  size_t b = (n + kThreads - 1) / kThreads;
  size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  return int(b < 1 ? 1 : b);
}

using Common = NkOptPenalty;

template <typename TW, typename TG>
__device__ __forceinline__ float penalised_grad(const Common& c, TW* w, TG* g, const float* master, size_t i, float* wv) {
  *wv = master ? master[i] : nk_to_f32<TW>(w[i]);
  const float gv = nk_opt_grad(c, nk_to_f32<TG>(g[i]), *wv);
  if (c.write_back_grad) g[i] = nk_from_f32<TG>(gv);  // the reference adds the penalty INTO the gradient (adam/mod.rs:146-148)
  return gv;
}

template <typename TW>
__device__ __forceinline__ void store_w(TW* w, float* master, size_t i, float wv) {
  if (master) master[i] = wv;
  w[i] = nk_from_f32<TW>(wv);
}

// adam/mod.rs:150-166, amsgrad/mod.rs:177-200
template <typename TW, typename TG>
__global__ void __launch_bounds__(kThreads) adam_kernel(TW* __restrict__ w, TG* __restrict__ g, float* __restrict__ exp_avg,
                                                        float* __restrict__ exp_avg_sq, float* __restrict__ max_sq,
                                                        float* __restrict__ master, size_t n, float beta1, float beta2,
                                                        float sqrt_bc2, float step_size, float eps, Common c) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float wv;
    const float gv = penalised_grad<TW, TG>(c, w, g, master, i, &wv);
    float m = exp_avg[i], v = exp_avg_sq[i], mx = max_sq ? max_sq[i] : 0.f;
    wv = nk_adam_update(wv, gv, m, v, max_sq != nullptr, mx, beta1, beta2, sqrt_bc2, step_size, eps);
    exp_avg[i] = m;
    exp_avg_sq[i] = v;
    if (max_sq) max_sq[i] = mx;
    store_w<TW>(w, master, i, wv);
  }
}

// rmsprop/mod.rs:193-300: the four (centered, momentum) variants
template <typename TW, typename TG>
__global__ void __launch_bounds__(kThreads) rmsprop_kernel(TW* __restrict__ w, TG* __restrict__ g, float* __restrict__ square_avg,
                                                           float* __restrict__ grad_avg, float* __restrict__ buf,
                                                           float* __restrict__ master, size_t n, float lr, float alpha,
                                                           float eps, float momentum, Common c) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float wv;
    const float gv = penalised_grad<TW, TG>(c, w, g, master, i, &wv);
    float sq = square_avg[i], ga = grad_avg ? grad_avg[i] : 0.f, b = buf ? buf[i] : 0.f;
    wv = nk_rmsprop_update(wv, gv, sq, grad_avg != nullptr, ga, buf != nullptr, b, lr, alpha, eps, momentum);
    square_avg[i] = sq;
    if (grad_avg) grad_avg[i] = ga;
    if (buf) buf[i] = b;
    store_w<TW>(w, master, i, wv);
  }
}

// adagrad/mod.rs:113-140
template <typename TW, typename TG>
__global__ void __launch_bounds__(kThreads) adagrad_kernel(TW* __restrict__ w, TG* __restrict__ g, float* __restrict__ grad_sq,
                                                           float* __restrict__ master, size_t n, float clr, float eps,
                                                           Common c) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float wv;
    const float gv = penalised_grad<TW, TG>(c, w, g, master, i, &wv);
    float s = grad_sq[i];
    wv = nk_adagrad_update(wv, gv, s, clr, eps);
    grad_sq[i] = s;
    store_w<TW>(w, master, i, wv);
  }
}

#define NK_OPT_DISPATCH(KERNEL, ...)                                                                              \
  do {                                                                                                            \
    if (w_dtype == NK_F32 && g_dtype == NK_F32)                                                                   \
      KERNEL<float, float><<<blocks, kThreads, 0, ctx->stream>>>((float*)w, (float*)g, __VA_ARGS__);              \
    else if (w_dtype == NK_BF16 && g_dtype == NK_BF16)                                                            \
      KERNEL<__nv_bfloat16, __nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)w, (__nv_bfloat16*)g, __VA_ARGS__); \
    else if (w_dtype == NK_BF16)                                                                                  \
      KERNEL<__nv_bfloat16, float><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)w, (float*)g, __VA_ARGS__); \
    else                                                                                                          \
      KERNEL<float, __nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((float*)w, (__nv_bfloat16*)g, __VA_ARGS__); \
  } while (0)

}  // namespace

extern "C" {

int nk_adam_step(nk_ctx* ctx, void* w, int w_dtype, void* g, int g_dtype, float* exp_avg, float* exp_avg_sq,
                 float* max_exp_avg_sq, float* master, size_t n, int64_t step, float lr, float beta1, float beta2,
                 float eps, float l1, float l2, float grad_scale, int write_back_grad) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(w_dtype) && nk_dtype_ok(g_dtype), "nk_adam_step: bad dtype");
  NK_REQUIRE(ctx, step >= 1, "nk_adam_step: step counts from 1 (got %lld)", (long long)step);
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, w && g && exp_avg && exp_avg_sq, "nk_adam_step: NULL pointer");
  // bias corrections on the host in f32 like the reference: 1 - beta.powi(step)  (adam/mod.rs:141-142)
  float p1 = 1.f, p2 = 1.f;
  {
    float b1 = beta1, b2 = beta2;
    for (uint64_t e = uint64_t(step); e; e >>= 1) {
      if (e & 1) p1 *= b1, p2 *= b2;
      b1 *= b1, b2 *= b2;
    }
  }
  const float bc1 = 1.f - p1, bc2 = 1.f - p2;
  const float sqrt_bc2 = sqrtf(bc2), step_size = lr / bc1;
  const int blocks = opt_blocks(ctx, n);
  const Common c{l1, 2.f * l2, grad_scale, write_back_grad};
  NK_OPT_DISPATCH(adam_kernel, exp_avg, exp_avg_sq, max_exp_avg_sq, master, n, beta1, beta2, sqrt_bc2, step_size, eps, c);
  NK_LAUNCHED(ctx, max_exp_avg_sq ? "amsgrad" : "adam");
  return NK_OK;
}

int nk_rmsprop_step(nk_ctx* ctx, void* w, int w_dtype, void* g, int g_dtype, float* square_avg, float* grad_avg,
                    float* momentum_buf, float* master, size_t n, float lr, float alpha, float eps, float momentum,
                    float l1, float l2, float grad_scale, int write_back_grad) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(w_dtype) && nk_dtype_ok(g_dtype), "nk_rmsprop_step: bad dtype");
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, w && g && square_avg, "nk_rmsprop_step: NULL pointer");
  // `.filter(|momentum| *momentum > f32::EPSILON)` (rmsprop/mod.rs:213-216): a tiny momentum is no momentum
  if (!(momentum > FLT_EPSILON)) momentum_buf = nullptr;
  const int blocks = opt_blocks(ctx, n);
  const Common c{l1, 2.f * l2, grad_scale, write_back_grad};
  NK_OPT_DISPATCH(rmsprop_kernel, square_avg, grad_avg, momentum_buf, master, n, lr, alpha, eps, momentum, c);
  NK_LAUNCHED(ctx, "rmsprop");
  return NK_OK;
}

int nk_adagrad_step(nk_ctx* ctx, void* w, int w_dtype, void* g, int g_dtype, float* grad_sq, float* master, size_t n,
                    int64_t step, float lr, float lr_decay, float eps, float l1, float l2, float grad_scale,
                    int write_back_grad) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(w_dtype) && nk_dtype_ok(g_dtype), "nk_adagrad_step: bad dtype");
  NK_REQUIRE(ctx, step >= 1, "nk_adagrad_step: step counts from 1 (got %lld)", (long long)step);
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, w && g && grad_sq, "nk_adagrad_step: NULL pointer");
  const float clr = lr / (1.f + float(step - 1) * lr_decay);  // adagrad/mod.rs:121
  const int blocks = opt_blocks(ctx, n);
  const Common c{l1, 2.f * l2, grad_scale, write_back_grad};
  NK_OPT_DISPATCH(adagrad_kernel, grad_sq, master, n, clr, eps, c);
  NK_LAUNCHED(ctx, "adagrad");
  return NK_OK;
}

}  // extern "C"
