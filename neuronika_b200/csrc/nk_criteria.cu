// The criteria beside MSE / NLL: mean absolute error (absolute_error/mod.rs), binary cross entropy (bce/mod.rs), binary
// cross entropy on logits (bce_with_logits/mod.rs) and Kullback-Leibler divergence (kldiv/mod.rs), with the reference's
// per-element maths and operation order, in f32 whatever the storage type.
//   forward:  one pass over (x, t) in 8-element vectors (16-byte loads) with a scalar tail, f32 partial sums carried
//             into double every 64 terms, one double per block; then the single-warp fixed-order stage 2 of
//             nk_elementwise.cu.  The partition depends only on n and the SM count, so repeated calls are bitwise equal.
//   backward: one elementwise pass dx = beta*dx + dloss/dx * g, dx in its own element type.
#include <float.h>

#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;

inline int grid_for(nk_ctx* ctx, size_t work_items) {
  size_t b = (work_items + kThreads - 1) / kThreads;
  const size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// f32::clamp(v, -100, f32::MAX): NaN stays NaN
__device__ __forceinline__ float clamp_log(float v) { return v < -100.f ? -100.f : (v > FLT_MAX ? FLT_MAX : v); }

// each criterion: fwd(x, t) is one element's term of the sum; bwd(x, t, g) its derivative times the seed, before the mean.
// Products that feed an addition are rounded on their own (__fmul_rn / __fadd_rn: no contraction into an FMA), as in
// the reference's f32 arithmetic, so that the backward is bit-exact against it.
struct MaeOp {  // absolute_error/mod.rs:45-57, 96-122
  static constexpr bool kUsesX = true;
  __device__ float fwd(float x, float t) const { return fabsf(x - t); }
  __device__ float bwd(float x, float t, float g) const {
    const float d = x - t;
    if (d == 0.f) return 0.f;
    return (d != d ? d : copysignf(1.f, d)) * g;  // f32::signum (NaN stays NaN)
  }
};
struct BceOp {  // bce/mod.rs:45-61, 100-125
  static constexpr bool kUsesX = true;
  __device__ float fwd(float x, float t) const {
    return __fmul_rn(t - 1.f, clamp_log(logf(1.f - x))) - __fmul_rn(t, clamp_log(logf(x)));
  }
  __device__ float bwd(float x, float t, float g) const { return (x - t) / fmaxf((1.f - x) * x, FLT_EPSILON) * g; }
};
struct BceLogitsOp {  // bce_with_logits/mod.rs:46-66, 106-131
  static constexpr bool kUsesX = true;
  __device__ float fwd(float x, float t) const {
    const float m = fmaxf(-x, 0.f);
    return __fmul_rn(1.f - t, x) + m + logf(expf(-m) + expf(-x - m));
  }
  __device__ float bwd(float x, float t, float g) const { return (1.f / (1.f + expf(-x)) - t) * g; }
};
struct KlDivOp {  // kldiv/mod.rs:46-61, 98-116; a zero target contributes 0 (SURVEY.md 8-c defect 9)
  static constexpr bool kUsesX = false;
  __device__ float fwd(float x, float t) const { return t > 0.f ? t * (logf(t) - x) : 0.f; }
  __device__ float bwd(float, float t, float g) const { return -t * g; }
};

template <typename T, typename Op, bool VEC>
__global__ void __launch_bounds__(kThreads) crit_fwd_kernel(double* __restrict__ partials, const T* __restrict__ x,
                                                           const T* __restrict__ t, size_t n, Op op) {
  const size_t tid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  float acc = 0.f;
  double dacc = 0.0;
  int cnt = 0;
  auto add = [&](float v) {
    acc = __fadd_rn(acc, v);
    if (++cnt == 64) {  // bound the f32 partial's error, then carry in double
      dacc += double(acc);
      acc = 0.f;
      cnt = 0;
    }
  };
  size_t done = 0;
  if (VEC) {
    const size_t npk = n / 8;
    for (size_t v = tid; v < npk; v += stride) {
      NkPack8<T> a, b;
      a.load(x + v * 8);
      b.load(t + v * 8);
#pragma unroll
      for (int i = 0; i < 8; ++i) add(op.fwd(a.get(i), b.get(i)));
    }
    done = npk * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) add(op.fwd(nk_to_f32<T>(x[i]), nk_to_f32<T>(t[i])));
  dacc += double(acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dacc += __shfl_xor_sync(0xffffffffu, dacc, o);
  __shared__ double sm[kThreads / 32];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = dacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += sm[i];
    partials[blockIdx.x] = s;
  }
}

// dx = (RMW ? beta*dx : 0) + (mean ? bwd / div : bwd)
template <typename T, typename TD, typename Op, bool RMW, bool VEC>
__global__ void __launch_bounds__(kThreads) crit_bwd_kernel(TD* __restrict__ dx, const T* __restrict__ x,
                                                           const T* __restrict__ t, const float* __restrict__ g,
                                                           size_t n, int mean, float div, float beta, Op op) {
  const size_t tid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  const float gv = *g;
  auto term = [&](float xv, float tv) {
    const float v = op.bwd(xv, tv, gv);
    return mean ? v / div : v;
  };
  size_t done = 0;
  if (VEC) {
    const size_t npk = n / 8;
    for (size_t v = tid; v < npk; v += stride) {
      NkPack8<T> a, b;
      NkPack8<TD> o;
      if (Op::kUsesX) a.load(x + v * 8);
      b.load(t + v * 8);
      if (RMW) o.load(dx + v * 8);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float r = term(Op::kUsesX ? a.get(i) : 0.f, b.get(i));
        if (RMW) r = __fadd_rn(__fmul_rn(beta, o.get(i)), r);
        o.set(i, r);
      }
      o.store(dx + v * 8);
    }
    done = npk * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    float r = term(Op::kUsesX ? nk_to_f32<T>(x[i]) : 0.f, nk_to_f32<T>(t[i]));
    if (RMW) r = __fadd_rn(__fmul_rn(beta, nk_to_f32<TD>(dx[i])), r);
    dx[i] = nk_from_f32<TD>(r);
  }
}

template <typename Op>
int crit_fwd(nk_ctx* ctx, const char* name, float* loss, const void* x, const void* t, size_t n, int dtype,
             double scale) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", name, dtype);
  NK_REQUIRE(ctx, loss && x && t && n > 0, "%s: NULL pointer or empty input", name);
  const bool vec = aligned16(x) && aligned16(t);
  const int blocks = grid_for(ctx, vec ? n / 8 + 1 : n);
  double* partials;
  int rc = nk_workspace(ctx, size_t(blocks) * sizeof(double), (void**)&partials);
  if (rc) return rc;
  NK_DISPATCH_DTYPE(dtype, T, {
    if (vec)
      crit_fwd_kernel<T, Op, true><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n, Op{});
    else
      crit_fwd_kernel<T, Op, false><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n, Op{});
  });
  NK_LAUNCHED(ctx, name);
  return nk_reduce_finish(ctx, loss, partials, blocks, scale);
}

template <typename T, typename TD, typename Op>
void launch_bwd(nk_ctx* ctx, int blocks, bool vec, void* dx, const void* x, const void* t, const float* g, size_t n,
                int mean, float div, float beta) {
  TD* d = static_cast<TD*>(dx);
  const T* a = static_cast<const T*>(x);
  const T* b = static_cast<const T*>(t);
  if (beta != 0.f) {
    if (vec)
      crit_bwd_kernel<T, TD, Op, true, true><<<blocks, kThreads, 0, ctx->stream>>>(d, a, b, g, n, mean, div, beta, Op{});
    else
      crit_bwd_kernel<T, TD, Op, true, false><<<blocks, kThreads, 0, ctx->stream>>>(d, a, b, g, n, mean, div, beta, Op{});
  } else {
    if (vec)
      crit_bwd_kernel<T, TD, Op, false, true><<<blocks, kThreads, 0, ctx->stream>>>(d, a, b, g, n, mean, div, beta, Op{});
    else
      crit_bwd_kernel<T, TD, Op, false, false><<<blocks, kThreads, 0, ctx->stream>>>(d, a, b, g, n, mean, div, beta, Op{});
  }
}

template <typename Op>
int crit_bwd(nk_ctx* ctx, const char* name, void* dx, int dx_dtype, const void* x, const void* t, const float* g,
             size_t n, int dtype, int mean, float div, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(dx_dtype), "%s: bad dtype %d / dx dtype %d", name, dtype, dx_dtype);
  NK_REQUIRE(ctx, dx && (x || !Op::kUsesX) && t && g && n > 0, "%s: NULL pointer or empty input", name);
  const bool vec = aligned16(dx) && (!Op::kUsesX || aligned16(x)) && aligned16(t);
  const int blocks = grid_for(ctx, vec ? n / 8 + 1 : n);
  NK_DISPATCH_DTYPE(dtype, T, {
    if (dx_dtype == NK_BF16)
      launch_bwd<T, __nv_bfloat16, Op>(ctx, blocks, vec, dx, x, t, g, n, mean, div, beta);
    else
      launch_bwd<T, float, Op>(ctx, blocks, vec, dx, x, t, g, n, mean, div, beta);
  });
  NK_LAUNCHED(ctx, name);
  return NK_OK;
}

}  // namespace

extern "C" {

int nk_mae_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean) {
  return crit_fwd<MaeOp>(ctx, "nk_mae_fwd", loss, x, t, n, dtype, mean ? 1.0 / double(n) : 1.0);
}
int nk_mae_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n, int dtype,
               int mean, float beta) {
  return crit_bwd<MaeOp>(ctx, "nk_mae_bwd", dx, dx_dtype, x, t, g, n, dtype, mean, float(n), beta);
}

int nk_bce_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean) {
  return crit_fwd<BceOp>(ctx, "nk_bce_fwd", loss, x, t, n, dtype, mean ? 1.0 / double(n) : 1.0);
}
int nk_bce_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n, int dtype,
               int mean, float beta) {
  return crit_bwd<BceOp>(ctx, "nk_bce_bwd", dx, dx_dtype, x, t, g, n, dtype, mean, float(n), beta);
}

int nk_bce_with_logits_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean) {
  return crit_fwd<BceLogitsOp>(ctx, "nk_bce_with_logits_fwd", loss, x, t, n, dtype, mean ? 1.0 / double(n) : 1.0);
}
int nk_bce_with_logits_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, const void* t, const float* g, size_t n,
                           int dtype, int mean, float beta) {
  return crit_bwd<BceLogitsOp>(ctx, "nk_bce_with_logits_bwd", dx, dx_dtype, x, t, g, n, dtype, mean, float(n), beta);
}

int nk_kldiv_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int64_t batch, int dtype, int mean) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, batch > 0, "nk_kldiv_fwd: batch must be positive");
  return crit_fwd<KlDivOp>(ctx, "nk_kldiv_fwd", loss, x, t, n, dtype, mean ? 1.0 / double(batch) : 1.0);
}
int nk_kldiv_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* t, const float* g, size_t n, int64_t batch, int dtype,
                 int mean, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, batch > 0, "nk_kldiv_bwd: batch must be positive");
  return crit_bwd<KlDivOp>(ctx, "nk_kldiv_bwd", dx, dx_dtype, nullptr, t, g, n, dtype, mean, float(batch), beta);
}

}  // extern "C"
