// Direct (CUDA-core) 2-D convolution kernels: the general engine for every stride / dilation /
// groups combination and both element types.  The tensor-core im2col engines take over for the shapes they support
// (bf16: nk_conv_gemm.cu; f32 once nk_conv_f32_config has set TF32 / TF32X3: nk_conv_tf32.cu); this file is the
// complete, always-valid path and what the reference's own golden cases (tiny, integer valued) run through.
// Reference semantics: convolution/mod.rs:85-123 (fwd, beta = 0), :146-189 (dX, accumulate),
// :191-226 (dW, accumulate), grouped variants :125-144, 228-294; arg checks utils.rs:427-496.
#include <stdlib.h>

#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;

struct ConvDims {
  int64_t n, cin, h, w, cout, kh, kw, sh, sw, dh, dw, groups, ho, wo;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) conv_fwd_direct(T* __restrict__ y, const T* __restrict__ x,
                                                           const T* __restrict__ wt, const T* __restrict__ bias,
                                                           int relu, ConvDims d) {
  const int64_t total = d.n * d.cout * d.ho * d.wo;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const int64_t q = idx % d.wo, p = (idx / d.wo) % d.ho, o = (idx / (d.wo * d.ho)) % d.cout,
                  n = idx / (d.wo * d.ho * d.cout);
    const int64_t g = o / cout_g;
    float acc = 0.f;
    for (int64_t c = 0; c < cin_g; ++c) {
      const T* xp = x + ((n * d.cin + g * cin_g + c) * d.h + p * d.sh) * d.w + q * d.sw;
      const T* wp = wt + ((o * cin_g + c) * d.kh) * d.kw;
      for (int64_t i = 0; i < d.kh; ++i)
        for (int64_t j = 0; j < d.kw; ++j)
          acc = fmaf(nk_to_f32<T>(wp[i * d.kw + j]), nk_to_f32<T>(xp[i * d.dh * d.w + j * d.dw]), acc);
    }
    if (bias) acc += nk_to_f32<T>(bias[o]);
    if (relu) acc = acc > 0.f ? acc : 0.f;
    y[idx] = nk_from_f32<T>(acc);
  }
}

// gather form of dX: dx[n,c,u,v] (+)= sum_{o,i,j : u = p*sh + i*dh, v = q*sw + j*dw} g[n,o,p,q] * w[o,c,i,j]
template <typename T>
__global__ void __launch_bounds__(kThreads) conv_bwd_input_direct(T* __restrict__ dx, const T* __restrict__ g,
                                                                 const T* __restrict__ wt, ConvDims d, float beta) {
  const int64_t total = d.n * d.cin * d.h * d.w;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const int64_t v = idx % d.w, u = (idx / d.w) % d.h, c = (idx / (d.w * d.h)) % d.cin,
                  n = idx / (d.w * d.h * d.cin);
    const int64_t grp = c / cin_g, cl = c - grp * cin_g;
    float acc = 0.f;
    for (int64_t i = 0; i < d.kh; ++i) {
      const int64_t pu = u - i * d.dh;
      if (pu < 0 || pu % d.sh != 0) continue;
      const int64_t p = pu / d.sh;
      if (p >= d.ho) continue;
      for (int64_t j = 0; j < d.kw; ++j) {
        const int64_t qv = v - j * d.dw;
        if (qv < 0 || qv % d.sw != 0) continue;
        const int64_t q = qv / d.sw;
        if (q >= d.wo) continue;
        for (int64_t ol = 0; ol < cout_g; ++ol) {
          const int64_t o = grp * cout_g + ol;
          acc = fmaf(nk_to_f32<T>(g[((n * d.cout + o) * d.ho + p) * d.wo + q]),
                     nk_to_f32<T>(wt[((o * cin_g + cl) * d.kh + i) * d.kw + j]), acc);
        }
      }
    }
    if (beta != 0.f) acc += beta * nk_to_f32<T>(dx[idx]);
    dx[idx] = nk_from_f32<T>(acc);
  }
}

// dW[o,c,i,j] = sum_{n,p,q} g[n,o,p,q] * x[n, c, p*sh + i*dh, q*sw + j*dw]
// grid.x = one weight element, grid.y = chunk of the batch; f32 atomics into scratch
template <typename T>
__global__ void __launch_bounds__(kThreads) conv_bwd_kernel_direct(float* __restrict__ scratch,
                                                                  const T* __restrict__ g, const T* __restrict__ x,
                                                                  ConvDims d, int64_t n_per_block) {
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  const int64_t widx = blockIdx.x;
  const int64_t j = widx % d.kw, i = (widx / d.kw) % d.kh, c = (widx / (d.kw * d.kh)) % cin_g,
                o = widx / (d.kw * d.kh * cin_g);
  const int64_t grp = o / cout_g;
  const int64_t n_begin = int64_t(blockIdx.y) * n_per_block;
  int64_t n_end = n_begin + n_per_block;
  if (n_end > d.n) n_end = d.n;
  const int64_t L = d.ho * d.wo;
  float acc = 0.f;
  for (int64_t n = n_begin; n < n_end; ++n) {
    const T* gp = g + (n * d.cout + o) * L;
    const T* xp = x + ((n * d.cin + grp * cin_g + c) * d.h + i * d.dh) * d.w + j * d.dw;
    for (int64_t l = threadIdx.x; l < L; l += blockDim.x) {
      const int64_t p = l / d.wo, q = l - p * d.wo;
      acc = fmaf(nk_to_f32<T>(gp[l]), nk_to_f32<T>(xp[p * d.sh * d.w + q * d.sw]), acc);
    }
  }
  acc = nk_warp_sum(acc);
  __shared__ float sm[kThreads / 32];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < kThreads / 32; ++k) s += sm[k];
    atomicAdd(&scratch[widx], s);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) finalize_dw(T* __restrict__ dst, const float* __restrict__ scratch,
                                                       int64_t n, float beta) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = scratch[i];
  if (beta != 0.f) v += beta * nk_to_f32<T>(dst[i]);
  dst[i] = nk_from_f32<T>(v);
}

int check_dims(nk_ctx* ctx, const char* who, ConvDims& d) {
  // same predicates as check_conv_args / check_groups_args (utils.rs:427-496)
  NK_REQUIRE(ctx, d.n >= 0 && d.cin > 0 && d.cout > 0 && d.kh > 0 && d.kw > 0, "%s: bad sizes", who);
  NK_REQUIRE(ctx, d.sh > 0 && d.sw > 0 && d.dh > 0 && d.dw > 0, "%s: stride and dilation must be positive", who);
  NK_REQUIRE(ctx, d.groups >= 1, "%s: groups must be >= 1", who);
  NK_REQUIRE(ctx, d.cin % d.groups == 0, "In channels %lld is not divisible by groups %lld", (long long)d.cin,
             (long long)d.groups);
  NK_REQUIRE(ctx, d.cout % d.groups == 0, "Out channels %lld is not divisible by groups %lld", (long long)d.cout,
             (long long)d.groups);
  NK_REQUIRE(ctx, d.h >= (d.kh - 1) * d.dh + 1 && d.w >= (d.kw - 1) * d.dw + 1,
             "The kernel size can't be greater than actual input size.");
  d.ho = (d.h - d.dh * (d.kh - 1) - 1) / d.sh + 1;  // conv_out_shape, utils.rs:207-237
  d.wo = (d.w - d.dw * (d.kw - 1) - 1) / d.sw + 1;
  return NK_OK;
}

inline int blocks_for(nk_ctx* ctx, int64_t total) {
  int64_t b = (total + kThreads - 1) / kThreads;
  const int64_t cap = int64_t(ctx->sm_count) * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}

}  // namespace

// im2col + batched wgmma GEMM for every other bf16, groups = 1 shape (nk_conv_gemm.cu)
int nk_conv_gemm_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, int64_t n, int64_t cin,
                     int64_t h, int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw);
int nk_conv_gemm_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int64_t n, int64_t cin, int64_t h, int64_t wd,
                           int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw, float beta);
int nk_conv_gemm_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int64_t n, int64_t cin, int64_t h,
                            int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw,
                            float beta);
extern "C" {

int nk_conv2d_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, int64_t n,
                  int64_t cin, int64_t h, int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw,
                  int64_t dh, int64_t dw, int64_t groups, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_conv2d_fwd: bad dtype %d", dtype);
  ConvDims d{n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw, groups, 0, 0};
  int rc = check_dims(ctx, "nk_conv2d_fwd", d);
  if (rc) return rc;
  const int64_t total = d.n * d.cout * d.ho * d.wo;
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x && w, "nk_conv2d_fwd: NULL pointer");
  const int64_t in_sp[2] = {h, wd}, ks[2] = {kh, kw}, st[2] = {sh, sw}, dl[2] = {dh, dw}, no_pad[2] = {0, 0};
  if (nk_conv_tf32_on(ctx, dtype, groups))
    return nk_conv_tf32_fwd(ctx, y, x, w, bias, relu, 2, n, cin, in_sp, cout, ks, st, dl, no_pad, NK_PAD_CONSTANT, 0.f, false);
  if (dtype == NK_BF16 && groups == 1 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_fwd(ctx, y, x, w, bias, relu, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  ctx->last_conv_kernel = "direct_fwd";
  int blocks = blocks_for(ctx, total);
  if (dtype == NK_BF16)
    conv_fwd_direct<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)y, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)bias, relu, d);
  else
    conv_fwd_direct<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)y, (const float*)x, (const float*)w, (const float*)bias, relu, d);
  NK_LAUNCHED(ctx, "conv_fwd_direct");
  return NK_OK;
}

int nk_conv2d_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int64_t n, int64_t cin, int64_t h,
                        int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh,
                        int64_t dw, int64_t groups, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_conv2d_bwd_input: bad dtype %d", dtype);
  ConvDims d{n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw, groups, 0, 0};
  int rc = check_dims(ctx, "nk_conv2d_bwd_input", d);
  if (rc) return rc;
  const int64_t total = d.n * d.cin * d.h * d.w;
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && g && w, "nk_conv2d_bwd_input: NULL pointer");
  const int64_t in_sp[2] = {h, wd}, ks[2] = {kh, kw}, st[2] = {sh, sw}, dl[2] = {dh, dw}, no_pad[2] = {0, 0};
  if (nk_conv_tf32_on(ctx, dtype, groups))
    return nk_conv_tf32_bwd_input(ctx, dx, g, w, 2, n, cin, in_sp, cout, ks, st, dl, no_pad, NK_PAD_CONSTANT, beta, false);
  if (dtype == NK_BF16 && groups == 1 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_bwd_input(ctx, dx, g, w, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw, beta);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  ctx->last_conv_kernel = "direct_bwd_input";
  int blocks = blocks_for(ctx, total);
  if (dtype == NK_BF16)
    conv_bwd_input_direct<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dx, (const __nv_bfloat16*)g, (const __nv_bfloat16*)w, d, beta);
  else
    conv_bwd_input_direct<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dx, (const float*)g, (const float*)w, d, beta);
  NK_LAUNCHED(ctx, "conv_bwd_input_direct");
  return NK_OK;
}

int nk_conv2d_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, void* dbias, const void* g, const void* x, int64_t n,
                         int64_t cin, int64_t h, int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh,
                         int64_t sw, int64_t dh, int64_t dw, int64_t groups, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(dw_dtype), "nk_conv2d_bwd_kernel: bad dtype");
  ConvDims d{n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw, groups, 0, 0};
  int rc = check_dims(ctx, "nk_conv2d_bwd_kernel", d);
  if (rc) return rc;
  const int64_t nw = d.cout * (d.cin / d.groups) * d.kh * d.kw;
  // an empty batch adds nothing: dW (and dbias) = beta * dW, as in nk_convnd_bwd_kernel; g and x may then be NULL
  NK_REQUIRE(ctx, dwt && (d.n == 0 || (g && x)), "nk_conv2d_bwd_kernel: NULL pointer");
  const int64_t in_sp[2] = {h, wd}, ks[2] = {kh, kw}, st[2] = {sh, sw}, dl[2] = {dh, dw}, no_pad[2] = {0, 0};
  if (d.n > 0 && nk_conv_tf32_on(ctx, dtype, groups)) {
    rc = nk_conv_tf32_bwd_kernel(ctx, dwt, dw_dtype, g, x, 2, n, cin, in_sp, cout, ks, st, dl, no_pad, NK_PAD_CONSTANT, 0.f,
                                 beta, false);
    if (rc == NK_OK && dbias) {
      int64_t dshape[3] = {d.cout, 1, 1};
      int64_t gshape[4] = {d.n, d.cout, d.ho, d.wo};
      rc = nk_unbroadcast_acc(ctx, dbias, dw_dtype, 3, dshape, g, dtype, 4, gshape, beta);
    }
    return rc;
  }
  if (d.n > 0 && dtype == NK_BF16 && groups == 1 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_bwd_kernel(ctx, dwt, dw_dtype, g, x, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw, beta);
    if (rc == NK_OK && dbias) {
      int64_t dshape[3] = {d.cout, 1, 1};
      int64_t gshape[4] = {d.n, d.cout, d.ho, d.wo};
      rc = nk_unbroadcast_acc(ctx, dbias, dw_dtype, 3, dshape, g, dtype, 4, gshape, beta);
    }
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  ctx->last_conv_kernel = "direct_bwd_kernel";
  if (dbias) {
    int64_t dshape[3] = {d.cout, 1, 1};
    int64_t gshape[4] = {d.n, d.cout, d.ho, d.wo};
    rc = nk_unbroadcast_acc(ctx, dbias, dw_dtype, 3, dshape, g, dtype, 4, gshape, beta);
    if (rc) return rc;
  }
  float* scratch;
  rc = nk_workspace(ctx, size_t(nw) * sizeof(float), (void**)&scratch);
  if (rc) return rc;
  NK_CUDA(ctx, cudaMemsetAsync(scratch, 0, size_t(nw) * sizeof(float), ctx->stream));
  if (d.n > 0) {
    int64_t want_y = (int64_t(ctx->sm_count) * 4 + nw - 1) / nw;
    if (want_y > d.n) want_y = d.n;
    if (want_y < 1) want_y = 1;
    const int64_t n_per_block = (d.n + want_y - 1) / want_y;
    const int64_t gy = (d.n + n_per_block - 1) / n_per_block;
    NK_REQUIRE(ctx, gy <= 65535, "nk_conv2d_bwd_kernel: batch grid too large");
    dim3 grid((unsigned)nw, (unsigned)gy);
    if (dtype == NK_BF16)
      conv_bwd_kernel_direct<__nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, (const __nv_bfloat16*)x, d, n_per_block);
    else
      conv_bwd_kernel_direct<float><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, (const float*)x, d, n_per_block);
    NK_LAUNCHED(ctx, "conv_bwd_kernel_direct");
  }
  int blocks = int((nw + kThreads - 1) / kThreads);
  if (dw_dtype == NK_BF16)
    finalize_dw<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dwt, scratch, nw, beta);
  else
    finalize_dw<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dwt, scratch, nw, beta);
  NK_LAUNCHED(ctx, "finalize_dw");
  return NK_OK;
}

}  // extern "C"
