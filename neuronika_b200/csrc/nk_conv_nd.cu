// 1-D and 3-D convolution (SURVEY.md 8-f rank 3): the reference's convolution is generic over the number of sample
// dimensions (convolution/mod.rs:85-123 fwd, 146-189 dX, 191-226 dW, grouped :125-144, 228-294; goldens
// convolution/test.rs:144-239 (1-D), 306-444 (3-D) and their strided / dilated / grouped siblings).  The 2-D case has
// its own engines (nk_conv_gemm.cu, nk_conv_direct.cu); this file is the CUDA-core gather engine for x (N, C, s0, s1, s2)
// with leading sample dims of extent 1 when there are fewer than three.  Same un-padded cross-correlation, same
// accumulate protocol (beta) and argument checks (utils.rs:427-496) as the 2-D entry points.
#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;

struct NdDims {
  int64_t n, cin, cout, groups;
  int64_t in[3], k[3], s[3], d[3], out[3];
};

template <typename T>
__global__ void __launch_bounds__(kThreads) convnd_fwd_kernel(T* __restrict__ y, const T* __restrict__ x,
                                                              const T* __restrict__ wt, NdDims d) {
  const int64_t L = d.out[0] * d.out[1] * d.out[2];
  const int64_t total = d.n * d.cout * L;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  const int64_t isz = d.in[0] * d.in[1] * d.in[2], ksz = d.k[0] * d.k[1] * d.k[2];
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    int64_t rem = idx;
    const int64_t p2 = rem % d.out[2];
    rem /= d.out[2];
    const int64_t p1 = rem % d.out[1];
    rem /= d.out[1];
    const int64_t p0 = rem % d.out[0];
    rem /= d.out[0];
    const int64_t o = rem % d.cout, n = rem / d.cout;
    const int64_t g = o / cout_g;
    float acc = 0.f;
    for (int64_t c = 0; c < cin_g; ++c) {
      const T* xp = x + (n * d.cin + g * cin_g + c) * isz;
      const T* wp = wt + (o * cin_g + c) * ksz;
      for (int64_t i0 = 0; i0 < d.k[0]; ++i0)
        for (int64_t i1 = 0; i1 < d.k[1]; ++i1)
          for (int64_t i2 = 0; i2 < d.k[2]; ++i2) {
            const int64_t u0 = p0 * d.s[0] + i0 * d.d[0], u1 = p1 * d.s[1] + i1 * d.d[1], u2 = p2 * d.s[2] + i2 * d.d[2];
            acc = fmaf(nk_to_f32<T>(wp[(i0 * d.k[1] + i1) * d.k[2] + i2]),
                       nk_to_f32<T>(xp[(u0 * d.in[1] + u1) * d.in[2] + u2]), acc);
          }
    }
    y[idx] = nk_from_f32<T>(acc);
  }
}

// output position along one axis that reads input coordinate u through tap i, or -1
__device__ __forceinline__ int64_t out_pos(int64_t u, int64_t i, int64_t s, int64_t dil, int64_t out) {
  const int64_t pu = u - i * dil;
  if (pu < 0 || pu % s != 0) return -1;
  const int64_t p = pu / s;
  return p < out ? p : -1;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) convnd_bwd_input_kernel(T* __restrict__ dx, const T* __restrict__ g,
                                                                    const T* __restrict__ wt, NdDims d, float beta) {
  const int64_t isz = d.in[0] * d.in[1] * d.in[2], L = d.out[0] * d.out[1] * d.out[2], ksz = d.k[0] * d.k[1] * d.k[2];
  const int64_t total = d.n * d.cin * isz;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    int64_t rem = idx;
    const int64_t u2 = rem % d.in[2];
    rem /= d.in[2];
    const int64_t u1 = rem % d.in[1];
    rem /= d.in[1];
    const int64_t u0 = rem % d.in[0];
    rem /= d.in[0];
    const int64_t c = rem % d.cin, n = rem / d.cin;
    const int64_t grp = c / cin_g, cl = c - grp * cin_g;
    float acc = 0.f;
    for (int64_t i0 = 0; i0 < d.k[0]; ++i0) {
      const int64_t p0 = out_pos(u0, i0, d.s[0], d.d[0], d.out[0]);
      if (p0 < 0) continue;
      for (int64_t i1 = 0; i1 < d.k[1]; ++i1) {
        const int64_t p1 = out_pos(u1, i1, d.s[1], d.d[1], d.out[1]);
        if (p1 < 0) continue;
        for (int64_t i2 = 0; i2 < d.k[2]; ++i2) {
          const int64_t p2 = out_pos(u2, i2, d.s[2], d.d[2], d.out[2]);
          if (p2 < 0) continue;
          const int64_t l = (p0 * d.out[1] + p1) * d.out[2] + p2, kidx = (i0 * d.k[1] + i1) * d.k[2] + i2;
          for (int64_t ol = 0; ol < cout_g; ++ol) {
            const int64_t o = grp * cout_g + ol;
            acc = fmaf(nk_to_f32<T>(g[(n * d.cout + o) * L + l]), nk_to_f32<T>(wt[(o * cin_g + cl) * ksz + kidx]), acc);
          }
        }
      }
    }
    if (beta != 0.f) acc += beta * nk_to_f32<T>(dx[idx]);
    dx[idx] = nk_from_f32<T>(acc);
  }
}

// one block per kernel element (x a chunk of the batch): reduce over (n, output positions), f32 atomics into scratch
template <typename T>
__global__ void __launch_bounds__(kThreads) convnd_bwd_kernel_kernel(float* __restrict__ scratch, const T* __restrict__ g,
                                                                     const T* __restrict__ x, NdDims d,
                                                                     int64_t n_per_block) {
  const int64_t cin_g = d.cin / d.groups, cout_g = d.cout / d.groups;
  const int64_t isz = d.in[0] * d.in[1] * d.in[2], L = d.out[0] * d.out[1] * d.out[2], ksz = d.k[0] * d.k[1] * d.k[2];
  const int64_t widx = blockIdx.x;
  int64_t rem = widx;
  const int64_t kidx = rem % ksz;
  rem /= ksz;
  const int64_t c = rem % cin_g, o = rem / cin_g;
  const int64_t i2 = kidx % d.k[2], i1 = (kidx / d.k[2]) % d.k[1], i0 = kidx / (d.k[2] * d.k[1]);
  const int64_t grp = o / cout_g;
  const int64_t n_begin = int64_t(blockIdx.y) * n_per_block;
  int64_t n_end = n_begin + n_per_block;
  if (n_end > d.n) n_end = d.n;
  float acc = 0.f;
  for (int64_t n = n_begin; n < n_end; ++n) {
    const T* gp = g + (n * d.cout + o) * L;
    const T* xp = x + (n * d.cin + grp * cin_g + c) * isz;
    for (int64_t l = threadIdx.x; l < L; l += blockDim.x) {
      const int64_t p2 = l % d.out[2], p1 = (l / d.out[2]) % d.out[1], p0 = l / (d.out[2] * d.out[1]);
      const int64_t u0 = p0 * d.s[0] + i0 * d.d[0], u1 = p1 * d.s[1] + i1 * d.d[1], u2 = p2 * d.s[2] + i2 * d.d[2];
      acc = fmaf(nk_to_f32<T>(gp[l]), nk_to_f32<T>(xp[(u0 * d.in[1] + u1) * d.in[2] + u2]), acc);
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
__global__ void __launch_bounds__(kThreads) finalize_dwnd(T* __restrict__ dst, const float* __restrict__ scratch,
                                                          int64_t n, float beta) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = scratch[i];
  if (beta != 0.f) v += beta * nk_to_f32<T>(dst[i]);
  dst[i] = nk_from_f32<T>(v);
}

int make_dims(nk_ctx* ctx, const char* who, int nsp, int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout,
              const int64_t* k, const int64_t* s, const int64_t* dil, int64_t groups, NdDims* d) {
  NK_REQUIRE(ctx, nsp >= 1 && nsp <= 3, "%s: 1 to 3 sample dimensions (got %d)", who, nsp);
  NK_REQUIRE(ctx, in_sp && k && s && dil, "%s: NULL shape pointer", who);
  NK_REQUIRE(ctx, n >= 0 && cin > 0 && cout > 0, "%s: bad sizes", who);
  NK_REQUIRE(ctx, groups >= 1, "%s: groups must be >= 1", who);
  NK_REQUIRE(ctx, cin % groups == 0, "In channels %lld is not divisible by groups %lld", (long long)cin, (long long)groups);
  NK_REQUIRE(ctx, cout % groups == 0, "Out channels %lld is not divisible by groups %lld", (long long)cout, (long long)groups);
  d->n = n, d->cin = cin, d->cout = cout, d->groups = groups;
  for (int a = 0; a < 3; ++a) d->in[a] = d->k[a] = d->s[a] = d->d[a] = d->out[a] = 1;
  for (int a = 0; a < nsp; ++a) {
    const int j = 3 - nsp + a;
    NK_REQUIRE(ctx, k[a] > 0 && s[a] > 0 && dil[a] > 0, "%s: kernel, stride and dilation must be positive", who);
    NK_REQUIRE(ctx, in_sp[a] >= (k[a] - 1) * dil[a] + 1, "The kernel size can't be greater than actual input size.");
    d->in[j] = in_sp[a], d->k[j] = k[a], d->s[j] = s[a], d->d[j] = dil[a];
    d->out[j] = (in_sp[a] - dil[a] * (k[a] - 1) - 1) / s[a] + 1;  // conv_out_shape, utils.rs:207-237
  }
  return NK_OK;
}

inline int nd_blocks(nk_ctx* ctx, int64_t total) {
  int64_t b = (total + kThreads - 1) / kThreads;
  const int64_t cap = int64_t(ctx->sm_count) * 16;
  if (b > cap) b = cap;
  return int(b < 1 ? 1 : b);
}

// ---- the 1-D / 3-D convolution layers: y = conv(pad(x), W) + b
struct LayerDims {
  NdDims d;            // the convolution of the padded input
  int64_t padded[3];   // its sample extents (nsp of them)
  bool any_pad;
};

int layer_dims(nk_ctx* ctx, const char* who, int nsp, int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout,
               const int64_t* k, const int64_t* s, const int64_t* dil, const int64_t* pad, int mode, LayerDims* ld) {
  NK_REQUIRE(ctx, nsp == 1 || nsp == 3, "%s: 1 or 3 sample dimensions (got %d); 2-d layers use nk_conv2d_*", who, nsp);
  NK_REQUIRE(ctx, in_sp && pad, "%s: NULL shape pointer", who);
  NK_REQUIRE(ctx, mode >= NK_PAD_CONSTANT && mode <= NK_PAD_REPLICATIVE, "pad: bad mode %d", mode);
  ld->any_pad = false;
  for (int a = 0; a < nsp; ++a) {
    NK_REQUIRE(ctx, in_sp[a] >= 0 && pad[a] >= 0, "pad: negative size");
    NK_REQUIRE(ctx, mode != NK_PAD_REFLECTIVE || pad[a] == 0 || pad[a] < in_sp[a],
               "pad: reflective padding %lld must be smaller than the dimension %lld", (long long)pad[a], (long long)in_sp[a]);
    NK_REQUIRE(ctx, mode != NK_PAD_REPLICATIVE || pad[a] == 0 || in_sp[a] > 0, "pad: replicative padding of an empty dimension");
    ld->padded[a] = in_sp[a] + 2 * pad[a];
    ld->any_pad = ld->any_pad || pad[a] > 0;
  }
  return make_dims(ctx, who, nsp, n, cin, ld->padded, cout, k, s, dil, 1, &ld->d);
}

// the (Cout, 1, ..) bias against the (N, Cout, out...) output: the shapes the Addition node of the composed graph uses
void bias_shapes(const NdDims& d, int nsp, int64_t* bshape, int64_t* yshape) {
  bshape[0] = d.cout, yshape[0] = d.n, yshape[1] = d.cout;
  for (int a = 0; a < nsp; ++a) bshape[1 + a] = 1, yshape[2 + a] = d.out[3 - nsp + a];
}

// the padded input (planes, padded...) in a stream-ordered temporary, as the composed graph's Pad node writes it
int padded_copy(nk_ctx* ctx, const void* x, const LayerDims& ld, int nsp, const int64_t* in_sp, const int64_t* pad, int mode,
                float value, int dtype, void** out) {
  int64_t elems = ld.d.n * ld.d.cin;
  for (int a = 0; a < nsp; ++a) elems *= ld.padded[a];
  int rc = nk_alloc_uninit(ctx, size_t(elems) * nk_dtype_size(dtype), out);
  if (rc) return rc;
  rc = nk_padnd_fwd(ctx, *out, x, ld.d.n * ld.d.cin, nsp, in_sp, pad, mode, value, dtype);
  if (rc) {
    nk_free(ctx, *out);
    *out = nullptr;
  }
  return rc;
}

}  // namespace

// im2col + batched wgmma GEMM with the padding folded into the gather (nk_conv_gemm.cu)
int nk_conv_gemm_nd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int nsp, int64_t n, int64_t cin,
                        const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                        const int64_t* pad, int mode, float value);
int nk_conv_gemm_nd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                              const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                              const int64_t* pad, int mode, float beta);
int nk_conv_gemm_nd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp, int64_t n,
                               int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s,
                               const int64_t* dil, const int64_t* pad, int mode, float value, float beta);

extern "C" {

int nk_convnd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, int nsp, int64_t n, int64_t cin,
                  const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride, const int64_t* dilation,
                  int64_t groups, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_convnd_fwd: bad dtype %d", dtype);
  NdDims d;
  int rc = make_dims(ctx, "nk_convnd_fwd", nsp, n, cin, in_sp, cout, k, stride, dilation, groups, &d);
  if (rc) return rc;
  const int64_t total = d.n * d.cout * d.out[0] * d.out[1] * d.out[2];
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x && w, "nk_convnd_fwd: NULL pointer");
  const int64_t no_pad[3] = {0, 0, 0};
  if (nk_conv_tf32_on(ctx, dtype, groups))
    return nk_conv_tf32_fwd(ctx, y, x, w, nullptr, 0, nsp, n, cin, in_sp, cout, k, stride, dilation, no_pad, NK_PAD_CONSTANT,
                            0.f, true);
  const int blocks = nd_blocks(ctx, total);
  if (dtype == NK_BF16)
    convnd_fwd_kernel<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)y, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, d);
  else
    convnd_fwd_kernel<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)y, (const float*)x, (const float*)w, d);
  NK_LAUNCHED(ctx, "convnd_fwd");
  ctx->last_conv_kernel = "direct_nd_fwd";
  return NK_OK;
}

int nk_convnd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                        const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                        const int64_t* dilation, int64_t groups, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_convnd_bwd_input: bad dtype %d", dtype);
  NdDims d;
  int rc = make_dims(ctx, "nk_convnd_bwd_input", nsp, n, cin, in_sp, cout, k, stride, dilation, groups, &d);
  if (rc) return rc;
  const int64_t total = d.n * d.cin * d.in[0] * d.in[1] * d.in[2];
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && g && w, "nk_convnd_bwd_input: NULL pointer");
  const int64_t no_pad[3] = {0, 0, 0};
  if (nk_conv_tf32_on(ctx, dtype, groups))
    return nk_conv_tf32_bwd_input(ctx, dx, g, w, nsp, n, cin, in_sp, cout, k, stride, dilation, no_pad, NK_PAD_CONSTANT, beta,
                                  true);
  const int blocks = nd_blocks(ctx, total);
  if (dtype == NK_BF16)
    convnd_bwd_input_kernel<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dx, (const __nv_bfloat16*)g, (const __nv_bfloat16*)w, d, beta);
  else
    convnd_bwd_input_kernel<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dx, (const float*)g, (const float*)w, d, beta);
  NK_LAUNCHED(ctx, "convnd_bwd_input");
  ctx->last_conv_kernel = "direct_nd_dx";
  return NK_OK;
}

int nk_convnd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp, int64_t n,
                         int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                         const int64_t* dilation, int64_t groups, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(dw_dtype), "nk_convnd_bwd_kernel: bad dtype");
  NdDims d;
  int rc = make_dims(ctx, "nk_convnd_bwd_kernel", nsp, n, cin, in_sp, cout, k, stride, dilation, groups, &d);
  if (rc) return rc;
  const int64_t welems = d.cout * (d.cin / d.groups) * d.k[0] * d.k[1] * d.k[2];
  NK_REQUIRE(ctx, dwt && (d.n == 0 || (g && x)), "nk_convnd_bwd_kernel: NULL pointer");
  const int64_t no_pad[3] = {0, 0, 0};
  if (d.n > 0 && nk_conv_tf32_on(ctx, dtype, groups))
    return nk_conv_tf32_bwd_kernel(ctx, dwt, dw_dtype, g, x, nsp, n, cin, in_sp, cout, k, stride, dilation, no_pad,
                                   NK_PAD_CONSTANT, 0.f, beta, true);
  float* scratch;
  rc = nk_workspace(ctx, size_t(welems) * sizeof(float), (void**)&scratch);
  if (rc) return rc;
  NK_CUDA(ctx, cudaMemsetAsync(scratch, 0, size_t(welems) * sizeof(float), ctx->stream));
  if (d.n > 0) {
    int64_t want_y = (int64_t(ctx->sm_count) * 4 + welems - 1) / welems;
    if (want_y > d.n) want_y = d.n;
    if (want_y < 1) want_y = 1;
    if (want_y > 65535) want_y = 65535;
    const int64_t n_per_block = (d.n + want_y - 1) / want_y;
    const int64_t gy = (d.n + n_per_block - 1) / n_per_block;
    dim3 grid((unsigned)welems, (unsigned)gy);
    if (dtype == NK_BF16)
      convnd_bwd_kernel_kernel<__nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, (const __nv_bfloat16*)x, d, n_per_block);
    else
      convnd_bwd_kernel_kernel<float><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, (const float*)x, d, n_per_block);
    NK_LAUNCHED(ctx, "convnd_bwd_kernel");
  }
  const int fb = int((welems + kThreads - 1) / kThreads);
  if (dw_dtype == NK_BF16)
    finalize_dwnd<__nv_bfloat16><<<fb, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dwt, scratch, welems, beta);
  else
    finalize_dwnd<float><<<fb, kThreads, 0, ctx->stream>>>((float*)dwt, scratch, welems, beta);
  NK_LAUNCHED(ctx, "convnd_finalize");
  ctx->last_conv_kernel = "direct_nd_dw";
  return NK_OK;
}

// The layers pick the engine as nk_conv2d_* do: the tensor cores for bf16 shapes the im2col engine takes and, in the
// TF32 / TF32X3 modes of nk_conv_f32_config, for every f32 call (nk_conv_tf32.cu; unless nk_conv_config(DIRECT));
// otherwise the padded input in a temporary and the CUDA-core kernels above, i.e. the calls of
// the composed graph pad -> convolution -> + bias, with the same results.
int nk_conv_layer_nd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int nsp, int64_t n, int64_t cin,
                         const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                         const int64_t* dilation, const int64_t* pad, int pad_mode, float pad_value, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_conv_layer_nd_fwd: bad dtype %d", dtype);
  LayerDims ld;
  int rc = layer_dims(ctx, "nk_conv_layer_nd_fwd", nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, &ld);
  if (rc) return rc;
  if (ld.d.n * ld.d.cout * ld.d.out[0] * ld.d.out[1] * ld.d.out[2] == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x && w, "nk_conv_layer_nd_fwd: NULL pointer");
  if (nk_conv_tf32_on(ctx, dtype, 1))
    return nk_conv_tf32_fwd(ctx, y, x, w, bias, 0, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, pad_value,
                            true);
  if (dtype == NK_BF16 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_nd_fwd(ctx, y, x, w, bias, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, pad_value);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  void* xp = nullptr;
  if (ld.any_pad) {
    rc = padded_copy(ctx, x, ld, nsp, in_sp, pad, pad_mode, pad_value, dtype, &xp);
    if (rc) return rc;
  }
  rc = nk_convnd_fwd(ctx, y, xp ? xp : x, w, nsp, n, cin, ld.padded, cout, k, stride, dilation, 1, dtype);
  nk_free(ctx, xp);
  if (rc || !bias) return rc;
  int64_t bshape[4], yshape[5];
  bias_shapes(ld.d, nsp, bshape, yshape);
  return nk_add_bcast_fwd(ctx, y, y, bias, dtype, nsp + 2, yshape, nsp + 2, yshape, nsp + 1, bshape);
}

int nk_conv_layer_nd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                               const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* stride,
                               const int64_t* dilation, const int64_t* pad, int pad_mode, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_conv_layer_nd_bwd_input: bad dtype %d", dtype);
  LayerDims ld;
  int rc = layer_dims(ctx, "nk_conv_layer_nd_bwd_input", nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, &ld);
  if (rc) return rc;
  int64_t total = n * cin;
  for (int a = 0; a < nsp; ++a) total *= in_sp[a];
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && g && w, "nk_conv_layer_nd_bwd_input: NULL pointer");
  if (nk_conv_tf32_on(ctx, dtype, 1))
    return nk_conv_tf32_bwd_input(ctx, dx, g, w, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, beta, true);
  if (dtype == NK_BF16 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_nd_bwd_input(ctx, dx, g, w, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, beta);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  if (!ld.any_pad)
    return nk_convnd_bwd_input(ctx, dx, g, w, nsp, n, cin, in_sp, cout, k, stride, dilation, 1, dtype, beta);
  // the gradient of the padded input, then its interior slice (pad/mod.rs:157-182)
  int64_t elems = n * cin;
  for (int a = 0; a < nsp; ++a) elems *= ld.padded[a];
  void* dxp = nullptr;
  rc = nk_alloc_uninit(ctx, size_t(elems) * nk_dtype_size(dtype), &dxp);
  if (rc) return rc;
  rc = nk_convnd_bwd_input(ctx, dxp, g, w, nsp, n, cin, ld.padded, cout, k, stride, dilation, 1, dtype, 0.f);
  if (rc == NK_OK) rc = nk_padnd_bwd(ctx, dx, dxp, n * cin, nsp, in_sp, pad, dtype, beta);
  nk_free(ctx, dxp);
  return rc;
}

int nk_conv_layer_nd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, void* dbias, const void* g, const void* x, int nsp,
                                int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k,
                                const int64_t* stride, const int64_t* dilation, const int64_t* pad, int pad_mode,
                                float pad_value, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(dw_dtype), "nk_conv_layer_nd_bwd_kernel: bad dtype");
  LayerDims ld;
  int rc = layer_dims(ctx, "nk_conv_layer_nd_bwd_kernel", nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode, &ld);
  if (rc) return rc;
  // an empty batch adds nothing: dW (and dbias) = beta * dW; g and x may then be NULL
  NK_REQUIRE(ctx, dwt && (n == 0 || (g && x)), "nk_conv_layer_nd_bwd_kernel: NULL pointer");
  int64_t bshape[4], gshape[5];
  bias_shapes(ld.d, nsp, bshape, gshape);
  if (dbias) {   // the composed graph's AdditionBackward: the un-broadcast of g onto (Cout, 1, ..)
    rc = nk_unbroadcast_acc(ctx, dbias, dw_dtype, nsp + 1, bshape, g, dtype, nsp + 2, gshape, beta);
    if (rc) return rc;
  }
  if (n > 0 && nk_conv_tf32_on(ctx, dtype, 1))
    return nk_conv_tf32_bwd_kernel(ctx, dwt, dw_dtype, g, x, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode,
                                   pad_value, beta, true);
  if (n > 0 && dtype == NK_BF16 && ctx->conv_engine != NK_CONV_DIRECT) {
    rc = nk_conv_gemm_nd_bwd_kernel(ctx, dwt, dw_dtype, g, x, nsp, n, cin, in_sp, cout, k, stride, dilation, pad, pad_mode,
                                    pad_value, beta);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  void* xp = nullptr;
  if (n > 0 && ld.any_pad) {
    rc = padded_copy(ctx, x, ld, nsp, in_sp, pad, pad_mode, pad_value, dtype, &xp);
    if (rc) return rc;
  }
  rc = nk_convnd_bwd_kernel(ctx, dwt, dw_dtype, g, xp ? xp : x, nsp, n, cin, ld.padded, cout, k, stride, dilation, 1, dtype,
                            beta);
  nk_free(ctx, xp);
  return rc;
}

}  // extern "C"
