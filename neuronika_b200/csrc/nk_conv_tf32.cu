// f32 convolution on the tensor cores (sm_90a): im2col + the TF32 / 3xTF32 wgmma GEMM of nk_gemm_tf32.cu, in the
// context's f32 convolution mode (nk_conv_f32_config).  Every f32, groups = 1 call of nk_conv2d_*, nk_convnd_* and
// nk_conv_layer_nd_* with a non-empty batch comes here once the mode is TF32 or TF32X3 (unless nk_conv_config(DIRECT)),
// whatever its shape, alignment or padding: the numerics of a mode never depend on the shape.
//
// tf32 wgmma reads both operands K-major only (nk_gemm_tf32.cu), so each product is laid out with its reduction axis
// contiguous in both operands; every element is rounded on its way in (tf32_put: TF32, or the [hi|hi|lo] / [hi|lo|hi]
// segments of 3xTF32), including the fill values of the constant padding mode:
//   forward  Y[n] (Cout x L) = W (Cout x K) . cols[n]^T     A = W packed, shared by the samples;  B = cols[n] (L rows x K),
//            + bias per row, ReLU (the GEMM epilogue)          written by the gather through a shared-memory transpose
//   dX       dcolsT[n] (K x L) = W^T . G[n], col2im          A = W^T packed (K rows x Cout);  B = G[n]^T (L rows x Cout)
//   dW       dW (Cout x K) = sum_n G[n] . cols[n]            A = G (Cout rows x (n, l));  B = colsT (K rows x (n, l)), the
//                                                           gather's other layout
// The dW reduction (N.L terms) is split into ranges of k-blocks, each range one batch entry of the GEMM writing its own
// (Cout x K) partial; tf32_dw_reduce sums the partials (and the sample chunks) in a fixed order, so two identical calls
// give the same bits.  The padding of the 1-D / 3-D layers is folded into the gather (pad_src_index, as the bf16 engine)
// and col2im writes only the interior dx positions (the reference's pad backward).
//
// Temporaries are stream-ordered (nk_alloc_uninit / nk_free: a captured step takes them from its arena).  With s = 1
// (TF32) or 3 (3xTF32) and ceil4 the TMA row pitch, per chunk of nn samples (chunks of <= 4 GB):
//   forward  Cout.ceil4(s.K).4 + nn.L.ceil4(s.K).4 bytes
//   dX       K.ceil4(s.Cout).4 + nn.L.ceil4(s.Cout).4 + nn.K.L.4
//   dW       (Cout + K).ceil4(s.nn.L).4, + (splits + 1).Cout.K.4
#include "nk_conv_im2col.cuh"
#include "nk_tf32.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int64_t kChunkBytes = int64_t(4) << 30;

inline int64_t ceil4(int64_t v) { return (v + 3) / 4 * 4; }

// Operand element (ns, k, l) of the im2col matrix -- x at padded coordinate p_a * s_a + i_a * d_a along each axis, or the
// fill value -- rounded by tf32_put into
//   kLK  (forward B, L rows x K):     dst[(ns * L + l) * ldp + k], segments seg_len = K apart
//   !kLK (dW B, K rows x (ns, l)):    dst[k * ldp + ns * L + l],   segments seg_len = nn * L apart
// One 32 (l) x 32 (k) tile at a time per block of 32 x 8 threads (grid.y steps through the k tiles, grid.z through the
// samples).  x is contiguous along l (unit stride), so the reads go with lanes along l; the !kLK layout is written the
// same way, the kLK one through a shared-memory transpose (lanes along k).
template <bool kLK>
__global__ void __launch_bounds__(kThreads) tf32_im2col_kernel(float* __restrict__ dst, const float* __restrict__ x, CgNdDims d,
                                                               int64_t n0, int64_t nn, int64_t ldp, int64_t seg_len,
                                                               int segments, int lo_seg) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t l0 = int64_t(blockIdx.x) * 32;
  const int in0 = int(d.in[0]), in1 = int(d.in[1]), in2 = int(d.in[2]), k1 = int(d.k[1]), k2 = int(d.k[2]);
  const int ksz = int(d.k[0]) * k1 * k2;
  const int64_t isz = int64_t(in0) * in1 * in2;
  // this thread's output position (read phase)
  const int64_t l = l0 + tx;
  const bool l_ok = l < d.L;
  int q0 = 0, q1 = 0, q2 = 0;
  if (l_ok) {
    q2 = int(l % d.out[2]);
    const int64_t r = l / d.out[2];
    q1 = int(r % d.out[1]), q0 = int(r / d.out[1]);
  }
  const int64_t k_tiles = (d.K + 31) / 32;
  bool first = true;
  for (int64_t ns = blockIdx.z; ns < nn; ns += gridDim.z) {
    const float* xs = x + (n0 + ns) * d.cin * isz;
    for (int64_t kt = blockIdx.y; kt < k_tiles; kt += gridDim.y) {
      const int64_t k0 = kt * 32;
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t k = k0 + ty + 8 * i;
        v[i] = 0.f;
        if (l_ok && k < d.K) {
          const int c = int(k) / ksz;
          int t = int(k) - c * ksz;
          const int i2 = t % k2;
          t /= k2;
          const int i1 = t % k1, i0 = t / k1;
          const int u0 = pad_src_index(q0 * int(d.s[0]) + i0 * int(d.d[0]), in0, int(d.pad[0]), d.mode);
          const int u1 = pad_src_index(q1 * int(d.s[1]) + i1 * int(d.d[1]), in1, int(d.pad[1]), d.mode);
          const int u2 = pad_src_index(q2 * int(d.s[2]) + i2 * int(d.d[2]), in2, int(d.pad[2]), d.mode);
          v[i] = (u0 < 0 || u1 < 0 || u2 < 0) ? d.value : __ldg(xs + c * isz + (int64_t(u0) * in1 + u1) * in2 + u2);
        }
      }
      if constexpr (kLK) {
        if (!first) __syncthreads();   // the previous tile has been read
        first = false;
#pragma unroll
        for (int i = 0; i < 4; ++i) tile[tx][ty + 8 * i] = v[i];
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int64_t lw = l0 + ty + 8 * i, k = k0 + tx;
          if (lw < d.L && k < d.K) tf32_put(dst + (ns * d.L + lw) * ldp + k, tile[ty + 8 * i][tx], segments, lo_seg, seg_len);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int64_t k = k0 + ty + 8 * i;
          if (l_ok && k < d.K) tf32_put(dst + k * ldp + ns * d.L + l, v[i], segments, lo_seg, seg_len);
        }
      }
    }
  }
}

// acc = (first ? 0 : acc) + part[0] + part[1] + ... + part[splits - 1], in that order; on the last sample chunk
// dw = acc + beta * dw in dw's type (the finalize of the other engines)
template <typename T>
__global__ void __launch_bounds__(kThreads) tf32_dw_reduce(T* __restrict__ dw, float* __restrict__ acc,
                                                           const float* __restrict__ part, int64_t count, int splits,
                                                           int first, int last, float beta) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float v = first ? 0.f : acc[i];
  for (int s = 0; s < splits; ++s) v += part[s * count + i];
  if (!last) {
    acc[i] = v;
    return;
  }
  if (beta != 0.f) v += beta * nk_to_f32<T>(dw[i]);
  dw[i] = nk_from_f32<T>(v);
}

struct Scratch {   // stream-ordered temporaries released on scope exit
  nk_ctx* ctx;
  void* p[4] = {nullptr, nullptr, nullptr, nullptr};
  explicit Scratch(nk_ctx* c) : ctx(c) {}
  ~Scratch() {
    for (void* q : p)
      if (q) nk_free(ctx, q);
  }
  int alloc(int i, int64_t bytes) { return nk_alloc_uninit(ctx, size_t(bytes), &p[i]); }
  float* f(int i) const { return static_cast<float*>(p[i]); }
};

struct Mode {
  bool x3;
  int segments;
};

int begin(nk_ctx* ctx, const char* who, CgNdDims& d, Mode& m, int nsp, int64_t n, int64_t cin, const int64_t* in_sp,
          int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil, const int64_t* pad, int mode, float value) {
  conv_nd_geometry(d, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value);
  d.Kp = d.K, d.Lp = d.L;   // f32 column gradients stored densely (col2im_nd_kernel's row pitch)
  m.x3 = ctx->f32_conv == NK_F32_GEMM_TF32X3;
  m.segments = m.x3 ? 3 : 1;
  // one sample's image, columns and gradient in 32-bit indices along each gathered axis
  NK_REQUIRE(ctx, d.L < (int64_t(1) << 31) && d.K < (int64_t(1) << 31) &&
                  d.cin * d.in[0] * d.in[1] * d.in[2] < (int64_t(1) << 31),
             "%s: shape too large for the tf32 engine (K=%lld L=%lld)", who, (long long)d.K, (long long)d.L);
  return NK_OK;
}

int64_t chunk(const CgNdDims& d, int64_t per_sample_bytes) {
  int64_t c = kChunkBytes / (per_sample_bytes > 0 ? per_sample_bytes : 1);
  if (c < 1) c = 1;
  return c < d.n ? c : d.n;
}

int launch_gather(nk_ctx* ctx, bool lk, float* dst, const float* x, const CgNdDims& d, int64_t n0, int64_t nn, int64_t ldp,
                  int64_t seg_len, const Mode& m, int lo_seg) {
  const int64_t k_tiles = (d.K + 31) / 32;
  const dim3 grid(unsigned((d.L + 31) / 32), unsigned(k_tiles < 65535 ? k_tiles : 65535), unsigned(nn < 65535 ? nn : 65535)),
      block(32, 8);
  if (lk)
    tf32_im2col_kernel<true><<<grid, block, 0, ctx->stream>>>(dst, x, d, n0, nn, ldp, seg_len, m.segments, lo_seg);
  else
    tf32_im2col_kernel<false><<<grid, block, 0, ctx->stream>>>(dst, x, d, n0, nn, ldp, seg_len, m.segments, lo_seg);
  NK_LAUNCHED(ctx, lk ? "tf32_im2col_lk" : "tf32_im2col_kl");
  return NK_OK;
}

int conv_fwd(nk_ctx* ctx, float* y, const float* x, const float* w, const float* bias, int relu, const CgNdDims& d,
             const Mode& m) {
  const int64_t ldp = ceil4(m.segments * d.K);
  Scratch s(ctx);
  int rc = s.alloc(0, d.cout * ldp * 4);
  if (!rc) rc = nk_tf32_pack(ctx, w, d.K, false, d.cout, d.K, s.f(0), ldp, m.segments, 2);
  const int64_t cs = chunk(d, d.L * ldp * 4);
  if (!rc) rc = s.alloc(1, cs * d.L * ldp * 4);
  for (int64_t n0 = 0; !rc && n0 < d.n; n0 += cs) {
    const int64_t nn = d.n - n0 < cs ? d.n - n0 : cs;
    rc = launch_gather(ctx, true, s.f(1), x, d, n0, nn, ldp, d.K, m, 1);
    if (rc) break;
    NkTf32Gemm g;
    g.x3 = m.x3, g.M = d.cout, g.N = d.L, g.batch = nn;
    g.A = s.f(0), g.lda = ldp, g.a_rows = d.cout;
    g.B = s.f(1), g.ldb = ldp, g.b_rows = nn * d.L, g.b_bstride = d.L;
    g.kp = m.segments * d.K, g.k_len = g.kp;
    g.C = y + n0 * d.cout * d.L, g.ldc = d.L, g.c_bstride = d.cout * d.L;
    g.bias = bias, g.row_bias = 1, g.relu = relu;
    rc = nk_gemm_tf32_packed(ctx, g);
  }
  return rc;
}

int conv_dx(nk_ctx* ctx, float* dx, const float* gr, const float* w, const CgNdDims& d, const Mode& m,
            float beta) {
  const int64_t ldp = ceil4(m.segments * d.cout);
  Scratch s(ctx);
  int rc = s.alloc(0, d.K * ldp * 4);
  // W^T: element (k, o) at w[o * K + k]
  if (!rc) rc = nk_tf32_pack(ctx, w, d.K, true, d.K, d.cout, s.f(0), ldp, m.segments, 2);
  const int64_t cs = chunk(d, d.L * ldp * 4 + d.K * d.L * 4);
  if (!rc) rc = s.alloc(1, cs * d.L * ldp * 4);
  if (!rc) rc = s.alloc(2, cs * d.K * d.L * 4);
  for (int64_t n0 = 0; !rc && n0 < d.n; n0 += cs) {
    const int64_t nn = d.n - n0 < cs ? d.n - n0 : cs;
    // G[n]^T: element (l, o) at g[n][o * L + l]
    rc = nk_tf32_pack(ctx, gr + n0 * d.cout * d.L, d.L, true, d.L, d.cout, s.f(1), ldp, m.segments, 1, nn, d.cout * d.L,
                      d.L * ldp);
    if (rc) break;
    NkTf32Gemm g;
    g.x3 = m.x3, g.M = d.K, g.N = d.L, g.batch = nn;
    g.A = s.f(0), g.lda = ldp, g.a_rows = d.K;
    g.B = s.f(1), g.ldb = ldp, g.b_rows = nn * d.L, g.b_bstride = d.L;
    g.kp = m.segments * d.cout, g.k_len = g.kp;
    g.C = s.f(2), g.ldc = d.L, g.c_bstride = d.K * d.L;
    rc = nk_gemm_tf32_packed(ctx, g);
    if (rc) break;
    const int64_t items = nn * d.cin * d.in[0] * d.in[1] * d.in[2];
    int64_t blocks = (items + kThreads - 1) / kThreads;
    if (blocks > int64_t(ctx->sm_count) * 16) blocks = int64_t(ctx->sm_count) * 16;
    col2im_nd_kernel<float><<<int(blocks), kThreads, 0, ctx->stream>>>(dx, s.f(2), d, n0, nn, beta);
    NK_LAUNCHED(ctx, "col2im_nd");
  }
  return rc;
}

int conv_dw(nk_ctx* ctx, void* dwt, int dw_dtype, const float* gr, const float* x, const CgNdDims& d, const Mode& m,
            float beta) {
  const int64_t cs = chunk(d, (d.cout + d.K) * m.segments * d.L * 4);
  const int64_t ldp = ceil4(m.segments * cs * d.L);
  // the split of the reduction: about one wave of output tiles, each summing at least 8 k-blocks
  const int64_t tiles = (d.cout + 127) / 128 * ((d.K + nk_tf32_block_n(d.K, m.x3) - 1) / nk_tf32_block_n(d.K, m.x3));
  const int64_t kblocks_max = (m.segments * cs * d.L + 31) / 32;
  int64_t splits = (ctx->sm_count + tiles - 1) / tiles;
  if (splits > (kblocks_max + 7) / 8) splits = (kblocks_max + 7) / 8;
  if (splits < 1) splits = 1;
  const int64_t count = d.cout * d.K;
  Scratch s(ctx);
  int rc = s.alloc(0, d.cout * ldp * 4);
  if (!rc) rc = s.alloc(1, d.K * ldp * 4);
  if (!rc) rc = s.alloc(2, splits * count * 4);
  if (!rc && cs < d.n) rc = s.alloc(3, count * 4);
  for (int64_t n0 = 0; !rc && n0 < d.n; n0 += cs) {
    const int64_t nn = d.n - n0 < cs ? d.n - n0 : cs;
    const int64_t R = nn * d.L;
    // G as (Cout rows x (n, l)): sample n's (Cout x L) block at column n * L
    rc = nk_tf32_pack(ctx, gr + n0 * d.cout * d.L, d.L, false, d.cout, d.L, s.f(0), ldp, m.segments, 2, nn, d.cout * d.L,
                      d.L, R);
    if (!rc) rc = launch_gather(ctx, false, s.f(1), x, d, n0, nn, ldp, R, m, 1);
    if (rc) break;
    const int64_t kb = (m.segments * R + 31) / 32;
    const int64_t per = (kb + splits - 1) / splits;
    const int64_t used = (kb + per - 1) / per;
    NkTf32Gemm g;
    g.x3 = m.x3, g.M = d.cout, g.N = d.K, g.batch = used;
    g.A = s.f(0), g.lda = ldp, g.a_rows = d.cout;
    g.B = s.f(1), g.ldb = ldp, g.b_rows = d.K;
    g.kp = m.segments * R, g.k_len = per * 32, g.k_bstride = per * 32;
    g.C = s.f(2), g.ldc = d.K, g.c_bstride = count;
    rc = nk_gemm_tf32_packed(ctx, g);
    if (rc) break;
    const int first = n0 == 0, last = n0 + nn >= d.n;
    const unsigned fb = unsigned((count + kThreads - 1) / kThreads);
    if (dw_dtype == NK_BF16)
      tf32_dw_reduce<__nv_bfloat16><<<fb, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dwt, s.f(3), s.f(2), count, int(used),
                                                                      first, last, beta);
    else
      tf32_dw_reduce<float><<<fb, kThreads, 0, ctx->stream>>>((float*)dwt, s.f(3), s.f(2), count, int(used), first, last,
                                                              beta);
    NK_LAUNCHED(ctx, "tf32_dw_reduce");
  }
  return rc;
}

const char* kernel_name(const Mode& m, bool nd, int product) {
  static const char* names[2][2][3] = {
      {{"tf32_im2col_fwd", "tf32_im2col_dx", "tf32_im2col_dw"}, {"tf32_im2col_nd_fwd", "tf32_im2col_nd_dx", "tf32_im2col_nd_dw"}},
      {{"tf32x3_im2col_fwd", "tf32x3_im2col_dx", "tf32x3_im2col_dw"},
       {"tf32x3_im2col_nd_fwd", "tf32x3_im2col_nd_dx", "tf32x3_im2col_nd_dw"}}};
  return names[m.x3][nd][product];
}

}  // namespace

int nk_conv_tf32_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, int nsp, int64_t n,
                     int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                     const int64_t* pad, int mode, float value, bool nd) {
  CgNdDims d;
  Mode m;
  int rc = begin(ctx, "conv fwd (tf32)", d, m, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value);
  if (!rc) rc = conv_fwd(ctx, (float*)y, (const float*)x, (const float*)w, (const float*)bias, relu, d, m);
  if (!rc) ctx->last_conv_kernel = kernel_name(m, nd, 0);
  return rc;
}

int nk_conv_tf32_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                           const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                           const int64_t* pad, int mode, float beta, bool nd) {
  CgNdDims d;
  Mode m;
  int rc = begin(ctx, "conv dX (tf32)", d, m, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, 0.f);
  if (!rc) rc = conv_dx(ctx, (float*)dx, (const float*)g, (const float*)w, d, m, beta);
  if (!rc) ctx->last_conv_kernel = kernel_name(m, nd, 1);
  return rc;
}

int nk_conv_tf32_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp, int64_t n,
                            int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s,
                            const int64_t* dil, const int64_t* pad, int mode, float value, float beta, bool nd) {
  CgNdDims d;
  Mode m;
  int rc = begin(ctx, "conv dW (tf32)", d, m, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value);
  if (!rc) rc = conv_dw(ctx, dwt, dw_dtype, (const float*)g, (const float*)x, d, m, beta);
  if (!rc) ctx->last_conv_kernel = kernel_name(m, nd, 2);
  return rc;
}
