// General 2-D convolution on the tensor cores: im2col + batched wgmma GEMM (bf16, groups = 1, any stride / dilation /
// channel count).  This is the reference's own formulation -- convolution/mod.rs:85-123 (out[n] = Wflat . cols[n]^T),
// :146-189 (dX = col2im(G[n]^T . Wflat)), :191-226 (dW += G[n] . cols[n]) -- with the GEMMs on wgmma instead of one
// sgemm per sample: ONE batched launch (3-D TMA maps over (k, row, sample)) per product, and the kernel gradient as a
// split reduction over the samples inside the GEMM's k loop.  It takes every bf16, groups = 1 shape with
// K = Cin*kh*kw >= 9 (config 3's thin 3 -> 64 layer as well as config 5's 32 -> 64 one); the rest falls through to the
// CUDA-core kernels.  Rows of Ho*Wo pixels are stored Lp = ceil8(Ho*Wo) apart (TMA row pitch: a multiple of 16 bytes);
// the tensor maps stop at Ho*Wo, so the pad columns are never read as operands (TMA zero-fills them) nor written.
//   colsT[n][k][l]  k = (c, i, j) as in the reference (utils.rs:332-353), l = output pixel: the TRANSPOSE of the
//   reference's (l, k) column matrix, so that a row is a shifted copy of image rows (im2col / col2im move contiguous
//   runs) and is the MN-major wgmma operand as it lies; the buffer lives in HBM for the duration of the call (sample
//   chunks of <= 4 GB).  The (Cout, K) kernel is copied once into rows of Kp = ceil8(K) elements (TMA row pitch).
// Compute bound for Cin >= 16 (K >= 144); the column buffer adds 2 x |cols| of HBM traffic.
//
// The same three GEMMs serve the 1-D / 3-D convolution LAYERS (nk_conv_layer_nd_*, nk_conv_nd.cu): x (N, Cin, s0[, s1,
// s2]), k = (c, i0, i1, i2), l = output position in row-major order, and the layer's padding applied inside the gather
// instead of through a padded copy of x: column element (c, i, p) reads padded coordinate u' = p*s + i*d along each axis,
// mapped to a source index by the padding mode exactly as nk_padnd_fwd maps it (a bit-exact copy or the fill value).
// col2im writes only the interior dx positions, each the f32 sum of the taps that read padded coordinate u + pad: the
// reference's pad backward, the interior slice for every mode (pad/mod.rs:157-182).
#include "nk_conv_im2col.cuh"

int nk_gemm_wgmma_batched(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                            int64_t lda, int64_t strideA, const void* B, int64_t ldb, int64_t strideB, void* C, int64_t ldc,
                            int64_t strideC, int64_t batch, int c_dtype, const void* row_bias, int bias_dtype, int relu,
                            int reduce);

namespace {

constexpr int kThreads = 256;
constexpr int64_t kChunkBytes = int64_t(4) << 30;

struct CgDims {
  int64_t n, cin, h, w, cout, kh, kw, sh, sw, dh, dw, ho, wo, K, Kp, L, Lp;
};

// eight consecutive bf16 source elements x[off .. off+7] (2-byte aligned): aligned 4-byte loads + a funnel shift when the
// run starts on an odd element
__device__ __forceinline__ uint4 load_run8(const __nv_bfloat16* __restrict__ x, int64_t off, int64_t x_elems) {
  const uint32_t* xw = reinterpret_cast<const uint32_t*>(x);
  if ((off & 1) == 0) {
    const uint32_t* s = xw + (off >> 1);
    return make_uint4(__ldg(s), __ldg(s + 1), __ldg(s + 2), __ldg(s + 3));
  }
  const uint32_t* s = xw + ((off - 1) >> 1);
  const uint32_t w0 = __ldg(s), w1 = __ldg(s + 1), w2 = __ldg(s + 2), w3 = __ldg(s + 3);
  // the fifth word holds source element off+7 in its low half; its high half may lie past the end of x
  const uint32_t w4 = (off + 9 <= x_elems) ? __ldg(s + 4) : uint32_t(reinterpret_cast<const unsigned short*>(x)[off + 7]);
  return make_uint4(__funnelshift_r(w0, w1, 16), __funnelshift_r(w1, w2, 16), __funnelshift_r(w2, w3, 16),
                    __funnelshift_r(w3, w4, 16));
}

// colsT[ns][k][l0 .. l0+7]: one thread per 16-byte vector of eight consecutive output pixels of one im2col row (rows Lp
// apart; the pixels l >= L of the last vector are written as zeros)
// k = (c, i, j).  With a unit horizontal stride the eight values are a contiguous (2-byte aligned) run of the image row:
// aligned 4-byte loads + a funnel shift when the run starts on an odd element; every store is a full 16-byte vector and a
// warp writes 512 contiguous bytes, so the kernel runs at copy speed (the first version gathered element by element into
// a k-contiguous buffer: 6.4 ms for config 5's 2.35 GB).
__global__ void __launch_bounds__(kThreads) im2col_kernel(__nv_bfloat16* __restrict__ cols, const __nv_bfloat16* __restrict__ x,
                                                          CgDims d, int64_t n0, int64_t nn) {
  const uint32_t lv_n = uint32_t(d.Lp / 8), L = uint32_t(d.L), K = uint32_t(d.K), wo = uint32_t(d.wo), kw = uint32_t(d.kw), kh = uint32_t(d.kh);
  const int64_t total = nn * int64_t(K) * lv_n;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t x_elems = d.n * d.cin * d.h * d.w;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const uint32_t row = uint32_t(idx / lv_n);          // (ns, k)
    const uint32_t lv = uint32_t(idx - int64_t(row) * lv_n);
    const uint32_t ns = row / K, k = row - ns * K;
    const uint32_t j = k % kw, ci = k / kw, i = ci % kh, c = ci / kh;
    const uint32_t l0 = lv * 8, p = l0 / wo, q = l0 - p * wo;
    const int64_t plane = ((n0 + ns) * d.cin + c) * d.h;
    uint4 out;
    if (d.sw == 1 && q + 8 <= wo && l0 + 8 <= L) {
      // first of 8 consecutive source elements
      out = load_run8(x, (plane + p * d.sh + i * d.dh) * d.w + q + j * d.dw, x_elems);
    } else {
      __align__(16) unsigned short e[8];
      const unsigned short* xs = reinterpret_cast<const unsigned short*>(x);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const uint32_t l = l0 + t, pp = l / wo, qq = l - pp * wo;
        e[t] = l < L ? __ldg(xs + (plane + pp * d.sh + i * d.dh) * d.w + qq * d.sw + j * d.dw) : (unsigned short)0;
      }
      out = *reinterpret_cast<const uint4*>(e);
    }
    reinterpret_cast<uint4*>(cols)[idx] = out;
  }
}

// dx[n,c,u,v] = beta*dx + sum_{i,j : u = p*sh + i*dh, v = q*sw + j*dw} dcolsT[ns][(c,i,j)][p*wo+q]
// one thread per dx element; for a fixed tap the reads of a warp are consecutive pixels of one dcolsT row (coalesced).
// The column gradients are f32: the up to kh*kw terms of a dx element are summed before the one rounding to bf16.
__global__ void __launch_bounds__(kThreads) col2im_kernel(__nv_bfloat16* __restrict__ dx, const float* __restrict__ dcols,
                                                          CgDims d, int64_t n0, int64_t nn, float beta) {
  const int64_t total = nn * d.cin * d.h * d.w;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int w = int(d.w), h = int(d.h), cin = int(d.cin), kh = int(d.kh), kw = int(d.kw), sh = int(d.sh), sw = int(d.sw),
            dh = int(d.dh), dw = int(d.dw), ho = int(d.ho), wo = int(d.wo);
  const uint32_t hw = uint32_t(h) * uint32_t(w);
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const uint32_t pl = uint32_t(idx / hw);             // (ns, c)
    const uint32_t uv = uint32_t(idx - int64_t(pl) * hw);
    const int u = int(uv / uint32_t(w)), v = int(uv) - u * w;
    const uint32_t ns = pl / uint32_t(cin), c = pl - ns * uint32_t(cin);
    const float* dc = dcols + (int64_t(ns) * d.K + int64_t(c) * kh * kw) * d.Lp;
    float acc = 0.f;
    for (int i = 0; i < kh; ++i) {
      const int pu = u - i * dh;
      if (pu < 0) break;
      const int p = pu / sh;
      if (p * sh != pu || p >= ho) continue;
      for (int j = 0; j < kw; ++j) {
        const int qv = v - j * dw;
        if (qv < 0) break;
        const int q = qv / sw;
        if (q * sw != qv || q >= wo) continue;
        acc += dc[int64_t(i * kw + j) * d.Lp + p * wo + q];
      }
    }
    __nv_bfloat16* o = dx + n0 * d.cin * d.h * d.w + idx;
    if (beta != 0.f) acc += beta * __bfloat162float(*o);
    *o = __float2bfloat16_rn(acc);
  }
}

// ---- unit stride / dilation: one block per (sample, channel) plane.  The kh*kw rows (c, i, j) of a channel are CONSECUTIVE
// rows of colsT, i.e. one contiguous block of kh*kw*L elements, and all of them are shifted views of ONE image plane:
// stage the x plane (h*w) in shared memory, then write the kh*kw*L elements out with full 16-byte vectors.
constexpr int kPlaneThreads = 256;

__global__ void __launch_bounds__(kPlaneThreads) im2col_plane_kernel(__nv_bfloat16* __restrict__ cols, const __nv_bfloat16* __restrict__ x,
                                                                     CgDims d, int64_t n0, int64_t nn) {
  extern __shared__ __align__(16) unsigned short plane[];   // h*w (+ slack) input pixels
  const int hw = int(d.h * d.w), kk = int(d.kh * d.kw), L = int(d.L), wo = int(d.wo), w = int(d.w), kw = int(d.kw);
  const int lv_n = int(d.Lp / 8);
  const int64_t planes = nn * d.cin;
  for (int64_t pl = blockIdx.x; pl < planes; pl += gridDim.x) {
    const int64_t ns = pl / d.cin, c = pl - ns * d.cin;
    const unsigned short* src = reinterpret_cast<const unsigned short*>(x) + ((n0 + ns) * d.cin + c) * hw;
    __syncthreads();
    for (int i = threadIdx.x; i < hw; i += kPlaneThreads) plane[i] = __ldg(src + i);
    __syncthreads();
    uint4* dst = reinterpret_cast<uint4*>(cols + (ns * d.K + c * kk) * d.Lp);
    for (int idx = threadIdx.x; idx < kk * lv_n; idx += kPlaneThreads) {
      const int t = idx / lv_n, lv = idx - t * lv_n;
      const int i = t / kw, j = t - i * kw;
      const int l0 = lv * 8, p = l0 / wo, q = l0 - p * wo;
      __align__(16) unsigned short e[8];
      if (q + 8 <= wo && l0 + 8 <= L) {
        const unsigned short* s0 = plane + (p + i) * w + q + j;
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = s0[k];
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int l = l0 + k, pp = l / wo, qq = l - pp * wo;
          e[k] = l < L ? plane[(pp + i) * w + qq + j] : (unsigned short)0;
        }
      }
      dst[idx] = *reinterpret_cast<const uint4*>(e);
    }
  }
}

// (Cout, Kp) bf16 copy of the (Cout, K) kernel, zero padded (the GEMM operand rows must be 16-byte multiples)
__global__ void __launch_bounds__(kThreads) pad_kernel_rows(__nv_bfloat16* __restrict__ wp, const __nv_bfloat16* __restrict__ w,
                                                            int64_t cout, int64_t K, int64_t Kp) {
  const int64_t total = cout * Kp;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += int64_t(gridDim.x) * blockDim.x) {
    const int64_t k = idx % Kp, o = idx / Kp;
    wp[idx] = k < K ? w[o * K + k] : __float2bfloat16_rn(0.f);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) finalize_dw_padded(T* __restrict__ dw, const float* __restrict__ scratch, int64_t cout,
                                                               int64_t K, int64_t Kp, float beta) {
  const int64_t total = cout * K;
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int64_t k = idx % K, o = idx / K;
  float v = scratch[o * Kp + k];
  if (beta != 0.f) v += beta * nk_to_f32<T>(dw[idx]);
  dw[idx] = nk_from_f32<T>(v);
}

// ---- 1-D / 3-D layers with the padding folded into the gather (pad_src_index: nk_conv_im2col.cuh)
// colsT[ns][(c, i0, i1, i2)][l0 .. l0+7] as im2col_kernel, through the padding map.  A vector of eight outputs along one
// output row (unit stride on the last axis) reads one source row: the fill value when the padding puts that row outside x
// (constant mode), else a contiguous run (load_run8) when the eight columns are interior; only runs that touch the border
// along the last axis, non-unit last-axis strides and vectors that wrap a row are gathered element by element.
__global__ void __launch_bounds__(kThreads) im2col_nd_kernel(__nv_bfloat16* __restrict__ cols, const __nv_bfloat16* __restrict__ x,
                                                             CgNdDims d, int64_t n0, int64_t nn) {
  const uint32_t lv_n = uint32_t(d.Lp / 8), L = uint32_t(d.L), K = uint32_t(d.K);
  const int in0 = int(d.in[0]), in1 = int(d.in[1]), in2 = int(d.in[2]), k1 = int(d.k[1]), k2 = int(d.k[2]);
  const int o1 = int(d.out[1]), o2 = int(d.out[2]), ksz = int(d.k[0]) * k1 * k2;
  const int s0 = int(d.s[0]), s1 = int(d.s[1]), s2 = int(d.s[2]), d0 = int(d.d[0]), d1 = int(d.d[1]), d2 = int(d.d[2]);
  const int p0 = int(d.pad[0]), p1 = int(d.pad[1]), p2 = int(d.pad[2]), mode = d.mode;
  const int64_t isz = int64_t(in0) * in1 * in2;
  const int64_t total = nn * int64_t(K) * lv_n;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t x_elems = d.n * d.cin * isz;
  const unsigned short fill = __bfloat16_as_ushort(__float2bfloat16_rn(d.value));
  const unsigned short* xs = reinterpret_cast<const unsigned short*>(x);
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const uint32_t row = uint32_t(idx / lv_n);          // (ns, k)
    const uint32_t lv = uint32_t(idx - int64_t(row) * lv_n);
    const uint32_t ns = row / K, k = row - ns * K;
    const int c = int(k) / ksz;
    int t = int(k) - c * ksz;
    const int i2 = t % k2;
    t /= k2;
    const int i1 = t % k1, i0 = t / k1;
    const int64_t plane = ((n0 + ns) * d.cin + c) * isz;
    const uint32_t l0 = lv * 8;
    const int q = int(l0 % uint32_t(o2)), r = int(l0 / uint32_t(o2));
    uint4 out;
    if (s2 == 1 && q + 8 <= o2 && l0 + 8 <= L) {
      const int r0 = pad_src_index((r / o1) * s0 + i0 * d0, in0, p0, mode);
      const int r1 = pad_src_index((r % o1) * s1 + i1 * d1, in1, p1, mode);
      const int u2 = q + i2 * d2 - p2;                  // source column of the first output
      if (r0 < 0 || r1 < 0) {
        const uint32_t f = uint32_t(fill) * 0x10001u;
        out = make_uint4(f, f, f, f);
      } else if (u2 >= 0 && u2 + 8 <= in2) {
        out = load_run8(x, plane + (int64_t(r0) * in1 + r1) * in2 + u2, x_elems);
      } else {
        __align__(16) unsigned short e[8];
        const unsigned short* src = xs + plane + (int64_t(r0) * in1 + r1) * in2;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int u = pad_src_index(q + j + i2 * d2, in2, p2, mode);
          e[j] = u < 0 ? fill : __ldg(src + u);
        }
        out = *reinterpret_cast<const uint4*>(e);
      }
    } else {
      __align__(16) unsigned short e[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t l = l0 + j;
        unsigned short v = 0;
        if (l < L) {
          const int c2 = int(l % uint32_t(o2)), rr = int(l / uint32_t(o2));
          const int u0 = pad_src_index((rr / o1) * s0 + i0 * d0, in0, p0, mode);
          const int u1 = pad_src_index((rr % o1) * s1 + i1 * d1, in1, p1, mode);
          const int u2 = pad_src_index(c2 * s2 + i2 * d2, in2, p2, mode);
          v = (u0 < 0 || u1 < 0 || u2 < 0) ? fill : __ldg(xs + plane + (int64_t(u0) * in1 + u1) * in2 + u2);
        }
        e[j] = v;
      }
      out = *reinterpret_cast<const uint4*>(e);
    }
    reinterpret_cast<uint4*>(cols)[idx] = out;
  }
}

inline int cg_blocks(nk_ctx* ctx, int64_t items) {
  int64_t b = (items + kThreads - 1) / kThreads;
  const int64_t cap = int64_t(ctx->sm_count) * 16;
  if (b > cap) b = cap;
  return int(b < 1 ? 1 : b);
}

bool make_dims(CgDims& d, int64_t n, int64_t cin, int64_t h, int64_t w, int64_t cout, int64_t kh, int64_t kw, int64_t sh,
               int64_t sw, int64_t dh, int64_t dw) {
  d = CgDims{n, cin, h, w, cout, kh, kw, sh, sw, dh, dw, 0, 0, 0, 0, 0, 0};
  d.ho = (h - dh * (kh - 1) - 1) / sh + 1;
  d.wo = (w - dw * (kw - 1) - 1) / sw + 1;
  d.K = cin * kh * kw;
  d.Kp = (d.K + 7) & ~int64_t(7);
  d.L = d.ho * d.wo;
  d.Lp = (d.L + 7) & ~int64_t(7);
  // TMA: every leading dimension / batch stride a multiple of 8 elements; a useful amount of work per GEMM tile
  return n > 0 && d.L > 0 && d.Kp >= 16 && d.Lp * d.Kp < (int64_t(1) << 31);
}

struct Scratch {   // stream-ordered temporaries released on scope exit
  nk_ctx* ctx;
  void* p[3] = {nullptr, nullptr, nullptr};
  explicit Scratch(nk_ctx* c) : ctx(c) {}
  ~Scratch() {
    for (void* q : p)
      if (q) nk_free(ctx, q);
  }
};

inline bool unit_steps(const CgDims& d) { return d.sh == 1 && d.sw == 1 && d.dh == 1 && d.dw == 1; }
inline int plane_blocks(nk_ctx* ctx, int64_t planes) {
  const int64_t cap = int64_t(ctx->sm_count) * 8;
  return int(planes < cap ? planes : cap);
}

int launch_im2col(nk_ctx* ctx, __nv_bfloat16* cols, const __nv_bfloat16* x, const CgDims& d, int64_t n0, int64_t nn) {
  const size_t smem = size_t(d.h * d.w + 8) * 2;
  if (unit_steps(d) && smem <= 48 * 1024) {
    im2col_plane_kernel<<<plane_blocks(ctx, nn * d.cin), kPlaneThreads, smem, ctx->stream>>>(cols, x, d, n0, nn);
  } else {
    im2col_kernel<<<cg_blocks(ctx, nn * d.K * (d.Lp / 8)), kThreads, 0, ctx->stream>>>(cols, x, d, n0, nn);
  }
  NK_LAUNCHED(ctx, "im2col");
  return NK_OK;
}

int launch_col2im(nk_ctx* ctx, __nv_bfloat16* dx, const float* dcols, const CgDims& d, int64_t n0, int64_t nn, float beta) {
  col2im_kernel<<<cg_blocks(ctx, nn * d.cin * d.h * d.w), kThreads, 0, ctx->stream>>>(dx, dcols, d, n0, nn, beta);
  NK_LAUNCHED(ctx, "col2im");
  return NK_OK;
}

// the 1-D / 3-D layer's gather / scatter (one launch per sample chunk)
int launch_im2col(nk_ctx* ctx, __nv_bfloat16* cols, const __nv_bfloat16* x, const CgNdDims& d, int64_t n0, int64_t nn) {
  im2col_nd_kernel<<<cg_blocks(ctx, nn * d.K * (d.Lp / 8)), kThreads, 0, ctx->stream>>>(cols, x, d, n0, nn);
  NK_LAUNCHED(ctx, "im2col_nd");
  return NK_OK;
}
int launch_col2im(nk_ctx* ctx, __nv_bfloat16* dx, const float* dcols, const CgNdDims& d, int64_t n0, int64_t nn, float beta) {
  col2im_nd_kernel<__nv_bfloat16><<<cg_blocks(ctx, nn * d.cin * d.in[0] * d.in[1] * d.in[2]), kThreads, 0, ctx->stream>>>(
      dx, dcols, d, n0, nn, beta);
  NK_LAUNCHED(ctx, "col2im_nd");
  return NK_OK;
}

// the helpers and drivers below read only the GEMM geometry (n, cout, K, Kp, L, Lp) of CgDims / CgNdDims
template <class D>
int64_t chunk_samples(const D& d, int64_t elem_bytes = 2) {
  int64_t per = d.Lp * d.Kp * elem_bytes;
  int64_t c = kChunkBytes / per;
  if (c < 1) c = 1;
  return c < d.n ? c : d.n;
}

// The output gradient as a GEMM operand: TMA needs its rows of L pixels 16-byte aligned, i.e. L % 8 == 0 and an aligned
// base.  Otherwise each sample chunk is first copied into rows Lp apart (slot `slot` of the scratch, cs samples).
template <class D>
int g_rows_scratch(nk_ctx* ctx, Scratch& s, int slot, const D& d, const void* g, int64_t cs, int64_t* ldg) {
  const bool copy = d.Lp != d.L || (reinterpret_cast<uintptr_t>(g) & 15);
  *ldg = copy ? d.Lp : d.L;
  return copy ? nk_alloc_uninit(ctx, size_t(cs * d.cout * d.Lp * 2), &s.p[slot]) : NK_OK;
}
template <class D>
int g_rows(nk_ctx* ctx, void* copy, const D& d, const void* g, int64_t n0, int64_t nn, const __nv_bfloat16** out) {
  const __nv_bfloat16* gn = static_cast<const __nv_bfloat16*>(g) + n0 * d.cout * d.L;
  *out = gn;
  if (d.Lp == d.L && (reinterpret_cast<uintptr_t>(g) & 15) == 0) return NK_OK;
  pad_kernel_rows<<<cg_blocks(ctx, nn * d.cout * d.Lp), kThreads, 0, ctx->stream>>>((__nv_bfloat16*)copy, gn, nn * d.cout, d.L,
                                                                                     d.Lp);
  NK_LAUNCHED(ctx, "conv_pad_gradient_rows");
  *out = static_cast<const __nv_bfloat16*>(copy);
  return NK_OK;
}

// ---- the three products, shared by the 2-D entry points and the 1-D / 3-D layers (launch_im2col / launch_col2im are
// overloaded on the dims type)
template <class D>
int gemm_conv_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, const D& d) {
  const int64_t n = d.n, cout = d.cout;
  Scratch s(ctx);
  int rc = nk_alloc_uninit(ctx, size_t(cout * d.Kp * 2), &s.p[0]);
  if (rc) return rc;
  pad_kernel_rows<<<cg_blocks(ctx, cout * d.Kp), kThreads, 0, ctx->stream>>>((__nv_bfloat16*)s.p[0], (const __nv_bfloat16*)w, cout, d.K, d.Kp);
  NK_LAUNCHED(ctx, "conv_pad_kernel");
  const int64_t cs = chunk_samples(d);
  rc = nk_alloc_uninit(ctx, size_t(cs * d.Lp * d.Kp * 2), &s.p[1]);
  if (rc) return rc;
  for (int64_t n0 = 0; n0 < n; n0 += cs) {
    const int64_t nn = n - n0 < cs ? n - n0 : cs;
    rc = launch_im2col(ctx, (__nv_bfloat16*)s.p[1], (const __nv_bfloat16*)x, d, n0, nn);
    if (rc) return rc;
    // y[n] (Cout x L) = Wp (Cout x K) . colsT[n] (K x L) : NN, A shared by every sample (TMA zero-fills k >= K)
    rc = nk_gemm_wgmma_batched(ctx, 0, 0, cout, d.L, d.K, 1.f, s.p[0], d.Kp, 0, s.p[1], d.Lp, d.K * d.Lp,
                                 static_cast<__nv_bfloat16*>(y) + n0 * cout * d.L, d.L, cout * d.L, nn, NK_BF16, bias, NK_BF16,
                                 relu, 0);
    if (rc) return rc;
  }
  return NK_OK;
}

template <class D>
int gemm_conv_dx(nk_ctx* ctx, void* dx, const void* g, const void* w, const D& d, float beta) {
  const int64_t n = d.n, cout = d.cout;
  Scratch s(ctx);
  int rc = nk_alloc_uninit(ctx, size_t(cout * d.Kp * 2), &s.p[0]);
  if (rc) return rc;
  pad_kernel_rows<<<cg_blocks(ctx, cout * d.Kp), kThreads, 0, ctx->stream>>>((__nv_bfloat16*)s.p[0], (const __nv_bfloat16*)w, cout, d.K, d.Kp);
  NK_LAUNCHED(ctx, "conv_pad_kernel");
  const int64_t cs = chunk_samples(d, 4);
  rc = nk_alloc_uninit(ctx, size_t(cs * d.Lp * d.Kp * 4), &s.p[1]);
  if (rc) return rc;
  int64_t ldg;
  rc = g_rows_scratch(ctx, s, 2, d, g, cs, &ldg);
  if (rc) return rc;
  for (int64_t n0 = 0; n0 < n; n0 += cs) {
    const int64_t nn = n - n0 < cs ? n - n0 : cs;
    const __nv_bfloat16* gn;
    rc = g_rows(ctx, s.p[2], d, g, n0, nn, &gn);
    if (rc) return rc;
    // dcolsT[n] (K x L, f32) = Wp^T (K x Cout) . G[n] (Cout x L) : TN (A = Wp stored (Cout, K), shared), B = G[n]
    rc = nk_gemm_wgmma_batched(ctx, 1, 0, d.K, d.L, cout, 1.f, s.p[0], d.Kp, 0, gn, ldg, cout * ldg, s.p[1], d.Lp, d.K * d.Lp,
                               nn, NK_F32, nullptr, NK_BF16, 0, 0);
    if (rc) return rc;
    rc = launch_col2im(ctx, (__nv_bfloat16*)dx, (const float*)s.p[1], d, n0, nn, beta);
    if (rc) return rc;
  }
  return NK_OK;
}

template <class D>
int gemm_conv_dw(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, const D& d, float beta) {
  const int64_t n = d.n, cout = d.cout;
  Scratch s(ctx);
  const int64_t cs = chunk_samples(d);
  int rc = nk_alloc_uninit(ctx, size_t(cs * d.Lp * d.Kp * 2), &s.p[1]);
  if (rc) return rc;
  int64_t ldg;
  rc = g_rows_scratch(ctx, s, 0, d, g, cs, &ldg);
  if (rc) return rc;
  rc = nk_alloc(ctx, size_t(cout * d.Kp * 4), &s.p[2]);   // f32 accumulator of the split reduction, zero filled
  if (rc) return rc;
  for (int64_t n0 = 0; n0 < n; n0 += cs) {
    const int64_t nn = n - n0 < cs ? n - n0 : cs;
    rc = launch_im2col(ctx, (__nv_bfloat16*)s.p[1], (const __nv_bfloat16*)x, d, n0, nn);
    if (rc) return rc;
    const __nv_bfloat16* gn;
    rc = g_rows(ctx, s.p[0], d, g, n0, nn, &gn);
    if (rc) return rc;
    // acc (Cout x K) += sum_n G[n] (Cout x L) . colsT[n]^T (L x K) : NT, reduced over the samples inside the k loop
    rc = nk_gemm_wgmma_batched(ctx, 0, 1, cout, d.K, d.L, 1.f, gn, ldg, cout * ldg, s.p[1], d.Lp, d.K * d.Lp, s.p[2], d.Kp, 0,
                               nn, NK_F32, nullptr, NK_F32, 0, 1);
    if (rc) return rc;
  }
  const int fb = int((cout * d.K + kThreads - 1) / kThreads);
  if (dw_dtype == NK_BF16)
    finalize_dw_padded<__nv_bfloat16><<<fb, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dwt, (const float*)s.p[2], cout, d.K, d.Kp, beta);
  else
    finalize_dw_padded<float><<<fb, kThreads, 0, ctx->stream>>>((float*)dwt, (const float*)s.p[2], cout, d.K, d.Kp, beta);
  NK_LAUNCHED(ctx, "conv_dw_finalize_padded");
  return NK_OK;
}

// the layer's geometry (conv_nd_geometry), and the 2-D engine's applicability rules (make_dims)
bool make_nd_dims(CgNdDims& d, int nsp, int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k,
                  const int64_t* s, const int64_t* dil, const int64_t* pad, int mode, float value) {
  conv_nd_geometry(d, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value);
  d.Kp = (d.K + 7) & ~int64_t(7);
  d.Lp = (d.L + 7) & ~int64_t(7);
  return n > 0 && d.L > 0 && d.Kp >= 16 && d.Lp * d.Kp < (int64_t(1) << 31);
}

}  // namespace

// all three return NK_ERR_UNSUPPORTED (last_error untouched) when the shape is outside this engine

int nk_conv_gemm_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, int64_t n, int64_t cin,
                     int64_t h, int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw) {
  CgDims d;
  if (!make_dims(d, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(x) & 3) || cout < 8) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_fwd(ctx, y, x, w, bias, relu, d);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_gemm_fwd";
  return rc;
}

int nk_conv_gemm_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int64_t n, int64_t cin, int64_t h, int64_t wd,
                           int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw, float beta) {
  CgDims d;
  if (!make_dims(d, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if (cout % 8 != 0) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_dx(ctx, dx, g, w, d, beta);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_gemm_dx";
  return rc;
}

int nk_conv_gemm_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int64_t n, int64_t cin, int64_t h,
                            int64_t wd, int64_t cout, int64_t kh, int64_t kw, int64_t sh, int64_t sw, int64_t dh, int64_t dw,
                            float beta) {
  CgDims d;
  if (!make_dims(d, n, cin, h, wd, cout, kh, kw, sh, sw, dh, dw) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(x) & 3) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_dw(ctx, dwt, dw_dtype, g, x, d, beta);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_gemm_dw";
  return rc;
}

// The 1-D / 3-D layer (nsp sample dims, groups = 1, padding `pad` with nk_pad_mode `mode`): arguments validated by the
// caller (nk_conv_layer_nd_*, nk_conv_nd.cu); same applicability and return protocol as the 2-D entry points above.
int nk_conv_gemm_nd_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int nsp, int64_t n, int64_t cin,
                        const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                        const int64_t* pad, int mode, float value) {
  CgNdDims d;
  if (!make_nd_dims(d, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(x) & 3) || cout < 8) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_fwd(ctx, y, x, w, bias, 0, d);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_nd_fwd";
  return rc;
}

int nk_conv_gemm_nd_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                              const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                              const int64_t* pad, int mode, float beta) {
  CgNdDims d;
  if (!make_nd_dims(d, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, 0.f) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if (cout % 8 != 0) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_dx(ctx, dx, g, w, d, beta);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_nd_dx";
  return rc;
}

int nk_conv_gemm_nd_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp, int64_t n,
                               int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s,
                               const int64_t* dil, const int64_t* pad, int mode, float value, float beta) {
  CgNdDims d;
  if (!make_nd_dims(d, nsp, n, cin, in_sp, cout, k, s, dil, pad, mode, value) || !ctx->encode_tiled) return NK_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(x) & 3) return NK_ERR_UNSUPPORTED;
  const int rc = gemm_conv_dw(ctx, dwt, dw_dtype, g, x, d, beta);
  if (rc == NK_OK) ctx->last_conv_kernel = "wgmma_im2col_nd_dw";
  return rc;
}
