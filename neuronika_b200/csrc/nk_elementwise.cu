// HBM-bound elementwise / broadcast / reduction kernels of the hot path:
//   fill, cast, broadcast add + un-broadcast (addition/mod.rs:39-135, utils.rs:97-192),
//   ReLU (relu/mod.rs:29-79), MSE / NLL / sum / mean (squared_error/mod.rs:46-122,
//   nll/mod.rs:42-133, sum/mod.rs, mean/mod.rs), constant pad (pad/mod.rs:97-182).
// All kernels: 128-bit vector loads/stores when pointers are 16-byte aligned, grid sized to a
// multiple of the SM count, warp-shuffle reductions, f32 arithmetic whatever the storage type.
#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;

inline int ew_blocks(nk_ctx* ctx, size_t work_items) {
  size_t b = (work_items + kThreads - 1) / kThreads;
  size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// out[i] = (RMW ? beta*out[i] : 0) + op(in0[i], in1[i], in2[i])
template <typename T, int NIN, bool RMW, bool VEC, typename Op>
__global__ void __launch_bounds__(kThreads) ew_kernel(T* __restrict__ out, const T* __restrict__ in0,
                                                      const T* __restrict__ in1, const T* __restrict__ in2,
                                                      size_t n, float beta, Op op) {
  const size_t tid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  size_t done = 0;
  if (VEC) {
    constexpr int V = NkVec<T>::N;
    const size_t nvec = n / V;
    for (size_t v = tid; v < nvec; v += stride) {
      NkVec<T> a, b, c, o;
      if (NIN > 0) a.load(in0 + v * V);
      if (NIN > 1) b.load(in1 + v * V);
      if (NIN > 2) c.load(in2 + v * V);
      if (RMW) o.load(out + v * V);
#pragma unroll
      for (int i = 0; i < V; ++i) {
        float r = op(NIN > 0 ? a.get(i) : 0.f, NIN > 1 ? b.get(i) : 0.f, NIN > 2 ? c.get(i) : 0.f);
        if (RMW) r = beta * o.get(i) + r;
        o.set(i, r);
      }
      o.store(out + v * V);
    }
    done = nvec * V;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    float r = op(NIN > 0 ? nk_to_f32<T>(in0[i]) : 0.f, NIN > 1 ? nk_to_f32<T>(in1[i]) : 0.f,
                 NIN > 2 ? nk_to_f32<T>(in2[i]) : 0.f);
    if (RMW) r = beta * nk_to_f32<T>(out[i]) + r;
    out[i] = nk_from_f32<T>(r);
  }
}

template <typename T, int NIN, typename Op>
int launch_ew(nk_ctx* ctx, const char* name, void* out, const void* in0, const void* in1, const void* in2,
              size_t n, float beta, Op op) {
  if (n == 0) return NK_OK;
  bool vec = aligned16(out) && (NIN < 1 || aligned16(in0)) && (NIN < 2 || aligned16(in1)) &&
             (NIN < 3 || aligned16(in2));
  int blocks = ew_blocks(ctx, vec ? n / NkVec<T>::N + 1 : n);
  T* o = static_cast<T*>(out);
  const T* a = static_cast<const T*>(in0);
  const T* b = static_cast<const T*>(in1);
  const T* c = static_cast<const T*>(in2);
  if (beta != 0.f) {
    if (vec)
      ew_kernel<T, NIN, true, true, Op><<<blocks, kThreads, 0, ctx->stream>>>(o, a, b, c, n, beta, op);
    else
      ew_kernel<T, NIN, true, false, Op><<<blocks, kThreads, 0, ctx->stream>>>(o, a, b, c, n, beta, op);
  } else {
    if (vec)
      ew_kernel<T, NIN, false, true, Op><<<blocks, kThreads, 0, ctx->stream>>>(o, a, b, c, n, beta, op);
    else
      ew_kernel<T, NIN, false, false, Op><<<blocks, kThreads, 0, ctx->stream>>>(o, a, b, c, n, beta, op);
  }
  NK_LAUNCHED(ctx, name);
  return NK_OK;
}

struct OpFill {
  float v;
  __device__ float operator()(float, float, float) const { return v; }
};
struct OpAdd {
  __device__ float operator()(float a, float b, float) const { return a + b; }
};
struct OpCopy {
  __device__ float operator()(float a, float, float) const { return a; }
};
struct OpRelu {  // f32::max(x, 0): NaN -> 0
  __device__ float operator()(float a, float, float) const { return a > 0.f ? a : 0.f; }
};
struct OpReluBwd {  // (x > 0) * g
  __device__ float operator()(float x, float g, float) const { return x > 0.f ? g : 0.f; }
};
struct OpMseBwd {  // 2 (x - t) * g [/ n], same operation order as squared_error/mod.rs:111-119
  const float* g;
  float nf;
  int mean;
  __device__ float operator()(float x, float t, float) const {
    float v = (2.f * (x - t)) * (*g);
    return mean ? v / nf : v;
  }
};
struct OpScalarBcast {  // sum/mean backward: g [* 1/n]
  const float* g;
  float div;
  __device__ float operator()(float, float, float) const { return (*g) / div; }
};

// ---------------------------------------------------------------- cast
template <typename TD, typename TS>
__global__ void __launch_bounds__(kThreads) cast_kernel(TD* __restrict__ dst, const TS* __restrict__ src, size_t n) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = nk_from_f32<TD>(nk_to_f32<TS>(src[i]));
}

// ---------------------------------------------------------------- broadcast add (generic strided)
struct BcastDims {
  int ndim;
  int64_t shape[NK_MAX_DIMS];
  int64_t ls[NK_MAX_DIMS];  // element strides, 0 on broadcast axes
  int64_t rs[NK_MAX_DIMS];
};

template <typename T>
__global__ void __launch_bounds__(kThreads) add_bcast_generic(T* __restrict__ y, const T* __restrict__ l,
                                                             const T* __restrict__ r, size_t n, BcastDims d) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    size_t rem = i;
    int64_t lo = 0, ro = 0;
#pragma unroll
    for (int k = NK_MAX_DIMS - 1; k >= 0; --k) {
      if (k < d.ndim) {
        int64_t c = int64_t(rem % size_t(d.shape[k]));
        rem /= size_t(d.shape[k]);
        lo += c * d.ls[k];
        ro += c * d.rs[k];
      }
    }
    y[i] = nk_from_f32<T>(nk_to_f32<T>(l[lo]) + nk_to_f32<T>(r[ro]));
  }
}

// y viewed as (outer, C, inner); small[c] broadcast.  inner == 1 -> row broadcast (Linear bias),
// inner = H*W -> channel broadcast (Conv2d bias (Cout,1,1)).
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads) add_bcast_channel(T* __restrict__ y, const T* __restrict__ big,
                                                             const T* __restrict__ small, size_t n,
                                                             int64_t C, int64_t inner) {
  const size_t tid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  if (VEC) {
    constexpr int V = NkVec<T>::N;  // host guarantees inner % V == 0 or (inner == 1 and C % V == 0)
    const size_t nvec = n / V;
    for (size_t v = tid; v < nvec; v += stride) {
      NkVec<T> a, o;
      a.load(big + v * V);
      const size_t e0 = v * V;
      if (inner == 1) {
        const size_t c0 = e0 % size_t(C);
#pragma unroll
        for (int i = 0; i < V; ++i) o.set(i, a.get(i) + nk_to_f32<T>(small[c0 + i]));
      } else {
        const float s = nk_to_f32<T>(small[(e0 / size_t(inner)) % size_t(C)]);
#pragma unroll
        for (int i = 0; i < V; ++i) o.set(i, a.get(i) + s);
      }
      o.store(y + v * V);
    }
  } else {
    for (size_t i = tid; i < n; i += stride) {
      const size_t c = (i / size_t(inner)) % size_t(C);
      y[i] = nk_from_f32<T>(nk_to_f32<T>(big[i]) + nk_to_f32<T>(small[c]));
    }
  }
}

// ---------------------------------------------------------------- un-broadcast reductions
// g viewed as (R0, K, R1): out[k] = sum_{r0, r1} g[r0][k][r1]   (f32 scratch, atomics between CTAs)
// R1 == 1: column sums of an (R0, K) matrix  -> coalesced across k
template <typename T>
__global__ void __launch_bounds__(kThreads) colsum_kernel(float* __restrict__ scratch, const T* __restrict__ g,
                                                         int64_t R0, int64_t K, int64_t rows_per_block) {
  // block = 32 columns x 8 row-lanes
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int64_t col = int64_t(blockIdx.x) * 32 + cx;
  const int64_t r_begin = int64_t(blockIdx.y) * rows_per_block;
  int64_t r_end = r_begin + rows_per_block;
  if (r_end > R0) r_end = R0;
  float acc = 0.f;
  if (col < K)
    for (int64_t r = r_begin + ry; r < r_end; r += 8) acc += nk_to_f32<T>(g[r * K + col]);
  __shared__ float sm[8][33];
  sm[ry][cx] = acc;
  __syncthreads();
  if (ry == 0 && col < K) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += sm[i][cx];
    atomicAdd(&scratch[col], s);
  }
}

// same, 16-byte loads: 32 column groups x 8 row lanes per block, V = 16/sizeof(T) columns per thread
template <typename T>
__global__ void __launch_bounds__(kThreads) colsum_vec_kernel(float* __restrict__ scratch, const T* __restrict__ g,
                                                             int64_t R0, int64_t K, int64_t rows_per_block) {
  constexpr int V = NkVec<T>::N;
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int64_t col = (int64_t(blockIdx.x) * 32 + cx) * V;
  const int64_t r_begin = int64_t(blockIdx.y) * rows_per_block;
  int64_t r_end = r_begin + rows_per_block;
  if (r_end > R0) r_end = R0;
  float acc[V];
#pragma unroll
  for (int i = 0; i < V; ++i) acc[i] = 0.f;
  if (col < K) {
    int64_t r = r_begin + ry;
    for (; r + 8 < r_end; r += 16) {  // two independent loads in flight
      NkVec<T> a, b;
      a.load(g + r * K + col);
      b.load(g + (r + 8) * K + col);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] += a.get(i) + b.get(i);
    }
    for (; r < r_end; r += 8) {
      NkVec<T> a;
      a.load(g + r * K + col);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] += a.get(i);
    }
  }
  __shared__ float sm[8][32 * V + 1];
#pragma unroll
  for (int i = 0; i < V; ++i) sm[ry][cx * V + i] = acc[i];
  __syncthreads();
  for (int c = threadIdx.x; c < 32 * V; c += kThreads) {
    const int64_t gc = int64_t(blockIdx.x) * 32 * V + c;
    if (gc < K) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += sm[i][c];
      atomicAdd(&scratch[gc], t);
    }
  }
}

// general (R0, K, R1) with R1 > 1: one block per (k, r0-chunk); contiguous runs of R1
template <typename T>
__global__ void __launch_bounds__(kThreads) chansum_kernel(float* __restrict__ scratch, const T* __restrict__ g,
                                                          int64_t R0, int64_t K, int64_t R1, int64_t r0_per_block) {
  const int64_t k = blockIdx.x;
  const int64_t r_begin = int64_t(blockIdx.y) * r0_per_block;
  int64_t r_end = r_begin + r0_per_block;
  if (r_end > R0) r_end = R0;
  float acc = 0.f;
  for (int64_t r0 = r_begin; r0 < r_end; ++r0) {
    const T* p = g + (r0 * K + k) * R1;
    for (int64_t i = threadIdx.x; i < R1; i += blockDim.x) acc += nk_to_f32<T>(p[i]);
  }
  acc = nk_warp_sum(acc);
  __shared__ float sm[kThreads / 32];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) s += sm[i];
    atomicAdd(&scratch[k], s);
  }
}

// slow but fully general: one thread per dst element, loops over every reduced coordinate
struct UnbDims {
  int ndim;                       // ndim of g
  int64_t gshape[NK_MAX_DIMS];
  int64_t dshape[NK_MAX_DIMS];    // dst shape left-padded with 1s to ndim
};
template <typename T>
__global__ void __launch_bounds__(kThreads) unbroadcast_generic(float* __restrict__ scratch, const T* __restrict__ g,
                                                               size_t n_dst, UnbDims d) {
  const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_dst) return;
  int64_t dc[NK_MAX_DIMS];
  size_t rem = i;
  for (int k = d.ndim - 1; k >= 0; --k) {
    dc[k] = int64_t(rem % size_t(d.dshape[k]));
    rem /= size_t(d.dshape[k]);
  }
  // iterate over the reduced sub-space
  int64_t red_total = 1;
  for (int k = 0; k < d.ndim; ++k)
    if (d.dshape[k] == 1 && d.gshape[k] != 1) red_total *= d.gshape[k];
  float acc = 0.f;
  for (int64_t r = 0; r < red_total; ++r) {
    int64_t rr = r, off = 0, mul = 1;
    for (int k = d.ndim - 1; k >= 0; --k) {
      int64_t c;
      if (d.dshape[k] == 1 && d.gshape[k] != 1) {
        c = rr % d.gshape[k];
        rr /= d.gshape[k];
      } else {
        c = dc[k];
      }
      off += c * mul;
      mul *= d.gshape[k];
    }
    acc += nk_to_f32<T>(g[off]);
  }
  scratch[i] = acc;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) finalize_acc(T* __restrict__ dst, const float* __restrict__ scratch,
                                                        size_t n, float beta) {
  const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = scratch[i];
  if (beta != 0.f) v += beta * nk_to_f32<T>(dst[i]);
  dst[i] = nk_from_f32<T>(v);
}

// dst(TD) = beta*dst + src(TS), same shape
template <typename TD, typename TS>
__global__ void __launch_bounds__(kThreads) axpy_mixed(TD* __restrict__ dst, const TS* __restrict__ src, size_t n,
                                                      float beta) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float v = nk_to_f32<TS>(src[i]);
    if (beta != 0.f) v += beta * nk_to_f32<TD>(dst[i]);
    dst[i] = nk_from_f32<TD>(v);
  }
}

// ---------------------------------------------------------------- scalar reductions
// stage 1: per-block partial of sum f(x[, t]) in double; stage 2: single block, fixed order.
template <typename T, int MODE>  // MODE 0: sum x ; 1: sum (x-t)^2
__global__ void __launch_bounds__(kThreads) reduce_stage1(double* __restrict__ partials, const T* __restrict__ x,
                                                         const T* __restrict__ t, size_t n) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  float acc = 0.f;
  double dacc = 0.0;
  int cnt = 0;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float v = nk_to_f32<T>(x[i]);
    if (MODE == 1) {
      float d = v - nk_to_f32<T>(t[i]);
      v = d * d;
    }
    acc += v;
    if (++cnt == 64) {  // bound the f32 partial's error, then carry in double
      dacc += double(acc);
      acc = 0.f;
      cnt = 0;
    }
  }
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

__global__ void reduce_stage2(float* __restrict__ out, const double* __restrict__ partials, int nparts, double scale) {
  double s = 0.0;
  for (int i = threadIdx.x; i < nparts; i += 32) s += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) *out = float(s * scale);
}

template <typename T, typename TT>
__global__ void __launch_bounds__(kThreads) nll_fwd_kernel(double* __restrict__ partials, const T* __restrict__ logp,
                                                          const TT* __restrict__ target, int64_t n, int64_t c) {
  double acc = 0.0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    int64_t cls = (int64_t)nk_to_f32<TT>(target[i]);  // `target as usize`, nll/mod.rs:55
    if (cls >= 0 && cls < c) acc += double(nk_to_f32<T>(logp[i * c + cls]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double sm[kThreads / 32];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += sm[i];
    partials[blockIdx.x] = s;
  }
}

template <typename T, typename TT>
__global__ void __launch_bounds__(kThreads) nll_bwd_kernel(T* __restrict__ d, const TT* __restrict__ target,
                                                          const float* __restrict__ g, int64_t n, int64_t c,
                                                          float scale, float beta) {
  const int64_t total = n * c;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const float gv = (*g) * scale;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t row = i / c, col = i - row * c;
    const int64_t cls = (int64_t)nk_to_f32<TT>(target[row]);
    float v = (cls == col) ? -gv : 0.f;
    if (beta != 0.f) v += beta * nk_to_f32<T>(d[i]);
    d[i] = nk_from_f32<T>(v);
  }
}

// ---------------------------------------------------------------- pad
// One thread per E consecutive elements of an output row (E = 2 when the row length is even: one 4- / 8-byte store, a warp
// writes a contiguous span), index arithmetic in 32 bits whenever the tensor allows it: the first version spent two
// 64-bit divisions per 2-byte element and ran at 0.6 TB/s.
template <typename T, int E>
struct alignas(sizeof(T) * E) PadPack {
  T v[E];
};

template <typename T, int E, typename IT>
__global__ void __launch_bounds__(kThreads) pad2d_fwd_kernel(T* __restrict__ y, const T* __restrict__ x, int64_t planes,
                                                            int64_t h, int64_t w, int64_t ph, int64_t pw, float value) {
  const IT ho = IT(h + 2 * ph), wo = IT(w + 2 * pw), wv = wo / E;
  const IT total = IT(planes) * ho * wv;
  const IT stride = IT(gridDim.x) * blockDim.x;
  const T fillv = nk_from_f32<T>(value);
  for (IT i = IT(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const IT r = i / wv, qv = i - r * wv;     // r = (plane, p)
    const IT pl = r / ho, p = r - pl * ho;
    const int sy = int(p) - int(ph);
    const bool row_in = sy >= 0 && sy < int(h);
    const T* xr = x + (int64_t(pl) * h + (row_in ? sy : 0)) * w;
    PadPack<T, E> o;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int sx = int(qv) * E + e - int(pw);
      o.v[e] = (row_in && sx >= 0 && sx < int(w)) ? xr[sx] : fillv;  // bit-exact copy
    }
    reinterpret_cast<PadPack<T, E>*>(y)[i] = o;
  }
}

template <typename T, int E, typename IT>
__global__ void __launch_bounds__(kThreads) pad2d_bwd_kernel(T* __restrict__ dx, const T* __restrict__ g, int64_t planes,
                                                            int64_t h, int64_t w, int64_t ph, int64_t pw, float beta) {
  const IT ho = IT(h + 2 * ph), wo = IT(w + 2 * pw), wv = IT(w) / E, hh = IT(h);
  const IT total = IT(planes) * hh * wv;
  const IT stride = IT(gridDim.x) * blockDim.x;
  for (IT i = IT(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const IT r = i / wv, qv = i - r * wv;     // r = (plane, p)
    const IT pl = r / hh, p = r - pl * hh;
    const T* gr = g + (int64_t(pl) * ho + p + ph) * wo + pw + int64_t(qv) * E;
    PadPack<T, E>* d = reinterpret_cast<PadPack<T, E>*>(dx) + i;
    PadPack<T, E> o;
    if (beta != 0.f) o = *d;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const T gv = gr[e];
      o.v[e] = beta != 0.f ? nk_from_f32<T>(beta * nk_to_f32<T>(o.v[e]) + nk_to_f32<T>(gv)) : gv;
    }
    *d = o;
  }
}

}  // namespace

int nk_reduce_finish(nk_ctx* ctx, float* out, const double* partials, int nparts, double scale) {
  reduce_stage2<<<1, 32, 0, ctx->stream>>>(out, partials, nparts, scale);
  NK_LAUNCHED(ctx, "reduce_stage2");
  return NK_OK;
}

extern "C" {

int nk_fill(nk_ctx* ctx, void* dptr, int dtype, size_t n, float value) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_fill: bad dtype %d", dtype);
  NK_REQUIRE(ctx, dptr || n == 0, "nk_fill: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 0>(ctx, "fill", dptr, nullptr, nullptr, nullptr, n, 0.f, OpFill{value})));
}

int nk_cast(nk_ctx* ctx, void* dst, int dst_dtype, const void* src, int src_dtype, size_t n) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dst_dtype) && nk_dtype_ok(src_dtype), "nk_cast: bad dtype");
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, dst && src, "nk_cast: NULL pointer");
  int blocks = ew_blocks(ctx, n);
  if (dst_dtype == NK_F32 && src_dtype == NK_F32)
    cast_kernel<float, float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dst, (const float*)src, n);
  else if (dst_dtype == NK_BF16 && src_dtype == NK_F32)
    cast_kernel<__nv_bfloat16, float><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dst, (const float*)src, n);
  else if (dst_dtype == NK_F32 && src_dtype == NK_BF16)
    cast_kernel<float, __nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((float*)dst, (const __nv_bfloat16*)src, n);
  else
    cast_kernel<__nv_bfloat16, __nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dst, (const __nv_bfloat16*)src, n);
  NK_LAUNCHED(ctx, "cast");
  return NK_OK;
}

// co-broadcast predicate of utils.rs:97-125
static int bcast_shape(nk_ctx* ctx, int l_ndim, const int64_t* ls, int r_ndim, const int64_t* rs, int* ndim,
                       int64_t* out) {
  NK_REQUIRE(ctx, l_ndim >= 0 && l_ndim <= NK_MAX_DIMS && r_ndim >= 0 && r_ndim <= NK_MAX_DIMS,
             "broadcast: at most %d dims", NK_MAX_DIMS);
  int nd = l_ndim > r_ndim ? l_ndim : r_ndim;
  for (int k = 0; k < nd; ++k) {
    int64_t a = (k - (nd - l_ndim)) >= 0 ? ls[k - (nd - l_ndim)] : 1;
    int64_t b = (k - (nd - r_ndim)) >= 0 ? rs[k - (nd - r_ndim)] : 1;
    NK_REQUIRE(ctx, a == b || a == 1 || b == 1, "The two tensors have incompatible shape.");
    out[k] = a == 1 ? b : a;
  }
  *ndim = nd;
  return NK_OK;
}

int nk_add_bcast_fwd(nk_ctx* ctx, void* y, const void* l, const void* r, int dtype, int y_ndim,
                     const int64_t* y_shape, int l_ndim, const int64_t* l_shape, int r_ndim,
                     const int64_t* r_shape) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_add_bcast_fwd: bad dtype %d", dtype);
  int nd = 0;
  int64_t shape[NK_MAX_DIMS];
  int rc = bcast_shape(ctx, l_ndim, l_shape, r_ndim, r_shape, &nd, shape);
  if (rc) return rc;
  NK_REQUIRE(ctx, nd == y_ndim, "nk_add_bcast_fwd: output rank %d != broadcast rank %d", y_ndim, nd);
  size_t n = 1, nl = 1, nr = 1;
  for (int k = 0; k < nd; ++k) {
    NK_REQUIRE(ctx, y_shape[k] == shape[k], "nk_add_bcast_fwd: output dim %d is %lld, expected %lld", k,
               (long long)y_shape[k], (long long)shape[k]);
    n *= size_t(shape[k]);
  }
  for (int k = 0; k < l_ndim; ++k) nl *= size_t(l_shape[k]);
  for (int k = 0; k < r_ndim; ++k) nr *= size_t(r_shape[k]);
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, y && l && r, "nk_add_bcast_fwd: NULL pointer");
  if (nl == n && nr == n) {
    NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 2>(ctx, "add", y, l, r, nullptr, n, 0.f, OpAdd{})));
  }
  // fast path: one operand is full, the other is (C) or (C,1,..,1) aligned somewhere inside
  {
    const void* big = nl == n ? l : (nr == n ? r : nullptr);
    const void* small = nl == n ? r : l;
    int s_ndim = nl == n ? r_ndim : l_ndim;
    const int64_t* s_shape = nl == n ? r_shape : l_shape;
    if (big) {
      // find the single non-1 axis of the small operand
      int ax = -1, cnt = 0;
      for (int k = 0; k < s_ndim; ++k)
        if (s_shape[k] != 1) {
          ax = k;
          ++cnt;
        }
      if (cnt <= 1) {
        int64_t C = 1, inner = 1;
        if (cnt == 1) {
          int yax = ax + (nd - s_ndim);
          C = shape[yax];
          for (int k = yax + 1; k < nd; ++k) inner *= shape[k];
        } else {
          C = 1;
          inner = int64_t(n);
        }
        int V = dtype == NK_BF16 ? 8 : 4;
        bool vec = aligned16(y) && aligned16(big) && ((inner == 1 && C % V == 0) || (inner > 1 && inner % V == 0));
        int blocks = ew_blocks(ctx, vec ? n / V : n);
        if (dtype == NK_BF16) {
          using T = __nv_bfloat16;
          if (vec)
            add_bcast_channel<T, true><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, (const T*)big, (const T*)small, n, C, inner);
          else
            add_bcast_channel<T, false><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, (const T*)big, (const T*)small, n, C, inner);
        } else {
          using T = float;
          if (vec)
            add_bcast_channel<T, true><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, (const T*)big, (const T*)small, n, C, inner);
          else
            add_bcast_channel<T, false><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, (const T*)big, (const T*)small, n, C, inner);
        }
        NK_LAUNCHED(ctx, "add_bcast_channel");
        return NK_OK;
      }
    }
  }
  BcastDims d;
  d.ndim = nd;
  int64_t lstride = 1, rstride = 1;
  for (int k = nd - 1; k >= 0; --k) {
    d.shape[k] = shape[k];
    int lk = k - (nd - l_ndim), rk = k - (nd - r_ndim);
    int64_t a = lk >= 0 ? l_shape[lk] : 1, b = rk >= 0 ? r_shape[rk] : 1;
    d.ls[k] = (a == 1 && shape[k] != 1) ? 0 : lstride;
    d.rs[k] = (b == 1 && shape[k] != 1) ? 0 : rstride;
    lstride *= a;
    rstride *= b;
  }
  for (int k = nd; k < NK_MAX_DIMS; ++k) d.shape[k] = 1, d.ls[k] = 0, d.rs[k] = 0;
  int blocks = ew_blocks(ctx, n);
  if (dtype == NK_BF16)
    add_bcast_generic<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)y, (const __nv_bfloat16*)l, (const __nv_bfloat16*)r, n, d);
  else
    add_bcast_generic<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)y, (const float*)l, (const float*)r, n, d);
  NK_LAUNCHED(ctx, "add_bcast_generic");
  return NK_OK;
}

int nk_unbroadcast_acc(nk_ctx* ctx, void* dst, int dst_dtype, int dst_ndim, const int64_t* dst_shape,
                       const void* g, int g_dtype, int g_ndim, const int64_t* g_shape, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dst_dtype) && nk_dtype_ok(g_dtype), "nk_unbroadcast_acc: bad dtype");
  NK_REQUIRE(ctx, dst_ndim >= 0 && g_ndim <= NK_MAX_DIMS && dst_ndim <= g_ndim,
             "nk_unbroadcast_acc: target rank %d must not exceed source rank %d (max %d)", dst_ndim, g_ndim, NK_MAX_DIMS);
  int64_t dsh[NK_MAX_DIMS];
  size_t n_dst = 1, n_g = 1;
  const int off = g_ndim - dst_ndim;
  for (int k = 0; k < g_ndim; ++k) {
    dsh[k] = k >= off ? dst_shape[k - off] : 1;
    NK_REQUIRE(ctx, dsh[k] == g_shape[k] || dsh[k] == 1, "nk_unbroadcast_acc: dim %d: %lld does not broadcast to %lld",
               k, (long long)dsh[k], (long long)g_shape[k]);
    n_dst *= size_t(dsh[k]);
    n_g *= size_t(g_shape[k]);
  }
  if (n_dst == 0) return NK_OK;
  if (n_g == 0) {  // nothing to sum: dst = beta*dst (a fill of 0 when beta = 0); g may be NULL
    NK_REQUIRE(ctx, dst, "nk_unbroadcast_acc: NULL pointer");
    if (beta == 1.f) return NK_OK;
    NK_DISPATCH_DTYPE(dst_dtype, T, return (launch_ew<T, 0>(ctx, "scale", dst, nullptr, nullptr, nullptr, n_dst, beta, OpFill{0.f})));
  }
  NK_REQUIRE(ctx, dst && g, "nk_unbroadcast_acc: NULL pointer");
  if (n_dst == n_g) {  // same shape: dst = beta*dst + g
    int blocks = ew_blocks(ctx, n_g);
    if (dst_dtype == g_dtype) {
      NK_DISPATCH_DTYPE(dst_dtype, T, return (launch_ew<T, 1>(ctx, "acc", dst, g, nullptr, nullptr, n_g, beta, OpCopy{})));
    } else if (dst_dtype == NK_F32) {
      axpy_mixed<float, __nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((float*)dst, (const __nv_bfloat16*)g, n_g, beta);
    } else {
      axpy_mixed<__nv_bfloat16, float><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dst, (const float*)g, n_g, beta);
    }
    NK_LAUNCHED(ctx, "axpy_mixed");
    return NK_OK;
  }
  // collapse to (R0, K, R1) when the kept axes are contiguous
  int first_keep = -1, last_keep = -1;
  bool contiguous = true;
  for (int k = 0; k < g_ndim; ++k) {
    bool keep = dsh[k] != 1 || g_shape[k] == 1;
    if (dsh[k] == 1 && g_shape[k] == 1) continue;  // neutral axis
    if (keep) {
      if (first_keep < 0) first_keep = k;
      last_keep = k;
    }
  }
  if (first_keep >= 0)
    for (int k = first_keep; k <= last_keep; ++k)
      if (dsh[k] == 1 && g_shape[k] != 1) contiguous = false;
  float* scratch;
  int rc = nk_workspace(ctx, n_dst * sizeof(float), (void**)&scratch);
  if (rc) return rc;
  if (contiguous) {
    int64_t R0 = 1, K = 1, R1 = 1;
    for (int k = 0; k < g_ndim; ++k) {
      if (first_keep < 0 || k < first_keep)
        R0 *= g_shape[k];
      else if (k <= last_keep)
        K *= g_shape[k];
      else
        R1 *= g_shape[k];
    }
    NK_CUDA(ctx, cudaMemsetAsync(scratch, 0, n_dst * sizeof(float), ctx->stream));
    const int V = g_dtype == NK_BF16 ? 8 : 4;
    if (R1 == 1 && K % V == 0 && aligned16(g) && K >= 32 * V) {
      const int64_t col_blocks = (K + 32 * V - 1) / (32 * V);
      int64_t want_y = (int64_t(ctx->sm_count) * 8 + col_blocks - 1) / col_blocks;
      int64_t rows_per_block = (R0 + want_y - 1) / want_y;
      if (rows_per_block < 64) rows_per_block = 64;
      const int64_t gy = (R0 + rows_per_block - 1) / rows_per_block;
      dim3 grid((unsigned)col_blocks, (unsigned)gy);
      if (g_dtype == NK_BF16)
        colsum_vec_kernel<__nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, R0, K, rows_per_block);
      else
        colsum_vec_kernel<float><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, R0, K, rows_per_block);
      NK_LAUNCHED(ctx, "colsum_vec");
    } else if (R1 == 1) {
      int64_t col_blocks = (K + 31) / 32;
      int64_t want_y = (int64_t(ctx->sm_count) * 8 + col_blocks - 1) / col_blocks;
      int64_t rows_per_block = (R0 + want_y - 1) / want_y;
      if (rows_per_block < 64) rows_per_block = 64;
      int64_t gy = (R0 + rows_per_block - 1) / rows_per_block;
      dim3 grid((unsigned)col_blocks, (unsigned)gy);
      if (g_dtype == NK_BF16)
        colsum_kernel<__nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, R0, K, rows_per_block);
      else
        colsum_kernel<float><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, R0, K, rows_per_block);
      NK_LAUNCHED(ctx, "colsum");
    } else {
      int64_t want_y = (int64_t(ctx->sm_count) * 8 + K - 1) / K;
      if (want_y > R0) want_y = R0;
      if (want_y < 1) want_y = 1;
      int64_t r0_per_block = (R0 + want_y - 1) / want_y;
      int64_t gy = (R0 + r0_per_block - 1) / r0_per_block;
      NK_REQUIRE(ctx, gy <= 65535, "nk_unbroadcast_acc: reduction grid too large");
      dim3 grid((unsigned)K, (unsigned)gy);
      if (g_dtype == NK_BF16)
        chansum_kernel<__nv_bfloat16><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, R0, K, R1, r0_per_block);
      else
        chansum_kernel<float><<<grid, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, R0, K, R1, r0_per_block);
      NK_LAUNCHED(ctx, "chansum");
    }
  } else {
    UnbDims d;
    d.ndim = g_ndim;
    for (int k = 0; k < NK_MAX_DIMS; ++k) {
      d.gshape[k] = k < g_ndim ? g_shape[k] : 1;
      d.dshape[k] = k < g_ndim ? dsh[k] : 1;
    }
    int blocks = int((n_dst + kThreads - 1) / kThreads);
    if (g_dtype == NK_BF16)
      unbroadcast_generic<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>(scratch, (const __nv_bfloat16*)g, n_dst, d);
    else
      unbroadcast_generic<float><<<blocks, kThreads, 0, ctx->stream>>>(scratch, (const float*)g, n_dst, d);
    NK_LAUNCHED(ctx, "unbroadcast_generic");
  }
  int blocks = int((n_dst + kThreads - 1) / kThreads);
  if (dst_dtype == NK_BF16)
    finalize_acc<__nv_bfloat16><<<blocks, kThreads, 0, ctx->stream>>>((__nv_bfloat16*)dst, scratch, n_dst, beta);
  else
    finalize_acc<float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dst, scratch, n_dst, beta);
  NK_LAUNCHED(ctx, "finalize_acc");
  return NK_OK;
}

int nk_relu_fwd(nk_ctx* ctx, void* y, const void* x, size_t n, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_relu_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, (y && x) || n == 0, "nk_relu_fwd: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 1>(ctx, "relu_fwd", y, x, nullptr, nullptr, n, 0.f, OpRelu{})));
}

int nk_relu_bwd(nk_ctx* ctx, void* dx, const void* x, const void* g, size_t n, int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_relu_bwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, (dx && x && g) || n == 0, "nk_relu_bwd: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 2>(ctx, "relu_bwd", dx, x, g, nullptr, n, beta, OpReluBwd{})));
}

static int reduce_to_scalar(nk_ctx* ctx, float* out, const void* x, const void* t, size_t n, int dtype, int mode,
                            double scale) {
  int blocks = ew_blocks(ctx, n);
  double* partials;
  int rc = nk_workspace(ctx, size_t(blocks) * sizeof(double), (void**)&partials);
  if (rc) return rc;
  if (dtype == NK_BF16) {
    using T = __nv_bfloat16;
    if (mode == 0)
      reduce_stage1<T, 0><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n);
    else
      reduce_stage1<T, 1><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n);
  } else {
    using T = float;
    if (mode == 0)
      reduce_stage1<T, 0><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n);
    else
      reduce_stage1<T, 1><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const T*)x, (const T*)t, n);
  }
  NK_LAUNCHED(ctx, "reduce_stage1");
  reduce_stage2<<<1, 32, 0, ctx->stream>>>(out, partials, blocks, scale);
  NK_LAUNCHED(ctx, "reduce_stage2");
  return NK_OK;
}

int nk_mse_fwd(nk_ctx* ctx, float* loss, const void* x, const void* t, size_t n, int dtype, int mean) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_mse_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, loss && x && t && n > 0, "nk_mse_fwd: NULL pointer or empty input");
  return reduce_to_scalar(ctx, loss, x, t, n, dtype, 1, mean ? 1.0 / double(n) : 1.0);
}

int nk_mse_bwd(nk_ctx* ctx, void* dx, const void* x, const void* t, const float* g, size_t n, int dtype, int mean,
               float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_mse_bwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, dx && x && t && g && n > 0, "nk_mse_bwd: NULL pointer or empty input");
  OpMseBwd op{g, float(n), mean};
  NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 2>(ctx, "mse_bwd", dx, x, t, nullptr, n, beta, op)));
}

static int nll_target_ok(nk_ctx* ctx, int target_dtype, int64_t c) {
  NK_REQUIRE(ctx, nk_dtype_ok(target_dtype), "nll: bad target dtype %d", target_dtype);
  // bf16 holds integers exactly only up to 256: larger class ids would silently select the wrong class
  NK_REQUIRE(ctx, target_dtype == NK_F32 || c <= 256, "nll: a bf16 target cannot hold class ids above 256 (c = %lld); "
             "pass the target as f32", (long long)c);
  return NK_OK;
}

int nk_nll_fwd(nk_ctx* ctx, float* loss, const void* logp, const void* target, int target_dtype, int64_t n, int64_t c,
               int dtype, int mean) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_nll_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, loss && logp && target && n > 0 && c > 0, "nk_nll_fwd: NULL pointer or empty input");
  int rc = nll_target_ok(ctx, target_dtype, c);
  if (rc) return rc;
  int blocks = ew_blocks(ctx, size_t(n));
  double* partials;
  rc = nk_workspace(ctx, size_t(blocks) * sizeof(double), (void**)&partials);
  if (rc) return rc;
  using B = __nv_bfloat16;
  if (dtype == NK_BF16 && target_dtype == NK_BF16)
    nll_fwd_kernel<B, B><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const B*)logp, (const B*)target, n, c);
  else if (dtype == NK_BF16)
    nll_fwd_kernel<B, float><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const B*)logp, (const float*)target, n, c);
  else if (target_dtype == NK_BF16)
    nll_fwd_kernel<float, B><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const float*)logp, (const B*)target, n, c);
  else
    nll_fwd_kernel<float, float><<<blocks, kThreads, 0, ctx->stream>>>(partials, (const float*)logp, (const float*)target, n, c);
  NK_LAUNCHED(ctx, "nll_fwd");
  reduce_stage2<<<1, 32, 0, ctx->stream>>>(loss, partials, blocks, mean ? -1.0 / double(n) : -1.0);
  NK_LAUNCHED(ctx, "reduce_stage2");
  return NK_OK;
}

int nk_nll_bwd(nk_ctx* ctx, void* dlogp, const void* target, int target_dtype, const float* g, int64_t n, int64_t c,
               int dtype, int mean, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_nll_bwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, dlogp && target && g && n > 0 && c > 0, "nk_nll_bwd: NULL pointer or empty input");
  int rc = nll_target_ok(ctx, target_dtype, c);
  if (rc) return rc;
  int blocks = ew_blocks(ctx, size_t(n * c));
  float scale = mean ? 1.f / float(n) : 1.f;
  using B = __nv_bfloat16;
  if (dtype == NK_BF16 && target_dtype == NK_BF16)
    nll_bwd_kernel<B, B><<<blocks, kThreads, 0, ctx->stream>>>((B*)dlogp, (const B*)target, g, n, c, scale, beta);
  else if (dtype == NK_BF16)
    nll_bwd_kernel<B, float><<<blocks, kThreads, 0, ctx->stream>>>((B*)dlogp, (const float*)target, g, n, c, scale, beta);
  else if (target_dtype == NK_BF16)
    nll_bwd_kernel<float, B><<<blocks, kThreads, 0, ctx->stream>>>((float*)dlogp, (const B*)target, g, n, c, scale, beta);
  else
    nll_bwd_kernel<float, float><<<blocks, kThreads, 0, ctx->stream>>>((float*)dlogp, (const float*)target, g, n, c, scale, beta);
  NK_LAUNCHED(ctx, "nll_bwd");
  return NK_OK;
}

int nk_sum_fwd(nk_ctx* ctx, float* out, const void* x, size_t n, int dtype, int mean) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_sum_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, out && x && n > 0, "nk_sum_fwd: NULL pointer or empty input");
  return reduce_to_scalar(ctx, out, x, nullptr, n, dtype, 0, mean ? 1.0 / double(n) : 1.0);
}

int nk_sum_bwd(nk_ctx* ctx, void* dx, const float* g, size_t n, int dtype, int mean, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_sum_bwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, dx && g && n > 0, "nk_sum_bwd: NULL pointer or empty input");
  OpScalarBcast op{g, mean ? float(n) : 1.f};
  NK_DISPATCH_DTYPE(dtype, T, return (launch_ew<T, 0>(ctx, "sum_bwd", dx, nullptr, nullptr, nullptr, n, beta, op)));
}

int nk_pad2d_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int64_t h, int64_t w, int64_t ph, int64_t pw,
                 float value, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_pad2d_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, planes >= 0 && h >= 0 && w >= 0 && ph >= 0 && pw >= 0, "nk_pad2d_fwd: negative size");
  size_t total = size_t(planes) * size_t(h + 2 * ph) * size_t(w + 2 * pw);
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x, "nk_pad2d_fwd: NULL pointer");
  // E = 2 elements per thread when rows are even (and the base pointer takes the wider store); 32-bit indices when they fit
  const bool pair = (w + 2 * pw) % 2 == 0 && (reinterpret_cast<uintptr_t>(y) % (2 * nk_dtype_size(dtype))) == 0;
  const bool small = total < (size_t(1) << 31);
  int blocks = ew_blocks(ctx, pair ? total / 2 : total);
#define NK_PAD_F(T, E, IT) pad2d_fwd_kernel<T, E, IT><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, (const T*)x, planes, h, w, ph, pw, value)
#define NK_PAD_F2(T) (pair ? (small ? NK_PAD_F(T, 2, uint32_t) : NK_PAD_F(T, 2, int64_t)) : (small ? NK_PAD_F(T, 1, uint32_t) : NK_PAD_F(T, 1, int64_t)))
  if (dtype == NK_BF16)
    NK_PAD_F2(__nv_bfloat16);
  else
    NK_PAD_F2(float);
#undef NK_PAD_F2
#undef NK_PAD_F
  NK_LAUNCHED(ctx, "pad2d_fwd");
  return NK_OK;
}

int nk_pad2d_bwd(nk_ctx* ctx, void* dx, const void* g, int64_t planes, int64_t h, int64_t w, int64_t ph, int64_t pw,
                 int dtype, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_pad2d_bwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, planes >= 0 && h >= 0 && w >= 0 && ph >= 0 && pw >= 0, "nk_pad2d_bwd: negative size");
  size_t total = size_t(planes) * size_t(h) * size_t(w);
  if (total == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && g, "nk_pad2d_bwd: NULL pointer");
  const bool pair = w % 2 == 0 && (reinterpret_cast<uintptr_t>(dx) % (2 * nk_dtype_size(dtype))) == 0;
  const bool small = size_t(planes) * size_t(h + 2 * ph) * size_t(w + 2 * pw) < (size_t(1) << 31);
  int blocks = ew_blocks(ctx, pair ? total / 2 : total);
#define NK_PAD_B(T, E, IT) pad2d_bwd_kernel<T, E, IT><<<blocks, kThreads, 0, ctx->stream>>>((T*)dx, (const T*)g, planes, h, w, ph, pw, beta)
#define NK_PAD_B2(T) (pair ? (small ? NK_PAD_B(T, 2, uint32_t) : NK_PAD_B(T, 2, int64_t)) : (small ? NK_PAD_B(T, 1, uint32_t) : NK_PAD_B(T, 1, int64_t)))
  if (dtype == NK_BF16)
    NK_PAD_B2(__nv_bfloat16);
  else
    NK_PAD_B2(float);
#undef NK_PAD_B2
#undef NK_PAD_B
  NK_LAUNCHED(ctx, "pad2d_bwd");
  return NK_OK;
}

}  // extern "C"
