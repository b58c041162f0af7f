// Batch norm over (N, C, S) and layer norm over (rows, cols), torch's semantics (nk_b200.h nk_batch_norm_* /
// nk_layer_norm_*).
//
// Statistics: each thread keeps (count, mean, M2) of its values minus a shift K (the first element of the channel or
// row), adding one 16-byte vector (or one scalar) at a time by Chan's merge of the vector's own two-pass mean and M2.
// The shift keeps the running mean near zero, so its rounding does not grow with |x| (x = 1000 + U(-1, 1) keeps full
// precision); Chan's merge never forms E[x^2] - E[x]^2.  Threads are merged in f64 by a fixed tree.
// Batch norm reduces a channel over many CTAs: each CTA writes its partial to a workspace (nk_alloc_uninit, from the
// capture arena inside a captured step) and a per-channel finalize merges the partials in ascending CTA order, so every
// output, the saved and running statistics included, is bitwise repeatable.  No float atomics anywhere.
// Layouts: (N, C, S) planes, a CTA per (channel, chunk of the channel's N*S elements), 8-element loads (NkPack8) when S
// is a multiple of 8 and every base is 16-byte aligned, scalars otherwise; (N, C) rows (S = 1), a CTA per (32
// channels, chunk of rows) whose threads walk the contiguous channels.  Layer norm: a warp per row up to kLnWarpRowBytes
// bytes, a CTA per row above.
#include <math.h>

#include <algorithm>

#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;
// Rows of at most this many bytes (of x) are normalized by one warp, longer rows by one CTA of kThreads.  Measured on an
// H100 80GB HBM3 at 700 W, 2^24 elements, forward / forward+backward in us, warp vs CTA: bf16 1024 cols 36 / 111 vs
// 110 / 201, bf16 2048 37 / 105 vs 61 / 139, bf16 4096 42 / 114 vs 44 / 115, bf16 8192 54 / 133 vs 41 / 107; f32 1024
// 72 / 181 vs 120 / 238, f32 2048 83 / 193 vs 77 / 188, f32 4096 86 / 199 vs 66 / 173.
constexpr int64_t kLnWarpRowBytes = 4096;
constexpr int kVec = 8;  // elements per vector load (one 16-byte vector of bf16, two of f32)

// ---------------------------------------------------------------- element access
template <typename T, int V>
__device__ __forceinline__ void load_vals(const T* p, float (&v)[V]) {
  if constexpr (V == kVec) {
    NkPack8<T> k;
    k.load(p);
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = k.get(i);
  } else {
    v[0] = nk_to_f32<T>(*p);
  }
}
// p = beta*p + v (the product and the add rounded separately; p is not read when beta = 0)
template <typename T, int V>
__device__ __forceinline__ void store_vals(T* p, const float (&v)[V], float beta) {
  if constexpr (V == kVec) {
    NkPack8<T> k;
    if (beta != 0.f) k.load(p);
#pragma unroll
    for (int i = 0; i < V; ++i) k.set(i, beta != 0.f ? __fadd_rn(__fmul_rn(beta, k.get(i)), v[i]) : v[i]);
    k.store(p);
  } else {
    p[0] = nk_from_f32<T>(beta != 0.f ? __fadd_rn(__fmul_rn(beta, nk_to_f32<T>(p[0])), v[0]) : v[0]);
  }
}
__device__ __forceinline__ float load_any(const void* p, int dt, int64_t i) {
  return dt == NK_BF16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]) : static_cast<const float*>(p)[i];
}
__device__ __forceinline__ void store_any(void* p, int dt, int64_t i, double v, float beta) {
  const float f = beta != 0.f ? __fadd_rn(__fmul_rn(beta, load_any(p, dt, i)), float(v)) : float(v);
  if (dt == NK_BF16)
    static_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(f);
  else
    static_cast<float*>(p)[i] = f;
}
template <typename T>
__device__ __forceinline__ float param(const T* p, int64_t i, float absent) {
  return p ? nk_to_f32<T>(p[i]) : absent;
}

// ---------------------------------------------------------------- (count, mean, M2) with Chan's merge
template <typename F>
struct Wf {
  F n, mean, m2;  // value-initialized ({}) to zeros; no initializers, so that it may live in shared memory
  // this, then b (the order is part of the result)
  __device__ __forceinline__ void merge(const Wf& b) {
    const F t = n + b.n;
    if (t == F(0)) return;
    const F delta = b.mean - mean, f = b.n / t;
    mean = mean + delta * f;
    m2 = m2 + b.m2 + delta * delta * n * f;
    n = t;
  }
};
template <int V>
__device__ __forceinline__ void wf_push(Wf<float>& a, const float (&v)[V]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) s += v[i];
  Wf<float> b{};
  b.n = float(V);
  b.mean = s / float(V);
#pragma unroll
  for (int i = 0; i < V; ++i) b.m2 = fmaf(v[i] - b.mean, v[i] - b.mean, b.m2);
  a.merge(b);
}
__device__ __forceinline__ Wf<float> wf_shfl_xor(const Wf<float>& a, int o) {
  Wf<float> b{};
  b.n = __shfl_xor_sync(0xffffffffu, a.n, o);
  b.mean = __shfl_xor_sync(0xffffffffu, a.mean, o);
  b.m2 = __shfl_xor_sync(0xffffffffu, a.m2, o);
  return b;
}
// every lane of the warp ends with the same merge of the 32 lanes: the lower lane of each pair is always merged first
__device__ __forceinline__ void wf_warp(Wf<float>& a) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Wf<float> b = wf_shfl_xor(a, o);
    if (lane & o) {
      b.merge(a);
      a = b;
    } else {
      a.merge(b);
    }
  }
}

// ---------------------------------------------------------------- batch norm: per-channel reductions
// One CTA's share of a channel, written to the workspace; merged in CTA order by the finalize.
struct StatPart {
  long long n;
  double mean, m2;  // of x - K
};
struct GradPart {
  double sg, sgx;  // sum of g, sum of g * xhat
};

// The forward's statistics of x - K, K = the channel's first element
struct StatOp {
  using Acc = Wf<float>;
  using AccD = Wf<double>;
  using Part = StatPart;
  static constexpr bool kGrad = false;
  float K = 0.f;
  template <typename TX>
  __device__ void begin(const TX* x, int64_t c, int64_t S) { K = nk_to_f32<TX>(x[c * S]); }
  template <int V>
  __device__ __forceinline__ void push(Acc& a, float (&xv)[V], const float (&)[V]) const {
#pragma unroll
    for (int i = 0; i < V; ++i) xv[i] -= K;
    wf_push<V>(a, xv);
  }
  __device__ static AccD widen(const Acc& a) { return AccD{double(a.n), double(a.mean), double(a.m2)}; }
  __device__ static void merge(AccD& a, const AccD& b) { a.merge(b); }
  __device__ static Part part(const AccD& a) { return Part{(long long)a.n, a.mean, a.m2}; }
};
// The backward's sums of g and g * xhat, xhat = (x - mean) * rstd with the saved statistics
struct GradOp {
  struct Acc {
    float sg = 0.f, sgx = 0.f;
  };
  struct AccD {
    double sg, sgx;
  };
  using Part = GradPart;
  static constexpr bool kGrad = true;
  const float* mean;
  const float* rstd;
  float m = 0.f, r = 0.f;
  template <typename TX>
  __device__ void begin(const TX*, int64_t c, int64_t) {
    m = mean[c];
    r = rstd[c];
  }
  template <int V>
  __device__ __forceinline__ void push(Acc& a, const float (&xv)[V], const float (&gv)[V]) const {
#pragma unroll
    for (int i = 0; i < V; ++i) {
      a.sg += gv[i];
      a.sgx = fmaf(gv[i], (xv[i] - m) * r, a.sgx);
    }
  }
  __device__ static AccD widen(const Acc& a) { return AccD{double(a.sg), double(a.sgx)}; }
  __device__ static void merge(AccD& a, const AccD& b) { a.sg += b.sg, a.sgx += b.sgx; }
  __device__ static Part part(const AccD& a) { return Part{a.sg, a.sgx}; }
};

// fixed tree over the kThreads / LANES groups of a CTA; sh[g * LANES + l] holds group g's value of lane l
template <class Op, int LANES>
__device__ __forceinline__ void block_tree(typename Op::AccD* sh) {
  const int l = threadIdx.x % LANES, grp = threadIdx.x / LANES;
  __syncthreads();
#pragma unroll
  for (int s = kThreads / LANES / 2; s > 0; s >>= 1) {
    if (grp < s) Op::merge(sh[grp * LANES + l], sh[(grp + s) * LANES + l]);
    __syncthreads();
  }
}

// (N, C, S) planes: block (c, p) reduces vectors [nvec*p/P, nvec*(p+1)/P) of channel c (element j of the channel is
// plane j / S, position j % S)
template <class Op, typename TX, typename TG, int V>
__global__ void __launch_bounds__(kThreads) bn_partial_planes(Op op, const TX* __restrict__ x, const TG* __restrict__ g,
                                                              int64_t C, int64_t S, int64_t nvec, int P,
                                                              typename Op::Part* __restrict__ part) {
  __shared__ typename Op::AccD sh[kThreads];
  const int64_t c = blockIdx.x;
  const int p = blockIdx.y;
  op.begin(x, c, S);
  typename Op::Acc a{};
  int64_t v = nvec * p / P + threadIdx.x;
  const int64_t v1 = nvec * (p + 1) / P;
  if (v < v1) {
    int64_t n = v * V / S, s = v * V - n * S;
    const int64_t step = int64_t(kThreads) * V, dn = step / S, ds = step - dn * S;
    for (; v < v1; v += kThreads) {
      const int64_t off = (n * C + c) * S + s;
      float xv[V], gv[V];
      load_vals<TX, V>(x + off, xv);
      if constexpr (Op::kGrad) load_vals<TG, V>(g + off, gv);
      op.template push<V>(a, xv, gv);
      s += ds;
      n += dn;
      if (s >= S) s -= S, ++n;
    }
  }
  sh[threadIdx.x] = Op::widen(a);
  block_tree<Op, 1>(sh);
  if (threadIdx.x == 0) part[c * P + p] = Op::part(sh[0]);
}

// (N, C) rows: block (b, p) reduces channels [32b, 32b + 32) over rows [N*p/P, N*(p+1)/P); lane = channel, the 8 warps
// take every 8th row
template <class Op, typename TX, typename TG>
__global__ void __launch_bounds__(kThreads) bn_partial_rows(Op op, const TX* __restrict__ x, const TG* __restrict__ g,
                                                            int64_t N, int64_t C, int P,
                                                            typename Op::Part* __restrict__ part) {
  __shared__ typename Op::AccD sh[kThreads];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t c = int64_t(blockIdx.x) * 32 + lane;
  const int p = blockIdx.y;
  typename Op::Acc a{};
  if (c < C) {
    op.begin(x, c, 1);
    for (int64_t r = N * p / P + w, r1 = N * (p + 1) / P; r < r1; r += kThreads / 32) {
      float xv[1], gv[1];
      load_vals<TX, 1>(x + r * C + c, xv);
      if constexpr (Op::kGrad) load_vals<TG, 1>(g + r * C + c, gv);
      op.template push<1>(a, xv, gv);
    }
  }
  sh[threadIdx.x] = Op::widen(a);
  block_tree<Op, 32>(sh);
  if (w == 0 && c < C) part[c * P + p] = Op::part(sh[lane]);
}

// per channel: the partials in CTA order -> saved mean and 1/sqrt(var + eps) (biased var), and the running statistics
// rm = (1 - momentum) rm + momentum mean, rv = (1 - momentum) rv + momentum var M / (M - 1)
template <typename T>
__global__ void bn_stats_finalize(const T* __restrict__ x, int64_t C, int64_t S, int P, const StatPart* __restrict__ part,
                                  float* save_mean, float* save_rstd, float* rm, float* rv, float momentum, float eps) {
  const int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= C) return;
  Wf<double> a{};
  long long n = 0;
  for (int p = 0; p < P; ++p) {
    const StatPart q = part[c * P + p];
    a.merge(Wf<double>{double(q.n), q.mean, q.m2});
    n += q.n;
  }
  const double mean = double(nk_to_f32<T>(x[c * S])) + a.mean, var = a.m2 / double(n);
  save_mean[c] = float(mean);
  save_rstd[c] = float(1.0 / sqrt(var + double(eps)));
  if (rm) {
    const double mom = momentum;
    rm[c] = float((1.0 - mom) * double(rm[c]) + mom * mean);
    rv[c] = float((1.0 - mom) * double(rv[c]) + mom * (var * double(n) / double(n - 1)));
  }
}

// Element i of (N, C, S) sits at position s = i % S of channel c = (i / S) % C; both are stepped by a fixed stride
// without a division per element
struct Pos {
  int64_t s, c, ds, dc;
  __device__ __forceinline__ Pos(int64_t i, int64_t step, int64_t S, int64_t C) {
    const int64_t pl = i / S, q = step / S;
    s = i - pl * S;
    c = pl % C;
    ds = step - q * S;
    dc = q % C;
  }
  __device__ __forceinline__ void next(int64_t S, int64_t C) {
    s += ds;
    c += dc;
    if (s >= S) s -= S, ++c;
    if (c >= C) c -= C;
  }
};

// y = (x - mean) * (rstd * w) + b over items of V elements.  ROWS: the V elements of an item are V consecutive channels
// (S = 1); else they share one channel.  With rv (eval), mean = running mean, rstd = 1/sqrt(rv + eps), both also written
// to save_mean / save_rstd for the backward.
template <typename T, int V, bool ROWS>
__global__ void __launch_bounds__(kThreads) bn_apply(T* __restrict__ y, const T* __restrict__ x, int64_t items,
                                                     int64_t C, int64_t S, const T* __restrict__ w,
                                                     const T* __restrict__ b, const float* __restrict__ mean,
                                                     const float* __restrict__ rstd, const float* __restrict__ rv,
                                                     float eps, float* save_mean, float* save_rstd) {
  const int64_t t0 = int64_t(blockIdx.x) * kThreads + threadIdx.x, nt = int64_t(gridDim.x) * kThreads;
  if (rv)
    for (int64_t c = t0; c < C; c += nt) {
      save_mean[c] = mean[c];
      save_rstd[c] = __frsqrt_rn(rv[c] + eps);
    }
  if (t0 >= items) return;
  Pos pos(t0 * V, nt * V, S, C);
  for (int64_t it = t0; it < items; it += nt, pos.next(S, C)) {
    float v[V];
    load_vals<T, V>(x + it * V, v);
    float m = 0.f, sc = 0.f, sh = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (ROWS || i == 0) {
        const int64_t c = pos.c + i;
        m = mean[c];
        sc = (rv ? __frsqrt_rn(rv[c] + eps) : rstd[c]) * param(w, c, 1.f);
        sh = param(b, c, 0.f);
      }
      v[i] = fmaf(v[i] - m, sc, sh);
    }
    store_vals<T, V>(y + it * V, v, 0.f);
  }
}

// per channel: db = beta*db + sum g, dw = beta*dw + sum g*xhat, and the dx coefficients sum/M of both
__global__ void bn_grad_finalize(int64_t C, int64_t M, int P, const GradPart* __restrict__ part, void* dw, int dw_dtype,
                                 float dw_beta, void* db, int db_dtype, float db_beta, float2* coef) {
  const int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sg = 0.0, sgx = 0.0;
  for (int p = 0; p < P; ++p) {
    const GradPart q = part[c * P + p];
    sg += q.sg;
    sgx += q.sgx;
  }
  if (db) store_any(db, db_dtype, c, sg, db_beta);
  if (dw) store_any(dw, dw_dtype, c, sgx, dw_beta);
  if (coef) coef[c] = make_float2(float(sg / double(M)), float(sgx / double(M)));
}

// dx = beta*dx + w*rstd * (g - sum(g)/M - xhat * sum(g*xhat)/M) with batch statistics (coef), w*rstd*g with running ones
template <typename TX, typename TG, typename TD, int V, bool ROWS>
__global__ void __launch_bounds__(kThreads) bn_dx(TD* __restrict__ dx, const TG* __restrict__ g,
                                                  const TX* __restrict__ x, int64_t items, int64_t C, int64_t S,
                                                  const TX* __restrict__ w, const float* __restrict__ mean,
                                                  const float* __restrict__ rstd, const float2* __restrict__ coef,
                                                  float beta) {
  const int64_t t0 = int64_t(blockIdx.x) * kThreads + threadIdx.x, nt = int64_t(gridDim.x) * kThreads;
  if (t0 >= items) return;
  Pos pos(t0 * V, nt * V, S, C);
  for (int64_t it = t0; it < items; it += nt, pos.next(S, C)) {
    float gv[V];
    load_vals<TG, V>(g + it * V, gv);
    if (coef) {
      float xv[V];
      load_vals<TX, V>(x + it * V, xv);
#pragma unroll
      for (int i = 0; i < (ROWS ? V : 1); ++i) {
        const int64_t c = pos.c + i;
        const float m = mean[c], r = rstd[c], k = r * param(w, c, 1.f);
        const float2 q = coef[c];
#pragma unroll
        for (int e = ROWS ? i : 0; e < (ROWS ? i + 1 : V); ++e) gv[e] = k * (gv[e] - q.x - (xv[e] - m) * r * q.y);
      }
    } else {
      float k = 0.f;
#pragma unroll
      for (int i = 0; i < V; ++i) {
        if (ROWS || i == 0) k = rstd[pos.c + i] * param(w, pos.c + i, 1.f);
        gv[i] *= k;
      }
    }
    store_vals<TD, V>(dx + it * V, gv, beta);
  }
}

// ---------------------------------------------------------------- layer norm
// A warp (RT = 32) or a CTA (RT = kThreads) per row; rows are dealt to the groups of RT threads with a grid stride.
// Group-wide sums and merges run in a fixed order (xor tree within a warp, then warps 0..7 in order).
template <int RT>
__device__ __forceinline__ void group_merge(Wf<float>& a, Wf<float>* sh) {
  wf_warp(a);
  if constexpr (RT > 32) {
    const int wid = threadIdx.x >> 5;
    __syncthreads();  // the previous row's readers are done
    if ((threadIdx.x & 31) == 0) sh[wid] = a;
    __syncthreads();
    a = sh[0];
#pragma unroll
    for (int k = 1; k < RT / 32; ++k) a.merge(sh[k]);
  }
}
template <int RT>
__device__ __forceinline__ float2 group_sum(float2 v, float2* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
  }
  if constexpr (RT > 32) {
    const int wid = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[wid] = v;
    __syncthreads();
    v = sh[0];
#pragma unroll
    for (int k = 1; k < RT / 32; ++k) v.x += sh[k].x, v.y += sh[k].y;
  }
  return v;
}

template <typename T, int RT, int V>
__global__ void __launch_bounds__(kThreads) ln_fwd(T* __restrict__ y, const T* __restrict__ x, int64_t rows,
                                                   int64_t cols, const T* __restrict__ w, const T* __restrict__ b,
                                                   float* __restrict__ save_mean, float* __restrict__ save_rstd,
                                                   float eps) {
  __shared__ Wf<float> sh[kThreads / 32];
  constexpr int G = kThreads / RT;
  const int lane = threadIdx.x % RT;
  for (int64_t r = int64_t(blockIdx.x) * G + threadIdx.x / RT; r < rows; r += int64_t(gridDim.x) * G) {
    const T* xr = x + r * cols;
    const float K = nk_to_f32<T>(xr[0]);
    Wf<float> a{};
    for (int64_t j = int64_t(lane) * V; j < cols; j += RT * V) {
      float v[V];
      load_vals<T, V>(xr + j, v);
#pragma unroll
      for (int i = 0; i < V; ++i) v[i] -= K;
      wf_push<V>(a, v);
    }
    group_merge<RT>(a, sh);
    const float mean = K + a.mean, rstd = 1.f / sqrtf(a.m2 / a.n + eps);
    if (lane == 0) save_mean[r] = mean, save_rstd[r] = rstd;
    for (int64_t j = int64_t(lane) * V; j < cols; j += RT * V) {
      float v[V];
      load_vals<T, V>(xr + j, v);
#pragma unroll
      for (int i = 0; i < V; ++i) v[i] = fmaf((v[i] - mean) * rstd, param(w, j + i, 1.f), param(b, j + i, 0.f));
      store_vals<T, V>(y + r * cols + j, v, 0.f);
    }
  }
}

// dx = beta*dx + rstd * (g' - sum(g')/D - xhat * sum(g'*xhat)/D), g' = g*w.  CTAs from row_blocks on finalize the
// column sums instead: dw / db column j = beta*d + the partials of ln_colpart in ascending order.
template <typename TX, typename TG, typename TD, int RT, int V>
__global__ void __launch_bounds__(kThreads) ln_bwd(TD* __restrict__ dx, const TG* __restrict__ g,
                                                   const TX* __restrict__ x, int64_t rows, int64_t cols,
                                                   const TX* __restrict__ w, const float* __restrict__ save_mean,
                                                   const float* __restrict__ save_rstd, float beta, int row_blocks,
                                                   const float* __restrict__ part, int P, void* dw, int dw_dtype,
                                                   float dw_beta, void* db, int db_dtype, float db_beta) {
  if (int(blockIdx.x) >= row_blocks) {
    const int64_t j = int64_t(blockIdx.x - row_blocks) * kThreads + threadIdx.x;
    if (j >= cols) return;
    double sgx = 0.0, sg = 0.0;
    for (int p = 0; p < P; ++p) {
      sgx += part[int64_t(p) * cols + j];
      sg += part[(int64_t(P) + p) * cols + j];
    }
    if (dw) store_any(dw, dw_dtype, j, sgx, dw_beta);
    if (db) store_any(db, db_dtype, j, sg, db_beta);
    return;
  }
  __shared__ float2 sh[kThreads / 32];
  constexpr int G = kThreads / RT;
  const int lane = threadIdx.x % RT;
  for (int64_t r = int64_t(blockIdx.x) * G + threadIdx.x / RT; r < rows; r += int64_t(row_blocks) * G) {
    const TX* xr = x + r * cols;
    const TG* gr = g + r * cols;
    const float m = save_mean[r], rs = save_rstd[r];
    float2 s = make_float2(0.f, 0.f);
    for (int64_t j = int64_t(lane) * V; j < cols; j += RT * V) {
      float xv[V], gv[V];
      load_vals<TX, V>(xr + j, xv);
      load_vals<TG, V>(gr + j, gv);
#pragma unroll
      for (int i = 0; i < V; ++i) {
        const float gw = __fmul_rn(gv[i], param(w, j + i, 1.f));  // not contracted: the same g' as below
        s.x += gw;
        s.y = fmaf(gw, (xv[i] - m) * rs, s.y);
      }
    }
    s = group_sum<RT>(s, sh);
    const float mg = s.x / float(cols), mgx = s.y / float(cols);
    for (int64_t j = int64_t(lane) * V; j < cols; j += RT * V) {
      float xv[V], gv[V];
      load_vals<TX, V>(xr + j, xv);
      load_vals<TG, V>(gr + j, gv);
#pragma unroll
      for (int i = 0; i < V; ++i) gv[i] = rs * (__fmul_rn(gv[i], param(w, j + i, 1.f)) - mg - (xv[i] - m) * rs * mgx);
      store_vals<TD, V>(dx + r * cols + j, gv, beta);
    }
  }
}

// block (b, p): columns [256b, 256b + 256) over rows [rows*p/P, rows*(p+1)/P): part[p][j] = sum g*xhat,
// part[P + p][j] = sum g
template <typename TX, typename TG>
__global__ void __launch_bounds__(kThreads) ln_colpart(const TG* __restrict__ g, const TX* __restrict__ x,
                                                       int64_t rows, int64_t cols, const float* __restrict__ save_mean,
                                                       const float* __restrict__ save_rstd, int P,
                                                       float* __restrict__ part) {
  const int64_t j = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  const int p = blockIdx.y;
  if (j >= cols) return;
  float sgx = 0.f, sg = 0.f;
  for (int64_t r = rows * p / P, r1 = rows * (p + 1) / P; r < r1; ++r) {
    const float gv = nk_to_f32<TG>(g[r * cols + j]);
    sg += gv;
    sgx = fmaf(gv, (nk_to_f32<TX>(x[r * cols + j]) - save_mean[r]) * save_rstd[r], sgx);
  }
  part[int64_t(p) * cols + j] = sgx;
  part[(int64_t(P) + p) * cols + j] = sg;
}

// ---------------------------------------------------------------- host side
inline int grid_for(nk_ctx* ctx, int64_t items) {
  const int64_t cap = int64_t(ctx->sm_count) * 8;
  return int(std::max<int64_t>(1, std::min<int64_t>((items + kThreads - 1) / kThreads, cap)));
}
inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline int cdiv(int64_t a, int64_t b) { return int((a + b - 1) / b); }

// CTAs per channel for the partial reductions: about 4 CTAs per SM in all, at least 4 vectors per thread, at most 65535
inline int parts_for(nk_ctx* ctx, int64_t groups, int64_t work) {
  int64_t p = std::min<int64_t>((4 * int64_t(ctx->sm_count) + groups - 1) / groups, (work + 4 * kThreads - 1) / (4 * kThreads));
  return int(std::max<int64_t>(1, std::min<int64_t>(p, 65535)));
}

struct Workspace {  // stream-ordered temporaries, freed on every exit path
  nk_ctx* ctx;
  void* p = nullptr;
  explicit Workspace(nk_ctx* c) : ctx(c) {}
  ~Workspace() {
    if (p) nk_free(ctx, p);
  }
  int alloc(size_t bytes) { return nk_alloc_uninit(ctx, bytes, &p); }
};

// the partial-reduction launch of either op over either layout; part holds C * P entries
template <class Op, typename TX, typename TG>
int launch_partial(nk_ctx* ctx, const Op& op, const TX* x, const TG* g, int64_t N, int64_t C, int64_t S, bool vec, int P,
                   typename Op::Part* part) {
  if (S == 1) {
    bn_partial_rows<Op, TX, TG><<<dim3(cdiv(C, 32), P), kThreads, 0, ctx->stream>>>(op, x, g, N, C, P, part);
  } else if (vec) {
    bn_partial_planes<Op, TX, TG, kVec><<<dim3(unsigned(C), P), kThreads, 0, ctx->stream>>>(op, x, g, C, S, N * S / kVec,
                                                                                           P, part);
  } else {
    bn_partial_planes<Op, TX, TG, 1><<<dim3(unsigned(C), P), kThreads, 0, ctx->stream>>>(op, x, g, C, S, N * S, P, part);
  }
  NK_LAUNCHED(ctx, "bn_partial");
  return NK_OK;
}
inline int bn_parts(nk_ctx* ctx, int64_t N, int64_t C, int64_t S) {
  return S == 1 ? parts_for(ctx, cdiv(C, 32), N * 32) : parts_for(ctx, C, N * S / kVec);
}

int check_bn(nk_ctx* ctx, const char* who, int64_t N, int64_t C, int64_t S) {
  NK_REQUIRE(ctx, N >= 0 && C >= 1 && S >= 1, "%s: bad shape (N %lld, C %lld, S %lld)", who, (long long)N, (long long)C,
             (long long)S);
  NK_REQUIRE(ctx, C <= INT32_MAX, "%s: more than 2^31 - 1 channels", who);
  return NK_OK;
}

template <typename T>
int bn_fwd(nk_ctx* ctx, T* y, const T* x, int64_t N, int64_t C, int64_t S, const T* w, const T* b, float* rm, float* rv,
           float* save_mean, float* save_rstd, bool batch, bool update, float momentum, float eps) {
  const bool rows = S == 1;
  const bool vec = al16(x) && al16(y) && (rows ? C % kVec == 0 : S % kVec == 0);
  Workspace ws(ctx);
  if (batch) {
    const int P = bn_parts(ctx, N, C, S);
    int rc = ws.alloc(size_t(C) * P * sizeof(StatPart));
    if (rc) return rc;
    StatPart* part = static_cast<StatPart*>(ws.p);
    rc = launch_partial(ctx, StatOp{}, x, (const T*)nullptr, N, C, S, vec && !rows, P, part);
    if (rc) return rc;
    bn_stats_finalize<T><<<cdiv(C, 128), 128, 0, ctx->stream>>>(x, C, S, P, part, save_mean, save_rstd,
                                                                 update ? rm : nullptr, update ? rv : nullptr, momentum, eps);
    NK_LAUNCHED(ctx, "bn_stats_finalize");
  }
  const float* mean = batch ? save_mean : rm;
  const float* var = batch ? nullptr : rv;
  const int64_t items = vec ? N * C * S / kVec : N * C * S;
  const int blocks = grid_for(ctx, std::max<int64_t>(items, batch ? 0 : C));
  if (vec && rows)
    bn_apply<T, kVec, true><<<blocks, kThreads, 0, ctx->stream>>>(y, x, items, C, S, w, b, mean, save_rstd, var, eps,
                                                                  save_mean, save_rstd);
  else if (vec)
    bn_apply<T, kVec, false><<<blocks, kThreads, 0, ctx->stream>>>(y, x, items, C, S, w, b, mean, save_rstd, var, eps,
                                                                   save_mean, save_rstd);
  else
    bn_apply<T, 1, false><<<blocks, kThreads, 0, ctx->stream>>>(y, x, items, C, S, w, b, mean, save_rstd, var, eps,
                                                                save_mean, save_rstd);
  NK_LAUNCHED(ctx, "bn_apply");
  return NK_OK;
}

template <typename TX, typename TG, typename TD>
int bn_dx_launch(nk_ctx* ctx, void* dx, const void* g, const void* x, int64_t N, int64_t C, int64_t S, const void* w,
                 const float* mean, const float* rstd, const float2* coef, float beta) {
  const bool rows = S == 1;
  const bool vec = al16(dx) && al16(g) && al16(x) && (rows ? C % kVec == 0 : S % kVec == 0);
  const int64_t items = vec ? N * C * S / kVec : N * C * S;
  const int blocks = grid_for(ctx, items);
  TD* d = static_cast<TD*>(dx);
  const TG* gg = static_cast<const TG*>(g);
  const TX* xx = static_cast<const TX*>(x);
  const TX* ww = static_cast<const TX*>(w);
  if (vec && rows)
    bn_dx<TX, TG, TD, kVec, true><<<blocks, kThreads, 0, ctx->stream>>>(d, gg, xx, items, C, S, ww, mean, rstd, coef, beta);
  else if (vec)
    bn_dx<TX, TG, TD, kVec, false><<<blocks, kThreads, 0, ctx->stream>>>(d, gg, xx, items, C, S, ww, mean, rstd, coef, beta);
  else
    bn_dx<TX, TG, TD, 1, false><<<blocks, kThreads, 0, ctx->stream>>>(d, gg, xx, items, C, S, ww, mean, rstd, coef, beta);
  NK_LAUNCHED(ctx, "bn_dx");
  return NK_OK;
}

template <typename TX, typename TG>
int bn_bwd(nk_ctx* ctx, void* dx, int dx_dtype, float dx_beta, void* dw, int dw_dtype, float dw_beta, void* db,
           int db_dtype, float db_beta, const void* g, const void* x, int64_t N, int64_t C, int64_t S, const void* w,
           const float* mean, const float* rstd, bool batch) {
  const int64_t M = N * S;
  const bool need_dx = dx && M > 0;
  const float2* coef = nullptr;
  Workspace ws(ctx);
  if (dw || db || (need_dx && batch)) {
    const bool rows = S == 1;
    const bool vec = !rows && al16(x) && al16(g) && S % kVec == 0;
    const int P = M > 0 ? bn_parts(ctx, N, C, S) : 0;
    const size_t coef_bytes = need_dx && batch ? size_t(C) * sizeof(float2) : 0;
    int rc = ws.alloc(size_t(C) * P * sizeof(GradPart) + coef_bytes);
    if (rc) return rc;
    GradPart* part = static_cast<GradPart*>(ws.p);
    float2* cf = coef_bytes ? reinterpret_cast<float2*>(part + size_t(C) * P) : nullptr;
    if (P > 0) {
      rc = launch_partial(ctx, GradOp{mean, rstd}, static_cast<const TX*>(x), static_cast<const TG*>(g), N, C, S, vec, P,
                          part);
      if (rc) return rc;
    }
    bn_grad_finalize<<<cdiv(C, 128), 128, 0, ctx->stream>>>(C, M, P, part, dw, dw_dtype, dw_beta, db, db_dtype, db_beta,
                                                            cf);
    NK_LAUNCHED(ctx, "bn_grad_finalize");
    coef = cf;
  }
  if (!need_dx) return NK_OK;
  if (dx_dtype == NK_BF16)
    return bn_dx_launch<TX, TG, __nv_bfloat16>(ctx, dx, g, x, N, C, S, w, mean, rstd, coef, dx_beta);
  return bn_dx_launch<TX, TG, float>(ctx, dx, g, x, N, C, S, w, mean, rstd, coef, dx_beta);
}

template <typename T>
int ln_fwd_launch(nk_ctx* ctx, T* y, const T* x, int64_t rows, int64_t cols, const T* w, const T* b, float* save_mean,
                  float* save_rstd, float eps) {
  const bool vec = cols % kVec == 0 && al16(x) && al16(y) && (!w || al16(w)) && (!b || al16(b));
  const bool warp = cols * int64_t(sizeof(T)) <= kLnWarpRowBytes;
  const int64_t cap = int64_t(ctx->sm_count) * 16;
  const int blocks = int(std::min<int64_t>(warp ? (rows + kThreads / 32 - 1) / (kThreads / 32) : rows, cap));
  auto go = [&](auto kern) {
    kern<<<blocks, kThreads, 0, ctx->stream>>>(y, x, rows, cols, w, b, save_mean, save_rstd, eps);
  };
  if (warp)
    vec ? go(ln_fwd<T, 32, kVec>) : go(ln_fwd<T, 32, 1>);
  else
    vec ? go(ln_fwd<T, kThreads, kVec>) : go(ln_fwd<T, kThreads, 1>);
  NK_LAUNCHED(ctx, "ln_fwd");
  return NK_OK;
}

template <typename TX, typename TG, typename TD>
int ln_bwd_launch(nk_ctx* ctx, void* dx, float dx_beta, void* dw, int dw_dtype, float dw_beta, void* db, int db_dtype,
                  float db_beta, const void* g, const void* x, int64_t rows, int64_t cols, const void* w,
                  const float* mean, const float* rstd) {
  const TX* xx = static_cast<const TX*>(x);
  const TG* gg = static_cast<const TG*>(g);
  Workspace ws(ctx);
  int P = 0;
  const bool sums = dw || db;
  if (sums && rows > 0) {
    const int cb = cdiv(cols, kThreads);
    P = int(std::max<int64_t>(1, std::min<int64_t>({(4 * int64_t(ctx->sm_count) + cb - 1) / cb, (rows + 15) / 16, 65535})));
    int rc = ws.alloc(size_t(2) * P * cols * sizeof(float));
    if (rc) return rc;
    ln_colpart<TX, TG><<<dim3(cb, P), kThreads, 0, ctx->stream>>>(gg, xx, rows, cols, mean, rstd, P,
                                                                   static_cast<float*>(ws.p));
    NK_LAUNCHED(ctx, "ln_colpart");
  }
  const bool warp = cols * int64_t(sizeof(TX)) <= kLnWarpRowBytes;
  const int64_t cap = int64_t(ctx->sm_count) * 16;
  const int row_blocks = dx && rows > 0
      ? int(std::min<int64_t>(warp ? (rows + kThreads / 32 - 1) / (kThreads / 32) : rows, cap)) : 0;
  const int fin_blocks = sums ? cdiv(cols, kThreads) : 0;
  if (row_blocks + fin_blocks == 0) return NK_OK;
  const bool vec = cols % kVec == 0 && al16(x) && al16(g) && (!dx || al16(dx)) && (!w || al16(w));
  auto go = [&](auto kern) {
    kern<<<row_blocks + fin_blocks, kThreads, 0, ctx->stream>>>(static_cast<TD*>(dx), gg, xx, rows, cols,
                                                                 static_cast<const TX*>(w), mean, rstd, dx_beta,
                                                                 row_blocks, static_cast<const float*>(ws.p), P, dw,
                                                                 dw_dtype, dw_beta, db, db_dtype, db_beta);
  };
  if (warp)
    vec ? go(ln_bwd<TX, TG, TD, 32, kVec>) : go(ln_bwd<TX, TG, TD, 32, 1>);
  else
    vec ? go(ln_bwd<TX, TG, TD, kThreads, kVec>) : go(ln_bwd<TX, TG, TD, kThreads, 1>);
  NK_LAUNCHED(ctx, "ln_bwd");
  return NK_OK;
}

}  // namespace

extern "C" {

int nk_batch_norm_fwd(nk_ctx* ctx, void* y, const void* x, int dtype, int64_t n, int64_t c, int64_t s, const void* w,
                      const void* b, float* running_mean, float* running_var, float* save_mean, float* save_rstd,
                      int training, float momentum, float eps) {
  static const char* who = "nk_batch_norm_fwd";
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", who, dtype);
  if (int rc = check_bn(ctx, who, n, c, s)) return rc;
  NK_REQUIRE(ctx, (running_mean == nullptr) == (running_var == nullptr),
             "%s: running_mean and running_var are both given or both NULL", who);
  NK_REQUIRE(ctx, eps >= 0.f, "%s: bad eps %g", who, eps);
  const bool batch = training || !running_mean;
  NK_REQUIRE(ctx, !(batch && n * s == 1),
             "Expected more than 1 value per channel when training, got input size (%lld, %lld, %lld)", (long long)n,
             (long long)c, (long long)s);
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x && save_mean && save_rstd, "%s: NULL pointer", who);
  NK_DISPATCH_DTYPE(dtype, T,
                    return bn_fwd<T>(ctx, (T*)y, (const T*)x, n, c, s, (const T*)w, (const T*)b, running_mean,
                                     running_var, save_mean, save_rstd, batch, training && running_mean, momentum, eps));
}

int nk_batch_norm_bwd(nk_ctx* ctx, void* dx, int dx_dtype, float dx_beta, void* dw, int dw_dtype, float dw_beta,
                      void* db, int db_dtype, float db_beta, const void* g, int g_dtype, const void* x, int dtype,
                      int64_t n, int64_t c, int64_t s, const void* w, const float* save_mean, const float* save_rstd,
                      int batch_stats) {
  static const char* who = "nk_batch_norm_bwd";
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(g_dtype) && (!dx || nk_dtype_ok(dx_dtype)) &&
                      (!dw || nk_dtype_ok(dw_dtype)) && (!db || nk_dtype_ok(db_dtype)),
             "%s: bad dtype", who);
  if (int rc = check_bn(ctx, who, n, c, s)) return rc;
  if (!dx && !dw && !db) return NK_OK;
  NK_REQUIRE(ctx, (n == 0 || (g && x)) && save_mean && save_rstd, "%s: NULL pointer", who);
  if (dtype == NK_BF16) {
    NK_DISPATCH_DTYPE(g_dtype, TG,
                      return (bn_bwd<__nv_bfloat16, TG>(ctx, dx, dx_dtype, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype,
                                                        db_beta, g, x, n, c, s, w, save_mean, save_rstd,
                                                        batch_stats != 0)));
  }
  NK_DISPATCH_DTYPE(g_dtype, TG,
                    return (bn_bwd<float, TG>(ctx, dx, dx_dtype, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype, db_beta,
                                              g, x, n, c, s, w, save_mean, save_rstd, batch_stats != 0)));
}

int nk_layer_norm_fwd(nk_ctx* ctx, void* y, const void* x, int dtype, int64_t rows, int64_t cols, const void* w,
                      const void* b, float* save_mean, float* save_rstd, float eps) {
  static const char* who = "nk_layer_norm_fwd";
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", who, dtype);
  NK_REQUIRE(ctx, rows >= 0 && cols >= 1, "%s: bad shape (rows %lld, cols %lld)", who, (long long)rows, (long long)cols);
  NK_REQUIRE(ctx, eps >= 0.f, "%s: bad eps %g", who, eps);
  if (rows == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x && save_mean && save_rstd, "%s: NULL pointer", who);
  NK_DISPATCH_DTYPE(dtype, T,
                    return ln_fwd_launch<T>(ctx, (T*)y, (const T*)x, rows, cols, (const T*)w, (const T*)b, save_mean,
                                            save_rstd, eps));
}

int nk_layer_norm_bwd(nk_ctx* ctx, void* dx, int dx_dtype, float dx_beta, void* dw, int dw_dtype, float dw_beta,
                      void* db, int db_dtype, float db_beta, const void* g, int g_dtype, const void* x, int dtype,
                      int64_t rows, int64_t cols, const void* w, const float* save_mean, const float* save_rstd) {
  static const char* who = "nk_layer_norm_bwd";
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(g_dtype) && (!dx || nk_dtype_ok(dx_dtype)) &&
                      (!dw || nk_dtype_ok(dw_dtype)) && (!db || nk_dtype_ok(db_dtype)),
             "%s: bad dtype", who);
  NK_REQUIRE(ctx, rows >= 0 && cols >= 1, "%s: bad shape (rows %lld, cols %lld)", who, (long long)rows, (long long)cols);
  if (!dx && !dw && !db) return NK_OK;
  NK_REQUIRE(ctx, rows == 0 || (g && x && save_mean && save_rstd), "%s: NULL pointer", who);
  auto run = [&](auto tx, auto tg) {
    using TX = decltype(tx);
    using TG = decltype(tg);
    if (dx_dtype == NK_BF16 && dx)
      return ln_bwd_launch<TX, TG, __nv_bfloat16>(ctx, dx, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype, db_beta, g, x,
                                                  rows, cols, w, save_mean, save_rstd);
    return ln_bwd_launch<TX, TG, float>(ctx, dx, dx_beta, dw, dw_dtype, dw_beta, db, db_dtype, db_beta, g, x, rows, cols,
                                        w, save_mean, save_rstd);
  };
  if (dtype == NK_BF16) {
    NK_DISPATCH_DTYPE(g_dtype, TG, return run(__nv_bfloat16(), TG()));
  }
  NK_DISPATCH_DTYPE(g_dtype, TG, return run(float(), TG()));
}

}  // extern "C"
