// Cross-entropy loss with class-index targets, torch's F.cross_entropy (nk_b200.h nk_cross_entropy_fwd / _bwd).
//
// x is (n, c, s): n samples, c classes, s spatial positions (s = 1 for 2-D input); one position is the c values of one
// (sample, spatial index) pair.  The forward reads x once and keeps per position an online (max, sum of exp) pair that
// is rescaled whenever the max grows; the same pass gathers x_t and, with label smoothing, sum_c w_c*x_c.  It saves
// lse = max + ln(sum) per position, so the backward reads x and lse once and writes dx once: no (n, c) intermediate.
// Layouts, chosen from the shape alone:
//   s == 1, rows of at most kWarpRowBytes bytes, or at least kWarpMinRows rows: a warp per row;
//   s == 1, fewer longer rows: a CTA per row, or, when the rows are too few to fill the SMs and long enough, a CTA per
//           (row, chunk) whose partial pairs are merged in ascending chunk order by a second kernel;
//   s > 1:  a thread per position, walking the classes with stride s, so each class step is coalesced across the
//           warp over the contiguous spatial positions.
// Rows take 8-element loads (NkPack8) when both bases are 16-byte aligned, whatever the row length: each row has a
// scalar head up to the first element whose flat index is a multiple of 8 and a scalar tail.
// Every partition depends only on the shape and the SM count, the pairs merge in a fixed tree and the per-block sums in
// a fixed order, and there are no float atomics: repeated calls give identical bits.
#include <math.h>

#include <algorithm>

#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kVec = 8;  // elements per vector load
// Layout thresholds, from forward / forward+backward times in us of a warp per row against a CTA per row and of split
// against unsplit rows, measured on an H100 80GB HBM3 at 700 W (f32 targets, mean, dx in x's dtype).
// Rows of at most kWarpRowBytes bytes take a warp each whatever their number: bf16 2^27 elements, warp vs CTA, 256
// classes 437 / 694 vs 2886 / 4194, 1024 classes 209 / 413 vs 788 / 1164, 2048 classes 168 / 369 vs 462 / 709; f32
// 2^26 elements, 1024 classes 123 / 312 vs 542 / 772.
constexpr int64_t kWarpRowBytes = 4096;
// Longer rows take a warp each too once there are at least kWarpMinRows of them: bf16 (32768, 4096) 155 / 357 vs
// 311 / 528, (16384, 8192) 148 / 349 vs 217 / 422, (8960, 10000) 115 / 283 vs 145 / 291, (4096, 32000) 135 / 337 vs
// 156 / 355; f32 (32768, 2048) 108 / 304 vs 295 / 497, (16384, 4096) 107 / 309 vs 202 / 390.  Fewer long rows take a
// CTA each (between 2*SMs and 4096 rows this was not measured against a warp per row).
constexpr int64_t kWarpMinRows = 4096;
// Rows are split over several CTAs when fewer than kSplitRowsPerSm * sm_count rows would leave SMs idle and a row has
// at least kSplitMinCols elements; a chunk keeps at least kMinChunk elements so that each thread of the CTA still has
// several vectors to load.  Split vs one CTA per row, bf16: 262144 classes, 16 rows 24 / 38 vs 71 / 134, 132 rows
// 48 / 103 vs 81 / 188, 263 rows 84 / 190 vs 92 / 226; 65536 classes, 16 rows 22 / 28 vs 25 / 44, 132 rows 22 / 35 vs
// 26 / 45; but 16384 classes (2 chunks), 16 rows 27 / 43 vs 13 / 29 and 132 rows 28 / 46 vs 15 / 24, hence
// kSplitMinCols.  8 rows per SM instead of 2 was no faster from 64 rows up (262144 classes, 64 rows 45 / 75 vs 34 / 72).
constexpr int64_t kSplitRowsPerSm = 2;
constexpr int64_t kSplitMinCols = 65536;
constexpr int64_t kMinChunk = kThreads * kVec * 4;

struct Acc {
  float m, s, xt, wx;  // running max, sum of exp(x - m), x_t (0 where t is elsewhere), sum of w_c * x_c
};

struct Args {
  int64_t n, c, s;      // samples, classes, spatial positions per sample
  int64_t chunk;        // elements of a row per work item (c unless rows are split), a multiple of kVec
  int splits;           // work items per row
  int group;            // threads per work item: 32 or kThreads
  int64_t ignore;       // ignore_index
  float eps, eps_c;     // label_smoothing and label_smoothing / c
};

// The class of one target value: trunc(v) for 0 <= v < c, else (NaN, negative, too large) or when it equals
// ignore_index, -1 (ignored).  The test is made on the float: a NaN converted to an integer would become class 0.
template <typename TT>
__device__ __forceinline__ int64_t target_class(TT raw, float fc, int64_t ignore) {
  const float v = nk_to_f32<TT>(raw);
  if (!(v >= 0.f && v < fc)) return -1;
  const int64_t k = int64_t(v);
  return k == ignore ? -1 : k;
}

__device__ __forceinline__ float wt_of(const float* w, int64_t k) { return w ? w[k] : 1.f; }

// A grid-stride walk over flat indices idx = row * cols + col that keeps (row, col) up to date without a 64-bit
// division per step (start and step are below 2^31, so 32-bit divisions suffice).
struct Walk {
  int64_t idx, row, col, drow, dcol, cols;
  __device__ __forceinline__ Walk(int64_t start, int64_t step, int64_t ncols) : idx(start), cols(ncols) {
    split(start, row, col);
    split(step, drow, dcol);
  }
  __device__ __forceinline__ void split(int64_t v, int64_t& r, int64_t& c) const {
    r = v < cols ? 0 : int64_t(uint32_t(v) / uint32_t(cols));
    c = v - r * cols;
  }
  __device__ __forceinline__ void next(int64_t step) {
    idx += step;
    row += drow;
    col += dcol;
    if (col >= cols) col -= cols, ++row;
  }
};

__device__ __forceinline__ Acc merge(const Acc& a, const Acc& b) {
  const float m = fmaxf(a.m, b.m);
  Acc r;
  r.m = m;
  r.s = (a.m == m ? a.s : a.s * expf(a.m - m)) + (b.m == m ? b.s : b.s * expf(b.m - m));
  r.xt = a.xt + b.xt;  // at most one side holds x_t, the other 0
  r.wx = a.wx + b.wx;
  return r;
}

// xor butterfly: every lane ends with the same merge of the 32 lanes (merge is commutative bit for bit)
__device__ __forceinline__ Acc warp_merge(Acc a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Acc b;
    b.m = __shfl_xor_sync(0xffffffffu, a.m, o);
    b.s = __shfl_xor_sync(0xffffffffu, a.s, o);
    b.xt = __shfl_xor_sync(0xffffffffu, a.xt, o);
    b.wx = __shfl_xor_sync(0xffffffffu, a.wx, o);
    a = merge(a, b);
  }
  return a;
}

// fold k values (element indices e0..e0+k-1 of the position) into the pair: one rescale per group of values
template <int K>
__device__ __forceinline__ void fold(Acc& a, const float (&v)[K], int64_t e0, int64_t t, const float* w, bool smooth) {
  float vm = v[0];
#pragma unroll
  for (int i = 1; i < K; ++i) vm = fmaxf(vm, v[i]);
  if (vm > a.m) {
    a.s *= expf(a.m - vm);
    a.m = vm;
  }
  // The max is still -inf only when every value so far is -inf (or NaN): subtract 0 then, so that each -inf adds
  // exp(-inf) = 0 instead of exp(-inf - -inf) = NaN; a NaN logit still makes the sum NaN, as in torch.
  const float m = a.m == -INFINITY ? 0.f : a.m;
  float ps = 0.f;
#pragma unroll
  for (int i = 0; i < K; ++i) ps += expf(v[i] - m);
  a.s += ps;
  const int64_t d = t - e0;
  if (d >= 0 && d < K) {
#pragma unroll
    for (int i = 0; i < K; ++i)
      if (i == d) a.xt = v[i];
  }
  if (smooth) {
#pragma unroll
    for (int i = 0; i < K; ++i) a.wx += wt_of(w, e0 + i) * v[i];
  }
}

// [v0, v1): the whole 8-element vectors of elements [e0, e1) of a row whose element 0 has flat index `base`, starting
// at the first element whose flat index is a multiple of 8, so that the vectors of a 16-byte aligned tensor are 16-byte
// aligned whatever the row length
__device__ __forceinline__ void vec_range(int64_t base, int64_t e0, int64_t e1, int64_t& v0, int64_t& v1) {
  v0 = min(e1, e0 + ((-(base + e0)) & (kVec - 1)));
  v1 = v0 + (e1 - v0) / kVec * kVec;
}

// Vectors per thread loaded before any is folded by the forward: enough bytes in flight to cover the memory latency
// (the backward's vectors are independent of each other, so its loads overlap without it).
constexpr int kUnroll = 4;

// this thread's share of elements [e0, e1) of the row that starts at flat index `base`: the scalar head, the vectors
// gt, gt + group, ... (kUnroll at a time), then the scalar tail
template <typename T, bool VEC>
__device__ __forceinline__ Acc scan_row(const T* __restrict__ row, int64_t base, int64_t e0, int64_t e1, int gt,
                                        int group, int64_t t, const float* __restrict__ w, bool smooth) {
  Acc a{-INFINITY, 0.f, 0.f, 0.f};
  int64_t v0 = e1, v1 = e1;
  if (VEC) vec_range(base, e0, e1, v0, v1);
  for (int64_t e = e0 + gt; e < v0; e += group) {
    const float v[1] = {nk_to_f32<T>(row[e])};
    fold(a, v, e, t, w, smooth);
  }
  if (VEC) {
    const int64_t npk = (v1 - v0) / kVec;
    int64_t p = gt;
    for (; p + (kUnroll - 1) * group < npk; p += kUnroll * group) {
      NkPack8<T> pk[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) pk[u].load(row + v0 + (p + u * group) * kVec);
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        float v[kVec];
#pragma unroll
        for (int i = 0; i < kVec; ++i) v[i] = pk[u].get(i);
        fold(a, v, v0 + (p + u * group) * kVec, t, w, smooth);
      }
    }
    for (; p < npk; p += group) {
      NkPack8<T> pk;
      pk.load(row + v0 + p * kVec);
      float v[kVec];
#pragma unroll
      for (int i = 0; i < kVec; ++i) v[i] = pk.get(i);
      fold(a, v, v0 + p * kVec, t, w, smooth);
    }
  }
  for (int64_t e = v1 + gt; e < e1; e += group) {
    const float v[1] = {nk_to_f32<T>(row[e])};
    fold(a, v, e, t, w, smooth);
  }
  return a;
}

// lse and the loss of one position from its merged pair; W = sum of the weights
__device__ __forceinline__ float position_loss(const Acc& a, float wt, float W, const Args& g, bool smooth, float* lse) {
  *lse = a.m + logf(a.s);
  float l = (1.f - g.eps) * wt * (*lse - a.xt);
  if (smooth) l += g.eps_c * (W * *lse - a.wx);
  return l;
}

// the block's (loss, weight) sums, in a fixed order, into part[blockIdx.x]
__device__ __forceinline__ void block_partial(double2* __restrict__ part, double dl, double dw) {
  __shared__ double2 red[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dl += __shfl_xor_sync(0xffffffffu, dl, o);
    dw += __shfl_xor_sync(0xffffffffu, dw, o);
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_double2(dl, dw);
  __syncthreads();
  if (threadIdx.x == 0) {
    double2 r = red[0];
    for (int i = 1; i < kThreads / 32; ++i) r.x += red[i].x, r.y += red[i].y;
    part[blockIdx.x] = r;
  }
}

// ------------------------------------------------------------------------------------------------------ forward
// s == 1: one work item = (row, chunk); `group` threads per item.  splits == 1: the item's pair gives the row's lse and
// loss here; otherwise the pair goes to split_part[item] for ce_fwd_merge.
template <typename T, typename TT, bool VEC>
__global__ void __launch_bounds__(kThreads) ce_fwd_rows(double2* __restrict__ part, Acc* __restrict__ split_part,
                                                        float* __restrict__ lse_out, const T* __restrict__ x,
                                                        const TT* __restrict__ target, const float* __restrict__ w,
                                                        const float* __restrict__ wsum, Args g, bool smooth) {
  __shared__ Acc wacc[kThreads / 32];
  const int group = g.group, gpb = kThreads / group;
  const int gid = threadIdx.x / group, gt = threadIdx.x % group;
  const float fc = float(g.c);
  const float W = wsum ? *wsum : fc;
  double dl = 0.0, dw = 0.0;
  const int64_t items = g.n * g.splits;
  const int64_t step = int64_t(gridDim.x) * gpb;
  for (Walk wk(int64_t(blockIdx.x) * gpb + gid, step, g.splits); wk.idx < items; wk.next(step)) {
    const int64_t it = wk.idx, row = wk.row, chunk = wk.col;
    const int64_t t = target_class<TT>(target[row], fc, g.ignore);
    if (t < 0) {  // the same for every thread of the item (the whole CTA when group == kThreads)
      if (gt == 0 && g.splits == 1) lse_out[row] = 0.f;
      continue;
    }
    const int64_t e0 = chunk * g.chunk, e1 = min(g.c, e0 + g.chunk);
    Acc a = warp_merge(scan_row<T, VEC>(x + row * g.c, row * g.c, e0, e1, gt, group, t, w, smooth));
    if (group > 32) {  // warps in order
      if ((threadIdx.x & 31) == 0) wacc[threadIdx.x >> 5] = a;
      __syncthreads();
      if (threadIdx.x == 0)
        for (int i = 1; i < kThreads / 32; ++i) a = merge(a, wacc[i]);
      __syncthreads();
    }
    if (gt != 0) continue;
    if (g.splits > 1) {
      split_part[it] = a;
    } else {
      const float wt = wt_of(w, t);
      dl += position_loss(a, wt, W, g, smooth, lse_out + row);
      dw += wt;
    }
  }
  if (part) block_partial(part, dl, dw);
}

// split rows: one thread per row merges the row's chunk pairs in ascending chunk order
template <typename TT>
__global__ void __launch_bounds__(kThreads) ce_fwd_merge(double2* __restrict__ part, float* __restrict__ lse_out,
                                                         const Acc* __restrict__ split_part, const TT* __restrict__ target,
                                                         const float* __restrict__ w, const float* __restrict__ wsum,
                                                         Args g, bool smooth) {
  const float fc = float(g.c);
  const float W = wsum ? *wsum : fc;
  double dl = 0.0, dw = 0.0;
  for (int64_t row = int64_t(blockIdx.x) * kThreads + threadIdx.x; row < g.n; row += int64_t(gridDim.x) * kThreads) {
    const int64_t t = target_class<TT>(target[row], fc, g.ignore);
    if (t < 0) {
      lse_out[row] = 0.f;
      continue;
    }
    Acc a = split_part[row * g.splits];
    for (int k = 1; k < g.splits; ++k) a = merge(a, split_part[row * g.splits + k]);
    const float wt = wt_of(w, t);
    dl += position_loss(a, wt, W, g, smooth, lse_out + row);
    dw += wt;
  }
  block_partial(part, dl, dw);
}

// s > 1: one thread per position q = (i, j), classes at x[(i*c + k)*s + j]
template <typename T, typename TT>
__global__ void __launch_bounds__(kThreads) ce_fwd_spatial(double2* __restrict__ part, float* __restrict__ lse_out,
                                                           const T* __restrict__ x, const TT* __restrict__ target,
                                                           const float* __restrict__ w, const float* __restrict__ wsum,
                                                           Args g, bool smooth) {
  const float fc = float(g.c);
  const float W = wsum ? *wsum : fc;
  double dl = 0.0, dw = 0.0;
  const int64_t total = g.n * g.s;
  const int64_t step = int64_t(gridDim.x) * kThreads;
  for (Walk wk(int64_t(blockIdx.x) * kThreads + threadIdx.x, step, g.s); wk.idx < total; wk.next(step)) {
    const int64_t q = wk.idx;
    const int64_t t = target_class<TT>(target[q], fc, g.ignore);
    if (t < 0) {
      lse_out[q] = 0.f;
      continue;
    }
    const T* p = x + wk.row * g.c * g.s + wk.col;
    Acc a{-INFINITY, 0.f, 0.f, 0.f};
    int64_t k = 0;
    for (; k + 4 <= g.c; k += 4) {
      float v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = nk_to_f32<T>(p[(k + u) * g.s]);
      fold(a, v, k, t, w, smooth);
    }
    for (; k < g.c; ++k) {
      const float v[1] = {nk_to_f32<T>(p[k * g.s])};
      fold(a, v, k, t, w, smooth);
    }
    const float wt = wt_of(w, t);
    dl += position_loss(a, wt, W, g, smooth, lse_out + q);
    dw += wt;
  }
  block_partial(part, dl, dw);
}

// denominator and loss from the per-block sums, one warp in a fixed order; an empty or fully ignored Mean is 0/0 = NaN
__global__ void ce_finish(float* __restrict__ loss, float* __restrict__ denom, const double2* __restrict__ part,
                          int nparts, int mean) {
  double l = 0.0, d = 0.0;
  for (int i = threadIdx.x; i < nparts; i += 32) l += part[i].x, d += part[i].y;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_xor_sync(0xffffffffu, l, o);
    d += __shfl_xor_sync(0xffffffffu, d, o);
  }
  if (threadIdx.x == 0) {
    *denom = float(d);
    *loss = float(mean ? l / d : l);
  }
}

// W = sum of the class weights, one block in a fixed order (needed with label smoothing only)
__global__ void __launch_bounds__(kThreads) ce_weight_sum(float* __restrict__ out, const float* __restrict__ w,
                                                          int64_t c) {
  __shared__ double red[kThreads / 32];
  double s = 0.0;
  for (int64_t k = threadIdx.x; k < c; k += kThreads) s += double(w[k]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) r += red[i];
    *out = float(r);
  }
}

// ----------------------------------------------------------------------------------------------------- backward
// Per non-ignored position, with p = exp(x - lse), gs = g (Sum) or g / denominator (Mean):
//   dx_k = a*p_k - b*[k == t] - cw*w_k,  a = gs*((1 - eps)*w_t + eps/c*W),  b = gs*(1 - eps)*w_t,  cw = gs*eps/c;
// dx = beta*dx + that, the product and the add rounded separately; beta = 0 never reads dx.  Ignored positions get
// beta*dx (nothing is written when beta == 1).
struct Coef {
  float a, b, cw, lse;
  int64_t t;  // -1: ignored
};

template <typename TD>
__device__ __forceinline__ void store_grad(TD* p, float r, float beta) {
  *p = nk_from_f32<TD>(beta != 0.f ? __fadd_rn(__fmul_rn(beta, nk_to_f32<TD>(*p)), r) : r);
}

__device__ __forceinline__ float grad_of(float v, int64_t k, const Coef& q, const float* w, bool smooth) {
  float r = q.a * expf(v - q.lse);
  if (k == q.t) r -= q.b;
  if (smooth) r -= q.cw * wt_of(w, k);
  return r;
}

template <typename TT>
__device__ __forceinline__ Coef coef_of(TT raw, const float* lse, int64_t pos, const float* w, float gs, float W,
                                        const Args& g, float fc) {
  Coef q{0.f, 0.f, 0.f, 0.f, target_class<TT>(raw, fc, g.ignore)};
  if (q.t >= 0) {
    const float wt = wt_of(w, q.t);
    q.b = gs * ((1.f - g.eps) * wt);
    q.a = gs * ((1.f - g.eps) * wt + g.eps_c * W);
    q.cw = gs * g.eps_c;
    q.lse = lse[pos];
  }
  return q;
}

template <typename T, typename TD, typename TT, bool VEC>
__global__ void __launch_bounds__(kThreads) ce_bwd_rows(TD* __restrict__ dx, const T* __restrict__ x,
                                                        const TT* __restrict__ target, const float* __restrict__ w,
                                                        const float* __restrict__ wsum, const float* __restrict__ lse,
                                                        const float* __restrict__ denom, const float* __restrict__ gp,
                                                        Args g, bool smooth, int mean, float beta) {
  const int group = g.group, gpb = kThreads / group;
  const int gid = threadIdx.x / group, gt = threadIdx.x % group;
  const float fc = float(g.c);
  const float W = wsum ? *wsum : fc;
  const float gs = mean ? *gp / *denom : *gp;
  const int64_t items = g.n * g.splits;
  const int64_t step = int64_t(gridDim.x) * gpb;
  for (Walk wk(int64_t(blockIdx.x) * gpb + gid, step, g.splits); wk.idx < items; wk.next(step)) {
    const int64_t row = wk.row, chunk = wk.col;
    const Coef q = coef_of<TT>(target[row], lse, row, w, gs, W, g, fc);
    if (q.t < 0 && beta == 1.f) continue;
    const int64_t e0 = chunk * g.chunk, e1 = min(g.c, e0 + g.chunk);
    const T* xr = x + row * g.c;
    TD* dr = dx + row * g.c;
    int64_t v0 = e1, v1 = e1;
    if (VEC) vec_range(row * g.c, e0, e1, v0, v1);
    auto scalar = [&](int64_t k) {
      const float r = q.t < 0 ? 0.f : grad_of(nk_to_f32<T>(xr[k]), k, q, w, smooth);
      store_grad(dr + k, r, beta);
    };
    for (int64_t k = e0 + gt; k < v0; k += group) scalar(k);
    if (VEC) {
      const int64_t npk = (v1 - v0) / kVec;
      for (int64_t p = gt; p < npk; p += group) {
        const int64_t k0 = v0 + p * kVec;
        NkPack8<TD> o;
        if (beta != 0.f) o.load(dr + k0);
        if (q.t < 0) {
#pragma unroll
          for (int i = 0; i < kVec; ++i) o.set(i, beta != 0.f ? __fmul_rn(beta, o.get(i)) : 0.f);
        } else {
          NkPack8<T> v;
          v.load(xr + k0);
#pragma unroll
          for (int i = 0; i < kVec; ++i) {
            const float r = grad_of(v.get(i), k0 + i, q, w, smooth);
            o.set(i, beta != 0.f ? __fadd_rn(__fmul_rn(beta, o.get(i)), r) : r);
          }
        }
        o.store(dr + k0);
      }
    }
    for (int64_t k = v1 + gt; k < e1; k += group) scalar(k);
  }
}

template <typename T, typename TD, typename TT>
__global__ void __launch_bounds__(kThreads) ce_bwd_spatial(TD* __restrict__ dx, const T* __restrict__ x,
                                                           const TT* __restrict__ target, const float* __restrict__ w,
                                                           const float* __restrict__ wsum, const float* __restrict__ lse,
                                                           const float* __restrict__ denom, const float* __restrict__ gp,
                                                           Args g, bool smooth, int mean, float beta) {
  const float fc = float(g.c);
  const float W = wsum ? *wsum : fc;
  const float gs = mean ? *gp / *denom : *gp;
  const int64_t total = g.n * g.s;
  const int64_t step = int64_t(gridDim.x) * kThreads;
  for (Walk wk(int64_t(blockIdx.x) * kThreads + threadIdx.x, step, g.s); wk.idx < total; wk.next(step)) {
    const int64_t q = wk.idx;
    const Coef cf = coef_of<TT>(target[q], lse, q, w, gs, W, g, fc);
    if (cf.t < 0 && beta == 1.f) continue;
    const int64_t off = wk.row * g.c * g.s + wk.col;
    const T* xp = x + off;
    TD* dp = dx + off;
    for (int64_t k = 0; k < g.c; ++k) {
      const float r = cf.t < 0 ? 0.f : grad_of(nk_to_f32<T>(xp[k * g.s]), k, cf, w, smooth);
      store_grad(dp + k * g.s, r, beta);
    }
  }
}

// ------------------------------------------------------------------------------------------------------- host
inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int grid_for(nk_ctx* ctx, int64_t threads) {
  int64_t b = (threads + kThreads - 1) / kThreads;
  const int64_t cap = int64_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  return int(b < 1 ? 1 : b);
}

int check(nk_ctx* ctx, const char* who, int dtype, int target_dtype, int64_t n, int64_t c, int64_t s,
          float label_smoothing) {
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(target_dtype), "%s: bad dtype", who);
  NK_REQUIRE(ctx, n >= 0 && s >= 1 && c >= 1, "%s: need n >= 0, c >= 1 and s >= 1 (n = %lld, c = %lld, s = %lld)", who,
             (long long)n, (long long)c, (long long)s);
  NK_REQUIRE(ctx, c <= (int64_t(1) << 24), "%s: c = %lld exceeds 2^24, the range where f32 class ids are exact", who,
             (long long)c);
  // bf16 holds integers exactly only up to 256: larger class ids would silently select the wrong class
  NK_REQUIRE(ctx, target_dtype == NK_F32 || c <= 256,
             "%s: a bf16 target cannot hold class ids above 256 (c = %lld); pass the target as f32", who, (long long)c);
  NK_REQUIRE(ctx, label_smoothing >= 0.f && label_smoothing <= 1.f, "%s: label_smoothing %g outside [0, 1]", who,
             double(label_smoothing));
  return NK_OK;
}

// the layout of one call (forward and backward choose the same for the same shape, except that the backward's vector
// loads also need dx's alignment)
Args plan(nk_ctx* ctx, int64_t n, int64_t c, int64_t s, int64_t ignore, float eps, int esize) {
  Args g{n, c, s, c, 1, 32, ignore, eps, eps / float(c)};
  if (s == 1 && c * esize > kWarpRowBytes && n < kWarpMinRows) {
    g.group = kThreads;
    const int64_t want = kSplitRowsPerSm * ctx->sm_count;
    if (n > 0 && n < want && c >= kSplitMinCols) {
      int64_t splits = std::min<int64_t>((want + n - 1) / n * 2, c / kMinChunk);
      int64_t chunk = (c + splits - 1) / splits;
      chunk = (chunk + kVec - 1) / kVec * kVec;
      g.chunk = chunk;
      g.splits = int((c + chunk - 1) / chunk);
    }
  }
  return g;
}

template <typename T, typename TT>
int fwd_launch(nk_ctx* ctx, float* loss, float* lse, float* denom, const void* xv, const void* tv, const float* w,
               const Args& g, bool smooth, int mean) {
  const T* x = static_cast<const T*>(xv);
  const TT* t = static_cast<const TT*>(tv);
  const bool wsum_needed = smooth && w;
  const int64_t positions = g.n * g.s;
  int blocks = 0;
  if (positions > 0) {
    if (g.s > 1)
      blocks = grid_for(ctx, positions);
    else if (g.splits > 1)
      blocks = 1;
    else
      blocks = grid_for(ctx, g.n * g.group);
  }
  const size_t split_bytes = g.splits > 1 ? size_t(g.n) * g.splits * sizeof(Acc) : 0;
  const size_t bytes = size_t(std::max(blocks, 1)) * sizeof(double2) + split_bytes + (wsum_needed ? 16 : 0);
  void* ws = nullptr;
  int rc = nk_alloc_uninit(ctx, bytes, &ws);
  if (rc) return rc;
  double2* part = static_cast<double2*>(ws);
  Acc* split = reinterpret_cast<Acc*>(static_cast<char*>(ws) + size_t(std::max(blocks, 1)) * sizeof(double2));
  float* wsum = wsum_needed ? reinterpret_cast<float*>(static_cast<char*>(ws) + bytes - 16) : nullptr;
  rc = [&]() -> int {
    if (positions > 0) {
      if (wsum) {
        ce_weight_sum<<<1, kThreads, 0, ctx->stream>>>(wsum, w, g.c);
        NK_LAUNCHED(ctx, "cross_entropy_weight_sum");
      }
      if (g.s > 1) {
        ce_fwd_spatial<T, TT><<<blocks, kThreads, 0, ctx->stream>>>(part, lse, x, t, w, wsum, g, smooth);
        NK_LAUNCHED(ctx, "cross_entropy_fwd_spatial");
      } else {
        const bool vec = al16(x);
        const int rb = g.splits > 1 ? int(std::min<int64_t>(g.n * g.splits, int64_t(ctx->sm_count) * 8)) : blocks;
        double2* p = g.splits > 1 ? nullptr : part;
        if (vec)
          ce_fwd_rows<T, TT, true><<<rb, kThreads, 0, ctx->stream>>>(p, split, lse, x, t, w, wsum, g, smooth);
        else
          ce_fwd_rows<T, TT, false><<<rb, kThreads, 0, ctx->stream>>>(p, split, lse, x, t, w, wsum, g, smooth);
        NK_LAUNCHED(ctx, "cross_entropy_fwd_rows");
        if (g.splits > 1) {
          ce_fwd_merge<TT><<<1, kThreads, 0, ctx->stream>>>(part, lse, split, t, w, wsum, g, smooth);
          NK_LAUNCHED(ctx, "cross_entropy_fwd_merge");
        }
      }
    }
    ce_finish<<<1, 32, 0, ctx->stream>>>(loss, denom, part, blocks, mean);
    NK_LAUNCHED(ctx, "cross_entropy_finish");
    return NK_OK;
  }();
  const int frc = nk_free(ctx, ws);
  return rc ? rc : frc;
}

template <typename T, typename TD, typename TT>
int bwd_launch(nk_ctx* ctx, void* dxv, const void* xv, const void* tv, const float* w, const float* lse,
               const float* denom, const float* g, const Args& a, bool smooth, int mean, float beta) {
  TD* dx = static_cast<TD*>(dxv);
  const T* x = static_cast<const T*>(xv);
  const TT* t = static_cast<const TT*>(tv);
  void* ws = nullptr;
  float* wsum = nullptr;
  if (smooth && w) {
    int rc = nk_alloc_uninit(ctx, 16, &ws);
    if (rc) return rc;
    wsum = static_cast<float*>(ws);
  }
  int rc = [&]() -> int {
    if (wsum) {
      ce_weight_sum<<<1, kThreads, 0, ctx->stream>>>(wsum, w, a.c);
      NK_LAUNCHED(ctx, "cross_entropy_weight_sum");
    }
    if (a.s > 1) {
      ce_bwd_spatial<T, TD, TT><<<grid_for(ctx, a.n * a.s), kThreads, 0, ctx->stream>>>(dx, x, t, w, wsum, lse, denom, g,
                                                                                        a, smooth, mean, beta);
      NK_LAUNCHED(ctx, "cross_entropy_bwd_spatial");
      return NK_OK;
    }
    const bool vec = al16(x) && al16(dx);
    const int blocks = grid_for(ctx, a.n * a.splits * a.group);
    if (vec)
      ce_bwd_rows<T, TD, TT, true><<<blocks, kThreads, 0, ctx->stream>>>(dx, x, t, w, wsum, lse, denom, g, a, smooth,
                                                                        mean, beta);
    else
      ce_bwd_rows<T, TD, TT, false><<<blocks, kThreads, 0, ctx->stream>>>(dx, x, t, w, wsum, lse, denom, g, a, smooth,
                                                                         mean, beta);
    NK_LAUNCHED(ctx, "cross_entropy_bwd_rows");
    return NK_OK;
  }();
  if (ws) {
    const int frc = nk_free(ctx, ws);
    if (!rc) rc = frc;
  }
  return rc;
}

}  // namespace

extern "C" {

int nk_cross_entropy_fwd(nk_ctx* ctx, float* loss, float* lse, float* denom, const void* x, int dtype,
                         const void* target, int target_dtype, const float* weight, int64_t n, int64_t c, int64_t s,
                         int64_t ignore_index, float label_smoothing, int mean) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  static const char* who = "nk_cross_entropy_fwd";
  int rc = check(ctx, who, dtype, target_dtype, n, c, s, label_smoothing);
  if (rc) return rc;
  NK_REQUIRE(ctx, loss && denom && (n == 0 || (lse && x && target)), "%s: NULL pointer", who);
  const Args g = plan(ctx, n, c, s, ignore_index, label_smoothing, int(nk_dtype_size(dtype)));
  const bool smooth = label_smoothing != 0.f;
  using B = __nv_bfloat16;
  if (dtype == NK_BF16)
    return target_dtype == NK_BF16 ? fwd_launch<B, B>(ctx, loss, lse, denom, x, target, weight, g, smooth, mean)
                                   : fwd_launch<B, float>(ctx, loss, lse, denom, x, target, weight, g, smooth, mean);
  return target_dtype == NK_BF16 ? fwd_launch<float, B>(ctx, loss, lse, denom, x, target, weight, g, smooth, mean)
                                 : fwd_launch<float, float>(ctx, loss, lse, denom, x, target, weight, g, smooth, mean);
}

int nk_cross_entropy_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* x, int dtype, const void* target,
                         int target_dtype, const float* weight, const float* lse, const float* denom, const float* g,
                         int64_t n, int64_t c, int64_t s, int64_t ignore_index, float label_smoothing, int mean,
                         float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  static const char* who = "nk_cross_entropy_bwd";
  NK_REQUIRE(ctx, nk_dtype_ok(dx_dtype), "%s: bad dx dtype %d", who, dx_dtype);
  int rc = check(ctx, who, dtype, target_dtype, n, c, s, label_smoothing);
  if (rc) return rc;
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && x && target && lse && denom && g, "%s: NULL pointer", who);
  const Args a = plan(ctx, n, c, s, ignore_index, label_smoothing, int(nk_dtype_size(dtype)));
  const bool smooth = label_smoothing != 0.f;
  using B = __nv_bfloat16;
#define NK_CE_BWD(T, TD)                                                                                            \
  (target_dtype == NK_BF16 ? bwd_launch<T, TD, B>(ctx, dx, x, target, weight, lse, denom, g, a, smooth, mean, beta) \
                           : bwd_launch<T, TD, float>(ctx, dx, x, target, weight, lse, denom, g, a, smooth, mean, beta))
  if (dtype == NK_BF16) return dx_dtype == NK_BF16 ? NK_CE_BWD(B, B) : NK_CE_BWD(B, float);
  return dx_dtype == NK_BF16 ? NK_CE_BWD(float, B) : NK_CE_BWD(float, float);
#undef NK_CE_BWD
}

}  // extern "C"
