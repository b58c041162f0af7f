// Max, average and adaptive average pooling over the 1..3 sample dims of (planes, s...) with torch's semantics
// (nk_b200.h nk_max_pool_nd_* / nk_avg_pool_nd_* / nk_adaptive_avg_pool_nd_*).
//
// Forward, small windows: one thread computes V adjacent outputs along the last axis (V = 8 bf16, 4 f32, one 16-byte
// vector) and stores them with 16-byte stores where aligned.  The common last-axis shapes (k2 s2 p0, k3 s2 p1) load each
// window row of the V outputs as one segment with 16-byte loads when the rows are 16-byte aligned and the segment is in
// bounds; every other shape, tail and misaligned base reads scalars.  Each output scans its window in row-major order:
// max keeps the first of equal maxima (the last NaN), averages add in f32 in that order.
// Forward, large windows (kLargeWindow elements or more): one warp per output.  The window's in-bounds elements, in
// row-major order, are dealt to the lanes in chunks of V (chunk c to lane c % 32); each lane scans its chunks in order,
// with one 16-byte load per chunk where the window is one aligned contiguous range (global pooling), and the lanes are
// combined by a fixed xor-shuffle tree (offsets 16, 8, 4, 2, 1).  Both orders depend on the shape alone.
// Backward: a gather without atomics: each input element sums, in f32 and in ascending output order, the gradients of
// the outputs whose windows hold it (max: where the saved index is the element; averages: g / divisor), then
// dx = beta*dx + sum with the product and the add rounded separately.
// Index math is 32-bit within a plane and 64-bit across planes.
#include <math.h>

#include "nk_internal.cuh"
#include "nk_pool.h"

namespace {

constexpr int kThreads = 256;
// Windows of at least this many elements (prod(k), or prod(ceil(L/O)) for the adaptive pool) are reduced by a warp: a
// thread scanning them alone would issue as many dependent loads per output as a warp has lanes.
constexpr int kLargeWindow = 32;
enum PoolKind { kMax = 0, kAvg = 1, kAdaptive = 2 };

struct PoolGeom {
  int in[3], out[3], k[3], s[3], p[3], d[3];  // 3 axes; a missing leading axis has in = out = k = s = d = 1, p = 0
  int in_plane, out_plane;
  int64_t planes;
  int include_pad;
};

inline int grid_for(nk_ctx* ctx, size_t work_items) {
  size_t b = (work_items + kThreads - 1) / kThreads;
  const size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}

// the in-bounds positions lo, lo + st, ... (n of them) of output o's window along axis a, and the window's divisor
// extent along that axis
struct Win {
  int lo, st, n, div;
};
template <int KIND>
__device__ __forceinline__ Win axis_window(const PoolGeom& g, int a, int o) {
  const int L = g.in[a];
  Win w;
  if (KIND == kAdaptive) {
    const int O = g.out[a];
    if (O == 1) {  // global along this axis: no division
      w.lo = 0, w.st = 1, w.n = L, w.div = L;
      return w;
    }
    w.lo = int(int64_t(o) * L / O);
    w.n = int((int64_t(o + 1) * L + O - 1) / O) - w.lo;
    w.st = 1;
    w.div = w.n;
    return w;
  }
  const int k = g.k[a], d = g.d[a], start = o * g.s[a] - g.p[a];
  int j0 = 0, j1 = 0;
  if (d == 1) {
    j0 = max(0, -start);
    j1 = min(k, L - start);
  } else {
    j0 = start < 0 ? (-start + d - 1) / d : 0;
    j1 = start >= L ? 0 : min(k, (L - start + d - 1) / d);
  }
  w.lo = start + j0 * d;
  w.st = d;
  w.n = max(0, j1 - j0);
  w.div = KIND == kAvg && g.include_pad ? min(start + k, L + g.p[a]) - start : w.n;
  return w;
}

// The outputs [lo, hi] along axis a whose windows can hold input position u, as quotients of numerators that grow by a
// fixed step with u: max / avg lo = ceil((u + p - d(k-1)) / s), hi = floor((u + p) / s); adaptive lo = floor(u*O / L),
// hi = floor(((u+1)*O - 1) / L).  Cand keeps quotient and remainder of both, so the next position costs no division.
struct Cand {
  int64_t qlo, rlo, qhi, rhi;  // floor quotients and remainders (lo's numerator is offset so that lo = qlo + (rlo > 0))
  int64_t step, den;
  __device__ __forceinline__ static void split(int64_t num, int64_t den, int64_t& q, int64_t& r) {
    if (num >= 0 && num <= INT32_MAX)  // the common case: a 32-bit division
      q = int(num) / int(den);
    else
      q = num >= 0 ? num / den : -((-num + den - 1) / den);
    r = num - q * den;
  }
  __device__ __forceinline__ static void bump(int64_t& q, int64_t& r, int64_t step, int64_t den) {
    r += step;
    while (r >= den) r -= den, ++q;
  }
  template <int KIND>
  __device__ __forceinline__ void init(const PoolGeom& g, int a, int u) {
    if (KIND == kAdaptive) {
      step = g.out[a], den = g.in[a];
      split(int64_t(u) * g.out[a], den, qlo, rlo);
      split(int64_t(u + 1) * g.out[a] - 1, den, qhi, rhi);
    } else {
      step = 1, den = g.s[a];
      split(int64_t(u) + g.p[a] - int64_t(g.d[a]) * (g.k[a] - 1), den, qlo, rlo);
      split(int64_t(u) + g.p[a], den, qhi, rhi);
    }
  }
  template <int KIND>
  __device__ __forceinline__ void range(const PoolGeom& g, int a, int& lo, int& hi) const {
    lo = int(KIND == kAdaptive ? qlo : max(int64_t(0), qlo + (rlo > 0)));
    hi = int(min(int64_t(g.out[a] - 1), qhi));
  }
  __device__ __forceinline__ void next() {
    bump(qlo, rlo, step, den);
    bump(qhi, rhi, step, den);
  }
};
template <int KIND>
__device__ __forceinline__ void candidates(const PoolGeom& g, int a, int u, int& lo, int& hi) {
  if (KIND == kAdaptive && g.out[a] == 1) {  // global along this axis
    lo = hi = 0;
    return;
  }
  Cand c;
  c.init<KIND>(g, a, u);
  c.range<KIND>(g, a, lo, hi);
}

// the scan of a max window: an element replaces the running maximum when it is greater or NaN; the first in-bounds
// element sets the index even when it is -inf
__device__ __forceinline__ void max_step(float& m, int& best, float v, int pos) {
  if (best < 0 || v > m || isnan(v)) {
    m = v;
    best = pos;
  }
}
// (va, ia) wins over (vb, ib) in the scan that holds both: the last NaN, else the greater value, else the first index
__device__ __forceinline__ bool max_wins(float va, int ia, float vb, int ib) {
  const bool na = isnan(va), nb = isnan(vb);
  if (na || nb) return na && (!nb || ia > ib);
  if (va != vb) return va > vb;
  return ia < ib;
}

template <typename T, int V>
__device__ __forceinline__ void store_outputs(T* y, int* idx, int64_t off, int count, const float (&val)[V],
                                              const int (&best)[V]) {
  if (count == V && (reinterpret_cast<uintptr_t>(y + off) & 15) == 0) {
    NkVec<T> v;
#pragma unroll
    for (int i = 0; i < V; ++i) v.set(i, val[i]);
    v.store(y + off);
  } else {
    for (int i = 0; i < V; ++i)
      if (i < count) y[off + i] = nk_from_f32<T>(val[i]);
  }
  if (!idx) return;
  if (count == V && (reinterpret_cast<uintptr_t>(idx + off) & 15) == 0) {
#pragma unroll
    for (int i = 0; i < V; i += 4)
      *reinterpret_cast<int4*>(idx + off + i) = make_int4(best[i], best[i + 1], best[i + 2], best[i + 3]);
  } else {
    for (int i = 0; i < V; ++i)
      if (i < count) idx[off + i] = best[i];
  }
}

// K2 > 0: the last axis has kernel K2, stride S2, padding P2 and dilation 1, so the window rows of V adjacent outputs
// are one segment of (V-1)*S2 + K2 elements; `rows_aligned`: every row of x starts on a 16-byte boundary
template <typename T, int KIND, int K2, int S2, int P2>
__global__ void __launch_bounds__(kThreads) pool_fwd_small(T* __restrict__ y, int* __restrict__ idx,
                                                           const T* __restrict__ x, PoolGeom g, bool rows_aligned) {
  constexpr int V = 16 / sizeof(T);
  const int groups = (g.out[2] + V - 1) / V;
  const int rows_per_plane = g.out[0] * g.out[1];
  const int64_t total = g.planes * rows_per_plane * groups;
  for (int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += int64_t(gridDim.x) * blockDim.x) {
    const int64_t row = t / groups;
    const int oc = int(t - row * groups) * V;
    const int64_t pl = row / rows_per_plane;
    const int r = int(row - pl * rows_per_plane);
    const int o0 = r / g.out[1], o1 = r - o0 * g.out[1];
    const T* xp = x + pl * g.in_plane;
    const Win w0 = axis_window<KIND>(g, 0, o0), w1 = axis_window<KIND>(g, 1, o1);
    Win w2[V];
    float acc[V];
    int best[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
      w2[i] = axis_window<KIND>(g, 2, min(oc + i, g.out[2] - 1));
      acc[i] = KIND == kMax ? -INFINITY : 0.f;
      best[i] = -1;
    }
    if constexpr (K2 > 0) {
      constexpr int SEG = (V - 1) * S2 + K2, MIS = (V - P2 % V) % V, NV = (MIS + SEG + V - 1) / V;
      const int a = oc * S2 - P2, al = a - MIS, L2 = g.in[2];
      const bool vec = rows_aligned && al >= 0 && al + NV * V <= L2;
      for (int j0 = 0; j0 < w0.n; ++j0)
        for (int j1 = 0; j1 < w1.n; ++j1) {
          const int rbase = ((w0.lo + j0 * w0.st) * g.in[1] + w1.lo + j1 * w1.st) * L2;
          const T* rp = xp + rbase;
          float seg[NV * V];
          if (vec) {
#pragma unroll
            for (int c = 0; c < NV; ++c) {
              NkVec<T> q;
              q.raw = __ldg(reinterpret_cast<const uint4*>(rp + al) + c);
#pragma unroll
              for (int e = 0; e < V; ++e) seg[c * V + e] = q.get(e);
            }
          } else {
#pragma unroll
            for (int e = 0; e < NV * V; ++e) seg[e] = al + e >= 0 && al + e < L2 ? nk_to_f32<T>(rp[al + e]) : 0.f;
          }
#pragma unroll
          for (int i = 0; i < V; ++i)
#pragma unroll
            for (int j = 0; j < K2; ++j) {
              const int u2 = a + i * S2 + j;
              if (u2 < 0 || u2 >= L2) continue;
              const float v = seg[MIS + i * S2 + j];
              if (KIND == kMax)
                max_step(acc[i], best[i], v, rbase + u2);
              else
                acc[i] = __fadd_rn(acc[i], v);
            }
        }
    } else {
      for (int j0 = 0; j0 < w0.n; ++j0)
        for (int j1 = 0; j1 < w1.n; ++j1) {
          const int rbase = ((w0.lo + j0 * w0.st) * g.in[1] + w1.lo + j1 * w1.st) * g.in[2];
          const T* rp = xp + rbase;
#pragma unroll
          for (int i = 0; i < V; ++i)
            for (int j2 = 0; j2 < w2[i].n; ++j2) {
              const int u2 = w2[i].lo + j2 * w2[i].st;
              const float v = nk_to_f32<T>(rp[u2]);
              if (KIND == kMax)
                max_step(acc[i], best[i], v, rbase + u2);
              else
                acc[i] = __fadd_rn(acc[i], v);
            }
        }
    }
    if (KIND != kMax) {
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] = __fdiv_rn(acc[i], float(int64_t(w0.div) * w1.div * w2[i].div));
    }
    store_outputs<T, V>(y, idx, pl * g.out_plane + int64_t(r) * g.out[2] + oc, min(V, g.out[2] - oc), acc, best);
  }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(kThreads) pool_fwd_large(T* __restrict__ y, int* __restrict__ idx,
                                                           const T* __restrict__ x, PoolGeom g) {
  constexpr int V = 16 / sizeof(T);
  const int lane = threadIdx.x & 31;
  const int64_t total = g.planes * g.out_plane;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  for (int64_t o = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; o < total; o += nwarps) {
    const int64_t pl = o / g.out_plane;
    const int r = int(o - pl * g.out_plane);
    const int o2 = r % g.out[2], o1 = (r / g.out[2]) % g.out[1], o0 = r / (g.out[2] * g.out[1]);
    const Win w0 = axis_window<KIND>(g, 0, o0), w1 = axis_window<KIND>(g, 1, o1), w2 = axis_window<KIND>(g, 2, o2);
    const int n12 = w1.n * w2.n, W = w0.n * n12;
    const int first = (w0.lo * g.in[1] + w1.lo) * g.in[2] + w2.lo;
    const int last = ((w0.lo + (w0.n - 1) * w0.st) * g.in[1] + w1.lo + (w1.n - 1) * w1.st) * g.in[2] + w2.lo +
                     (w2.n - 1) * w2.st;
    const T* xp = x + pl * g.in_plane;
    const bool contig = W > 0 && last - first + 1 == W;  // strictly increasing positions: contiguous iff span == count
    const bool vec = contig && (reinterpret_cast<uintptr_t>(xp + first) & 15) == 0;
    float acc = KIND == kMax ? -INFINITY : 0.f;
    int best = -1;
    for (int c = lane; c * V < W; c += 32) {
      const int q0 = c * V;
      if (vec && q0 + V <= W) {
        NkVec<T> q;
        q.raw = __ldg(reinterpret_cast<const uint4*>(xp + first + q0));
#pragma unroll
        for (int e = 0; e < V; ++e) {
          if (KIND == kMax)
            max_step(acc, best, q.get(e), first + q0 + e);
          else
            acc = __fadd_rn(acc, q.get(e));
        }
      } else {
        for (int q = q0; q < q0 + V && q < W; ++q) {
          int pos = first + q;
          if (!contig) {
            const int i0 = q / n12, rem = q - i0 * n12, i1 = rem / w2.n, i2 = rem - i1 * w2.n;
            pos = ((w0.lo + i0 * w0.st) * g.in[1] + w1.lo + i1 * w1.st) * g.in[2] + w2.lo + i2 * w2.st;
          }
          const float v = nk_to_f32<T>(xp[pos]);
          if (KIND == kMax)
            max_step(acc, best, v, pos);
          else
            acc = __fadd_rn(acc, v);
        }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float oa = __shfl_xor_sync(0xffffffffu, acc, off);
      if (KIND == kMax) {
        const int ob = __shfl_xor_sync(0xffffffffu, best, off);
        // a lane without elements (best < 0) never wins
        if (ob >= 0 && (best < 0 || max_wins(oa, ob, acc, best))) {
          acc = oa;
          best = ob;
        }
      } else {
        acc = __fadd_rn(acc, oa);
      }
    }
    if (lane == 0) {
      if (KIND == kMax) {
        y[o] = nk_from_f32<T>(acc);
        if (idx) idx[o] = best;
      } else {
        y[o] = nk_from_f32<T>(__fdiv_rn(acc, float(int64_t(w0.div) * w1.div * w2.div)));
      }
    }
  }
}

// dx = beta*dx + the gathered gradient, V adjacent elements of dx's last axis per thread
template <typename TD, typename TG, int KIND>
__global__ void __launch_bounds__(kThreads) pool_bwd(TD* __restrict__ dx, const TG* __restrict__ gy,
                                                     const int* __restrict__ idx, PoolGeom g, float beta) {
  constexpr int V = 16 / sizeof(TD);
  const int groups = (g.in[2] + V - 1) / V;
  const int rows_per_plane = g.in[0] * g.in[1];
  const int64_t total = g.planes * rows_per_plane * groups;
  for (int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += int64_t(gridDim.x) * blockDim.x) {
    const int64_t row = t / groups;
    const int uc = int(t - row * groups) * V;
    const int64_t pl = row / rows_per_plane;
    const int r = int(row - pl * rows_per_plane);
    const int u0 = r / g.in[1], u1 = r - u0 * g.in[1];
    int lo0, hi0, lo1, hi1;
    candidates<KIND>(g, 0, u0, lo0, hi0);
    candidates<KIND>(g, 1, u1, lo1, hi1);
    const TG* gp = gy + pl * g.out_plane;
    const int* ip = idx ? idx + pl * g.out_plane : nullptr;
    const int count = min(V, g.in[2] - uc);
    // the V elements' last-axis candidate ranges grow with u: visit their union once, each output's gradient (and
    // index, or divisor) loaded once, and add it to every element whose range holds it -- per element still in
    // ascending output order
    float sum[V];
    int lo2[V], hi2[V];
    Cand c2;
    c2.init<KIND>(g, 2, uc);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      sum[i] = 0.f;
      if (i > 0) c2.next();
      c2.range<KIND>(g, 2, lo2[i], hi2[i]);
      if (i >= count) lo2[i] = 0, hi2[i] = -1;  // past the row: no candidates, and the union ends at the last element's
    }
    const int rowflat = (u0 * g.in[1] + u1) * g.in[2] + uc;
    int last = hi2[0];
#pragma unroll
    for (int i = 1; i < V; ++i) last = max(last, hi2[i]);
    for (int a0 = lo0; a0 <= hi0; ++a0) {
      const int d0 = KIND == kMax ? 1 : axis_window<KIND>(g, 0, a0).div;
      for (int a1 = lo1; a1 <= hi1; ++a1) {
        const int d1 = KIND == kMax ? 1 : axis_window<KIND>(g, 1, a1).div;
        const int obase = (a0 * g.out[1] + a1) * g.out[2];
        for (int a2 = lo2[0]; a2 <= last; ++a2) {
          if (KIND == kMax) {
            const int hit = ip[obase + a2] - rowflat;  // the element this output's maximum came from
            if (hit < 0 || hit >= count) continue;
            const float gv = nk_to_f32<TG>(gp[obase + a2]);
#pragma unroll
            for (int i = 0; i < V; ++i)
              if (hit == i) sum[i] = __fadd_rn(sum[i], gv);
          } else {
            const float div = float(int64_t(d0) * d1 * axis_window<KIND>(g, 2, a2).div);
            const float c = __fdiv_rn(nk_to_f32<TG>(gp[obase + a2]), div);
#pragma unroll
            for (int i = 0; i < V; ++i)
              if (a2 >= lo2[i] && a2 <= hi2[i]) sum[i] = __fadd_rn(sum[i], c);
          }
        }
      }
    }
    TD* dp = dx + pl * g.in_plane + int64_t(r) * g.in[2] + uc;
    if (count == V && (reinterpret_cast<uintptr_t>(dp) & 15) == 0) {
      NkVec<TD> v;
      if (beta != 0.f) v.load(dp);
#pragma unroll
      for (int i = 0; i < V; ++i) v.set(i, beta != 0.f ? __fadd_rn(__fmul_rn(beta, v.get(i)), sum[i]) : sum[i]);
      v.store(dp);
    } else {
      for (int i = 0; i < count; ++i)
        dp[i] = nk_from_f32<TD>(beta != 0.f ? __fadd_rn(__fmul_rn(beta, nk_to_f32<TD>(dp[i])), sum[i]) : sum[i]);
    }
  }
}

// checks the arguments of every entry point and fills the geometry; *empty when there is nothing to compute
int make_geom(nk_ctx* ctx, const char* who, int kind, int64_t planes, int nsp, const int64_t* in_sp,
              const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
              const int64_t* dilation, int include_pad, PoolGeom* g, bool* empty) {
  NK_REQUIRE(ctx, nsp >= 1 && nsp <= 3, "%s: 1 to 3 sample dimensions (got %d)", who, nsp);
  NK_REQUIRE(ctx, planes >= 0 && in_sp && out_sp && (kind == kAdaptive || (k && stride && pad && dilation)),
             "%s: bad arguments", who);
  int64_t isz = 1, osz = 1;
  for (int a = 0; a < 3; ++a) g->in[a] = g->out[a] = g->k[a] = g->s[a] = g->d[a] = 1, g->p[a] = 0;
  for (int i = 0; i < nsp; ++i) {
    const int a = 3 - nsp + i;
    const int64_t L = in_sp[i], O = out_sp[i];
    if (kind == kAdaptive) {
      NK_REQUIRE(ctx, L >= 1 && O >= 1, "%s: input and output sizes must be >= 1 (axis %d: %lld, %lld)", who, i,
                 (long long)L, (long long)O);
    } else {
      char msg[160];
      NK_REQUIRE(ctx, !nk_pool_check_axis(who, i, L, k[i], stride[i], pad[i], dilation[i], msg, sizeof msg), "%s", msg);
      const int64_t lo = nk_pool_out_extent(L, k[i], stride[i], pad[i], dilation[i], false);
      const int64_t hi = nk_pool_out_extent(L, k[i], stride[i], pad[i], dilation[i], true);
      NK_REQUIRE(ctx, lo >= 1 && hi >= 1, "%s: output size would be < 1 (axis %d, input %lld)", who, i, (long long)L);
      NK_REQUIRE(ctx, O == lo || O == hi, "%s: output size %lld is neither %lld nor (ceil_mode) %lld (axis %d)", who,
                 (long long)O, (long long)lo, (long long)hi, i);
      g->k[a] = int(k[i]);
      g->s[a] = int(stride[i]);
      g->p[a] = int(pad[i]);
      g->d[a] = int(dilation[i]);
    }
    g->in[a] = int(L);
    g->out[a] = int(O);
    isz *= L;
    osz *= O;
    if (isz > INT32_MAX || osz > INT32_MAX || (k && k[i] * dilation[i] > INT32_MAX))
      return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 elements in a plane", who);
  }
  g->in_plane = int(isz);
  g->out_plane = int(osz);
  g->planes = planes;
  g->include_pad = include_pad;
  *empty = planes == 0;
  return NK_OK;
}

bool large_window(int kind, const PoolGeom& g) {
  int64_t vol = 1;
  for (int a = 0; a < 3; ++a) vol *= kind == kAdaptive ? (g.in[a] + g.out[a] - 1) / g.out[a] : g.k[a];
  return vol >= kLargeWindow;
}

template <typename T, int KIND>
int launch_fwd(nk_ctx* ctx, void* y, int* idx, const void* x, const PoolGeom& g) {
  constexpr int V = 16 / sizeof(T);
  if (large_window(KIND, g)) {
    const int blocks = grid_for(ctx, size_t(g.planes) * g.out_plane * 32);
    pool_fwd_large<T, KIND><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, idx, (const T*)x, g);
    NK_LAUNCHED(ctx, "pool_fwd_large");
    return NK_OK;
  }
  const int blocks = grid_for(ctx, size_t(g.planes) * g.out[0] * g.out[1] * ((g.out[2] + V - 1) / V));
  const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (size_t(g.in[2]) * sizeof(T)) % 16 == 0;
  const bool d1 = g.d[2] == 1;
  if (KIND != kAdaptive && d1 && g.k[2] == 2 && g.s[2] == 2 && g.p[2] == 0)
    pool_fwd_small<T, KIND, 2, 2, 0><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, idx, (const T*)x, g, aligned);
  else if (KIND != kAdaptive && d1 && g.k[2] == 3 && g.s[2] == 2 && g.p[2] == 1)
    pool_fwd_small<T, KIND, 3, 2, 1><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, idx, (const T*)x, g, aligned);
  else
    pool_fwd_small<T, KIND, 0, 0, 0><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, idx, (const T*)x, g, aligned);
  NK_LAUNCHED(ctx, "pool_fwd_small");
  return NK_OK;
}

template <int KIND>
int pool_fwd(nk_ctx* ctx, const char* who, void* y, int* idx, const void* x, int64_t planes, int nsp,
             const int64_t* in_sp, const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
             const int64_t* dilation, int include_pad, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", who, dtype);
  PoolGeom g;
  bool empty = false;
  int rc = make_geom(ctx, who, KIND, planes, nsp, in_sp, out_sp, k, stride, pad, dilation, include_pad, &g, &empty);
  if (rc || empty) return rc;
  NK_REQUIRE(ctx, y && x, "%s: NULL pointer", who);
  NK_DISPATCH_DTYPE(dtype, T, return (launch_fwd<T, KIND>(ctx, y, idx, x, g)));
}

template <typename TD, typename TG, int KIND>
int launch_bwd(nk_ctx* ctx, void* dx, const void* g, const int* idx, const PoolGeom& geo, float beta) {
  constexpr int V = 16 / sizeof(TD);
  const int blocks = grid_for(ctx, size_t(geo.planes) * geo.in[0] * geo.in[1] * ((geo.in[2] + V - 1) / V));
  pool_bwd<TD, TG, KIND><<<blocks, kThreads, 0, ctx->stream>>>((TD*)dx, (const TG*)g, idx, geo, beta);
  NK_LAUNCHED(ctx, "pool_bwd");
  return NK_OK;
}

template <int KIND>
int pool_bwd_entry(nk_ctx* ctx, const char* who, void* dx, int dx_dtype, const void* g, int g_dtype, const int* idx,
                   int64_t planes, int nsp, const int64_t* in_sp, const int64_t* out_sp, const int64_t* k,
                   const int64_t* stride, const int64_t* pad, const int64_t* dilation, int include_pad, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dx_dtype) && nk_dtype_ok(g_dtype), "%s: bad dtype", who);
  PoolGeom geo;
  bool empty = false;
  int rc = make_geom(ctx, who, KIND, planes, nsp, in_sp, out_sp, k, stride, pad, dilation, include_pad, &geo, &empty);
  if (rc || empty) return rc;
  NK_REQUIRE(ctx, dx && g && (KIND != kMax || idx), "%s: NULL pointer", who);
  if (dx_dtype == NK_BF16) {
    NK_DISPATCH_DTYPE(g_dtype, TG, return (launch_bwd<__nv_bfloat16, TG, KIND>(ctx, dx, g, idx, geo, beta)));
  }
  NK_DISPATCH_DTYPE(g_dtype, TG, return (launch_bwd<float, TG, KIND>(ctx, dx, g, idx, geo, beta)));
}

}  // namespace

extern "C" {

int nk_max_pool_nd_fwd(nk_ctx* ctx, void* y, int32_t* idx, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                       const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
                       const int64_t* dilation, int dtype) {
  return pool_fwd<kMax>(ctx, "nk_max_pool_nd_fwd", y, idx, x, planes, nsp, in_sp, out_sp, k, stride, pad, dilation, 1,
                        dtype);
}

int nk_max_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, const int32_t* idx,
                       int64_t planes, int nsp, const int64_t* in_sp, const int64_t* out_sp, const int64_t* k,
                       const int64_t* stride, const int64_t* pad, const int64_t* dilation, float beta) {
  return pool_bwd_entry<kMax>(ctx, "nk_max_pool_nd_bwd", dx, dx_dtype, g, g_dtype, idx, planes, nsp, in_sp, out_sp, k,
                              stride, pad, dilation, 1, beta);
}

int nk_avg_pool_nd_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                       const int64_t* out_sp, const int64_t* k, const int64_t* stride, const int64_t* pad,
                       int count_include_pad, int dtype) {
  const int64_t ones[3] = {1, 1, 1};
  return pool_fwd<kAvg>(ctx, "nk_avg_pool_nd_fwd", y, nullptr, x, planes, nsp, in_sp, out_sp, k, stride, pad, ones,
                        count_include_pad != 0, dtype);
}

int nk_avg_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int64_t planes, int nsp,
                       const int64_t* in_sp, const int64_t* out_sp, const int64_t* k, const int64_t* stride,
                       const int64_t* pad, int count_include_pad, float beta) {
  const int64_t ones[3] = {1, 1, 1};
  return pool_bwd_entry<kAvg>(ctx, "nk_avg_pool_nd_bwd", dx, dx_dtype, g, g_dtype, nullptr, planes, nsp, in_sp, out_sp,
                              k, stride, pad, ones, count_include_pad != 0, beta);
}

int nk_adaptive_avg_pool_nd_fwd(nk_ctx* ctx, void* y, const void* x, int64_t planes, int nsp, const int64_t* in_sp,
                                const int64_t* out_sp, int dtype) {
  return pool_fwd<kAdaptive>(ctx, "nk_adaptive_avg_pool_nd_fwd", y, nullptr, x, planes, nsp, in_sp, out_sp, nullptr,
                             nullptr, nullptr, nullptr, 0, dtype);
}

int nk_adaptive_avg_pool_nd_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int64_t planes,
                                int nsp, const int64_t* in_sp, const int64_t* out_sp, float beta) {
  return pool_bwd_entry<kAdaptive>(ctx, "nk_adaptive_avg_pool_nd_bwd", dx, dx_dtype, g, g_dtype, nullptr, planes, nsp,
                                   in_sp, out_sp, nullptr, nullptr, nullptr, nullptr, 0, beta);
}

}  // extern "C"
