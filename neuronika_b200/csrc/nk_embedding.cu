// Embedding lookup and its deterministic gradient (nk_b200.h nk_embedding_fwd / nk_embedding_bwd).
//
// Forward: a gather of whole weight rows, one launch.  A block walks `rpb` output rows at a time, its threads spread
// over the row's 16-byte units (or elements, when the row length or a base rules 16-byte accesses out); the bits are
// copied, never converted.
// Backward, without float atomics:
//   1. a stable LSD radix sort of (key, position) pairs, 8 bits per pass, keys = the ids with invalid ids and
//      padding_idx mapped to the sentinel v: per pass a per-tile digit histogram, one exclusive scan of all tiles'
//      counts in digit-major order, and a stable scatter (warp match + per-warp counts keep each tile's order);
//   2. the sorted positions are cut into slots of kChunk consecutive entries.  One thread per (slot, column group)
//      sums each run of equal keys inside its slot sequentially, in ascending position order.  A row whose run lies
//      wholly in the slot is finished there; the first and last runs of a slot whose rows cross the slot's edges go to
//      f32 partials;
//   3. one thread per (row, column group) adds the partials of rows that span several slots in slot order, and writes
//      beta*dw into rows that received nothing.
// So a row's sum is a fixed function of the ids alone, and at most kChunk additions of it are chained before a
// partial is handed on: one id at every position is spread over n/kChunk slots instead of one serial chain.
#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 16;                      // keys per thread in a sort tile
constexpr int kTile = kThreads * kItems;        // keys per sort tile
constexpr int kChunk = 32;                      // sorted entries per slot of the backward's first summation level
constexpr int kScanThreads = 1024;

inline int grid_for(nk_ctx* ctx, int64_t rows, int rpb) {
  int64_t b = (rows + rpb - 1) / rpb;
  const int64_t cap = int64_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}
// rows walked at once by a block over rows of `units` work items each
inline int rows_per_block(int64_t units) { return units >= kThreads ? 1 : int(kThreads / units); }

// The key of one id: trunc(x) for 0 <= x < v, else (NaN, negative, too large, padding_idx) the sentinel v.  The test
// is made on the float: a NaN converted to an integer on the device would become the valid row 0.
template <typename TI>
__device__ __forceinline__ uint32_t id_key(TI raw, float fv, uint32_t v, int64_t pad) {
  const float x = nk_to_f32<TI>(raw);
  if (!(x >= 0.f && x < fv)) return v;
  const uint32_t k = uint32_t(x);
  return int64_t(k) == pad ? v : k;
}

// ------------------------------------------------------------------------------------------------------ forward
template <typename TI, typename U>
__global__ void __launch_bounds__(kThreads) emb_fwd(U* __restrict__ y, const U* __restrict__ w,
                                                    const TI* __restrict__ ids, int64_t n, int64_t units, float fv,
                                                    uint32_t v, int rpb) {
  const int tid = threadIdx.x;
  const int r0 = rpb == 1 ? 0 : tid / int(units);
  if (r0 >= rpb) return;
  const int64_t u0 = rpb == 1 ? tid : tid - int64_t(r0) * units;
  const int64_t ustep = rpb == 1 ? kThreads : units;
  for (int64_t p = int64_t(blockIdx.x) * rpb + r0; p < n; p += int64_t(gridDim.x) * rpb) {
    const uint32_t k = id_key<TI>(ids[p], fv, v, -1);
    U* yp = y + p * units;
    if (k == v) {
      for (int64_t u = u0; u < units; u += ustep) yp[u] = U{};
    } else {
      const U* wp = w + int64_t(k) * units;
      for (int64_t u = u0; u < units; u += ustep) yp[u] = wp[u];
    }
  }
}

// ------------------------------------------------------------------------------------------------- radix sort
// pass 0 reads the ids (keys computed on the fly, values = positions); later passes read the previous pass's pairs
template <typename TI>
__global__ void __launch_bounds__(kThreads) sort_hist(uint32_t* __restrict__ counts, const uint32_t* __restrict__ keys,
                                                      const TI* __restrict__ ids, int64_t n, int shift, int nblk,
                                                      float fv, uint32_t v, int64_t pad) {
  __shared__ uint32_t h[256];
  const int tid = threadIdx.x;
  h[tid] = 0;
  __syncthreads();
  const int64_t base = int64_t(blockIdx.x) * kTile;
#pragma unroll 4
  for (int i = 0; i < kItems; ++i) {
    const int64_t idx = base + i * kThreads + tid;
    if (idx < n) {
      const uint32_t k = keys ? keys[idx] : id_key<TI>(ids[idx], fv, v, pad);
      atomicAdd(&h[(k >> shift) & 255], 1u);
    }
  }
  __syncthreads();
  counts[int64_t(tid) * nblk + blockIdx.x] = h[tid];
}

// exclusive scan, in place, of `total` counts by one block
__global__ void __launch_bounds__(kScanThreads) sort_scan(uint32_t* __restrict__ counts, int64_t total) {
  __shared__ uint32_t wsum[kScanThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t per = (total + kScanThreads - 1) / kScanThreads;
  const int64_t beg = min(total, tid * per), end = min(total, beg + per);
  uint32_t s = 0;
  for (int64_t i = beg; i < end; ++i) s += counts[i];
  uint32_t incl = s;  // inclusive scan of the thread sums within the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t ws = wsum[lane], wi = ws;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    wsum[lane] = wi - ws;  // exclusive over warps
  }
  __syncthreads();
  uint32_t run = wsum[warp] + incl - s;
  for (int64_t i = beg; i < end; ++i) {
    const uint32_t c = counts[i];
    counts[i] = run;
    run += c;
  }
}

// Stable scatter of one tile: the tile is read in rounds of kThreads consecutive keys; inside a round, a key's place
// is its digit's running offset + the same digit's count in the lower warps + its rank among the equal digits of its
// own warp, so equal digits keep their order.
template <typename TI>
__global__ void __launch_bounds__(kThreads) sort_scatter(uint32_t* __restrict__ keys_out, uint32_t* __restrict__ pos_out,
                                                         const uint32_t* __restrict__ keys, const uint32_t* __restrict__ pos,
                                                         const TI* __restrict__ ids, const uint32_t* __restrict__ offsets,
                                                         int64_t n, int shift, int nblk, float fv, uint32_t v,
                                                         int64_t pad) {
  constexpr int kWarps = kThreads / 32;
  __shared__ uint32_t base[256];
  __shared__ uint32_t wc[kWarps][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  base[tid] = offsets[int64_t(tid) * nblk + blockIdx.x];
#pragma unroll
  for (int w = 0; w < kWarps; ++w) wc[w][tid] = 0;
  __syncthreads();
  const uint32_t lower = (1u << lane) - 1u;
  const int64_t tile = int64_t(blockIdx.x) * kTile;
  for (int i = 0; i < kItems; ++i) {
    const int64_t idx = tile + i * kThreads + tid;
    const bool valid = idx < n;
    uint32_t k = 0, p = 0;
    if (valid) {
      k = keys ? keys[idx] : id_key<TI>(ids[idx], fv, v, pad);
      p = keys ? pos[idx] : uint32_t(idx);
    }
    const uint32_t d = valid ? (k >> shift) & 255 : 256u + lane;  // an idle lane matches nobody
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    if (valid && __ffs(peers) - 1 == lane) wc[warp][d] = __popc(peers);
    __syncthreads();
    if (valid) {
      uint32_t off = base[d] + __popc(peers & lower);
      for (int w = 0; w < warp; ++w) off += wc[w][d];
      keys_out[off] = k;
      pos_out[off] = p;
    }
    __syncthreads();
    uint32_t t = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += wc[w][tid], wc[w][tid] = 0;
    base[tid] += t;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------ gradient summation
template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) Pack {
  T x[VEC];
};
template <typename T, int VEC>
__device__ __forceinline__ void load_f32(float (&out)[VEC], const T* p) {
  const Pack<T, VEC> v = *reinterpret_cast<const Pack<T, VEC>*>(p);
#pragma unroll
  for (int i = 0; i < VEC; ++i) out[i] = nk_to_f32<T>(v.x[i]);
}
template <typename T, int VEC>
__device__ __forceinline__ void store_f32(T* p, const float (&in)[VEC]) {
  Pack<T, VEC> v;
#pragma unroll
  for (int i = 0; i < VEC; ++i) v.x[i] = nk_from_f32<T>(in[i]);
  *reinterpret_cast<Pack<T, VEC>*>(p) = v;
}
// dw = beta*dw + sum, the product and the add rounded separately; beta = 0 never reads dw
template <typename TD, int VEC>
__device__ __forceinline__ void finish(TD* p, const float (&sum)[VEC], float beta) {
  float r[VEC];
  if (beta != 0.f) {
    load_f32<TD, VEC>(r, p);
#pragma unroll
    for (int i = 0; i < VEC; ++i) r[i] = __fadd_rn(__fmul_rn(beta, r[i]), sum[i]);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) r[i] = sum[i];
  }
  store_f32<TD, VEC>(p, r);
}

// first summation level: one thread per (slot, group of VEC columns)
template <typename TG, typename TD, int VEC>
__global__ void __launch_bounds__(kThreads) emb_slots(TD* __restrict__ dw, float* __restrict__ part,
                                                      const uint32_t* __restrict__ skey, const uint32_t* __restrict__ spos,
                                                      const TG* __restrict__ g, int64_t n, int64_t e, uint32_t v,
                                                      int64_t slots, int64_t units, int rpb, float beta) {
  const int tid = threadIdx.x;
  const int r0 = rpb == 1 ? 0 : tid / int(units);
  if (r0 >= rpb) return;
  const int64_t u0 = rpb == 1 ? tid : tid - int64_t(r0) * units;
  const int64_t ustep = rpb == 1 ? kThreads : units;
  for (int64_t j = int64_t(blockIdx.x) * rpb + r0; j < slots; j += int64_t(gridDim.x) * rpb) {
    const int64_t i0 = j * kChunk, i1 = min(i0 + kChunk, n);
    const uint32_t first = skey[i0];
    if (first == v) continue;  // the sentinel sorts last: nothing of this slot is summed
    const bool first_open = i0 > 0 && skey[i0 - 1] == first;
    for (int64_t u = u0; u < units; u += ustep) {
      const int64_t c = u * VEC;
      uint32_t cur = first;
      bool open = first_open;  // the running row began in an earlier slot
      // a finished run: the first run of a row begun earlier -> partial 2j, the last run of a row that goes on ->
      // partial 2j + 1, a whole row -> dw
      auto flush = [&](const float(&acc)[VEC], bool continues) {
        if (open)
          store_f32<float, VEC>(part + (2 * j) * e + c, acc);
        else if (continues)
          store_f32<float, VEC>(part + (2 * j + 1) * e + c, acc);
        else
          finish<TD, VEC>(dw + int64_t(cur) * e + c, acc, beta);
      };
      float acc[VEC];
      load_f32<TG, VEC>(acc, g + int64_t(spos[i0]) * e + c);
      bool done = false;
      for (int64_t i = i0 + 1; i < i1; ++i) {
        const uint32_t k = skey[i];
        float x[VEC];
        load_f32<TG, VEC>(x, g + int64_t(spos[i]) * e + c);
        if (k == cur) {
#pragma unroll
          for (int q = 0; q < VEC; ++q) acc[q] = __fadd_rn(acc[q], x[q]);
          continue;
        }
        flush(acc, false);
        if (k == v) {  // the sentinel sorts last: the rest of the slot is not summed
          done = true;
          break;
        }
        cur = k;
        open = false;
#pragma unroll
        for (int q = 0; q < VEC; ++q) acc[q] = x[q];
      }
      if (!done) flush(acc, i1 < n && skey[i1] == cur);
    }
  }
}

// first sorted index whose key is >= r, in [lo, n)
__device__ __forceinline__ int64_t lower_bound(const uint32_t* __restrict__ skey, int64_t lo, int64_t n, uint32_t r) {
  int64_t hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (skey[mid] < r)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// second level: one thread per (row, group of VEC columns).  A row spanning slots js..je is the last run of slot js
// (partial 2*js + 1) followed by the first run of each later slot (partial 2*k); a row without positions gets beta*dw.
template <typename TD, int VEC>
__global__ void __launch_bounds__(kThreads) emb_rows(TD* __restrict__ dw, const float* __restrict__ part,
                                                     const uint32_t* __restrict__ skey, int64_t n, int64_t e, int64_t v,
                                                     int64_t units, int rpb, float beta) {
  const int tid = threadIdx.x;
  const int r0 = rpb == 1 ? 0 : tid / int(units);
  if (r0 >= rpb) return;
  const int64_t u0 = rpb == 1 ? tid : tid - int64_t(r0) * units;
  const int64_t ustep = rpb == 1 ? kThreads : units;
  for (int64_t r = int64_t(blockIdx.x) * rpb + r0; r < v; r += int64_t(gridDim.x) * rpb) {
    const int64_t lb = lower_bound(skey, 0, n, uint32_t(r));
    TD* row = dw + r * e;
    if (lb == n || skey[lb] != uint32_t(r)) {
      if (beta == 1.f) continue;
      for (int64_t u = u0; u < units; u += ustep) {
        float x[VEC];
        if (beta != 0.f) {
          load_f32<TD, VEC>(x, row + u * VEC);
#pragma unroll
          for (int q = 0; q < VEC; ++q) x[q] = __fmul_rn(beta, x[q]);
        } else {
#pragma unroll
          for (int q = 0; q < VEC; ++q) x[q] = 0.f;
        }
        store_f32<TD, VEC>(row + u * VEC, x);
      }
      continue;
    }
    const int64_t js = lb / kChunk, je = (lower_bound(skey, lb, n, uint32_t(r) + 1) - 1) / kChunk;
    if (js == je) continue;  // finished by emb_slots
    for (int64_t u = u0; u < units; u += ustep) {
      const int64_t c = u * VEC;
      float acc[VEC];
      load_f32<float, VEC>(acc, part + (2 * js + 1) * e + c);
      for (int64_t k = js + 1; k <= je; ++k) {
        float x[VEC];
        load_f32<float, VEC>(x, part + (2 * k) * e + c);
#pragma unroll
        for (int q = 0; q < VEC; ++q) acc[q] = __fadd_rn(acc[q], x[q]);
      }
      finish<TD, VEC>(row + c, acc, beta);
    }
  }
}

int ids_ok(nk_ctx* ctx, const char* who, int ids_dtype, int64_t n, int64_t v, int64_t e) {
  NK_REQUIRE(ctx, nk_dtype_ok(ids_dtype), "%s: bad ids dtype %d", who, ids_dtype);
  NK_REQUIRE(ctx, n >= 0 && e >= 0 && v >= 0, "%s: negative size", who);
  NK_REQUIRE(ctx, v <= (int64_t(1) << 24), "%s: v = %lld exceeds 2^24, the range where f32 ids are exact", who,
             (long long)v);
  // bf16 holds integers exactly only up to 256: larger ids would silently select the wrong row
  NK_REQUIRE(ctx, ids_dtype == NK_F32 || v <= 256,
             "%s: a bf16 id table cannot hold ids above 256 (v = %lld); pass the ids as f32", who, (long long)v);
  return NK_OK;
}

template <typename TI, typename U>
int launch_fwd(nk_ctx* ctx, void* y, const void* w, const void* ids, int64_t n, int64_t units, int64_t v) {
  const int rpb = rows_per_block(units);
  emb_fwd<TI, U><<<grid_for(ctx, n, rpb), kThreads, 0, ctx->stream>>>((U*)y, (const U*)w, (const TI*)ids, n, units,
                                                                     float(v), uint32_t(v), rpb);
  NK_LAUNCHED(ctx, "embedding_fwd");
  return NK_OK;
}

template <typename TI>
int fwd_units(nk_ctx* ctx, void* y, const void* w, const void* ids, int64_t n, int64_t v, int64_t e, int dtype) {
  const int64_t row_bytes = e * int64_t(nk_dtype_size(dtype));
  const bool vec = row_bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(w) & 15) == 0;
  if (vec) return launch_fwd<TI, uint4>(ctx, y, w, ids, n, row_bytes / 16, v);
  if (dtype == NK_BF16) return launch_fwd<TI, uint16_t>(ctx, y, w, ids, n, e, v);
  return launch_fwd<TI, uint32_t>(ctx, y, w, ids, n, e, v);
}

// the sorted (key, position) pairs of the ids; *keys / *pos point into ws
template <typename TI>
int radix_sort(nk_ctx* ctx, const TI* ids, int64_t n, int64_t v, int64_t pad, uint32_t* ws, int nblk,
               const uint32_t** keys, const uint32_t** pos) {
  uint32_t *ka = ws, *kb = ws + n, *pa = ws + 2 * n, *pb = ws + 3 * n, *counts = ws + 4 * n;
  int bits = 0;
  while ((int64_t(1) << bits) <= v) ++bits;  // the keys are 0..v
  const int passes = (bits + 7) / 8;
  const uint32_t *kin = nullptr, *pin = nullptr;
  for (int p = 0; p < passes; ++p) {
    uint32_t* kout = p & 1 ? kb : ka;
    uint32_t* pout = p & 1 ? pb : pa;
    sort_hist<TI><<<nblk, kThreads, 0, ctx->stream>>>(counts, kin, ids, n, 8 * p, nblk, float(v), uint32_t(v), pad);
    NK_LAUNCHED(ctx, "embedding_sort_hist");
    sort_scan<<<1, kScanThreads, 0, ctx->stream>>>(counts, int64_t(256) * nblk);
    NK_LAUNCHED(ctx, "embedding_sort_scan");
    sort_scatter<TI><<<nblk, kThreads, 0, ctx->stream>>>(kout, pout, kin, pin, ids, counts, n, 8 * p, nblk, float(v),
                                                          uint32_t(v), pad);
    NK_LAUNCHED(ctx, "embedding_sort_scatter");
    kin = kout;
    pin = pout;
  }
  *keys = kin;
  *pos = pin;
  return NK_OK;
}

template <typename TG, typename TD, int VEC>
int launch_sums(nk_ctx* ctx, void* dw, float* part, const uint32_t* skey, const uint32_t* spos, const void* g,
                int64_t n, int64_t v, int64_t e, float beta) {
  const int64_t units = e / VEC;
  const int rpb = rows_per_block(units);
  if (n > 0) {
    const int64_t slots = (n + kChunk - 1) / kChunk;
    emb_slots<TG, TD, VEC><<<grid_for(ctx, slots, rpb), kThreads, 0, ctx->stream>>>(
        (TD*)dw, part, skey, spos, (const TG*)g, n, e, uint32_t(v), slots, units, rpb, beta);
    NK_LAUNCHED(ctx, "embedding_bwd_slots");
  }
  if (beta != 1.f || n > kChunk) {  // rows without positions to scale, or rows that may span slots
    emb_rows<TD, VEC><<<grid_for(ctx, v, rpb), kThreads, 0, ctx->stream>>>((TD*)dw, part, skey, n, e, v, units, rpb,
                                                                          beta);
    NK_LAUNCHED(ctx, "embedding_bwd_rows");
  }
  return NK_OK;
}

template <typename TG, typename TD>
int bwd_sums(nk_ctx* ctx, void* dw, float* part, const uint32_t* skey, const uint32_t* spos, const void* g, int64_t n,
             int64_t v, int64_t e, float beta) {
  const bool vec = e % 4 == 0 && (reinterpret_cast<uintptr_t>(dw) % (4 * sizeof(TD))) == 0 &&
                   (reinterpret_cast<uintptr_t>(g) % (4 * sizeof(TG))) == 0;
  if (vec) return launch_sums<TG, TD, 4>(ctx, dw, part, skey, spos, g, n, v, e, beta);
  return launch_sums<TG, TD, 1>(ctx, dw, part, skey, spos, g, n, v, e, beta);
}

}  // namespace

extern "C" {

int nk_embedding_fwd(nk_ctx* ctx, void* y, const void* w, const void* ids, int ids_dtype, int64_t n, int64_t v,
                     int64_t e, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  static const char* who = "nk_embedding_fwd";
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", who, dtype);
  int rc = ids_ok(ctx, who, ids_dtype, n, v, e);
  if (rc) return rc;
  if (n == 0 || e == 0) return NK_OK;
  NK_REQUIRE(ctx, y && ids && (w || v == 0), "%s: NULL pointer", who);
  if (ids_dtype == NK_BF16) return fwd_units<__nv_bfloat16>(ctx, y, w, ids, n, v, e, dtype);
  return fwd_units<float>(ctx, y, w, ids, n, v, e, dtype);
}

int nk_embedding_bwd(nk_ctx* ctx, void* dw, int dw_dtype, const void* ids, int ids_dtype, const void* g, int g_dtype,
                     int64_t n, int64_t v, int64_t e, int64_t padding_idx, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  static const char* who = "nk_embedding_bwd";
  NK_REQUIRE(ctx, nk_dtype_ok(dw_dtype) && nk_dtype_ok(g_dtype), "%s: bad dtype", who);
  int rc = ids_ok(ctx, who, ids_dtype, n, v, e);
  if (rc) return rc;
  NK_REQUIRE(ctx, padding_idx >= -1 && padding_idx < v, "%s: padding_idx %lld outside [-1, %lld)", who,
             (long long)padding_idx, (long long)v);
  if (n >= (int64_t(1) << 31))
    return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "%s: %lld positions exceed 2^31 - 1", who, (long long)n);
  if (v == 0 || e == 0 || (n == 0 && beta == 1.f)) return NK_OK;
  NK_REQUIRE(ctx, dw && (n == 0 || (ids && g)), "%s: NULL pointer", who);
  const int nblk = int((n + kTile - 1) / kTile);
  const int64_t slots = (n + kChunk - 1) / kChunk;
  const size_t sort_bytes = n > 0 ? (size_t(4) * n + size_t(256) * nblk) * 4 : 0;
  const size_t part_bytes = slots > 1 ? size_t(2) * slots * e * 4 : 0;
  void* ws = nullptr;
  if (sort_bytes + part_bytes) {
    rc = nk_alloc_uninit(ctx, sort_bytes + part_bytes, &ws);
    if (rc) return rc;
  }
  const uint32_t *skey = nullptr, *spos = nullptr;
  if (n > 0) {
    if (ids_dtype == NK_BF16)
      rc = radix_sort<__nv_bfloat16>(ctx, (const __nv_bfloat16*)ids, n, v, padding_idx, (uint32_t*)ws, nblk, &skey,
                                     &spos);
    else
      rc = radix_sort<float>(ctx, (const float*)ids, n, v, padding_idx, (uint32_t*)ws, nblk, &skey, &spos);
  }
  float* part = part_bytes ? (float*)((char*)ws + sort_bytes) : nullptr;
  if (!rc) {
    using B = __nv_bfloat16;
    if (dw_dtype == NK_BF16 && g_dtype == NK_BF16)
      rc = bwd_sums<B, B>(ctx, dw, part, skey, spos, g, n, v, e, beta);
    else if (dw_dtype == NK_BF16)
      rc = bwd_sums<float, B>(ctx, dw, part, skey, spos, g, n, v, e, beta);
    else if (g_dtype == NK_BF16)
      rc = bwd_sums<B, float>(ctx, dw, part, skey, spos, g, n, v, e, beta);
    else
      rc = bwd_sums<float, float>(ctx, dw, part, skey, spos, g, n, v, e, beta);
  }
  if (ws) {
    const int frc = nk_free(ctx, ws);
    if (!rc) rc = frc;
  }
  return rc;
}

}  // extern "C"
