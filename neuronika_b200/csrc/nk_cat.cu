// Concatenation along one axis (multi_concatenate/mod.rs, multi_stack/mod.rs: `cat` and `stack` are the same copy).
// The operands and the output are seen as (outer, len, inner) blocks: per output row (one `outer` index) operand i owns
// the contiguous run of run_i = len_i * inner elements at element col_i = sum_{j<i} run_j of that row.  So operand i is
// an (outer x run_i) 2-D copy with source pitch run_i and destination pitch sum_j run_j.
//
// One launch per NK_CAT_OPS_PER_LAUNCH operands: the operand table travels in the kernel parameters (__grid_constant__,
// read in place from the constant bank), so there is no allocation, no host-to-device copy and nothing that a stream
// capture cannot record.  The grid is the concatenation of every operand's CTAs: the host computes a CTA prefix over the
// operands and each CTA finds its operand with a binary search, so a 1-row operand beside a 4096-row one costs one CTA
// and does not serialise anything.  Each operand takes 16-byte accesses when its run, its column, the row pitch and its
// base pointers allow it, element accesses otherwise.
// When a launch's part of an output row is short (stack along the last axis: runs of one element) the forward walks the
// output in order instead and gathers each element from its operand, so the stores stay coalesced.
// All index maths is 64-bit.
#include <algorithm>
#include <limits.h>

#include "nk_internal.cuh"

// a named namespace: the kernels keep the same symbol names from build to build (torch.profiler traces)
namespace nk_cat {

constexpr int kThreads = 256;
constexpr int kOps = NK_CAT_OPS_PER_LAUNCH;
constexpr int kFwdUnroll = 4;        // 16-byte units (or elements) per thread and CTA in the forward
constexpr int kBwdVec = 8;           // elements per vector unit of the backward (16 bytes of the narrower type)
constexpr int kBwdUnrollVec = 2;
constexpr int kBwdUnrollScalar = 4;
constexpr int64_t kGatherBytes = 256; // a launch whose share of an output row is at most this long gathers

struct FwdTable {
  const void* src[kOps];
  int64_t run[kOps];       // elements of operand i per output row
  int64_t col[kOps];       // element offset of operand i's run within an output row
  int64_t blk[kOps + 1];   // CTA prefix
  uint64_t vec;            // bit i: operand i takes the 16-byte path
  int64_t pitch, outer;
  int count;
};
struct BwdTable {
  void* dst[kOps];
  int64_t run[kOps];
  int64_t col[kOps];
  int64_t blk[kOps + 1];
  float beta[kOps];
  uint64_t vec;            // bit i: 16-byte path
  uint64_t bf16;           // bit i: dst i holds bf16
  int64_t pitch, outer;
  int count;
};
static_assert(sizeof(FwdTable) + sizeof(void*) <= 4096, "forward operand table exceeds the kernel parameter limit");
static_assert(sizeof(BwdTable) + sizeof(void*) <= 4096, "backward operand table exceeds the kernel parameter limit");

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// the operand whose CTAs include CTA b: the largest i with blk[i] <= b (empty operands own no CTA)
__device__ __forceinline__ int find_op(const int64_t* blk, int count, int64_t b) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (blk[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// q = a / b, r = a % b for non-negative a, b > 0; 32-bit division when both fit
__device__ __forceinline__ void divmod(int64_t a, int64_t b, int64_t& q, int64_t& r) {
  if (((uint64_t(a) | uint64_t(b)) >> 32) == 0) {
    const uint32_t q32 = uint32_t(a) / uint32_t(b);
    q = q32;
    r = int64_t(uint32_t(a) - q32 * uint32_t(b));
  } else {
    q = a / b;
    r = a - q * b;
  }
}

// ------------------------------------------------------------------------------------------------- forward
// CTA `cta` of one operand: units [cta*U, cta*U + U) of its (outer x run) block, U = kThreads * kFwdUnroll.  A unit is
// one element of type W (a 16-byte vector or one element); run, col and pitch are in units.
template <typename W>
__device__ __forceinline__ void copy_rows(W* __restrict__ y, const W* __restrict__ x, int64_t run, int64_t col,
                                          int64_t pitch, int64_t outer, int64_t cta) {
  const int64_t n = outer * run;
  const int64_t base = cta * (kThreads * kFwdUnroll) + threadIdx.x;
  W v[kFwdUnroll];
  int64_t d[kFwdUnroll];
#pragma unroll
  for (int k = 0; k < kFwdUnroll; ++k) {
    const int64_t u = base + k * kThreads;
    if (u < n) {
      int64_t row, c;
      divmod(u, run, row, c);
      d[k] = row * pitch + col + c;
      v[k] = x[u];
    }
  }
#pragma unroll
  for (int k = 0; k < kFwdUnroll; ++k)
    if (base + k * kThreads < n) y[d[k]] = v[k];
}

template <typename E>
__global__ void __launch_bounds__(kThreads) nk_cat_fwd_kernel(E* __restrict__ y, const __grid_constant__ FwdTable t) {
  const int64_t b = blockIdx.x;
  const int i = find_op(t.blk, t.count, b);
  constexpr int V = 16 / int(sizeof(E));
  if ((t.vec >> i) & 1)
    copy_rows<uint4>(reinterpret_cast<uint4*>(y), static_cast<const uint4*>(t.src[i]), t.run[i] / V, t.col[i] / V,
                     t.pitch / V, t.outer, b - t.blk[i]);
  else
    copy_rows<E>(y, static_cast<const E*>(t.src[i]), t.run[i], t.col[i], t.pitch, t.outer, b - t.blk[i]);
}

// short rows: thread e writes element e of the launch's (outer x width) slice of the output, in order
template <typename E>
__global__ void __launch_bounds__(kThreads) nk_cat_gather_kernel(E* __restrict__ y, const __grid_constant__ FwdTable t) {
  __shared__ const E* s_src[kOps];
  __shared__ int64_t s_col[kOps], s_run[kOps];
  const int64_t col0 = t.col[0];
  for (int k = threadIdx.x; k < t.count; k += kThreads) {
    s_src[k] = static_cast<const E*>(t.src[k]);
    s_col[k] = t.col[k] - col0;
    s_run[k] = t.run[k];
  }
  __syncthreads();
  const int64_t width = t.col[t.count - 1] + t.run[t.count - 1] - col0;
  const int64_t n = t.outer * width;
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  for (int64_t e = int64_t(blockIdx.x) * kThreads + threadIdx.x; e < n; e += stride) {
    int64_t o, j;
    divmod(e, width, o, j);
    int lo = 0, hi = t.count - 1;   // the largest k with s_col[k] <= j: the operand that owns column j
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_col[mid] <= j) lo = mid; else hi = mid - 1;
    }
    y[o * t.pitch + col0 + j] = s_src[lo][o * s_run[lo] + (j - s_col[lo])];
  }
}

// ------------------------------------------------------------------------------------------------- backward
// 8 elements of T at a 16-byte aligned p
template <typename T>
__device__ __forceinline__ void ld8(float (&v)[8], const T* __restrict__ p) {
  constexpr int per = 16 / int(sizeof(T));
#pragma unroll
  for (int k = 0; k < 8 / per; ++k) {
    const uint4 r = reinterpret_cast<const uint4*>(p)[k];
    const T* e = reinterpret_cast<const T*>(&r);
#pragma unroll
    for (int i = 0; i < per; ++i) v[k * per + i] = nk_to_f32<T>(e[i]);
  }
}
template <typename T>
__device__ __forceinline__ void st8(T* __restrict__ p, const float (&v)[8]) {
  constexpr int per = 16 / int(sizeof(T));
#pragma unroll
  for (int k = 0; k < 8 / per; ++k) {
    uint4 r;
    T* e = reinterpret_cast<T*>(&r);
#pragma unroll
    for (int i = 0; i < per; ++i) e[i] = nk_from_f32<T>(v[k * per + i]);
    reinterpret_cast<uint4*>(p)[k] = r;
  }
}

// dx = beta*dx + g; dx is not read when beta is 0 (it may hold anything, NaN included)
template <typename TG, typename TD>
__device__ __forceinline__ void acc_rows(TD* __restrict__ dx, const TG* __restrict__ g, float beta, bool vec,
                                         int64_t run, int64_t col, int64_t pitch, int64_t outer, int64_t cta) {
  if (vec) {
    const int64_t runv = run / kBwdVec, n = outer * runv;
    const int64_t base = cta * (kThreads * kBwdUnrollVec) + threadIdx.x;
    float v[kBwdUnrollVec][8];
#pragma unroll
    for (int k = 0; k < kBwdUnrollVec; ++k) {
      const int64_t u = base + k * kThreads;
      if (u < n) {
        int64_t row, c;
        divmod(u, runv, row, c);
        ld8<TG>(v[k], g + row * pitch + col + c * kBwdVec);
      }
    }
#pragma unroll
    for (int k = 0; k < kBwdUnrollVec; ++k) {
      const int64_t u = base + k * kThreads;
      if (u < n) {
        if (beta != 0.f) {
          float d[8];
          ld8<TD>(d, dx + u * kBwdVec);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[k][i] = __fmaf_rn(beta, d[i], v[k][i]);
        }
        st8<TD>(dx + u * kBwdVec, v[k]);
      }
    }
  } else {
    const int64_t n = outer * run;
    const int64_t base = cta * (kThreads * kBwdUnrollScalar) + threadIdx.x;
    float v[kBwdUnrollScalar];
#pragma unroll
    for (int k = 0; k < kBwdUnrollScalar; ++k) {
      const int64_t u = base + k * kThreads;
      if (u < n) {
        int64_t row, c;
        divmod(u, run, row, c);
        v[k] = nk_to_f32<TG>(g[row * pitch + col + c]);
      }
    }
#pragma unroll
    for (int k = 0; k < kBwdUnrollScalar; ++k) {
      const int64_t u = base + k * kThreads;
      if (u < n) {
        float r = v[k];
        if (beta != 0.f) r = __fmaf_rn(beta, nk_to_f32<TD>(dx[u]), r);
        dx[u] = nk_from_f32<TD>(r);
      }
    }
  }
}

template <typename TG>
__global__ void __launch_bounds__(kThreads) nk_cat_bwd_kernel(const TG* __restrict__ g,
                                                               const __grid_constant__ BwdTable t) {
  const int64_t b = blockIdx.x;
  const int i = find_op(t.blk, t.count, b);
  const bool vec = (t.vec >> i) & 1;
  if ((t.bf16 >> i) & 1)
    acc_rows<TG, __nv_bfloat16>(static_cast<__nv_bfloat16*>(t.dst[i]), g, t.beta[i], vec, t.run[i], t.col[i], t.pitch,
                                t.outer, b - t.blk[i]);
  else
    acc_rows<TG, float>(static_cast<float*>(t.dst[i]), g, t.beta[i], vec, t.run[i], t.col[i], t.pitch, t.outer,
                        b - t.blk[i]);
}

// ------------------------------------------------------------------------------------------------- host side
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// shared argument checks: sizes, and the row pitch / element count without int64 overflow
static int cat_sizes(nk_ctx* ctx, const char* who, const int64_t* lens, int count, int64_t outer, int64_t inner,
                     int64_t& pitch, int64_t& n) {
  NK_REQUIRE(ctx, count >= 0, "%s: negative operand count %d", who, count);
  NK_REQUIRE(ctx, count == 0 || lens, "%s: NULL lens", who);
  NK_REQUIRE(ctx, outer >= 0 && inner >= 0, "%s: negative outer (%lld) or inner (%lld)", who, (long long)outer,
             (long long)inner);
  int64_t total = 0;
  for (int i = 0; i < count; ++i) {
    NK_REQUIRE(ctx, lens[i] >= 0, "%s: operand %d has negative length %lld", who, i, (long long)lens[i]);
    NK_REQUIRE(ctx, !__builtin_add_overflow(total, lens[i], &total), "%s: total length overflows", who);
  }
  NK_REQUIRE(ctx, !__builtin_mul_overflow(total, inner, &pitch) && !__builtin_mul_overflow(pitch, outer, &n),
             "%s: output size overflows int64", who);
  return NK_OK;
}

}  // namespace nk_cat

using namespace nk_cat;

extern "C" {

int nk_cat_fwd(nk_ctx* ctx, void* y, const void* const* xs, const int64_t* lens, int count, int64_t outer,
               int64_t inner, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_cat_fwd: bad dtype %d", dtype);
  int64_t pitch, n;
  if (int rc = cat_sizes(ctx, "nk_cat_fwd", lens, count, outer, inner, pitch, n)) return rc;
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, y && xs, "nk_cat_fwd: NULL pointer");
  const int64_t es = int64_t(nk_dtype_size(dtype)), V = 16 / es;
  // every table first: nothing is launched when one of them is invalid
  std::vector<FwdTable> tabs;
  int64_t col = 0;
  for (int first = 0; first < count; first += kOps) {
    FwdTable t = {};
    t.count = std::min(kOps, count - first);
    t.pitch = pitch;
    t.outer = outer;
    int64_t blocks = 0;
    for (int k = 0; k < t.count; ++k) {
      const int i = first + k;
      const int64_t run = lens[i] * inner;
      NK_REQUIRE(ctx, run == 0 || xs[i], "nk_cat_fwd: operand %d is NULL", i);
      t.src[k] = xs[i];
      t.run[k] = run;
      t.col[k] = col;
      const bool vec = run % V == 0 && col % V == 0 && pitch % V == 0 && aligned16(xs[i]) && aligned16(y);
      if (vec) t.vec |= uint64_t(1) << k;
      t.blk[k] = blocks;
      blocks += ceil_div(outer * (vec ? run / V : run), kThreads * kFwdUnroll);
      col += run;
    }
    t.blk[t.count] = blocks;
    NK_REQUIRE(ctx, blocks <= INT_MAX, "nk_cat_fwd: %lld CTAs exceed the grid limit", (long long)blocks);
    if (blocks > 0) tabs.push_back(t);
  }
  for (const FwdTable& t : tabs) {
    const int64_t width = t.col[t.count - 1] + t.run[t.count - 1] - t.col[0];
    if (width * es <= kGatherBytes) {
      const int grid = int(std::min<int64_t>(ceil_div(t.outer * width, kThreads), int64_t(ctx->sm_count) * 8));
      NK_DISPATCH_DTYPE(dtype, T, { nk_cat_gather_kernel<T><<<grid, kThreads, 0, ctx->stream>>>((T*)y, t); });
    } else {
      const int grid = int(t.blk[t.count]);
      NK_DISPATCH_DTYPE(dtype, T, { nk_cat_fwd_kernel<T><<<grid, kThreads, 0, ctx->stream>>>((T*)y, t); });
    }
    NK_LAUNCHED(ctx, "cat_fwd");
  }
  return NK_OK;
}

int nk_cat_bwd(nk_ctx* ctx, void* const* dxs, const int* dx_dtypes, const float* betas, const void* g, int g_dtype,
               const int64_t* lens, int count, int64_t outer, int64_t inner) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(g_dtype), "nk_cat_bwd: bad gradient dtype %d", g_dtype);
  int64_t pitch, n;
  if (int rc = cat_sizes(ctx, "nk_cat_bwd", lens, count, outer, inner, pitch, n)) return rc;
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, g && dxs && dx_dtypes && betas, "nk_cat_bwd: NULL pointer");
  std::vector<void*> seen;
  for (int i = 0; i < count; ++i) {
    if (!dxs[i] || lens[i] * inner == 0) continue;
    NK_REQUIRE(ctx, nk_dtype_ok(dx_dtypes[i]), "nk_cat_bwd: operand %d has bad dtype %d", i, dx_dtypes[i]);
    seen.push_back(dxs[i]);
  }
  std::sort(seen.begin(), seen.end());
  NK_REQUIRE(ctx, std::adjacent_find(seen.begin(), seen.end()) == seen.end(),
             "nk_cat_bwd: two operands share one gradient buffer (accumulate them in separate calls)");
  std::vector<BwdTable> tabs;
  int64_t col = 0;
  for (int first = 0; first < count; first += kOps) {
    BwdTable t = {};
    t.count = std::min(kOps, count - first);
    t.pitch = pitch;
    t.outer = outer;
    int64_t blocks = 0;
    for (int k = 0; k < t.count; ++k) {
      const int i = first + k;
      const int64_t run = lens[i] * inner;
      t.dst[k] = dxs[i];
      t.run[k] = run;
      t.col[k] = col;
      t.blk[k] = blocks;
      col += run;
      if (!dxs[i] || run == 0) continue;
      t.beta[k] = betas[i];
      if (dx_dtypes[i] == NK_BF16) t.bf16 |= uint64_t(1) << k;
      const bool vec = run % kBwdVec == 0 && t.col[k] % kBwdVec == 0 && pitch % kBwdVec == 0 && aligned16(g) &&
                       aligned16(dxs[i]);
      if (vec) t.vec |= uint64_t(1) << k;
      blocks += vec ? ceil_div(outer * (run / kBwdVec), kThreads * kBwdUnrollVec)
                    : ceil_div(outer * run, kThreads * kBwdUnrollScalar);
    }
    t.blk[t.count] = blocks;
    NK_REQUIRE(ctx, blocks <= INT_MAX, "nk_cat_bwd: %lld CTAs exceed the grid limit", (long long)blocks);
    if (blocks > 0) tabs.push_back(t);
  }
  for (const BwdTable& t : tabs) {
    NK_DISPATCH_DTYPE(g_dtype, TG, {
      nk_cat_bwd_kernel<TG><<<int(t.blk[t.count]), kThreads, 0, ctx->stream>>>((const TG*)g, t);
    });
    NK_LAUNCHED(ctx, "cat_bwd");
  }
  return NK_OK;
}

}  // extern "C"
