// Dropout (dropout/mod.rs) with a counter-based generator, so that a mask is a pure function of (seed, call id, element)
// and can be restated exactly on the host, and so that a captured step draws a new mask on every replay.
//
// Generator: Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11), the
// generator of Random123 and cuRAND's philox4_32_10.  Key = the context's 64-bit seed; counter = (e/4, call id), both
// 64-bit; element e takes output word e%4.  u = (r >> 8) * 2^-24 is exact in f32, and the element is kept iff u < q,
// q = 1 - (float)p: P(keep) = q up to 2^-24.
//
// The call id lives in device memory (ctx->rng_state = {seed, calls, ticket}), never in a kernel parameter, which a
// captured graph would freeze.  Every block of a drawing forward reads `calls` first thing, then takes a ticket; the
// block that takes the last ticket knows every block has read the id and advances it (and resets the ticket).  So the
// kernel needs no second launch, and a later dropout forward on the stream sees the next id.
#include <random>

#include "nk_internal.cuh"

namespace {

constexpr int kThreads = 256;

inline int grid_for(nk_ctx* ctx, size_t work_items) {
  size_t b = (work_items + kThreads - 1) / kThreads;
  const size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}

inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {  // key schedule: bump before every round after the first
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// bits 0..7 of b to bits 0, 4, 8, ..., 28
__device__ __forceinline__ uint32_t spread_nibbles(uint32_t b) {
  b &= 0xffu;
  b = (b | (b << 12)) & 0x000F000Fu;
  b = (b | (b << 6)) & 0x03030303u;
  b = (b | (b << 3)) & 0x11111111u;
  return b;
}

template <typename T>
struct alignas(4 * sizeof(T)) Quad {
  T v[4];
};

// One thread per group of 4 elements (one Philox block); a warp covers 128 consecutive elements = 4 mask words, which
// its lanes 0..3 store after four ballots (bit j of every lane's 4-bit keep nibble).  The whole warp runs every trip of
// the loop so the ballots see all 32 lanes.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads) dropout_fwd_kernel(T* __restrict__ y, uint32_t* __restrict__ mask,
                                                              const T* __restrict__ x, size_t n, float q,
                                                              unsigned long long* __restrict__ state) {
  __shared__ unsigned long long s_call;
  if (threadIdx.x == 0) {
    s_call = *reinterpret_cast<volatile unsigned long long*>(&state[1]);
    __threadfence();
    if (atomicAdd(&state[2], 1ull) == gridDim.x - 1) {  // the last block to read the call id advances it
      state[1] = s_call + 1;
      state[2] = 0;
    }
  }
  __syncthreads();
  const unsigned long long call = s_call, seed = state[0];
  const uint2 key = make_uint2(uint32_t(seed), uint32_t(seed >> 32));
  const size_t groups = (n + 3) / 4, words = (n + 31) / 32;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  for (size_t g = size_t(blockIdx.x) * blockDim.x + threadIdx.x; g - lane < groups; g += stride) {
    uint32_t keep = 0;
    if (g < groups) {
      const uint4 r = philox4x32_10(make_uint4(uint32_t(g), uint32_t(g >> 32), uint32_t(call), uint32_t(call >> 32)), key);
      const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
      const size_t e0 = g * 4;
      if (VEC && e0 + 4 <= n) {
        Quad<T> xv = *reinterpret_cast<const Quad<T>*>(x + e0), yv;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool k = float(rr[j] >> 8) * 0x1p-24f < q;
          yv.v[j] = nk_from_f32<T>(k ? nk_to_f32<T>(xv.v[j]) / q : 0.f);
          keep |= uint32_t(k) << j;
        }
        *reinterpret_cast<Quad<T>*>(y + e0) = yv;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e0 + j < n) {
            const bool k = float(rr[j] >> 8) * 0x1p-24f < q;
            y[e0 + j] = nk_from_f32<T>(k ? nk_to_f32<T>(x[e0 + j]) / q : 0.f);
            keep |= uint32_t(k) << j;
          }
      }
    }
    uint32_t b[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = __ballot_sync(0xffffffffu, (keep >> j) & 1u);
    if (lane < 4) {  // word `lane` of this warp's 4: lanes 8*lane .. 8*lane+7, 4 bits each
      uint32_t word = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) word |= spread_nibbles(b[j] >> (8 * lane)) << j;
      const size_t w = (g - lane) / 8 + lane;
      if (w < words) mask[w] = word;
    }
  }
}

// MODE 0: identity (eval / p == 0); 1: masked, g*keep/q; 2: zero (p == 1).  dx = (RMW ? beta*dx : 0) + that.
template <typename T, typename TD, int MODE, bool RMW, bool VEC>
__global__ void __launch_bounds__(kThreads) dropout_bwd_kernel(TD* __restrict__ dx, const uint32_t* __restrict__ mask,
                                                              const T* __restrict__ g, size_t n, float q, float beta) {
  const size_t tid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  auto term = [&](float gv, uint32_t bit) { return MODE == 0 ? gv : (MODE == 1 && bit ? gv / q : 0.f); };
  size_t done = 0;
  if (VEC) {
    const size_t npk = n / 8;
    const uint8_t* mbytes = reinterpret_cast<const uint8_t*>(mask);  // bit e%8 of byte e/8 (little endian words)
    for (size_t v = tid; v < npk; v += stride) {
      NkPack8<T> a;
      NkPack8<TD> o;
      if (MODE != 2) a.load(g + v * 8);
      if (RMW) o.load(dx + v * 8);
      const uint32_t m = MODE == 1 ? mbytes[v] : 0u;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float r = term(MODE != 2 ? a.get(i) : 0.f, (m >> i) & 1u);
        if (RMW) r = __fadd_rn(__fmul_rn(beta, o.get(i)), r);  // no FMA: the reference's `+=`
        o.set(i, r);
      }
      o.store(dx + v * 8);
    }
    done = npk * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    const uint32_t bit = MODE == 1 ? (mask[i / 32] >> (i % 32)) & 1u : 0u;
    float r = term(MODE != 2 ? nk_to_f32<T>(g[i]) : 0.f, bit);
    if (RMW) r = __fadd_rn(__fmul_rn(beta, nk_to_f32<TD>(dx[i])), r);
    dx[i] = nk_from_f32<TD>(r);
  }
}

__global__ void rng_seed_kernel(unsigned long long* state, unsigned long long seed) {
  state[0] = seed;
  state[1] = 0;
  state[2] = 0;
}

// the device state, created on first use (seeded from OS entropy, like the reference's thread_rng, unless `seed` is set)
int rng_state(nk_ctx* ctx, const unsigned long long* seed, unsigned long long** out) {
  if (!ctx->rng_state) {
    if (ctx->capturing)
      return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "the dropout generator state is created on first use, which cannot "
                          "be captured: run the step once before capturing it");
    NK_CUDA(ctx, cudaMalloc(&ctx->rng_state, 3 * sizeof(unsigned long long)));
    if (!seed) {
      std::random_device rd;
      const unsigned long long s = (unsigned long long)rd() << 32 | rd();
      rng_seed_kernel<<<1, 1, 0, ctx->stream>>>(ctx->rng_state, s);
      NK_LAUNCHED(ctx, "rng_seed");
    }
  }
  if (seed) {
    rng_seed_kernel<<<1, 1, 0, ctx->stream>>>(ctx->rng_state, *seed);
    NK_LAUNCHED(ctx, "rng_seed");
  }
  *out = ctx->rng_state;
  return NK_OK;
}

template <typename T, typename TD, int MODE>
void launch_bwd(nk_ctx* ctx, int blocks, bool vec, void* dx, const uint32_t* mask, const void* g, size_t n, float q,
                float beta) {
  TD* d = static_cast<TD*>(dx);
  const T* gg = static_cast<const T*>(g);
  if (beta != 0.f) {
    if (vec)
      dropout_bwd_kernel<T, TD, MODE, true, true><<<blocks, kThreads, 0, ctx->stream>>>(d, mask, gg, n, q, beta);
    else
      dropout_bwd_kernel<T, TD, MODE, true, false><<<blocks, kThreads, 0, ctx->stream>>>(d, mask, gg, n, q, beta);
  } else {
    if (vec)
      dropout_bwd_kernel<T, TD, MODE, false, true><<<blocks, kThreads, 0, ctx->stream>>>(d, mask, gg, n, q, beta);
    else
      dropout_bwd_kernel<T, TD, MODE, false, false><<<blocks, kThreads, 0, ctx->stream>>>(d, mask, gg, n, q, beta);
  }
}

template <typename T, typename TD>
void launch_bwd_mode(nk_ctx* ctx, int mode, int blocks, bool vec, void* dx, const uint32_t* mask, const void* g,
                     size_t n, float q, float beta) {
  if (mode == 0)
    launch_bwd<T, TD, 0>(ctx, blocks, vec, dx, mask, g, n, q, beta);
  else if (mode == 1)
    launch_bwd<T, TD, 1>(ctx, blocks, vec, dx, mask, g, n, q, beta);
  else
    launch_bwd<T, TD, 2>(ctx, blocks, vec, dx, mask, g, n, q, beta);
}

}  // namespace

extern "C" {

int nk_dropout_fwd(nk_ctx* ctx, void* y, uint32_t* mask, const void* x, size_t n, int dtype, double p) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_dropout_fwd: bad dtype %d", dtype);
  NK_REQUIRE(ctx, p >= 0.0 && p <= 1.0, "Wrong probability received: %g.", p);
  NK_REQUIRE(ctx, y && x && n > 0, "nk_dropout_fwd: NULL pointer or empty input");
  const size_t bytes = n * nk_dtype_size(dtype);
  if (p == 0.0) {  // dropout/mod.rs:59-62
    if (y != x) NK_CUDA(ctx, cudaMemcpyAsync(y, x, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return NK_OK;
  }
  if (1.0 - p == 0.0) {  // :64-67
    NK_CUDA(ctx, cudaMemsetAsync(y, 0, bytes, ctx->stream));
    return NK_OK;
  }
  NK_REQUIRE(ctx, mask, "nk_dropout_fwd: NULL mask");
  unsigned long long* state;
  int rc = rng_state(ctx, nullptr, &state);
  if (rc) return rc;
  const float q = 1.f - float(p);
  const size_t groups = (n + 3) / 4;
  const int blocks = grid_for(ctx, groups);
  NK_DISPATCH_DTYPE(dtype, T, {
    const bool vec = aligned(x, sizeof(Quad<T>)) && aligned(y, sizeof(Quad<T>));
    if (vec)
      dropout_fwd_kernel<T, true><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, mask, (const T*)x, n, q, state);
    else
      dropout_fwd_kernel<T, false><<<blocks, kThreads, 0, ctx->stream>>>((T*)y, mask, (const T*)x, n, q, state);
  });
  NK_LAUNCHED(ctx, "dropout_fwd");
  return NK_OK;
}

int nk_dropout_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const uint32_t* mask, const void* g, size_t n, int dtype,
                   double p, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype) && nk_dtype_ok(dx_dtype), "nk_dropout_bwd: bad dtype %d / dx dtype %d", dtype,
             dx_dtype);
  NK_REQUIRE(ctx, p >= 0.0 && p <= 1.0, "Wrong probability received: %g.", p);
  NK_REQUIRE(ctx, dx && g && n > 0, "nk_dropout_bwd: NULL pointer or empty input");
  const int mode = p == 0.0 ? 0 : (1.0 - p == 0.0 ? 2 : (mask ? 1 : 0));
  const bool vec = aligned(dx, 16) && aligned(g, 16);
  const int blocks = grid_for(ctx, vec ? n / 8 + 1 : n);
  const float q = 1.f - float(p);
  NK_DISPATCH_DTYPE(dtype, T, {
    if (dx_dtype == NK_BF16)
      launch_bwd_mode<T, __nv_bfloat16>(ctx, mode, blocks, vec, dx, mask, g, n, q, beta);
    else
      launch_bwd_mode<T, float>(ctx, mode, blocks, vec, dx, mask, g, n, q, beta);
  });
  NK_LAUNCHED(ctx, "dropout_bwd");
  return NK_OK;
}

int nk_rng_seed(nk_ctx* ctx, uint64_t seed) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (ctx->capturing)
    return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "nk_rng_seed cannot be captured: a replay would reset the generator");
  const unsigned long long s = seed;
  unsigned long long* state;
  return rng_state(ctx, &s, &state);
}

int nk_rng_state(nk_ctx* ctx, uint64_t* seed, uint64_t* calls) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, seed && calls, "nk_rng_state: NULL pointer");
  if (ctx->capturing) return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "nk_rng_state reads device memory: not while capturing");
  unsigned long long* state;
  int rc = rng_state(ctx, nullptr, &state);
  if (rc) return rc;
  unsigned long long host[2];
  NK_CUDA(ctx, cudaMemcpyAsync(host, state, sizeof(host), cudaMemcpyDeviceToHost, ctx->stream));
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *seed = host[0];
  *calls = host[1];
  return NK_OK;
}

}  // extern "C"
