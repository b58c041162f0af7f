// CUDA-core GEMM engine: C = alpha * op(A).op(B) + beta*C (+bias, ReLU), f32 FFMA accumulate.
// This is the parity-grade path for f32 tensors (the tensor cores have no true-f32 kind) and the fallback
// for operands TMA cannot address (leading dimension not a multiple of 16 bytes, e.g. the
// (N, 10) logits of config 4).  Reference call sites: matrix_matrix_mul/mod.rs:33,65,97 and
// matrix_matrix_mul_t/mod.rs:33,65,97 (general_mat_mul).
// Tiling: 64x64x16 per CTA, 256 threads, 4x4 register micro-tile, split-K over gridDim.z into an
// f32 workspace when the (M, N) grid alone cannot fill the SMs.
#include "nk_internal.cuh"

namespace {

// two-lane fused multiply-add, lane by lane (the same IEEE result as two fmaf)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
constexpr int kThreads = 256;

struct Epilogue {
  float alpha, beta;
  const void* bias;
  int bias_bf16;
  int relu;
  const void* mask = nullptr;   // small-K kernel only: (M, N) tensor of C's type and pitch; v = mask > 0 ? v : 0 before the
                                // beta accumulate (the ReLU backward of the layer below, relu/mod.rs:71-78)
  float* colsum = nullptr;      // small-K kernel only: N floats, += column sums of the stored values (the bias gradient of
                                // the layer below), f32 atomics; beta must be 0
};

template <typename TC>
__device__ __forceinline__ void store_out(TC* C, int64_t ldc, int64_t m, int64_t n, float acc, const Epilogue& ep) {
  float v = ep.alpha * acc;
  if (ep.beta != 0.f) v += ep.beta * nk_to_f32<TC>(C[m * ldc + n]);
  if (ep.bias)
    v += ep.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(ep.bias)[n])
                      : static_cast<const float*>(ep.bias)[n];
  if (ep.relu) v = v > 0.f ? v : 0.f;
  C[m * ldc + n] = nk_from_f32<TC>(v);
}

template <typename TAB, typename TC, bool TA, bool TB>
__global__ void __launch_bounds__(kThreads) gemm_simt_kernel(const TAB* __restrict__ A, const TAB* __restrict__ B,
                                                            TC* __restrict__ C, float* __restrict__ partial,
                                                            int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                                                            int64_t ldc, int64_t k_per_split, Epilogue ep) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = int64_t(blockIdx.y) * BM, n0 = int64_t(blockIdx.x) * BN;
  const int64_t k_begin = int64_t(blockIdx.z) * k_per_split;
  int64_t k_end = k_begin + k_per_split;
  if (k_end > K) k_end = K;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int64_t k0 = k_begin; k0 < k_end; k0 += BK) {
    // A tile (BM x BK): 1024 elements, 4 per thread
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * kThreads;
      int mm, kk;
      if (TA) {  // stored (K, M): consecutive threads along m
        kk = idx / BM;
        mm = idx % BM;
      } else {  // stored (M, K): consecutive threads along k
        mm = idx / BK;
        kk = idx % BK;
      }
      const int64_t gm = m0 + mm, gk = k0 + kk;
      float v = 0.f;
      if (gm < M && gk < k_end) v = nk_to_f32<TAB>(TA ? A[gk * lda + gm] : A[gm * lda + gk]);
      As[kk][mm] = v;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * kThreads;
      int nn, kk;
      if (TB) {  // stored (N, K): consecutive threads along k
        nn = idx / BK;
        kk = idx % BK;
      } else {  // stored (K, N): consecutive threads along n
        kk = idx / BN;
        nn = idx % BN;
      }
      const int64_t gn = n0 + nn, gk = k0 + kk;
      float v = 0.f;
      if (gn < N && gk < k_end) v = nk_to_f32<TAB>(TB ? B[gn * ldb + gk] : B[gk * ldb + gn]);
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t n = n0 + tx * TN + j;
      if (n >= N) continue;
      if (partial)
        partial[(int64_t(blockIdx.z) * M + m) * N + n] = acc[i][j];
      else
        store_out<TC>(C, ldc, m, n, acc[i][j], ep);
    }
  }
}

template <typename TC>
__global__ void __launch_bounds__(kThreads) splitk_reduce_kernel(TC* __restrict__ C, const float* __restrict__ partial,
                                                                int64_t M, int64_t N, int64_t ldc, int splits,
                                                                Epilogue ep) {
  const int64_t total = M * N;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    float s = 0.f;
    for (int z = 0; z < splits; ++z) s += partial[int64_t(z) * total + i];
    store_out<TC>(C, ldc, i / N, i % N, s, ep);
  }
}

template <typename TAB, typename TC>
int launch(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
           const void* B, int64_t ldb, void* C, int64_t ldc, Epilogue ep) {
  const int64_t gm = (M + BM - 1) / BM, gn = (N + BN - 1) / BN;
  NK_REQUIRE(ctx, gm <= 65535, "nk_gemm(simt): M too large");
  // split-K when the output grid underfills the machine and K is deep
  int splits = 1;
  const int64_t tiles = gm * gn;
  if (tiles < ctx->sm_count && K >= 512) {
    int64_t s = (2 * int64_t(ctx->sm_count) + tiles - 1) / tiles;
    const int64_t max_s = K / 128;
    if (s > max_s) s = max_s;
    if (s > 64) s = 64;
    if (s > 1) splits = int(s);
  }
  int64_t k_per_split = (K + splits - 1) / splits;
  k_per_split = (k_per_split + BK - 1) / BK * BK;
  if (k_per_split == 0) k_per_split = BK;   // K = 0: one pass of no steps, the epilogue alone (C = beta*C + bias)
  splits = int((K + k_per_split - 1) / k_per_split);
  if (splits < 1) splits = 1;
  float* partial = nullptr;
  if (splits > 1) {
    int rc = nk_workspace(ctx, size_t(splits) * size_t(M) * size_t(N) * sizeof(float), (void**)&partial);
    if (rc) return rc;
  }
  dim3 grid((unsigned)gn, (unsigned)gm, (unsigned)splits);
  const TAB* a = static_cast<const TAB*>(A);
  const TAB* b = static_cast<const TAB*>(B);
  TC* c = static_cast<TC*>(C);
#define NK_L(TA_, TB_) \
  gemm_simt_kernel<TAB, TC, TA_, TB_><<<grid, kThreads, 0, ctx->stream>>>(a, b, c, partial, M, N, K, lda, ldb, ldc, k_per_split, ep)
  if (!transA && !transB)
    NK_L(false, false);
  else if (!transA && transB)
    NK_L(false, true);
  else if (transA && !transB)
    NK_L(true, false);
  else
    NK_L(true, true);
#undef NK_L
  NK_LAUNCHED(ctx, "gemm_simt");
  if (splits > 1) {
    int64_t blocks = (M * N + kThreads - 1) / kThreads;
    if (blocks > int64_t(ctx->sm_count) * 8) blocks = int64_t(ctx->sm_count) * 8;
    splitk_reduce_kernel<TC><<<(unsigned)blocks, kThreads, 0, ctx->stream>>>(c, partial, M, N, ldc, splits, ep);
    NK_LAUNCHED(ctx, "gemm_simt_splitk_reduce");
  }
  return NK_OK;
}


// ------------------------------------------------------------------------------------------------------
// Skinny shapes of config 4's last layer (Linear 4096 -> 10): the (N,10) logits and their gradient have a
// 20-byte row pitch that TMA cannot address, and 64x64 tiles waste >80 % of their work on them.  Both kernels are
// HBM-bound on the large operand and read/write it exactly once.
//   small-K  (NN, K <= 16):  dH = G . W        C[m][n] = sum_k A[m][k] * B[k][n]
//   small-M  (TN, M <= 16):  dW = G^T . H      C[m][n] = sum_k A[k][m] * B[k][n]   (split over k, f32 atomics)
// ------------------------------------------------------------------------------------------------------
constexpr int kSkinnyMax = 16;

// 4 consecutive elements of a row, as one 8-byte (bf16) or 16-byte (f32) access when `vec`, else scalars
template <typename T>
__device__ __forceinline__ void load4(const T* p, bool vec, int valid, float* out) {
  if (vec) {
    if constexpr (sizeof(T) == 2) {
      const uint2 w = *reinterpret_cast<const uint2*>(p);
      out[0] = __uint_as_float(w.x << 16), out[1] = __uint_as_float(w.x & 0xffff0000u);
      out[2] = __uint_as_float(w.y << 16), out[3] = __uint_as_float(w.y & 0xffff0000u);
    } else {
      const float4 w = *reinterpret_cast<const float4*>(p);
      out[0] = w.x, out[1] = w.y, out[2] = w.z, out[3] = w.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = j < valid ? nk_to_f32<T>(p[j]) : 0.f;
  }
}
template <typename T>
__device__ __forceinline__ void store4(T* p, bool vec, int valid, const float* v) {
  if (vec) {
    if constexpr (sizeof(T) == 2) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
      uint2 w;
      w.x = *reinterpret_cast<uint32_t*>(&lo), w.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(p) = w;
    } else {
      *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < valid) p[j] = nk_from_f32<T>(v[j]);
  }
}

// raw 4-element group of a row (8 bytes of bf16 / 16 bytes of f32) kept as loaded: conversion happens at use, so that
// eight rows' worth of mask / old values can be in flight without eight rows' worth of converted registers
template <typename T>
struct Raw4 {
  uint32_t w[sizeof(T) == 2 ? 2 : 4];
};
template <typename T>
__device__ __forceinline__ Raw4<T> load_raw4(const T* p, bool vec, int valid) {
  Raw4<T> r;
  if (vec) {
    if constexpr (sizeof(T) == 2) {
      const uint2 v = *reinterpret_cast<const uint2*>(p);
      r.w[0] = v.x, r.w[1] = v.y;
    } else {
      const uint4 v = *reinterpret_cast<const uint4*>(p);
      r.w[0] = v.x, r.w[1] = v.y, r.w[2] = v.z, r.w[3] = v.w;
    }
  } else {
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = j < valid ? nk_to_f32<T>(p[j]) : 0.f;
    if constexpr (sizeof(T) == 2) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(f[0], f[1]), hi = __floats2bfloat162_rn(f[2], f[3]);   // exact: they were bf16
      r.w[0] = *reinterpret_cast<uint32_t*>(&lo), r.w[1] = *reinterpret_cast<uint32_t*>(&hi);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) r.w[j] = __float_as_uint(f[j]);
    }
  }
  return r;
}
template <typename T>
__device__ __forceinline__ float raw_get(const Raw4<T>& r, int j) {
  if constexpr (sizeof(T) == 2) return __uint_as_float((j & 1) ? (r.w[j >> 1] & 0xffff0000u) : (r.w[j >> 1] << 16));
  else return __uint_as_float(r.w[j]);
}

template <typename TAB, typename TC, int KP>
__global__ void __launch_bounds__(256, 2) gemm_small_k_kernel(const TAB* __restrict__ A, const TAB* __restrict__ B,
                                                           TC* __restrict__ C, int64_t M, int64_t N, int K,
                                                           int64_t lda, int64_t ldb, int64_t ldc, Epilogue ep) {
  // block: 64 rows x 1024 columns; thread: 4 consecutive columns of all rows, 8 rows in flight at a time so that the
  // (optional) reads of the mask / old C overlap the arithmetic; every access to C is one 8/16-byte vector.  The kernel
  // is issue bound, K x 4 FMAs per 8 bytes stored -- KP = K rounded up to 4 bounds them (10 -> 12, not 16).
  constexpr int kRows = 64, kFlight = 8;
  __shared__ __align__(16) float As[kRows][KP];
  const int64_t m0 = int64_t(blockIdx.y) * kRows;
  const int64_t n = (int64_t(blockIdx.x) * 256 + threadIdx.x) * 4;
  for (int i = threadIdx.x; i < kRows * KP; i += 256) {
    const int r = i / KP, k = i - r * KP;
    As[r][k] = (k < K && m0 + r < M) ? nk_to_f32<TAB>(A[(m0 + r) * lda + k]) : 0.f;
  }
  __syncthreads();
  if (n >= N) return;
  const int valid = int(N - n < 4 ? N - n : 4);
  const bool vb = valid == 4 && (ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
  const bool vc = valid == 4 && (ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
  const bool vmask = vc && ((reinterpret_cast<uintptr_t>(ep.mask) & 15) == 0);
  float2 b01[KP], b23[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    if (k < K) load4<TAB>(B + int64_t(k) * ldb + n, vb, valid, t);
    b01[k] = make_float2(t[0], t[1]), b23[k] = make_float2(t[2], t[3]);
  }
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (ep.bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < valid)
        bias[j] = ep.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(ep.bias)[n + j])
                               : static_cast<const float*>(ep.bias)[n + j];
  }
  const int rows = int(M - m0 < kRows ? M - m0 : kRows);
  float csum[4] = {0.f, 0.f, 0.f, 0.f};
  for (int r0 = 0; r0 < rows; r0 += kFlight) {
    Raw4<TC> old[kFlight], msk[kFlight];
    if (ep.beta != 0.f) {
#pragma unroll
      for (int rr = 0; rr < kFlight; ++rr)
        if (r0 + rr < rows) old[rr] = load_raw4<TC>(C + (m0 + r0 + rr) * ldc + n, vc, valid);
    }
    if (ep.mask) {
#pragma unroll
      for (int rr = 0; rr < kFlight; ++rr)
        if (r0 + rr < rows) msk[rr] = load_raw4<TC>(static_cast<const TC*>(ep.mask) + (m0 + r0 + rr) * ldc + n, vmask, valid);
    }
#pragma unroll
    for (int rr = 0; rr < kFlight; ++rr) {
      if (r0 + rr >= rows) break;
      float2 a01 = make_float2(0.f, 0.f), a23 = make_float2(0.f, 0.f);
#pragma unroll
      for (int k4 = 0; k4 < KP / 4; ++k4) {
        const float4 av = *reinterpret_cast<const float4*>(&As[r0 + rr][k4 * 4]);  // zero for k >= K
        const float a[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 aa = make_float2(a[i], a[i]);
          a01 = fma2(aa, b01[k4 * 4 + i], a01);
          a23 = fma2(aa, b23[k4 * 4 + i], a23);
        }
      }
      float acc[4] = {a01.x, a01.y, a23.x, a23.y};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = ep.alpha * acc[j];
        if (ep.mask) v = raw_get<TC>(msk[rr], j) > 0.f ? v : 0.f;
        if (ep.beta != 0.f) v += ep.beta * raw_get<TC>(old[rr], j);
        v += bias[j];
        if (ep.relu) v = v > 0.f ? v : 0.f;
        acc[j] = v;
        csum[j] += nk_to_f32<TC>(nk_from_f32<TC>(v));   // what the output tensor will hold
      }
      store4<TC>(C + (m0 + r0 + rr) * ldc + n, vc, valid, acc);
    }
  }
  if (ep.colsum) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < valid) atomicAdd(ep.colsum + n + j, csum[j]);
  }
}

// small-M: block = 8 warps x 128 columns (lane: 4 consecutive) x one slab of k.  Warp w takes the rows k = w, w + 8, ...
// of the slab with eight 8/16-byte loads of the streamed operand in flight; the M (<= 16) values of A for a row come
// from shared memory as broadcast 16-byte reads; MP = M rounded up to 4 bounds the FMAs (10 -> 12, not 16), which are
// the packed two-lane form.  The eight warps' partial sums meet in a three-round tree through shared memory (shared
// f32 atomicAdd is a compare-and-swap loop in SASS, ATOMS.CAST.SPIN: 8-way contended it cost more than the loop), and
// one warp ends the block with M x 128 global reductions.
constexpr int kSmChunk = 512;   // rows of A staged per pass (a whole k slab of the usual launch)
template <typename TAB, int MP>
__global__ void __launch_bounds__(256) gemm_small_m_kernel(const TAB* __restrict__ A, const TAB* __restrict__ B,
                                                           float* __restrict__ scratch, int M, int64_t N, int64_t K,
                                                           int64_t lda, int64_t ldb, int64_t k_per_block) {
  constexpr int kAsFloats = kSmChunk * MP, kRedFloats = 4 * MP * 128;
  __shared__ __align__(16) float smem[kAsFloats > kRedFloats ? kAsFloats : kRedFloats];
  float (*As)[MP] = reinterpret_cast<float (*)[MP]>(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n = int64_t(blockIdx.x) * 128 + lane * 4;
  const int64_t k_begin = int64_t(blockIdx.y) * k_per_block;
  int64_t k_end = k_begin + k_per_block;
  if (k_end > K) k_end = K;
  const int valid = n < N ? int(N - n < 4 ? N - n : 4) : 0;
  const bool vb = valid == 4 && (ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
  float2 acc01[MP], acc23[MP];
#pragma unroll
  for (int m = 0; m < MP; ++m) acc01[m] = make_float2(0.f, 0.f), acc23[m] = make_float2(0.f, 0.f);
  for (int64_t k0 = k_begin; k0 < k_end; k0 += kSmChunk) {
    __syncthreads();
    const int rows = int(k_end - k0 < kSmChunk ? k_end - k0 : kSmChunk);
    for (int i = threadIdx.x; i < kSmChunk * MP; i += 256) {
      const int r = i / MP, m = i - r * MP;
      As[r][m] = (m < M && r < rows) ? nk_to_f32<TAB>(A[(k0 + r) * lda + m]) : 0.f;
    }
    __syncthreads();
    if (valid) {
      // software pipeline: the 8 loads of the NEXT pass are issued before the FMAs of the current one, so a warp always has
      // loads in flight (kept raw, converted at use: 16 registers per set)
      Raw4<TAB> cur[8], nxt[8];
      auto fetch = [&](Raw4<TAB>* dst, int kb) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (kb + 8 * u < rows) dst[u] = load_raw4<TAB>(B + (k0 + kb + 8 * u) * ldb + n, vb, valid);
          else dst[u] = Raw4<TAB>{};
        }
      };
      fetch(cur, warp);
      for (int kb = warp; kb < rows; kb += 64) {      // 8 rows of this warp per pass: kb, kb + 8, ..., kb + 56
        if (kb + 64 < rows) fetch(nxt, kb + 64);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = kb + 8 * u < rows ? kb + 8 * u : 0;   // (the operand is zero beyond the slab)
          const float2 b01 = make_float2(raw_get<TAB>(cur[u], 0), raw_get<TAB>(cur[u], 1));
          const float2 b23 = make_float2(raw_get<TAB>(cur[u], 2), raw_get<TAB>(cur[u], 3));
#pragma unroll
          for (int m4 = 0; m4 < MP / 4; ++m4) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[r][m4 * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 aa = make_float2(a[i], a[i]);
              acc01[m4 * 4 + i] = fma2(aa, b01, acc01[m4 * 4 + i]);
              acc23[m4 * 4 + i] = fma2(aa, b23, acc23[m4 * 4 + i]);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) cur[u] = nxt[u];
      }
    }
  }
  // tree over the 8 warps: the upper half of the live warps stores, the lower half adds
  float4* red = reinterpret_cast<float4*>(smem);            // [4 warps][MP][32 lanes] float4, aliases As (no longer needed)
#pragma unroll
  for (int half = 4; half >= 1; half >>= 1) {
    __syncthreads();
    if (warp >= half && warp < 2 * half) {
#pragma unroll
      for (int m = 0; m < MP; ++m)
        red[((warp - half) * MP + m) * 32 + lane] = make_float4(acc01[m].x, acc01[m].y, acc23[m].x, acc23[m].y);
    }
    __syncthreads();
    if (warp < half) {
#pragma unroll
      for (int m = 0; m < MP; ++m) {
        const float4 v = red[(warp * MP + m) * 32 + lane];
        acc01[m].x += v.x, acc01[m].y += v.y, acc23[m].x += v.z, acc23[m].y += v.w;
      }
    }
  }
  if (warp == 0 && valid) {
#pragma unroll
    for (int m = 0; m < MP; ++m) {
      if (m >= M) break;
      const float v[4] = {acc01[m].x, acc01[m].y, acc23[m].x, acc23[m].y};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < valid) atomicAdd(&scratch[int64_t(m) * N + n + j], v[j]);
    }
  }
}

template <typename TAB, typename TC>
int launch_skinny(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                  const void* B, int64_t ldb, void* C, int64_t ldc, Epilogue ep, bool* handled) {
  *handled = false;
  if (!transA && !transB && K <= kSkinnyMax && K > 0 && N >= 256) {
    dim3 grid((unsigned)((N + 1023) / 1024), (unsigned)((M + 63) / 64));
    if (grid.y > 65535) return NK_OK;
#define NK_SK(KP_) gemm_small_k_kernel<TAB, TC, KP_><<<grid, 256, 0, ctx->stream>>>((const TAB*)A, (const TAB*)B, (TC*)C, M, N, (int)K, lda, ldb, ldc, ep)
    if (K <= 4)
      NK_SK(4);
    else if (K <= 8)
      NK_SK(8);
    else if (K <= 12)
      NK_SK(12);
    else
      NK_SK(16);
#undef NK_SK
    NK_LAUNCHED(ctx, "gemm_small_k");
    ctx->last_gemm_kernel = "simt_small_k";
    *handled = true;
    return NK_OK;
  }
  if (transA && !transB && M <= kSkinnyMax && N >= 256 && K >= 256) {
    float* scratch;
    int rc = nk_workspace(ctx, size_t(M) * size_t(N) * sizeof(float), (void**)&scratch);
    if (rc) return rc;
    NK_CUDA(ctx, cudaMemsetAsync(scratch, 0, size_t(M) * size_t(N) * sizeof(float), ctx->stream));
    const int64_t gx = (N + 127) / 128;
    // ~4 blocks of 8 warps per SM, each warp with 8 loads of the streamed operand in flight
    int64_t gy = (int64_t(ctx->sm_count) * 4 + gx - 1) / gx;
    int64_t k_per_block = (K + gy - 1) / gy;
    k_per_block = (k_per_block + kSmChunk - 1) / kSmChunk * kSmChunk;
    gy = (K + k_per_block - 1) / k_per_block;
    dim3 grid((unsigned)gx, (unsigned)gy);
#define NK_SM(MP_) gemm_small_m_kernel<TAB, MP_><<<grid, 256, 0, ctx->stream>>>((const TAB*)A, (const TAB*)B, scratch, (int)M, N, K, lda, ldb, k_per_block)
    if (M <= 4)
      NK_SM(4);
    else if (M <= 8)
      NK_SM(8);
    else if (M <= 12)
      NK_SM(12);
    else
      NK_SM(16);
#undef NK_SM
    NK_LAUNCHED(ctx, "gemm_small_m");
    int64_t blocks = (M * N + kThreads - 1) / kThreads;
    splitk_reduce_kernel<TC><<<(unsigned)blocks, kThreads, 0, ctx->stream>>>((TC*)C, scratch, M, N, ldc, 1, ep);
    NK_LAUNCHED(ctx, "gemm_small_m_finalize");
    ctx->last_gemm_kernel = "simt_small_m";
    *handled = true;
    return NK_OK;
  }
  return NK_OK;
}

}  // namespace

// C = mask > 0 ? A.B : 0  (+ beta*C) for the skinny NN shape only (K <= 16): the dX product of a 10-wide layer with the ReLU
// backward of the layer below applied on the way out.  NK_ERR_UNSUPPORTED (nothing done) for every other shape.
int nk_gemm_simt_small_k_masked(nk_ctx* ctx, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                                int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype, const void* mask,
                                float* colsum) {
  if (K > kSkinnyMax || K <= 0 || N < 256 || (M + 63) / 64 > 65535 || (colsum && beta != 0.f)) return NK_ERR_UNSUPPORTED;
  Epilogue ep{1.f, beta, nullptr, 0, 0, mask, colsum};
  bool handled = false;
  int rc;
  if (ab_dtype == NK_F32 && c_dtype == NK_F32)
    rc = launch_skinny<float, float>(ctx, 0, 0, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else if (ab_dtype == NK_BF16 && c_dtype == NK_BF16)
    rc = launch_skinny<__nv_bfloat16, __nv_bfloat16>(ctx, 0, 0, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else if (ab_dtype == NK_BF16 && c_dtype == NK_F32)
    rc = launch_skinny<__nv_bfloat16, float>(ctx, 0, 0, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else
    rc = launch_skinny<float, __nv_bfloat16>(ctx, 0, 0, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  if (rc) return rc;
  return handled ? NK_OK : NK_ERR_UNSUPPORTED;
}

int nk_gemm_simt(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                 int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype,
                 int c_dtype, const void* bias, int bias_dtype, int relu) {
  Epilogue ep{alpha, beta, bias, bias_dtype == NK_BF16, relu};
  bool handled = false;
  int rc;
  if (ab_dtype == NK_F32 && c_dtype == NK_F32)
    rc = launch_skinny<float, float>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else if (ab_dtype == NK_BF16 && c_dtype == NK_BF16)
    rc = launch_skinny<__nv_bfloat16, __nv_bfloat16>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else if (ab_dtype == NK_BF16 && c_dtype == NK_F32)
    rc = launch_skinny<__nv_bfloat16, float>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  else
    rc = launch_skinny<float, __nv_bfloat16>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep, &handled);
  if (rc || handled) return rc;
  ctx->last_gemm_kernel = "simt_64x64x16";
  if (ab_dtype == NK_F32 && c_dtype == NK_F32)
    return launch<float, float>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep);
  if (ab_dtype == NK_BF16 && c_dtype == NK_BF16)
    return launch<__nv_bfloat16, __nv_bfloat16>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep);
  if (ab_dtype == NK_BF16 && c_dtype == NK_F32)
    return launch<__nv_bfloat16, float>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep);
  return launch<float, __nv_bfloat16>(ctx, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, ep);
}
