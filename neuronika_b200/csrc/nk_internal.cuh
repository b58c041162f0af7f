// Internal declarations shared by the kernel translation units of libnk_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "nk_b200.h"

// a captured step (nk_capture_begin / nk_capture_end): the instantiated CUDA graph plus the arena its buffers live in
struct nk_graph {
  nk_ctx* ctx = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  char* arena = nullptr;
  size_t arena_bytes = 0, arena_used = 0;
  uint64_t kernel_nodes = 0;
};

struct nk_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int sm_count = 132;
  size_t smem_optin = 0;
  std::string last_error;
  uint64_t launches = 0;
  void* workspace = nullptr;  // grow-only device scratch (split-K partials, reductions)
  size_t workspace_bytes = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int gemm_engine = NK_GEMM_AUTO;
  int f32_gemm = NK_F32_GEMM_IEEE;   // nk_gemm_f32_config: how f32 products use the tensor cores
  int conv_engine = NK_CONV_AUTO;
  int f32_conv = NK_F32_GEMM_IEEE;   // nk_conv_f32_config: how f32 convolutions use the tensor cores
  const char* last_gemm_kernel = "none";
  const char* last_conv_kernel = "none";
  void* encode_tiled = nullptr;  // cuTensorMapEncodeTiled, fetched through the runtime
  // reduce-scatter plan of the NEXT tensor-core GEMM (set by nk_gemm_rs around its call): row shard o of the product is
  // stored to rs_dst[o] (rank o's slot buffer, peer-mapped, already offset to this rank's slot) instead of C
  int rs_world = 0, rs_rank = 0;
  void* rs_dst[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // stream capture of a whole step (nk_ctx.cu): while capturing, nk_alloc* hand out memory from the graph's arena
  // (fixed addresses for every replay, freed blocks are recycled within the capture) and nk_free of an arena pointer
  // is a no-op, during the capture and for as long as the graph lives
  nk_graph* capturing = nullptr;
  std::multimap<size_t, void*> arena_free;      // (rounded size -> block) freed during the running capture
  std::map<void*, size_t> capturing_sizes;      // rounded size of every block handed out by the running capture
  std::vector<nk_graph*> graphs;
  std::vector<std::pair<char*, size_t>> retired_arenas;  // ranges of destroyed graphs (late frees of their blocks are no-ops)
  std::vector<void*> deferred_frees;            // pool memory released while capturing: freed for real at capture end
  // NCCL communicator owned by the context (nk_comm.cu; libnccl is bound at run time)
  void* comm = nullptr;
  int comm_world = 0, comm_rank = 0;
  // dropout generator state in device memory (nk_dropout.cu): {seed, call counter, block ticket}, allocated on first use
  unsigned long long* rng_state = nullptr;
};

int nk_set_error(nk_ctx* ctx, int code, const char* fmt, ...);
int nk_workspace(nk_ctx* ctx, size_t bytes, void** out);
// stage 2 of the fixed-order scalar reductions (nk_elementwise.cu): *out = float(scale * sum of the nparts double
// partials), summed by one warp in a fixed order
int nk_reduce_finish(nk_ctx* ctx, float* out, const double* partials, int nparts, double scale);

#define NK_REQUIRE(ctx, cond, ...)                                      \
  do {                                                                  \
    if (!(cond)) return nk_set_error((ctx), NK_ERR_INVALID_ARG, __VA_ARGS__); \
  } while (0)

#define NK_CUDA(ctx, expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return nk_set_error((ctx), _e == cudaErrorMemoryAllocation ? NK_ERR_OOM : NK_ERR_CUDA, \
                          "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// after every kernel launch: count it and surface launch-configuration errors
#define NK_LAUNCHED(ctx, name)                                                          \
  do {                                                                                  \
    (ctx)->launches++;                                                                  \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess)                                                              \
      return nk_set_error((ctx), NK_ERR_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e)); \
  } while (0)

static inline size_t nk_dtype_size(int dt) { return dt == NK_BF16 ? 2 : 4; }
static inline bool nk_dtype_ok(int dt) { return dt == NK_F32 || dt == NK_BF16; }

// ------------------------------------------------------------------ device helpers
template <typename T>
__device__ __forceinline__ float nk_to_f32(T v);
template <>
__device__ __forceinline__ float nk_to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float nk_to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T nk_from_f32(float v);
template <>
__device__ __forceinline__ float nk_from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __nv_bfloat16 nk_from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// 16-byte vector of T with float accessors
template <typename T>
struct NkVec {
  static constexpr int N = 16 / sizeof(T);
  uint4 raw;
  __device__ __forceinline__ float get(int i) const { return nk_to_f32<T>(reinterpret_cast<const T*>(&raw)[i]); }
  __device__ __forceinline__ void set(int i, float v) { reinterpret_cast<T*>(&raw)[i] = nk_from_f32<T>(v); }
  __device__ __forceinline__ void load(const T* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(T* p) const { *reinterpret_cast<uint4*>(p) = raw; }
};

// 8 consecutive elements of T (one 16-byte vector of bf16, two of f32) with float accessors: lets kernels whose
// operands have different element types step through all of them 8 elements at a time
template <typename T>
struct NkPack8 {
  static constexpr int R = sizeof(T) / 2;
  uint4 raw[R];
  __device__ __forceinline__ float get(int i) const { return nk_to_f32<T>(reinterpret_cast<const T*>(raw)[i]); }
  __device__ __forceinline__ void set(int i, float v) { reinterpret_cast<T*>(raw)[i] = nk_from_f32<T>(v); }
  __device__ __forceinline__ void load(const T* p) {
#pragma unroll
    for (int r = 0; r < R; ++r) raw[r] = reinterpret_cast<const uint4*>(p)[r];
  }
  __device__ __forceinline__ void store(T* p) const {
#pragma unroll
    for (int r = 0; r < R; ++r) reinterpret_cast<uint4*>(p)[r] = raw[r];
  }
};

__device__ __forceinline__ float nk_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float nk_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// dispatch helper: call f.template operator()<T>() for the dtype
#define NK_DISPATCH_DTYPE(dt, T, ...)              \
  do {                                             \
    if ((dt) == NK_BF16) {                         \
      using T = __nv_bfloat16;                     \
      __VA_ARGS__;                                 \
    } else {                                       \
      using T = float;                             \
      __VA_ARGS__;                                 \
    }                                              \
  } while (0)

// engines implemented in other translation units
int nk_gemm_simt_small_k_masked(nk_ctx* ctx, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                                int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype, const void* mask,
                                float* colsum);
int nk_gemm_simt(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
                 const void* A, int64_t lda, const void* B, int64_t ldb, float beta, void* C,
                 int64_t ldc, int ab_dtype, int c_dtype, const void* bias, int bias_dtype, int relu);
// returns NK_ERR_UNSUPPORTED (without touching last_error) when the operands cannot be
// addressed by TMA, so that the caller may choose the SIMT engine
int nk_gemm_wgmma(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
                    const void* A, int64_t lda, const void* B, int64_t ldb, float beta, void* C,
                    int64_t ldc, int c_dtype, const void* bias, int bias_dtype, int relu, const void* mask, float* colsum);
// 2-D tensor map (bf16 or f32 elements) of a `rows` x `cols` row-major matrix with leading dimension ld: boxes of
// box_cols (= 128 bytes) x box_rows elements, 128B-swizzled (nk_gemm_tc.cu)
int make_tmap_2d(nk_ctx* ctx, CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld, uint32_t box_cols,
                 uint32_t box_rows, int dtype = NK_BF16);
// f32 products on the tensor cores in the context's TF32 / 3xTF32 mode (nk_gemm_tf32.cu); the caller has checked the
// arguments, K > 0
int nk_gemm_tf32(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                 int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int c_dtype, const void* bias,
                 int bias_dtype, int relu);
// f32 convolution on the tensor cores (nk_conv_tf32.cu): every f32, groups = 1 call with a non-empty batch once
// nk_conv_f32_config has set TF32 or TF32X3, unless nk_conv_config(DIRECT).  Arguments checked by the caller; the
// convolution of x padded by `pad` (nk_pad_mode `mode`, fill `value`) with nsp sample dims; `nd` picks the kernel names
// of the 1-D / 3-D entry points ("tf32_im2col_nd_*") over the 2-D ones ("tf32_im2col_*").
static inline bool nk_conv_tf32_on(const nk_ctx* ctx, int dtype, int64_t groups) {
  return dtype == NK_F32 && groups == 1 && ctx->f32_conv != NK_F32_GEMM_IEEE && ctx->conv_engine != NK_CONV_DIRECT;
}
int nk_conv_tf32_fwd(nk_ctx* ctx, void* y, const void* x, const void* w, const void* bias, int relu, int nsp, int64_t n,
                     int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                     const int64_t* pad, int mode, float value, bool nd);
int nk_conv_tf32_bwd_input(nk_ctx* ctx, void* dx, const void* g, const void* w, int nsp, int64_t n, int64_t cin,
                           const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s, const int64_t* dil,
                           const int64_t* pad, int mode, float beta, bool nd);
int nk_conv_tf32_bwd_kernel(nk_ctx* ctx, void* dwt, int dw_dtype, const void* g, const void* x, int nsp, int64_t n,
                            int64_t cin, const int64_t* in_sp, int64_t cout, const int64_t* k, const int64_t* s,
                            const int64_t* dil, const int64_t* pad, int mode, float value, float beta, bool nd);
bool nk_gemm_wgmma_supported(int transA, int transB, int64_t M, int64_t N, int64_t K,
                             const void* A, int64_t lda, const void* B, int64_t ldb);
