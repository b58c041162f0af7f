// nk_peer.cu -- data-parallel gradient exchange over NVLink peer memory (SURVEY.md 8-e).
//
// The reference has no multi-device path; the hot path's only exchange step is the sum of the weight gradients over
// the replicas before the SGD step (neuronika-optim/src/sgd/mod.rs:191-231 then runs identically on every replica).
// Instead of calling a library all-reduce after the dW GEMM, the exchange is fused into the kernels around it:
//   1. reduce-scatter inside the GEMM epilogue: nk_gemm_rs runs the wgmma dW GEMM, and the epilogue stores row shard
//      o of the local product straight into rank o's slot buffer over NVLink (slot index = this rank) -- the transfer
//      overlaps the MMAs tile by tile and the local gradient is never written to local HBM;
//   2. nk_reduce_exchange: ONE kernel for "all pushes landed" (flag exchange through peer memory) -> the owner sums its
//      `world` slots in rank order (so every replica receives bit-identical sums) and stores the result into EVERY
//      replica's gradient buffer over NVLink (the all-gather half) -> "all sums landed"; device-resident epoch, so the
//      launch is the same every step and can live in a CUDA graph (the r01 three-launch form -- nk_peer_barrier,
//      nk_reduce_bcast, nk_peer_barrier -- is kept);
//   3. nk_peer_allreduce_small: biases and other small tensors, one single-CTA kernel through peer memory, issued the
//      moment the gradient is final;
//   4. then the ordinary optimizer step (nk_multi_sgd_step) on every replica.
// Memory that peers touch comes from nk_ipc_alloc (plain cudaMalloc: CUDA IPC cannot export pool memory) and is
// mapped into the other processes with nk_ipc_export / nk_ipc_open.
#include "nk_internal.cuh"

#include <cstring>

namespace {

constexpr int kMaxWorld = 8;

struct PeerPtrs {
  void* p[kMaxWorld];
};

// one thread per peer: publish `epoch` in the peer's flag array, then wait for the peer's epoch in our own
__global__ void peer_barrier_kernel(PeerPtrs flags, int world, int rank, uint32_t epoch, int* error) {
  const int r = threadIdx.x;
  if (r >= world) return;
  __threadfence_system();
  volatile uint32_t* theirs = static_cast<uint32_t*>(flags.p[r]) + rank;
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(theirs), "r"(epoch) : "memory");
  const uint32_t* mine = static_cast<const uint32_t*>(flags.p[rank]) + r;
  const long long t0 = clock64();
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
    if (int32_t(v - epoch) >= 0) break;
    if (clock64() - t0 > 8000000000LL) {  // ~4 s: a peer died; fail loudly instead of hanging the GPU
      *error = 1;
      __trap();
    }
    __nanosleep(64);
  }
  __threadfence_system();
}

// out[e] = sum_s slots[s][e] (rank order), stored to every replica's gradient at `offset + e`
__global__ void __launch_bounds__(1024) reduce_bcast_kernel(const float4* __restrict__ slots, PeerPtrs grads, int world,
                                                            int64_t shard_vec, int64_t offset_vec) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  constexpr int U = 4;  // independent 16-byte loads in flight per thread and slot: few CTAs must still fill the pipes
  for (int64_t i0 = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i0 < shard_vec; i0 += U * stride) {
    float4 acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      acc[u] = i < shard_vec ? __ldcs(slots + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int s = 1; s < world; ++s) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = i < shard_vec ? __ldcs(slots + s * shard_vec + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) acc[u].x += v[u].x, acc[u].y += v[u].y, acc[u].z += v[u].z, acc[u].w += v[u].w;
    }
    for (int r = 0; r < world; ++r) {
      float4* g = static_cast<float4*>(grads.p[r]) + offset_vec;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        if (i < shard_vec) g[i] = acc[u];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// One kernel for "barrier -> owner reduce + broadcast -> barrier", with the epoch kept on the device so that the launch
// is identical every step (capturable in a CUDA graph) and with the work handed out dynamically, so that it may be
// launched with a CTA per SM: the CTAs that find an SM free while a GEMM runs start at once, the others pick up
// whatever is left when the GEMM's CTAs retire.
//   phase A  every rank tells every peer "my pushes into your slots have landed" (the GEMM that pushed them precedes
//            this kernel in stream order) and waits for the same word from all peers;
//   phase B  32 KB chunks of the local slot buffers are summed in rank order and stored into every replica's gradient;
//   phase C  the last CTA to finish tells every peer "my sums have landed in your gradient" and waits for theirs, so
//            the kernel's completion means this replica's gradient is final.
struct ExState {
  uint32_t epoch, done, next_chunk, error;
};
constexpr long long kPeerTimeout = 60000000000LL;  // ~30 s of SM clocks: a peer died; fail loudly instead of hanging

__device__ __forceinline__ void peer_signal(void* flag_base, int index, uint32_t epoch) {
  uint32_t* p = static_cast<uint32_t*>(flag_base) + index;
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(epoch) : "memory");
}
__device__ __forceinline__ void peer_wait(const void* flag_base, int index, uint32_t epoch, ExState* st) {
  const uint32_t* p = static_cast<const uint32_t*>(flag_base) + index;
  const long long t0 = clock64();
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    if (int32_t(v - epoch) >= 0) break;
    if (clock64() - t0 > kPeerTimeout) {
      st->error = 1;
      __trap();
    }
    __nanosleep(32);
  }
}

constexpr int kExThreads = 512;
constexpr int kExChunkVec = 2048;  // float4 per chunk and slot (32 KB)

__global__ void __launch_bounds__(kExThreads) reduce_exchange_kernel(const float4* __restrict__ slots, PeerPtrs grads,
                                                                     PeerPtrs flags, int world, int rank,
                                                                     int64_t shard_vec, int64_t offset_vec, ExState* st) {
  __shared__ uint32_t s_epoch;
  __shared__ uint32_t s_chunk;
  __shared__ int s_last;
  if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile uint32_t*>(&st->epoch) + 1u;
  __syncthreads();
  const uint32_t epoch = s_epoch;
  // ---- phase A
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    peer_signal(flags.p[threadIdx.x], rank, epoch);
  }
  if (threadIdx.x < world) peer_wait(flags.p[rank], threadIdx.x, epoch, st);
  __syncthreads();
  // ---- phase B
  const int64_t chunks = (shard_vec + kExChunkVec - 1) / kExChunkVec;
  for (;;) {
    if (threadIdx.x == 0) s_chunk = atomicAdd(&st->next_chunk, 1u);
    __syncthreads();
    const int64_t c = s_chunk;
    __syncthreads();
    if (c >= chunks) break;
    const int64_t base = c * kExChunkVec;
#pragma unroll
    for (int u = 0; u < kExChunkVec / kExThreads; ++u) {
      const int64_t i = base + u * kExThreads + threadIdx.x;
      if (i < shard_vec) {
        float4 acc = __ldcs(slots + i);
        for (int s = 1; s < world; ++s) {
          const float4 v = __ldcs(slots + s * shard_vec + i);
          acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
        }
        for (int r = 0; r < world; ++r) {
          const int rr = (r + rank) % world;  // every rank starts with a different replica: spreads the links
          static_cast<float4*>(grads.p[rr])[offset_vec + i] = acc;
        }
      }
    }
  }
  // ---- phase C
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&st->done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last) {
    if (threadIdx.x < world) {
      peer_signal(flags.p[threadIdx.x], world + rank, epoch);
      peer_wait(flags.p[rank], world + threadIdx.x, epoch, st);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      st->done = 0;
      st->next_chunk = 0;
      __threadfence();
      st->epoch = epoch;
    }
  }
}

// all-reduce of a SMALL vector (biases, the 10-wide layer) through peer memory, one CTA: every rank stores its local
// values into slot `rank` of every peer, signals, waits for all peers, then sums the `world` slots it received in rank
// order -- so every replica computes bit-identical sums -- into its own gradient.
__global__ void __launch_bounds__(1024) small_allreduce_kernel(float* __restrict__ grad, PeerPtrs slots, PeerPtrs flags,
                                                               int world, int rank, int64_t n, ExState* st) {
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile uint32_t*>(&st->epoch) + 1u;
  __syncthreads();
  const uint32_t epoch = s_epoch;
  // 16-byte accesses with 8 of them in flight per thread where the addresses allow it: one CTA moving 160 KB (the
  // 10 x 4096 weight gradient of config 4) element by element spent 60 us on load -> store round trips
  constexpr int U = 8;
  const bool vec = (n % 4 == 0) && ((reinterpret_cast<uintptr_t>(grad) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(slots.p[rank]) & 15) == 0);   // same slot offset on every rank
  const int64_t nv = vec ? n / 4 : 0;
  for (int64_t i0 = threadIdx.x; i0 < nv; i0 += int64_t(U) * blockDim.x) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + int64_t(u) * blockDim.x;
      if (i < nv) v[u] = reinterpret_cast<const float4*>(grad)[i];
    }
    for (int r = 0; r < world; ++r) {
      float4* dst = reinterpret_cast<float4*>(static_cast<float*>(slots.p[(r + rank) % world]) + int64_t(rank) * n);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + int64_t(u) * blockDim.x;
        if (i < nv) dst[i] = v[u];
      }
    }
  }
  if (!vec) {
    for (int r = 0; r < world; ++r) {
      float* dst = static_cast<float*>(slots.p[(r + rank) % world]) + int64_t(rank) * n;
      for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = grad[i];
    }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < world) {
    peer_signal(flags.p[threadIdx.x], rank, epoch);
    peer_wait(flags.p[rank], threadIdx.x, epoch, st);
  }
  __syncthreads();
  const float* mine = static_cast<const float*>(slots.p[rank]);
  for (int64_t i0 = threadIdx.x; i0 < nv; i0 += int64_t(U) * blockDim.x) {
    float4 acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + int64_t(u) * blockDim.x;
      acc[u] = i < nv ? __ldcv(reinterpret_cast<const float4*>(mine) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int s = 1; s < world; ++s) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + int64_t(u) * blockDim.x;
        v[u] = i < nv ? __ldcv(reinterpret_cast<const float4*>(mine + int64_t(s) * n) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) acc[u].x += v[u].x, acc[u].y += v[u].y, acc[u].z += v[u].z, acc[u].w += v[u].w;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + int64_t(u) * blockDim.x;
      if (i < nv) reinterpret_cast<float4*>(grad)[i] = acc[u];
    }
  }
  for (int64_t i = (vec ? n : 0) + threadIdx.x; i < n; i += blockDim.x) {
    float acc = __ldcv(mine + i);
    for (int s = 1; s < world; ++s) acc += __ldcv(mine + int64_t(s) * n + i);
    grad[i] = acc;
  }
  // second handshake: nobody may overwrite a slot (next step) before every rank has read it
  __syncthreads();
  if (threadIdx.x < world) {
    peer_signal(flags.p[threadIdx.x], world + rank, epoch);
    peer_wait(flags.p[rank], world + threadIdx.x, epoch, st);
  }
  __syncthreads();
  if (threadIdx.x == 0) st->epoch = epoch;
}

}  // namespace

extern "C" {

int nk_reduce_exchange(nk_ctx* ctx, const float* slots, void* const* grads, void* const* flags, int world, int rank,
                       int64_t shard_elems, void* state, int max_ctas) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, slots && grads && flags && state && world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world,
             "nk_reduce_exchange: bad arguments");
  NK_REQUIRE(ctx, shard_elems > 0 && shard_elems % 4 == 0, "nk_reduce_exchange: shard of %lld elements is not a positive multiple of 4",
             (long long)shard_elems);
  PeerPtrs g, f;
  for (int i = 0; i < kMaxWorld; ++i) g.p[i] = i < world ? grads[i] : nullptr, f.p[i] = i < world ? flags[i] : nullptr;
  const int64_t vec = shard_elems / 4;
  const int64_t chunks = (vec + kExChunkVec - 1) / kExChunkVec;
  int grid = max_ctas > 0 ? max_ctas : ctx->sm_count;
  if (grid > chunks) grid = int(chunks);
  reduce_exchange_kernel<<<grid, kExThreads, 0, ctx->stream>>>(reinterpret_cast<const float4*>(slots), g, f, world, rank, vec,
                                                               int64_t(rank) * vec, static_cast<ExState*>(state));
  NK_LAUNCHED(ctx, "reduce_exchange");
  return NK_OK;
}

int nk_peer_allreduce_small(nk_ctx* ctx, float* grad, void* const* slots, void* const* flags, int world, int rank,
                            int64_t n, void* state) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, grad && slots && flags && state && world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world,
             "nk_peer_allreduce_small: bad arguments");
  NK_REQUIRE(ctx, n > 0 && n <= (int64_t(1) << 20), "nk_peer_allreduce_small: n = %lld outside (0, 2^20]; use nk_allreduce_sum",
             (long long)n);
  PeerPtrs s, f;
  for (int i = 0; i < kMaxWorld; ++i) s.p[i] = i < world ? slots[i] : nullptr, f.p[i] = i < world ? flags[i] : nullptr;
  small_allreduce_kernel<<<1, 1024, 0, ctx->stream>>>(grad, s, f, world, rank, n, static_cast<ExState*>(state));
  NK_LAUNCHED(ctx, "peer_allreduce_small");
  return NK_OK;
}

int nk_ipc_alloc(nk_ctx* ctx, size_t bytes, void** out) {
  if (!ctx || !out) return NK_ERR_INVALID_ARG;
  *out = nullptr;
  if (bytes == 0) return NK_OK;
  NK_CUDA(ctx, cudaMalloc(out, bytes));
  NK_CUDA(ctx, cudaMemsetAsync(*out, 0, bytes, ctx->stream));
  NK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NK_OK;
}

int nk_ipc_free(nk_ctx* ctx, void* ptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (ptr) NK_CUDA(ctx, cudaFree(ptr));
  return NK_OK;
}

int nk_ipc_export(nk_ctx* ctx, void* ptr, void* handle64) {
  if (!ctx || !ptr || !handle64) return NK_ERR_INVALID_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  NK_CUDA(ctx, cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return NK_OK;
}

int nk_ipc_open(nk_ctx* ctx, const void* handle64, void** out) {
  if (!ctx || !handle64 || !out) return NK_ERR_INVALID_ARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  NK_CUDA(ctx, cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
  return NK_OK;
}

int nk_ipc_close(nk_ctx* ctx, void* peer_ptr) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (peer_ptr) NK_CUDA(ctx, cudaIpcCloseMemHandle(peer_ptr));
  return NK_OK;
}

int nk_peer_barrier(nk_ctx* ctx, void* const* flags, int world, int rank, uint32_t epoch) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, flags && world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world,
             "nk_peer_barrier: bad world %d / rank %d", world, rank);
  PeerPtrs f;
  for (int i = 0; i < kMaxWorld; ++i) f.p[i] = i < world ? flags[i] : nullptr;
  int* err;
  int rc = nk_workspace(ctx, 256, (void**)&err);
  if (rc) return rc;
  peer_barrier_kernel<<<1, 32, 0, ctx->stream>>>(f, world, rank, epoch, err);
  NK_LAUNCHED(ctx, "peer_barrier");
  return NK_OK;
}

int nk_reduce_bcast(nk_ctx* ctx, const float* slots, void* const* grads, int world, int rank, int64_t shard_elems,
                    int max_ctas) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, slots && grads && world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world,
             "nk_reduce_bcast: bad arguments");
  NK_REQUIRE(ctx, shard_elems % 4 == 0, "nk_reduce_bcast: shard of %lld elements is not a multiple of 4",
             (long long)shard_elems);
  if (shard_elems == 0) return NK_OK;
  PeerPtrs g;
  for (int i = 0; i < kMaxWorld; ++i) g.p[i] = i < world ? grads[i] : nullptr;
  const int64_t vec = shard_elems / 4;
  int grid = max_ctas > 0 ? max_ctas : 20;
  if (int64_t(grid) * 1024 > vec) grid = int((vec + 1023) / 1024);
  reduce_bcast_kernel<<<grid, 1024, 0, ctx->stream>>>(reinterpret_cast<const float4*>(slots), g, world, vec,
                                                      int64_t(rank) * vec);
  NK_LAUNCHED(ctx, "reduce_bcast");
  return NK_OK;
}

int nk_gemm_rs(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
               int64_t lda, const void* B, int64_t ldb, void* const* slots, int world, int rank, int ab_dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, slots && world >= 2 && world <= kMaxWorld && rank >= 0 && rank < world,
             "nk_gemm_rs: bad world %d / rank %d", world, rank);
  NK_REQUIRE(ctx, ab_dtype == NK_BF16, "nk_gemm_rs: the fused exchange runs on the tensor-core engine (bf16 operands)");
  NK_REQUIRE(ctx, M >= 0 && N >= 0 && K >= 0, "nk_gemm_rs: negative dimension");
  NK_REQUIRE(ctx, M % (int64_t(world) * 128) == 0, "nk_gemm_rs: M = %lld is not a multiple of world * 128",
             (long long)M);
  // the epilogue's conditions (launch_cfg), checked here so that the error names them: nk_gemm_bias_act would report
  // any refusal of the forced tensor-core engine as operands that TMA cannot address
  NK_REQUIRE(ctx, N > 128 && N % 4 == 0,
             "nk_gemm_rs: N = %lld: the reduce-scatter epilogue runs 128x256 tiles (N > 128) with 16-byte row stores "
             "(N %% 4 == 0)", (long long)N);
  for (int o = 0; o < world; ++o)
    NK_REQUIRE(ctx, slots[o] && (reinterpret_cast<uintptr_t>(slots[o]) & 15) == 0,
               "nk_gemm_rs: slot buffer %d is NULL or not 16-byte aligned", o);
  const int64_t shard = (M / world) * N;  // elements per (owner, source) slot
  if (M == 0) return NK_OK;
  if (K == 0) {
    // an empty local batch: the product is zero, and every owner still receives this rank's (zero) shard, so that all
    // ranks go on to the same exchange
    for (int o = 0; o < world; ++o) {
      const int rc = nk_memset0(ctx, static_cast<float*>(slots[o]) + int64_t(rank) * shard, size_t(shard) * sizeof(float));
      if (rc) return rc;
    }
    return NK_OK;
  }
  NK_REQUIRE(ctx, nk_gemm_wgmma_supported(transA, transB, M, N, K, A, lda, B, ldb),
             "nk_gemm_rs: operands are not TMA-addressable (16-byte aligned base, leading dimension multiple of 8 "
             "elements)");
  ctx->rs_world = world;
  ctx->rs_rank = rank;
  for (int o = 0; o < world; ++o) ctx->rs_dst[o] = static_cast<float*>(slots[o]) + int64_t(rank) * shard;
  const int saved = ctx->gemm_engine;
  ctx->gemm_engine = NK_GEMM_TC;
  const int rc = nk_gemm_bias_act(ctx, transA, transB, M, N, K, alpha, A, lda, B, ldb, 0.f, ctx->rs_dst[rank], N, ab_dtype,
                                  NK_F32, nullptr, NK_F32, 0);
  ctx->gemm_engine = saved;
  ctx->rs_world = 0;
  return rc;
}

}  // extern "C"
