// wgmma GEMM engine (sm_90a): C = alpha * op(A).op(B) + beta*C (+bias[n], ReLU)
// bf16 operands, f32 accumulation in registers, f32 or bf16 output.
//
// Serves the three GEMM forms of every matmul node (SURVEY.md 8-a):
//   NT  Y  = X.W^T   (MatrixMatrixMulT::forward, matrix_matrix_mul_t/mod.rs:31-41;  mm dA :63-73)
//   NN  dX = G.W     (MatrixMatrixMulTBackwardLeft :63-73;  mm forward matrix_matrix_mul/mod.rs:31-41)
//   TN  dW = G^T.X   (MatrixMatrixMulTBackwardRight :95-105;  mm dB :95-105)
// A "transposed" operand is never copied: TMA loads it as stored and the wgmma shared-memory
// descriptor is MN-major instead of K-major.
//
// Structure (persistent over 128 x BLOCK_N output tiles, one CTA per SM, three warpgroups):
//   warpgroup 0    : TMA producer (one thread) -- cp.async.bulk.tensor 128B-swizzled boxes into a kStages smem ring
//   warpgroups 1-2 : consumers -- each runs wgmma m64nBLOCK_Nk16 on its 64 rows of the tile with the accumulator in
//                    registers, keeping one k-block's wgmma group in flight: it issues k-block k, waits for k-1's group
//                    (wgmma.wait_group 1) and only then releases k-1's ring slot, so the tensor pipe never drains
//                    between k-blocks (the consumer holds two slots; the producer prefetches kStages - 2 ahead).
//                    Then the epilogue, one of two:
//                    - TMA store (column bias, alpha, ReLU, beta == 0, no mask / column sums / reduce-scatter, C
//                      TMA-addressable): every warp converts its 16 rows of fragments to C's type straight into one of
//                      two 128B-swizzled 16-row x 128-byte staging buffers of its own (stmatrix for bf16) and writes
//                      them with cp.async.bulk.tensor stores it issues itself, so the warps of a warpgroup never wait
//                      for each other; the stores drain while the warpgroup already runs the next tile's main loop.
//                      A bf16 column bias is copied into shared memory by the producer with the tile's first k-block,
//                      so the epilogue reads it without a global-memory round trip;
//                    - the drain: through a swizzled shared-memory stage, alpha/bias/ReLU, mask, beta, column sums,
//                      reduce-scatter over NVLink and batched outputs as 16-byte global stores per row.
// Pipeline: smem full/empty mbarriers (TMA <-> the two consumer warpgroups); bulk async-groups for the output stores.
#include "nk_internal.cuh"
#include "nk_ptx.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int kNumThreads = 384;   // producer warpgroup (registers given to the consumers) + two consumer warpgroups
constexpr uint32_t kSmemLimit = 232448;  // 227 KB
constexpr int kEpiCols = 64;                                       // accumulator columns staged per drain step
constexpr uint32_t kEpiStageBytes = 2 * 64 * kEpiCols * 4;         // 2 consumer warpgroups x 64 rows x 64 f32 = 32 KB

struct GemmParams {
  int64_t M, N, K;
  int64_t ldc;
  void* C;
  const void* bias;
  float alpha, beta;
  int bias_bf16;
  int bias_per_row;  // the bias is indexed by the output ROW (convolution: C rows are output channels) instead of the column
  int relu;
  const void* mask;    // optional (M, N) tensor of C's element type and leading dimension: v = mask > 0 ? v : 0 before the
                       // beta accumulate -- the ReLU backward of the layer below fused into the dX GEMM (relu/mod.rs:71-78)
  float* colsum;       // optional (N floats, accumulated with atomics; beta must be 0): column sums of the values the
                       // epilogue stores -- the bias gradient of the layer below (un-broadcast of its Addition,
                       // addition/mod.rs:81-135) without a separate pass over the (M, N) gradient
  int num_m_blocks, num_n_blocks, num_k_blocks;
  // wgmma descriptor parameters (bytes)
  uint32_t a_lbo, a_sbo, a_kstep;
  uint32_t b_lbo, b_sbo, b_kstep;
  // fused reduce-scatter epilogue (data parallel dW): rows [o*rs_rows, (o+1)*rs_rows) go to rs_dst[o]; m_rot = rank
  // staggers the owner order between ranks (tile_m_block)
  int rs_world, m_rot;
  int64_t rs_rows;
  void* rs_dst[8];
  // batched operation (im2col convolution, nk_gemm_batched): `batch` independent products whose operands are 3-D
  // tensor maps (k, rows, batch); C of product b starts c_batch_stride elements further.  batch_reduce: ONE output,
  // the products of all batches are summed (the k loop runs over (batch, k)); the batch range is split over
  // `splits` CTAs per tile, which add their partial sums into C with f32 atomics (C zeroed / scaled by the host).
  int batch, a_batched, b_batched, batch_reduce, splits;
  int64_t c_batch_stride;
  int tma_store;   // the epilogue writes C through the C tensor map (see the header); the host checks the conditions
  int bias_stage;  // TMA-store epilogue: the producer copies each tile's slice of the (bf16, 16-byte aligned, N % 8 == 0)
                   // column bias into shared memory
  int64_t bias_batch_stride;   // the bias of product b starts this many elements further (nk_gemm_strided_batched)
};

__device__ __forceinline__ int tile_m_block(const GemmParams& p, int tile) {
  const int t = tile % p.num_m_blocks;
  if (p.rs_world == 0) return t;
  // consecutive tiles go to consecutive owners (starting with a different one on every rank), so that the remote
  // stores are spread evenly over the whole kernel and over all links instead of bunching up at the end
  const int owner = (t + p.m_rot) % p.rs_world;
  return owner * (p.num_m_blocks / p.rs_world) + t / p.rs_world;
}

// tile index -> (m block, n block).  Tiles that run concurrently are consecutive indices (persistent CTAs stride by the
// grid), so consecutive indices walk kGroupM m-blocks before moving to the next n-block: a wave of ~128 tiles then
// covers a near-square 16 x 8 patch of the output and re-reads far less of A and B than an m-fastest order.
constexpr int kGroupM = 16;
__device__ __forceinline__ void tile_coords(const GemmParams& p, int tile, int& m_blk, int& n_blk) {
  if (p.rs_world) {
    m_blk = tile_m_block(p, tile);
    n_blk = tile / p.num_m_blocks;
    return;
  }
  const int group_size = kGroupM * p.num_n_blocks;
  const int group = tile / group_size, in_group = tile - group * group_size;
  const int first_m = group * kGroupM;
  const int gm = min(p.num_m_blocks - first_m, kGroupM);
  m_blk = first_m + in_group % gm;
  n_blk = in_group / gm;
}

template <int BLOCK_N>
struct Cfg {
  static constexpr uint32_t A_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
  static constexpr uint32_t B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  // after the ring: 1 KB of barriers, kEpiStageBytes of epilogue staging, then two BLOCK_N-wide bf16 bias slots (1 KB)
  static constexpr int kStagesMax = (kSmemLimit - 3072 - kEpiStageBytes) / STAGE_BYTES;
  static constexpr int kStages = kStagesMax > 8 ? 8 : kStagesMax;
  static constexpr uint32_t SMEM_BYTES = kStages * STAGE_BYTES + 3072 + kEpiStageBytes;  // + alignment slack + barriers
  static_assert(2 * BLOCK_N * 2 <= 1024, "bias slots");
};

// v[j] = alpha * acc[j] + bias (row- or column-indexed) for one 32-column chunk of one output row.  The product is
// rounded before the bias is added (__fmul_rn: never contracted into an FMA), in every epilogue, so that all of them
// store the same bits
// `bias` is p.bias, or the bias of the batch being drained
__device__ __forceinline__ void scale_and_bias(const GemmParams& p, const void* bias, int64_t row, int64_t col0,
                                               const uint32_t* r, bool full, float* v) {
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __fmul_rn(p.alpha, __uint_as_float(r[j]));
  if (bias && p.bias_per_row) {
    const float b = p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(bias)[row]) : static_cast<const float*>(bias)[row];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] += b;
  } else if (bias) {
    // 32 scalar loads here serialise on L1 latency and made the epilogue slower than a K = 1024 main loop:
    // fetch the 32 bias values of a full chunk with 16-byte loads
    if (full && (reinterpret_cast<uintptr_t>(bias) & 15) == 0) {
      if (p.bias_bf16) {
        const uint4* bp = reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(bias) + col0);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint4 w = __ldg(bp + q);
          const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            v[q * 8 + 2 * i] += __uint_as_float(ww[i] << 16);
            v[q * 8 + 2 * i + 1] += __uint_as_float(ww[i] & 0xffff0000u);
          }
        }
      } else {
        const float4* bp = reinterpret_cast<const float4*>(static_cast<const float*>(bias) + col0);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 w = __ldg(bp + q);
          v[q * 4] += w.x, v[q * 4 + 1] += w.y, v[q * 4 + 2] += w.z, v[q * 4 + 3] += w.w;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j < p.N)
          v[j] += p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(bias)[col0 + j])
                              : static_cast<const float*>(bias)[col0 + j];
    }
  }
}

// column sums of one 32-row x 32-column chunk (all 32 lanes of the warp take part; lane = row): the values are exactly the
// ones epilogue_store_chunk32 stores (alpha, mask, rounding to the output type), rows / columns outside the matrix count as
// zero.  A butterfly of 31 shuffles leaves the sum of column j on lane j; one atomic per column and chunk.
template <typename TC>
__device__ __forceinline__ void epilogue_colsum_chunk32(const GemmParams& p, int64_t row, int64_t col0, const uint32_t* r,
                                                        int lane, bool vec_ok) {
  float v[32];
  const bool live = row < p.M;
  const TC* mrow = (p.mask && live) ? static_cast<const TC*>(p.mask) + row * p.ldc + col0 : nullptr;
  const bool full = col0 + 32 <= p.N;
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = (live && col0 + j < p.N) ? p.alpha * __uint_as_float(r[j]) : 0.f;
  if (mrow) {
    if (full && vec_ok) {
      // the same four 16-byte loads per row the store path issues right after (then L1 hits): 32 scalar loads per row,
      // each a first touch of the mask, made the epilogue of an 8192 x 4096 GEMM longer than its main loop
      constexpr int V = 16 / sizeof(TC);
#pragma unroll
      for (int q = 0; q < 32 / V; ++q) {
        NkVec<TC> mk;
        mk.load(mrow + q * V);
#pragma unroll
        for (int i = 0; i < V; ++i) v[q * V + i] = mk.get(i) > 0.f ? v[q * V + i] : 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (col0 + j < p.N) v[j] = nk_to_f32<TC>(mrow[j]) > 0.f ? v[j] : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = nk_to_f32<TC>(nk_from_f32<TC>(v[j]));   // what the output tensor will hold
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const float send = upper ? v[i] : v[i + off];
      const float keep = upper ? v[i + off] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  if (col0 + lane < p.N) atomicAdd(p.colsum + col0 + lane, v[0]);
}

// The bias of the product whose C starts c_off elements into p.C (kernels instantiated with BATCH_BIAS, for
// nk_gemm_strided_batched: biases bias_batch_stride apart).  Derived from c_off where it is used rather than kept as a
// pointer across the drain: one more 64-bit value live in the 256-wide kernels, which run at the register cap, costs
// spills.  The other kernels (the convolution's batched ones among them) read p.bias as before.
template <bool BATCH_BIAS>
__device__ __forceinline__ const void* batch_bias(const GemmParams& p, int64_t c_off) {
  if (!BATCH_BIAS || !c_off) return p.bias;
  return static_cast<const char*>(p.bias) + (c_off / p.c_batch_stride) * p.bias_batch_stride * (p.bias_bf16 ? 2 : 4);
}

template <typename TC, bool BATCH_BIAS>
__device__ __forceinline__ void epilogue_store_chunk32(const GemmParams& p, int64_t row, int64_t col0, const uint32_t* r,
                                                       int ncols, bool vec_ok, int64_t c_off, bool atomic) {
  TC* crow = static_cast<TC*>(p.C) + c_off + row * p.ldc + col0;
  if (atomic) {  // partial sum of a split reduction: f32 atomics (alpha applied, beta handled by the host)
    if constexpr (sizeof(TC) == 4) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < ncols && col0 + j < p.N) atomicAdd(reinterpret_cast<float*>(crow) + j, p.alpha * __uint_as_float(r[j]));
    }
    return;
  }
  if (p.rs_world) {
    const int owner = int(row / p.rs_rows);
    crow = static_cast<TC*>(p.rs_dst[owner]) + (row - owner * p.rs_rows) * p.ldc + col0;
  }
  float v[32];
  const bool full = (col0 + 32 <= p.N) && ncols == 32;
  scale_and_bias(p, batch_bias<BATCH_BIAS>(p, c_off), row, col0, r, full, v);
  const TC* mrow = p.mask ? static_cast<const TC*>(p.mask) + row * p.ldc + col0 : nullptr;
  if (full && vec_ok) {
    constexpr int V = 16 / sizeof(TC);
    if (mrow) {
#pragma unroll
      for (int q = 0; q < 32 / V; ++q) {
        NkVec<TC> mk;
        mk.load(mrow + q * V);
#pragma unroll
        for (int i = 0; i < V; ++i) v[q * V + i] = mk.get(i) > 0.f ? v[q * V + i] : 0.f;
      }
    }
    if (p.beta != 0.f) {
#pragma unroll
      for (int q = 0; q < 32 / V; ++q) {
        NkVec<TC> c;
        c.load(crow + q * V);
#pragma unroll
        for (int i = 0; i < V; ++i) v[q * V + i] += p.beta * c.get(i);
      }
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : 0.f;
    }
#pragma unroll
    for (int q = 0; q < 32 / V; ++q) {
      NkVec<TC> o;
#pragma unroll
      for (int i = 0; i < V; ++i) o.set(i, v[q * V + i]);
      o.store(crow + q * V);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (j < ncols && col0 + j < p.N) {
        float x = v[j];
        if (mrow) x = nk_to_f32<TC>(mrow[j]) > 0.f ? x : 0.f;
        if (p.beta != 0.f) x += p.beta * nk_to_f32<TC>(crow[j]);
        if (p.relu) x = x > 0.f ? x : 0.f;
        crow[j] = nk_from_f32<TC>(x);
      }
    }
  }
}

// float offset of (row, col) in a consumer's 64 x kEpiCols f32 stage: the 16-byte units of a row are XOR-swizzled with
// the row, so that the eight rows a phase of row-wise 16-byte reads touches fall on distinct banks
__device__ __forceinline__ int epi_index(int row, int col) {
  return row * kEpiCols + ((((col >> 2) ^ (row & 7))) << 2) + (col & 3);
}

// bias[col] of the column-indexed bias, 0 past the last column
__device__ __forceinline__ float col_bias(const GemmParams& p, int64_t col) {
  if (col >= p.N) return 0.f;
  return p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(p.bias)[col]) : static_cast<const float*>(p.bias)[col];
}

// one output value of the TMA-store epilogue: the drain's alpha (rounded product), bias and ReLU
template <bool kAddBias>
__device__ __forceinline__ float epi_value(const GemmParams& p, float acc, float bias) {
  float v = __fmul_rn(p.alpha, acc);
  if (kAddBias) v += bias;
  return p.relu ? (v > 0.f ? v : 0.f) : v;
}

// where the TMA-store epilogue takes the column bias from
enum { kBiasNone, kBiasStaged, kBiasLoaded };

// TMA-store epilogue of one tile, per warp: chunk ch = columns [ch kStoreCols, +kStoreCols) of the warp's 16 rows.
// Lane holds rows r, r + 8 (r = lane / 4) and columns 8 jj + 2 (lane & 3) + {0, 1} of each 8-column block jj; they go,
// converted, to the 128B-swizzled layout of the C tensor map's 16-row box (16-byte unit u of row r at unit u ^ (r & 7);
// conflict-free: the eight rows of one 8 x 8 block hit eight different units).  Lane 0 issues and waits for the warp's
// own bulk stores, so a __syncwarp is all the hand-off a chunk needs.  The bias source is a template parameter: with a
// run-time choice inside the chunk loop the bias-free NN form paid about 2.5 kcycles more per tile (H100 SXM, 700 W)
template <int BLOCK_N, typename TC, int kBias>
__device__ __forceinline__ void tma_store_tile(const GemmParams& p, const CUtensorMap* tmap_c, const float (&acc)[BLOCK_N / 2],
                                               int lane, int row0, int64_t n0, uint32_t stg0, uint32_t bias_s,
                                               uint32_t& store_buf) {
  constexpr int kStoreCols = 128 / int(sizeof(TC));
  const int r = lane >> 2;
  const int q = lane & 3;
  // stmatrix: lanes 8i .. 8i + 7 address the rows of matrix i = (rows 8 (i & 1) + [0, 8), 8-column block jj + (i >> 1))
  // of a pair of blocks jj, jj + 1
  const int sm_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int sm_blk = lane >> 4;
#pragma unroll
  for (int ch = 0; ch < BLOCK_N / kStoreCols; ++ch) {
    const uint32_t buf = stg0 + store_buf * (64 * 128);
    if (lane == 0) ptx::tma_store_wait_read<1>();   // the store that last read this buffer is done with it
    __syncwarp();
    const int64_t col0 = n0 + ch * kStoreCols;
    uint32_t packed[4];   // bf16: blocks jj - 1 and jj, rows r and r + 8, for one stmatrix per pair of blocks
#pragma unroll
    for (int jj = 0; jj < kStoreCols / 8; ++jj) {
      const int j = (ch * (kStoreCols / 8) + jj) * 4;   // acc[j..j+1]: row r, acc[j+2..j+3]: row r + 8
      float b0 = 0.f, b1 = 0.f;
      if constexpr (kBias == kBiasStaged) {
        const uint32_t w = ptx::ld_shared_b32(bias_s + uint32_t(ch * kStoreCols + jj * 8 + 2 * q) * 2);
        b0 = __uint_as_float(w << 16), b1 = __uint_as_float(w & 0xffff0000u);
      } else if constexpr (kBias == kBiasLoaded) {
        const int64_t col = col0 + jj * 8 + 2 * q;
        b0 = col_bias(p, col), b1 = col_bias(p, col + 1);
      }
      constexpr bool kAdd = kBias != kBiasNone;
      const float v0 = epi_value<kAdd>(p, acc[j], b0), v1 = epi_value<kAdd>(p, acc[j + 1], b1);
      const float v2 = epi_value<kAdd>(p, acc[j + 2], b0), v3 = epi_value<kAdd>(p, acc[j + 3], b1);
      if constexpr (sizeof(TC) == 2) {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(v0, v1), hi = __floats2bfloat162_rn(v2, v3);
        packed[2 * (jj & 1)] = *reinterpret_cast<const uint32_t*>(&lo);
        packed[2 * (jj & 1) + 1] = *reinterpret_cast<const uint32_t*>(&hi);
        if (jj & 1) {
          const uint32_t off = sm_row * 128 + (((jj - 1 + sm_blk) ^ (sm_row & 7)) << 4);
          ptx::stmatrix_x4(buf + off, packed[0], packed[1], packed[2], packed[3]);
        }
      } else {
        // two f32 per row and block (stmatrix is b16 only): 8-byte stores, the eight rows of a store on distinct units
        const uint32_t off = r * 128 + (((2 * jj + (q >> 1)) ^ r) << 4) + (q & 1) * 8;
        ptx::st_shared_v2_f32(buf + off, v0, v1);
        ptx::st_shared_v2_f32(buf + off + 8 * 128, v2, v3);
      }
    }
    ptx::fence_proxy_async();   // the staged chunk is visible to the TMA unit ...
    __syncwarp();
    if (lane == 0) {            // ... which clips the box at M, N (the ldc - N gap is never written)
      if (row0 < p.M && col0 < p.N) ptx::tma_store_2d(tmap_c, buf, int(col0), row0);
      ptx::tma_store_commit();   // (an empty group when nothing was issued: one group per chunk)
    }
    store_buf ^= 1u;
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, typename TC, bool BATCH = false, bool BATCH_BIAS = false>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_c, const GemmParams p) {
  using C_ = Cfg<BLOCK_N>;
  constexpr int kStages = C_::kStages;
  // TMA-store epilogue: chunks of one 128-byte swizzle row (64 bf16 / 32 f32 columns) x 16 rows per warp, two 2 KB
  // staging buffers per consumer warp (two 8 KB buffers per warpgroup in its half of the epilogue stage)
  constexpr int kStoreCols = 128 / int(sizeof(TC));
  constexpr bool kTmaStore = !BATCH && BLOCK_N % kStoreCols == 0;
  static_assert(2 * 2 * 64 * 128 <= kEpiStageBytes, "staging buffers");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms: 1024 B aligned
  const uint32_t smem_a0 = smem_base;
  const uint32_t smem_b0 = smem_base + kStages * C_::A_BYTES;
  const uint32_t bar_base = smem_base + kStages * C_::STAGE_BYTES;  // 8-byte aligned
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  // bias slot s (tiles of even / odd local index) is free again once all eight consumer warps have read it
  auto bias_empty_bar = [&](int s) { return bar_base + 8u * (2 * kStages + s); };
  const uint32_t epi_stage = bar_base + 1024;
  float* epi = reinterpret_cast<float*>(smem_raw + (epi_stage - ptx::smem_u32(smem_raw)));
  auto bias_slot = [&](int s) { return epi_stage + kEpiStageBytes + uint32_t(s) * (BLOCK_N * 2); };
  const bool stage_bias = kTmaStore && p.tma_store && p.bias_stage;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
    if (kTmaStore && p.tma_store) ptx::prefetch_tmap(&tmap_c);
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    for (int s = 0; s < 2; ++s) ptx::mbar_init(bias_empty_bar(s), 8);   // one arrive per consumer warp
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int tiles_mn = p.num_m_blocks * p.num_n_blocks;
  // BATCH: a "tile" is (batch or split, m block, n block); the k loop of a reducing launch walks its share of the batches
  const int num_tiles = BATCH ? tiles_mn * (p.batch_reduce ? p.splits : p.batch) : tiles_mn;
  auto batch_range = [&](int outer, int& b0, int& b1) {   // batches whose products tile `outer` accumulates
    if (!p.batch_reduce) {
      b0 = outer, b1 = outer + 1;
    } else {
      const int per = (p.batch + p.splits - 1) / p.splits;
      b0 = outer * per;
      b1 = min(p.batch, b0 + per);
    }
  };

  if (wg == 0) {
    // ===================================================== TMA producer
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x, local = 0; tile < num_tiles; tile += gridDim.x, ++local) {
        int m_blk, n_blk, b0 = 0, b1 = 1;
        tile_coords(p, BATCH ? tile % tiles_mn : tile, m_blk, n_blk);
        if (BATCH) batch_range(tile / tiles_mn, b0, b1);
        const int m0 = m_blk * BLOCK_M, n0 = n_blk * BLOCK_N;
        for (int bb = b0; bb < b1; ++bb)
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          ptx::mbar_wait_spin(empty_bar(stage), phase ^ 1u);
          if (stage_bias && kb == 0) {
            // the tile's bias slice rides on its first k-block's barrier.  With one or two k-blocks per tile this thread
            // can run more than a tile ahead of the consumers: the slot is reused only after they have read it
            const int s = local & 1;
            const uint32_t bytes = 2u * uint32_t(min(int64_t(BLOCK_N), p.N - n0));   // a multiple of 16: N % 8 == 0
            ptx::mbar_wait_spin(bias_empty_bar(s), ((local >> 1) & 1) ^ 1u);
            ptx::mbar_expect_tx(full_bar(stage), C_::STAGE_BYTES + bytes);
            ptx::bulk_load(bias_slot(s), static_cast<const __nv_bfloat16*>(p.bias) + n0, bytes, full_bar(stage));
          } else {
            ptx::mbar_expect_tx(full_bar(stage), C_::STAGE_BYTES);
          }
          const int k0 = kb * BLOCK_K;
          const uint32_t sa = smem_a0 + stage * C_::A_BYTES;
          const uint32_t sb = smem_b0 + stage * C_::B_BYTES;
          if (A_MN) {  // stored (K, M): boxes of 64 (m) x 64 (k)
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c) {
              if (BATCH && p.a_batched)
                ptx::tma_load_3d(sa + c * (64 * BLOCK_K * 2), &tmap_a, full_bar(stage), m0 + c * 64, k0, bb);
              else
                ptx::tma_load_2d(sa + c * (64 * BLOCK_K * 2), &tmap_a, full_bar(stage), m0 + c * 64, k0);
            }
          } else {  // stored (M, K): one box of 64 (k) x 128 (m)
            if (BATCH && p.a_batched)
              ptx::tma_load_3d(sa, &tmap_a, full_bar(stage), k0, m0, bb);
            else
              ptx::tma_load_2d(sa, &tmap_a, full_bar(stage), k0, m0);
          }
          if (B_MN) {  // stored (K, N)
#pragma unroll
            for (int c = 0; c < BLOCK_N / 64; ++c) {
              if (BATCH && p.b_batched)
                ptx::tma_load_3d(sb + c * (64 * BLOCK_K * 2), &tmap_b, full_bar(stage), n0 + c * 64, k0, bb);
              else
                ptx::tma_load_2d(sb + c * (64 * BLOCK_K * 2), &tmap_b, full_bar(stage), n0 + c * 64, k0);
            }
          } else {  // stored (N, K)
            if (BATCH && p.b_batched)
              ptx::tma_load_3d(sb, &tmap_b, full_bar(stage), k0, n0, bb);
            else
              ptx::tma_load_2d(sb, &tmap_b, full_bar(stage), k0, n0);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup 1 owns tile rows [0, 64), warpgroup 2 [64, 128)
  ptx::setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5;
  const bool vec_ok = ((p.ldc * int64_t(sizeof(TC))) % 16 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.mask) & 15) == 0);
  float* stg = epi + cw * (64 * kEpiCols);
  // A rows of this warpgroup: K-major, 64 rows x 128 B further; MN-major, the second 64-wide m box -- 8 KB either way
  const uint32_t a_off = uint32_t(cw) * (64 * BLOCK_K * 2);
  float acc[BLOCK_N / 2];
  int stage = 0;
  uint32_t phase = 0;
  uint32_t store_buf = 0;   // TMA-store epilogue: the staging buffer the next chunk goes to
  for (int tile = blockIdx.x, local = 0; tile < num_tiles; tile += gridDim.x, ++local) {
    int m_blk, n_blk;
    tile_coords(p, BATCH ? tile % tiles_mn : tile, m_blk, n_blk);
    int k_total = p.num_k_blocks;
    if (BATCH) {
      int b0, b1;
      batch_range(tile / tiles_mn, b0, b1);
      k_total *= (b1 - b0);
    }
    int prev_stage = 0;
    for (int kb = 0; kb < k_total; ++kb) {
      ptx::mbar_wait_spin(full_bar(stage), phase);
      const uint64_t adesc = ptx::make_smem_desc_sw128(smem_a0 + stage * C_::A_BYTES + a_off, p.a_lbo, p.a_sbo);
      const uint64_t bdesc = ptx::make_smem_desc_sw128(smem_b0 + stage * C_::B_BYTES, p.b_lbo, p.b_sbo);
      ptx::fence_regs(acc);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
        ptx::Wgmma<BLOCK_N>::template mma<int(A_MN), int(B_MN)>(acc, adesc + uint64_t((k * p.a_kstep) >> 4),
                                                                 bdesc + uint64_t((k * p.b_kstep) >> 4), (kb | k) != 0 ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();   // k-block kb - 1's group is done; kb's stays in flight
      ptx::fence_regs(acc);
      if (kb > 0 && t == 0) ptx::mbar_arrive(empty_bar(prev_stage));  // this warpgroup is done reading kb - 1's slot
      prev_stage = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1u;
      }
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    if (t == 0) ptx::mbar_arrive(empty_bar(prev_stage));

    if constexpr (kTmaStore) {
      if (p.tma_store) {
        // ---- TMA-store epilogue (tma_store_tile), each warp on its own two 16-row staging buffers
        const int row0 = m_blk * BLOCK_M + cw * 64 + warp * 16;
        const int64_t n0 = int64_t(n_blk) * BLOCK_N;
        const uint32_t stg0 = epi_stage + uint32_t(cw) * (2 * 64 * 128) + uint32_t(warp) * (16 * 128);
        const uint32_t bias_s = bias_slot(local & 1);
        if (stage_bias)
          tma_store_tile<BLOCK_N, TC, kBiasStaged>(p, &tmap_c, acc, lane, row0, n0, stg0, bias_s, store_buf);
        else if (p.bias)
          tma_store_tile<BLOCK_N, TC, kBiasLoaded>(p, &tmap_c, acc, lane, row0, n0, stg0, bias_s, store_buf);
        else
          tma_store_tile<BLOCK_N, TC, kBiasNone>(p, &tmap_c, acc, lane, row0, n0, stg0, bias_s, store_buf);
        if (stage_bias) {   // this warp is done with the tile's bias slot
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(bias_empty_bar(local & 1));
        }
        continue;   // the stores drain while the next tile's main loop runs
      }
    }

    // ---- epilogue: kEpiCols accumulator columns at a time through the stage; warp w then drains row
    // 32 (w & 1) + lane, columns [32 (w >> 1), +32) of the staged chunk with the row-wise store / column-sum code
    const int64_t c_off = (BATCH && !p.batch_reduce) ? int64_t(tile / tiles_mn) * p.c_batch_stride : 0;
    const bool atomic = BATCH && p.batch_reduce;
    const int fr = warp * 16 + (lane >> 2);   // fragment rows fr, fr + 8
    const int fc = (lane & 3) * 2;
    const int half = warp >> 1;
    const int rloc = (warp & 1) * 32 + lane;
    const int64_t row = int64_t(m_blk) * BLOCK_M + cw * 64 + rloc;
    constexpr int kChunks = (BLOCK_N + kEpiCols - 1) / kEpiCols;
#pragma unroll
    for (int ch = 0; ch < kChunks; ++ch) {
      constexpr int kFullBlocks = kEpiCols / 8;
      ptx::named_barrier(1 + cw, 128);   // the previous chunk has been drained
#pragma unroll
      for (int nb = 0; nb < kFullBlocks; ++nb) {
        if (ch * kFullBlocks + nb < BLOCK_N / 8) {
          const int j = (ch * kFullBlocks + nb) * 4;
          *reinterpret_cast<float2*>(stg + epi_index(fr, nb * 8 + fc)) = make_float2(acc[j], acc[j + 1]);
          *reinterpret_cast<float2*>(stg + epi_index(fr + 8, nb * 8 + fc)) = make_float2(acc[j + 2], acc[j + 3]);
        }
      }
      ptx::named_barrier(1 + cw, 128);
      const int chunk_cols = BLOCK_N - ch * kEpiCols < kEpiCols ? BLOCK_N - ch * kEpiCols : kEpiCols;
      if (!vec_ok && !p.colsum && !p.mask && !p.rs_world) {
        // rows that 16-byte stores cannot address (odd leading dimension, e.g. a convolution with Ho*Wo % 8 != 0): warp w
        // drains rows [16w, 16w + 16) of the chunk with lane = column, so that every store instruction writes one
        // contiguous run of a row instead of 32 scattered elements
        const int64_t col_base = int64_t(n_blk) * BLOCK_N + ch * kEpiCols;
        for (int rr = 0; rr < 16; ++rr) {
          const int srow = warp * 16 + rr;
          const int64_t grow = int64_t(m_blk) * BLOCK_M + cw * 64 + srow;
          if (grow >= p.M) break;
          const void* bias = p.bias;
          if constexpr (BATCH_BIAS) bias = batch_bias<true>(p, c_off);
          float rb = 0.f;
          if (bias && p.bias_per_row)
            rb = p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(bias)[grow]) : static_cast<const float*>(bias)[grow];
          for (int c = lane; c < chunk_cols; c += 32) {
            const int64_t col = col_base + c;
            if (col >= p.N) break;
            float v = __fmul_rn(p.alpha, stg[epi_index(srow, c)]);
            TC* cp = static_cast<TC*>(p.C) + c_off + grow * p.ldc + col;
            if (atomic) {
              if constexpr (sizeof(TC) == 4) atomicAdd(reinterpret_cast<float*>(cp), v);
              continue;
            }
            if (bias) {
              v += p.bias_per_row ? rb
                                  : (p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(bias)[col])
                                                 : static_cast<const float*>(bias)[col]);
            }
            if (p.beta != 0.f) v += p.beta * nk_to_f32<TC>(*cp);
            if (p.relu) v = v > 0.f ? v : 0.f;
            *cp = nk_from_f32<TC>(v);
          }
        }
        continue;
      }
      const int ncols = min(32, chunk_cols - half * 32);
      if (ncols > 0) {   // warp-uniform
        uint32_t r[32];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (q * 4 < ncols) v = *reinterpret_cast<const float4*>(stg + epi_index(rloc, half * 32 + q * 4));
          r[4 * q] = __float_as_uint(v.x), r[4 * q + 1] = __float_as_uint(v.y);
          r[4 * q + 2] = __float_as_uint(v.z), r[4 * q + 3] = __float_as_uint(v.w);
        }
        const int64_t col0 = int64_t(n_blk) * BLOCK_N + ch * kEpiCols + half * 32;
        if (p.colsum && col0 < p.N) epilogue_colsum_chunk32<TC>(p, row, col0, r, lane, vec_ok);
        if (row < p.M && col0 < p.N) epilogue_store_chunk32<TC, BATCH_BIAS>(p, row, col0, r, ncols, vec_ok, c_off, atomic);
      }
    }
  }
  if (kTmaStore && p.tma_store && lane == 0) ptx::tma_store_wait<0>();   // the staging buffers outlive the last stores
}

}  // namespace

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D tensor map (bf16 or f32 elements): `rows` x `cols` row-major with leading dimension ld, box (box_cols, box_rows)
// with box_cols elements = 128 bytes, 128B-swizzled
int make_tmap_2d(nk_ctx* ctx, CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld,
                 uint32_t box_cols, uint32_t box_rows, int dtype) {
  if (!ctx->encode_tiled) return nk_set_error(ctx, NK_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * nk_dtype_size(dtype)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled)(
      tm, dtype == NK_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
      const_cast<void*>(base), dims, strides, box, estr,
      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return nk_set_error(ctx, NK_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r,
                        (long long)rows, (long long)cols, (long long)ld);
  return NK_OK;
}

namespace {

template <int BLOCK_N, bool A_MN, bool B_MN, typename TC, bool BATCH = false, bool BATCH_BIAS = false>
int launch_cfg(nk_ctx* ctx, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, GemmParams& p) {
  using C_ = Cfg<BLOCK_N>;
  auto kern = gemm_tc_kernel<BLOCK_N, A_MN, B_MN, TC, BATCH, BATCH_BIAS>;
  static bool attr_done[64] = {};  // per template instantiation and device (the attribute is per device)
  if (!attr_done[ctx->device & 63]) {
    static_assert(C_::SMEM_BYTES <= kSmemLimit, "shared memory budget");
    NK_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C_::SMEM_BYTES));
    attr_done[ctx->device & 63] = true;
  }
  p.num_n_blocks = int((p.N + BLOCK_N - 1) / BLOCK_N);
  int num_tiles = p.num_m_blocks * p.num_n_blocks;
  if (BATCH) {
    if (p.batch_reduce) {
      // split the batch range so that the launch fills the machine; every split gets at least one batch
      int want = (ctx->sm_count + num_tiles - 1) / num_tiles;
      if (want > p.batch) want = p.batch;
      const int per = (p.batch + want - 1) / want;
      p.splits = (p.batch + per - 1) / per;
      num_tiles *= p.splits;
    } else {
      num_tiles *= p.batch;
    }
  }
  // persistent grid balanced over the waves the tiles need anyway: 256 tiles on 132 SMs take 2 waves whether 132
  // or 128 CTAs run them, and the SMs left free let a concurrent NCCL all-reduce make progress
  const int units = ctx->sm_count;
  const int waves = (num_tiles + units - 1) / units;
  const int grid = (num_tiles + waves - 1) / waves;
  const size_t smem = C_::SMEM_BYTES;
  if (p.rs_world) {
    if (BLOCK_N != 256 || sizeof(TC) != 4 || p.N % 4 != 0)
      return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "wgmma gemm: reduce-scatter epilogue needs 128x256 tiles, f32, N %% 4 == 0");
  }
  kern<<<grid, kNumThreads, smem, ctx->stream>>>(ta, tb, tc, p);
  ctx->launches++;
  cudaError_t le = cudaGetLastError();
  if (le != cudaSuccess)
    return nk_set_error(ctx, NK_ERR_CUDA, "launch of gemm_wgmma failed: %s (M=%lld N=%lld K=%lld BLOCK_N=%d grid=%d smem=%zu "
                        "a_mn=%d b_mn=%d out=%s)", cudaGetErrorString(le), (long long)p.M, (long long)p.N, (long long)p.K,
                        BLOCK_N, grid, smem, int(A_MN), int(B_MN), sizeof(TC) == 4 ? "f32" : "bf16");
  return NK_OK;
}

template <bool A_MN, bool B_MN, typename TC>
int launch_bn(nk_ctx* ctx, int block_n, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, GemmParams& p) {
  switch (block_n) {
    case 256: return launch_cfg<256, A_MN, B_MN, TC>(ctx, ta, tb, tc, p);
    case 128: return launch_cfg<128, A_MN, B_MN, TC>(ctx, ta, tb, tc, p);
    case 64: return launch_cfg<64, A_MN, B_MN, TC>(ctx, ta, tb, tc, p);
    default:
      if (!B_MN) {
        if (block_n == 32) return launch_cfg<32, A_MN, false, TC>(ctx, ta, tb, tc, p);
        if (block_n == 16) return launch_cfg<16, A_MN, false, TC>(ctx, ta, tb, tc, p);
      }
      return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "wgmma gemm: unsupported BLOCK_N %d", block_n);
  }
}

}  // namespace

bool nk_gemm_wgmma_supported(int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                             const void* B, int64_t ldb) {
  (void)transA;
  (void)transB;
  if (M <= 0 || N <= 0 || K <= 0) return false;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return false;
  if ((lda * 2) % 16 != 0 || (ldb * 2) % 16 != 0) return false;  // TMA global strides: multiples of 16 bytes
  if (M > (int64_t(1) << 30) || N > (int64_t(1) << 30) || K > (int64_t(1) << 30)) return false;
  return true;
}

int nk_gemm_wgmma(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                  int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int c_dtype,
                  const void* bias, int bias_dtype, int relu, const void* mask, float* colsum) {
  if (!nk_gemm_wgmma_supported(transA, transB, M, N, K, A, lda, B, ldb)) return NK_ERR_UNSUPPORTED;
  if (colsum && (N <= 16 || beta != 0.f)) return NK_ERR_UNSUPPORTED;   // (the narrow-tile epilogue has no column-sum path)
  const bool a_mn = transA != 0;   // op(A) = A^T  -> A stored (K, M), M contiguous
  const bool b_mn = transB == 0;   // op(B) = B    -> B stored (K, N), N contiguous
  // tile width: widest that does not leave most of a tile empty
  int block_n = 256;
  if (N <= 16 && !b_mn)
    block_n = 16;
  else if (N <= 32 && !b_mn)
    block_n = 32;
  else if (N <= 64)
    block_n = 64;
  else if (N <= 128)
    block_n = 128;

  GemmParams p;
  p.M = M;
  p.N = N;
  p.K = K;
  p.ldc = ldc;
  p.C = C;
  p.bias = bias;
  p.alpha = alpha;
  p.beta = beta;
  p.bias_bf16 = bias_dtype == NK_BF16;
  p.bias_per_row = 0;
  p.relu = relu;
  p.mask = mask;
  p.colsum = colsum;
  p.batch = 1, p.a_batched = p.b_batched = p.batch_reduce = 0, p.splits = 1, p.c_batch_stride = 0, p.bias_batch_stride = 0;
  p.num_m_blocks = int((M + BLOCK_M - 1) / BLOCK_M);
  p.num_n_blocks = 0;
  p.num_k_blocks = int((K + BLOCK_K - 1) / BLOCK_K);
  p.rs_world = 0;
  p.m_rot = 0;
  p.rs_rows = M;
  for (int i = 0; i < 8; ++i) p.rs_dst[i] = nullptr;
  if (ctx->rs_world > 1) {
    if (M % (int64_t(ctx->rs_world) * BLOCK_M) != 0 || beta != 0.f || c_dtype != NK_F32)
      return nk_set_error(ctx, NK_ERR_INVALID_ARG, "wgmma gemm: reduce-scatter epilogue needs M %% (world*128) == 0, "
                          "beta == 0 and f32 output");
    p.rs_world = ctx->rs_world;
    p.rs_rows = M / ctx->rs_world;
    p.m_rot = ctx->rs_rank;
    for (int i = 0; i < ctx->rs_world; ++i) p.rs_dst[i] = ctx->rs_dst[i];
  }
  // K-major: 8-row groups 1024 B apart, +32 B per WGMMA_K.  MN-major: 64-wide chunks
  // BLOCK_K*128 B apart (LBO), 8-k groups 1024 B apart (SBO), +16 rows * 128 B per WGMMA_K.
  p.a_lbo = a_mn ? BLOCK_K * 128 : 16;
  p.a_sbo = 1024;
  p.a_kstep = a_mn ? WGMMA_K * 128 : WGMMA_K * 2;
  p.b_lbo = b_mn ? BLOCK_K * 128 : 16;
  p.b_sbo = 1024;
  p.b_kstep = b_mn ? WGMMA_K * 128 : WGMMA_K * 2;

  CUtensorMap ta, tb;
  int rc;
  if (a_mn)
    rc = make_tmap_2d(ctx, &ta, A, K, M, lda, 64, BLOCK_K);
  else
    rc = make_tmap_2d(ctx, &ta, A, M, K, lda, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  if (b_mn)
    rc = make_tmap_2d(ctx, &tb, B, K, N, ldb, 64, BLOCK_K);
  else
    rc = make_tmap_2d(ctx, &tb, B, N, K, ldb, BLOCK_K, (uint32_t)block_n);
  if (rc) return rc;
  // TMA-store epilogue: an output the epilogue only writes (beta 0; alpha, column bias and ReLU are applied on the way)
  // and that TMA can address; box = one warp's 16-row x 128-byte staging buffer, whole chunks per tile.  The rows must also end
  // on a 16-byte boundary: a store box clips at the last row exactly but at the last column only to the 16-byte unit
  // that holds it, which would write into the ldc - N gap
  const int64_t c_size = int64_t(nk_dtype_size(c_dtype));
  CUtensorMap tc;
  memset(&tc, 0, sizeof(tc));
  p.tma_store = beta == 0.f && !mask && !colsum && !p.rs_world && (block_n * c_size) % 128 == 0 &&
                (reinterpret_cast<uintptr_t>(C) & 15) == 0 && (ldc * c_size) % 16 == 0 && (N * c_size) % 16 == 0;
  if (p.tma_store) {
    rc = make_tmap_2d(ctx, &tc, C, M, N, ldc, uint32_t(128 / c_size), 16, c_dtype);
    if (rc) return rc;
  }
  // a bias slice every tile can fetch with one bulk copy: bf16 (f32 would not fit the slots), 16-byte aligned, and
  // N % 8 == 0 so that the last tile's slice is a whole number of 16-byte units; otherwise the epilogue loads it
  p.bias_stage = p.tma_store && bias && bias_dtype == NK_BF16 && (reinterpret_cast<uintptr_t>(bias) & 15) == 0 && N % 8 == 0;

  static const char* names[2][2][5] = {
      {{"wgmma_nt_128x256", "wgmma_nt_128x128", "wgmma_nt_128x64", "wgmma_nt_128x32", "wgmma_nt_128x16"},
       {"wgmma_nn_128x256", "wgmma_nn_128x128", "wgmma_nn_128x64", "", ""}},
      {{"wgmma_tt_128x256", "wgmma_tt_128x128", "wgmma_tt_128x64", "wgmma_tt_128x32", "wgmma_tt_128x16"},
       {"wgmma_tn_128x256", "wgmma_tn_128x128", "wgmma_tn_128x64", "", ""}}};
  const int bi = block_n == 256 ? 0 : block_n == 128 ? 1 : block_n == 64 ? 2 : block_n == 32 ? 3 : 4;
  ctx->last_gemm_kernel = names[a_mn][b_mn][bi];

#define NK_TC(AM, BM_)                                                              \
  (c_dtype == NK_BF16 ? launch_bn<AM, BM_, __nv_bfloat16>(ctx, block_n, ta, tb, tc, p) \
                      : launch_bn<AM, BM_, float>(ctx, block_n, ta, tb, tc, p))
  if (!a_mn && !b_mn) return NK_TC(false, false);
  if (!a_mn && b_mn) return NK_TC(false, true);
  if (a_mn && !b_mn) return NK_TC(true, false);
  return NK_TC(true, true);
#undef NK_TC
}

// 3-D bf16 tensor map (cols, rows, batch)
static int make_tmap_3d(nk_ctx* ctx, CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld, int64_t batch,
                        int64_t batch_stride, uint32_t box_cols, uint32_t box_rows) {
  if (!ctx->encode_tiled) return nk_set_error(ctx, NK_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)batch_stride * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled)(
      tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return nk_set_error(ctx, NK_ERR_CUDA, "cuTensorMapEncodeTiled (3-d) failed (%d) rows=%lld cols=%lld ld=%lld batch=%lld stride=%lld",
                        (int)r, (long long)rows, (long long)cols, (long long)ld, (long long)batch, (long long)batch_stride);
  return NK_OK;
}

// `batch` products C_b = alpha * op(A_b).op(B_b) + beta*C_b (+ bias, ReLU) with operands batch_stride elements apart
// (stride 0 = the same operand for every batch), or -- reduce != 0 -- ONE product C += alpha * sum_b op(A_b).op(B_b) (C
// f32, accumulated with atomics: the caller zeroes / scales C first; beta is ignored).  The bias is indexed by the output
// row (bias_per_row) or column; that of product b starts bias_stride elements further.
static int gemm_wgmma_batched(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                              int64_t lda, int64_t strideA, const void* B, int64_t ldb, int64_t strideB, float beta, void* C,
                              int64_t ldc, int64_t strideC, int64_t batch, int c_dtype, const void* bias, int bias_dtype,
                              int bias_per_row, int64_t bias_stride, int relu, int reduce) {
  if (!nk_gemm_wgmma_supported(transA, transB, M, N, K, A, lda, B, ldb)) return NK_ERR_UNSUPPORTED;
  if (batch < 1 || batch > (int64_t(1) << 30) || (strideA * 2) % 16 != 0 || (strideB * 2) % 16 != 0) return NK_ERR_UNSUPPORTED;
  if (reduce && c_dtype != NK_F32) return NK_ERR_UNSUPPORTED;
  const bool a_mn = transA != 0, b_mn = transB == 0;
  int block_n = N <= 64 ? 64 : (N <= 128 ? 128 : 256);
  GemmParams p;
  p.M = M, p.N = N, p.K = K, p.ldc = ldc, p.C = C;
  p.bias = bias, p.bias_bf16 = bias_dtype == NK_BF16, p.bias_per_row = bias_per_row;
  p.bias_batch_stride = bias ? bias_stride : 0;   // the drain finds a product's bias from its C offset (batch_bias)
  p.alpha = alpha, p.beta = reduce ? 0.f : beta, p.relu = relu, p.mask = nullptr, p.colsum = nullptr;
  p.num_m_blocks = int((M + BLOCK_M - 1) / BLOCK_M);
  p.num_n_blocks = 0;
  p.num_k_blocks = int((K + BLOCK_K - 1) / BLOCK_K);
  p.rs_world = 0, p.m_rot = 0, p.rs_rows = M;
  for (int i = 0; i < 8; ++i) p.rs_dst[i] = nullptr;
  p.batch = int(batch), p.a_batched = strideA != 0, p.b_batched = strideB != 0, p.batch_reduce = reduce ? 1 : 0, p.splits = 1;
  p.c_batch_stride = strideC;
  p.tma_store = 0;   // batched outputs (and the row-indexed bias) keep the drain
  p.bias_stage = 0;
  p.a_lbo = a_mn ? BLOCK_K * 128 : 16, p.a_sbo = 1024, p.a_kstep = a_mn ? WGMMA_K * 128 : WGMMA_K * 2;
  p.b_lbo = b_mn ? BLOCK_K * 128 : 16, p.b_sbo = 1024, p.b_kstep = b_mn ? WGMMA_K * 128 : WGMMA_K * 2;
  CUtensorMap ta, tb;
  int rc;
  if (p.a_batched)
    rc = a_mn ? make_tmap_3d(ctx, &ta, A, K, M, lda, batch, strideA, 64, BLOCK_K)
              : make_tmap_3d(ctx, &ta, A, M, K, lda, batch, strideA, BLOCK_K, BLOCK_M);
  else
    rc = a_mn ? make_tmap_2d(ctx, &ta, A, K, M, lda, 64, BLOCK_K) : make_tmap_2d(ctx, &ta, A, M, K, lda, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  if (p.b_batched)
    rc = b_mn ? make_tmap_3d(ctx, &tb, B, K, N, ldb, batch, strideB, 64, BLOCK_K)
              : make_tmap_3d(ctx, &tb, B, N, K, ldb, batch, strideB, BLOCK_K, (uint32_t)block_n);
  else
    rc = b_mn ? make_tmap_2d(ctx, &tb, B, K, N, ldb, 64, BLOCK_K) : make_tmap_2d(ctx, &tb, B, N, K, ldb, BLOCK_K, (uint32_t)block_n);
  if (rc) return rc;
  CUtensorMap tc;
  memset(&tc, 0, sizeof(tc));
  ctx->last_gemm_kernel = "wgmma_batched";
  // products with biases of their own get the kernels that find each product's bias (batch_bias)
  const bool per_batch_bias = p.bias && p.bias_batch_stride && !reduce;
#define NK_TCB(BN, AM, BM_)                                                                                      \
  (per_batch_bias ? (c_dtype == NK_BF16 ? launch_cfg<BN, AM, BM_, __nv_bfloat16, true, true>(ctx, ta, tb, tc, p) \
                                        : launch_cfg<BN, AM, BM_, float, true, true>(ctx, ta, tb, tc, p))        \
                  : (c_dtype == NK_BF16 ? launch_cfg<BN, AM, BM_, __nv_bfloat16, true>(ctx, ta, tb, tc, p)       \
                                        : launch_cfg<BN, AM, BM_, float, true>(ctx, ta, tb, tc, p)))
#define NK_TCB_BN(AM, BM_) (block_n == 256 ? NK_TCB(256, AM, BM_) : block_n == 128 ? NK_TCB(128, AM, BM_) : NK_TCB(64, AM, BM_))
  if (!a_mn && !b_mn) return NK_TCB_BN(false, false);
  if (!a_mn && b_mn) return NK_TCB_BN(false, true);
  if (a_mn && b_mn) return NK_TCB_BN(true, true);
  return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "batched gemm: the TT form is not instantiated");
#undef NK_TCB_BN
#undef NK_TCB
}

// The engine behind the im2col convolution path (nk_conv_gemm.cu): beta 0, row-indexed bias shared by the batches.
// Returns NK_ERR_UNSUPPORTED (last_error untouched) when the operands are not TMA-addressable.
int nk_gemm_wgmma_batched(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                            int64_t lda, int64_t strideA, const void* B, int64_t ldb, int64_t strideB, void* C, int64_t ldc,
                            int64_t strideC, int64_t batch, int c_dtype, const void* row_bias, int bias_dtype, int relu,
                            int reduce) {
  return gemm_wgmma_batched(ctx, transA, transB, M, N, K, alpha, A, lda, strideA, B, ldb, strideB, 0.f, C, ldc, strideC, batch,
                            c_dtype, row_bias, bias_dtype, 1, 0, relu, reduce);
}

// f32 products go to the tf32 engine (nk_gemm_tf32.cu) in a non-IEEE f32 mode unless the SIMT engine is forced; the
// data-parallel reduce-scatter epilogue (ctx->rs_world) exists on the bf16 engine only
static bool f32_on_tensor_cores(const nk_ctx* ctx, int ab_dtype, int64_t K) {
  return ab_dtype == NK_F32 && ctx->f32_gemm != NK_F32_GEMM_IEEE && ctx->gemm_engine != NK_GEMM_SIMT && K > 0 &&
         ctx->rs_world == 0;
}

extern "C" {

int nk_gemm_bias_act(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha,
                     const void* A, int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc,
                     int ab_dtype, int c_dtype, const void* bias, int bias_dtype, int relu) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(ab_dtype) && nk_dtype_ok(c_dtype), "nk_gemm: bad dtype");
  NK_REQUIRE(ctx, M >= 0 && N >= 0 && K >= 0, "nk_gemm: negative dimension");
  if (M == 0 || N == 0) return NK_OK;
  NK_REQUIRE(ctx, C != nullptr && (K == 0 || (A && B)), "nk_gemm: NULL pointer");
  NK_REQUIRE(ctx, lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N,
             "nk_gemm: leading dimension too small (lda=%lld ldb=%lld ldc=%lld for M=%lld N=%lld K=%lld tA=%d tB=%d)",
             (long long)lda, (long long)ldb, (long long)ldc, (long long)M, (long long)N, (long long)K, transA, transB);
  NK_REQUIRE(ctx, !bias || nk_dtype_ok(bias_dtype), "nk_gemm: bad bias dtype");
  // f32 operands in TF32 / 3xTF32 mode: every shape goes to the tf32 engine (it packs whatever TMA cannot read)
  if (f32_on_tensor_cores(ctx, ab_dtype, K))
    return nk_gemm_tf32(ctx, transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, c_dtype, bias, bias_dtype, relu);
  const bool want_tc = ab_dtype == NK_BF16 && ctx->gemm_engine != NK_GEMM_SIMT && K > 0;
  if (want_tc) {
    int rc = nk_gemm_wgmma(ctx, transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, c_dtype, bias,
                             bias_dtype, relu, nullptr, nullptr);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
    if (ctx->gemm_engine == NK_GEMM_TC)
      return nk_set_error(ctx, NK_ERR_UNSUPPORTED,
                          "nk_gemm: tensor-core engine forced but operands are not TMA-addressable "
                          "(16-byte aligned base, leading dimension multiple of 8 elements)");
  } else if (ctx->gemm_engine == NK_GEMM_TC) {
    return nk_set_error(ctx, NK_ERR_UNSUPPORTED, "nk_gemm: tensor-core engine forced but operands are not bf16");
  }
  return nk_gemm_simt(ctx, transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ab_dtype, c_dtype, bias,
                      bias_dtype, relu);
}

int nk_gemm_strided_batched(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                            int64_t lda, int64_t strideA, const void* B, int64_t ldb, int64_t strideB, float beta, void* C,
                            int64_t ldc, int64_t strideC, int64_t batch, int ab_dtype, int c_dtype, const void* bias,
                            int64_t bias_stride, int bias_dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(ab_dtype) && nk_dtype_ok(c_dtype), "nk_gemm_strided_batched: bad dtype");
  NK_REQUIRE(ctx, M >= 0 && N >= 0 && K >= 0 && batch >= 0, "nk_gemm_strided_batched: negative dimension");
  NK_REQUIRE(ctx, !bias || nk_dtype_ok(bias_dtype), "nk_gemm_strided_batched: bad bias dtype");
  if (M == 0 || N == 0 || batch == 0) return NK_OK;
  // one launch of the batched wgmma kernel (TMA needs non-negative operand strides); its drain epilogue decides on 16-byte
  // stores from the first product's C, so every product's C must sit on a 16-byte boundary like the first one's
  const size_t cs = nk_dtype_size(c_dtype), bs = bias ? nk_dtype_size(bias_dtype) : 0;
  const bool tc = ab_dtype == NK_BF16 && ctx->gemm_engine != NK_GEMM_SIMT && K > 0 && !(transA && transB) &&
                  strideA >= 0 && strideB >= 0 && strideC >= 0 && bias_stride >= 0 && (strideC * int64_t(cs)) % 16 == 0 &&
                  (!bias || !bias_stride || batch == 1 || strideC > 0) &&
                  lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N;
  if (tc) {
    NK_REQUIRE(ctx, A && B && C, "nk_gemm_strided_batched: NULL pointer");
    const int rc = gemm_wgmma_batched(ctx, transA, transB, M, N, K, alpha, A, lda, strideA, B, ldb, strideB, beta, C, ldc,
                                      strideC, batch, c_dtype, bias, bias_dtype, 0, bias_stride, 0, 0);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  // everything else: one GEMM per product (which checks the arguments)
  const size_t as = nk_dtype_size(ab_dtype);
  for (int64_t b = 0; b < batch; ++b) {
    const int rc = nk_gemm_bias_act(
        ctx, transA, transB, M, N, K, alpha, A ? static_cast<const char*>(A) + b * strideA * int64_t(as) : nullptr, lda,
        B ? static_cast<const char*>(B) + b * strideB * int64_t(as) : nullptr, ldb, beta,
        C ? static_cast<char*>(C) + b * strideC * int64_t(cs) : nullptr, ldc, ab_dtype, c_dtype,
        bias ? static_cast<const char*>(bias) + b * bias_stride * int64_t(bs) : nullptr, bias_dtype, 0);
    if (rc) return rc;
  }
  return NK_OK;
}

int nk_gemm_relu_bwd_colsum(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                            const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype,
                            const void* relu_operand, float* colsum) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(ab_dtype) && nk_dtype_ok(c_dtype), "nk_gemm_relu_bwd: bad dtype");
  NK_REQUIRE(ctx, M >= 0 && N >= 0 && K > 0, "nk_gemm_relu_bwd: bad dimension");
  if (M == 0 || N == 0) return NK_OK;
  NK_REQUIRE(ctx, A && B && C && relu_operand, "nk_gemm_relu_bwd: NULL pointer");
  NK_REQUIRE(ctx, lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N, "nk_gemm_relu_bwd: leading dimension too small");
  NK_REQUIRE(ctx, !colsum || beta == 0.f, "nk_gemm_relu_bwd_colsum: the column sums are those of the product (beta must be 0)");
  if (ab_dtype == NK_BF16 && ctx->gemm_engine != NK_GEMM_SIMT) {
    int rc = nk_gemm_wgmma(ctx, transA, transB, M, N, K, 1.f, A, lda, B, ldb, beta, C, ldc, c_dtype, nullptr, NK_F32, 0,
                             relu_operand, colsum);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  // the skinny NN shape (K <= 16: the layer above is 10 wide) masks (and sums) in its own epilogue
  if (!transA && !transB) {
    int rc = nk_gemm_simt_small_k_masked(ctx, M, N, K, A, lda, B, ldb, beta, C, ldc, ab_dtype, c_dtype, relu_operand, colsum);
    if (rc != NK_ERR_UNSUPPORTED) return rc;
  }
  if (colsum) return NK_ERR_UNSUPPORTED;   // nothing done: the caller sums the columns itself after the plain call
  // operands the tensor-core engine cannot take: the product into a temporary, then the ordinary ReLU backward.  The
  // product of f32 operands in TF32 / 3xTF32 mode runs on the tf32 engine (the skinny K <= 16 kernel above stays on the
  // CUDA cores in every mode: it masks and sums in its own epilogue)
  void* tmp = nullptr;
  int rc = nk_alloc_uninit(ctx, size_t(M) * size_t(N) * nk_dtype_size(c_dtype), &tmp);
  if (rc) return rc;
  if (f32_on_tensor_cores(ctx, ab_dtype, K))
    rc = nk_gemm_tf32(ctx, transA, transB, M, N, K, 1.f, A, lda, B, ldb, 0.f, tmp, N, c_dtype, nullptr, NK_F32, 0);
  else
    rc = nk_gemm_simt(ctx, transA, transB, M, N, K, 1.f, A, lda, B, ldb, 0.f, tmp, N, ab_dtype, c_dtype, nullptr, NK_F32, 0);
  if (rc == NK_OK) {
    if (ldc == N) {
      rc = nk_relu_bwd(ctx, C, relu_operand, tmp, size_t(M) * size_t(N), c_dtype, beta);
    } else {
      rc = nk_set_error(ctx, NK_ERR_UNSUPPORTED, "nk_gemm_relu_bwd: strided output needs the tensor-core engine");
    }
  }
  nk_free(ctx, tmp);
  return rc;
}

int nk_gemm_relu_bwd(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, const void* A, int64_t lda,
                     const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype,
                     const void* relu_operand) {
  return nk_gemm_relu_bwd_colsum(ctx, transA, transB, M, N, K, A, lda, B, ldb, beta, C, ldc, ab_dtype, c_dtype, relu_operand,
                                 nullptr);
}

int nk_gemm(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
            int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int ab_dtype, int c_dtype) {
  return nk_gemm_bias_act(ctx, transA, transB, M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ab_dtype, c_dtype,
                          nullptr, NK_F32, 0);
}

}  // extern "C"
