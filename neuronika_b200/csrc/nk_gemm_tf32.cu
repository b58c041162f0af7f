// f32 products on the tensor cores (sm_90a): C = alpha * op(A).op(B) + beta*C (+bias[n], ReLU) with f32 operands, in the
// context's TF32 or 3xTF32 mode (nk_gemm_f32_config).  The bf16 engine (nk_gemm_tc.cu) is not involved.
//
// wgmma takes tf32 operands only K-major in shared memory (the transpose immediates the bf16 engine uses for MN-major
// operands do not exist for tf32), so every operand goes through one pass of the pack kernel first:
//   tf32_pack : op(X) (R x K, K- or MN-major as stored) -> a K-major temporary (R rows, leading dimension rounded up to
//               4 elements = TMA's 16 bytes), every element rounded with cvt.rna.tf32.f32 (to nearest, ties away from
//               zero).  In 3xTF32 mode each element x becomes hi = tf32(x) and lo = tf32(x - hi), written along K as
//               A' = [A_hi | A_hi | A_lo] and B' = [B_hi | B_lo | B_hi]: the product over K' = 3K is
//               A_hi.B_hi + A_hi.B_lo + A_lo.B_hi, an ordinary TF32 GEMM.
// Packing every operand, K-major ones included, means every element reaches the tensor cores rounded the same way, so
// the four forms NN / NT / TN / TT of one product give the same bits.  The temporaries are stream-ordered
// (nk_alloc_uninit / nk_free: a captured step takes them from its arena): (M + N) x ceil4(K) floats in TF32 mode,
// (M + N) x ceil4(3K) in 3xTF32 mode.
//
// tf32_gemm (persistent over 128 x BLOCK_N output tiles, one CTA per SM, three warpgroups, as the bf16 engine):
//   warpgroup 0    : TMA producer (one thread) -- 128B-swizzled boxes of 32 f32 (one swizzle row) per k-block into a
//                    kStages smem ring
//   warpgroups 1-2 : consumers, 64 rows each -- wgmma m64nBLOCK_Nk8.f32.tf32.tf32 with the accumulator in registers, one
//                    k-block's group kept in flight; then a register-to-global drain applying nk_gemm_simt.cu's
//                    store_out epilogue (alpha, beta, column bias, ReLU) in its order.
// 3xTF32 (kSplitAcc): the tensor cores' f32 accumulation does not round to nearest, and its error grows with the number
// of k-steps summed into one accumulator (measured on H100: a 256 x 256 x 2048 product 98x further from float64 than
// the CUDA-core engine, only 12x closer than one TF32 pass).  So each k-block's product goes into a fresh partial
// accumulator, which the warpgroup adds to the tile's accumulator with ordinary f32 adds once its group is done: the
// tensor cores never sum more than 32 products.  Two accumulators per thread limit 3xTF32 tiles to 128 columns.
// No split-K: every output element is one accumulator's sum in a fixed order, so repeated calls give the same bits.
// nk_gemm_tf32_packed (nk_tf32.cuh) is the same kernel on operands the caller packed: a batch index is the slowest index
// of the tile order (A shared or batched, row / reduction-column / C offsets per batch entry) and the bias may be per
// row; the f32 convolution engine (nk_conv_tf32.cu) runs its three products on it.
#include "nk_tf32.cuh"
#include "nk_ptx.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;   // 32 f32 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 8;
constexpr int kNumThreads = 384;
constexpr uint32_t kSmemLimit = 232448;  // 227 KB
constexpr int kGroupM = 16;              // tile order as the bf16 engine: kGroupM m-blocks per n-block step

struct Tf32Params {
  int64_t M, N, ldc;
  void* C;
  const void* bias;
  float alpha, beta;
  int bias_bf16, relu, row_bias;
  int num_m_blocks, num_n_blocks, num_k_blocks;
  int k_blocks_total;   // of the packed operands: a batch entry's k-blocks stop there
  // batch entry b (the slowest index of the tile order): operand rows from b * a_bstride / b * b_bstride, reduction
  // columns from b * k_bstride, output at C + b * c_bstride
  int batch, a_bstride, b_bstride, k_bstride;
  int64_t c_bstride;
};

template <int BLOCK_N>
struct Tf32Cfg {
  static constexpr uint32_t A_BYTES = BLOCK_M * BLOCK_K * 4;  // 16 KB
  static constexpr uint32_t B_BYTES = BLOCK_N * BLOCK_K * 4;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int kStagesMax = (kSmemLimit - 2048) / STAGE_BYTES;
  static constexpr int kStages = kStagesMax > 8 ? 8 : kStagesMax;
  static constexpr uint32_t SMEM_BYTES = kStages * STAGE_BYTES + 2048;  // + alignment slack + barriers
};

__device__ __forceinline__ void tile_coords(const Tf32Params& p, int tile, int& b, int& m_blk, int& n_blk) {
  const int per_batch = p.num_m_blocks * p.num_n_blocks;
  b = tile / per_batch;
  tile -= b * per_batch;
  const int group_size = kGroupM * p.num_n_blocks;
  const int group = tile / group_size, in_group = tile - group * group_size;
  const int first_m = group * kGroupM;
  const int gm = min(p.num_m_blocks - first_m, kGroupM);
  m_blk = first_m + in_group % gm;
  n_blk = in_group / gm;
}

// One 32 (rows) x 32 (k) tile of op(X) per block of 32 x 8 threads, through shared memory so that both the read of an
// MN-major operand (along rows) and the write (along k) are coalesced; every element written by tf32_put.  grid.y
// steps through the k tiles and grid.z through the batch entries, so K and the batch have no grid limit.
template <bool MN>
__global__ void __launch_bounds__(256) tf32_pack_kernel(const float* __restrict__ src, int64_t ld, int64_t R, int64_t K,
                                                       float* __restrict__ dst, int64_t ldp, int segments, int lo_seg,
                                                       int64_t batch, int64_t src_bstride, int64_t dst_bstride,
                                                       int64_t seg_len) {
  __shared__ float tile[32][33];
  const int64_t r0 = int64_t(blockIdx.x) * 32, k_tiles = (K + 31) / 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  bool first = true;
  for (int64_t b = blockIdx.z; b < batch; b += gridDim.z) {
    const float* sb = src + b * src_bstride;
    for (int64_t kt = blockIdx.y; kt < k_tiles; kt += gridDim.y) {
      const int64_t k0 = kt * 32;
      if (!first) __syncthreads();   // the previous tile has been read
      first = false;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int yy = ty + 8 * i;
        if (MN) {   // element (r, k) at src[k * ld + r]: lanes along r
          const int64_t r = r0 + tx, k = k0 + yy;
          if (r < R && k < K) tile[tx][yy] = sb[k * ld + r];
        } else {    // element (r, k) at src[r * ld + k]: lanes along k
          const int64_t r = r0 + yy, k = k0 + tx;
          if (r < R && k < K) tile[yy][tx] = sb[r * ld + k];
        }
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int yy = ty + 8 * i;
        const int64_t r = r0 + yy, k = k0 + tx;
        if (r < R && k < K) tf32_put(dst + b * dst_bstride + r * ldp + k, tile[yy][tx], segments, lo_seg, seg_len);
      }
    }
  }
}

template <typename TC>
__device__ __forceinline__ void store_pair(const Tf32Params& p, TC* cb, int64_t row, int64_t col, float a0, float a1,
                                           bool pair_ok) {
  if (row >= p.M || col >= p.N) return;
  TC* c = cb + row * p.ldc + col;
  float v[2] = {a0, a1};
  const int n = col + 1 < p.N ? 2 : 1;
  // nk_gemm_simt.cu store_out: alpha, beta.C, bias, ReLU, rounding to C's type
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (e >= n) break;
    float x = p.alpha * v[e];
    if (p.beta != 0.f) x += p.beta * nk_to_f32<TC>(c[e]);
    if (p.bias) {
      const int64_t bi = p.row_bias ? row : col + e;
      x += p.bias_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(p.bias)[bi])
                       : static_cast<const float*>(p.bias)[bi];
    }
    if (p.relu) x = x > 0.f ? x : 0.f;
    v[e] = x;
  }
  if (n == 2 && pair_ok) {
    if constexpr (sizeof(TC) == 4) {
      *reinterpret_cast<float2*>(c) = make_float2(v[0], v[1]);
    } else {
      *reinterpret_cast<__nv_bfloat162*>(c) = __floats2bfloat162_rn(v[0], v[1]);
    }
  } else {
    for (int e = 0; e < n; ++e) c[e] = nk_from_f32<TC>(v[e]);
  }
}

template <int BLOCK_N, typename TC, bool kSplitAcc>
__global__ void __launch_bounds__(kNumThreads, 1)
tf32_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Tf32Params p) {
  using C_ = Tf32Cfg<BLOCK_N>;
  constexpr int kStages = C_::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms: 1024 B aligned
  const uint32_t smem_a0 = smem_base;
  const uint32_t smem_b0 = smem_base + kStages * C_::A_BYTES;
  const uint32_t bar_base = smem_base + kStages * C_::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  const int num_tiles = p.batch * p.num_m_blocks * p.num_n_blocks;

  if (wg == 0) {
    // ===================================================== TMA producer
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int b, m_blk, n_blk;
        tile_coords(p, tile, b, m_blk, n_blk);
        const int a_row = b * p.a_bstride + m_blk * BLOCK_M, b_row = b * p.b_bstride + n_blk * BLOCK_N;
        const int k0 = b * p.k_bstride;
        const int nkb = min(p.num_k_blocks, p.k_blocks_total - k0 / BLOCK_K);
        for (int kb = 0; kb < nkb; ++kb) {
          ptx::mbar_wait_spin(empty_bar(stage), phase ^ 1u);
          ptx::mbar_expect_tx(full_bar(stage), C_::STAGE_BYTES);
          ptx::tma_load_2d(smem_a0 + stage * C_::A_BYTES, &tmap_a, full_bar(stage), k0 + kb * BLOCK_K, a_row);
          ptx::tma_load_2d(smem_b0 + stage * C_::B_BYTES, &tmap_b, full_bar(stage), k0 + kb * BLOCK_K, b_row);
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
  const int warp = t >> 5, lane = t & 31;
  const uint32_t a_off = uint32_t(cw) * (64 * BLOCK_K * 4);   // 64 K-major rows of 128 B
  float acc[BLOCK_N / 2];
  float part[kSplitAcc ? BLOCK_N / 2 : 1];   // kSplitAcc: the current k-block's product
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int b, m_blk, n_blk;
    tile_coords(p, tile, b, m_blk, n_blk);
    int prev_stage = 0;
    const int nkb = min(p.num_k_blocks, p.k_blocks_total - b * p.k_bstride / BLOCK_K);
    for (int kb = 0; kb < nkb; ++kb) {
      ptx::mbar_wait_spin(full_bar(stage), phase);
      // K-major SW128: 8-row groups 1024 B apart (SBO), +32 B per k8 step inside the swizzle row
      const uint64_t adesc = ptx::make_smem_desc_sw128(smem_a0 + stage * C_::A_BYTES + a_off, 16, 1024);
      const uint64_t bdesc = ptx::make_smem_desc_sw128(smem_b0 + stage * C_::B_BYTES, 16, 1024);
      if constexpr (kSplitAcc) {
        ptx::fence_regs(part);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
          ptx::WgmmaTf32<BLOCK_N>::mma(part, adesc + uint64_t((k * WGMMA_K * 4) >> 4),
                                       bdesc + uint64_t((k * WGMMA_K * 4) >> 4), k != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(part);
        if (t == 0) ptx::mbar_arrive(empty_bar(stage));   // this warpgroup is done reading the slot
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = kb == 0 ? part[i] : __fadd_rn(acc[i], part[i]);
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1u;
        }
        continue;
      }
      ptx::fence_regs(acc);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
        ptx::WgmmaTf32<BLOCK_N>::mma(acc, adesc + uint64_t((k * WGMMA_K * 4) >> 4), bdesc + uint64_t((k * WGMMA_K * 4) >> 4),
                                     (kb | k) != 0 ? 1u : 0u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();   // k-block kb - 1's group is done; kb's stays in flight
      ptx::fence_regs(acc);
      if (kb > 0 && t == 0) ptx::mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1u;
      }
    }
    if constexpr (!kSplitAcc) {
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (t == 0) ptx::mbar_arrive(empty_bar(prev_stage));
    }

    // ---- drain: thread holds rows r, r + 8 (r = 16 warp + lane / 4) and columns 8j + 2 (lane % 4) + {0, 1}
    const int64_t row = int64_t(m_blk) * BLOCK_M + cw * 64 + warp * 16 + (lane >> 2);
    const int64_t col = int64_t(n_blk) * BLOCK_N + 2 * (lane & 3);
    TC* cb = static_cast<TC*>(p.C) + b * p.c_bstride;
    const bool pair_ok = (p.ldc % 2 == 0) && (reinterpret_cast<uintptr_t>(cb) % (2 * sizeof(TC)) == 0);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      store_pair<TC>(p, cb, row, col + 8 * j, acc[4 * j], acc[4 * j + 1], pair_ok);
      store_pair<TC>(p, cb, row + 8, col + 8 * j, acc[4 * j + 2], acc[4 * j + 3], pair_ok);
    }
  }
}

template <int BLOCK_N, typename TC, bool kSplitAcc>
int launch_tf32(nk_ctx* ctx, const CUtensorMap& ta, const CUtensorMap& tb, Tf32Params& p) {
  using C_ = Tf32Cfg<BLOCK_N>;
  auto kern = tf32_gemm_kernel<BLOCK_N, TC, kSplitAcc>;
  static bool attr_done[64] = {};  // per template instantiation and device (the attribute is per device)
  if (!attr_done[ctx->device & 63]) {
    static_assert(C_::SMEM_BYTES <= kSmemLimit, "shared memory budget");
    NK_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C_::SMEM_BYTES));
    attr_done[ctx->device & 63] = true;
  }
  p.num_n_blocks = int((p.N + BLOCK_N - 1) / BLOCK_N);
  const int num_tiles = p.batch * p.num_m_blocks * p.num_n_blocks;
  const int waves = (num_tiles + ctx->sm_count - 1) / ctx->sm_count;
  const int grid = (num_tiles + waves - 1) / waves;
  kern<<<grid, kNumThreads, C_::SMEM_BYTES, ctx->stream>>>(ta, tb, p);
  NK_LAUNCHED(ctx, "tf32_gemm");
  return NK_OK;
}

}  // namespace

int nk_tf32_pack(nk_ctx* ctx, const float* src, int64_t ld, bool mn, int64_t R, int64_t K, float* dst, int64_t ldp,
                 int segments, int lo_seg, int64_t batch, int64_t src_bstride, int64_t dst_bstride, int64_t seg_len) {
  NK_REQUIRE(ctx, (R + 31) / 32 < (int64_t(1) << 31), "tf32 pack: operand too large (R=%lld K=%lld)", (long long)R,
             (long long)K);
  const int64_t k_tiles = (K + 31) / 32;
  const dim3 grid(unsigned((R + 31) / 32), unsigned(k_tiles < 65535 ? k_tiles : 65535), unsigned(batch < 65535 ? batch : 65535)),
      block(32, 8);
  if (seg_len < 0) seg_len = K;
  if (mn)
    tf32_pack_kernel<true><<<grid, block, 0, ctx->stream>>>(src, ld, R, K, dst, ldp, segments, lo_seg, batch, src_bstride,
                                                            dst_bstride, seg_len);
  else
    tf32_pack_kernel<false><<<grid, block, 0, ctx->stream>>>(src, ld, R, K, dst, ldp, segments, lo_seg, batch, src_bstride,
                                                             dst_bstride, seg_len);
  NK_LAUNCHED(ctx, "tf32_pack");
  return NK_OK;
}

int nk_gemm_tf32_packed(nk_ctx* ctx, const NkTf32Gemm& g) {
  const int block_n = nk_tf32_block_n(g.N, g.x3);
  const int64_t m_blocks = (g.M + BLOCK_M - 1) / BLOCK_M, n_blocks = (g.N + block_n - 1) / block_n;
  NK_REQUIRE(ctx, g.batch >= 1 && g.batch * m_blocks * n_blocks < (int64_t(1) << 31) && g.a_rows < (int64_t(1) << 31) &&
                  g.b_rows < (int64_t(1) << 31) && g.kp < (int64_t(1) << 31) &&
                  (g.batch - 1) * (g.a_bstride + g.b_bstride + g.k_bstride) < (int64_t(1) << 31),
             "tf32 gemm: shape too large (M=%lld N=%lld K=%lld batch=%lld)", (long long)g.M, (long long)g.N,
             (long long)g.kp, (long long)g.batch);
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(ctx, &ta, g.A, g.a_rows, g.kp, g.lda, BLOCK_K, BLOCK_M, NK_F32);
  if (!rc) rc = make_tmap_2d(ctx, &tb, g.B, g.b_rows, g.kp, g.ldb, BLOCK_K, uint32_t(block_n), NK_F32);
  if (rc) return rc;
  Tf32Params p;
  p.M = g.M, p.N = g.N, p.ldc = g.ldc, p.C = g.C, p.bias = g.bias, p.alpha = g.alpha, p.beta = g.beta;
  p.bias_bf16 = g.bias_dtype == NK_BF16, p.relu = g.relu, p.row_bias = g.row_bias;
  p.num_m_blocks = int(m_blocks);
  p.num_n_blocks = 0;
  p.num_k_blocks = int((g.k_len + BLOCK_K - 1) / BLOCK_K);
  p.k_blocks_total = int((g.kp + BLOCK_K - 1) / BLOCK_K);
  p.batch = int(g.batch), p.a_bstride = int(g.a_bstride), p.b_bstride = int(g.b_bstride), p.k_bstride = int(g.k_bstride);
  p.c_bstride = g.c_bstride;
  const bool cb = g.c_dtype == NK_BF16;
#define NK_TF32(BN, SPLIT) (cb ? launch_tf32<BN, __nv_bfloat16, SPLIT>(ctx, ta, tb, p) : launch_tf32<BN, float, SPLIT>(ctx, ta, tb, p))
  if (g.x3)
    rc = block_n == 128 ? NK_TF32(128, true) : NK_TF32(64, true);
  else
    rc = block_n == 256 ? NK_TF32(256, false) : block_n == 128 ? NK_TF32(128, false) : NK_TF32(64, false);
#undef NK_TF32
  return rc;
}

int nk_gemm_tf32(nk_ctx* ctx, int transA, int transB, int64_t M, int64_t N, int64_t K, float alpha, const void* A,
                 int64_t lda, const void* B, int64_t ldb, float beta, void* C, int64_t ldc, int c_dtype, const void* bias,
                 int bias_dtype, int relu) {
  const bool x3 = ctx->f32_gemm == NK_F32_GEMM_TF32X3;
  const int segments = x3 ? 3 : 1;
  const int64_t kp = K * segments;
  const int64_t ldp = (kp + 3) / 4 * 4;
  NK_REQUIRE(ctx, (M + 31) / 32 < (int64_t(1) << 31) && (N + 31) / 32 < (int64_t(1) << 31) && (K + 31) / 32 <= 65535 &&
                  (M + BLOCK_M - 1) / BLOCK_M * ((N + 63) / 64) < (int64_t(1) << 31),
             "nk_gemm (tf32): shape too large (M=%lld N=%lld K=%lld)", (long long)M, (long long)N, (long long)K);
  const int block_n = nk_tf32_block_n(N, x3);

  void* pa = nullptr;
  void* pb = nullptr;
  int rc = nk_alloc_uninit(ctx, size_t(M) * size_t(ldp) * 4, &pa);
  if (rc) return rc;
  rc = nk_alloc_uninit(ctx, size_t(N) * size_t(ldp) * 4, &pb);
  if (rc) {
    nk_free(ctx, pa);
    return rc;
  }
  // A' = [A_hi | A_hi | A_lo], B' = [B_hi | B_lo | B_hi]
  rc = nk_tf32_pack(ctx, static_cast<const float*>(A), lda, transA != 0, M, K, static_cast<float*>(pa), ldp, segments, 2);
  if (!rc) rc = nk_tf32_pack(ctx, static_cast<const float*>(B), ldb, transB == 0, N, K, static_cast<float*>(pb), ldp, segments, 1);
  if (!rc) {
    static const char* names[2][2][2][3] = {
        {{{"tf32_nn_128x256", "tf32_nn_128x128", "tf32_nn_128x64"}, {"tf32_nt_128x256", "tf32_nt_128x128", "tf32_nt_128x64"}},
         {{"tf32_tn_128x256", "tf32_tn_128x128", "tf32_tn_128x64"}, {"tf32_tt_128x256", "tf32_tt_128x128", "tf32_tt_128x64"}}},
        {{{"tf32x3_nn_128x256", "tf32x3_nn_128x128", "tf32x3_nn_128x64"},
          {"tf32x3_nt_128x256", "tf32x3_nt_128x128", "tf32x3_nt_128x64"}},
         {{"tf32x3_tn_128x256", "tf32x3_tn_128x128", "tf32x3_tn_128x64"},
          {"tf32x3_tt_128x256", "tf32x3_tt_128x128", "tf32x3_tt_128x64"}}}};
    ctx->last_gemm_kernel = names[x3][transA != 0][transB != 0][block_n == 256 ? 0 : block_n == 128 ? 1 : 2];
    NkTf32Gemm g;
    g.x3 = x3, g.M = M, g.N = N;
    g.A = static_cast<const float*>(pa), g.lda = ldp, g.a_rows = M;
    g.B = static_cast<const float*>(pb), g.ldb = ldp, g.b_rows = N;
    g.kp = kp, g.k_len = kp;
    g.C = C, g.ldc = ldc, g.c_dtype = c_dtype, g.alpha = alpha, g.beta = beta;
    g.bias = bias, g.bias_dtype = bias_dtype, g.relu = relu;
    rc = nk_gemm_tf32_packed(ctx, g);
  }
  nk_free(ctx, pa);
  nk_free(ctx, pb);
  return rc;
}
