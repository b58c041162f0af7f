// The f32 tensor-core engine's internal interface (nk_gemm_tf32.cu), shared by the TF32 GEMM and the TF32 convolution
// engine (nk_conv_tf32.cu): the rounding of an operand element and the K-major packed operand layout, the pack kernel,
// and the GEMM entry that takes operands already packed.
#pragma once
#include "nk_internal.cuh"

// cvt.rna.tf32.f32: to nearest on the 10-bit mantissa, ties away from zero
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Writes operand element x to its place d in a packed row.  segments = 1 (TF32): d[0] = tf32(x).  segments = 3
// (3xTF32): hi = tf32(x), lo = tf32(x - hi); segment s (seg_len elements apart along the row) gets lo when s == lo_seg,
// else hi -- A' = [hi | hi | lo] (lo_seg 2) against B' = [hi | lo | hi] (lo_seg 1) sums hi.hi + hi.lo + lo.hi.
__device__ __forceinline__ void tf32_put(float* d, float x, int segments, int lo_seg, int64_t seg_len) {
  const float hi = tf32_rna(x);
  if (segments == 1) {
    d[0] = hi;
  } else {
    const float lo = tf32_rna(__fsub_rn(x, hi));
    for (int s = 0; s < segments; ++s) d[s * seg_len] = s == lo_seg ? lo : hi;
  }
}

// op(X) (R x K per batch entry; mn: stored (K, R), element (r, k) at src[k * ld + r], else at src[r * ld + k]) -> dst,
// K-major with leading dimension ldp, through tf32_put.  Batch entry b reads src + b * src_bstride and writes
// dst + b * dst_bstride; segments are seg_len elements apart (K for a plain operand).
int nk_tf32_pack(nk_ctx* ctx, const float* src, int64_t ld, bool mn, int64_t R, int64_t K, float* dst, int64_t ldp,
                 int segments, int lo_seg, int64_t batch = 1, int64_t src_bstride = 0, int64_t dst_bstride = 0,
                 int64_t seg_len = -1);

// C[b] (M x N) = alpha * A[b] . B[b]^T + beta * C[b] (+ bias, ReLU) for b < batch, with A (rows x kp) and B (rows x kp)
// packed K-major by the caller (tf32_put's layout).  Batch entry b reads the rows from b * a_bstride (b_bstride) and the
// reduction columns [b * k_bstride, b * k_bstride + k_len) of its operands -- rows and columns past the end of an operand
// read as zeros -- and writes C + b * c_bstride.  The bias is per column, or per row with row_bias.
struct NkTf32Gemm {
  bool x3 = false;   // 3xTF32: every k-block's product summed into the tile with IEEE adds
  int64_t M = 0, N = 0, batch = 1;
  const float* A = nullptr;
  int64_t lda = 0, a_rows = 0, a_bstride = 0;
  const float* B = nullptr;
  int64_t ldb = 0, b_rows = 0, b_bstride = 0;
  int64_t kp = 0, k_len = 0, k_bstride = 0;
  void* C = nullptr;
  int64_t ldc = 0, c_bstride = 0;
  int c_dtype = NK_F32;
  float alpha = 1.f, beta = 0.f;
  const void* bias = nullptr;
  int bias_dtype = NK_F32, row_bias = 0, relu = 0;
};
// the tile width nk_gemm_tf32_packed uses for N columns: the widest that does not leave most of a tile empty (3xTF32:
// at most 128)
inline int nk_tf32_block_n(int64_t N, bool x3) { return N <= 64 ? 64 : (N <= 128 || x3) ? 128 : 256; }
int nk_gemm_tf32_packed(nk_ctx* ctx, const NkTf32Gemm& g);
