// Geometry, padding map and column-gradient scatter shared by the two im2col convolution engines: bf16 (nk_conv_gemm.cu)
// and TF32 / 3xTF32 (nk_conv_tf32.cu).  x is (N, Cin, s0, s1, s2) with leading sample dims of extent 1 when there are
// fewer than three (the 2-D convolution is the case nsp = 2 with no padding); k = (c, i0, i1, i2) indexes the reduction
// of the forward product and l the output position in row-major order.
#pragma once
#include "nk_internal.cuh"

// the 1-D / 3-D layer: sample dims padded to three with leading extents of 1 (kernel 1, stride 1, dilation 1, pad 0)
struct CgNdDims {
  int64_t n, cin, cout, K, Kp, L, Lp;
  int64_t in[3], k[3], s[3], d[3], pad[3], out[3];
  int mode;        // nk_pad_mode
  float value;     // fill of the constant mode
};

// the convolution of the input padded by `pad` (mode / value as nk_padnd_fwd): output extents, K = Cin * prod(k),
// L = prod(out); Kp = Lp = 0 (each engine sets the row pitches it needs)
inline void conv_nd_geometry(CgNdDims& d, int nsp, int64_t n, int64_t cin, const int64_t* in_sp, int64_t cout,
                             const int64_t* k, const int64_t* s, const int64_t* dil, const int64_t* pad, int mode,
                             float value) {
  d = CgNdDims{};
  d.n = n, d.cin = cin, d.cout = cout, d.mode = mode, d.value = value;
  d.K = cin, d.L = 1;
  for (int a = 0; a < 3; ++a) d.in[a] = d.k[a] = d.s[a] = d.d[a] = d.out[a] = 1, d.pad[a] = 0;
  for (int a = 0; a < nsp; ++a) {
    const int j = 3 - nsp + a;
    d.in[j] = in_sp[a], d.k[j] = k[a], d.s[j] = s[a], d.d[j] = dil[a], d.pad[j] = pad[a];
    d.out[j] = (in_sp[a] + 2 * pad[a] - dil[a] * (k[a] - 1) - 1) / s[a] + 1;
    d.K *= k[a];
    d.L *= d.out[j];
  }
}

// source index of padded coordinate u along an axis of length len padded by p on both sides, or -1 for the fill value:
// the map of nk_padnd_fwd (nk_pointwise.cu pad_src; reflective/mod.rs:22-31, replicative/mod.rs:22-31)
__device__ __forceinline__ int pad_src_index(int u, int len, int p, int mode) {
  if (u >= p && u < len + p) return u - p;
  if (mode == NK_PAD_REFLECTIVE) return (u < p ? 2 * p - u : 2 * (len + p - 1) - u) - p;
  if (mode == NK_PAD_REPLICATIVE) return u < p ? 0 : len - 1;
  return -1;
}

// dx[n,c,u] = beta*dx + sum over the taps i and output positions p with p*s + i*d = u + pad (per axis) of
// dcolsT[ns][(c,i)][p] (rows Lp apart): only the interior positions of the padded input, whatever the mode; one thread
// per dx element (256 per block), the taps summed in f32 and rounded once to dx's type
template <typename T>
__global__ void __launch_bounds__(256) col2im_nd_kernel(T* __restrict__ dx, const float* __restrict__ dcols, CgNdDims d,
                                                        int64_t n0, int64_t nn, float beta) {
  const int in0 = int(d.in[0]), in1 = int(d.in[1]), in2 = int(d.in[2]);
  const int k0 = int(d.k[0]), k1 = int(d.k[1]), k2 = int(d.k[2]);
  const int o0 = int(d.out[0]), o1 = int(d.out[1]), o2 = int(d.out[2]);
  const int s0 = int(d.s[0]), s1 = int(d.s[1]), s2 = int(d.s[2]), d0 = int(d.d[0]), d1 = int(d.d[1]), d2 = int(d.d[2]);
  const int cin = int(d.cin), ksz = k0 * k1 * k2;
  const uint32_t isz = uint32_t(in0) * uint32_t(in1) * uint32_t(in2);
  const int64_t total = nn * d.cin * int64_t(isz);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const uint32_t pl = uint32_t(idx / isz);            // (ns, c)
    const uint32_t uv = uint32_t(idx - int64_t(pl) * isz);
    const int U2 = int(uv % uint32_t(in2)) + int(d.pad[2]);
    const int t = int(uv / uint32_t(in2));
    const int U1 = t % in1 + int(d.pad[1]), U0 = t / in1 + int(d.pad[0]);
    const uint32_t ns = pl / uint32_t(cin), c = pl - ns * uint32_t(cin);
    const float* dc = dcols + (int64_t(ns) * d.K + int64_t(c) * ksz) * d.Lp;
    float acc = 0.f;
    for (int i0 = 0; i0 < k0; ++i0) {
      const int pu0 = U0 - i0 * d0;
      if (pu0 < 0) break;
      const int q0 = pu0 / s0;
      if (q0 * s0 != pu0 || q0 >= o0) continue;
      for (int i1 = 0; i1 < k1; ++i1) {
        const int pu1 = U1 - i1 * d1;
        if (pu1 < 0) break;
        const int q1 = pu1 / s1;
        if (q1 * s1 != pu1 || q1 >= o1) continue;
        for (int i2 = 0; i2 < k2; ++i2) {
          const int pu2 = U2 - i2 * d2;
          if (pu2 < 0) break;
          const int q2 = pu2 / s2;
          if (q2 * s2 != pu2 || q2 >= o2) continue;
          acc += dc[int64_t((i0 * k1 + i1) * k2 + i2) * d.Lp + (int64_t(q0) * o1 + q1) * o2 + q2];
        }
      }
    }
    T* o = dx + n0 * d.cin * int64_t(isz) + idx;
    if (beta != 0.f) acc += beta * nk_to_f32<T>(*o);
    *o = nk_from_f32<T>(acc);
  }
}
