// Recurrent cells and the `chunks` op (SURVEY.md 8-f rank 4):
//   LSTM / GRU gate maths    the pointwise half of neuronika-nn/src/lib.rs:510-540 (LSTMCell::forward, with the intended
//                            gate assignment i, f, o = sigmoid, g = tanh; SURVEY.md 8-c defect 7) and :607-624
//                            (GRUCell::forward = torch.nn.GRUCell), forward and backward, one kernel each
//   chunk                    chunk/mod.rs: block `index` of ndarray's exact_chunks, and its backward (dx[block] += g)
// The cell's GEMMs write the gate pre-activations in f32, so the activations never see a bf16-rounded input.  Every
// thread owns V consecutive hidden units of one row: columns j, H+j, 2H+j (, 3H+j) of that row.  16-byte vector accesses
// when H and the base pointers allow it, a scalar body otherwise; grid-stride with 64-bit indexing.  The activations are
// those of nk_pointwise.cu (1/(1+expf(-x)), tanhf), so the fused cell and the cell composed from primitives differ only
// by the composed graph's rounded intermediates.  Saturated or infinite pre-activations give 0 / 1 / +-1, never NaN.
// The backward recomputes the activations (and c') from the f32 gates instead of keeping them.
//   sequence steps           nk_lstm_seq_bwd_step / nk_gru_seq_bwd_step: the same gate gradients for one time step of the
//                            LSTM / GRU sequence node (nk_graph.cpp, RnnSeqBackward).  The gradient carried from step to
//                            step (dc, and the recurrent part of dh) stays in f32 whatever the element type and is updated
//                            in place, so a bf16 sequence rounds it once at the end instead of once per step.
//   two directions           nk_{lstm,gru}_bidir_{fwd,bwd}_step: one time step of both directions of a bidirectional
//                            layer in one launch (blockIdx.y = direction), each direction's operands a given distance apart.
// All of them share the per-unit gate maths below (lstm_fwd_unit, lstm_bwd_unit, gru_fwd_unit, gru_bwd_unit).
#include "nk_internal.cuh"

// a named namespace: the kernels keep the same symbol names from build to build (profiler traces, torch.profiler)
namespace nk_rnn {

constexpr int kThreads = 256;

static inline int rnn_blocks(nk_ctx* ctx, size_t work_items) {
  size_t b = (work_items + kThreads - 1) / kThreads;
  size_t cap = size_t(ctx->sm_count) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return int(b);
}
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// The gate maths of one hidden unit, shared by the cell, sequence-step and two-direction step kernels.
// LSTM forward: the new cell state cn and hidden state hn from the gate pre-activations and the previous cell state c.
__device__ __forceinline__ void lstm_fwd_unit(float gi, float gf, float gg, float go, float c, float& cn, float& hn) {
  cn = sigm(gf) * c + sigm(gi) * tanhf(gg);
  hn = sigm(go) * tanhf(cn);
}
// LSTM backward: the gate pre-activations are replaced by their gradients, given the hidden-state gradient dh and the
// cell-state gradient dc that reach this step; returns sigmoid(f)*dc_total, the part of the previous cell state's gradient
__device__ __forceinline__ float lstm_bwd_unit(float& gi, float& gf, float& gg, float& go, float c, float dh, float dc) {
  const float i = sigm(gi), f = sigm(gf), g = tanhf(gg), o = sigm(go);
  const float tc = tanhf(f * c + i * g);
  const float dct = dc + dh * o * (1.f - tc * tc);
  gi = dct * g * i * (1.f - i);
  gf = dct * c * f * (1.f - f);
  gg = dct * i * (1.f - g * g);
  go = dh * tc * o * (1.f - o);
  return f * dct;
}
// GRU forward: the new hidden state from both gate pre-activations and the previous hidden state h
__device__ __forceinline__ float gru_fwd_unit(float ir, float iz, float in, float hr, float hz, float hn, float h) {
  const float r = sigm(ir + hr), z = sigm(iz + hz);
  const float nn = tanhf(in + r * hn);
  return (h - nn) * z + nn;
}
// GRU backward: ir, iz, in become d(i_r) = d(h_r), d(i_z) = d(h_z), d(i_n) and hn becomes d(h_n); returns z*dh, the
// pointwise part of the previous hidden state's gradient
__device__ __forceinline__ float gru_bwd_unit(float& ir, float& iz, float& in, float hr, float hz, float& hn, float h,
                                              float dh) {
  const float r = sigm(ir + hr), z = sigm(iz + hz);
  const float nn = tanhf(in + r * hn);
  const float dpn = dh * (1.f - z) * (1.f - nn * nn);
  const float dpz = dh * (h - nn) * z * (1.f - z);
  const float dpr = dpn * hn * r * (1.f - r);
  ir = dpr;
  iz = dpz;
  in = dpn;
  hn = dpn * r;
  return z * dh;
}

// V elements of T at p (16 / 8 byte vector accesses when V * sizeof(T) allows it; the caller guarantees alignment)
template <typename T, int V>
__device__ __forceinline__ void ldv(float (&o)[V], const T* __restrict__ p) {
  constexpr int B = V * int(sizeof(T));
  if constexpr (B % 16 == 0) {
#pragma unroll
    for (int k = 0; k < B / 16; ++k) {
      uint4 r = reinterpret_cast<const uint4*>(p)[k];
      const T* e = reinterpret_cast<const T*>(&r);
#pragma unroll
      for (int i = 0; i < 16 / int(sizeof(T)); ++i) o[k * (16 / int(sizeof(T))) + i] = nk_to_f32<T>(e[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) o[i] = nk_to_f32<T>(p[i]);
  }
}
template <typename T, int V>
__device__ __forceinline__ void stv(T* __restrict__ p, const float (&v)[V]) {
  constexpr int B = V * int(sizeof(T));
  if constexpr (B % 16 == 0) {
#pragma unroll
    for (int k = 0; k < B / 16; ++k) {
      uint4 r;
      T* e = reinterpret_cast<T*>(&r);
#pragma unroll
      for (int i = 0; i < 16 / int(sizeof(T)); ++i) e[i] = nk_from_f32<T>(v[k * (16 / int(sizeof(T))) + i]);
      reinterpret_cast<uint4*>(p)[k] = r;
    }
  } else if constexpr (B == 8) {
    uint2 r;
    T* e = reinterpret_cast<T*>(&r);
#pragma unroll
    for (int i = 0; i < V; ++i) e[i] = nk_from_f32<T>(v[i]);
    *reinterpret_cast<uint2*>(p) = r;
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) p[i] = nk_from_f32<T>(v[i]);
  }
}

// ------------------------------------------------------------------------------------------------- LSTM
// gates (n, 4H) f32, chunks [i | f | g | o]
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) nk_lstm_cell_fwd_kernel(T* __restrict__ c_out, T* __restrict__ h_out,
                                                                    const float* __restrict__ gates,
                                                                    const T* __restrict__ c_prev, int64_t n, int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const float* g = gates + row * 4 * H + j;
    float gi[V], gf[V], gg[V], go[V], c[V], co[V], ho[V];
    ldv<float, V>(gi, g);
    ldv<float, V>(gf, g + H);
    ldv<float, V>(gg, g + 2 * H);
    ldv<float, V>(go, g + 3 * H);
    ldv<T, V>(c, c_prev + row * H + j);
#pragma unroll
    for (int k = 0; k < V; ++k) lstm_fwd_unit(gi[k], gf[k], gg[k], go[k], c[k], co[k], ho[k]);
    stv<T, V>(c_out + row * H + j, co);
    stv<T, V>(h_out + row * H + j, ho);
  }
}

// dgates (beta 0) and dc_prev = beta*dc_prev + f*dc_total, dc_total = dc_out + dh_out*o*(1 - tanh(c')^2).
// c' is recomputed in f32 from the gates and c_prev (read anyway for the forget-gate gradient).
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_lstm_cell_bwd_kernel(TG* __restrict__ dgates, T* __restrict__ dc_prev,
                                                                    float beta_dc, const float* __restrict__ gates,
                                                                    const T* __restrict__ c_prev,
                                                                    const T* __restrict__ dh_out,
                                                                    const T* __restrict__ dc_out, int64_t n, int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 4 * H + j, ss = row * H + j;
    float gi[V], gf[V], gg[V], go[V], c[V], dh[V], dc[V], dcp[V];
    ldv<float, V>(gi, gates + gs);
    ldv<float, V>(gf, gates + gs + H);
    ldv<float, V>(gg, gates + gs + 2 * H);
    ldv<float, V>(go, gates + gs + 3 * H);
    ldv<T, V>(c, c_prev + ss);
    if (dh_out) ldv<T, V>(dh, dh_out + ss);
    if (dc_out) ldv<T, V>(dc, dc_out + ss);
    if (dc_prev && beta_dc != 0.f) ldv<T, V>(dcp, dc_prev + ss);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      float r = lstm_bwd_unit(gi[k], gf[k], gg[k], go[k], c[k], dh_out ? dh[k] : 0.f, dc_out ? dc[k] : 0.f);
      if (dc_prev && beta_dc != 0.f) r += beta_dc * dcp[k];
      dcp[k] = r;
    }
    stv<TG, V>(dgates + gs, gi);
    stv<TG, V>(dgates + gs + H, gf);
    stv<TG, V>(dgates + gs + 2 * H, gg);
    stv<TG, V>(dgates + gs + 3 * H, go);
    if (dc_prev) stv<T, V>(dc_prev + ss, dcp);
  }
}

// One backward time step of the LSTM sequence node.  dh = dh_out (this step's slice of the output gradient, element type
// T) + dh_rec (f32, what came back through h.W_hh^T from step t+1); either may be NULL = zero.  dc is the running f32
// cell-state gradient: read as dc_out, overwritten with dc_prev = f*dc_total.
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_lstm_seq_bwd_step_kernel(TG* __restrict__ dgates, float* __restrict__ dc,
                                                                        const float* __restrict__ gates,
                                                                        const T* __restrict__ c_prev,
                                                                        const T* __restrict__ dh_out,
                                                                        const float* __restrict__ dh_rec, int64_t n,
                                                                        int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 4 * H + j, ss = row * H + j;
    float gi[V], gf[V], gg[V], go[V], c[V], dh[V], dr[V], dcr[V];
    ldv<float, V>(gi, gates + gs);
    ldv<float, V>(gf, gates + gs + H);
    ldv<float, V>(gg, gates + gs + 2 * H);
    ldv<float, V>(go, gates + gs + 3 * H);
    ldv<T, V>(c, c_prev + ss);
    ldv<float, V>(dcr, dc + ss);
    if (dh_out) ldv<T, V>(dh, dh_out + ss);
    if (dh_rec) ldv<float, V>(dr, dh_rec + ss);
#pragma unroll
    for (int k = 0; k < V; ++k)
      dcr[k] = lstm_bwd_unit(gi[k], gf[k], gg[k], go[k], c[k], (dh_out ? dh[k] : 0.f) + (dh_rec ? dr[k] : 0.f), dcr[k]);
    stv<TG, V>(dgates + gs, gi);
    stv<TG, V>(dgates + gs + H, gf);
    stv<TG, V>(dgates + gs + 2 * H, gg);
    stv<TG, V>(dgates + gs + 3 * H, go);
    stv<float, V>(dc + ss, dcr);
  }
}

// ------------------------------------------------------------------------------------------------- GRU
// igates = x.W_ih^T + b_ih, hgates = h.W_hh^T + b_hh, (n, 3H) f32 each, chunks [r | z | n]
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) nk_gru_cell_fwd_kernel(T* __restrict__ h_out, const float* __restrict__ igates,
                                                                   const float* __restrict__ hgates,
                                                                   const T* __restrict__ h_prev, int64_t n, int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 3 * H + j, ss = row * H + j;
    float ir[V], iz[V], in[V], hr[V], hz[V], hn[V], h[V], ho[V];
    ldv<float, V>(ir, igates + gs);
    ldv<float, V>(iz, igates + gs + H);
    ldv<float, V>(in, igates + gs + 2 * H);
    ldv<float, V>(hr, hgates + gs);
    ldv<float, V>(hz, hgates + gs + H);
    ldv<float, V>(hn, hgates + gs + 2 * H);
    ldv<T, V>(h, h_prev + ss);
#pragma unroll
    for (int k = 0; k < V; ++k) ho[k] = gru_fwd_unit(ir[k], iz[k], in[k], hr[k], hz[k], hn[k], h[k]);
    stv<T, V>(h_out + ss, ho);
  }
}

// digates, dhgates (beta 0; equal but for the n chunk: d(i_n) = dpre_n, d(h_n) = dpre_n * r) and the pointwise part of
// the hidden-state gradient, dh_prev = beta*dh_prev + z*dh_out
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_gru_cell_bwd_kernel(TG* __restrict__ digates, TG* __restrict__ dhgates,
                                                                   T* __restrict__ dh_prev, float beta_dh,
                                                                   const float* __restrict__ igates,
                                                                   const float* __restrict__ hgates,
                                                                   const T* __restrict__ h_prev,
                                                                   const T* __restrict__ dh_out, int64_t n, int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 3 * H + j, ss = row * H + j;
    float ir[V], iz[V], in[V], hr[V], hz[V], hn[V], h[V], dh[V], dhp[V];
    ldv<float, V>(ir, igates + gs);
    ldv<float, V>(iz, igates + gs + H);
    ldv<float, V>(in, igates + gs + 2 * H);
    ldv<float, V>(hr, hgates + gs);
    ldv<float, V>(hz, hgates + gs + H);
    ldv<float, V>(hn, hgates + gs + 2 * H);
    ldv<T, V>(h, h_prev + ss);
    ldv<T, V>(dh, dh_out + ss);
    if (dh_prev && beta_dh != 0.f) ldv<T, V>(dhp, dh_prev + ss);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      float v = gru_bwd_unit(ir[k], iz[k], in[k], hr[k], hz[k], hn[k], h[k], dh[k]);
      if (dh_prev && beta_dh != 0.f) v += beta_dh * dhp[k];
      dhp[k] = v;
    }
    stv<TG, V>(digates + gs, ir);
    stv<TG, V>(digates + gs + H, iz);
    stv<TG, V>(digates + gs + 2 * H, in);
    stv<TG, V>(dhgates + gs, ir);
    stv<TG, V>(dhgates + gs + H, iz);
    stv<TG, V>(dhgates + gs + 2 * H, hn);
    if (dh_prev) stv<T, V>(dh_prev + ss, dhp);
  }
}

// One backward time step of the GRU sequence node.  dh = dh_out (element type T, NULL = zero) + dh_rec (f32).  dh_rec is
// the running hidden-state gradient: read, then overwritten with the pointwise part z*dh of the previous step's gradient
// (the caller adds dhgates.W_hh to it).  dh_rec may be NULL when nothing is carried (a single step whose hidden state is
// not differentiable).
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_gru_seq_bwd_step_kernel(TG* __restrict__ digates, TG* __restrict__ dhgates,
                                                                       float* __restrict__ dh_rec,
                                                                       const float* __restrict__ igates,
                                                                       const float* __restrict__ hgates,
                                                                       const T* __restrict__ h_prev,
                                                                       const T* __restrict__ dh_out, int64_t n, int64_t H) {
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 3 * H + j, ss = row * H + j;
    float ir[V], iz[V], in[V], hr[V], hz[V], hn[V], h[V], dh[V], dr[V];
    ldv<float, V>(ir, igates + gs);
    ldv<float, V>(iz, igates + gs + H);
    ldv<float, V>(in, igates + gs + 2 * H);
    ldv<float, V>(hr, hgates + gs);
    ldv<float, V>(hz, hgates + gs + H);
    ldv<float, V>(hn, hgates + gs + 2 * H);
    ldv<T, V>(h, h_prev + ss);
    if (dh_out) ldv<T, V>(dh, dh_out + ss);
    if (dh_rec) ldv<float, V>(dr, dh_rec + ss);
#pragma unroll
    for (int k = 0; k < V; ++k)
      dr[k] = gru_bwd_unit(ir[k], iz[k], in[k], hr[k], hz[k], hn[k], h[k], (dh_out ? dh[k] : 0.f) + (dh_rec ? dr[k] : 0.f));
    stv<TG, V>(digates + gs, ir);
    stv<TG, V>(digates + gs + H, iz);
    stv<TG, V>(digates + gs + 2 * H, in);
    stv<TG, V>(dhgates + gs, ir);
    stv<TG, V>(dhgates + gs + H, iz);
    stv<TG, V>(dhgates + gs + 2 * H, hn);
    if (dh_rec) stv<float, V>(dh_rec + ss, dr);
  }
}

// ------------------------------------------------------------------------------------------------- two directions
// One time step of both directions of a bidirectional layer (nk_graph.cpp, RnnSeq with D = 2) in one launch:
// blockIdx.y = d is the direction, and every per-direction operand of direction d starts d * <its _ds> elements after the
// pointer passed (the graph passes the step's forward-direction slices and the distance to the reverse direction's).
// The state buffers h_next, dc and dh_rec are (2, n, H), direction stride n*H.  Rows of y / dh_out / h_prev are ld apart.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads) nk_lstm_bidir_fwd_step_kernel(T* __restrict__ y, int64_t y_ds, int64_t ldy,
                                                                          T* __restrict__ h_next, T* __restrict__ c_out,
                                                                          int64_t c_out_ds, const float* __restrict__ gates,
                                                                          int64_t g_ds, const T* __restrict__ c_prev,
                                                                          int64_t c_prev_ds, int64_t n, int64_t H) {
  const int64_t d = blockIdx.y;
  y += d * y_ds, h_next += d * n * H, c_out += d * c_out_ds, gates += d * g_ds, c_prev += d * c_prev_ds;
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const float* g = gates + row * 4 * H + j;
    float gi[V], gf[V], gg[V], go[V], c[V], co[V], ho[V];
    ldv<float, V>(gi, g);
    ldv<float, V>(gf, g + H);
    ldv<float, V>(gg, g + 2 * H);
    ldv<float, V>(go, g + 3 * H);
    ldv<T, V>(c, c_prev + row * H + j);
#pragma unroll
    for (int k = 0; k < V; ++k) lstm_fwd_unit(gi[k], gf[k], gg[k], go[k], c[k], co[k], ho[k]);
    stv<T, V>(c_out + row * H + j, co);
    stv<T, V>(y + row * ldy + j, ho);
    stv<T, V>(h_next + row * H + j, ho);
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads) nk_gru_bidir_fwd_step_kernel(T* __restrict__ y, int64_t y_ds, int64_t ldy,
                                                                         T* __restrict__ h_next,
                                                                         const float* __restrict__ igates,
                                                                         const float* __restrict__ hgates, int64_t g_ds,
                                                                         const T* __restrict__ h_prev, int64_t h_prev_ds,
                                                                         int64_t n, int64_t H) {
  const int64_t d = blockIdx.y;
  y += d * y_ds, h_next += d * n * H, igates += d * g_ds, hgates += d * g_ds, h_prev += d * h_prev_ds;
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 3 * H + j;
    float ir[V], iz[V], in[V], hr[V], hz[V], hn[V], h[V], ho[V];
    ldv<float, V>(ir, igates + gs);
    ldv<float, V>(iz, igates + gs + H);
    ldv<float, V>(in, igates + gs + 2 * H);
    ldv<float, V>(hr, hgates + gs);
    ldv<float, V>(hz, hgates + gs + H);
    ldv<float, V>(hn, hgates + gs + 2 * H);
    ldv<T, V>(h, h_prev + row * H + j);
#pragma unroll
    for (int k = 0; k < V; ++k) ho[k] = gru_fwd_unit(ir[k], iz[k], in[k], hr[k], hz[k], hn[k], h[k]);
    stv<T, V>(y + row * ldy + j, ho);
    stv<T, V>(h_next + row * H + j, ho);
  }
}

// dgates share the gates' layout (direction distance g_ds); dc (f32) is read as dc_out and overwritten with dc_prev
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_lstm_bidir_bwd_step_kernel(TG* __restrict__ dgates, int64_t g_ds,
                                                                          float* __restrict__ dc,
                                                                          const float* __restrict__ gates,
                                                                          const T* __restrict__ c_prev, int64_t c_prev_ds,
                                                                          const T* __restrict__ dh_out, int64_t dh_ds,
                                                                          int64_t ld_dh, const float* __restrict__ dh_rec,
                                                                          int64_t n, int64_t H) {
  const int64_t d = blockIdx.y;
  dgates += d * g_ds, gates += d * g_ds, dc += d * n * H, c_prev += d * c_prev_ds;
  if (dh_out) dh_out += d * dh_ds;
  if (dh_rec) dh_rec += d * n * H;
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 4 * H + j, ss = row * H + j;
    float gi[V], gf[V], gg[V], go[V], c[V], dh[V], dr[V], dcr[V];
    ldv<float, V>(gi, gates + gs);
    ldv<float, V>(gf, gates + gs + H);
    ldv<float, V>(gg, gates + gs + 2 * H);
    ldv<float, V>(go, gates + gs + 3 * H);
    ldv<T, V>(c, c_prev + ss);
    ldv<float, V>(dcr, dc + ss);
    if (dh_out) ldv<T, V>(dh, dh_out + row * ld_dh + j);
    if (dh_rec) ldv<float, V>(dr, dh_rec + ss);
#pragma unroll
    for (int k = 0; k < V; ++k)
      dcr[k] = lstm_bwd_unit(gi[k], gf[k], gg[k], go[k], c[k], (dh_out ? dh[k] : 0.f) + (dh_rec ? dr[k] : 0.f), dcr[k]);
    stv<TG, V>(dgates + gs, gi);
    stv<TG, V>(dgates + gs + H, gf);
    stv<TG, V>(dgates + gs + 2 * H, gg);
    stv<TG, V>(dgates + gs + 3 * H, go);
    stv<float, V>(dc + ss, dcr);
  }
}

// dh_rec (f32) is read and overwritten with z*dh (the caller adds dhgates.W_hh)
template <typename T, typename TG, int V>
__global__ void __launch_bounds__(kThreads) nk_gru_bidir_bwd_step_kernel(TG* __restrict__ digates, TG* __restrict__ dhgates,
                                                                         int64_t g_ds, float* __restrict__ dh_rec,
                                                                         const float* __restrict__ igates,
                                                                         const float* __restrict__ hgates,
                                                                         const T* __restrict__ h_prev, int64_t h_prev_ds,
                                                                         int64_t ld_h, const T* __restrict__ dh_out,
                                                                         int64_t dh_ds, int64_t ld_dh, int64_t n,
                                                                         int64_t H) {
  const int64_t d = blockIdx.y;
  digates += d * g_ds, dhgates += d * g_ds, igates += d * g_ds, hgates += d * g_ds, h_prev += d * h_prev_ds;
  if (dh_out) dh_out += d * dh_ds;
  if (dh_rec) dh_rec += d * n * H;
  const int64_t per_row = H / V;
  const size_t units = size_t(n) * size_t(per_row);
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t u = size_t(blockIdx.x) * blockDim.x + threadIdx.x; u < units; u += stride) {
    const int64_t row = int64_t(u / size_t(per_row)), j = int64_t(u % size_t(per_row)) * V;
    const int64_t gs = row * 3 * H + j, ss = row * H + j;
    float ir[V], iz[V], in[V], hr[V], hz[V], hn[V], h[V], dh[V], dr[V];
    ldv<float, V>(ir, igates + gs);
    ldv<float, V>(iz, igates + gs + H);
    ldv<float, V>(in, igates + gs + 2 * H);
    ldv<float, V>(hr, hgates + gs);
    ldv<float, V>(hz, hgates + gs + H);
    ldv<float, V>(hn, hgates + gs + 2 * H);
    ldv<T, V>(h, h_prev + row * ld_h + j);
    if (dh_out) ldv<T, V>(dh, dh_out + row * ld_dh + j);
    if (dh_rec) ldv<float, V>(dr, dh_rec + ss);
#pragma unroll
    for (int k = 0; k < V; ++k)
      dr[k] = gru_bwd_unit(ir[k], iz[k], in[k], hr[k], hz[k], hn[k], h[k], (dh_out ? dh[k] : 0.f) + (dh_rec ? dr[k] : 0.f));
    stv<TG, V>(digates + gs, ir);
    stv<TG, V>(digates + gs + H, iz);
    stv<TG, V>(digates + gs + 2 * H, in);
    stv<TG, V>(dhgates + gs, ir);
    stv<TG, V>(dhgates + gs + H, iz);
    stv<TG, V>(dhgates + gs + 2 * H, hn);
    if (dh_rec) stv<float, V>(dh_rec + ss, dr);
  }
}

// ------------------------------------------------------------------------------------------------- chunk
struct ChunkDims {
  int ndim;
  int64_t cshape[NK_MAX_DIMS];   // chunk shape
  int64_t xstride[NK_MAX_DIMS];  // element strides of the operand
  int64_t origin;                // operand offset of the block's first element
};

__device__ __forceinline__ int64_t chunk_offset(const ChunkDims& d, size_t i) {
  int64_t off = d.origin;
  size_t rem = i;
#pragma unroll
  for (int k = NK_MAX_DIMS - 1; k >= 0; --k) {
    if (k < d.ndim) {
      off += int64_t(rem % size_t(d.cshape[k])) * d.xstride[k];
      rem /= size_t(d.cshape[k]);
    }
  }
  return off;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) nk_chunk_fwd_kernel(T* __restrict__ y, const T* __restrict__ x, size_t n,
                                                                ChunkDims d) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = x[chunk_offset(d, i)];
}

template <typename TD, typename TGr>
__global__ void __launch_bounds__(kThreads) nk_chunk_bwd_kernel(TD* __restrict__ dx, const TGr* __restrict__ g, size_t n,
                                                                ChunkDims d, float beta) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t o = chunk_offset(d, i);
    float v = nk_to_f32<TGr>(g[i]);
    if (beta != 0.f) v += beta * nk_to_f32<TD>(dx[o]);
    dx[o] = nk_from_f32<TD>(v);
  }
}

static int chunk_dims(nk_ctx* ctx, ChunkDims& d, int ndim, const int64_t* x_shape, const int64_t* chunk_shape, int64_t index,
               size_t& n) {
  NK_REQUIRE(ctx, ndim >= 1 && ndim <= NK_MAX_DIMS && x_shape && chunk_shape, "nk_chunk: bad shape arguments");
  d.ndim = ndim;
  int64_t blocks[NK_MAX_DIMS], nblocks = 1;
  n = 1;
  for (int k = 0; k < ndim; ++k) {
    NK_REQUIRE(ctx, x_shape[k] >= 0 && chunk_shape[k] >= 1 && chunk_shape[k] <= x_shape[k],
               "nk_chunk: chunk dimension %d (%lld) must be in [1, %lld]", k, (long long)chunk_shape[k],
               (long long)x_shape[k]);
    d.cshape[k] = chunk_shape[k];
    blocks[k] = x_shape[k] / chunk_shape[k];   // exact_chunks: trailing partial blocks are dropped
    nblocks *= blocks[k];
    n *= size_t(chunk_shape[k]);
  }
  NK_REQUIRE(ctx, index >= 0 && index < nblocks, "nk_chunk: index %lld out of range (%lld chunks)", (long long)index,
             (long long)nblocks);
  int64_t s = 1, rem = index;
  d.origin = 0;
  for (int k = ndim - 1; k >= 0; --k) {
    d.xstride[k] = s;
    d.origin += (rem % blocks[k]) * chunk_shape[k] * s;
    rem /= blocks[k];
    s *= x_shape[k];
  }
  for (int k = ndim; k < NK_MAX_DIMS; ++k) d.cshape[k] = 1, d.xstride[k] = 0;
  return NK_OK;
}

// the vector bodies need 16-byte aligned bases and every stride (ld, direction distance) a multiple of 16 bytes
static inline bool bytes16(int64_t elems, size_t esize) { return (elems * int64_t(esize)) % 16 == 0; }
static inline dim3 bidir_grid(nk_ctx* ctx, size_t units) { return dim3(unsigned(rnn_blocks(ctx, units)), 2u); }

static int cell_args(nk_ctx* ctx, const char* who, int64_t n, int64_t hidden, int dtype) {
  NK_REQUIRE(ctx, n >= 0 && hidden >= 0, "%s: negative size", who);
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "%s: bad dtype %d", who, dtype);
  return NK_OK;
}

}  // namespace nk_rnn

using namespace nk_rnn;

extern "C" {

int nk_lstm_cell_fwd(nk_ctx* ctx, void* c_out, void* h_out, const float* gates, const void* c_prev, int64_t n,
                     int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_lstm_cell_fwd", n, hidden, dtype)) return rc;
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, c_out && h_out && gates && c_prev, "nk_lstm_cell_fwd: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    constexpr int V = NkVec<T>::N;
    const bool vec = hidden % V == 0 && aligned16(c_out) && aligned16(h_out) && aligned16(gates) && aligned16(c_prev);
    const int64_t units = n * (vec ? hidden / V : hidden);
    if (vec)
      nk_lstm_cell_fwd_kernel<T, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)c_out, (T*)h_out, gates, (const T*)c_prev, n, hidden);
    else
      nk_lstm_cell_fwd_kernel<T, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)c_out, (T*)h_out, gates, (const T*)c_prev, n, hidden);
  });
  NK_LAUNCHED(ctx, "lstm_cell_fwd");
  return NK_OK;
}

int nk_lstm_cell_bwd(nk_ctx* ctx, void* dgates, int dgates_dtype, void* dc_prev, float beta_dc, const float* gates,
                     const void* c_prev, const void* dh_out, const void* dc_out, int64_t n, int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_lstm_cell_bwd", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dgates_dtype), "nk_lstm_cell_bwd: bad dgates dtype %d", dgates_dtype);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, dgates && gates && c_prev, "nk_lstm_cell_bwd: NULL pointer");
  const bool al = aligned16(dgates) && aligned16(gates) && aligned16(c_prev) && (!dc_prev || aligned16(dc_prev)) &&
                  (!dh_out || aligned16(dh_out)) && (!dc_out || aligned16(dc_out));
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dgates_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const bool vec = al && hidden % V == 0;
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_lstm_cell_bwd_kernel<T, TG, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, (T*)dc_prev, beta_dc, gates, (const T*)c_prev, (const T*)dh_out, (const T*)dc_out, n, hidden);
      else
        nk_lstm_cell_bwd_kernel<T, TG, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, (T*)dc_prev, beta_dc, gates, (const T*)c_prev, (const T*)dh_out, (const T*)dc_out, n, hidden);
    });
  });
  NK_LAUNCHED(ctx, "lstm_cell_bwd");
  return NK_OK;
}

int nk_gru_cell_fwd(nk_ctx* ctx, void* h_out, const float* igates, const float* hgates, const void* h_prev, int64_t n,
                    int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_gru_cell_fwd", n, hidden, dtype)) return rc;
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, h_out && igates && hgates && h_prev, "nk_gru_cell_fwd: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    constexpr int V = NkVec<T>::N;
    const bool vec = hidden % V == 0 && aligned16(h_out) && aligned16(igates) && aligned16(hgates) && aligned16(h_prev);
    const int64_t units = n * (vec ? hidden / V : hidden);
    if (vec)
      nk_gru_cell_fwd_kernel<T, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)h_out, igates, hgates, (const T*)h_prev, n, hidden);
    else
      nk_gru_cell_fwd_kernel<T, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)h_out, igates, hgates, (const T*)h_prev, n, hidden);
  });
  NK_LAUNCHED(ctx, "gru_cell_fwd");
  return NK_OK;
}

int nk_gru_cell_bwd(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, void* dh_prev, float beta_dh,
                    const float* igates, const float* hgates, const void* h_prev, const void* dh_out, int64_t n,
                    int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_gru_cell_bwd", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dg_dtype), "nk_gru_cell_bwd: bad dgates dtype %d", dg_dtype);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, digates && dhgates && igates && hgates && h_prev && dh_out, "nk_gru_cell_bwd: NULL pointer");
  const bool al = aligned16(digates) && aligned16(dhgates) && aligned16(igates) && aligned16(hgates) &&
                  aligned16(h_prev) && aligned16(dh_out) && (!dh_prev || aligned16(dh_prev));
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dg_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const bool vec = al && hidden % V == 0;
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_gru_cell_bwd_kernel<T, TG, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, (T*)dh_prev, beta_dh, igates, hgates, (const T*)h_prev, (const T*)dh_out, n,
            hidden);
      else
        nk_gru_cell_bwd_kernel<T, TG, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, (T*)dh_prev, beta_dh, igates, hgates, (const T*)h_prev, (const T*)dh_out, n,
            hidden);
    });
  });
  NK_LAUNCHED(ctx, "gru_cell_bwd");
  return NK_OK;
}

int nk_lstm_seq_bwd_step(nk_ctx* ctx, void* dgates, int dgates_dtype, float* dc, const float* gates, const void* c_prev,
                         const void* dh_out, const float* dh_rec, int64_t n, int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_lstm_seq_bwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dgates_dtype), "nk_lstm_seq_bwd_step: bad dgates dtype %d", dgates_dtype);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, dgates && dc && gates && c_prev, "nk_lstm_seq_bwd_step: NULL pointer");
  const bool al = aligned16(dgates) && aligned16(dc) && aligned16(gates) && aligned16(c_prev) &&
                  (!dh_out || aligned16(dh_out)) && (!dh_rec || aligned16(dh_rec));
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dgates_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const bool vec = al && hidden % V == 0;
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_lstm_seq_bwd_step_kernel<T, TG, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, dc, gates, (const T*)c_prev, (const T*)dh_out, dh_rec, n, hidden);
      else
        nk_lstm_seq_bwd_step_kernel<T, TG, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, dc, gates, (const T*)c_prev, (const T*)dh_out, dh_rec, n, hidden);
    });
  });
  NK_LAUNCHED(ctx, "lstm_seq_bwd_step");
  return NK_OK;
}

int nk_gru_seq_bwd_step(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, float* dh_rec, const float* igates,
                        const float* hgates, const void* h_prev, const void* dh_out, int64_t n, int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_gru_seq_bwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dg_dtype), "nk_gru_seq_bwd_step: bad dgates dtype %d", dg_dtype);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, digates && dhgates && igates && hgates && h_prev, "nk_gru_seq_bwd_step: NULL pointer");
  const bool al = aligned16(digates) && aligned16(dhgates) && aligned16(igates) && aligned16(hgates) &&
                  aligned16(h_prev) && (!dh_out || aligned16(dh_out)) && (!dh_rec || aligned16(dh_rec));
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dg_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const bool vec = al && hidden % V == 0;
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_gru_seq_bwd_step_kernel<T, TG, V><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, dh_rec, igates, hgates, (const T*)h_prev, (const T*)dh_out, n, hidden);
      else
        nk_gru_seq_bwd_step_kernel<T, TG, 1><<<rnn_blocks(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, dh_rec, igates, hgates, (const T*)h_prev, (const T*)dh_out, n, hidden);
    });
  });
  NK_LAUNCHED(ctx, "gru_seq_bwd_step");
  return NK_OK;
}

int nk_lstm_bidir_fwd_step(nk_ctx* ctx, void* y, int64_t y_dstride, int64_t ldy, void* h_next, void* c_out,
                           int64_t c_out_dstride, const float* gates, int64_t gates_dstride, const void* c_prev,
                           int64_t c_prev_dstride, int64_t n, int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_lstm_bidir_fwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, ldy >= hidden, "nk_lstm_bidir_fwd_step: ldy %lld < hidden %lld", (long long)ldy, (long long)hidden);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, y && h_next && c_out && gates && c_prev, "nk_lstm_bidir_fwd_step: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    constexpr int V = NkVec<T>::N;
    const size_t es = sizeof(T);
    const bool vec = hidden % V == 0 && aligned16(y) && aligned16(h_next) && aligned16(c_out) && aligned16(gates) &&
                     aligned16(c_prev) && bytes16(y_dstride, es) && bytes16(ldy, es) && bytes16(c_out_dstride, es) &&
                     bytes16(gates_dstride, 4) && bytes16(c_prev_dstride, es);
    const int64_t units = n * (vec ? hidden / V : hidden);
    if (vec)
      nk_lstm_bidir_fwd_step_kernel<T, V><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)y, y_dstride, ldy, (T*)h_next, (T*)c_out, c_out_dstride, gates, gates_dstride, (const T*)c_prev,
          c_prev_dstride, n, hidden);
    else
      nk_lstm_bidir_fwd_step_kernel<T, 1><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)y, y_dstride, ldy, (T*)h_next, (T*)c_out, c_out_dstride, gates, gates_dstride, (const T*)c_prev,
          c_prev_dstride, n, hidden);
  });
  NK_LAUNCHED(ctx, "lstm_bidir_fwd_step");
  return NK_OK;
}

int nk_gru_bidir_fwd_step(nk_ctx* ctx, void* y, int64_t y_dstride, int64_t ldy, void* h_next, const float* igates,
                          const float* hgates, int64_t gates_dstride, const void* h_prev, int64_t h_prev_dstride, int64_t n,
                          int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_gru_bidir_fwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, ldy >= hidden, "nk_gru_bidir_fwd_step: ldy %lld < hidden %lld", (long long)ldy, (long long)hidden);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, y && h_next && igates && hgates && h_prev, "nk_gru_bidir_fwd_step: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    constexpr int V = NkVec<T>::N;
    const size_t es = sizeof(T);
    const bool vec = hidden % V == 0 && aligned16(y) && aligned16(h_next) && aligned16(igates) && aligned16(hgates) &&
                     aligned16(h_prev) && bytes16(y_dstride, es) && bytes16(ldy, es) && bytes16(gates_dstride, 4) &&
                     bytes16(h_prev_dstride, es);
    const int64_t units = n * (vec ? hidden / V : hidden);
    if (vec)
      nk_gru_bidir_fwd_step_kernel<T, V><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)y, y_dstride, ldy, (T*)h_next, igates, hgates, gates_dstride, (const T*)h_prev, h_prev_dstride, n, hidden);
    else
      nk_gru_bidir_fwd_step_kernel<T, 1><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
          (T*)y, y_dstride, ldy, (T*)h_next, igates, hgates, gates_dstride, (const T*)h_prev, h_prev_dstride, n, hidden);
  });
  NK_LAUNCHED(ctx, "gru_bidir_fwd_step");
  return NK_OK;
}

int nk_lstm_bidir_bwd_step(nk_ctx* ctx, void* dgates, int dgates_dtype, int64_t gates_dstride, float* dc, const float* gates,
                           const void* c_prev, int64_t c_prev_dstride, const void* dh_out, int64_t dh_out_dstride,
                           int64_t ld_dh_out, const float* dh_rec, int64_t n, int64_t hidden, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_lstm_bidir_bwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dgates_dtype), "nk_lstm_bidir_bwd_step: bad dgates dtype %d", dgates_dtype);
  NK_REQUIRE(ctx, !dh_out || ld_dh_out >= hidden, "nk_lstm_bidir_bwd_step: ld_dh_out %lld < hidden %lld",
             (long long)ld_dh_out, (long long)hidden);
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, dgates && dc && gates && c_prev, "nk_lstm_bidir_bwd_step: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dgates_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const size_t es = sizeof(T);
      const bool vec = hidden % V == 0 && aligned16(dgates) && aligned16(dc) && aligned16(gates) && aligned16(c_prev) &&
                       bytes16(gates_dstride, sizeof(TG)) && bytes16(gates_dstride, 4) && bytes16(c_prev_dstride, es) &&
                       (!dh_out || (aligned16(dh_out) && bytes16(dh_out_dstride, es) && bytes16(ld_dh_out, es))) &&
                       (!dh_rec || aligned16(dh_rec));
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_lstm_bidir_bwd_step_kernel<T, TG, V><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, gates_dstride, dc, gates, (const T*)c_prev, c_prev_dstride, (const T*)dh_out, dh_out_dstride,
            ld_dh_out, dh_rec, n, hidden);
      else
        nk_lstm_bidir_bwd_step_kernel<T, TG, 1><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)dgates, gates_dstride, dc, gates, (const T*)c_prev, c_prev_dstride, (const T*)dh_out, dh_out_dstride,
            ld_dh_out, dh_rec, n, hidden);
    });
  });
  NK_LAUNCHED(ctx, "lstm_bidir_bwd_step");
  return NK_OK;
}

int nk_gru_bidir_bwd_step(nk_ctx* ctx, void* digates, void* dhgates, int dg_dtype, int64_t gates_dstride, float* dh_rec,
                          const float* igates, const float* hgates, const void* h_prev, int64_t h_prev_dstride, int64_t ld_h_prev,
                          const void* dh_out, int64_t dh_out_dstride, int64_t ld_dh_out, int64_t n, int64_t hidden,
                          int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  if (int rc = cell_args(ctx, "nk_gru_bidir_bwd_step", n, hidden, dtype)) return rc;
  NK_REQUIRE(ctx, nk_dtype_ok(dg_dtype), "nk_gru_bidir_bwd_step: bad dgates dtype %d", dg_dtype);
  NK_REQUIRE(ctx, ld_h_prev >= hidden && (!dh_out || ld_dh_out >= hidden), "nk_gru_bidir_bwd_step: leading dimension too small");
  if (n == 0 || hidden == 0) return NK_OK;
  NK_REQUIRE(ctx, digates && dhgates && igates && hgates && h_prev, "nk_gru_bidir_bwd_step: NULL pointer");
  NK_DISPATCH_DTYPE(dtype, T, {
    NK_DISPATCH_DTYPE(dg_dtype, TG, {
      constexpr int V = NkVec<T>::N;
      const size_t es = sizeof(T);
      const bool vec = hidden % V == 0 && aligned16(digates) && aligned16(dhgates) && aligned16(igates) &&
                       aligned16(hgates) && aligned16(h_prev) && bytes16(gates_dstride, sizeof(TG)) &&
                       bytes16(gates_dstride, 4) && bytes16(h_prev_dstride, es) && bytes16(ld_h_prev, es) &&
                       (!dh_out || (aligned16(dh_out) && bytes16(dh_out_dstride, es) && bytes16(ld_dh_out, es))) &&
                       (!dh_rec || aligned16(dh_rec));
      const int64_t units = n * (vec ? hidden / V : hidden);
      if (vec)
        nk_gru_bidir_bwd_step_kernel<T, TG, V><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, gates_dstride, dh_rec, igates, hgates, (const T*)h_prev, h_prev_dstride, ld_h_prev,
            (const T*)dh_out, dh_out_dstride, ld_dh_out, n, hidden);
      else
        nk_gru_bidir_bwd_step_kernel<T, TG, 1><<<bidir_grid(ctx, units), kThreads, 0, ctx->stream>>>(
            (TG*)digates, (TG*)dhgates, gates_dstride, dh_rec, igates, hgates, (const T*)h_prev, h_prev_dstride, ld_h_prev,
            (const T*)dh_out, dh_out_dstride, ld_dh_out, n, hidden);
    });
  });
  NK_LAUNCHED(ctx, "gru_bidir_bwd_step");
  return NK_OK;
}

int nk_chunk_fwd(nk_ctx* ctx, void* y, const void* x, int ndim, const int64_t* x_shape, const int64_t* chunk_shape,
                 int64_t index, int dtype) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dtype), "nk_chunk_fwd: bad dtype %d", dtype);
  ChunkDims d;
  size_t n;
  if (int rc = chunk_dims(ctx, d, ndim, x_shape, chunk_shape, index, n)) return rc;
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, y && x, "nk_chunk_fwd: NULL pointer");
  if (dtype == NK_BF16)   // a copy: moved as 16-bit words, bit exact
    nk_chunk_fwd_kernel<uint16_t><<<rnn_blocks(ctx, n), kThreads, 0, ctx->stream>>>((uint16_t*)y, (const uint16_t*)x, n, d);
  else
    nk_chunk_fwd_kernel<uint32_t><<<rnn_blocks(ctx, n), kThreads, 0, ctx->stream>>>((uint32_t*)y, (const uint32_t*)x, n, d);
  NK_LAUNCHED(ctx, "chunk_fwd");
  return NK_OK;
}

int nk_chunk_bwd(nk_ctx* ctx, void* dx, int dx_dtype, const void* g, int g_dtype, int ndim, const int64_t* x_shape,
                 const int64_t* chunk_shape, int64_t index, float beta) {
  if (!ctx) return NK_ERR_INVALID_ARG;
  NK_REQUIRE(ctx, nk_dtype_ok(dx_dtype) && nk_dtype_ok(g_dtype), "nk_chunk_bwd: bad dtype");
  ChunkDims d;
  size_t n;
  if (int rc = chunk_dims(ctx, d, ndim, x_shape, chunk_shape, index, n)) return rc;
  if (n == 0) return NK_OK;
  NK_REQUIRE(ctx, dx && g, "nk_chunk_bwd: NULL pointer");
  NK_DISPATCH_DTYPE(dx_dtype, TD, {
    NK_DISPATCH_DTYPE(g_dtype, TGr, {
      nk_chunk_bwd_kernel<TD, TGr><<<rnn_blocks(ctx, n), kThreads, 0, ctx->stream>>>((TD*)dx, (const TGr*)g, n, d, beta);
    });
  });
  NK_LAUNCHED(ctx, "chunk_bwd");
  return NK_OK;
}

}  // extern "C"
