// Per-element arithmetic of the five optimizers, shared by the per-parameter kernels (nk_elementwise.cu: SGD,
// nk_optim.cu: the Adam family) and the multi-tensor kernels (nk_optim_multi.cu).  Both paths inline the same
// statements in the same order, so they compile to the same instructions (including nvcc's FMA contractions) and give
// the same bits.  `wv` is the f32 weight (the master copy when there is one), `gv` the penalised gradient.
#pragma once

// SGD penalty (sgd/mod.rs:191-231, penalty.rs:63-67): g' = grad_scale*g + 2*l2*w.  The SGD update spells out its
// fused multiply-adds: left to nvcc, the contraction of `a*b + c*d` can differ between two kernels that inline the same
// expression.  These are the contractions the SGD kernels have always compiled to.
__device__ __forceinline__ float nk_sgd_grad(float g, float wv, float grad_scale, float l2x2) {
  return __fmaf_rn(l2x2, wv, __fmul_rn(g, grad_scale));  // grad += penalty.penalize(w) = 2*lambda*w
}

__device__ __forceinline__ float nk_sgd_update(float wv, float gv, float& buf, float lr, float mu, float one_minus_damp,
                                               int use_momentum, int nesterov) {
  if (!use_momentum) return __fmaf_rn(-gv, lr, wv);
  const float b = __fmaf_rn(gv, one_minus_damp, __fmul_rn(buf, mu));
  buf = b;
  return __fmaf_rn(-(nesterov ? __fmaf_rn(b, mu, gv) : b), lr, wv);
}

// Adam-family penalties (penalty.rs:63-79): g' = grad_scale*g + l1*signum(w) + 2*l2*w
struct NkOptPenalty {
  float l1, l2x2, grad_scale;
  int write_back_grad;
};

__device__ __forceinline__ float nk_signum_f32(float w) {  // f32::signum: 1.0 for +0.0, -1.0 for -0.0, NaN for NaN
  return w != w ? w : copysignf(1.f, w);
}

__device__ __forceinline__ float nk_opt_grad(const NkOptPenalty& c, float g, float wv) {
  float gv = g * c.grad_scale;
  if (c.l1 != 0.f) gv += c.l1 * nk_signum_f32(wv);
  gv += c.l2x2 * wv;
  return gv;
}

// adam/mod.rs:150-166, amsgrad/mod.rs:177-200; `max_sq` is read and written only when `ams`
__device__ __forceinline__ float nk_adam_update(float wv, float gv, float& exp_avg, float& exp_avg_sq, bool ams,
                                                float& max_sq, float beta1, float beta2, float sqrt_bc2,
                                                float step_size, float eps) {
  const float m = exp_avg * beta1 + gv * (1.f - beta1);
  const float v = exp_avg_sq * beta2 + gv * gv * (1.f - beta2);
  exp_avg = m;
  exp_avg_sq = v;
  float vv = v;
  if (ams) {  // AMSGrad: running maximum of the second moment
    vv = fmaxf(max_sq, v);
    max_sq = vv;
  }
  wv -= m / ((sqrtf(vv) / sqrt_bc2) + eps) * step_size;
  return wv;
}

// rmsprop/mod.rs:193-300: the four (centered, momentum) variants
__device__ __forceinline__ float nk_rmsprop_update(float wv, float gv, float& square_avg, bool centered,
                                                   float& grad_avg, bool momentum_on, float& buf, float lr,
                                                   float alpha, float eps, float momentum) {
  const float sq = square_avg * alpha + gv * gv * (1.f - alpha);
  square_avg = sq;
  float denom;
  if (centered) {
    const float ga = grad_avg * alpha + gv * (1.f - alpha);
    grad_avg = ga;
    denom = sqrtf(sq + (-ga * ga)) + eps;
  } else {
    denom = sqrtf(sq) + eps;
  }
  if (momentum_on) {
    const float b = buf * momentum + gv / denom;
    buf = b;
    wv -= b * lr;
  } else {
    wv -= gv / denom * lr;
  }
  return wv;
}

// adagrad/mod.rs:113-140
__device__ __forceinline__ float nk_adagrad_update(float wv, float gv, float& grad_sq, float clr, float eps) {
  const float s = grad_sq + gv * gv;
  grad_sq = s;
  wv -= gv / (sqrtf(s) + eps) * clr;
  return wv;
}
