// Output extents and argument checks of the pooling ops (nk_pool.cu), shared with the graph recorder (nk_graph.cpp) so
// that both reject exactly what torch rejects, with the same messages.  Plain host C++.
#pragma once
#include <stdint.h>
#include <stdio.h>

// torch's pooling_output_shape: O = floor_or_ceil((L + 2p - d(k-1) - 1) / s) + 1; with ceil_mode the last window is
// dropped when it would start in the right padding
static inline int64_t nk_pool_floordiv(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
static inline int64_t nk_pool_out_extent(int64_t L, int64_t k, int64_t s, int64_t p, int64_t d, bool ceil_mode) {
  const int64_t num = L + 2 * p - d * (k - 1) - 1;
  int64_t o = nk_pool_floordiv(ceil_mode ? num + s - 1 : num, s) + 1;
  if (ceil_mode && (o - 1) * s >= L + p) --o;
  return o;
}

// checks one axis of a max / avg pool; 0 when valid, else writes the reason into msg
static inline int nk_pool_check_axis(const char* who, int axis, int64_t L, int64_t k, int64_t s, int64_t p, int64_t d,
                                     char* msg, size_t n) {
  if (k < 1 || s < 1 || d < 1) {
    snprintf(msg, n, "%s: kernel size, stride and dilation must be >= 1 (axis %d: %lld, %lld, %lld)", who, axis,
             (long long)k, (long long)s, (long long)d);
    return 1;
  }
  if (p < 0 || p > k / 2) {
    snprintf(msg, n, "%s: padding %lld must be >= 0 and at most half the kernel size %lld (axis %d)", who, (long long)p,
             (long long)k, axis);
    return 1;
  }
  if (L < 0) {
    snprintf(msg, n, "%s: negative input size %lld (axis %d)", who, (long long)L, axis);
    return 1;
  }
  return 0;
}
