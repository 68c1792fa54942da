// hadamard.cuh — the Hadamard butterfly networks of get_satd (dist.rs:55-149) and the 2-D transforms
// built from them.  Every SATD kernel runs these networks; where kernels differ (IDP.4A horizontal
// passes on packed bytes, shuffle-based vertical passes, a last stage folded into 2*max) they call
// the 1-D networks below and keep the differing part themselves.
//
// The transforms are exact integer arithmetic and only sum |coeff| is consumed, so the pass order and
// the order of outputs inside a vector do not change any result; the networks keep the reference's
// order anyway.  The abs-sums are u32: 64 coefficients of at most 64 * 4095 (12-bit) stay below 2^25.
#pragma once

#include <cstdint>

__device__ __forceinline__ void bfly(int &a, int &b) {
  const int s = a + b, t = a - b;
  a = s;
  b = t;
}

// hadamard4_1d (dist.rs:55-73)
__device__ __forceinline__ void hadamard4(int (&a)[4]) {
  bfly(a[0], a[1]);
  bfly(a[2], a[3]);
  bfly(a[0], a[2]);
  bfly(a[1], a[3]);
}

// hadamard8_1d (dist.rs:88-121).  kStages < 3 stops early: a caller that folds the last stage into
// its sum (|x + y| + |x - y| = 2 max(|x|, |y|) over the pairs (k, k + 4)) runs the first two.
template <int kStages = 3>
__device__ __forceinline__ void hadamard8(int (&a)[8]) {
  bfly(a[0], a[1]);
  bfly(a[2], a[3]);
  bfly(a[4], a[5]);
  bfly(a[6], a[7]);
  bfly(a[0], a[2]);
  bfly(a[1], a[3]);
  bfly(a[4], a[6]);
  bfly(a[5], a[7]);
  if (kStages < 3) return;
  bfly(a[0], a[4]);
  bfly(a[1], a[5]);
  bfly(a[2], a[6]);
  bfly(a[3], a[7]);
}

// sum |H4 d H4^T| over a 4x4 difference block: vertical (stride 4 over rows) then horizontal,
// dist.rs:125-143; no rounding
__device__ __forceinline__ uint32_t hadamard4x4_abs_sum(int (&d)[16]) {
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int s0 = pass == 0 ? 1 : 4, s1 = pass == 0 ? 4 : 1;
      int a[4];
#pragma unroll
      for (int k = 0; k < 4; k++) a[k] = d[i * s0 + k * s1];
      hadamard4(a);
#pragma unroll
      for (int k = 0; k < 4; k++) d[i * s0 + k * s1] = a[k];
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) s += (uint32_t)abs(d[i]);
  return s;
}

// sum |H8 d H8^T| over an 8x8 difference block; no rounding
__device__ __forceinline__ uint32_t hadamard8x8_abs_sum(int (&d)[64]) {
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int s0 = pass == 0 ? 1 : 8, s1 = pass == 0 ? 8 : 1;
      int a[8];
#pragma unroll
      for (int k = 0; k < 8; k++) a[k] = d[i * s0 + k * s1];
      hadamard8(a);
#pragma unroll
      for (int k = 0; k < 8; k++) d[i * s0 + k * s1] = a[k];
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 64; i++) s += (uint32_t)abs(d[i]);
  return s;
}

// get_satd of one 8x8 block (dist.rs:156-221): the abs-sum with its single final rounding (ln = 3).
// The lookahead's importance blocks (api/lookahead.rs, api/internal.rs:963-970) are all 8x8.
__device__ __forceinline__ uint32_t satd8x8(int (&d)[64]) { return (hadamard8x8_abs_sum(d) + 4) >> 3; }
