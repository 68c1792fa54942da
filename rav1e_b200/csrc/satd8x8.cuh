// satd8x8.cuh — the 8x8 SATD of the lookahead's importance blocks, shared by lookahead.cu and
// temporal_rdo.cu (both call get_satd on 8x8 blocks, api/lookahead.rs and api/internal.rs:963-970).
#pragma once

#include <cstdint>

namespace b200_satd8 {

__device__ __forceinline__ void bfly(int &a, int &b) {
  const int s = a + b, t = a - b;
  a = s;
  b = t;
}

// sum |H8 d H8^T| with the single final rounding of get_satd (dist.rs:156-221, 8x8: ln = 3)
__device__ __forceinline__ uint32_t satd8x8(int (&d)[64]) {
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int s0 = pass == 0 ? 1 : 8, s1 = pass == 0 ? 8 : 1;
      int v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = d[i * s0 + k * s1];
      bfly(v[0], v[1]);
      bfly(v[2], v[3]);
      bfly(v[4], v[5]);
      bfly(v[6], v[7]);
      bfly(v[0], v[2]);
      bfly(v[1], v[3]);
      bfly(v[4], v[6]);
      bfly(v[5], v[7]);
      bfly(v[0], v[4]);
      bfly(v[1], v[5]);
      bfly(v[2], v[6]);
      bfly(v[3], v[7]);
#pragma unroll
      for (int k = 0; k < 8; k++) d[i * s0 + k * s1] = v[k];
    }
  }
  unsigned long long s = 0;
#pragma unroll
  for (int i = 0; i < 64; i++) s += (uint32_t)abs(d[i]);
  return (uint32_t)((s + 4) >> 3);
}

}  // namespace b200_satd8
