// warp_satd.cuh — get_satd (dist.rs:156-221) of one W x H block by ONE warp, against a packed W x H
// prediction.  The result is the block's SATD on every lane.  Used by the sub-pel RDO kernel
// (subpel_rdo.cu) and the inter mode screen (inter_screen.cu).
#pragma once
#include "hadamard.cuh"

namespace {

// SATD of the W x H block: 8 lanes per 8x8 chunk (lane = row), four chunks per step
template <typename T, int W, int H>
__device__ __forceinline__ uint32_t warp_satd(const T *org, int os, const T *pred, int lane) {
  constexpr int NCH = (W / 8) * (H / 8);
  const int row = lane & 7, g = lane >> 3;
  uint32_t acc = 0;
#pragma unroll
  for (int c0 = 0; c0 < NCH; c0 += 4) {
    const int ch = c0 + g;
    int v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = 0;
    if (NCH % 4 == 0 || ch < NCH) {
      const int cy = (ch / (W / 8)) * 8, cx = (ch % (W / 8)) * 8;
      const T *o = org + (long long)(cy + row) * os + cx;
      const T *p = pred + (cy + row) * W + cx;
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = (int)o[k] - (int)p[k];
    }
    hadamard8(v);  // horizontal pass in registers
    // vertical pass across the 8 lanes of the chunk
#pragma unroll
    for (int s = 1; s < 8; s <<= 1) {
      const bool hi = (row & s) != 0;
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int other = __shfl_xor_sync(0xffffffffu, v[k], s);
        v[k] = hi ? other - v[k] : v[k] + other;
      }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) acc += (uint32_t)abs(v[k]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return (acc + 4u) >> 3;  // dist.rs:219-220 (8x8 chunks: ln = 3), one rounding for the block
}

// SATD of a block with a side below 8: 4x4 chunks (dist.rs:166-167), at most four of them (16x4, 4x16),
// one lane per chunk with the whole 2-D Hadamard in its registers
template <typename T, int W, int H>
__device__ __forceinline__ uint32_t warp_satd4(const T *org, int os, const T *pred, int lane) {
  constexpr int NCH = (W / 4) * (H / 4);
  static_assert(NCH <= 32, "one lane per 4x4 chunk");
  uint32_t acc = 0;
  if (lane < NCH) {
    const int cy = (lane / (W / 4)) * 4, cx = (lane % (W / 4)) * 4;
    int d[16];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
      for (int k = 0; k < 4; k++) d[r * 4 + k] = (int)org[(long long)(cy + r) * os + cx + k] - (int)pred[(cy + r) * W + cx + k];
    acc = hadamard4x4_abs_sum(d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return (acc + 2u) >> 2;  // dist.rs:219-220 (4x4 chunks: ln = 2)
}

template <typename T, int W, int H>
__device__ __forceinline__ uint32_t block_satd(const T *org, int os, const T *pred, int lane) {
  if constexpr (W < 8 || H < 8)
    return warp_satd4<T, W, H>(org, os, pred, lane);
  else
    return warp_satd<T, W, H>(org, os, pred, lane);
}

}  // namespace
