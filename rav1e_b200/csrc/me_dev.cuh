// me_dev.cuh — device primitives of the motion-estimation kernels: the empty-result sentinels, packed
// 8-bit SAD and SATD steps, the mv-range test, the block's mv predictors, the packed first-minimum key
// with its warp minimum and result epilogue, (cost, index) reductions, and the distortion of a block of
// any size.  Used by the candidate-list kernels (me_cand.cu, me_chunk.cu), the full search
// (me_full_search.cu), the search stages (me_search_dev.cuh) and the fused sub-pel RDO (subpel_rdo.cu).
#pragma once

#include <cuda_runtime.h>

#include "common.cuh"
#include "hadamard.cuh"

namespace {

constexpr unsigned long long kEmptyCost = ~0ull;  // MVCandidateRD::empty(), me.rs:139-146
constexpr uint32_t kEmptySad = ~0u;

// VABSDIFF4.U8.ACC with the accumulator fused (nvcc's __vsadu4(a,b)+c emits a separate IADD3).
__device__ __forceinline__ uint32_t sad4_acc(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// d = sum_i a.u8[i] * b.s8[i] + c   (IDP.4A.U8.S8)
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Row of W pixels at byte offset `off` (arbitrary alignment) inside a word-addressed shared
// window row; org row as W/4 packed words.  Returns sum |org - ref| over the row.
template <int W>
__device__ __forceinline__ uint32_t row_sad_u8(const uint32_t *__restrict__ wrow, int word0,
                                               int shift_bits, const uint32_t *__restrict__ orow,
                                               uint32_t acc) {
  uint32_t lo = wrow[word0];
#pragma unroll
  for (int k = 0; k < W / 4; k++) {
    const uint32_t hi = wrow[word0 + k + 1];
    const uint32_t v = __funnelshift_r(lo, hi, shift_bits);
    acc = sad4_acc(v, orow[k], acc);
    lo = hi;
  }
  return acc;
}

// get_fullpel_mv_rd's range test (me.rs:1392-1398): the vector lies outside get_mv_range's bounds `r`.
// A macro rather than an inline function: nvcc orders the compares of the function form differently
// in the kernels that test it (same results, different and in places larger machine code).
#define B200_MV_OUTSIDE(mv_row, mv_col, r) \
  ((mv_col) < (r).x_min || (mv_col) > (r).x_max || (mv_row) < (r).y_min || (mv_row) > (r).y_max)

// The block's two mv predictors from a table of 4 shorts per block (row0, col0, row1, col1); zero
// without a table.
struct Pmv {
  int r0, c0, r1, c1;
};
__device__ __forceinline__ Pmv load_pmv(const short *pmv, size_t blk) {
  Pmv p{0, 0, 0, 0};
  if (pmv) {
    const short *q = pmv + 4 * blk;
    p.r0 = q[0], p.c0 = q[1], p.r1 = q[2], p.c1 = q[3];
  }
  return p;
}

// Packed first-minimum key: cost << 24 | index of the candidate inside its block.  cost < 2^39 always
// (256*sad <= 2^34 for 128x128x12 bit, rate <= 64, lambda < 2^32), so the key orders exactly like
// (cost, index): the first minimum in list order.  An empty candidate is ~0.
constexpr int kKeyIdxBits = 24;
__device__ __forceinline__ unsigned long long pack_key(unsigned long long cost, uint32_t idx) {
  return cost == kEmptyCost ? ~0ull : ((cost << kKeyIdxBits) | idx);
}

// The warp's minimum key, in every lane: REDUX is 32 bits wide, so the high words first, then the low
// words of the lanes that hold the high minimum.
__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long key) {
  const uint32_t khi = (uint32_t)(key >> 32);
  const uint32_t mh = __reduce_min_sync(0xffffffffu, khi);
  const uint32_t klo = khi == mh ? (uint32_t)key : 0xffffffffu;
  const uint32_t ml = __reduce_min_sync(0xffffffffu, klo);
  return ((unsigned long long)mh << 32) | ml;
}

// Lexicographic (cost, index) min == "first minimum in scan order" (me.rs:898, :1501).
struct CostIdx {
  unsigned long long cost;
  uint32_t idx;
};
__device__ __forceinline__ CostIdx best_min(CostIdx a, CostIdx b) {
  return (b.cost < a.cost || (b.cost == a.cost && b.idx < a.idx)) ? b : a;
}
__device__ __forceinline__ CostIdx warp_best(CostIdx v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    CostIdx t;
    t.cost = __shfl_xor_sync(0xffffffffu, v.cost, o);
    t.idx = __shfl_xor_sync(0xffffffffu, v.idx, o);
    v = best_min(v, t);
  }
  return v;
}
// Block-wide reduction; result valid in thread 0.  `red` holds >= 32 entries.
__device__ __forceinline__ CostIdx block_best(CostIdx v, CostIdx *red) {
  v = warp_best(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    CostIdx t = lane < nw ? red[lane] : CostIdx{kEmptyCost, 0xffffffffu};
    v = warp_best(t);
  }
  return v;
}

// Warp-cooperative distortion of one w x h block pair (any size).  All 32 lanes call it
// with the same arguments; every lane returns the final value.
template <typename T>
__device__ uint32_t warp_block_dist(const T *org, int os, const T *ref, int rs, int w, int h,
                                    int use_satd, int lane) {
  if (!use_satd) {
    uint32_t s = 0;
    const int n = w * h;
    for (int i = lane; i < n; i += 32) {
      int y = i / w, x = i - y * w;
      int d = (int)org[(long long)y * os + x] - (int)ref[(long long)y * rs + x];
      s += (uint32_t)abs(d);
    }
    return warp_sum_u32(s);
  }
  // dist.rs:166: size = min(w, h, 8): 4x4 transform when either side is 4, else 8x8
  const int size = min(min(w, h), 8);
  const int nx = (w + size - 1) / size, ny = (h + size - 1) / size;
  unsigned long long sum = 0;
  for (int c = lane; c < nx * ny; c += 32) {
    const int cy = (c / nx) * size, cx = (c % nx) * size;
    const int cw = min(size, w - cx), ch = min(size, h - cy);
    const T *o = org + (long long)cy * os + cx;
    const T *r = ref + (long long)cy * rs + cx;
    if (cw != size || ch != size) {  // dist.rs:185-191: partial chunk -> SAD
      uint32_t s = 0;
      for (int y = 0; y < ch; y++)
        for (int x = 0; x < cw; x++)
          s += (uint32_t)abs((int)o[(long long)y * os + x] - (int)r[(long long)y * rs + x]);
      sum += s;
    } else if (size == 4) {
      int d[16];
#pragma unroll
      for (int y = 0; y < 4; y++)
#pragma unroll
        for (int x = 0; x < 4; x++)
          d[y * 4 + x] = (int)o[(long long)y * os + x] - (int)r[(long long)y * rs + x];
      sum += hadamard4x4_abs_sum(d);
    } else {
      int d[64];
#pragma unroll
      for (int y = 0; y < 8; y++)
#pragma unroll
        for (int x = 0; x < 8; x++)
          d[y * 8 + x] = (int)o[(long long)y * os + x] - (int)r[(long long)y * rs + x];
      sum += hadamard8x8_abs_sum(d);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const int ln = size == 4 ? 2 : 3;  // msb(size)
  return (uint32_t)((sum + ((1ull << ln) >> 1)) >> ln);
}

}  // namespace
