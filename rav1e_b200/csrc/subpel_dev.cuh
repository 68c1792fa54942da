// subpel_dev.cuh — get_subpel_mv_rd (me.rs:1411-1442) of one block and subpel_diamond_search's move-to-best
// loop (me.rs:1311-1383), one warp per block, shared by the fused sub-pel RDO (subpel_rdo.cu) and the
// encode-time motion search (encode_me.cu).  A candidate's (W + 7) x (H + 7) reference footprint is staged in
// shared memory, the 8-tap prediction formed there and measured against the source block with SAD or SATD.
#pragma once

#include <cuda_runtime.h>

#include "mc_dev.cuh"
#include "me_dev.cuh"
#include "warp_satd.cuh"

namespace {

template <typename T, int W, int H>
__device__ __forceinline__ uint32_t warp_sad(const T *org, int os, const T *pred, int lane) {
  uint32_t acc = 0;
#pragma unroll 4
  for (int i = lane; i < W * H; i += 32) {
    const int r = i / W, c = i - r * W;
    acc += (uint32_t)abs((int)org[(long long)r * os + c] - (int)pred[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// One block's sub-pel evaluation context.  tile / inter: the warp's McLayout<T, W, H> staging buffers.
template <typename T, int W, int H>
struct SubpelBlock {
  const T *org;  // block pixel (0,0) in the source
  int org_stride;
  const T *ref;  // reference pixel (0,0)
  int ref_stride;
  int x, y;  // block position, px
  MvRange rng;
  Pmv pm;
  uint32_t lambda;
  int allow_hp, use_satd, bit_depth, xb, yb;  // xb / yb: filter banks of fi.default_filter
  T *tile;
  short *inter;

  // get_subpel_mv_rd of one vector: prediction into `pred`, distortion into `sad`, the cost returned
  __device__ __forceinline__ unsigned long long rd(int mv_row, int mv_col, T *pred, uint32_t &sad, int lane) const {
    sad = kEmptySad;
    if (B200_MV_OUTSIDE(mv_row, mv_col, rng)) return kEmptyCost;
    // predict.rs:284-297 get_mv_params (luma)
    const int y0 = y + (mv_row >> 3), x0 = x + (mv_col >> 3);
    const int row_frac = (int)(((unsigned)mv_row << 1) & 0xf), col_frac = (int)(((unsigned)mv_col << 1) & 0xf);
    const T *src = ref + (long long)(y0 - 3) * ref_stride + (x0 - 3);
    __syncwarp();
    mc_stage_tile<T, W, H>(tile, src, ref_stride, lane);
    __syncwarp();
    mc_put_warp<T, W, H>(tile, inter, pred, xb, col_frac, yb, row_frac, bit_depth, lane);
    __syncwarp();
    sad = use_satd ? block_satd<T, W, H>(org, org_stride, pred, lane) : warp_sad<T, W, H>(org, org_stride, pred, lane);
    return b200_mv_cost(sad, mv_row, mv_col, pm.r0, pm.c0, pm.r1, pm.c1, lambda, allow_hp);
  }

  // subpel_diamond_search, me.rs:1311-1383: move to the best of the four diamond points while one is strictly
  // better, then halve the radius (1/2 pel down to 1/4, or 1/8 with high precision).  (cost, sad, row, col)
  // is the running result, in and out; `pred` is scratch.
  __device__ __forceinline__ void diamond(unsigned long long &best_cost, uint32_t &best_sad, int &best_row,
                                          int &best_col, T *pred, int lane) const {
    int radius_log2 = 2;
    const int end_log2 = allow_hp ? 0 : 1;
    for (;;) {
      unsigned long long cc = kEmptyCost;
      uint32_t cs = kEmptySad;
      int cr = 0, ccol = 0;
#pragma unroll 1
      for (int k = 0; k < 4; k++) {  // DIAMOND_R1_PATTERN_SUBPEL, me.rs:931-934: row+1, col+1, row-1, col-1
        const int dr = (k == 0) - (k == 2), dc = (k == 1) - (k == 3);
        const int mr = (short)(best_row + (short)(dr << radius_log2)), mc = (short)(best_col + (short)(dc << radius_log2));
        uint32_t s;
        const unsigned long long cost = rd(mr, mc, pred, s, lane);
        if (cost < cc) cc = cost, cs = s, cr = mr, ccol = mc;
      }
      if (best_cost <= cc) {
        if (radius_log2 == end_log2) break;
        radius_log2--;
      } else {
        best_cost = cc, best_sad = cs, best_row = cr, best_col = ccol;
      }
    }
  }
};

}  // namespace
