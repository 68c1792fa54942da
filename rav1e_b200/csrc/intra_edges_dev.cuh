// intra_edges_dev.cuh — get_intra_edges (rav1e src/partition.rs:639-898) for one transform block,
// evaluated by a group of threads: shared by the batched edge kernel (intra_edges.cu) and the intra
// mode screening (intra_screen.cu).
//
//   has_top_right / has_bottom_left     src/recon_intra.rs:174-255, :374-452
//   supersample_chroma_bsize            src/partition.rs:559-598
//
// Every entry of the 257-entry IntraEdge buffer is a closed-form function of its index: thread k
// computes "which plane pixel (or which documented constant) does entry k hold" directly, including
// the replication of the last available pixel into the unavailable part of each segment, so there is
// no dependent chain inside a buffer.  The has_tr_* / has_bl_* availability bitmaps
// (recon_intra.rs:30-136, :258-354) are not stored: the bit is computed from the rule the tables
// encode (Z-order of the 4x4 units of a 128x128 superblock; checked table by table against the
// reference's digests on the oracle side, which uses the same rule independently written).
#pragma once

#include "common.cuh"

namespace intra_edges {

static __constant__ unsigned char kBsW[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64};
static __constant__ unsigned char kBsH[22] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16};
// transform/mod.rs:101-123
static __constant__ unsigned char kTxW[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
static __constant__ unsigned char kTxH[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
static __constant__ short kModeAngle[9] = {0, 90, 180, 45, 135, 113, 157, 203, 67};  // predict.rs:138-150

__device__ __forceinline__ unsigned morton6(unsigned x, unsigned y) {
  unsigned m = 0;
#pragma unroll
  for (int b = 0; b < 6; b++) m |= ((x >> b) & 1u) << (2 * b) | ((y >> b) & 1u) << (2 * b + 1);
  return m;
}

// bit (blk_row, blk_col) of has_tr_<bsize> (kind 0) / has_bl_<bsize> (kind 1)
__device__ inline int avail_bit(int kind, int bw, int bh, int br, int bc) {
  const int S = max(bw, bh);
  const int x = bc * bw, y = br * bh, ox = x % S, oy = y % S, tx = x - ox, ty = y - oy;
  if (kind == 0) {
    if (oy > 0) return 0;
    if (ox + bw < S) return 1;
    if (ty == 0) return 1;
    if (tx + S >= 32) return 0;
    return morton6(tx + S, ty - 1) < morton6(tx, ty);
  }
  if (x == 0) return 0;
  if (ox > 0) return 0;
  if (oy + bh < S) return 1;
  if (ty + S >= 32) return 0;
  return morton6(tx - 1, ty + S) < morton6(tx, ty);
}

__device__ __forceinline__ int ilog2(int v) { return 31 - __clz(v); }

// recon_intra.rs:174-255; bw/bh = partition size in pixels (after supersample_chroma_bsize)
__device__ inline int has_top_right(int bw, int bh, int mi_col, int mi_row, int top_avail, int right_avail, int tx_w,
                             int row_off, int col_off, int ss_x, int ss_y) {
  if (!top_avail || !right_avail) return 0;
  const int plane_bw_unit = max((bw >> 2) >> ss_x, 1), cnt = tx_w >> 2;
  if (row_off > 0) {
    if (bw > 64) {
      if (row_off == (16 >> ss_y) && col_off + cnt == (16 >> ss_x)) return 0;
      const int u64w = 16 >> ss_x;
      return col_off % u64w + cnt < u64w;
    }
    return col_off + cnt < plane_bw_unit;
  }
  if (col_off + cnt < plane_bw_unit) return 1;
  const int bwl = ilog2(bw) - 2, bhl = ilog2(bh) - 2;
  const int r = (mi_row & 15) >> bhl, c = (mi_col & 15) >> bwl;
  if (r == 0) return 1;
  if (((c + 1) << bwl) >= 16) return 0;
  return avail_bit(0, bw >> 2, bh >> 2, r, c);
}

// recon_intra.rs:374-452
__device__ inline int has_bottom_left(int bw, int bh, int mi_col, int mi_row, int bottom_avail, int left_avail, int tx_h,
                               int row_off, int col_off, int ss_x, int ss_y) {
  if (!bottom_avail || !left_avail) return 0;
  if (bw > 64 && col_off > 0) {
    const int u64w = 16 >> ss_x;
    if (col_off % u64w == 0) {
      const int u64h = 16 >> ss_y;
      const int plane_bh_unit = min((bh >> 2) >> ss_y, u64h);
      return row_off % u64h + (tx_h >> 2) < plane_bh_unit;
    }
  }
  if (col_off > 0) return 0;
  const int plane_bh_unit = max((bh >> 2) >> ss_y, 1), cnt = tx_h >> 2;
  if (row_off + cnt < plane_bh_unit) return 1;
  const int bwl = ilog2(bw) - 2, bhl = ilog2(bh) - 2;
  const int r = (mi_row & 15) >> bhl, c = (mi_col & 15) >> bwl;
  if (c == 0) return ((r << bhl) >> ss_y) + row_off + cnt < (16 >> ss_y);
  if (((r + 1) << bhl) >= 16) return 0;
  return avail_bit(1, bw >> 2, bh >> 2, r, c);
}

// The region (tile) of the plane the edges are gathered from.
struct EdgeGeom {
  const void *data;  // region pixel (0,0)
  int stride;
  int plane_w, plane_h;  // plane_cfg.width / height
  int rect_x, rect_y, rect_w, rect_h;
  int xdec, ydec, bit_depth;
};

struct EdgeLens {
  int left, above;  // init_left, init_above: the slice lengths IntraEdge::new records
};

// Entries rank, rank + nthreads, ... of item e's IntraEdge buffer into out[0..257) (entries outside
// the initialised slices are zero), the region's pixels read through PX(y, x) (region coordinates).
// Every thread returns the lengths.
template <typename O, typename F>
__device__ __forceinline__ EdgeLens gather_intra_edge_px(const EdgeGeom &a, const b200_edge_item &e, int rank,
                                                         int nthreads, O *out, const F &PX) {
  const int x = e.po_x, y = e.po_y;
  const int tx_w = kTxW[e.tx_size], tx_h = kTxH[e.tx_size];
  const unsigned base = 128u << (a.bit_depth - 8);
  int needs_left = 1, needs_topleft = 1, needs_topright = 1, needs_bottomleft = 1, tl_filter = 0;
  if (e.mode != 255) {  // partition.rs:669-703
    int m = e.mode;
    if (m == 12) m = (x == 0 && y == 0) ? 0 : x == 0 ? 1 : y == 0 ? 2 : 12;
    const int p_angle = (m >= 1 && m <= 8 ? (int)kModeAngle[m] : 0) + (int)e.angle_delta * 3;
    const bool dc_or_cfl = m == 0 || m == 13, directional = m >= 1 && m <= 8;
    needs_left = (!dc_or_cfl || x != 0) || (p_angle > 90 && p_angle != 180);
    needs_topleft = m == 12 || (directional && p_angle != 90 && p_angle != 180);
    // needs_top is true for every mode: `p_angle != 90 && p_angle < 180` holds for the
    // non-directional modes' p_angle = 0 (:695)
    needs_topright = directional && p_angle < 90;
    needs_bottomleft = directional && p_angle > 180;
    tl_filter = e.enable_ief && p_angle > 90 && p_angle < 180;
  }
  const int rw = min(a.rect_w, a.plane_w - a.rect_x), rh = min(a.rect_h, a.plane_h - a.rect_y);
  const int txh = y + tx_h > rh ? rh - y : tx_h, txw = x + tx_w > rw ? rw - x : tx_w;
  const int bx4 = e.bx * (tx_w >> 2), by4 = e.by * (tx_h >> 2);
  const int have_top = by4 != 0 || (a.ydec ? e.part_y > 1 : e.part_y > 0);
  const int have_left = bx4 != 0 || (a.xdec ? e.part_x > 1 : e.part_x > 0);
  const int right_avail = x + tx_w < rw, bottom_avail = y + tx_h < rh;
  // supersample_chroma_bsize, partition.rs:559-598: 4-pixel sides grow to 8 along decimated axes
  int pbw = kBsW[e.bsize], pbh = kBsH[e.bsize];
  {
    const int w0 = pbw, h0 = pbh;
    if (w0 == 4 && a.xdec && (h0 == 4 || h0 == 8 || h0 == 16)) pbw = 8;
    if (h0 == 4 && a.ydec && (w0 == 4 || w0 == 8 || w0 == 16)) pbh = 8;
  }
  int ntr = 0, nbl = 0;
  if (needs_topright && y != 0 &&
      has_top_right(pbw, pbh, e.part_x, e.part_y, have_top, right_avail, tx_w, by4, bx4, a.xdec, a.ydec))
    ntr = min(tx_w, rw - x - tx_w);
  if (needs_bottomleft && x != 0 &&
      has_bottom_left(pbw, pbh, e.part_x, e.part_y, bottom_avail, have_left, tx_h, by4, bx4, a.xdec, a.ydec))
    nbl = min(tx_h, rh - y - tx_h);
  const int init_left = needs_left ? tx_h + (needs_bottomleft ? tx_w : 0) : 0;
  const int init_above = tx_w + (needs_topright ? tx_h : 0);
  // entry i of the left segment (i = 0 next to the top-left pixel, growing downwards)
  auto leftv = [&](int i) -> unsigned {
    if (i >= tx_h) {  // bottom-left: available rows, then the last available one (:835-870)
      const int k = i - tx_h;
      if (k < nbl) return PX(y + tx_h + k, x - 1);
      i = tx_h + nbl - 1;
      if (i >= tx_h) return PX(y + tx_h + nbl - 1, x - 1);
    }
    if (x != 0) return PX(y + min(i, txh - 1), x - 1);  // :711-725
    return y != 0 ? PX(y - 1, 0) : base + 1;            // :726-731
  };
  auto abovev = [&](int j) -> unsigned {
    if (j >= tx_w) {  // top-right (:789-829)
      const int k = j - tx_w;
      if (k < ntr) return PX(y - 1, x + tx_w + k);
      j = tx_w + ntr - 1;
      if (j >= tx_w) return PX(y - 1, x + tx_w + ntr - 1);
    }
    if (y != 0) return PX(y - 1, x + min(j, txw - 1));  // :736-752
    return x != 0 ? PX(0, x - 1) : base - 1;            // :753-758
  };
  for (int idx = rank; idx < 257; idx += nthreads) {
    unsigned v = 0;
    if (idx < 128) {
      const int i = 127 - idx;
      if (i < init_left) v = leftv(i);
    } else if (idx > 128) {
      const int j = idx - 129;
      if (j < init_above) v = abovev(j);
    } else if (needs_topleft) {  // :878-894
      v = (x == 0 && y == 0) ? base : y == 0 ? PX(0, x - 1) : x == 0 ? PX(y - 1, 0) : PX(y - 1, x - 1);
      if (tl_filter && tx_w + tx_h >= 24) v = (leftv(0) * 5 + v * 6 + abovev(0) * 5 + 8u) >> 4;
    } else {
      v = base;
    }
    out[idx] = (O)v;
  }
  return EdgeLens{init_left, init_above};
}

// gather_intra_edge_px over the region of a.data.
template <typename T, typename O>
__device__ EdgeLens gather_intra_edge(const EdgeGeom &a, const b200_edge_item &e, int rank, int nthreads, O *out) {
  const T *reg = (const T *)a.data;
  return gather_intra_edge_px(a, e, rank, nthreads, out,
                              [&](int yy, int xx) -> unsigned { return (unsigned)reg[(long long)yy * a.stride + xx]; });
}

}  // namespace intra_edges
