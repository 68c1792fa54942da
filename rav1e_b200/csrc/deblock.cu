// deblock.cu — the deblocking filter (rav1e src/deblock.rs) for lists of items: the level search
// (sse_optimize, deblock.rs:1553-1617) and the edge filter (deblock_filter_frame -> deblock_plane,
// :1292-1551).  An item is the TileBlocks rect of one call site: the frame, a tile or a loop-restoration
// area; edges are found on the item's own grid.
//
// Both kernels run one 256-thread CTA per (64x64 luma tile of an item, plane).
//  - Level search: a work unit is one 4-pixel edge segment of one direction.  Its four lines read `rec` and
//    `src` from global memory and add their none / narrow / wide SSE deltas at their threshold levels to
//    per-direction tallies in shared memory (i64 atomics), which are flushed to a per-item tally in the
//    context's scratch.  Integer sums do not depend on order, so the result is exact.  A finish kernel takes
//    the prefix sums and the first minimum per item.
//  - Filter: the tile plus a 7-pixel halo is staged in shared memory; every vertical edge line of the staged
//    rows is filtered in place, then (after a barrier) every horizontal edge line of the tile's columns,
//    then the tile is written.  Within one direction no two edges of a consistent block grid touch the same
//    pixels, and a horizontal edge reads only rows whose vertical edges are done, so this equals the
//    reference's lagged order (tests/test_oracle_deblock_spec.py carries that argument).
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

constexpr int kDbThreads = 256;
constexpr int kDbMaxItems = 160;  // items per launch (kernel-parameter table)
constexpr int kHalo = 7;
constexpr int kStage = 64 + 2 * kHalo;  // staged tile side (luma; chroma tiles use part of it)
constexpr int kMaxLevel = 63;

// BlockSize width / height in 4x4 units, TxSize width / height in 4x4 units (partition.rs:130-153,
// transform/mod.rs:101-123), subsampled_size (partition.rs:337-379; -1 = invalid, read as 4x4) and
// max_txsize_rect_lookup (context/transform_unit.rs:60-83) with av1_get_coded_tx_size folded in.
__constant__ uint8_t kBlkW[22] = {1, 1, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 1, 4, 2, 8, 4, 16};
__constant__ uint8_t kBlkH[22] = {1, 2, 1, 2, 4, 2, 4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 4, 1, 8, 2, 16, 4};
__constant__ uint8_t kTxW[19] = {1, 2, 4, 8, 16, 1, 2, 2, 4, 4, 8, 8, 16, 1, 4, 2, 8, 4, 16};
__constant__ uint8_t kTxH[19] = {1, 2, 4, 8, 16, 2, 1, 4, 2, 8, 4, 16, 8, 4, 1, 8, 2, 16, 4};
__constant__ int8_t kSub[3][22] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21},      // 4:4:4
    {0, -1, 0, 1, -1, 3, 4, -1, 6, 7, -1, 9, 10, -1, 12, 13, -1, 2, -1, 5, -1, 8},       // 4:2:2
    {0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 1, 2, 16, 17, 18, 19}};          // 4:2:0
__constant__ uint8_t kChromaTx[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 3, 3, 3, 3, 3, 3, 13, 14, 15, 16, 9, 10};

struct DbArgs {
  PlaneView a[3], b[3];  // level search: rec, src; filter: in, out
  int planes, xdec, ydec, bit_depth;
  const uint8_t *mi;
  int mi_stride;
  const uint8_t *levels_in;  // filter
  uint8_t *levels_out;       // finish
  long long *acc;            // level search: per item x plane x dir x 64, unsummed
  long long *tally;          // finish: prefix-summed copy for the caller, may be NULL
  // b200_deblock_state
  int deltas_enabled, block_deltas_enabled, block_delta_shift, block_delta_multi;
  int8_t ref_deltas[8], mode_deltas[2];
};

// The items of one launch and their 64x64 luma tiles: tile0[k] .. tile0[k + 1] belong to local item k.
struct DbItems {
  uint32_t item0;  // index of local item 0 in the caller's array
  int n;
  int32_t mx[kDbMaxItems], my[kDbMaxItems];  // origin, luma mi
  uint16_t cmi[kDbMaxItems], rmi[kDbMaxItems];  // min(mi_w, ceil(vis_w / 4)), likewise rows
  uint16_t ww[kDbMaxItems], wh[kDbMaxItems];    // working rect, luma px
  uint32_t tile0[kDbMaxItems + 1];
};
static_assert(sizeof(DbArgs) + sizeof(DbItems) <= 4096, "kernel parameters over 4 KB");

struct Mi {
  int bsize, tx, mode, skip, ref0;
  uint32_t deltas;  // Block::deblock_deltas, byte i = deltas[i]
};

__device__ __forceinline__ Mi load_mi(const DbArgs &A, int fx, int fy) {
  const uint8_t *r = A.mi + ((long long)fy * A.mi_stride + fx) * 12;
  Mi m;
  const int bs = __ldg(r), tx = __ldg(r + 1);
  m.bsize = bs < 22 ? bs : 0;  // out-of-range records: the reference panics, any bounded read will do
  m.tx = tx < 19 ? tx : 0;
  m.mode = __ldg(r + 2);
  m.skip = __ldg(r + 3) != 0;
  m.ref0 = (int8_t)__ldg(r + 4);
  m.deltas = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) m.deltas |= (uint32_t)__ldg(r + 5 + i) << (8 * i);
  return m;
}

// largest_chroma_tx_size (partition.rs:385-393)
__device__ __forceinline__ int plane_tx(const Mi &m, int pli, int xdec, int ydec) {
  if (pli == 0) return m.tx;
  int sub = kSub[xdec + ydec][m.bsize];
  return kChromaTx[sub < 0 ? 0 : sub];
}

struct Edge {
  int size;  // 0: no filtered edge here
  Mi blk, prev;
};

// tx-edge test, deblock_left / deblock_up and deblock_size (deblock.rs:71-129) at item-relative luma mi
// (x, y); the size from the transform widths when size_vertical (sse_h_edge passes `true`, :1257)
__device__ __forceinline__ Edge edge_at(const DbArgs &A, int mx, int my, int pli, int xd, int yd, int x, int y,
                                        bool vertical, bool size_vertical) {
  Edge e;
  e.size = 0;
  e.blk = load_mi(A, mx + x, my + y);
  const int tx = plane_tx(e.blk, pli, xd, yd);
  if (vertical ? ((x >> xd) & (kTxW[tx] - 1)) : ((y >> yd) & (kTxH[tx] - 1))) return e;
  e.prev = vertical ? load_mi(A, mx + ((x | xd) - (1 << xd)), my + (y | yd))
                    : load_mi(A, mx + (x | xd), my + ((y | yd) - (1 << yd)));
  const bool block_edge = vertical ? (x & (kBlkW[e.blk.bsize] - 1)) == 0 : (y & (kBlkH[e.blk.bsize] - 1)) == 0;
  if (!(block_edge || !e.blk.skip || !e.prev.skip || e.blk.ref0 == 0 || e.prev.ref0 == 0)) return e;
  const int ptx = plane_tx(e.prev, pli, xd, yd);
  const int n = size_vertical ? kTxW[tx] : kTxH[tx], pn = size_vertical ? kTxW[ptx] : kTxH[ptx];
  e.size = min(pli == 0 ? 14 : 6, min(n, pn) << 2);
  return e;
}

// deblock_adjusted_level (deblock.rs:23-69)
__device__ __forceinline__ int adjusted_level(const DbArgs &A, const uint8_t *lv, const Mi &b, int pli,
                                              bool vertical) {
  const int idx = pli == 0 ? !vertical : pli + 1;
  int level;
  if (A.block_deltas_enabled) {
    const int8_t d = (int8_t)(b.deltas >> (A.block_delta_multi ? 8 * idx : 0));
    const int8_t sum = (int8_t)((int8_t)(d << A.block_delta_shift) + (int8_t)lv[idx]);  // i8 arithmetic
    level = min(max((int)sum, 0), kMaxLevel);
  } else {
    level = lv[idx];
  }
  if (!A.deltas_enabled) return level;
  const int mode_type = b.mode >= 14 && b.mode != 18 && b.mode != 32;  // NEARESTMV, GLOBALMV, GLOBAL_GLOBALMV
  const int l5 = level >> 5;
  const int v = level + A.ref_deltas[b.ref0 & 7] * (1 << l5) + (b.ref0 == 0 ? 0 : A.mode_deltas[mode_type] * (1 << l5));
  return min(max(v, 0), kMaxLevel);
}

// ---------------------------------------------------------------- filters and thresholds (:145-875)
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

__device__ __forceinline__ void narrow(int p1, int p0, int q0, int q1, int shift, bool four, int o[4]) {
  const int lo = -128 * (1 << shift), hi = (128 << shift) - 1, mx = (256 << shift) - 1;
  const int f0 = four ? 0 : clampi(p1 - q1, lo, hi);
  const int f1 = clampi(f0 + 3 * (q0 - p0) + 4, lo, hi) >> 3;
  const int f2 = clampi(f0 + 3 * (q0 - p0) + 3, lo, hi) >> 3;
  const int f3 = (f1 + 1) >> 1;
  o[0] = four ? clampi(p1 + f3, 0, mx) : p1;
  o[1] = clampi(p0 + f2, 0, mx);
  o[2] = clampi(q0 - f1, 0, mx);
  o[3] = four ? clampi(q1 - f3, 0, mx) : q1;
}

__device__ __forceinline__ void wide6(const int *v, int *o) {  // v = p2 .. q2 -> p1 .. q1
  o[0] = (v[0] * 3 + v[1] * 2 + v[2] * 2 + v[3] + 4) >> 3;
  o[1] = (v[0] + v[1] * 2 + v[2] * 2 + v[3] * 2 + v[4] + 4) >> 3;
  o[2] = (v[1] + v[2] * 2 + v[3] * 2 + v[4] * 2 + v[5] + 4) >> 3;
  o[3] = (v[2] + v[3] * 2 + v[4] * 2 + v[5] * 3 + 4) >> 3;
}

__device__ __forceinline__ void wide8(const int *v, int *o) {  // v = p3 .. q3 -> p2 .. q2
  o[0] = (v[0] * 3 + v[1] * 2 + v[2] + v[3] + v[4] + 4) >> 3;
  o[1] = (v[0] * 2 + v[1] + v[2] * 2 + v[3] + v[4] + v[5] + 4) >> 3;
  o[2] = (v[0] + v[1] + v[2] + v[3] * 2 + v[4] + v[5] + v[6] + 4) >> 3;
  o[3] = (v[1] + v[2] + v[3] + v[4] * 2 + v[5] + v[6] + v[7] + 4) >> 3;
  o[4] = (v[2] + v[3] + v[4] + v[5] * 2 + v[6] + v[7] * 2 + 4) >> 3;
  o[5] = (v[3] + v[4] + v[5] + v[6] * 2 + v[7] * 3 + 4) >> 3;
}

// filter_wide14_12 as a running sum: output i (p5 .. q5) = (sum of the 14-tap window with the edge taps
// repeated, each inner tap once more) >> 4
__device__ __forceinline__ void wide14(const int *v, int *o) {  // v = p6 .. q6 -> p5 .. q5
  o[0] = (v[0] * 7 + v[1] * 2 + v[2] * 2 + v[3] + v[4] + v[5] + v[6] + v[7] + 8) >> 4;
  o[1] = (v[0] * 5 + v[1] * 2 + v[2] * 2 + v[3] * 2 + v[4] + v[5] + v[6] + v[7] + v[8] + 8) >> 4;
  o[2] = (v[0] * 4 + v[1] + v[2] * 2 + v[3] * 2 + v[4] * 2 + v[5] + v[6] + v[7] + v[8] + v[9] + 8) >> 4;
  o[3] = (v[0] * 3 + v[1] + v[2] + v[3] * 2 + v[4] * 2 + v[5] * 2 + v[6] + v[7] + v[8] + v[9] + v[10] + 8) >> 4;
  o[4] = (v[0] * 2 + v[1] + v[2] + v[3] + v[4] * 2 + v[5] * 2 + v[6] * 2 + v[7] + v[8] + v[9] + v[10] + v[11] + 8) >> 4;
  o[5] = (v[0] + v[1] + v[2] + v[3] + v[4] + v[5] * 2 + v[6] * 2 + v[7] * 2 + v[8] + v[9] + v[10] + v[11] + v[12] + 8) >> 4;
  o[6] = (v[1] + v[2] + v[3] + v[4] + v[5] + v[6] * 2 + v[7] * 2 + v[8] * 2 + v[9] + v[10] + v[11] + v[12] + v[13] + 8) >> 4;
  o[7] = (v[2] + v[3] + v[4] + v[5] + v[6] + v[7] * 2 + v[8] * 2 + v[9] * 2 + v[10] + v[11] + v[12] + v[13] * 2 + 8) >> 4;
  o[8] = (v[3] + v[4] + v[5] + v[6] + v[7] + v[8] * 2 + v[9] * 2 + v[10] * 2 + v[11] + v[12] + v[13] * 3 + 8) >> 4;
  o[9] = (v[4] + v[5] + v[6] + v[7] + v[8] + v[9] * 2 + v[10] * 2 + v[11] * 2 + v[12] + v[13] * 4 + 8) >> 4;
  o[10] = (v[5] + v[6] + v[7] + v[8] + v[9] + v[10] * 2 + v[11] * 2 + v[12] * 2 + v[13] * 5 + 8) >> 4;
  o[11] = (v[6] + v[7] + v[8] + v[9] + v[10] + v[11] * 2 + v[12] * 2 + v[13] * 7 + 8) >> 4;
}

__device__ __forceinline__ int limit_lv(int limit, int shift) { return (limit + (1 << shift) - 1) >> shift; }
__device__ __forceinline__ int blimit_lv(int p1, int p0, int q0, int q1, int shift) {
  return (((abs(p0 - q0) * 2 + abs(p1 - q1) / 2 + (1 << shift) - 1) >> shift) - 2) / 3;
}
__device__ __forceinline__ int nhev_lv(int p1, int p0, int q0, int q1, int shift) {
  return (max(abs(p1 - p0), abs(q1 - q0)) + (1 << shift) - 1) >> shift << 4;
}

// The thresholds of one line of a SIZE-tap edge, v = the SIZE taps: mask (filter vs none), nhev (narrow2 vs
// narrow4), flat (wide vs narrow) and, for 14, flat14 (wide14 vs wide8).
template <int SIZE>
__device__ __forceinline__ void thresholds(const int *v, int shift, int *mask, int *nhev, bool *flat, bool *flat14) {
  constexpr int P = SIZE == 14 ? 3 : 0;  // p3 inside the 14 taps
  const int fl = 1 << shift;
  const int *c = v + SIZE / 2 - 2;  // p1 p0 q0 q1
  int m = max(abs(c[0] - c[1]), abs(c[3] - c[2]));
  int f = m;
  if (SIZE >= 6) {
    const int *w = v + SIZE / 2 - 3;  // p2 .. q2
    m = max(m, max(abs(w[0] - w[1]), abs(w[5] - w[4])));
    f = max(f, max(abs(w[0] - w[2]), abs(w[5] - w[3])));
  }
  if (SIZE >= 8) {
    const int *w = v + P;  // p3 .. q3
    m = max(m, max(abs(w[0] - w[1]), abs(w[7] - w[6])));
    f = max(f, max(abs(w[0] - w[3]), abs(w[7] - w[4])));
  }
  *mask = max(limit_lv(m, shift), blimit_lv(c[0], c[1], c[2], c[3], shift));
  *nhev = nhev_lv(c[0], c[1], c[2], c[3], shift);
  *flat = SIZE > 4 && f <= fl;
  *flat14 = false;
  if (SIZE == 14)
    *flat14 = max(max(abs(v[2] - v[6]), abs(v[11] - v[7])),
                  max(max(abs(v[1] - v[6]), abs(v[12] - v[7])), max(abs(v[0] - v[6]), abs(v[13] - v[7])))) <= fl;
}

// deblock_size{4,6,8,14}_inner on v[0 .. SIZE) in place
template <int SIZE>
__device__ __forceinline__ void filter_line(int *v, int level, int shift) {
  int mask, nhev;
  bool flat, flat14;
  thresholds<SIZE>(v, shift, &mask, &nhev, &flat, &flat14);
  if (mask > level) return;
  int o[12];
  if (flat) {
    if (SIZE == 6) {
      wide6(v, o);
#pragma unroll
      for (int i = 0; i < 4; i++) v[1 + i] = o[i];
    } else if (SIZE == 8 || !flat14) {
      constexpr int P = SIZE == 14 ? 3 : 0;
      wide8(v + P, o);
#pragma unroll
      for (int i = 0; i < 6; i++) v[P + 1 + i] = o[i];
    } else {
      wide14(v, o);
#pragma unroll
      for (int i = 0; i < 12; i++) v[1 + i] = o[i];
    }
    return;
  }
  constexpr int C = SIZE / 2 - 2;
  narrow(v[C], v[C + 1], v[C + 2], v[C + 3], shift, nhev <= level, o);
#pragma unroll
  for (int i = 0; i < 4; i++) v[C + i] = o[i];
}

// sse_size{4,6,8,14} (:418-1097) for one line: r = rec taps, s = src taps.  Adds tally[0] into *t0 and
// the threshold entries into the shared tallies (entry 64 is never read: the prefix sums stop at 63).
template <int SIZE>
__device__ __forceinline__ void sse_line(const int *r, const int *s, int shift, long long *t0,
                                         unsigned long long *tally) {
  constexpr int NW = SIZE == 4 ? 4 : SIZE == 6 ? 4 : SIZE == 8 ? 6 : 12;  // compared pixels
  constexpr int OFF = SIZE == 4 ? 0 : 1;
  constexpr int C = SIZE / 2 - 2;
  int mask, nhev;
  bool flat, flat14;
  thresholds<SIZE>(r, shift, &mask, &nhev, &flat, &flat14);
  mask = clampi(mask, 1, kMaxLevel + 1);
  nhev = clampi(nhev, mask, kMaxLevel + 1);
  int sse_none = 0;
#pragma unroll
  for (int i = 0; i < NW; i++) {
    const int d = s[OFF + i] - r[OFF + i];
    sse_none += d * d;
  }
  *t0 += sse_none;
  if (mask > kMaxLevel) return;  // every other term lands on entry 64
  int o[12];
  if (flat) {
    int sse_wide = 0;
    if (SIZE == 6) {
      wide6(r, o);
    } else if (SIZE == 8 || !flat14) {
      constexpr int P = SIZE == 14 ? 3 : 0;
      wide8(r + P, o + (SIZE == 14 ? 3 : 0));
      if (SIZE == 14) {
#pragma unroll
        for (int i = 0; i < 3; i++) o[i] = r[1 + i], o[9 + i] = r[10 + i];
      }
    } else {
      wide14(r, o);
    }
#pragma unroll
    for (int i = 0; i < NW; i++) {
      const int d = s[OFF + i] - o[i];
      sse_wide += d * d;
    }
    atomicAdd(tally + mask, (unsigned long long)(long long)(sse_wide - sse_none));
    return;
  }
  // narrow2 / narrow4 change p1 p0 q0 q1 only: the other compared pixels cancel
  int n2 = sse_none, n4 = sse_none;
  int base = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int d = s[C + i] - r[C + i];
    base += d * d;
  }
  if (nhev != mask) {
    narrow(r[C], r[C + 1], r[C + 2], r[C + 3], shift, false, o);
    n2 = sse_none - base;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int d = s[C + i] - o[i];
      n2 += d * d;
    }
  }
  if (nhev <= kMaxLevel) {
    narrow(r[C], r[C + 1], r[C + 2], r[C + 3], shift, true, o);
    n4 = sse_none - base;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int d = s[C + i] - o[i];
      n4 += d * d;
    }
  }
  // tally[mask] += n2 - none; tally[nhev] += n4 - n2 (the same entry when nhev == mask)
  atomicAdd(tally + mask, (unsigned long long)(long long)(n2 - sse_none));
  if (nhev <= kMaxLevel) atomicAdd(tally + nhev, (unsigned long long)(long long)(n4 - n2));
}

template <typename T>
__device__ __forceinline__ int gpx(const PlaneView &p, int x, int y) {
  return (int)*px<T>(p, x, y);
}

// The item, tile and plane of this CTA.
struct TileCtx {
  int k, mx, my, pli, xd, yd, cols, rows, wp, hp, tx0, ty0, tw, th;
};

__device__ __forceinline__ TileCtx tile_ctx(const DbArgs &A, const DbItems &S) {
  TileCtx c;
  const uint32_t t = blockIdx.x;
  int lo = 0, hi = S.n - 1;  // the last k with tile0[k] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (S.tile0[mid] <= t) lo = mid;
    else hi = mid - 1;
  }
  c.k = lo;
  c.pli = blockIdx.y;
  c.xd = c.pli ? A.xdec : 0;
  c.yd = c.pli ? A.ydec : 0;
  c.mx = S.mx[lo];
  c.my = S.my[lo];
  // the plane's edge extent (deblock.rs:1321-1333), in luma mi
  c.cols = (S.cmi[lo] + (1 << c.xd >> 1)) >> c.xd << c.xd;
  c.rows = (S.rmi[lo] + (1 << c.yd >> 1)) >> c.yd << c.yd;
  c.wp = S.ww[lo] >> c.xd;
  c.hp = S.wh[lo] >> c.yd;
  const int ntx = (S.ww[lo] + 63) >> 6;
  const int tl = (int)(t - S.tile0[lo]);
  c.tw = 64 >> c.xd;
  c.th = 64 >> c.yd;
  c.tx0 = (tl % ntx) * c.tw;
  c.ty0 = (tl / ntx) * c.th;
  return c;
}

// ---------------------------------------------------------------- level search
template <typename T>
__global__ void __launch_bounds__(kDbThreads) deblock_sse_kernel(const __grid_constant__ DbArgs A,
                                                                 const __grid_constant__ DbItems S) {
  __shared__ unsigned long long s_t[2][64];
  const TileCtx c = tile_ctx(A, S);
  if (c.pli >= A.planes) return;
  for (int i = threadIdx.x; i < 128; i += kDbThreads) s_t[i >> 6][i & 63] = 0;
  __syncthreads();
  const int shift = A.bit_depth - 8;
  const PlaneView R = A.a[c.pli], Sr = A.b[c.pli];
  const int ox = (c.mx * 4) >> c.xd, oy = (c.my * 4) >> c.yd;
  // segments of this tile: (tw / 4) x (th / 4) positions, two directions
  const int npx = c.tw >> 2, npos = npx * (c.th >> 2);
  long long t0v = 0, t0h = 0;
  for (int w = threadIdx.x; w < 2 * npos; w += kDbThreads) {
    const bool vertical = w < npos;
    const int pos = vertical ? w : w - npos;
    const int sx = (c.tx0 >> 2) + pos % npx, sy = (c.ty0 >> 2) + pos / npx;  // plane 4x4 units
    const int x = sx << c.xd, y = sy << c.yd;                                 // luma mi
    if (x >= c.cols || y >= c.rows || (vertical ? x == 0 : y == 0)) continue;
    const Edge e = edge_at(A, c.mx, c.my, c.pli, c.xd, c.yd, x, y, vertical, true);
    if (!e.size) continue;
    const int px = ox + sx * 4, py = oy + sy * 4;
    unsigned long long *tally = s_t[vertical ? 0 : 1];
    long long acc = 0;
    for (int i = 0; i < 4; i++) {
      int r[14], s[14];
#define DB_LOAD(N)                                                                                   \
  _Pragma("unroll") for (int k = 0; k < N; k++) {                                                    \
    const int xx = vertical ? px - (N / 2) + k : px + i, yy = vertical ? py + i : py - (N / 2) + k; \
    r[k] = gpx<T>(R, xx, yy);                                                                        \
    s[k] = gpx<T>(Sr, xx, yy);                                                                       \
  }
      switch (e.size) {
        case 4: { DB_LOAD(4) sse_line<4>(r, s, shift, &acc, tally); break; }
        case 6: { DB_LOAD(6) sse_line<6>(r, s, shift, &acc, tally); break; }
        case 8: { DB_LOAD(8) sse_line<8>(r, s, shift, &acc, tally); break; }
        default: { DB_LOAD(14) sse_line<14>(r, s, shift, &acc, tally); break; }
      }
#undef DB_LOAD
    }
    if (vertical) t0v += acc;
    else t0h += acc;
  }
#pragma unroll
  for (int d = 0; d < 2; d++) {
    long long v = d ? t0h : t0v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_t[d][0], (unsigned long long)v);
  }
  __syncthreads();
  long long *g = A.acc + ((size_t)(S.item0 + c.k) * 3 + c.pli) * 128;
  for (int i = threadIdx.x; i < 128; i += kDbThreads) {
    const unsigned long long v = s_t[i >> 6][i & 63];
    if (v) atomicAdd((unsigned long long *)(g + i), v);
  }
}

// prefix sums and the first strict minimum (sse_optimize, deblock.rs:1582-1614), one thread per item
__global__ void deblock_levels_finish_kernel(const __grid_constant__ DbArgs A, int n_items) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_items) return;
  uint8_t lv[4] = {0, 0, 0, 0};
  for (int p = 0; p < 3; p++) {
    const long long *g = A.acc + ((size_t)k * 3 + p) * 128;
    long long *t = A.tally ? A.tally + ((size_t)k * 3 + p) * 128 : nullptr;
    long long sv = 0, sh = 0, bvv = 0, bhv = 0, bsv = 0;
    int bv = 0, bh = 0, bs = 0;
    for (int i = 0; i < 64; i++) {
      sv += g[i];
      sh += g[64 + i];
      if (t) t[i] = sv, t[64 + i] = sh;
      if (i == 0 || bvv > sv) bvv = sv, bv = i;
      if (i == 0 || bhv > sh) bhv = sh, bh = i;
      if (i == 0 || bsv > sv + sh) bsv = sv + sh, bs = i;
    }
    if (p >= A.planes) continue;
    if (p == 0) {
      lv[0] = (uint8_t)bv;
      lv[1] = (uint8_t)bh;
    } else {
      lv[p + 1] = (uint8_t)bs;
    }
  }
  for (int i = 0; i < 4; i++) A.levels_out[(size_t)k * 4 + i] = lv[i];
}

// ---------------------------------------------------------------- filter
template <typename T>
__global__ void __launch_bounds__(kDbThreads) deblock_filter_kernel(const __grid_constant__ DbArgs A,
                                                                    const __grid_constant__ DbItems S) {
  __shared__ uint16_t buf[kStage * kStage];
  const TileCtx c = tile_ctx(A, S);
  if (c.pli >= A.planes) return;
  const uint8_t *lv = A.levels_in + (size_t)(S.item0 + c.k) * 4;
  // encoder.rs:3280 / :3598 / rdo.rs:2311 gate all planes on the luma levels; deblock_plane, :1302-1319
  const bool active = (lv[0] | lv[1]) && (c.pli == 0 || lv[c.pli + 1]);
  const int ox = (c.mx * 4) >> c.xd, oy = (c.my * 4) >> c.yd;
  const PlaneView in = A.a[c.pli];
  // staged window: rows / cols [t0 - 7, t0 + tile + 7) of the item, clipped to the working rect
  const int bx = c.tx0 - kHalo, by = c.ty0 - kHalo;
  const int x0 = max(bx, 0), x1 = min(c.tx0 + c.tw + kHalo, c.wp);
  const int y0 = max(by, 0), y1 = min(c.ty0 + c.th + kHalo, c.hp);
  const int sw = x1 - x0;
  if (sw <= 0 || y1 <= y0) return;
  const int nst = sw * (y1 - y0);
  for (int i = threadIdx.x; i < nst; i += kDbThreads) {
    const int y = y0 + i / sw, x = x0 + i % sw;
    buf[(y - by) * kStage + x - bx] = (uint16_t)gpx<T>(in, ox + x, oy + y);
  }
  __syncthreads();
  const int shift = A.bit_depth - 8;
  if (active) {
    // vertical edges at plane columns tx0, tx0 + 4, .., tx0 + tw (edge line per staged row)
    const int ne = (c.tw >> 2) + 1, nl = ne * (y1 - y0);
    for (int w = threadIdx.x; w < nl; w += kDbThreads) {
      const int yy = y0 + w / ne, ex = c.tx0 + 4 * (w % ne);
      const int x = (ex >> 2) << c.xd, y = (yy >> 2) << c.yd;
      if (x == 0 || x >= c.cols || y >= c.rows) continue;
      const Edge e = edge_at(A, c.mx, c.my, c.pli, c.xd, c.yd, x, y, true, true);
      if (!e.size) continue;
      int level = adjusted_level(A, lv, e.blk, c.pli, true);
      if (level == 0) level = adjusted_level(A, lv, e.prev, c.pli, true);
      if (level == 0) continue;
      uint16_t *row = buf + (yy - by) * kStage;
      const int base = ex - (e.size >> 1) - bx;
      int v[14];
#define DB_FILTER(N)                                                                         \
  {                                                                                          \
    _Pragma("unroll") for (int k = 0; k < N; k++) v[k] = row[clampi(base + k, 0, kStage - 1)]; \
    filter_line<N>(v, level, shift);                                                         \
    _Pragma("unroll") for (int k = 0; k < N; k++) row[clampi(base + k, 0, kStage - 1)] = (uint16_t)v[k]; \
  }
      switch (e.size) {
        case 4: DB_FILTER(4) break;
        case 6: DB_FILTER(6) break;
        case 8: DB_FILTER(8) break;
        default: DB_FILTER(14) break;
      }
#undef DB_FILTER
    }
    __syncthreads();
    // horizontal edges at plane rows ty0, ty0 + 4, .., ty0 + th (edge line per tile column)
    const int cx1 = min(c.tx0 + c.tw, c.wp), ncol = cx1 - c.tx0;
    const int nh = (c.th >> 2) + 1, nl2 = nh * max(ncol, 0);
    for (int w = threadIdx.x; w < nl2; w += kDbThreads) {
      const int xx = c.tx0 + w % ncol, ey = c.ty0 + 4 * (w / ncol);
      const int x = (xx >> 2) << c.xd, y = (ey >> 2) << c.yd;
      if (y == 0 || x >= c.cols || y >= c.rows) continue;
      const Edge e = edge_at(A, c.mx, c.my, c.pli, c.xd, c.yd, x, y, false, false);
      if (!e.size) continue;
      int level = adjusted_level(A, lv, e.blk, c.pli, false);
      if (level == 0) level = adjusted_level(A, lv, e.prev, c.pli, false);
      if (level == 0) continue;
      uint16_t *col = buf + xx - bx;
      const int base = ey - (e.size >> 1) - by;
      int v[14];
#define DB_FILTER(N)                                                                                          \
  {                                                                                                           \
    _Pragma("unroll") for (int k = 0; k < N; k++) v[k] = col[clampi(base + k, 0, kStage - 1) * kStage];      \
    filter_line<N>(v, level, shift);                                                                          \
    _Pragma("unroll") for (int k = 0; k < N; k++) col[clampi(base + k, 0, kStage - 1) * kStage] = (uint16_t)v[k]; \
  }
      switch (e.size) {
        case 4: DB_FILTER(4) break;
        case 6: DB_FILTER(6) break;
        case 8: DB_FILTER(8) break;
        default: DB_FILTER(14) break;
      }
#undef DB_FILTER
    }
    __syncthreads();
  }
  // the tile's own pixels of the working rect
  const int wx1 = min(c.tx0 + c.tw, c.wp), wy1 = min(c.ty0 + c.th, c.hp), ow = wx1 - c.tx0;
  if (ow <= 0) return;
  const int no = ow * max(wy1 - c.ty0, 0);
  T *out = (T *)A.b[c.pli].data;
  const int ostride = A.b[c.pli].stride;
  for (int i = threadIdx.x; i < no; i += kDbThreads) {
    const int y = c.ty0 + i / ow, x = c.tx0 + i % ow;
    out[(long long)(oy + y) * ostride + ox + x] = (T)buf[(y - by) * kStage + x - bx];
  }
}

// ---------------------------------------------------------------- host side
struct ItemGeom {
  int wx, wy;    // working rect, luma px
  int cmi, rmi;  // edge extents before decimation, luma mi
};

ItemGeom item_geom(const b200_deblock_item &it) {
  ItemGeom g;
  g.wx = std::min(it.mi_w * 4, (it.vis_w + 7) & ~7);
  g.wy = std::min(it.mi_h * 4, (it.vis_h + 7) & ~7);
  g.cmi = std::min(it.mi_w, (it.vis_w + 3) >> 2);
  g.rmi = std::min(it.mi_h, (it.vis_h + 3) >> 2);
  return g;
}

// Checks shared by both calls: everything but the planes' pixels and the mi records.
int check_common(b200_ctx *ctx, const b200_plane *p0, const b200_plane *p1, int planes, int xdec, int ydec,
                 int bit_depth, const b200_deblock_mi *d_mi, int mi_stride, const b200_deblock_item *items,
                 size_t n_items, int margin) {
  B200_REQUIRE(ctx, p0 && p1 && d_mi && items, "NULL planes / mi / items");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, mi_stride > 0, "mi_stride %d", mi_stride);
  const int bpp = bit_depth == 8 ? 1 : 2;
  for (int p = 0; p < planes; p++)
    for (const b200_plane *pl : {p0, p1}) {
      B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
      B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
      B200_REQUIRE(ctx, pl[p].stride >= pl[p].width && pl[p].pad >= 0, "plane %d: stride %d below its width %d", p,
                   pl[p].stride, pl[p].width);
    }
  struct Rect {
    long long x0, y0, x1, y1;
  };
  std::vector<Rect> rects(n_items);
  for (size_t k = 0; k < n_items; k++) {
    const b200_deblock_item &it = items[k];
    B200_REQUIRE(ctx, it.mi_x >= 0 && it.mi_y >= 0 && it.mi_x % 16 == 0 && it.mi_y % 16 == 0,
                 "item %zu: origin (%d, %d) not on the superblock grid", k, it.mi_x, it.mi_y);
    B200_REQUIRE(ctx, it.mi_w > 0 && it.mi_h > 0 && it.mi_w % 2 == 0 && it.mi_h % 2 == 0,
                 "item %zu: %dx%d 4x4 blocks (empty or odd)", k, it.mi_w, it.mi_h);
    B200_REQUIRE(ctx, it.mi_w < 16384 && it.mi_h < 16384 && (long long)it.mi_x + it.mi_w <= mi_stride,
                 "item %zu: columns %d..%d past mi_stride %d", k, it.mi_x, it.mi_x + it.mi_w, mi_stride);
    B200_REQUIRE(ctx, it.vis_w > 0 && it.vis_h > 0, "item %zu: visible size %dx%d", k, it.vis_w, it.vis_h);
    const ItemGeom g = item_geom(it);
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      const long long x0 = (it.mi_x * 4LL) >> xd, y0 = ((it.mi_y * 4LL) >> yd) - (margin >> yd);
      const long long x1 = x0 + (g.wx >> xd), y1 = ((it.mi_y * 4LL) >> yd) + (g.wy >> yd) + (margin >> yd);
      for (const b200_plane *pl : {p0, p1})
        B200_REQUIRE(ctx, x0 >= -pl[p].pad && y0 >= -pl[p].pad && x1 <= (long long)pl[p].width + pl[p].pad &&
                              y1 <= (long long)pl[p].height + pl[p].pad,
                     "item %zu: plane %d rect outside the %dx%d plane (pad %d)", k, p, pl[p].width, pl[p].height,
                     pl[p].pad);
    }
    rects[k] = Rect{it.mi_x, it.mi_y, (long long)it.mi_x + it.mi_w, (long long)it.mi_y + it.mi_h};
    for (size_t j = 0; j < k; j++)
      B200_REQUIRE(ctx, rects[k].x0 >= rects[j].x1 || rects[j].x0 >= rects[k].x1 || rects[k].y0 >= rects[j].y1 ||
                            rects[j].y0 >= rects[k].y1,
                   "item %zu overlaps item %zu", k, j);
  }
  return B200_OK;
}

// Items in launch-sized groups; run(S, ntiles) launches one group.
template <typename F>
int for_each_group(const b200_deblock_item *items, size_t n_items, F run) {
  DbItems S;
  size_t k = 0;
  while (k < n_items) {
    S.item0 = (uint32_t)k;
    int n = 0;
    uint32_t tiles = 0;
    while (k < n_items && n < kDbMaxItems) {
      const b200_deblock_item &it = items[k];
      const ItemGeom g = item_geom(it);
      S.mx[n] = it.mi_x;
      S.my[n] = it.mi_y;
      S.cmi[n] = (uint16_t)g.cmi;
      S.rmi[n] = (uint16_t)g.rmi;
      S.ww[n] = (uint16_t)g.wx;
      S.wh[n] = (uint16_t)g.wy;
      S.tile0[n] = tiles;
      tiles += (uint32_t)(((g.wx + 63) >> 6) * ((g.wy + 63) >> 6));
      n++, k++;
    }
    S.tile0[n] = tiles;
    S.n = n;
    if (int st = run(S, tiles)) return st;
  }
  return B200_OK;
}

void fill_planes(DbArgs &a, const b200_plane *p0, const b200_plane *p1, int planes) {
  for (int p = 0; p < planes; p++) {
    a.a[p] = PlaneView{p0[p].data, p0[p].stride};
    a.b[p] = PlaneView{p1[p].data, p1[p].stride};
  }
}

}  // namespace

extern "C" int b200_deblock_levels_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int planes,
                                       int xdec, int ydec, int bit_depth, const b200_deblock_mi *d_mi, int mi_stride,
                                       const b200_deblock_item *items, size_t n_items, uint8_t *d_levels,
                                       int64_t *d_tally) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, d_levels != nullptr, "NULL d_levels");
  if (int st = check_common(ctx, rec, src, planes, xdec, ydec, bit_depth, d_mi, mi_stride, items, n_items, 4))
    return st;
  if (n_items == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t acc_bytes = n_items * 3 * 128 * sizeof(long long);
  if (int st = b200_reserve_dwork(ctx, acc_bytes)) return st;
  B200_CUDA(ctx, cudaMemsetAsync(ctx->dwork, 0, acc_bytes, ctx->stream));
  DbArgs a{};
  fill_planes(a, rec, src, planes);
  a.planes = planes;
  a.xdec = xdec;
  a.ydec = ydec;
  a.bit_depth = bit_depth;
  a.mi = (const uint8_t *)d_mi;
  a.mi_stride = mi_stride;
  a.acc = (long long *)ctx->dwork;
  a.levels_out = d_levels;
  a.tally = (long long *)d_tally;
  const bool hbd = bit_depth > 8;
  if (int st = for_each_group(items, n_items, [&](const DbItems &S, uint32_t tiles) {
        const dim3 grid(tiles, planes);
        if (hbd) deblock_sse_kernel<uint16_t><<<grid, kDbThreads, 0, ctx->stream>>>(a, S);
        else deblock_sse_kernel<uint8_t><<<grid, kDbThreads, 0, ctx->stream>>>(a, S);
        B200_LAUNCH_CHECK(ctx);
        return (int)B200_OK;
      }))
    return st;
  deblock_levels_finish_kernel<<<(unsigned)((n_items + 127) / 128), 128, 0, ctx->stream>>>(a, (int)n_items);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_deblock_filter_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out, int planes,
                                       int xdec, int ydec, int bit_depth, const b200_deblock_state *state,
                                       const uint8_t *d_levels, const b200_deblock_mi *d_mi, int mi_stride,
                                       const b200_deblock_item *items, size_t n_items) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, state && d_levels, "NULL state / d_levels");
  B200_REQUIRE(ctx, state->block_delta_shift <= 3, "block_delta_shift %d above 3", state->block_delta_shift);
  if (int st = check_common(ctx, in, out, planes, xdec, ydec, bit_depth, d_mi, mi_stride, items, n_items, 0))
    return st;
  for (int p = 0; p < planes; p++)
    for (int r = 0; r < planes; r++)
      B200_REQUIRE(ctx, out[p].data != in[r].data, "out plane %d aliases in plane %d", p, r);
  if (n_items == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  DbArgs a{};
  fill_planes(a, in, out, planes);
  a.planes = planes;
  a.xdec = xdec;
  a.ydec = ydec;
  a.bit_depth = bit_depth;
  a.mi = (const uint8_t *)d_mi;
  a.mi_stride = mi_stride;
  a.levels_in = d_levels;
  a.deltas_enabled = state->deltas_enabled != 0;
  a.block_deltas_enabled = state->block_deltas_enabled != 0;
  a.block_delta_shift = state->block_delta_shift;
  a.block_delta_multi = state->block_delta_multi != 0;
  for (int i = 0; i < 8; i++) a.ref_deltas[i] = state->ref_deltas[i];
  for (int i = 0; i < 2; i++) a.mode_deltas[i] = state->mode_deltas[i];
  const bool hbd = bit_depth > 8;
  return for_each_group(items, n_items, [&](const DbItems &S, uint32_t tiles) {
    const dim3 grid(tiles, planes);
    if (hbd) deblock_filter_kernel<uint16_t><<<grid, kDbThreads, 0, ctx->stream>>>(a, S);
    else deblock_filter_kernel<uint8_t><<<grid, kDbThreads, 0, ctx->stream>>>(a, S);
    B200_LAUNCH_CHECK(ctx);
    return (int)B200_OK;
  });
}
