/*
 * oracle/deblock.c — the deblocking level search and edge filter, item by item, the way rav1e runs them
 * (TEST INFRASTRUCTURE ONLY; see deblock.h for the contract and what pins it).
 */
#include "deblock.h"

#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#define MAX_LOOP_FILTER 63

/* BlockSize (partition.rs:130-153): width / height in 4x4 units */
static const int kBlkW[22] = {1, 1, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 1, 4, 2, 8, 4, 16};
static const int kBlkH[22] = {1, 2, 1, 2, 4, 2, 4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 4, 1, 8, 2, 16, 4};
/* TxSize (transform/mod.rs:101-123): width / height in 4x4 units */
static const int kTxW[19] = {1, 2, 4, 8, 16, 1, 2, 2, 4, 4, 8, 8, 16, 1, 4, 2, 8, 4, 16};
static const int kTxH[19] = {1, 2, 4, 8, 16, 2, 1, 4, 2, 8, 4, 16, 8, 4, 1, 8, 2, 16, 4};
/* BlockSize::subsampled_size (partition.rs:337-379); -1 = InvalidBlockSize */
static const int kSub422[22] = {0, -1, 0, 1, -1, 3, 4, -1, 6, 7, -1, 9, 10, -1, 12, 13, -1, 2, -1, 5, -1, 8};
static const int kSub420[22] = {0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 1, 2, 16, 17, 18, 19};
/* max_txsize_rect_lookup (context/transform_unit.rs:60-83) */
static const int kMaxTx[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18};

/* the fields of one b200_deblock_mi record */
typedef struct {
  int bsize, txsize, mode, skip, ref0;
  int8_t deltas[4];
} Mi;

typedef struct {
  const uint8_t *mi;
  ptrdiff_t stride;
  int mi_x, mi_y; /* item origin: TileBlocks index (x, y) is frame mi (mi_x + x, mi_y + y) */
} Blocks;

static Mi mi_at(const Blocks *b, int x, int y) {
  const uint8_t *r = b->mi + ((ptrdiff_t)(b->mi_y + y) * b->stride + b->mi_x + x) * 12;
  Mi m;
  /* out-of-range values are the reference's panics; any in-range stand-in keeps the oracle defined */
  m.bsize = r[0] < 22 ? r[0] : 0;
  m.txsize = r[1] < 19 ? r[1] : 0;
  m.mode = r[2];
  m.skip = r[3] != 0;
  m.ref0 = (int8_t)r[4];
  memcpy(m.deltas, r + 5, 4);
  return m;
}

/* BlockSize::largest_chroma_tx_size (partition.rs:385-393) with av1_get_coded_tx_size (context/mod.rs:95) */
static int chroma_tx(int bsize, int xdec, int ydec) {
  int sub = xdec && ydec ? kSub420[bsize] : xdec ? kSub422[bsize] : bsize;
  if (sub < 0) sub = 0;
  const int tx = kMaxTx[sub];
  switch (tx) {
    case 4: case 11: case 12: return 3;  /* 64x64, 32x64, 64x32 -> 32x32 */
    case 17: return 9;                   /* 16x64 -> 16x32 */
    case 18: return 10;                  /* 64x16 -> 32x16 */
    default: return tx;
  }
}

static int plane_tx(const Mi *m, int pli, int xdec, int ydec) {
  return pli == 0 ? m->txsize : chroma_tx(m->bsize, xdec, ydec);
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* deblock_adjusted_level (deblock.rs:23-69); levels = the frame's four levels */
static int adjusted_level(const uint8_t *st, const uint8_t *levels, const Mi *b, int pli, int vertical) {
  const int idx = pli == 0 ? !vertical : pli + 1;
  int level;
  if (st[11]) { /* block_deltas_enabled; st[12] = block_delta_shift, st[13] = block_delta_multi */
    const int shift = st[12];
    const int8_t d = st[13] ? b->deltas[idx] : b->deltas[0];
    const int8_t block_delta = (int8_t)(d << shift);            /* i8 << u8 */
    const int8_t sum = (int8_t)(block_delta + (int8_t)levels[idx]); /* i8 + i8 */
    level = clampi(sum, 0, MAX_LOOP_FILTER);
  } else {
    level = levels[idx];
  }
  if (st[0]) { /* deltas_enabled */
    const int mode_type = b->mode >= 14 && b->mode != 18 && b->mode != 32; /* NEARESTMV, GLOBALMV, GLOBAL_GLOBALMV */
    const int l5 = level >> 5;
    const int8_t *ref_deltas = (const int8_t *)st + 1, *mode_deltas = (const int8_t *)st + 9;
    return clampi(level + (ref_deltas[b->ref0 & 7] * (1 << l5)) + (b->ref0 == 0 ? 0 : mode_deltas[mode_type] * (1 << l5)),
                  0, MAX_LOOP_FILTER);
  }
  return level;
}

/* deblock_level (deblock.rs:131-143) */
static int edge_level(const uint8_t *st, const uint8_t *levels, const Mi *b, const Mi *prev, int pli, int vertical) {
  const int level = adjusted_level(st, levels, b, pli, vertical);
  return level == 0 ? adjusted_level(st, levels, prev, pli, vertical) : level;
}

/* The tx-edge test of filter_v_edge / filter_h_edge / sse_*_edge, deblock_left / deblock_up (:71-93) and
 * deblock_size (:94-129).  Returns the filter size (0: not a filtered edge) and the two blocks.  The size
 * takes the transform width when size_vertical, the height otherwise: sse_h_edge passes `true` (:1257). */
static int edge_size(const Blocks *bl, int pli, int xdec, int ydec, int x, int y, int vertical, int size_vertical,
                     Mi *blk, Mi *prev) {
  *blk = mi_at(bl, x, y);
  const int tx = plane_tx(blk, pli, xdec, ydec);
  if (vertical ? ((x >> xdec) & (kTxW[tx] - 1)) : ((y >> ydec) & (kTxH[tx] - 1))) return 0;
  *prev = vertical ? mi_at(bl, (x | xdec) - (1 << xdec), y | ydec) : mi_at(bl, x | xdec, (y | ydec) - (1 << ydec));
  const int block_edge = vertical ? (x & (kBlkW[blk->bsize] - 1)) == 0 : (y & (kBlkH[blk->bsize] - 1)) == 0;
  if (!(block_edge || !blk->skip || !prev->skip || blk->ref0 == 0 || prev->ref0 == 0)) return 0;
  const int ptx = plane_tx(prev, pli, xdec, ydec);
  const int n = size_vertical ? kTxW[tx] : kTxH[tx], pn = size_vertical ? kTxW[ptx] : kTxH[ptx];
  const int m = (n < pn ? n : pn) << 2;
  const int cap = pli == 0 ? 14 : 6;
  return m < cap ? m : cap;
}

/* ---------------------------------------------------------------- the filters (deblock.rs:145-306) */
static void narrow2_4(int p1, int p0, int q0, int q1, int shift, int *o) {
  const int lo = -128 * (1 << shift), hi = (128 << shift) - 1, mx = (256 << shift) - 1;
  const int f0 = clampi(p1 - q1, lo, hi);
  const int f1 = clampi(f0 + 3 * (q0 - p0) + 4, lo, hi) >> 3;
  const int f2 = clampi(f0 + 3 * (q0 - p0) + 3, lo, hi) >> 3;
  o[0] = p1;
  o[1] = clampi(p0 + f2, 0, mx);
  o[2] = clampi(q0 - f1, 0, mx);
  o[3] = q1;
}

static void narrow4_4(int p1, int p0, int q0, int q1, int shift, int *o) {
  const int lo = -128 * (1 << shift), hi = (128 << shift) - 1, mx = (256 << shift) - 1;
  const int f1 = clampi(3 * (q0 - p0) + 4, lo, hi) >> 3;
  const int f2 = clampi(3 * (q0 - p0) + 3, lo, hi) >> 3;
  const int f3 = (f1 + 1) >> 1;
  o[0] = clampi(p1 + f3, 0, mx);
  o[1] = clampi(p0 + f2, 0, mx);
  o[2] = clampi(q0 - f1, 0, mx);
  o[3] = clampi(q1 - f3, 0, mx);
}

static void wide6_4(const int *v, int *o) { /* v = p2 p1 p0 q0 q1 q2 */
  const int p2 = v[0], p1 = v[1], p0 = v[2], q0 = v[3], q1 = v[4], q2 = v[5];
  o[0] = (p2 * 3 + p1 * 2 + p0 * 2 + q0 + 4) >> 3;
  o[1] = (p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1 + 4) >> 3;
  o[2] = (p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2 + 4) >> 3;
  o[3] = (p0 + q0 * 2 + q1 * 2 + q2 * 3 + 4) >> 3;
}

static void wide8_6(const int *v, int *o) { /* v = p3 .. q3 */
  const int p3 = v[0], p2 = v[1], p1 = v[2], p0 = v[3], q0 = v[4], q1 = v[5], q2 = v[6], q3 = v[7];
  o[0] = (p3 * 3 + p2 * 2 + p1 + p0 + q0 + 4) >> 3;
  o[1] = (p3 * 2 + p2 + p1 * 2 + p0 + q0 + q1 + 4) >> 3;
  o[2] = (p3 + p2 + p1 + p0 * 2 + q0 + q1 + q2 + 4) >> 3;
  o[3] = (p2 + p1 + p0 + q0 * 2 + q1 + q2 + q3 + 4) >> 3;
  o[4] = (p1 + p0 + q0 + q1 * 2 + q2 + q3 * 2 + 4) >> 3;
  o[5] = (p0 + q0 + q1 + q2 * 2 + q3 * 3 + 4) >> 3;
}

static void wide14_12(const int *v, int *o) { /* v = p6 .. q6 */
  const int p6 = v[0], p5 = v[1], p4 = v[2], p3 = v[3], p2 = v[4], p1 = v[5], p0 = v[6];
  const int q0 = v[7], q1 = v[8], q2 = v[9], q3 = v[10], q4 = v[11], q5 = v[12], q6 = v[13];
  o[0] = (p6 * 7 + p5 * 2 + p4 * 2 + p3 + p2 + p1 + p0 + q0 + 8) >> 4;
  o[1] = (p6 * 5 + p5 * 2 + p4 * 2 + p3 * 2 + p2 + p1 + p0 + q0 + q1 + 8) >> 4;
  o[2] = (p6 * 4 + p5 + p4 * 2 + p3 * 2 + p2 * 2 + p1 + p0 + q0 + q1 + q2 + 8) >> 4;
  o[3] = (p6 * 3 + p5 + p4 + p3 * 2 + p2 * 2 + p1 * 2 + p0 + q0 + q1 + q2 + q3 + 8) >> 4;
  o[4] = (p6 * 2 + p5 + p4 + p3 + p2 * 2 + p1 * 2 + p0 * 2 + q0 + q1 + q2 + q3 + q4 + 8) >> 4;
  o[5] = (p6 + p5 + p4 + p3 + p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1 + q2 + q3 + q4 + q5 + 8) >> 4;
  o[6] = (p5 + p4 + p3 + p2 + p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2 + q3 + q4 + q5 + q6 + 8) >> 4;
  o[7] = (p4 + p3 + p2 + p1 + p0 + q0 * 2 + q1 * 2 + q2 * 2 + q3 + q4 + q5 + q6 * 2 + 8) >> 4;
  o[8] = (p3 + p2 + p1 + p0 + q0 + q1 * 2 + q2 * 2 + q3 * 2 + q4 + q5 + q6 * 3 + 8) >> 4;
  o[9] = (p2 + p1 + p0 + q0 + q1 + q2 * 2 + q3 * 2 + q4 * 2 + q5 + q6 * 4 + 8) >> 4;
  o[10] = (p1 + p0 + q0 + q1 + q2 + q3 * 2 + q4 * 2 + q5 * 2 + q6 * 5 + 8) >> 4;
  o[11] = (p0 + q0 + q1 + q2 + q3 + q4 * 2 + q5 * 2 + q6 * 7 + 8) >> 4;
}

/* ---------------------------------------------------------------- thresholds (deblock.rs:333-362, 363-374, ...) */
static int iabs(int v) { return v < 0 ? -v : v; }
static int imax(int a, int b) { return a > b ? a : b; }
static int limit_to_level(int limit, int shift) { return (limit + (1 << shift) - 1) >> shift; }
static int blimit_to_level(int blimit, int shift) { return (((blimit + (1 << shift) - 1) >> shift) - 2) / 3; }
static int thresh_to_level(int thresh, int shift) { return (thresh + (1 << shift) - 1) >> shift << 4; }

static int nhev4(int p1, int p0, int q0, int q1, int shift) {
  return thresh_to_level(imax(iabs(p1 - p0), iabs(q1 - q0)), shift);
}
static int blimit_lv(int p1, int p0, int q0, int q1, int shift) {
  return blimit_to_level(iabs(p0 - q0) * 2 + iabs(p1 - q1) / 2, shift);
}
static int mask4(const int *v, int shift) { /* p1 p0 q0 q1 */
  return imax(limit_to_level(imax(iabs(v[0] - v[1]), iabs(v[3] - v[2])), shift), blimit_lv(v[0], v[1], v[2], v[3], shift));
}
static int mask6(const int *v, int shift) { /* p2 .. q2 */
  const int m = imax(imax(iabs(v[0] - v[1]), iabs(v[1] - v[2])), imax(iabs(v[5] - v[4]), iabs(v[4] - v[3])));
  return imax(limit_to_level(m, shift), blimit_lv(v[1], v[2], v[3], v[4], shift));
}
static int flat6(const int *v) {
  return imax(imax(iabs(v[1] - v[2]), iabs(v[4] - v[3])), imax(iabs(v[0] - v[2]), iabs(v[5] - v[3])));
}
static int mask8(const int *v, int shift) { /* p3 .. q3 */
  const int m = imax(imax(iabs(v[0] - v[1]), imax(iabs(v[1] - v[2]), iabs(v[2] - v[3]))),
                     imax(iabs(v[7] - v[6]), imax(iabs(v[6] - v[5]), iabs(v[5] - v[4]))));
  return imax(limit_to_level(m, shift), blimit_lv(v[2], v[3], v[4], v[5], shift));
}
static int flat8(const int *v) {
  return imax(imax(iabs(v[2] - v[3]), iabs(v[5] - v[4])),
              imax(imax(iabs(v[1] - v[3]), iabs(v[6] - v[4])), imax(iabs(v[0] - v[3]), iabs(v[7] - v[4]))));
}
static int flat14_outer(const int *v) { /* v = p6 .. q6 */
  return imax(imax(iabs(v[2] - v[6]), iabs(v[11] - v[7])),
              imax(imax(iabs(v[1] - v[6]), iabs(v[12] - v[7])), imax(iabs(v[0] - v[6]), iabs(v[13] - v[7]))));
}

/* deblock_size{4,6,8,14}_inner (:376-390, :498-515, :669-686, :845-875) on one line v[0 .. size) in place */
static void filter_line(int *v, int size, int level, int bd) {
  const int shift = bd - 8, flat = 1 << shift;
  int o[12];
  switch (size) {
    case 4:
      if (mask4(v, shift) > level) return;
      if (nhev4(v[0], v[1], v[2], v[3], shift) <= level) narrow4_4(v[0], v[1], v[2], v[3], shift, o);
      else narrow2_4(v[0], v[1], v[2], v[3], shift, o);
      memcpy(v, o, 4 * sizeof(int));
      return;
    case 6:
      if (mask6(v, shift) > level) return;
      if (flat6(v) <= flat) wide6_4(v, o);
      else if (nhev4(v[1], v[2], v[3], v[4], shift) <= level) narrow4_4(v[1], v[2], v[3], v[4], shift, o);
      else narrow2_4(v[1], v[2], v[3], v[4], shift, o);
      memcpy(v + 1, o, 4 * sizeof(int));
      return;
    case 8:
      if (mask8(v, shift) > level) return;
      if (flat8(v) <= flat) {
        wide8_6(v, o);
        memcpy(v + 1, o, 6 * sizeof(int));
        return;
      }
      if (nhev4(v[2], v[3], v[4], v[5], shift) <= level) narrow4_4(v[2], v[3], v[4], v[5], shift, o);
      else narrow2_4(v[2], v[3], v[4], v[5], shift, o);
      memcpy(v + 2, o, 4 * sizeof(int));
      return;
    case 14:
      if (mask8(v + 3, shift) > level) return;
      if (flat8(v + 3) <= flat) {
        if (flat14_outer(v) <= flat) {
          wide14_12(v, o);
          memcpy(v + 1, o, 12 * sizeof(int));
        } else {
          wide8_6(v + 3, o);
          memcpy(v + 4, o, 6 * sizeof(int));
        }
        return;
      }
      if (nhev4(v[5], v[6], v[7], v[8], shift) <= level) narrow4_4(v[5], v[6], v[7], v[8], shift, o);
      else narrow2_4(v[5], v[6], v[7], v[8], shift, o);
      memcpy(v + 5, o, 4 * sizeof(int));
      return;
  }
}

static int get_px(const void *base, ptrdiff_t stride, int bpp, int x, int y) {
  const ptrdiff_t i = (ptrdiff_t)y * stride + x;
  return bpp == 1 ? ((const uint8_t *)base)[i] : ((const uint16_t *)base)[i];
}
static void set_px(void *base, ptrdiff_t stride, int bpp, int x, int y, int v) {
  const ptrdiff_t i = (ptrdiff_t)y * stride + x;
  if (bpp == 1) ((uint8_t *)base)[i] = (uint8_t)v;
  else ((uint16_t *)base)[i] = (uint16_t)v;
}

/* the rows / cols of deblock_plane and sse_plane (:1321-1333, :1470-1482) */
static int extent(int mi_n, int vis, int dec) {
  const int v = (vis + 3) >> 2;
  return ((mi_n < v ? mi_n : v) + (1 << dec >> 1)) >> dec << dec;
}

typedef struct {
  void *p;
  ptrdiff_t stride;
  int bpp, ox, oy; /* item origin in plane pixels */
} Px;

/* filter_v_edge / filter_h_edge (:1099-1143, :1195-1239) */
static void filter_edge(const uint8_t *st, const uint8_t *levels, const Blocks *bl, const Px *P, int pli, int bd,
                        int xdec, int ydec, int x, int y, int vertical) {
  Mi blk, prev;
  const int size = edge_size(bl, pli, xdec, ydec, x, y, vertical, vertical, &blk, &prev);
  if (!size) return;
  const int level = edge_level(st, levels, &blk, &prev, pli, vertical);
  if (level == 0) return;
  const int px = P->ox + ((x * 4) >> xdec), py = P->oy + ((y * 4) >> ydec);
  for (int i = 0; i < 4; i++) {
    int v[14];
    for (int k = 0; k < size; k++)
      v[k] = vertical ? get_px(P->p, P->stride, P->bpp, px - size / 2 + k, py + i)
                      : get_px(P->p, P->stride, P->bpp, px + i, py - size / 2 + k);
    filter_line(v, size, level, bd);
    for (int k = 0; k < size; k++) {
      if (vertical) set_px(P->p, P->stride, P->bpp, px - size / 2 + k, py + i, v[k]);
      else set_px(P->p, P->stride, P->bpp, px + i, py - size / 2 + k, v[k]);
    }
  }
}

/* deblock_plane (:1292-1458), the lagged order taken literally */
static void deblock_plane(const uint8_t *st, const uint8_t *levels, const Px *P, int pli, const Blocks *bl,
                          int mi_w, int mi_h, int vis_w, int vis_h, int bd, int xdec, int ydec) {
  if (pli == 0 && levels[0] == 0 && levels[1] == 0) return;
  if (pli > 0 && levels[pli + 1] == 0) return;
  const int cols = extent(mi_w, vis_w, xdec), rows = extent(mi_h, vis_h, ydec);
  const int sx = 1 << xdec, sy = 1 << ydec;
#define FV(X, Y) filter_edge(st, levels, bl, P, pli, bd, xdec, ydec, (X), (Y), 1)
#define FH(X, Y) filter_edge(st, levels, bl, P, pli, bd, xdec, ydec, (X), (Y), 0)
  if (rows > 0) {
    for (int x = sx; x < cols; x += sx) FV(x, 0);
    if (rows > sy)
      for (int x = sx; x < cols; x += sx) FV(x, sy);
  }
  for (int y = 2 << ydec; y < rows; y += sy) {
    if (cols > sx) FV(sx, y);
    for (int x = 2 << xdec; x < cols; x += sx) {
      FV(x, y);
      FH(x - (2 << xdec), y - sy);
    }
    if (cols >= 2 << xdec) FH(cols - (2 << xdec), y - sy);
    if (cols >= 1 << xdec) FH(cols - sx, y - sy);
  }
  if (rows > sy)
    for (int x = 0; x < cols; x += sx) FH(x, rows - sy);
#undef FV
#undef FH
}

void orc_deblock_filter(void *const *pl, const ptrdiff_t *stride, int bpp, int planes, int xdec, int ydec,
                        int bit_depth, const uint8_t *state, const uint8_t *levels, const uint8_t *mi,
                        ptrdiff_t mi_stride, const int32_t *items, size_t n_items) {
  /* items are disjoint and each reads and writes only its own working rect: they run in parallel */
#pragma omp parallel for schedule(dynamic)
  for (size_t k = 0; k < n_items; k++) {
    const int32_t *it = items + 6 * k;
    const uint8_t *lv = levels + 4 * k;
    if (lv[0] == 0 && lv[1] == 0) continue; /* encoder.rs:3280, :3598, rdo.rs:2311 */
    const Blocks bl = {mi, mi_stride, it[0], it[1]};
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      const Px P = {pl[p], stride[p], bpp, (it[0] * 4) >> xd, (it[1] * 4) >> yd};
      deblock_plane(state, lv, &P, p, &bl, it[2], it[3], it[4], it[5], bit_depth, xd, yd);
    }
  }
}

/* ---------------------------------------------------------------- the level search */
static int64_t sse_n(const int *a, const int *b, int n) {
  int s = 0;
  for (int i = 0; i < n; i++) s += (a[i] - b[i]) * (a[i] - b[i]);
  return s;
}

/* sse_size4 / 6 / 8 / 14 (:418-472, :550-625, :731-827, :932-1097) for one line: r = rec taps, a = src taps */
static void sse_line(const int *r, const int *s, int size, int bd, int64_t *tally) {
  const int shift = bd - 8, flat = 1 << shift;
  int none[12], n2[12], n4[12], wide[12], nw;
  const int *c; /* p1 p0 q0 q1 inside r */
  int mask, flatp = 0, flat14p = 0;
  switch (size) {
    case 4: nw = 4; c = r; mask = mask4(r, shift); break;
    case 6: nw = 4; c = r + 1; mask = mask6(r, shift); flatp = flat6(r) <= flat; break;
    case 8: nw = 6; c = r + 2; mask = mask8(r, shift); flatp = flat8(r) <= flat; break;
    default: nw = 12; c = r + 5; mask = mask8(r + 3, shift); flatp = flat8(r + 3) <= flat;
      flat14p = flat14_outer(r) <= flat; break;
  }
  const int off = size == 4 ? 0 : 1; /* compared pixels start one tap in, except for size 4 */
  const int *a = s + off;
  memcpy(none, r + off, nw * sizeof(int));
  const int lead = (nw - 4) / 2; /* untouched taps before p1 in the compared window */
  memcpy(n2, none, sizeof none);
  memcpy(n4, none, sizeof none);
  narrow2_4(c[0], c[1], c[2], c[3], shift, n2 + lead);
  narrow4_4(c[0], c[1], c[2], c[3], shift, n4 + lead);
  if (size == 6) wide6_4(r, wide);
  else if (size == 8) wide8_6(r, wide);
  else if (size == 14) {
    if (flat14p) wide14_12(r, wide);
    else {
      memcpy(wide, none, sizeof none);
      wide8_6(r + 3, wide + 3);
    }
  }
  mask = clampi(mask, 1, MAX_LOOP_FILTER + 1);
  const int nhev = clampi(nhev4(c[0], c[1], c[2], c[3], shift), mask, MAX_LOOP_FILTER + 1);
  const int64_t sse_none = sse_n(a, none, nw);
  const int64_t sse_wide = flatp && mask <= MAX_LOOP_FILTER ? sse_n(a, wide, nw) : sse_none;
  const int64_t sse_n2 = !flatp && nhev != mask ? sse_n(a, n2, nw) : sse_none;
  const int64_t sse_n4 = !flatp && nhev <= MAX_LOOP_FILTER ? sse_n(a, n4, nw) : sse_none;
  tally[0] += sse_none;
  tally[mask] -= sse_none;
  if (flatp) {
    tally[mask] += sse_wide;
  } else {
    tally[mask] += sse_n2;
    tally[nhev] -= sse_n2;
    tally[nhev] += sse_n4;
  }
}

/* sse_v_edge / sse_h_edge (:1145-1193, :1241-1290) */
static void sse_edge(const Blocks *bl, const Px *R, const Px *S, int64_t *tally, int pli, int bd, int xdec, int ydec,
                     int x, int y, int vertical) {
  Mi blk, prev;
  const int size = edge_size(bl, pli, xdec, ydec, x, y, vertical, 1, &blk, &prev);
  if (!size) return;
  const int px = (x * 4) >> xdec, py = (y * 4) >> ydec;
  for (int i = 0; i < 4; i++) {
    int r[14], s[14];
    for (int k = 0; k < size; k++) {
      const int xx = vertical ? px - size / 2 + k : px + i, yy = vertical ? py + i : py - size / 2 + k;
      r[k] = get_px(R->p, R->stride, R->bpp, R->ox + xx, R->oy + yy);
      s[k] = get_px(S->p, S->stride, S->bpp, S->ox + xx, S->oy + yy);
    }
    sse_line(r, s, size, bd, tally);
  }
}

void orc_deblock_levels(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                        const ptrdiff_t *src_stride, int bpp, int planes, int xdec, int ydec, int bit_depth,
                        const uint8_t *mi, ptrdiff_t mi_stride, const int32_t *items, size_t n_items,
                        uint8_t *levels, int64_t *tally) {
#pragma omp parallel for schedule(dynamic)
  for (size_t k = 0; k < n_items; k++) {
    const int32_t *it = items + 6 * k;
    const Blocks bl = {mi, mi_stride, it[0], it[1]};
    uint8_t *lv = levels + 4 * k;
    memset(lv, 0, 4);
    if (tally) memset(tally + k * 3 * 2 * 64, 0, 3 * 2 * 64 * sizeof(int64_t));
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      const Px R = {(void *)rec[p], rec_stride[p], bpp, (it[0] * 4) >> xd, (it[1] * 4) >> yd};
      const Px S = {(void *)src[p], src_stride[p], bpp, (it[0] * 4) >> xd, (it[1] * 4) >> yd};
      int64_t v[MAX_LOOP_FILTER + 2] = {0}, h[MAX_LOOP_FILTER + 2] = {0};
      const int cols = extent(it[2], it[4], xd), rows = extent(it[3], it[5], yd);
      const int sx = 1 << xd, sy = 1 << yd;
      /* sse_plane (:1460-1540) */
      for (int x = sx; x < cols; x += sx) sse_edge(&bl, &R, &S, v, p, bit_depth, xd, yd, x, 0, 1);
      for (int y = sy; y < rows; y += sy) {
        sse_edge(&bl, &R, &S, h, p, bit_depth, xd, yd, 0, y, 0);
        for (int x = sx; x < cols; x += sx) {
          sse_edge(&bl, &R, &S, v, p, bit_depth, xd, yd, x, y, 1);
          sse_edge(&bl, &R, &S, h, p, bit_depth, xd, yd, x, y, 0);
        }
      }
      /* sse_optimize (:1582-1614): prefix sums, first strict minimum */
      for (int i = 1; i <= MAX_LOOP_FILTER; i++) {
        v[i] += v[i - 1];
        h[i] += h[i - 1];
      }
      if (p == 0) {
        int bv = 0, bh = 0;
        for (int i = 1; i <= MAX_LOOP_FILTER; i++) {
          if (v[bv] > v[i]) bv = i;
          if (h[bh] > h[i]) bh = i;
        }
        lv[0] = (uint8_t)bv;
        lv[1] = (uint8_t)bh;
      } else {
        int b = 0;
        for (int i = 1; i <= MAX_LOOP_FILTER; i++)
          if (v[b] + h[b] > v[i] + h[i]) b = i;
        lv[p + 1] = (uint8_t)b;
      }
      if (tally) {
        int64_t *t = tally + (k * 3 + p) * 2 * 64;
        memcpy(t, v, 64 * sizeof(int64_t));
        memcpy(t + 64, h, 64 * sizeof(int64_t));
      }
    }
  }
}
