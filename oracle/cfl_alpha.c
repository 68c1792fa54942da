/* cfl_alpha.c — CPU restatement of rav1e's CfL alpha search (TEST INFRASTRUCTURE ONLY, see oracle.h and
 * cfl_alpha.h).
 *
 *   rdo_cfl_alpha                          src/rdo.rs:1593-1689
 *   clip_visible_bsize                     src/rdo.rs:228-253
 *   luma_ac                                src/predict.rs:644-698
 *   PredictionMode::predict_intra          src/predict.rs:205-249
 *   BlockSize::subsampled_size, is_sub8x8, sub8x8_offset, cfl_allowed   src/partition.rs:337-379, :401-413, :228-231
 *   has_chroma                             src/context/transform_unit.rs:108-121
 *   fi.w_in_b / fi.h_in_b                  src/encoder.rs:852-853
 *
 * Composed only of the pinned or second-sourced pieces orc_pred_cfl_ac, orc_get_intra_edges,
 * orc_predict_intra (DC_PRED / UV_CFL_PRED) and orc_weighted_sse_* with a unit scale map.  The orchestration
 * has no stored vectors upstream ("parity unpinned"); tests/test_oracle_cfl_alpha.py checks it against an
 * independent Python restatement.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "cfl_alpha.h"
#include "oracle.h"

enum { DC_PRED = 0, UV_CFL_PRED = 13, NALPHA = 33, BLOCK_32X32 = 9 };
/* BlockSize 0..BLOCK_32X32 in enum order (partition.rs:130-153) */
static const uint8_t BS_W[10] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32};
static const uint8_t BS_H[10] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32};

/* rdo.rs:228-253, one direction */
static int clip_visible(int frame, int blk, int pos) {
  if (pos + blk <= frame) return blk;
  if (pos >= frame) return 0;
  return frame - pos;
}

static int item_valid(const orc_cfl_item *it, int xdec, int ydec, int rect_w, int rect_h) {
  if (it->bsize > BLOCK_32X32) return 0; /* cfl_allowed: self <= BLOCK_32X32 */
  /* subsampled_size (partition.rs:342-357): 4:2:2 has no BLOCK_4X8, BLOCK_8X16, BLOCK_16X32 */
  if (xdec && !ydec && (it->bsize == 1 || it->bsize == 4 || it->bsize == 7)) return 0;
  if (it->tx_size >= 19) return 0;
  const int bw = BS_W[it->bsize], bh = BS_H[it->bsize];
  if (orc_tx_width(it->tx_size) > bw || orc_tx_height(it->tx_size) > bh) return 0;
  if (it->x < 0 || it->y < 0 || it->x >= rect_w || it->y >= rect_h || (it->x & 3) || (it->y & 3)) return 0;
  const int bx = it->x >> 2, by = it->y >> 2;
  /* has_chroma with width_mi / height_mi */
  return ((bx & 1) || !((bw >> 2) & 1) || !xdec) && ((by & 1) || !((bh >> 2) & 1) || !ydec);
}

static void cfl_one(const void *const rec[3], const ptrdiff_t rec_stride[3], const void *const src[3],
                    const ptrdiff_t src_stride[3], int bpp, int chroma_w, int chroma_h, int xdec, int ydec, int rect_x,
                    int rect_y, int rect_w, int rect_h, int frame_width, int frame_height, int bit_depth,
                    const orc_cfl_item *it, int8_t *alpha_out, uint64_t *sse_out) {
  const int bsize = it->bsize, bw = BS_W[bsize], bh = BS_H[bsize];
  const int bx = it->x >> 2, by = it->y >> 2; /* tile_bo */
  /* rdo.rs:1598: uv_tx_size = largest_chroma_tx_size, whose block size is subsampled_size (rdo.rs:1599-1601):
     the chroma block of a cfl_allowed size is max(side >> dec, 4) on each side */
  const int tw = (bw >> xdec) > 4 ? bw >> xdec : 4, th = (bh >> ydec) > 4 ? bh >> ydec : 4;
  /* rdo.rs:1603-1610: frame_bo = tile origin + tile_bo; x = (frame_bo.x << 2) >> xdec */
  const int vis_w = clip_visible((frame_width + xdec) >> xdec, tw, (rect_x + 4 * bx) >> xdec);
  const int vis_h = clip_visible((frame_height + ydec) >> ydec, th, (rect_y + 4 * by) >> ydec);
  if (vis_w == 0 || vis_h == 0) return; /* rdo.rs:1612-1614: None, the caller keeps the sentinels */

  /* luma_ac (predict.rs:644-698) */
  const int off_x = (xdec && bw == 4) ? -1 : 0, off_y = (ydec && bh == 4) ? -1 : 0; /* sub8x8_offset */
  const int lbx = bx + off_x, lby = by + off_y;
  const int fbx = (rect_x >> 2) + lbx, fby = (rect_y >> 2) + lby; /* ts.to_frame_block_offset(bo) */
  const int w_in_b = 2 * ((frame_width + 7) >> 3), h_in_b = 2 * ((frame_height + 7) >> 3);
  const int clip_bw = ((w_in_b - fbx) << 2) < bw ? (w_in_b - fbx) << 2 : bw;
  const int clip_bh = ((h_in_b - fby) << 2) < bh ? (h_in_b - fby) << 2 : bh;
  const int txw = orc_tx_width(it->tx_size), txh = orc_tx_height(it->tx_size);
  const int max_luma_w = bw > 8 ? (clip_bw + txw - 1) / txw * txw : bw;
  const int max_luma_h = bh > 8 ? (clip_bh + txh - 1) / txh * txh : bh;
  const int w_pad = (bw - max_luma_w) >> (2 + xdec), h_pad = (bh - max_luma_h) >> (2 + ydec);
  int16_t ac[32 * 32];
  const uint8_t *luma = (const uint8_t *)rec[0] + ((ptrdiff_t)(rect_y + 4 * lby) * rec_stride[0] + rect_x + 4 * lbx) * bpp;
  orc_pred_cfl_ac(ac, luma, rec_stride[0], bpp, tw, th, w_pad, h_pad, xdec, ydec);

  uint32_t unit[8 * 8]; /* |_, _| DistortionScale::default() */
  for (int k = 0; k < 64; k++) unit[k] = 1u << 14;
  const int crx = rect_x >> xdec, cry = rect_y >> ydec; /* tile_rect().decimated(xdec, ydec) */
  const int po_x = (bx >> xdec) << 2, po_y = (by >> ydec) << 2; /* tile_bo.plane_offset */
  /* predict.rs:214-218: PredictionVariant::new of the tile-relative destination */
  const int variant = po_x == 0 && po_y == 0 ? 0 : po_y == 0 ? 1 : po_x == 0 ? 2 : 3;
  for (int p = 1; p < 3; p++) {
    /* rdo.rs:1625-1638 */
    uint16_t edge[4 * 64 + 1];
    int init_left = 0, init_above = 0;
    const uint8_t *region = (const uint8_t *)rec[p] + ((ptrdiff_t)cry * rec_stride[p] + crx) * bpp;
    orc_get_intra_edges(edge, region, rec_stride[p], bpp, chroma_w, chroma_h, crx, cry, rect_w >> xdec,
                        rect_h >> ydec, xdec, ydec, bx, by, 0, 0, bsize, po_x, po_y, tw, th, bit_depth, UV_CFL_PRED,
                        0, 0, &init_left, &init_above);
    const uint8_t *org = (const uint8_t *)src[p] + ((ptrdiff_t)(cry + po_y) * src_stride[p] + crx + po_x) * bpp;
    uint64_t *sse = sse_out ? sse_out + (size_t)(p - 1) * NALPHA : NULL;
    uint16_t pred[32 * 32];
    /* rdo.rs:1639-1663: predict_intra (alpha 0 -> DC_PRED, predict.rs:236), then sse_wxh */
#define ALPHA_COST(AL, OUT)                                                                                       \
  do {                                                                                                           \
    orc_predict_intra((AL) == 0 ? DC_PRED : UV_CFL_PRED, variant, pred, tw, bpp, tw, th, bit_depth, ac, (AL), -1, \
                      edge, init_left, init_above, chroma_w, chroma_h, crx + po_x, cry + po_y);                  \
    OUT = bpp == 1 ? orc_weighted_sse_u8(org, src_stride[p], (const uint8_t *)pred, tw, unit, 8, vis_w, vis_h)   \
                   : orc_weighted_sse_u16((const uint16_t *)org, src_stride[p], pred, tw, unit, 8, vis_w, vis_h); \
    if (sse) sse[(AL) + 16] = OUT;                                                                               \
  } while (0)
    /* rdo.rs:1664-1680 */
    uint64_t best_cost, c0, c1;
    int best = 0, count = 2;
    ALPHA_COST(0, best_cost);
    for (int al = 1; al <= 16; al++) {
      ALPHA_COST(al, c0);
      ALPHA_COST(-al, c1);
      if (c0 < best_cost) {
        best_cost = c0;
        best = al;
        count += 2;
      }
      if (c1 < best_cost) {
        best_cost = c1;
        best = -al;
        count += 2;
      }
      if (count < al) break;
    }
#undef ALPHA_COST
    if (alpha_out) alpha_out[p - 1] = (int8_t)best;
  }
}

void orc_cfl_alpha(const void *const rec[3], const ptrdiff_t rec_stride[3], const void *const src[3],
                   const ptrdiff_t src_stride[3], int bpp, int chroma_w, int chroma_h, int xdec, int ydec, int rect_x,
                   int rect_y, int rect_w, int rect_h, int frame_width, int frame_height, int bit_depth,
                   const orc_cfl_item *items, size_t n, int8_t *alpha, uint64_t *sse, int threads) {
#pragma omp parallel for schedule(dynamic, 16) num_threads(threads > 0 ? threads : orc_num_threads())
  for (size_t i = 0; i < n; i++) {
    int8_t *a = alpha ? alpha + i * 2 : NULL;
    uint64_t *s = sse ? sse + i * 2 * NALPHA : NULL;
    if (a) a[0] = a[1] = 0;
    if (s)
      for (int k = 0; k < 2 * NALPHA; k++) s[k] = UINT64_MAX;
    if (!item_valid(&items[i], xdec, ydec, rect_w, rect_h)) continue;
    cfl_one(rec, rec_stride, src, src_stride, bpp, chroma_w, chroma_h, xdec, ydec, rect_x, rect_y, rect_w, rect_h,
            frame_width, frame_height, bit_depth, &items[i], a, s);
  }
}
